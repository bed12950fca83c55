/* bm_oracle_mismatch.c -- TEST INFRASTRUCTURE ONLY: the restated contract of bmb200_sv_mismatch / bmb200_sv_first_mismatch.
 *
 * sparse_vector_find_mismatch (src/bmsparsevec_algo.h:657) and sparse_vector_find_first_mismatch (:479) restated as the two
 * closed forms of include/bmb200.h, block by block over a packed set: the planes A_j / B_j, the NOT-NULL vectors NA / NB and
 * the bit ranges [x, y) of a column, combined word by word.  Same outputs as orc_scan (bm_oracle.c) with ONE result group of
 * n_cols columns.  Built by oracle/mismatch.mk into oracle/liboracle_mismatch.so together with the rest of the oracle. */
#include <stdlib.h>
#include <string.h>

#include "bm_oracle.h"

#define BW   BMB200_BLOCK_WORDS
#define GMAX BMB200_GAP_MAX_WORDS
#define NONE 0xffffffffu

int orc_sv_mismatch(const bmb200_packed_set* s, const bmb200_mismatch_args* a,
                    uint8_t* kind, uint32_t* popcnt, uint64_t* digest, uint32_t* nruns, uint32_t* blocks, uint16_t* gaps);
int orc_sv_first_mismatch(const bmb200_packed_set* s, const bmb200_mismatch_args* a, uint64_t* pos, int* found);

static int check(const bmb200_packed_set* s, const bmb200_mismatch_args* a, uint32_t* nb_to)
{
    if (!s || !a) return BMB200_ERR_BADARG;
    if (a->null_proc > BMB200_MM_USE_NULL || (a->flags & ~(BMB200_F_COUNT_ONLY | BMB200_F_OPT_COMPRESS))) return BMB200_ERR_BADARG;
    if (a->n_planes_a > 64 || a->n_planes_b > 64) return BMB200_ERR_BADARG;
    if ((uint64_t)a->plane0_a + a->n_planes_a > s->n_vec || (uint64_t)a->plane0_b + a->n_planes_b > s->n_vec) return BMB200_ERR_BADARG;
    if ((a->not_null_a != NONE && a->not_null_a >= s->n_vec) || (a->not_null_b != NONE && a->not_null_b >= s->n_vec)) return BMB200_ERR_BADARG;
    *nb_to = a->nb_to ? a->nb_to : s->n_blocks;
    if (a->nb_from >= *nb_to || *nb_to > s->n_blocks) return BMB200_ERR_RANGE;
    return BMB200_OK;
}

/* bit i of column nb in [lo, hi)? */
static int in_range(uint32_t nb, uint32_t i, uint64_t lo, uint64_t hi)
{
    const uint64_t p = ((uint64_t)nb << 16) + i;
    return p >= lo && p < hi;
}

/* the column's D (vector form, first = 0) or F (first form, first = 1) into out[2048]; ta / tb / na / nb2 are scratch blocks */
static void column(const bmb200_packed_set* s, const bmb200_mismatch_args* a, uint32_t nb, int first, uint32_t* out,
                   uint32_t* ta, uint32_t* tb, uint32_t* na, uint32_t* nbv)
{
    const uint32_t np = a->n_planes_a > a->n_planes_b ? a->n_planes_a : a->n_planes_b;
    const int ha = a->not_null_a != NONE, hb = a->not_null_b != NONE, use = a->null_proc == BMB200_MM_USE_NULL;
    const uint64_t sa = a->size_a, sb = a->size_b, lo = sa < sb ? sa : sb, hi = sa < sb ? sb : sa;
    memset(out, 0, BMB200_BLOCK_BYTES);
    for (uint32_t j = 0; j < np; ++j) {
        if (j < a->n_planes_a) orc_expand_block(s, a->plane0_a + j, nb, ta); else memset(ta, 0, BMB200_BLOCK_BYTES);
        if (j < a->n_planes_b) orc_expand_block(s, a->plane0_b + j, nb, tb); else memset(tb, 0, BMB200_BLOCK_BYTES);
        for (uint32_t w = 0; w < BW; ++w) out[w] |= ta[w] ^ tb[w];
    }
    if (ha) orc_expand_block(s, a->not_null_a, nb, na);
    if (hb) orc_expand_block(s, a->not_null_b, nb, nbv);
    for (uint32_t i = 0; i < BMB200_BLOCK_BITS; ++i) {
        const uint32_t w = i >> 5, m = 1u << (i & 31);
        const int A = ha && (na[w] & m), B = hb && (nbv[w] & m);
        int d = (out[w] & m) != 0;
        if (!first) {
            d |= in_range(nb, i, lo, hi);
            if (use) {
                if (ha && hb) d |= A ^ B;
                else if (ha) d |= in_range(nb, i, 0, sa) && !A;
                else if (hb) d |= in_range(nb, i, 0, sb) && !B;
            } else {
                if (ha && hb) d &= A | B;
                else if (ha) d &= A;
                else if (hb) d &= B;
            }
        } else if (use) {
            if (ha && hb) d |= A ^ B;
            else if (ha) d |= A ^ in_range(nb, i, 0, sb);
            else if (hb) d |= B ^ in_range(nb, i, 0, sa);
        }
        if (d) out[w] |= m; else out[w] &= ~m;
    }
}

static int scratch(uint32_t** t, int n)
{
    for (int k = 0; k < n; ++k) {
        t[k] = (uint32_t*)malloc(BMB200_BLOCK_BYTES);
        if (!t[k]) { for (int q = 0; q < k; ++q) free(t[q]); return BMB200_ERR_BADALLOC; }
    }
    return BMB200_OK;
}

int orc_sv_mismatch(const bmb200_packed_set* s, const bmb200_mismatch_args* a,
                    uint8_t* kind, uint32_t* popcnt, uint64_t* digest, uint32_t* nruns, uint32_t* blocks, uint16_t* gaps)
{
    uint32_t nb_to = 0, *t[5];
    int rc = check(s, a, &nb_to);
    if (rc) return rc;
    uint16_t* tg = (uint16_t*)malloc(sizeof(uint16_t) * 65540);
    if (!tg || scratch(t, 5)) { free(tg); return BMB200_ERR_BADALLOC; }
    const int compress = (a->flags & BMB200_F_OPT_COMPRESS) != 0;
    for (uint32_t nb = a->nb_from; nb < nb_to; ++nb) {
        uint32_t* r = t[0];
        column(s, a, nb, 0, r, t[1], t[2], t[3], t[4]);
        size_t c = nb - a->nb_from;
        uint32_t pc = orc_bit_block_count(r), nr = orc_bit_block_calc_change(r);
        uint64_t dg = orc_block_digest(r);
        uint8_t kd;                                   /* stored like an AND-SUB result: empty digest => nothing */
        if (dg == 0) kd = BMB200_BLK_NULL;
        else if (!compress) kd = BMB200_BLK_BIT;
        else if (nr == 1) kd = BMB200_BLK_FULL;
        else if (nr < BMB200_GAP_THRESHOLD) kd = BMB200_BLK_GAP;
        else kd = BMB200_BLK_BIT;
        if (kind) kind[c] = kd;
        if (popcnt) popcnt[c] = pc;
        if (digest) digest[c] = dg;
        if (nruns) nruns[c] = nr;
        if (blocks) memcpy(blocks + c * BW, r, BMB200_BLOCK_BYTES);
        if (gaps) {
            uint16_t* gout = gaps + c * GMAX;
            memset(gout, 0, sizeof(uint16_t) * GMAX);
            if (kd == BMB200_BLK_GAP) { uint32_t len = orc_bit_to_gap(tg, r); memcpy(gout, tg, sizeof(uint16_t) * (len + 1)); }
        }
    }
    for (int k = 0; k < 5; ++k) free(t[k]);
    free(tg);
    return BMB200_OK;
}

int orc_sv_first_mismatch(const bmb200_packed_set* s, const bmb200_mismatch_args* a, uint64_t* pos, int* found)
{
    uint32_t nb_to = 0, *t[5];
    if (!pos || !found) return BMB200_ERR_BADARG;
    int rc = check(s, a, &nb_to);
    if (rc) return rc;
    if (scratch(t, 5)) return BMB200_ERR_BADALLOC;
    *pos = UINT64_MAX; *found = 0;
    for (uint32_t nb = a->nb_from; nb < nb_to && !*found; ++nb) {
        column(s, a, nb, 1, t[0], t[1], t[2], t[3], t[4]);
        for (uint32_t w = 0; w < BW; ++w)
            if (t[0][w]) { *pos = ((uint64_t)nb << 16) + 32u * w + (uint32_t)__builtin_ctz(t[0][w]); *found = 1; break; }
    }
    for (int k = 0; k < 5; ++k) free(t[k]);
    return BMB200_OK;
}
