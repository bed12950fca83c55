/* bm_oracle_in.c -- TEST INFRASTRUCTURE ONLY: the restated contract of bmb200_scan with BMB200_SCAN_IN.
 *
 * sparse_vector_scanner::find_eq(sv, start, end, bv_out) (src/bmsparsevec_algo.h:1398-1423) restated: the elements whose
 * stored code is the code of some listed value, inside the universe U.  code(i) is element i rebuilt from its planes; the code
 * of a listed value is the value itself, or s2u(v) (src/bmbmatrix.h:2536-2569) with BMB200_F_SIGNED.  A listed code with a bit
 * at or above n_planes is simply never equal to an element's code, and value 0 matches the zero elements inside U.
 * Same arguments and outputs as orc_scan (bm_oracle.c), with ONE result group of n_cols columns.  Built by oracle/in.mk into
 * oracle/liboracle_in.so together with the rest of the oracle. */
#include <stdlib.h>
#include <string.h>

#include "bm_oracle.h"

#define BW   BMB200_BLOCK_WORDS
#define GMAX BMB200_GAP_MAX_WORDS

static int cmp_u64(const void* a, const void* b)
{
    const uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
    return x < y ? -1 : x > y;
}

static int listed(const uint64_t* c, uint32_t n, uint64_t u)
{
    return n && bsearch(&u, c, n, sizeof(uint64_t), cmp_u64) != NULL;
}

int orc_scan_in(const bmb200_packed_set* s, const bmb200_scan_args* a,
                uint8_t* kind, uint32_t* popcnt, uint64_t* digest, uint32_t* nruns, uint32_t* blocks, uint16_t* gaps)
{
    if (!s || !a || !a->values || !a->n_values || !a->n_planes || a->n_planes > 64) return BMB200_ERR_BADARG;
    if (a->pred != BMB200_SCAN_IN || (a->flags & BMB200_F_FLOAT)) return BMB200_ERR_BADARG;
    if ((uint64_t)a->plane0 + a->n_planes > s->n_vec) return BMB200_ERR_RANGE;
    if (a->universe != 0xffffffffu && a->universe >= s->n_vec) return BMB200_ERR_RANGE;
    uint32_t nb_to = a->nb_to ? a->nb_to : s->n_blocks;
    if (a->nb_from >= nb_to || nb_to > s->n_blocks) return BMB200_ERR_RANGE;
    int compress = (a->flags & BMB200_F_OPT_COMPRESS) != 0, sgn = (a->flags & BMB200_F_SIGNED) != 0;
    uint32_t* planes = (uint32_t*)malloc((size_t)BMB200_BLOCK_BYTES * (a->n_planes + 1));
    uint64_t* codes = (uint64_t*)malloc(sizeof(uint64_t) * a->n_values);
    uint32_t* tb = (uint32_t*)malloc(BMB200_BLOCK_BYTES);
    uint16_t* tg = (uint16_t*)malloc(sizeof(uint16_t) * 65540);
    if (!planes || !codes || !tb || !tg) { free(planes); free(codes); free(tb); free(tg); return BMB200_ERR_BADALLOC; }
    for (uint32_t k = 0; k < a->n_values; ++k) {
        uint64_t v = a->values[k];
        codes[k] = !sgn ? v : (int64_t)v >= 0 ? v << 1 : ((~v) << 1) | 1u;
    }
    qsort(codes, a->n_values, sizeof(uint64_t), cmp_u64);
    for (uint32_t nb = a->nb_from; nb < nb_to; ++nb) {
        uint32_t* uni = planes + (size_t)a->n_planes * BW;
        for (uint32_t j = 0; j < a->n_planes; ++j) orc_expand_block(s, a->plane0 + j, nb, planes + (size_t)j * BW);
        if (a->universe == 0xffffffffu) memset(uni, 0xFF, BMB200_BLOCK_BYTES); else orc_expand_block(s, a->universe, nb, uni);
        memset(tb, 0, BMB200_BLOCK_BYTES);
        for (uint32_t i = 0; i < BMB200_BLOCK_BITS; ++i) {
            if (!((uni[i >> 5] >> (i & 31)) & 1u)) continue;
            uint64_t u = 0;
            for (uint32_t j = 0; j < a->n_planes; ++j) u |= (uint64_t)((planes[(size_t)j * BW + (i >> 5)] >> (i & 31)) & 1u) << j;
            if (listed(codes, a->n_values, u)) tb[i >> 5] |= 1u << (i & 31);
        }
        size_t c = nb - a->nb_from;
        uint32_t pc = orc_bit_block_count(tb), nr = orc_bit_block_calc_change(tb);
        uint64_t dg = orc_block_digest(tb);
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
        if (blocks) memcpy(blocks + c * BW, tb, BMB200_BLOCK_BYTES);
        if (gaps) {
            uint16_t* gout = gaps + c * GMAX;
            memset(gout, 0, sizeof(uint16_t) * GMAX);
            if (kd == BMB200_BLK_GAP) { uint32_t len = orc_bit_to_gap(tg, tb); memcpy(gout, tg, sizeof(uint16_t) * (len + 1)); }
        }
    }
    free(planes); free(codes); free(tb); free(tg);
    return BMB200_OK;
}
