/* bm_oracle_signed.c -- TEST INFRASTRUCTURE ONLY: the restated contract of bmb200_scan with BMB200_F_SIGNED.
 *
 * sparse_vector_scanner searches over a signed sparse vector (bm::sparse_vector<int32_t / int64_t>), restated from their
 * contract (src/bmsparsevec_algo.h:1083-1176: "search result is a vector of 1s when sv[i] == / > / >= / < / <= value",
 * find_range: closed interval [from, to], reversed bounds swapped, :2871; NULL elements and indexes >= size() never match).
 * The planes hold u = s2u(x) (src/bmbmatrix.h:2536-2569: x >= 0 -> x << 1, x < 0 -> (-(x+1)) << 1 | 1, plane 0 = sign):
 * element i is rebuilt from its planes as u2s(u) and compared with the int64_t search values as a signed integer.
 * Same arguments and outputs as orc_scan (bm_oracle.c); the values are int64_t in the uint64_t slots.  Built by
 * oracle/signed.mk into oracle/liboracle_signed.so together with the rest of the oracle. */
#include <stdlib.h>
#include <string.h>

#include "bm_oracle.h"

#define BW   BMB200_BLOCK_WORDS
#define GMAX BMB200_GAP_MAX_WORDS

static int64_t u2s(uint64_t u) { return (u & 1u) ? -(int64_t)(u >> 1) - 1 : (int64_t)(u >> 1); }

int orc_scan_signed(const bmb200_packed_set* s, const bmb200_scan_args* a,
                    uint8_t* kind, uint32_t* popcnt, uint64_t* digest, uint32_t* nruns, uint32_t* blocks, uint16_t* gaps)
{
    if (!s || !a || !a->values || !a->n_values || !a->n_planes || a->n_planes > 64) return BMB200_ERR_BADARG;
    if (a->pred < BMB200_SCAN_EQ || a->pred > BMB200_SCAN_RANGE) return BMB200_ERR_BADARG;
    if ((uint64_t)a->plane0 + a->n_planes > s->n_vec) return BMB200_ERR_RANGE;
    if (a->universe != 0xffffffffu && a->universe >= s->n_vec) return BMB200_ERR_RANGE;
    uint32_t nb_to = a->nb_to ? a->nb_to : s->n_blocks;
    if (a->nb_from >= nb_to || nb_to > s->n_blocks) return BMB200_ERR_RANGE;
    int compress = (a->flags & BMB200_F_OPT_COMPRESS) != 0;
    uint32_t n_cols = nb_to - a->nb_from;
    uint32_t* planes = (uint32_t*)malloc((size_t)BMB200_BLOCK_BYTES * (a->n_planes + 1));
    int64_t* elem = (int64_t*)malloc(sizeof(int64_t) * BMB200_BLOCK_BITS);
    uint32_t* tb = (uint32_t*)malloc(BMB200_BLOCK_BYTES);
    uint16_t* tg = (uint16_t*)malloc(sizeof(uint16_t) * 65540);
    if (!planes || !elem || !tb || !tg) { free(planes); free(elem); free(tb); free(tg); return BMB200_ERR_BADALLOC; }
    for (uint32_t nb = a->nb_from; nb < nb_to; ++nb) {
        uint32_t* uni = planes + (size_t)a->n_planes * BW;
        for (uint32_t j = 0; j < a->n_planes; ++j) orc_expand_block(s, a->plane0 + j, nb, planes + (size_t)j * BW);
        if (a->universe == 0xffffffffu) memset(uni, 0xFF, BMB200_BLOCK_BYTES); else orc_expand_block(s, a->universe, nb, uni);
        for (uint32_t i = 0; i < BMB200_BLOCK_BITS; ++i) {
            uint64_t u = 0;
            for (uint32_t j = 0; j < a->n_planes; ++j) u |= (uint64_t)((planes[(size_t)j * BW + (i >> 5)] >> (i & 31)) & 1u) << j;
            elem[i] = u2s(u);
        }
        for (uint32_t k = 0; k < a->n_values; ++k) {
            int64_t va = (int64_t)a->values[a->pred == BMB200_SCAN_RANGE ? 2 * k : k];
            int64_t vb = a->pred == BMB200_SCAN_RANGE ? (int64_t)a->values[2 * k + 1] : 0;
            if (a->pred == BMB200_SCAN_RANGE && vb < va) { int64_t t = va; va = vb; vb = t; }   /* signed order, :2871-2872 */
            memset(tb, 0, BMB200_BLOCK_BYTES);
            for (uint32_t i = 0; i < BMB200_BLOCK_BITS; ++i) {
                if (!((uni[i >> 5] >> (i & 31)) & 1u)) continue;
                int64_t x = elem[i]; int hit;
                switch (a->pred) {
                case BMB200_SCAN_EQ: hit = x == va; break;
                case BMB200_SCAN_GT: hit = x >  va; break;
                case BMB200_SCAN_GE: hit = x >= va; break;
                case BMB200_SCAN_LT: hit = x <  va; break;
                case BMB200_SCAN_LE: hit = x <= va; break;
                default:             hit = x >= va && x <= vb; break;
                }
                if (hit) tb[i >> 5] |= 1u << (i & 31);
            }
            size_t c = (size_t)k * n_cols + (nb - a->nb_from);
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
    }
    free(planes); free(elem); free(tb); free(tg);
    return BMB200_OK;
}
