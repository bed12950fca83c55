/* bm_oracle_float.c -- TEST INFRASTRUCTURE ONLY: the restated contract of bmb200_scan with BMB200_F_FLOAT.
 *
 * sparse_vector_scanner's float searches over bm::sparse_vector_float<sparse_vector<unsigned>> (find_gt_float,
 * find_ge_float, find_lt_float, find_le_float, find_range_float, find_range_float_unbounded; src/bmsparsevec_algo.h:3692-4009),
 * restated from what they compute: a comparison in the IEEE sign-magnitude total order of the raw bits,
 *     key(b) = sign ? ~b : b | 0x80000000          (-0 < +0, NaNs beyond the infinities, payloads by their bits),
 * with the bounds of both ranges swapped when from > to as C++ floats (:3819, :3846: a NaN bound never swaps, +0 / -0 do
 * not swap).  NULL elements and indexes outside the universe never match.
 * Plane plane0 is the sign vector and plane plane0 + 1 + k bit k of the magnitude: element i is rebuilt as its 32 bits and
 * compared through key().  Same arguments and outputs as orc_scan (bm_oracle.c); values hold float bits, zero-extended.
 * The argument rules of bmb200_scan with the flag are restated too (BMB200_ERR_BADARG).  Built by oracle/float.mk into
 * oracle/liboracle_float.so together with the rest of the oracle. */
#include <stdlib.h>
#include <string.h>

#include "bm_oracle.h"

#define BW   BMB200_BLOCK_WORDS
#define GMAX BMB200_GAP_MAX_WORDS

static uint32_t key(uint32_t b) { return (b >> 31) ? ~b : b | 0x80000000u; }
static int is_nan(uint32_t b) { return (b & 0x7fffffffu) > 0x7f800000u; }
/* from > to as C++ floats, without a float compare (no flush-to-zero mode can change it) */
static int ieee_gt(uint32_t a, uint32_t b)
{
    if (is_nan(a) || is_nan(b) || !((a | b) & 0x7fffffffu)) return 0;
    return key(a) > key(b);
}

int orc_scan_float(const bmb200_packed_set* s, const bmb200_scan_args* a,
                   uint8_t* kind, uint32_t* popcnt, uint64_t* digest, uint32_t* nruns, uint32_t* blocks, uint16_t* gaps)
{
    if (!s || !a || !a->values || !a->n_values || !a->n_planes || a->n_planes > 32) return BMB200_ERR_BADARG;
    if (!(a->flags & BMB200_F_FLOAT) || (a->flags & BMB200_F_SIGNED)) return BMB200_ERR_BADARG;
    if (a->pred < BMB200_SCAN_GT || a->pred > BMB200_SCAN_RANGE_OPEN) return BMB200_ERR_BADARG;
    int two = a->pred == BMB200_SCAN_RANGE || a->pred == BMB200_SCAN_RANGE_OPEN;
    for (uint64_t k = 0; k < (uint64_t)a->n_values * (two ? 2 : 1); ++k)
        if (a->values[k] >> 32) return BMB200_ERR_BADARG;
    if ((uint64_t)a->plane0 + a->n_planes > s->n_vec) return BMB200_ERR_RANGE;
    if (a->universe != 0xffffffffu && a->universe >= s->n_vec) return BMB200_ERR_RANGE;
    uint32_t nb_to = a->nb_to ? a->nb_to : s->n_blocks;
    if (a->nb_from >= nb_to || nb_to > s->n_blocks) return BMB200_ERR_RANGE;
    int compress = (a->flags & BMB200_F_OPT_COMPRESS) != 0;
    uint32_t n_cols = nb_to - a->nb_from;
    uint32_t* planes = (uint32_t*)malloc((size_t)BMB200_BLOCK_BYTES * (a->n_planes + 1));
    uint32_t* elem = (uint32_t*)malloc(sizeof(uint32_t) * BMB200_BLOCK_BITS);
    uint32_t* tb = (uint32_t*)malloc(BMB200_BLOCK_BYTES);
    uint16_t* tg = (uint16_t*)malloc(sizeof(uint16_t) * 65540);
    if (!planes || !elem || !tb || !tg) { free(planes); free(elem); free(tb); free(tg); return BMB200_ERR_BADALLOC; }
    for (uint32_t nb = a->nb_from; nb < nb_to; ++nb) {
        uint32_t* uni = planes + (size_t)a->n_planes * BW;
        for (uint32_t j = 0; j < a->n_planes; ++j) orc_expand_block(s, a->plane0 + j, nb, planes + (size_t)j * BW);
        if (a->universe == 0xffffffffu) memset(uni, 0xFF, BMB200_BLOCK_BYTES); else orc_expand_block(s, a->universe, nb, uni);
        for (uint32_t i = 0; i < BMB200_BLOCK_BITS; ++i) {       /* the element's bits: sign from plane 0, magnitude bit k from plane 1 + k */
            uint32_t b = ((planes[i >> 5] >> (i & 31)) & 1u) << 31;
            for (uint32_t j = 1; j < a->n_planes; ++j) b |= ((planes[(size_t)j * BW + (i >> 5)] >> (i & 31)) & 1u) << (j - 1);
            elem[i] = key(b);
        }
        for (uint32_t k = 0; k < a->n_values; ++k) {
            uint32_t va = (uint32_t)a->values[two ? 2 * k : k], vb = two ? (uint32_t)a->values[2 * k + 1] : 0;
            if (two && ieee_gt(va, vb)) { uint32_t t = va; va = vb; vb = t; }
            uint32_t ka = key(va), kb = key(vb);
            memset(tb, 0, BMB200_BLOCK_BYTES);
            for (uint32_t i = 0; i < BMB200_BLOCK_BITS; ++i) {
                if (!((uni[i >> 5] >> (i & 31)) & 1u)) continue;
                uint32_t x = elem[i]; int hit;
                switch (a->pred) {
                case BMB200_SCAN_GT:    hit = x >  ka; break;
                case BMB200_SCAN_GE:    hit = x >= ka; break;
                case BMB200_SCAN_LT:    hit = x <  ka; break;
                case BMB200_SCAN_LE:    hit = x <= ka; break;
                case BMB200_SCAN_RANGE: hit = x >= ka && x <= kb; break;
                default:                hit = x >  ka && x <  kb; break;
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
