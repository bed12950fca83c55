/* bm_oracle_str.c -- TEST INFRASTRUCTURE ONLY: the restated contract of bmb200_scan_str.
 *
 * sparse_vector_scanner string searches over a str_sparse_vector<char, ...> (src/bmsparsevec_algo.h:3263-3436), restated
 * from their contract: plane 8k+b holds bit b of byte k of element i (basic_bmatrix::set_octet, src/bmbmatrix.h:1571-1605),
 * so element i is rebuilt byte by byte from the planes and compared with the query as a byte string:
 *   exact:  every byte k < ceil(n_planes / 8) equals the query's (zero past its end), on the planes that exist;
 *   prefix: the same for the bytes k < strlen(query) only (the empty query: exact);
 *   a query byte with a bit at a plane >= n_planes: no element matches (get_slice_mask pre-screen, :2569-2570);
 * then AND the universe.  Same arguments checks and outputs as orc_scan (bm_oracle.c).  Built by oracle/str.mk into
 * oracle/liboracle_str.so together with the rest of the oracle. */
#include <stdlib.h>
#include <string.h>

#include "bm_oracle.h"

#define BW   BMB200_BLOCK_WORDS
#define GMAX BMB200_GAP_MAX_WORDS

int orc_scan_str(const bmb200_packed_set* s, const bmb200_scan_str_args* a,
                 uint8_t* kind, uint32_t* popcnt, uint64_t* digest, uint32_t* nruns, uint32_t* blocks, uint16_t* gaps)
{
    if (!s || !a || !a->strs || !a->stride || !a->n_values || !a->n_planes || a->n_planes > 2048) return BMB200_ERR_BADARG;
    if (a->flags & ~(BMB200_F_COUNT_ONLY | BMB200_F_OPT_COMPRESS | BMB200_F_STR_PREFIX)) return BMB200_ERR_BADARG;
    if ((uint64_t)a->plane0 + a->n_planes > s->n_vec) return BMB200_ERR_RANGE;
    if (a->universe != 0xffffffffu && a->universe >= s->n_vec) return BMB200_ERR_RANGE;
    uint32_t nb_to = a->nb_to ? a->nb_to : s->n_blocks;
    if (a->nb_from >= nb_to || nb_to > s->n_blocks) return BMB200_ERR_RANGE;
    for (uint32_t k = 0; k < a->n_values; ++k)
        if (!memchr(a->strs + (size_t)k * a->stride, 0, a->stride)) return BMB200_ERR_BADARG;
    const int compress = (a->flags & BMB200_F_OPT_COMPRESS) != 0, prefix = (a->flags & BMB200_F_STR_PREFIX) != 0;
    const uint32_t n_cols = nb_to - a->nb_from, np = a->n_planes, nbytes = (np + 7) / 8;
    /* elem: the bytes of the column's 65536 elements, rebuilt from the planes */
    uint32_t* plane = (uint32_t*)malloc(BMB200_BLOCK_BYTES);
    uint32_t* uni = (uint32_t*)malloc(BMB200_BLOCK_BYTES);
    uint8_t* elem = (uint8_t*)malloc((size_t)BMB200_BLOCK_BITS * nbytes);
    uint8_t* q = (uint8_t*)calloc(nbytes, 1);
    uint32_t* tb = (uint32_t*)malloc(BMB200_BLOCK_BYTES);
    uint16_t* tg = (uint16_t*)malloc(sizeof(uint16_t) * 65540);
    if (!plane || !uni || !elem || !q || !tb || !tg) { free(plane); free(uni); free(elem); free(q); free(tb); free(tg); return BMB200_ERR_BADALLOC; }
    for (uint32_t nb = a->nb_from; nb < nb_to; ++nb) {
        memset(elem, 0, (size_t)BMB200_BLOCK_BITS * nbytes);
        for (uint32_t j = 0; j < np; ++j) {
            orc_expand_block(s, a->plane0 + j, nb, plane);
            for (uint32_t w = 0; w < BW; ++w)
                for (uint32_t x = plane[w]; x; x &= x - 1) {
                    uint32_t i = w * 32 + (uint32_t)__builtin_ctz(x);
                    elem[(size_t)i * nbytes + (j >> 3)] |= (uint8_t)(1u << (j & 7));
                }
        }
        if (a->universe == 0xffffffffu) memset(uni, 0xFF, BMB200_BLOCK_BYTES); else orc_expand_block(s, a->universe, nb, uni);
        for (uint32_t k = 0; k < a->n_values; ++k) {
            const uint8_t* str = (const uint8_t*)a->strs + (size_t)k * a->stride;
            const uint32_t len = (uint32_t)strlen((const char*)str);
            int possible = 1;
            memset(q, 0, nbytes);
            for (uint32_t b = 0; b < len; ++b) {
                const uint32_t have = 8 * b >= np ? 0 : (np - 8 * b >= 8 ? 8 : np - 8 * b);   /* planes of byte b that exist */
                if (str[b] >> have) possible = 0;
                if (b < nbytes) q[b] = str[b];
            }
            const uint32_t cmp = (prefix && len) ? (len < nbytes ? len : nbytes) : nbytes;   /* bytes compared */
            memset(tb, 0, BMB200_BLOCK_BYTES);
            for (uint32_t i = 0; possible && i < BMB200_BLOCK_BITS; ++i)
                if (((uni[i >> 5] >> (i & 31)) & 1u) && memcmp(elem + (size_t)i * nbytes, q, cmp) == 0)
                    tb[i >> 5] |= 1u << (i & 31);
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
                if (kd == BMB200_BLK_GAP) { uint32_t glen = orc_bit_to_gap(tg, tb); memcpy(gout, tg, sizeof(uint16_t) * (glen + 1)); }
            }
        }
    }
    free(plane); free(uni); free(elem); free(q); free(tb); free(tg);
    return BMB200_OK;
}
