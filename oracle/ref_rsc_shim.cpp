/*
 * ref_rsc_shim.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * extern "C" wrapper around the UNMODIFIED reference's rank-select compressed sparse vector and rank compressor
 * (bm::rsc_sparse_vector<unsigned>, src/bmsparsevec_compr.h; bm::sparse_vector_scanner<>, src/bmsparsevec_algo.h;
 * bm::rank_compressor<>, src/bmalgo.h:451-644).  Built by oracle/rsc.mk into oracle/_ref/libbmref_rsc.so with the
 * reference's own AVX2 flags, where the reference tree exists.  Never linked into the product.
 *
 * Bit vectors cross the wrapper as dense little-endian u32 words (bit p = word p / 32, bit p % 32).
 *   ref_rsc_planes: a nullable sparse_vector (values[n], nulls[n] != 0 => NULL) rank-compressed by load_from + sync(); its
 *                   compressed planes (get_slice(j), j < n_planes) and NN (get_null_bvector()) as dense words, n_cols columns
 *                   each, plane-major with NN last; *eff = effective_size().
 *   ref_rsc_scan:   sparse_vector_scanner<rsc_sparse_vector<unsigned>> on that vector, pred = BMB200_SCAN_*; one result per
 *                   search value (RANGE: (lo, hi) pairs), value-major, dense words of n_cols columns + count().
 *   ref_rank_compress / ref_rank_decompress: rank_compressor<bvector<>>::compress / decompress (target, idx, src) on dense
 *                   inputs of n_in_cols columns; the target as n_out_cols columns of dense words + count().
 */
#include <cstdint>
#include <cstring>
#include <vector>

#include "bm.h"
#include "bmalgo.h"
#include "bmsparsevec.h"
#include "bmsparsevec_compr.h"
#include "bmsparsevec_algo.h"

#include "../include/bmb200.h"

typedef bm::bvector<> bvect;
typedef bm::sparse_vector<unsigned, bvect> svect;
typedef bm::rsc_sparse_vector<unsigned, svect> rsc_vect;

namespace {

void from_words(bvect& bv, const uint32_t* w, uint32_t n_cols)
{
    bv.clear(true);
    std::vector<bvect::size_type> ids;
    for (uint64_t i = 0; i < (uint64_t)n_cols * BMB200_BLOCK_WORDS; ++i)
        for (uint32_t x = w[i]; x; x &= x - 1u) ids.push_back((bvect::size_type)(i * 32u + (uint32_t)__builtin_ctz(x)));
    if (!ids.empty()) bv.set(ids.data(), (bvect::size_type)ids.size(), bm::BM_SORTED);
}

void to_words(const bvect& bv, uint32_t* w, uint32_t n_cols)
{
    const uint64_t nbits = (uint64_t)n_cols * BMB200_BLOCK_BITS;
    std::memset(w, 0, (size_t)n_cols * BMB200_BLOCK_BYTES);
    for (bvect::enumerator en = bv.first(); en.valid(); ++en) {
        const uint64_t p = *en;
        if (p >= nbits) break;
        w[p >> 5] |= 1u << (p & 31u);
    }
}

void build_rsc(rsc_vect& rsc, const uint32_t* values, const uint8_t* nulls, uint64_t n)
{
    svect sv(bm::use_null);
    sv.resize((svect::size_type)n);
    for (uint64_t i = 0; i < n; ++i)
        if (!nulls[i]) sv.set((svect::size_type)i, values[i]);
    BM_DECLARE_TEMP_BLOCK(tb)
    sv.optimize(tb);
    rsc.load_from(sv);
    rsc.sync();
}

} // namespace

extern "C" {

int ref_rsc_planes(const uint32_t* values, const uint8_t* nulls, uint64_t n, uint32_t n_cols, uint32_t max_planes,
                   uint32_t* n_planes_out, uint64_t* eff_out, uint32_t* words)
{
    try {
        rsc_vect rsc;
        build_rsc(rsc, values, nulls, n);
        unsigned np = rsc.effective_slices();
        while (np > 1 && !rsc.get_slice(np - 1)) --np;
        if (np > max_planes) return 3;
        *n_planes_out = np;
        *eff_out = (uint64_t)rsc.effective_size();
        bvect empty;
        for (unsigned j = 0; j <= np; ++j) {
            const bvect* bv = j < np ? rsc.get_slice(j) : rsc.get_null_bvector();
            to_words(bv ? *bv : empty, words + (size_t)j * n_cols * BMB200_BLOCK_WORDS, n_cols);
        }
        return 0;
    } catch (...) { return 1; }
}

int ref_rsc_scan(const uint32_t* values, const uint8_t* nulls, uint64_t n, int pred, const uint32_t* search, uint32_t n_search,
                 uint32_t n_cols, uint64_t* counts, uint32_t* words)
{
    try {
        rsc_vect rsc;
        build_rsc(rsc, values, nulls, n);
        bm::sparse_vector_scanner<rsc_vect> scanner;
        for (uint32_t k = 0; k < n_search; ++k) {
            bvect bv;
            switch (pred) {
            case BMB200_SCAN_EQ: scanner.find_eq(rsc, search[k], bv); break;
            case BMB200_SCAN_GT: scanner.find_gt(rsc, search[k], bv); break;
            case BMB200_SCAN_GE: scanner.find_ge(rsc, search[k], bv); break;
            case BMB200_SCAN_LT: scanner.find_lt(rsc, search[k], bv); break;
            case BMB200_SCAN_LE: scanner.find_le(rsc, search[k], bv); break;
            case BMB200_SCAN_RANGE: scanner.find_range(rsc, search[2 * k], search[2 * k + 1], bv); break;
            default: return 2;
            }
            counts[k] = (uint64_t)bv.count();
            to_words(bv, words + (size_t)k * n_cols * BMB200_BLOCK_WORDS, n_cols);
        }
        return 0;
    } catch (...) { return 1; }
}

int ref_rank_compress(const uint32_t* idx, const uint32_t* src, uint32_t n_in_cols, uint32_t n_out_cols, uint32_t* out, uint64_t* count)
{
    try {
        bvect bi, bs, bt;
        from_words(bi, idx, n_in_cols); from_words(bs, src, n_in_cols);
        bm::rank_compressor<bvect> rc;
        rc.compress(bt, bi, bs);
        *count = (uint64_t)bt.count();
        to_words(bt, out, n_out_cols);
        return 0;
    } catch (...) { return 1; }
}

int ref_rank_decompress(const uint32_t* idx, const uint32_t* src, uint32_t n_in_cols, uint32_t n_out_cols, uint32_t* out, uint64_t* count)
{
    try {
        bvect bi, bs, bt;
        from_words(bi, idx, n_in_cols); from_words(bs, src, n_in_cols);
        bm::rank_compressor<bvect> rc;
        rc.decompress(bt, bi, bs);
        *count = (uint64_t)bt.count();
        to_words(bt, out, n_out_cols);
        return 0;
    } catch (...) { return 1; }
}

} // extern "C"
