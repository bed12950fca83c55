/*
 * ref_signed_shim.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * extern "C" wrapper around the UNMODIFIED reference's signed sparse vectors and their scanner:
 * bm::sparse_vector<int32_t / int64_t> (plain and nullable) and bm::rsc_sparse_vector<int32_t / int64_t>
 * (src/bmsparsevec.h, src/bmsparsevec_compr.h, src/bmbmatrix.h:2536-2569 for the s2u plane encoding) searched by
 * bm::sparse_vector_scanner<> (src/bmsparsevec_algo.h, find_gt_horizontal_s :3032-3219).  Built by oracle/signed.mk into
 * oracle/_ref/libbmref_signed.so with the reference's own AVX2 flags, where the reference tree exists.  Never linked into
 * the product.
 *
 * is64 == 0 selects the int32_t vector, otherwise int64_t; values and search values cross as int64_t (narrowed for int32_t).
 * pred = BMB200_SCAN_*, plus REF_SCAN_ZERO = find_zero and REF_SCAN_NONZERO = find_nonzero (search values unused).
 *   ref_svs_planes:    the vector's own s2u planes (get_slice(j), j < effective_slices(), plane 0 = sign) and, last, the
 *                      searchable universe (NOT-NULL plane of a nullable vector, else [0, n)) as per-column kind / blocks / GAP
 *                      words, (n_planes + 1) * n_cols columns, plane-major.
 *   ref_svs_scan:      one result per search value (RANGE: (lo, hi) pairs), value-major, as bit-block words + count().
 *   ref_svs_time_scan: seconds (best of `repeats`) of the n_search scanner calls alone + the summed cardinality.
 *   ref_rscs_planes:   the nullable vector rank-compressed (load_from + sync): its compressed planes and NN as dense words,
 *                      plane-major with NN last; *eff = effective_size().
 *   ref_rscs_scan:     sparse_vector_scanner<rsc_sparse_vector<>> on that vector; dense words of n_cols columns + count().
 */
#include <chrono>
#include <cstdint>
#include <cstring>

#include "bm.h"
#include "bmsparsevec.h"
#include "bmsparsevec_compr.h"
#include "bmsparsevec_algo.h"

#include "../include/bmb200.h"

#define REF_SCAN_ZERO    6
#define REF_SCAN_NONZERO 7

typedef bm::bvector<> bvect;
typedef bm::sparse_vector<int32_t, bvect> svect_i32;
typedef bm::sparse_vector<int64_t, bvect> svect_i64;
typedef bm::rsc_sparse_vector<int32_t, svect_i32> rsc_i32;
typedef bm::rsc_sparse_vector<int64_t, svect_i64> rsc_i64;

namespace {

/* a bvector's block tree -> per-column kind / bit-block words / GAP words (GAP words: only for GAP columns) */
void export_bvector(const bvect& bv, uint32_t n_cols, uint8_t* kind, uint32_t* blocks, uint16_t* gaps)
{
    const bvect::blocks_manager_type& bman = bv.get_blocks_manager();
    BM_DECLARE_TEMP_BLOCK(tb)
    for (uint32_t c = 0; c < n_cols; ++c) {
        unsigned i = c >> 8, j = c & 255u;
        const bm::word_t* blk = 0;
        if (bman.is_init() && i < bman.top_block_size()) blk = bman.get_block_ptr(i, j);
        uint8_t kd;
        uint32_t* bout = blocks ? blocks + (size_t)c * BMB200_BLOCK_WORDS : 0;
        uint16_t* gout = gaps ? gaps + (size_t)c * BMB200_GAP_MAX_WORDS : 0;
        if (gout) std::memset(gout, 0, sizeof(uint16_t) * BMB200_GAP_MAX_WORDS);
        if (!blk) { kd = BMB200_BLK_NULL; if (bout) std::memset(bout, 0, BMB200_BLOCK_BYTES); }
        else if (blk == FULL_BLOCK_FAKE_ADDR || blk == FULL_BLOCK_REAL_ADDR) { kd = BMB200_BLK_FULL; if (bout) std::memset(bout, 0xFF, BMB200_BLOCK_BYTES); }
        else if (BM_IS_GAP(blk)) {
            const bm::gap_word_t* g = BMGAP_PTR(blk);
            kd = BMB200_BLK_GAP;
            if (bout) { bm::gap_convert_to_bitset(tb.begin(), g); std::memcpy(bout, tb.begin(), BMB200_BLOCK_BYTES); }
            if (gout) std::memcpy(gout, g, sizeof(uint16_t) * bm::gap_length(g));
        } else { kd = BMB200_BLK_BIT; if (bout) std::memcpy(bout, blk, BMB200_BLOCK_BYTES); }
        if (kind) kind[c] = kd;
    }
}

/* dense little-endian u32 words of n_cols columns */
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

template<class SV>
void build_sv(SV& sv, const int64_t* values, const uint8_t* nulls, uint64_t n)
{
    sv.resize((typename SV::size_type)n);
    for (uint64_t i = 0; i < n; ++i) {
        if (nulls && nulls[i]) continue;             /* stays NULL */
        sv.set((typename SV::size_type)i, (typename SV::value_type)values[i]);
    }
    BM_DECLARE_TEMP_BLOCK(tb)
    sv.optimize(tb);
}

template<class RSC>
void build_rsc(RSC& rsc, const int64_t* values, const uint8_t* nulls, uint64_t n)
{
    typename RSC::sparse_vector_type sv(bm::use_null);
    build_sv(sv, values, nulls, n);
    rsc.load_from(sv);
    rsc.sync();
}

/* one scanner call; false for an unknown predicate */
template<class SV>
bool search(bm::sparse_vector_scanner<SV>& sc, const SV& sv, int pred, const int64_t* s, uint32_t k, bvect& bv)
{
    typedef typename SV::value_type V;
    switch (pred) {
    case BMB200_SCAN_EQ: sc.find_eq(sv, (V)s[k], bv); return true;
    case BMB200_SCAN_GT: sc.find_gt(sv, (V)s[k], bv); return true;
    case BMB200_SCAN_GE: sc.find_ge(sv, (V)s[k], bv); return true;
    case BMB200_SCAN_LT: sc.find_lt(sv, (V)s[k], bv); return true;
    case BMB200_SCAN_LE: sc.find_le(sv, (V)s[k], bv); return true;
    case BMB200_SCAN_RANGE: sc.find_range(sv, (V)s[2 * k], (V)s[2 * k + 1], bv); return true;
    case REF_SCAN_ZERO: sc.find_zero(sv, bv); return true;
    case REF_SCAN_NONZERO: sc.find_nonzero(sv, bv); return true;
    default: return false;
    }
}

template<class SV>
int svs_planes(const int64_t* values, const uint8_t* nulls, uint64_t n, uint32_t n_cols, uint32_t max_planes,
               uint32_t* n_planes_out, uint8_t* kind, uint32_t* blocks, uint16_t* gaps)
{
    SV sv(nulls ? bm::use_null : bm::no_null);
    build_sv(sv, values, nulls, n);
    unsigned np = sv.effective_slices();
    while (np > 1 && !sv.get_slice(np - 1)) --np;           /* trailing absent planes carry no bits */
    if (np > max_planes) return 3;
    *n_planes_out = np;
    bvect empty;
    for (unsigned j = 0; j <= np; ++j) {
        const bvect* bv;
        bvect uni;
        if (j < np) bv = sv.get_slice(j);
        else if (nulls) bv = sv.get_null_bvector();
        else { if (n) uni.set_range(0, (bvect::size_type)(n - 1)); uni.optimize(); bv = &uni; }
        size_t o = (size_t)j * n_cols;
        export_bvector(bv ? *bv : empty, n_cols, kind + o, blocks + o * BMB200_BLOCK_WORDS, gaps + o * BMB200_GAP_MAX_WORDS);
    }
    return 0;
}

template<class SV>
int svs_scan(const int64_t* values, const uint8_t* nulls, uint64_t n, int pred, const int64_t* s, uint32_t n_search,
             uint32_t n_cols, uint64_t* counts, uint32_t* blocks)
{
    SV sv(nulls ? bm::use_null : bm::no_null);
    build_sv(sv, values, nulls, n);
    bm::sparse_vector_scanner<SV> sc;
    for (uint32_t k = 0; k < n_search; ++k) {
        bvect bv;
        if (!search(sc, sv, pred, s, k, bv)) return 2;
        counts[k] = (uint64_t)bv.count();
        export_bvector(bv, n_cols, 0, blocks + (size_t)k * n_cols * BMB200_BLOCK_WORDS, 0);
    }
    return 0;
}

template<class SV>
int svs_time_scan(const int64_t* values, const uint8_t* nulls, uint64_t n, int pred, const int64_t* s, uint32_t n_search,
                  int repeats, double* best_sec, uint64_t* total)
{
    SV sv(nulls ? bm::use_null : bm::no_null);
    build_sv(sv, values, nulls, n);
    bm::sparse_vector_scanner<SV> sc;
    double best = 1e30; uint64_t tot = 0;
    for (int r = 0; r < repeats; ++r) {
        tot = 0;
        auto t0 = std::chrono::steady_clock::now();
        for (uint32_t k = 0; k < n_search; ++k) {
            bvect bv;
            if (!search(sc, sv, pred, s, k, bv)) return 2;
            tot += (uint64_t)bv.count();
        }
        double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        if (sec < best) best = sec;
    }
    *best_sec = best; *total = tot;
    return 0;
}

template<class RSC>
int rscs_planes(const int64_t* values, const uint8_t* nulls, uint64_t n, uint32_t n_cols, uint32_t max_planes,
                uint32_t* n_planes_out, uint64_t* eff_out, uint32_t* words)
{
    RSC rsc;
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
}

template<class RSC>
int rscs_scan(const int64_t* values, const uint8_t* nulls, uint64_t n, int pred, const int64_t* s, uint32_t n_search,
              uint32_t n_cols, uint64_t* counts, uint32_t* words)
{
    RSC rsc;
    build_rsc(rsc, values, nulls, n);
    bm::sparse_vector_scanner<RSC> sc;
    for (uint32_t k = 0; k < n_search; ++k) {
        bvect bv;
        if (!search(sc, rsc, pred, s, k, bv)) return 2;
        counts[k] = (uint64_t)bv.count();
        to_words(bv, words + (size_t)k * n_cols * BMB200_BLOCK_WORDS, n_cols);
    }
    return 0;
}

} // namespace

extern "C" {

int ref_svs_planes(int is64, const int64_t* values, const uint8_t* nulls, uint64_t n, uint32_t n_cols, uint32_t max_planes,
                   uint32_t* n_planes_out, uint8_t* kind, uint32_t* blocks, uint16_t* gaps)
{
    try {
        return is64 ? svs_planes<svect_i64>(values, nulls, n, n_cols, max_planes, n_planes_out, kind, blocks, gaps)
                    : svs_planes<svect_i32>(values, nulls, n, n_cols, max_planes, n_planes_out, kind, blocks, gaps);
    } catch (...) { return 1; }
}

int ref_svs_scan(int is64, const int64_t* values, const uint8_t* nulls, uint64_t n, int pred, const int64_t* search,
                 uint32_t n_search, uint32_t n_cols, uint64_t* counts, uint32_t* blocks)
{
    try {
        return is64 ? svs_scan<svect_i64>(values, nulls, n, pred, search, n_search, n_cols, counts, blocks)
                    : svs_scan<svect_i32>(values, nulls, n, pred, search, n_search, n_cols, counts, blocks);
    } catch (...) { return 1; }
}

int ref_svs_time_scan(int is64, const int64_t* values, const uint8_t* nulls, uint64_t n, int pred, const int64_t* search,
                      uint32_t n_search, int repeats, double* best_sec, uint64_t* total)
{
    try {
        return is64 ? svs_time_scan<svect_i64>(values, nulls, n, pred, search, n_search, repeats, best_sec, total)
                    : svs_time_scan<svect_i32>(values, nulls, n, pred, search, n_search, repeats, best_sec, total);
    } catch (...) { return 1; }
}

int ref_rscs_planes(int is64, const int64_t* values, const uint8_t* nulls, uint64_t n, uint32_t n_cols, uint32_t max_planes,
                    uint32_t* n_planes_out, uint64_t* eff_out, uint32_t* words)
{
    try {
        return is64 ? rscs_planes<rsc_i64>(values, nulls, n, n_cols, max_planes, n_planes_out, eff_out, words)
                    : rscs_planes<rsc_i32>(values, nulls, n, n_cols, max_planes, n_planes_out, eff_out, words);
    } catch (...) { return 1; }
}

int ref_rscs_scan(int is64, const int64_t* values, const uint8_t* nulls, uint64_t n, int pred, const int64_t* search,
                  uint32_t n_search, uint32_t n_cols, uint64_t* counts, uint32_t* words)
{
    try {
        return is64 ? rscs_scan<rsc_i64>(values, nulls, n, pred, search, n_search, n_cols, counts, words)
                    : rscs_scan<rsc_i32>(values, nulls, n, pred, search, n_search, n_cols, counts, words);
    } catch (...) { return 1; }
}

} // extern "C"
