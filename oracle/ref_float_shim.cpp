/*
 * ref_float_shim.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * extern "C" wrapper around the UNMODIFIED reference's float sparse vector and its scanner:
 * bm::sparse_vector_float<bm::sparse_vector<unsigned>> (src/bmsparsevec_float.h; plain and nullable) searched by
 * bm::sparse_vector_scanner<> (find_gt_float & co., src/bmsparsevec_algo.h:3692-4009).  Built by oracle/float.mk into
 * oracle/_ref/libbmref_float.so with the reference's own AVX2 flags, where the reference tree exists.  Never linked into
 * the product.
 *
 * Values and search values cross as float.  pred = BMB200_SCAN_GT / GE / LT / LE / RANGE / RANGE_OPEN
 * (find_gt_float / find_ge_float / find_lt_float / find_le_float / find_range_float / find_range_float_unbounded).
 *   ref_svf_planes:    the vector's planes in the device layout [signs_, mantissas_.get_slice(0..22), exponents_.get_slice(0..7)]
 *                      (absent slices as empty vectors, trailing absent ones trimmed) and, last, the searchable universe (the
 *                      NOT-NULL vector of a nullable vector, else [0, n)) as per-column kind / blocks / GAP words,
 *                      (n_planes + 1) * n_cols columns, plane-major.
 *   ref_svf_scan:      one result per search value (RANGE / RANGE_OPEN: (from, to) pairs), value-major, as bit-block words
 *                      + count().
 *   ref_svf_time_scan: seconds (best of `repeats`) of the n_search scanner calls alone + the summed cardinality.
 */
#include <chrono>
#include <cstdint>
#include <cstring>

#include "bm.h"
#include "bmsparsevec.h"
#include "bmsparsevec_algo.h"
#include "bmsparsevec_float.h"

#include "../include/bmb200.h"

typedef bm::bvector<> bvect;
typedef bm::sparse_vector<unsigned, bvect> svect_u32;
typedef bm::sparse_vector_float<svect_u32> svf_t;

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

/* n elements; NULL where nulls[i] (nullable vector), else set(i, values[i]); positions never set hold +0.0 */
void build_svf(svf_t& svf, const float* values, const uint8_t* nulls, uint64_t n)
{
    svf.exponents_.resize((svf_t::size_type)n);
    svf.mantissas_.resize((svf_t::size_type)n);
    for (uint64_t i = 0; i < n; ++i) {
        if (nulls && nulls[i]) continue;
        svf.set((svf_t::size_type)i, values[i]);
    }
    BM_DECLARE_TEMP_BLOCK(tb)
    svf.optimize(tb);
}

/* plane j of the device layout: 0 = signs_, 1..23 = mantissa slice j - 1, 24..31 = exponent slice j - 24 (0 when absent) */
const bvect* plane(const svf_t& svf, unsigned j)
{
    if (j == 0) return &svf.signs_;
    return j <= 23 ? svf.mantissas_.get_slice(j - 1) : svf.exponents_.get_slice(j - 24);
}

/* one scanner call; false for an unknown predicate */
bool search(bm::sparse_vector_scanner<svf_t>& sc, const svf_t& svf, int pred, const float* s, uint32_t k, bvect& bv)
{
    switch (pred) {
    case BMB200_SCAN_GT: sc.find_gt_float(svf, s[k], bv); return true;
    case BMB200_SCAN_GE: sc.find_ge_float(svf, s[k], bv); return true;
    case BMB200_SCAN_LT: sc.find_lt_float(svf, s[k], bv); return true;
    case BMB200_SCAN_LE: sc.find_le_float(svf, s[k], bv); return true;
    case BMB200_SCAN_RANGE: sc.find_range_float(svf, s[2 * k], s[2 * k + 1], bv); return true;
    case BMB200_SCAN_RANGE_OPEN: sc.find_range_float_unbounded(svf, s[2 * k], s[2 * k + 1], bv); return true;
    default: return false;
    }
}

} // namespace

extern "C" {

int ref_svf_planes(const float* values, const uint8_t* nulls, uint64_t n, uint32_t n_cols, uint32_t* n_planes_out,
                   uint8_t* kind, uint32_t* blocks, uint16_t* gaps)
{
    try {
        svf_t svf(nulls ? bm::use_null : bm::no_null);
        build_svf(svf, values, nulls, n);
        unsigned np = 32;
        while (np > 1 && !plane(svf, np - 1)) --np;              /* trailing absent planes carry no bits */
        *n_planes_out = np;
        bvect empty, uni;
        for (unsigned j = 0; j <= np; ++j) {
            const bvect* bv;
            if (j < np) bv = plane(svf, j);
            else if (nulls) bv = svf.get_null_bvector();
            else { if (n) uni.set_range(0, (bvect::size_type)(n - 1)); uni.optimize(); bv = &uni; }
            size_t o = (size_t)j * n_cols;
            export_bvector(bv ? *bv : empty, n_cols, kind + o, blocks + o * BMB200_BLOCK_WORDS, gaps + o * BMB200_GAP_MAX_WORDS);
        }
        return 0;
    } catch (...) { return 1; }
}

int ref_svf_scan(const float* values, const uint8_t* nulls, uint64_t n, int pred, const float* s, uint32_t n_search,
                 uint32_t n_cols, uint64_t* counts, uint32_t* blocks)
{
    try {
        svf_t svf(nulls ? bm::use_null : bm::no_null);
        build_svf(svf, values, nulls, n);
        bm::sparse_vector_scanner<svf_t> sc;
        for (uint32_t k = 0; k < n_search; ++k) {
            bvect bv;
            if (!search(sc, svf, pred, s, k, bv)) return 2;
            counts[k] = (uint64_t)bv.count();
            export_bvector(bv, n_cols, 0, blocks + (size_t)k * n_cols * BMB200_BLOCK_WORDS, 0);
        }
        return 0;
    } catch (...) { return 1; }
}

int ref_svf_time_scan(const float* values, const uint8_t* nulls, uint64_t n, int pred, const float* s, uint32_t n_search,
                      int repeats, double* best_sec, uint64_t* total)
{
    try {
        svf_t svf(nulls ? bm::use_null : bm::no_null);
        build_svf(svf, values, nulls, n);
        bm::sparse_vector_scanner<svf_t> sc;
        double best = 1e30; uint64_t tot = 0;
        for (int r = 0; r < repeats; ++r) {
            tot = 0;
            auto t0 = std::chrono::steady_clock::now();
            for (uint32_t k = 0; k < n_search; ++k) {
                bvect bv;
                if (!search(sc, svf, pred, s, k, bv)) return 2;
                tot += (uint64_t)bv.count();
            }
            double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            if (sec < best) best = sec;
        }
        *best_sec = best; *total = tot;
        return 0;
    } catch (...) { return 1; }
}

} // extern "C"
