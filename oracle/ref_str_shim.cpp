/*
 * ref_str_shim.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * extern "C" wrapper around the UNMODIFIED reference's string sparse vector and its scanner:
 * bm::str_sparse_vector<char, bvector<>, 32> (src/bmstrsparsevec.h), plain or nullable, optionally remap()ed, searched by
 * bm::sparse_vector_scanner<> (src/bmsparsevec_algo.h: find_eq_str / find_eq_str_prefix :3263-3419, pipeline :4579-4651).
 * Built by oracle/str.mk into oracle/_ref/libbmref_str.so with the reference's own AVX2 flags, where the reference tree
 * exists.  Never linked into the product.
 *
 * Strings cross as n slots of `stride` bytes (C strings); nulls[i] != 0 leaves element i NULL (nulls may be 0: no NULLs).
 *   ref_str_planes: the vector's planes (get_slice(j), j < rows_not_null() with trailing absent planes trimmed) and, last,
 *                   the searchable universe (NOT-NULL vector of a nullable vector, else [0, n)) as per-column kind / blocks /
 *                   GAP words, (n_planes + 1) * n_cols columns, plane-major; *max_str = effective_max_str().
 *   ref_str_remap:  remap_tosv(buf, effective_max_str(), q) of every query into a zeroed slot of qstride bytes; ok[k] = its
 *                   return value.  The caller passes only queries the reference defines an answer for (see DESIGN.md).
 *   ref_str_find:   mode 0 find_eq_str, 1 find_eq_str_prefix, 2 find_eq_str(str, pos) (found[k], pos[k]), 3 pipeline
 *                   results (agg_opt_bvect_and_counts), 4 pipeline counts (agg_opt_only_counts).  counts[k] and, for modes
 *                   0, 1, 3, the result bit-block words of n_cols columns per query; found[k] = the call's return value
 *                   (modes 0-2).
 *   ref_str_time:   seconds (best of `repeats`) of the nq scanner calls of `mode` (0, 1 or 4) alone + the summed cardinality.
 */
#include <chrono>
#include <cstdint>
#include <cstring>
#include <vector>

#include "bm.h"
#include "bmstrsparsevec.h"
#include "bmsparsevec_algo.h"

#include "../include/bmb200.h"

typedef bm::bvector<> bvect;
typedef bm::str_sparse_vector<char, bvect, 32> str_svect;
typedef bm::sparse_vector_scanner<str_svect> str_scanner;

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

void build(str_svect& sv, const char* strs, uint32_t stride, uint64_t n, const uint8_t* nulls, int remap)
{
    for (uint64_t i = 0; i < n; ++i) {
        if (nulls && nulls[i]) sv.push_back_null();
        else sv.push_back(strs + i * stride);
    }
    if (remap) sv.remap();
    BM_DECLARE_TEMP_BLOCK(tb)
    sv.optimize(tb);
}

template<class Opt>
void run_pipeline(const str_svect& sv, const char* q, uint32_t qstride, uint32_t nq, uint32_t n_cols, uint64_t* counts, uint32_t* blocks)
{
    str_scanner sc;
    typename str_scanner::template pipeline<Opt> pipe(sv);
    for (uint32_t k = 0; k < nq; ++k) pipe.add(q + (size_t)k * qstride);
    pipe.complete();
    sc.find_eq_str(pipe);
    auto& cnt = pipe.get_bv_count_vector();
    for (uint32_t k = 0; k < nq; ++k) {
        counts[k] = (uint64_t)cnt[k];
        if (blocks) {
            const bvect* bv = pipe.get_bv_res_vector()[k];
            bvect empty;
            export_bvector(bv ? *bv : empty, n_cols, 0, blocks + (size_t)k * n_cols * BMB200_BLOCK_WORDS, 0);
        }
    }
}

} // namespace

extern "C" {

int ref_str_planes(const char* strs, uint32_t stride, uint64_t n, const uint8_t* nulls, int remap, uint32_t n_cols,
                   uint32_t max_planes, uint32_t* n_planes_out, uint32_t* max_str, uint8_t* kind, uint32_t* blocks, uint16_t* gaps)
{
    try {
        str_svect sv(nulls ? bm::use_null : bm::no_null);
        build(sv, strs, stride, n, nulls, remap);
        unsigned np = (unsigned)sv.get_bmatrix().rows_not_null();
        while (np > 1 && !sv.get_slice(np - 1)) --np;       /* trailing absent planes carry no bits */
        if (!np) np = 1;
        if (np > max_planes) return 3;
        *n_planes_out = np;
        *max_str = (uint32_t)sv.effective_max_str();
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
    } catch (...) { return 1; }
}

int ref_str_remap(const char* strs, uint32_t stride, uint64_t n, const uint8_t* nulls, const char* q, uint32_t qstride, uint32_t nq,
                  char* out, uint8_t* ok)
{
    try {
        str_svect sv(nulls ? bm::use_null : bm::no_null);
        build(sv, strs, stride, n, nulls, 1);
        const size_t ms = sv.effective_max_str();
        std::vector<char> buf(ms + 1 > qstride ? ms + 1 : qstride);
        for (uint32_t k = 0; k < nq; ++k) {
            std::fill(buf.begin(), buf.end(), 0);
            ok[k] = sv.remap_tosv(buf.data(), ms, q + (size_t)k * qstride) ? 1 : 0;
            std::memcpy(out + (size_t)k * qstride, buf.data(), qstride);
        }
        return 0;
    } catch (...) { return 1; }
}

int ref_str_find(const char* strs, uint32_t stride, uint64_t n, const uint8_t* nulls, int remap, int mode, const char* q,
                 uint32_t qstride, uint32_t nq, uint32_t n_cols, uint8_t* found, uint64_t* pos, uint64_t* counts, uint32_t* blocks)
{
    try {
        str_svect sv(nulls ? bm::use_null : bm::no_null);
        build(sv, strs, stride, n, nulls, remap);
        if (mode == 3) { run_pipeline<bm::agg_opt_bvect_and_counts>(sv, q, qstride, nq, n_cols, counts, blocks); return 0; }
        if (mode == 4) { run_pipeline<bm::agg_opt_only_counts>(sv, q, qstride, nq, n_cols, counts, 0); return 0; }
        str_scanner sc;
        for (uint32_t k = 0; k < nq; ++k) {
            const char* s = q + (size_t)k * qstride;
            if (mode == 2) {
                str_svect::size_type p = 0;
                found[k] = sc.find_eq_str(sv, s, p) ? 1 : 0;
                pos[k] = found[k] ? (uint64_t)p : 0;
                continue;
            }
            bvect bv;
            const bool f = mode == 1 ? sc.find_eq_str_prefix(sv, s, bv) : sc.find_eq_str(sv, s, bv);
            found[k] = f ? 1 : 0;
            counts[k] = (uint64_t)bv.count();
            export_bvector(bv, n_cols, 0, blocks + (size_t)k * n_cols * BMB200_BLOCK_WORDS, 0);
        }
        return 0;
    } catch (...) { return 1; }
}

int ref_str_time(const char* strs, uint32_t stride, uint64_t n, const uint8_t* nulls, int remap, int mode, const char* q,
                 uint32_t qstride, uint32_t nq, int repeats, double* best_sec, uint64_t* total)
{
    try {
        str_svect sv(nulls ? bm::use_null : bm::no_null);
        build(sv, strs, stride, n, nulls, remap);
        double best = 1e30; uint64_t tot = 0;
        for (int r = 0; r < repeats; ++r) {
            tot = 0;
            auto t0 = std::chrono::steady_clock::now();
            if (mode == 4) {
                std::vector<uint64_t> cnt(nq);
                run_pipeline<bm::agg_opt_only_counts>(sv, q, qstride, nq, 0, cnt.data(), 0);
                for (uint64_t c : cnt) tot += c;
            } else {
                str_scanner sc;
                for (uint32_t k = 0; k < nq; ++k) {
                    bvect bv;
                    if (mode == 1) sc.find_eq_str_prefix(sv, q + (size_t)k * qstride, bv);
                    else sc.find_eq_str(sv, q + (size_t)k * qstride, bv);
                    tot += (uint64_t)bv.count();
                }
            }
            double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            if (sec < best) best = sec;
        }
        *best_sec = best; *total = tot;
        return 0;
    } catch (...) { return 1; }
}

} // extern "C"
