/*
 * ref_remap_shim.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * extern "C" wrapper around the UNMODIFIED reference's bm::set2set_11_transform<SV>::remap (src/bmsparsevec_algo.h:2097-2205)
 * over SV = bm::sparse_vector<bvector<>::size_type>, the only vector it compiles for.  Built by oracle/remap.mk into
 * oracle/_ref/libbmref_remap.so (32-bit addressing: size_type = uint32_t) and libbmref_remap64.so (-DBM64ADDR: uint64_t)
 * with the reference's own AVX2 flags, where the reference tree exists.  Never linked into the product.
 *
 * Values and ids cross as size_type arrays (ref_remap_word_bytes() tells which).  nulls (may be null: a non-nullable
 * vector) marks the NULL elements; the vector is import()ed from values[0..n), NULLs set, then optimize()d.  bv_in is the
 * set of ids[0..n_ids) (any order, any value, also past n).
 *   ref_remap:      mode bits: 1 = attach_sv(&sv, true) + remap(bv_in, bv_out) instead of remap(bv_in, sv, bv_out),
 *                   2 = bv_out pre-filled with {1, 3, 77, 65536 * 5 + 9} before the call.
 *                   -> bv_out.count() and its first `cap` values in order.
 *   ref_remap_time: seconds (best of `repeats`) of remap(bv_in, sv, bv_out) alone, one core -> count().
 */
#include <algorithm>
#include <chrono>
#include <cstdint>
#include <vector>

#include "bm.h"
#include "bmsparsevec.h"
#include "bmsparsevec_algo.h"

typedef bm::bvector<> bvect;
typedef bvect::size_type size_type;
typedef bm::sparse_vector<size_type, bvect> svect;

namespace {

void build_sv(svect& sv, const size_type* values, const uint8_t* nulls, uint64_t n)
{
    std::vector<size_type> v(values, values + n);
    if (nulls) for (uint64_t i = 0; i < n; ++i) if (nulls[i]) v[i] = 0;
    if (n) sv.import(v.data(), (size_type)n);
    if (nulls) {
        bvect bn;
        for (uint64_t i = 0; i < n; ++i) if (nulls[i]) bn.set((size_type)i);
        sv.set_null(bn);
    }
    BM_DECLARE_TEMP_BLOCK(tb)
    sv.optimize(tb);
}

void build_bv(bvect& bv, const size_type* ids, uint64_t n_ids)
{
    std::vector<size_type> v(ids, ids + n_ids);
    std::sort(v.begin(), v.end());
    if (!v.empty()) bv.set(v.data(), (size_type)v.size(), bm::BM_SORTED);
    bv.optimize();
}

} // namespace

extern "C" {

int ref_remap_word_bytes() { return (int)sizeof(size_type); }

int ref_remap(const size_type* values, const uint8_t* nulls, uint64_t n, const size_type* ids, uint64_t n_ids, int mode,
              uint64_t* count, size_type* out, uint64_t cap)
{
    try {
        svect sv(nulls ? bm::use_null : bm::no_null);
        build_sv(sv, values, nulls, n);
        bvect bv_in, bv_out;
        build_bv(bv_in, ids, n_ids);
        if (mode & 2) { bv_out.set(1); bv_out.set(3); bv_out.set(77); bv_out.set(65536u * 5u + 9u); }
        bm::set2set_11_transform<svect> tr;
        if (mode & 1) { tr.attach_sv(&sv, true); tr.remap(bv_in, bv_out); }
        else tr.remap(bv_in, sv, bv_out);
        *count = bv_out.count();
        uint64_t k = 0;
        for (bvect::enumerator en = bv_out.first(); en.valid() && k < cap; ++en) out[k++] = *en;
        return 0;
    } catch (...) {
        return 1;
    }
}

int ref_remap_time(const size_type* values, const uint8_t* nulls, uint64_t n, const size_type* ids, uint64_t n_ids, int repeats,
                   uint64_t* count, double* seconds)
{
    try {
        svect sv(nulls ? bm::use_null : bm::no_null);
        build_sv(sv, values, nulls, n);
        bvect bv_in;
        build_bv(bv_in, ids, n_ids);
        double best = 1e30;
        for (int r = 0; r < std::max(repeats, 1); ++r) {
            bvect bv_out;
            bm::set2set_11_transform<svect> tr;
            const auto t0 = std::chrono::steady_clock::now();
            tr.remap(bv_in, sv, bv_out);
            const auto t1 = std::chrono::steady_clock::now();
            best = std::min(best, std::chrono::duration<double>(t1 - t0).count());
            *count = bv_out.count();
        }
        *seconds = best;
        return 0;
    } catch (...) {
        return 1;
    }
}

} // extern "C"
