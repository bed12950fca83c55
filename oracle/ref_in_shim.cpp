/*
 * ref_in_shim.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * extern "C" wrapper around the UNMODIFIED reference's set-membership search: the iterator form of
 * bm::sparse_vector_scanner<SV>::find_eq(sv, start, end, bv_out) (src/bmsparsevec_algo.h:1398-1423) over
 * bm::sparse_vector<uint32_t / uint64_t / int32_t / int64_t> (plain and nullable), and the single-value find_eq over
 * bm::rsc_sparse_vector<> of the same types.  Built by oracle/in.mk into oracle/_ref/libbmref_in.so with the reference's own
 * AVX2 flags, where the reference tree exists.  Never linked into the product.
 *
 * type: 0 = uint32_t, 1 = uint64_t, 2 = int32_t, 3 = int64_t.  Element values and listed values cross as int64_t (the bits of
 * a uint64_t; narrowed for the 32-bit types).  nulls (may be null: a non-nullable vector) marks NULL elements.
 *   ref_in_planes: the vector's own planes (get_slice(j), j < effective_slices(), trailing absent ones trimmed) and, last, the
 *                  universe (NOT-NULL plane, else [0, n)) as per-column kind / blocks / GAP words, plane-major.
 *   ref_in_find:   bv_out = pre-fill (every `prefill`-th position of [0, n + 1000) when prefill > 0, else empty), then the
 *                  iterator find_eq over list[0..n_list); dense words of n_cols columns + count().
 *   ref_in_rsc:    the nullable vector rank-compressed (load_from + sync); mode 0: the OR over the list of the single-value
 *                  find_eq(sv, v, bv); mode 1: the iterator find_eq into an empty bv_out.  Dense words + count().
 *   ref_in_time:   seconds (best of `repeats`) of the iterator find_eq alone, one core, + the result's count().
 */
#include <chrono>
#include <cstdint>
#include <cstring>
#include <vector>

#include "bm.h"
#include "bmsparsevec.h"
#include "bmsparsevec_compr.h"
#include "bmsparsevec_algo.h"

#include "../include/bmb200.h"

typedef bm::bvector<> bvect;

namespace {

void export_bvector(const bvect& bv, uint32_t n_cols, uint8_t* kind, uint32_t* blocks, uint16_t* gaps)
{
    const bvect::blocks_manager_type& bman = bv.get_blocks_manager();
    BM_DECLARE_TEMP_BLOCK(tb)
    for (uint32_t c = 0; c < n_cols; ++c) {
        unsigned i = c >> 8, j = c & 255u;
        const bm::word_t* blk = 0;
        if (bman.is_init() && i < bman.top_block_size()) blk = bman.get_block_ptr(i, j);
        uint8_t kd;
        uint32_t* bout = blocks + (size_t)c * BMB200_BLOCK_WORDS;
        uint16_t* gout = gaps + (size_t)c * BMB200_GAP_MAX_WORDS;
        std::memset(gout, 0, sizeof(uint16_t) * BMB200_GAP_MAX_WORDS);
        if (!blk) { kd = BMB200_BLK_NULL; std::memset(bout, 0, BMB200_BLOCK_BYTES); }
        else if (blk == FULL_BLOCK_FAKE_ADDR || blk == FULL_BLOCK_REAL_ADDR) { kd = BMB200_BLK_FULL; std::memset(bout, 0xFF, BMB200_BLOCK_BYTES); }
        else if (BM_IS_GAP(blk)) {
            const bm::gap_word_t* g = BMGAP_PTR(blk);
            kd = BMB200_BLK_GAP;
            bm::gap_convert_to_bitset(tb.begin(), g); std::memcpy(bout, tb.begin(), BMB200_BLOCK_BYTES);
            std::memcpy(gout, g, sizeof(uint16_t) * bm::gap_length(g));
        } else { kd = BMB200_BLK_BIT; std::memcpy(bout, blk, BMB200_BLOCK_BYTES); }
        kind[c] = kd;
    }
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

template<class SV>
void build_sv(SV& sv, const int64_t* values, const uint8_t* nulls, uint64_t n)
{
    typedef typename SV::value_type V;
    std::vector<V> v(n);
    for (uint64_t i = 0; i < n; ++i) v[i] = (nulls && nulls[i]) ? V(0) : (V)values[i];
    if (n) sv.import(v.data(), (typename SV::size_type)n);
    else sv.resize(0);
    if (nulls) {
        bvect bn;
        for (uint64_t i = 0; i < n; ++i) if (nulls[i]) bn.set((bvect::size_type)i);
        sv.set_null(bn);
    }
    BM_DECLARE_TEMP_BLOCK(tb)
    sv.optimize(tb);
}

template<class SV>
std::vector<typename SV::value_type> list_of(const int64_t* list, uint64_t n_list)
{
    std::vector<typename SV::value_type> l(n_list);
    for (uint64_t k = 0; k < n_list; ++k) l[k] = (typename SV::value_type)list[k];
    return l;
}

template<class SV>
int planes(const int64_t* values, const uint8_t* nulls, uint64_t n, uint32_t n_cols, uint32_t max_planes,
           uint32_t* n_planes_out, uint8_t* kind, uint32_t* blocks, uint16_t* gaps)
{
    SV sv(nulls ? bm::use_null : bm::no_null);
    build_sv(sv, values, nulls, n);
    unsigned np = sv.effective_slices();
    while (np > 1 && !sv.get_slice(np - 1)) --np;
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
int find(const int64_t* values, const uint8_t* nulls, uint64_t n, const int64_t* list, uint64_t n_list, uint32_t prefill,
         uint32_t n_cols, uint64_t* count, uint32_t* words)
{
    SV sv(nulls ? bm::use_null : bm::no_null);
    build_sv(sv, values, nulls, n);
    std::vector<typename SV::value_type> l = list_of<SV>(list, n_list);
    bvect bv;
    if (prefill) for (uint64_t i = 0; i < n + 1000; i += prefill) bv.set((bvect::size_type)i);
    bm::sparse_vector_scanner<SV> sc;
    sc.find_eq(sv, l.begin(), l.end(), bv);
    *count = (uint64_t)bv.count();
    to_words(bv, words, n_cols);
    return 0;
}

template<class RSC>
int rsc(const int64_t* values, const uint8_t* nulls, uint64_t n, const int64_t* list, uint64_t n_list, int mode,
        uint32_t n_cols, uint64_t* count, uint32_t* words)
{
    typename RSC::sparse_vector_type sv(bm::use_null);
    build_sv(sv, values, nulls, n);
    RSC r;
    r.load_from(sv);
    r.sync();
    std::vector<typename RSC::value_type> l = list_of<RSC>(list, n_list);
    bm::sparse_vector_scanner<RSC> sc;
    bvect bv;
    if (mode == 0) {
        for (uint64_t k = 0; k < n_list; ++k) { bvect one; sc.find_eq(r, l[k], one); bv.bit_or(one); }
    } else sc.find_eq(r, l.begin(), l.end(), bv);
    *count = (uint64_t)bv.count();
    to_words(bv, words, n_cols);
    return 0;
}

template<class SV>
int time_find(const int64_t* values, const uint8_t* nulls, uint64_t n, const int64_t* list, uint64_t n_list, int repeats,
              double* best_sec, uint64_t* total)
{
    SV sv(nulls ? bm::use_null : bm::no_null);
    build_sv(sv, values, nulls, n);
    std::vector<typename SV::value_type> l = list_of<SV>(list, n_list);
    bm::sparse_vector_scanner<SV> sc;
    double best = 1e30;
    for (int r = 0; r < repeats; ++r) {
        bvect bv;
        auto t0 = std::chrono::steady_clock::now();
        sc.find_eq(sv, l.begin(), l.end(), bv);
        double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        if (sec < best) best = sec;
        *total = (uint64_t)bv.count();
    }
    *best_sec = best;
    return 0;
}

typedef bm::sparse_vector<uint32_t, bvect> sv_u32;
typedef bm::sparse_vector<uint64_t, bvect> sv_u64;
typedef bm::sparse_vector<int32_t, bvect> sv_i32;
typedef bm::sparse_vector<int64_t, bvect> sv_i64;

} // namespace

#define REF_IN_DISPATCH(F, ...) \
    try { \
        switch (type) { \
        case 0: return F<sv_u32>(__VA_ARGS__); \
        case 1: return F<sv_u64>(__VA_ARGS__); \
        case 2: return F<sv_i32>(__VA_ARGS__); \
        case 3: return F<sv_i64>(__VA_ARGS__); \
        default: return 2; \
        } \
    } catch (...) { return 1; }

extern "C" {

int ref_in_planes(int type, const int64_t* values, const uint8_t* nulls, uint64_t n, uint32_t n_cols, uint32_t max_planes,
                  uint32_t* n_planes_out, uint8_t* kind, uint32_t* blocks, uint16_t* gaps)
{
    REF_IN_DISPATCH(planes, values, nulls, n, n_cols, max_planes, n_planes_out, kind, blocks, gaps)
}

int ref_in_find(int type, const int64_t* values, const uint8_t* nulls, uint64_t n, const int64_t* list, uint64_t n_list,
                uint32_t prefill, uint32_t n_cols, uint64_t* count, uint32_t* words)
{
    REF_IN_DISPATCH(find, values, nulls, n, list, n_list, prefill, n_cols, count, words)
}

int ref_in_rsc(int type, const int64_t* values, const uint8_t* nulls, uint64_t n, const int64_t* list, uint64_t n_list, int mode,
               uint32_t n_cols, uint64_t* count, uint32_t* words)
{
    try {
        switch (type) {
        case 0: return rsc<bm::rsc_sparse_vector<uint32_t, sv_u32>>(values, nulls, n, list, n_list, mode, n_cols, count, words);
        case 1: return rsc<bm::rsc_sparse_vector<uint64_t, sv_u64>>(values, nulls, n, list, n_list, mode, n_cols, count, words);
        case 2: return rsc<bm::rsc_sparse_vector<int32_t, sv_i32>>(values, nulls, n, list, n_list, mode, n_cols, count, words);
        case 3: return rsc<bm::rsc_sparse_vector<int64_t, sv_i64>>(values, nulls, n, list, n_list, mode, n_cols, count, words);
        default: return 2;
        }
    } catch (...) { return 1; }
}

int ref_in_time(int type, const int64_t* values, const uint8_t* nulls, uint64_t n, const int64_t* list, uint64_t n_list,
                int repeats, double* best_sec, uint64_t* total)
{
    REF_IN_DISPATCH(time_find, values, nulls, n, list, n_list, repeats, best_sec, total)
}

} // extern "C"
