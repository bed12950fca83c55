/*
 * ref_mismatch_shim.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * extern "C" wrapper around the UNMODIFIED reference's sparse-vector mismatch functions
 *   bm::sparse_vector_find_mismatch(bv, sv1, sv2, null_proc)          src/bmsparsevec_algo.h:657
 *   bm::sparse_vector_find_first_mismatch(sv1, sv2, midx, null_proc)   src/bmsparsevec_algo.h:479
 * over bm::sparse_vector<uint32_t / uint64_t / int32_t / int64_t>, and the closed forms of include/bmb200.h evaluated with the
 * reference's own bvector operations (bit_xor, |=, &=, set_range, find), so a difference between the two tells a reference
 * defect from a contract error.  Built by oracle/mismatch.mk into oracle/_ref/libbmref_mismatch.so with the reference's own
 * AVX2 flags, where the reference tree exists.  Never linked into the product.
 *
 * type: 0 = uint32_t, 1 = uint64_t, 2 = int32_t, 3 = int64_t.  Element values cross as int64_t (the bits of a uint64_t;
 * narrowed for the 32-bit types).  nullsK (may be null: a non-nullable vector) marks the NULL elements of vector K.
 * null_proc: 0 = bm::no_null, 1 = bm::use_null.
 *   ref_mm_find:   sparse_vector_find_mismatch -> count() + dense words of n_cols columns.
 *   ref_mm_first:  sparse_vector_find_first_mismatch -> found, midx.
 *   ref_mm_closed: the closed form through bvector ops; first = 0: the vector form (count + words), 1: the first form
 *                  (count + words of F, and F.find() as found / midx).
 *   ref_mm_time:   seconds (best of `repeats`) of each reference call alone, one core: find_mismatch (-> count()) and
 *                  find_first_mismatch (-> found, midx) on the same pair.
 */
#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstring>
#include <vector>

#include "bm.h"
#include "bmsparsevec.h"
#include "bmsparsevec_algo.h"

typedef bm::bvector<> bvect;

namespace {

constexpr uint64_t kBlockBits = 65536;

void to_words(const bvect& bv, uint32_t* w, uint32_t n_cols)
{
    const uint64_t nbits = (uint64_t)n_cols * kBlockBits;
    std::memset(w, 0, (size_t)n_cols * 8192);
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
struct Pair {
    SV a, b;
    Pair(const int64_t* v1, const uint8_t* n1, uint64_t s1, const int64_t* v2, const uint8_t* n2, uint64_t s2)
        : a(n1 ? bm::use_null : bm::no_null), b(n2 ? bm::use_null : bm::no_null)
    {
        build_sv(a, v1, n1, s1);
        build_sv(b, v2, n2, s2);
    }
};

bm::null_support np_of(int null_proc) { return null_proc ? bm::use_null : bm::no_null; }

#define PAIR_ARGS const int64_t* v1, const uint8_t* n1, uint64_t s1, const int64_t* v2, const uint8_t* n2, uint64_t s2

template<class SV>
int find(PAIR_ARGS, int null_proc, uint32_t n_cols, uint64_t* count, uint32_t* words)
{
    Pair<SV> p(v1, n1, s1, v2, n2, s2);
    bvect bv;
    bm::sparse_vector_find_mismatch(bv, p.a, p.b, np_of(null_proc));
    *count = (uint64_t)bv.count();
    to_words(bv, words, n_cols);
    return 0;
}

template<class SV>
int first(PAIR_ARGS, int null_proc, int* found, uint64_t* midx)
{
    Pair<SV> p(v1, n1, s1, v2, n2, s2);
    typename SV::size_type m = 0;
    *found = bm::sparse_vector_find_first_mismatch(p.a, p.b, m, np_of(null_proc)) ? 1 : 0;
    *midx = (uint64_t)m;
    return 0;
}

template<class SV>
const bvect* plane(const SV& sv, unsigned j)
{
    if (j >= sv.slices()) return 0;
    const bvect* bv = sv.get_slice(j);
    return bv == sv.get_null_bvector() ? 0 : bv;
}

// [0, s) as a bvector
bvect prefix(uint64_t s)
{
    bvect r;
    if (s) r.set_range(0, (bvect::size_type)(s - 1));
    return r;
}

template<class SV>
int closed(PAIR_ARGS, int null_proc, int first_form, uint32_t n_cols, uint64_t* count, uint32_t* words, int* found, uint64_t* midx)
{
    Pair<SV> p(v1, n1, s1, v2, n2, s2);
    const unsigned np = std::max(p.a.effective_slices(), p.b.effective_slices());
    bvect D;
    for (unsigned j = 0; j < np; ++j) {
        const bvect* a = plane(p.a, j);
        const bvect* b = plane(p.b, j);
        bvect x;
        if (a && b) x.bit_xor(*a, *b, bvect::opt_none);
        else if (a) x = *a;
        else if (b) x = *b;
        D |= x;
    }
    const uint64_t sa = p.a.size(), sb = p.b.size();
    if (!first_form && sa != sb) D.set_range((bvect::size_type)std::min(sa, sb), (bvect::size_type)(std::max(sa, sb) - 1));
    const bvect* na = p.a.get_null_bvector();
    const bvect* nb = p.b.get_null_bvector();
    if (null_proc) {
        if (na && nb) { bvect x; x.bit_xor(*na, *nb, bvect::opt_none); D |= x; }
        else if (na) { bvect r = prefix(first_form ? sb : sa); if (first_form) r ^= *na; else r -= *na; D |= r; }
        else if (nb) { bvect r = prefix(first_form ? sa : sb); if (first_form) r ^= *nb; else r -= *nb; D |= r; }
    } else if (!first_form) {
        if (na && nb) { bvect x; x.bit_or(*na, *nb, bvect::opt_none); D &= x; }
        else if (na) D &= *na;
        else if (nb) D &= *nb;
    }
    *count = (uint64_t)D.count();
    to_words(D, words, n_cols);
    bvect::size_type m = 0;
    *found = D.find(m) ? 1 : 0;
    *midx = *found ? (uint64_t)m : (uint64_t)bm::id_max;
    return 0;
}

template<class SV>
int time_mm(PAIR_ARGS, int null_proc, int repeats, double* sec_find, uint64_t* count, double* sec_first, int* found, uint64_t* midx)
{
    Pair<SV> p(v1, n1, s1, v2, n2, s2);
    *sec_find = *sec_first = 1e30;
    for (int r = 0; r < repeats; ++r) {
        bvect bv;
        auto t0 = std::chrono::steady_clock::now();
        bm::sparse_vector_find_mismatch(bv, p.a, p.b, np_of(null_proc));
        *sec_find = std::min(*sec_find, std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count());
        *count = (uint64_t)bv.count();
        typename SV::size_type m = 0;
        t0 = std::chrono::steady_clock::now();
        *found = bm::sparse_vector_find_first_mismatch(p.a, p.b, m, np_of(null_proc)) ? 1 : 0;
        *sec_first = std::min(*sec_first, std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count());
        *midx = (uint64_t)m;
    }
    return 0;
}

typedef bm::sparse_vector<uint32_t, bvect> sv_u32;
typedef bm::sparse_vector<uint64_t, bvect> sv_u64;
typedef bm::sparse_vector<int32_t, bvect> sv_i32;
typedef bm::sparse_vector<int64_t, bvect> sv_i64;

} // namespace

#define REF_MM_DISPATCH(F, ...) \
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

int ref_mm_find(int type, PAIR_ARGS, int null_proc, uint32_t n_cols, uint64_t* count, uint32_t* words)
{
    REF_MM_DISPATCH(find, v1, n1, s1, v2, n2, s2, null_proc, n_cols, count, words)
}

int ref_mm_first(int type, PAIR_ARGS, int null_proc, int* found, uint64_t* midx)
{
    REF_MM_DISPATCH(first, v1, n1, s1, v2, n2, s2, null_proc, found, midx)
}

int ref_mm_closed(int type, PAIR_ARGS, int null_proc, int first_form, uint32_t n_cols, uint64_t* count, uint32_t* words,
                  int* found, uint64_t* midx)
{
    REF_MM_DISPATCH(closed, v1, n1, s1, v2, n2, s2, null_proc, first_form, n_cols, count, words, found, midx)
}

int ref_mm_time(int type, PAIR_ARGS, int null_proc, int repeats, double* sec_find, uint64_t* count, double* sec_first, int* found,
                uint64_t* midx)
{
    REF_MM_DISPATCH(time_mm, v1, n1, s1, v2, n2, s2, null_proc, repeats, sec_find, count, sec_first, found, midx)
}

} // extern "C"
