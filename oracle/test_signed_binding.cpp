/*
 * test_signed_binding.cpp -- TEST INFRASTRUCTURE.  Drop-in check of the signed scanner at the bm::bvector<> level: the
 * UNMODIFIED reference's bm::sparse_vector_scanner<> (headers from the reference tree) against bm::b200::scanner<>
 * (bitmagic_b200/include/bmb200_scanner.hpp, which talks to libbmb200.so) on real signed vectors:
 * sparse_vector<int32_t / int64_t> plain and nullable, rsc_sparse_vector<int32_t / int64_t>; every public search, the
 * batched forms and the counts.  Parity criterion = the reference's own: compare() == 0 and equal count().
 * Built by oracle/signed.mk into oracle/_ref/.
 *
 * Search values stay within [INT32_MIN, INT32_MAX] also for int64_t vectors: the reference's signed int64_t searches with
 * a value outside that range do not compute the comparison (see DESIGN.md, signed scanner), so there the product is
 * checked against the restated contract (orc_scan_signed, oracle/bm_oracle_signed.c) instead.  Stored int64_t elements span the whole range.
 */
#include <cstdio>
#include <cstdint>
#include <limits>
#include <random>
#include <vector>

#include "bm.h"
#include "bmalgo.h"
#include "bmsparsevec.h"
#include "bmsparsevec_compr.h"
#include "bmsparsevec_algo.h"
#include "bmb200_aggregator.hpp"
#include "bmb200_scanner.hpp"

typedef bm::bvector<> bvect;
static int g_fail = 0, g_checks = 0;
#define CHECK(cond, ...) do { ++g_checks; if (!(cond)) { ++g_fail; std::printf("FAIL %s:%d: ", __FILE__, __LINE__); std::printf(__VA_ARGS__); std::printf("\n"); } } while (0)

// n elements: runs of one value (GAP / FULL planes), an iid region (bit planes), NULLs (nullable only), and the extremes
template<class SV>
static void fill(SV& sv, std::mt19937_64& rng, uint64_t n, bool nullable, int64_t lo, int64_t hi)
{
    typedef typename SV::value_type V;
    sv.resize((typename SV::size_type)n);
    std::uniform_int_distribution<int64_t> val(lo, hi);
    std::uniform_real_distribution<double> u(0.0, 1.0);
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t nb = i >> 16;
        if (nullable && (nb % 5 == 2 || u(rng) < 0.3)) continue;
        V x;
        if (nb % 5 == 1) x = V(((i >> 11) & 1u) ? hi : lo);              // long runs
        else if (i % 997 == 0) x = std::numeric_limits<V>::min();
        else if (i % 991 == 0) x = std::numeric_limits<V>::max();
        else x = V(val(rng));
        sv.set((typename SV::size_type)i, x);
    }
    BM_DECLARE_TEMP_BLOCK(tb)
    sv.optimize(tb);
}

template<class SV>
static void ref_search(bm::sparse_vector_scanner<SV>& sc, const SV& v, int pred, int64_t a, int64_t b, bvect& out)
{
    typedef typename SV::value_type V;
    switch (pred) {
    case BMB200_SCAN_EQ: sc.find_eq(v, V(a), out); break;
    case BMB200_SCAN_GT: sc.find_gt(v, V(a), out); break;
    case BMB200_SCAN_GE: sc.find_ge(v, V(a), out); break;
    case BMB200_SCAN_LT: sc.find_lt(v, V(a), out); break;
    case BMB200_SCAN_LE: sc.find_le(v, V(a), out); break;
    default: sc.find_range(v, V(a), V(b), out); break;
    }
}

template<class SV>
static void gpu_search(bm::b200::scanner<SV>& sc, int pred, int64_t a, int64_t b, bvect& out)
{
    typedef typename SV::value_type V;
    switch (pred) {
    case BMB200_SCAN_EQ: sc.find_eq(V(a), out); break;
    case BMB200_SCAN_GT: sc.find_gt(V(a), out); break;
    case BMB200_SCAN_GE: sc.find_ge(V(a), out); break;
    case BMB200_SCAN_LT: sc.find_lt(V(a), out); break;
    case BMB200_SCAN_LE: sc.find_le(V(a), out); break;
    default: sc.find_range(V(a), V(b), out); break;
    }
}

// few = true: four of the search values and no batched forms (the vectors past 2^32, where every search spans 65 539 columns)
template<class SV>
static void check_vector(bm::b200::context& ctx, const SV& sv, const char* what, int64_t lo, int64_t hi, bool few = false)
{
    const int64_t i32min = std::numeric_limits<int32_t>::min(), i32max = std::numeric_limits<int32_t>::max();
    bm::sparse_vector_scanner<SV> ref_sc;
    bm::b200::scanner<SV> sc(ctx, sv);
    const int64_t vals[][2] = {{0, 0}, {lo, hi}, {-9, 9}, {i32min, i32max}, {-1, 1}, {-2, -1}, {1, -2}, {hi, lo}, {lo - 1, lo + 1},
                               {hi + 1, hi + 9}, {-3, 3}, {7, 7}, {i32max, i32min}, {i32min + 1, -i32max}};
    auto in_i32 = [&](int64_t x) { return x < i32min ? i32min : x > i32max ? i32max : x; };   // see the file comment
    for (int pred = BMB200_SCAN_EQ; pred <= BMB200_SCAN_RANGE; ++pred) {
        for (size_t q = 0; q < (few ? 4u : sizeof(vals) / sizeof(vals[0])); ++q) {
            const auto& vv = vals[q];
            const int64_t v[2] = {in_i32(vv[0]), in_i32(vv[1])};
            bvect r, g;
            ref_search(ref_sc, sv, pred, v[0], v[1], r);
            gpu_search(sc, pred, v[0], v[1], g);
            CHECK(r.compare(g) == 0 && r.count() == g.count(), "%s pred=%d value=%lld/%lld: count ref %llu gpu %llu", what, pred,
                  (long long)v[0], (long long)v[1], (unsigned long long)r.count(), (unsigned long long)g.count());
        }
        if (few) continue;
        // batched and count-only forms: two's-complement int64 values in the uint64_t slots
        std::vector<int64_t> sv64 = pred == BMB200_SCAN_RANGE ? std::vector<int64_t>{-2, 40, 300, -10, 0, 0, i32min, -1}
                                                                : std::vector<int64_t>{0, -3, 77, i32min, -1, i32max};
        std::vector<uint64_t> slots(sv64.begin(), sv64.end());
        std::vector<bvect> outs; std::vector<bvect::size_type> counts;
        sc.find_batch(pred, slots, outs); sc.count_batch(pred, slots, counts);
        for (size_t k = 0; k < outs.size(); ++k) {
            bvect r;
            if (pred == BMB200_SCAN_RANGE) ref_search(ref_sc, sv, pred, sv64[2 * k], sv64[2 * k + 1], r);
            else ref_search(ref_sc, sv, pred, sv64[k], 0, r);
            CHECK(r.compare(outs[k]) == 0 && r.count() == counts[k], "%s batch pred=%d k=%zu", what, pred, k);
        }
    }
    bvect r, g;
    ref_sc.find_zero(sv, r); sc.find_zero(g);
    CHECK(r.compare(g) == 0 && r.count() == g.count(), "%s find_zero", what);
    bvect rn, gn;
    ref_sc.find_nonzero(sv, rn); sc.find_nonzero(gn);
    if constexpr (SV::is_compressed()) {
        // the reference's find_nonzero of an RSC vector leaves its answer in the compressed index space (no decompress);
        // the binding answers in logical positions like every other search: the two agree through the NOT-NULL vector
        bvect rl;
        bm::rank_compressor<bvect>().decompress(rl, *sv.get_null_bvector(), rn);
        CHECK(rl.compare(gn) == 0 && rn.count() == gn.count(), "%s find_nonzero", what);
    } else {
        CHECK(rn.compare(gn) == 0 && rn.count() == gn.count(), "%s find_nonzero", what);
    }
}

#ifdef BM64ADDR
// the reference's signed searches are several times slower in a BM64ADDR build: the vectors below get the short value list there
static const bool few64 = true;
#else
static const bool few64 = false;
#endif

template<class V>
static void run_type(bm::b200::context& ctx, std::mt19937_64& rng, const char* tname)
{
    typedef bm::sparse_vector<V, bvect> svect;
    typedef bm::rsc_sparse_vector<V, svect> rsc_vect;
    const int64_t vmin = std::numeric_limits<V>::min(), vmax = std::numeric_limits<V>::max();
    struct Case { uint64_t n; int64_t lo, hi; } cases[] = {
        {3u * 65536u + 77u, -1000, 1000}, {2u * 65536u, 1, 500}, {70000u, -600, -1}, {0u, -5, 5}, {65536u, vmin + 1, vmax - 9}};      // hi + 9 stays in range
    char what[96];
    for (const Case& cs : cases) {
        for (int nullable = 0; nullable < 2; ++nullable) {
            svect sv(nullable ? bm::use_null : bm::no_null);
            fill(sv, rng, cs.n, nullable != 0, cs.lo, cs.hi);
            std::snprintf(what, sizeof(what), "%s n=%llu [%lld,%lld] nullable=%d", tname, (unsigned long long)cs.n,
                          (long long)cs.lo, (long long)cs.hi, nullable);
            check_vector(ctx, sv, what, cs.lo, cs.hi, few64);
            if (nullable) {
                rsc_vect rsc;
                rsc.load_from(sv);
                rsc.sync();
                std::snprintf(what, sizeof(what), "rsc<%s> n=%llu [%lld,%lld]", tname, (unsigned long long)cs.n, (long long)cs.lo,
                              (long long)cs.hi);
                check_vector(ctx, rsc, what, cs.lo, cs.hi, few64);
            }
        }
    }
}

#ifdef BM64ADDR
// ---- BM64ADDR: a nullable sparse_vector<int64_t> and its rsc_sparse_vector of more than 2^32 elements, whose stored elements sit
// on both sides of 2^32 (columns 65535 / 65536).  test_cxx_binding covers a plain (not nullable) vector past 2^32 ----
static void check_past_2_32(bm::b200::context& ctx, std::mt19937_64& rng)
{
    typedef bm::sparse_vector<int64_t, bvect> svect;
    typedef bm::rsc_sparse_vector<int64_t, svect> rsc_vect;
    const uint64_t B = 65536u, G = uint64_t(1) << 32, n = G + 2 * B + 321;
    svect sv(bm::use_null);
    sv.resize((svect::size_type)n);
    std::uniform_int_distribution<int64_t> val(-700, 700);
    for (uint64_t i = G - 2 * B + 3; i < n; ++i) {
        if (rng() % 4 == 0) continue;
        int64_t x = val(rng);
        if ((i >> 16) == 65536) x = ((i >> 10) & 1u) ? -9 : 9;                                    // runs in the first column past 2^32
        else if (i % 991 == 0) x = std::numeric_limits<int64_t>::min();
        sv.set((svect::size_type)i, x);
    }
    for (uint64_t i = 0; i < 3000; ++i) sv.set((svect::size_type)(i * 11), int64_t(i % 50) - 25);
    { BM_DECLARE_TEMP_BLOCK(tb) sv.optimize(tb); }
    check_vector(ctx, sv, "64: int64_t n=2^32+2*65536+321 nullable", -700, 700, true);
    rsc_vect rsc;
    rsc.load_from(sv);
    rsc.sync();
    check_vector(ctx, rsc, "64: rsc<int64_t> n=2^32+2*65536+321", -700, 700, true);
}
#endif

int main()
{
    std::mt19937_64 rng(20261016);
    bm::b200::context ctx(0);
#ifdef BM64ADDR
    check_past_2_32(ctx, rng);
#endif
    run_type<int32_t>(ctx, rng, "int32_t");
    run_type<int64_t>(ctx, rng, "int64_t");
    std::printf("test_signed_binding: %d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
