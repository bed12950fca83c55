/*
 * test_in_binding.cpp -- TEST INFRASTRUCTURE.  Drop-in check of the set-membership search at the bm::bvector<> level: the
 * UNMODIFIED reference's iterator bm::sparse_vector_scanner<>::find_eq(sv, start, end, bv_out) (src/bmsparsevec_algo.h:1398-1423)
 * against bm::b200::scanner<>::find_eq(first, last, bv_out) and count_eq(first, last) on sparse_vector<uint32_t / uint64_t /
 * int32_t / int64_t>, plain and nullable, with an empty and with a pre-filled bv_out (the reference ORs into it, and a listed 0
 * then ANDs it with the NOT-NULL vector).  Parity criterion = the reference's own: compare() == 0 and equal count().
 *
 * rsc_sparse_vector<>: the reference's iterator form answers a non-zero value in compressed positions but 0 (find_zero) in
 * logical ones.  The harness confirms that reading -- the iterator result over the non-zero values, decompressed, is the OR of
 * the single-value find_eq(v), and a listed 0 adds find_zero(0)'s logical answer to the compressed bits -- and holds the binding
 * to the OR of the single-value find_eq(v), which is in logical positions throughout.
 * Signed lists stay within [INT32_MIN, INT32_MAX] as in test_signed_binding.  Built by oracle/in.mk into oracle/_ref/.
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

// n elements: runs of two values (GAP / FULL planes), an iid region (bit planes), a sparse region, NULLs (nullable only)
template<class SV>
static void fill(SV& sv, std::mt19937_64& rng, uint64_t n, bool nullable, int64_t lo, int64_t hi)
{
    typedef typename SV::value_type V;
    sv.resize((typename SV::size_type)n);
    std::uniform_int_distribution<int64_t> val(lo, hi);
    std::uniform_real_distribution<double> u(0.0, 1.0);
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t nb = i >> 16;
        if (nullable && (nb % 4 == 3 || u(rng) < 0.3)) continue;
        V x;
        if (nb % 4 == 1) x = V(((i >> 11) & 1u) ? hi : lo);
        else if (nb % 4 == 2) x = u(rng) < 0.01 ? V(val(rng)) : V(0);
        else x = V(val(rng));
        sv.set((typename SV::size_type)i, x);
    }
    BM_DECLARE_TEMP_BLOCK(tb)
    sv.optimize(tb);
}

template<class V>
static std::vector<std::vector<V>> lists(std::mt19937_64& rng, int64_t lo, int64_t hi)
{
    const bool sgn = std::numeric_limits<V>::is_signed;
    const int64_t tmin = sgn ? (int64_t)std::numeric_limits<int32_t>::min() : 0;
    const int64_t tmax = sgn ? (int64_t)std::numeric_limits<int32_t>::max() : (int64_t)std::numeric_limits<uint32_t>::max();
    std::uniform_int_distribution<int64_t> val(lo, hi);
    std::vector<std::vector<V>> out;
    out.push_back({V(0)});
    out.push_back({V(lo)});
    out.push_back({V(hi), V(hi), V(lo + 1), V(hi + 1), V(tmax), V(tmin)});                   // duplicates, absent, beyond the planes
    out.push_back({V(7), V(0), V(lo), V(7), V(tmax)});
    std::vector<V> big;
    for (int k = 0; k < 2000; ++k) big.push_back(V(k % 3 ? val(rng) : int64_t(rng() % 5000)));
    out.push_back(big);
    big.push_back(V(0));
    out.push_back(big);
    return out;
}

template<class SV>
static void check_vector(bm::b200::context& ctx, std::mt19937_64& rng, const SV& sv, const char* what, int64_t lo, int64_t hi)
{
    typedef typename SV::value_type V;
    bm::sparse_vector_scanner<SV> ref_sc;
    bm::b200::scanner<SV> sc(ctx, sv);
    const uint64_t n = sv.size();
    for (const std::vector<V>& l : lists<V>(rng, lo, hi)) {
        for (int pre = 0; pre < 2; ++pre) {
            bvect r, g;
            if (pre) for (uint64_t i = 0; i < n + 1000; i += 7) { r.set((bvect::size_type)i); g.set((bvect::size_type)i); }
            ref_sc.find_eq(sv, l.begin(), l.end(), r);
            sc.find_eq(l.begin(), l.end(), g);
            CHECK(r.compare(g) == 0 && r.count() == g.count(), "%s list of %zu (first %lld) prefill=%d: count ref %llu gpu %llu", what,
                  l.size(), (long long)l[0], pre, (unsigned long long)r.count(), (unsigned long long)g.count());
            if (!pre) CHECK(sc.count_eq(l.begin(), l.end()) == r.count(), "%s count_eq list of %zu", what, l.size());
        }
    }
    bvect e;                                                   // an empty range: bv_out untouched
    e.set(5); e.set(100000);
    const std::vector<V> none;
    sc.find_eq(none.begin(), none.end(), e);
    CHECK(e.count() == 2 && e.test(5) && e.test(100000) && sc.count_eq(none.begin(), none.end()) == 0, "%s empty range", what);
}

template<class RSC>
static void check_rsc(bm::b200::context& ctx, std::mt19937_64& rng, const RSC& rsc, const char* what, int64_t lo, int64_t hi)
{
    typedef typename RSC::value_type V;
    bm::sparse_vector_scanner<RSC> ref_sc;
    bm::b200::scanner<RSC> sc(ctx, rsc);
    const bvect& nn = *rsc.get_null_bvector();
    for (const std::vector<V>& l : lists<V>(rng, lo, hi)) {
        bvect want, zero, g;
        bool has0 = false;
        std::vector<V> nz;
        for (V v : l) { bvect one; ref_sc.find_eq(rsc, v, one); want.bit_or(one); if (v == 0) has0 = true; else nz.push_back(v); }
        sc.find_eq(l.begin(), l.end(), g);
        CHECK(want.compare(g) == 0 && want.count() == g.count(), "%s list of %zu: count OR-of-find_eq %llu gpu %llu", what, l.size(),
              (unsigned long long)want.count(), (unsigned long long)g.count());
        CHECK(sc.count_eq(l.begin(), l.end()) == want.count(), "%s count_eq list of %zu", what, l.size());
        // the reference's iterator form: non-zero values in compressed positions, 0 in logical positions
        bvect it_nz, it_all, dec;
        ref_sc.find_eq(rsc, nz.begin(), nz.end(), it_nz);
        ref_sc.find_eq(rsc, l.begin(), l.end(), it_all);
        bm::rank_compressor<bvect>().decompress(dec, nn, it_nz);
        bvect want_nz;
        for (V v : nz) { bvect one; ref_sc.find_eq(rsc, v, one); want_nz.bit_or(one); }
        CHECK(dec.compare(want_nz) == 0, "%s: the iterator find_eq over non-zero values answers in compressed positions", what);
        if (has0) {
            ref_sc.find_eq(rsc, V(0), zero);
            bvect mixed(it_nz);
            mixed.bit_or(zero);
            mixed.bit_and(nn);
            CHECK(mixed.compare(it_all) == 0, "%s: a listed 0 adds find_zero's logical answer to the compressed bits", what);
        }
    }
}

template<class V>
static void run_type(bm::b200::context& ctx, std::mt19937_64& rng, const char* tname)
{
    typedef bm::sparse_vector<V, bvect> svect;
    typedef bm::rsc_sparse_vector<V, svect> rsc_vect;
    const bool sgn = std::numeric_limits<V>::is_signed;
    struct Case { uint64_t n; int64_t lo, hi; } cases[] = {
        {3u * 65536u + 77u, sgn ? -1000 : 1, 1000}, {2u * 65536u + 5u, sgn ? -300000 : 1, 1250000}, {0u, 1, 5}};
    char what[96];
    for (const Case& cs : cases) {
        for (int nullable = 0; nullable < 2; ++nullable) {
            svect sv(nullable ? bm::use_null : bm::no_null);
            fill(sv, rng, cs.n, nullable != 0, cs.lo, cs.hi);
            std::snprintf(what, sizeof(what), "%s n=%llu [%lld,%lld] nullable=%d", tname, (unsigned long long)cs.n, (long long)cs.lo,
                          (long long)cs.hi, nullable);
            check_vector(ctx, rng, sv, what, cs.lo, cs.hi);
            if (nullable && cs.n) {
                rsc_vect rsc;
                rsc.load_from(sv);
                rsc.sync();
                std::snprintf(what, sizeof(what), "rsc<%s> n=%llu", tname, (unsigned long long)cs.n);
                check_rsc(ctx, rng, rsc, what, cs.lo, cs.hi);
            }
        }
    }
}

int main()
{
    std::mt19937_64 rng(20261018);
    bm::b200::context ctx(0);
    run_type<uint32_t>(ctx, rng, "uint32_t");
    run_type<uint64_t>(ctx, rng, "uint64_t");
    run_type<int32_t>(ctx, rng, "int32_t");
    run_type<int64_t>(ctx, rng, "int64_t");
    std::printf("test_in_binding: %d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
