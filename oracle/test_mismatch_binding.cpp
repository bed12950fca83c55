/*
 * test_mismatch_binding.cpp -- TEST INFRASTRUCTURE.  Drop-in check of the sparse-vector mismatch at the bm::bvector<> level: the
 * UNMODIFIED reference's bm::sparse_vector_find_mismatch / bm::sparse_vector_find_first_mismatch (src/bmsparsevec_algo.h:657,479)
 * against bm::b200::sparse_vector_find_mismatch / sparse_vector_find_first_mismatch on sparse_vector<uint32_t / uint64_t /
 * int32_t / int64_t>, every nullable / plain pairing, both null_proc values, equal and different sizes.
 * Parity criterion = the reference's own: compare() == 0 and equal count(); the first form: equal found and midx.
 * Where the reference is defective (DESIGN.md 3.5f) the binding is held to the closed form evaluated with the reference's own
 * bvector operations instead:
 *   - the vector form with bm::use_null and two non-nullable vectors (the reference reports [0, bm::id_max)): no NULL term;
 *   - the first form, whose GAP x GAP comparison can miss or postpone a difference: the true lowest position of F, and the
 *     reference's answer must then be "not found" or later.
 * Built by oracle/mismatch.mk into oracle/_ref/ twice: as is and with -DBM64ADDR (then also vectors past 2^32).
 */
#include <algorithm>
#include <cstdio>
#include <cstdint>
#include <random>
#include <vector>

#include "bm.h"
#include "bmsparsevec.h"
#include "bmsparsevec_algo.h"
#include "bmb200_aggregator.hpp"
#include "bmb200_scanner.hpp"

typedef bm::bvector<> bvect;
static int g_fail = 0, g_checks = 0, g_first_defects = 0;
#define CHECK(cond, ...) do { ++g_checks; if (!(cond)) { ++g_fail; std::printf("FAIL %s:%d: ", __FILE__, __LINE__); std::printf(__VA_ARGS__); std::printf("\n"); } } while (0)

// n elements: runs of two values (GAP / FULL planes), an iid region (bit planes), a sparse region, NULLs (nullable only)
template<class SV>
static void fill(SV& sv, std::mt19937_64& rng, uint64_t n, bool nullable)
{
    typedef typename SV::value_type V;
    sv.resize((typename SV::size_type)n);
    std::uniform_int_distribution<int64_t> val(-1000, 100000);
    std::uniform_real_distribution<double> u(0.0, 1.0);
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t nb = i >> 16;
        if (nullable && (nb % 4 == 3 || u(rng) < 0.2)) continue;
        V x;
        if (nb % 4 == 1) x = V(((i >> 11) & 1u) ? 77 : 5);
        else if (nb % 4 == 2) x = u(rng) < 0.01 ? V(val(rng)) : V(0);
        else x = V(val(rng));
        sv.set((typename SV::size_type)i, x);
    }
    BM_DECLARE_TEMP_BLOCK(tb)
    sv.optimize(tb);
}

// the closed forms of include/bmb200.h through the reference's bvector operations
template<class SV>
static bvect closed(const SV& s1, const SV& s2, bm::null_support np, bool first)
{
    auto plane = [](const SV& sv, unsigned j) -> const bvect* {
        const bvect* bv = sv.get_slice(j);
        return bv == sv.get_null_bvector() ? nullptr : bv;
    };
    bvect D;
    const unsigned n = std::max(s1.effective_slices(), s2.effective_slices());
    for (unsigned j = 0; j < n; ++j) {
        const bvect* a = j < s1.slices() ? plane(s1, j) : nullptr;
        const bvect* b = j < s2.slices() ? plane(s2, j) : nullptr;
        bvect x;
        if (a && b) x.bit_xor(*a, *b, bvect::opt_none); else if (a) x = *a; else if (b) x = *b;
        D |= x;
    }
    const uint64_t sa = s1.size(), sb = s2.size();
    auto prefix = [](uint64_t s) { bvect r; if (s) r.set_range(0, (bvect::size_type)(s - 1)); return r; };
    if (!first && sa != sb) D.set_range((bvect::size_type)std::min(sa, sb), (bvect::size_type)(std::max(sa, sb) - 1));
    const bvect* na = s1.get_null_bvector();
    const bvect* nb = s2.get_null_bvector();
    if (np == bm::use_null) {
        if (na && nb) { bvect x; x.bit_xor(*na, *nb, bvect::opt_none); D |= x; }
        else if (na) { bvect r = prefix(first ? sb : sa); if (first) r ^= *na; else r -= *na; D |= r; }
        else if (nb) { bvect r = prefix(first ? sa : sb); if (first) r ^= *nb; else r -= *nb; D |= r; }
    } else if (!first) {
        if (na && nb) { bvect x; x.bit_or(*na, *nb, bvect::opt_none); D &= x; }
        else if (na) D &= *na;
        else if (nb) D &= *nb;
    }
    return D;
}

template<class SV>
static void check_pair(bm::b200::context& ctx, const SV& s1, const SV& s2, const char* what)
{
    for (bm::null_support np : {bm::no_null, bm::use_null}) {
        const char* nps = np == bm::use_null ? "use_null" : "no_null";
        bvect want, got;
        const bool defect1 = np == bm::use_null && !s1.get_null_bvector() && !s2.get_null_bvector();
        bm::sparse_vector_find_mismatch(want, s1, s2, defect1 ? bm::no_null : np);
        bm::b200::sparse_vector_find_mismatch(ctx, got, s1, s2, np);
        CHECK(got.compare(want) == 0 && got.count() == want.count(), "%s %s find_mismatch: count %llu vs %llu", what, nps,
              (unsigned long long)got.count(), (unsigned long long)want.count());
        CHECK(got.compare(closed(s1, s2, np, false)) == 0, "%s %s find_mismatch vs the closed form", what, nps);

        typename SV::size_type rpos = 0, gpos = 0, fpos = 0;
        const bool rf = bm::sparse_vector_find_first_mismatch(s1, s2, rpos, np);
        const bool gf = bm::b200::sparse_vector_find_first_mismatch(ctx, s1, s2, gpos, np);
        const bool ff = closed(s1, s2, np, true).find(fpos);
        CHECK(gf == ff && (gf ? gpos == fpos : gpos == (typename SV::size_type)bm::id_max), "%s %s find_first_mismatch: %d/%llu vs %d/%llu",
              what, nps, (int)gf, (unsigned long long)gpos, (int)ff, (unsigned long long)fpos);
        if (rf != gf || rpos != gpos) {
            ++g_first_defects;       // the reference's GAP x GAP comparison: it can only miss or postpone the first difference
            CHECK(gf && (!rf || rpos > gpos), "%s %s reference first mismatch %d/%llu vs %d/%llu", what, nps, (int)rf,
                  (unsigned long long)rpos, (int)gf, (unsigned long long)gpos);
        }
    }
}

template<class V>
static void run_type(bm::b200::context& ctx, std::mt19937_64& rng, const char* tname)
{
    typedef bm::sparse_vector<V, bvect> svect;
    const uint64_t B = 65536u;
    char what[160];
    for (uint64_t n : {uint64_t(1), B, 4 * B + 1234}) {
        for (int nl1 = 0; nl1 < 2; ++nl1) for (int nl2 = 0; nl2 < 2; ++nl2) {
            svect a(nl1 ? bm::use_null : bm::no_null);
            fill(a, rng, n, nl1 != 0);
            // b: a copy (or the same values in the other nullability), then versions of it
            svect b(nl2 ? bm::use_null : bm::no_null);
            b.resize(a.size());
            for (uint64_t i = 0; i < n; ++i)
                if (!a.is_null((typename svect::size_type)i)) b.set((typename svect::size_type)i, a.get((typename svect::size_type)i));
            b.optimize();
            std::snprintf(what, sizeof(what), "%s n=%llu null=%d/%d identical", tname, (unsigned long long)n, nl1, nl2);
            check_pair(ctx, a, b, what);
            svect c(b);                                            // a single difference at 0, the last element, a column edge
            c.set(0, V(c.get(0) + 1));
            c.set((typename svect::size_type)(n - 1), V(3));
            if (n > B) { c.set((typename svect::size_type)(B - 1), V(999)); c.set((typename svect::size_type)B, V(12)); }
            c.optimize();
            std::snprintf(what, sizeof(what), "%s n=%llu null=%d/%d edits", tname, (unsigned long long)n, nl1, nl2);
            check_pair(ctx, a, c, what);
            svect d(b);                                            // a different size: inside a column, then on a column edge
            d.resize((typename svect::size_type)(n + 777));
            d.set((typename svect::size_type)(n + 500), V(9));
            std::snprintf(what, sizeof(what), "%s n=%llu null=%d/%d longer", tname, (unsigned long long)n, nl1, nl2);
            check_pair(ctx, a, d, what);
            check_pair(ctx, d, a, what);
            if (n > B) {
                svect e(b);
                e.resize((typename svect::size_type)B);
                std::snprintf(what, sizeof(what), "%s n=%llu null=%d/%d cut at a column edge", tname, (unsigned long long)n, nl1, nl2);
                check_pair(ctx, a, e, what);
            }
            svect f(nl2 ? bm::use_null : bm::no_null);              // an unrelated vector: many planes differ
            fill(f, rng, n, nl2 != 0);
            std::snprintf(what, sizeof(what), "%s n=%llu null=%d/%d unrelated", tname, (unsigned long long)n, nl1, nl2);
            check_pair(ctx, a, f, what);
        }
    }
    // GAP x GAP planes whose first runs differ: every element differs, the reference's first form misses it
    svect g1, g2;
    g1.resize((typename svect::size_type)B); g2.resize((typename svect::size_type)B);
    for (uint64_t i = 0; i < B; ++i) { if (i < 1000) g1.set((typename svect::size_type)i, V(1)); else g2.set((typename svect::size_type)i, V(1)); }
    g1.optimize(); g2.optimize();
    std::snprintf(what, sizeof(what), "%s GAP first runs", tname);
    check_pair(ctx, g1, g2, what);
}

#ifdef BM64ADDR
// ---- BM64ADDR: two vectors of more than 2^32 elements with values on both sides of 2^32 (columns 65535 / 65536) ----
static void check_past_2_32(bm::b200::context& ctx)
{
    typedef bm::sparse_vector<uint32_t, bvect> svect;
    const uint64_t B = 65536u, G = uint64_t(1) << 32, n = G + 2 * B + 321;
    for (int nl = 0; nl < 2; ++nl) {
        svect a(nl ? bm::use_null : bm::no_null);
        a.resize((svect::size_type)n);
        for (uint64_t i = G - 3000; i < G + 3000; i += 7) a.set((svect::size_type)i, uint32_t(i % 1000));
        a.set((svect::size_type)(n - 1), 42u);
        a.optimize();
        svect b(a);
        b.set((svect::size_type)(G + 100), 5555u);
        b.optimize();
        check_pair(ctx, a, b, nl ? "past 2^32 nullable" : "past 2^32");
        svect::size_type pos = 0;                                    // the default null_proc (bm::use_null)
        CHECK(bm::b200::sparse_vector_find_first_mismatch(ctx, a, b, pos) && pos == G + 100, "past 2^32: first at %llu",
              (unsigned long long)pos);
    }
}
#endif

int main()
{
    std::mt19937_64 rng(20261018);
    bm::b200::context ctx(0);
#ifdef BM64ADDR
    check_past_2_32(ctx);
#endif
    run_type<uint32_t>(ctx, rng, "uint32_t");
    run_type<uint64_t>(ctx, rng, "uint64_t");
    run_type<int32_t>(ctx, rng, "int32_t");
    run_type<int64_t>(ctx, rng, "int64_t");
    std::printf("test_mismatch_binding: %d checks, %d failed (%d first-mismatch answers where the reference misses or postpones)\n",
                g_checks, g_fail, g_first_defects);
    return g_fail ? 1 : 0;
}
