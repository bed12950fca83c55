/*
 * test_remap_binding.cpp -- TEST INFRASTRUCTURE.  Drop-in check of the set image at the bm::bvector<> level: the UNMODIFIED
 * reference's bm::set2set_11_transform<SV>::remap / run (src/bmsparsevec_algo.h:1902-2205) against
 * bm::b200::set2set_11_transform on SV = bm::sparse_vector<bvector<>::size_type>, nullable and not, with ids past size(),
 * unassigned elements, explicit zeros, the value 0xffffffff, an empty vector, a pre-filled bv_out and attach_sv(sv, true).
 * Parity criterion: the binding's bv_out == the contract's image, built here from the reference's own sv.get() and NOT-NULL
 * vector over the ids of bv_in (compare() == 0, equal count()); and == the reference's remap wherever that equals the contract's
 * image.  The reference's remap departs from it on two kinds of input (DESIGN.md 3.5g), counted and reported, not failed:
 *   - the value bm::id_max: bvector::set(ids, n, BM_SORTED) stores it as bit 65535, so it can come back as the value 65535;
 *   - a non-nullable vector filled with set() around unassigned elements, under an input that holds part of its ids: values no
 *     id maps to appear, and values some id maps to are missing.
 * Built by oracle/remap.mk into oracle/_ref/ twice: as is and with -DBM64ADDR (then 0xffffffff is an ordinary value and a
 * vector with more than 32 planes must be refused with std::length_error).
 */
#include <cstdio>
#include <cstdint>
#include <random>
#include <stdexcept>
#include <vector>

#include "bm.h"
#include "bmsparsevec.h"
#include "bmsparsevec_algo.h"
#include "bmb200_aggregator.hpp"
#include "bmb200_scanner.hpp"

typedef bm::bvector<> bvect;
typedef bvect::size_type size_type;
typedef bm::sparse_vector<size_type, bvect> svect;
static int g_fail = 0, g_checks = 0;
#define CHECK(cond, ...) do { ++g_checks; if (!(cond)) { ++g_fail; std::printf("FAIL %s:%d: ", __FILE__, __LINE__); std::printf(__VA_ARGS__); std::printf("\n"); } } while (0)

static int g_ref_defects = 0;

// the contract's image: sv[i] for the ids i of bv_in (inside NOT-NULL when nullable; a plain vector maps ids past size() to 0),
// without bm::id_max; an empty vector has an empty image
static bvect contract_image(const svect& sv, const bvect& bv_in)
{
    bvect img;
    if (sv.empty()) return img;
    const bvect* nn = sv.get_null_bvector();
    for (bvect::enumerator en = bv_in.first(); en.valid(); ++en) {
        const size_type i = *en;
        if (nn && !nn->test(i)) continue;
        const size_type v = i < sv.size() ? sv.get(i) : size_type(0);
        if (v != size_type(bm::id_max)) img.set(v);
    }
    return img;
}

// every entry point of both sides on one (sv, bv_in), bv_out empty and pre-filled
static void compare(bm::b200::context& ctx, const svect& sv, const bvect& bv_in, const char* what)
{
    const bvect want = contract_image(sv, bv_in);
    for (int form = 0; form < 3; ++form) {
        for (int pre = 0; pre < 2; ++pre) {
            bvect ref_out, got;
            if (pre) { ref_out.set(5); ref_out.set(65536u * 3u + 1u); got = ref_out; }
            bm::set2set_11_transform<svect> ref;
            bm::b200::set2set_11_transform<svect> dev(ctx);
            if (form == 0) { ref.remap(bv_in, sv, ref_out); dev.remap(bv_in, sv, got); }
            else if (form == 1) { ref.run(bv_in, sv, ref_out); dev.run(bv_in, sv, got); }
            else { ref.attach_sv(&sv, true); ref.remap(bv_in, ref_out); dev.attach_sv(&sv, true); dev.remap(bv_in, got); }
            CHECK(want.compare(got) == 0 && want.count() == got.count(), "%s form %d prefilled %d: contract count %llu vs %llu", what,
                  form, pre, (unsigned long long)want.count(), (unsigned long long)got.count());
            if (ref_out.compare(want) == 0) {
                CHECK(ref_out.compare(got) == 0 && ref_out.count() == got.count(), "%s form %d prefilled %d: reference count %llu vs %llu",
                      what, form, pre, (unsigned long long)ref_out.count(), (unsigned long long)got.count());
            } else {
                ++g_ref_defects;
            }
        }
    }
}

static void build(svect& sv, std::mt19937_64& rng, uint64_t n, uint64_t range, double null_p, bool top)
{
    std::uniform_int_distribution<uint64_t> val(0, range - 1);
    std::uniform_real_distribution<double> u(0.0, 1.0);
    for (uint64_t i = 0; i < n; ++i) {
        if (null_p > 0 && u(rng) < null_p) continue;                      // NULL (nullable) / unassigned (plain)
        uint64_t x = ((i >> 16) % 3 == 1) ? ((i >> 12) & 1u ? 7u : 3u) : val(rng);   // runs: GAP / FULL planes
        if (top && i % 1009 == 0) x = 0xffffffffull;
        sv.set((size_type)i, (size_type)x);
    }
    BM_DECLARE_TEMP_BLOCK(tb)
    sv.optimize(tb);
}

static void ids(bvect& bv, std::mt19937_64& rng, uint64_t n, double density)
{
    std::uniform_real_distribution<double> u(0.0, 1.0);
    for (uint64_t i = 0; i < n; ++i) if (u(rng) < density) bv.set((size_type)i);
    bv.set_range((size_type)(n / 3), (size_type)(n / 3 + 70000));         // a FULL block inside
    bv.set((size_type)(n + 12345));                                       // past size()
    bv.optimize();
}

int main()
{
    std::mt19937_64 rng(20261019);
    bm::b200::context ctx(0);
    // the contract's example, plain and nullable with an explicit 9:0
    for (int nullable = 0; nullable < 2; ++nullable) {
        svect sv(nullable ? bm::use_null : bm::no_null);
        sv.set(2, 25); sv.set(3, 35); sv.set(7, 75); sv.set(256, 2001); sv.set(1000, 2000);
        if (nullable) sv.set(9, 0);
        bvect in; in.set(1); in.set(2); in.set(7); in.set(9); in.set(300); in.set(5000000);
        compare(ctx, sv, in, nullable ? "example nullable" : "example");
    }
    {
        svect empty; bvect in; in.set(4);
        compare(ctx, empty, in, "empty vector");
    }
    const uint64_t n = 65536u * 3u + 777u;
    const uint64_t ranges[] = {1u, 10u, 1000u, 1u << 20, 0xffffffffull};
    for (uint64_t range : ranges) {
        for (int nullable = 0; nullable < 2; ++nullable) {
            for (double dens : {0.001, 0.3, 1.0}) {
                svect sv(nullable ? bm::use_null : bm::no_null);
                build(sv, rng, n, range, 0.2, range == 0xffffffffull);
                bvect in; ids(in, rng, n, dens);
                char what[128];
                std::snprintf(what, sizeof what, "range %llu nullable %d density %g", (unsigned long long)range, nullable, dens);
                compare(ctx, sv, in, what);
            }
        }
    }
#ifdef BM64ADDR
    {
        svect wide; wide.set(3, (size_type)1 << 40);
        bm::b200::set2set_11_transform<svect> dev(ctx);
        bool thrown = false;
        try { dev.attach_sv(&wide); } catch (const std::length_error&) { thrown = true; }
        CHECK(thrown, "a vector with 41 planes must be refused");
    }
#endif
    std::printf("test_remap_binding: %d checks, %d failed (%d reference answers off the contract's image)\n", g_checks, g_fail,
                g_ref_defects);
    return g_fail ? 1 : 0;
}
