/*
 * test_float_binding.cpp -- TEST INFRASTRUCTURE.  Drop-in check of the float scanner at the bm::bvector<> level: the UNMODIFIED
 * reference's bm::sparse_vector_scanner<> (headers from the reference tree) against bm::b200::scanner<> (bitmagic_b200/include/
 * bmb200_scanner.hpp, which talks to libbmb200.so) on real bm::sparse_vector_float<sparse_vector<unsigned>> vectors, plain and
 * nullable: every public float search at special values (+-0, denormals, +-inf, NaNs with payloads), every ordered pair of them as
 * range bounds, the batched forms, the counts, a rebind and the empty vector.  Parity criterion = the reference's own:
 * compare() == 0 and equal count().  Built by oracle/float.mk into oracle/_ref/.
 *
 * On an EMPTY non-nullable vector the reference's find_ge_float / find_le_float / find_range_float, and find_gt_float at a
 * negative value, return every index of the 32-bit space (set_range(0, size() - 1) with size() == 0; count() then wraps to 0),
 * not a comparison (DESIGN.md 3.5d); there the binding is held to the empty answer.
 */
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <random>
#include <vector>

#include "bm.h"
#include "bmsparsevec.h"
#include "bmsparsevec_algo.h"
#include "bmsparsevec_float.h"
#include "bmb200_aggregator.hpp"
#include "bmb200_scanner.hpp"

typedef bm::bvector<> bvect;
typedef bm::sparse_vector<unsigned, bvect> svect_u32;
typedef bm::sparse_vector_float<svect_u32> svf_t;
static int g_fail = 0, g_checks = 0;
#define CHECK(cond, ...) do { ++g_checks; if (!(cond)) { ++g_fail; std::printf("FAIL %s:%d: ", __FILE__, __LINE__); std::printf(__VA_ARGS__); std::printf("\n"); } } while (0)

static float fl(uint32_t b) { float f; std::memcpy(&f, &b, sizeof f); return f; }
static uint32_t bits(float f) { uint32_t b; std::memcpy(&b, &f, sizeof b); return b; }

static const uint32_t kSpecials[] = {0x00000000u, 0x80000000u, 0x00000001u, 0x80000001u, 0x00800000u, 0x80800000u, 0x7F7FFFFFu,
                                     0xFF7FFFFFu, 0x7F800000u, 0xFF800000u, 0x7FC00000u, 0xFFC00000u, 0x7F800001u, 0xFF800001u};

// n elements: iid bit patterns with the specials sprinkled in (bit planes), long runs of two values (GAP / FULL planes), a sparse
// region of +0.0 left unassigned (GAP planes), NULLs (nullable only)
static void fill(svf_t& svf, std::mt19937_64& rng, uint64_t n, bool nullable)
{
    svf.exponents_.resize((svf_t::size_type)n);
    svf.mantissas_.resize((svf_t::size_type)n);
    std::uniform_real_distribution<double> u(0.0, 1.0);
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t nb = i >> 16;
        if (nullable && (nb % 4 == 2 || u(rng) < 0.3)) continue;
        uint32_t b;
        if (nb % 4 == 1) b = ((i >> 11) & 1u) ? bits(-2.5f) : bits(1.0f);
        else if (nb % 4 == 3) { if (u(rng) > 0.01) continue; b = (uint32_t)rng(); }
        else if (i % 331 == 0) b = kSpecials[(i / 331) % (sizeof(kSpecials) / sizeof(kSpecials[0]))];
        else b = (uint32_t)rng();
        svf.set((svf_t::size_type)i, fl(b));
    }
    BM_DECLARE_TEMP_BLOCK(tb)
    svf.optimize(tb);
}

static void ref_search(bm::sparse_vector_scanner<svf_t>& sc, const svf_t& v, int pred, float a, float b, bvect& out)
{
    switch (pred) {
    case BMB200_SCAN_GT: sc.find_gt_float(v, a, out); break;
    case BMB200_SCAN_GE: sc.find_ge_float(v, a, out); break;
    case BMB200_SCAN_LT: sc.find_lt_float(v, a, out); break;
    case BMB200_SCAN_LE: sc.find_le_float(v, a, out); break;
    case BMB200_SCAN_RANGE: sc.find_range_float(v, a, b, out); break;
    default: sc.find_range_float_unbounded(v, a, b, out); break;
    }
}

static void gpu_search(bm::b200::scanner<svf_t>& sc, int pred, float a, float b, bvect& out)
{
    switch (pred) {
    case BMB200_SCAN_GT: sc.find_gt_float(a, out); break;
    case BMB200_SCAN_GE: sc.find_ge_float(a, out); break;
    case BMB200_SCAN_LT: sc.find_lt_float(a, out); break;
    case BMB200_SCAN_LE: sc.find_le_float(a, out); break;
    case BMB200_SCAN_RANGE: sc.find_range_float(a, b, out); break;
    default: sc.find_range_float_unbounded(a, b, out); break;
    }
}

static void check_vector(bm::b200::context& ctx, bm::b200::scanner<svf_t>& sc, const svf_t& svf, const char* what)
{
    bm::sparse_vector_scanner<svf_t> ref_sc;
    std::vector<float> q;
    for (uint32_t b : kSpecials) q.push_back(fl(b));
    for (float f : {1.0f, -1.0f, -2.5f, 2.5f, 0.5f, -7.0f, 3e-39f, -3e-39f, 1e30f}) q.push_back(f);
    for (int pred = BMB200_SCAN_GT; pred <= BMB200_SCAN_RANGE_OPEN; ++pred) {
        const bool two = pred >= BMB200_SCAN_RANGE;
        std::vector<float> flat;
        for (size_t i = 0; i < q.size(); ++i)
            for (size_t j = 0; j < (two ? q.size() : 1); ++j) {
                const float a = q[i], b = two ? q[j] : 0.0f;
                bvect r, g;
                ref_search(ref_sc, svf, pred, a, b, r);
                if (!svf.size()) r.clear();                      // see the file comment
                gpu_search(sc, pred, a, b, g);
                CHECK(r.compare(g) == 0 && r.count() == g.count(), "%s pred=%d value=%08x/%08x: count ref %llu gpu %llu", what, pred,
                      bits(a), bits(b), (unsigned long long)r.count(), (unsigned long long)g.count());
                if ((i + j) % 5 == 0) { flat.push_back(a); if (two) flat.push_back(b); }
            }
        // batched and count-only forms: one launch over a subset of the searches above
        std::vector<bvect> outs; std::vector<bvect::size_type> counts;
        sc.find_batch(pred, flat, outs); sc.count_batch(pred, flat, counts);
        CHECK(outs.size() == (two ? flat.size() / 2 : flat.size()) && counts.size() == outs.size(), "%s batch sizes pred=%d", what, pred);
        for (size_t k = 0; k < outs.size(); ++k) {
            bvect r;
            if (two) ref_search(ref_sc, svf, pred, flat[2 * k], flat[2 * k + 1], r);
            else ref_search(ref_sc, svf, pred, flat[k], 0.0f, r);
            if (!svf.size()) r.clear();
            CHECK(r.compare(outs[k]) == 0 && r.count() == counts[k], "%s batch pred=%d k=%zu: count ref %llu gpu %llu / %llu", what, pred, k,
                  (unsigned long long)r.count(), (unsigned long long)outs[k].count(), (unsigned long long)counts[k]);
        }
    }
    (void)ctx;
}

int main()
{
    std::mt19937_64 rng(20261017);
    bm::b200::context ctx(0);
    const uint64_t sizes[] = {3u * 65536u + 77u, 70000u, 0u};
    char what[96];
    for (uint64_t n : sizes) {
        for (int nullable = 0; nullable < 2; ++nullable) {
            svf_t svf(nullable ? bm::use_null : bm::no_null);
            fill(svf, rng, n, nullable != 0);
            std::snprintf(what, sizeof(what), "n=%llu nullable=%d", (unsigned long long)n, nullable);
            bm::b200::scanner<svf_t> sc(ctx, svf);
            check_vector(ctx, sc, svf, what);
            // rebind the same scanner to another vector
            svf_t other(nullable ? bm::use_null : bm::no_null);
            fill(other, rng, n / 2 + 5, nullable != 0);
            sc.bind(other);
            std::snprintf(what, sizeof(what), "rebound n=%llu nullable=%d", (unsigned long long)(n / 2 + 5), nullable);
            check_vector(ctx, sc, other, what);
        }
    }
    std::printf("test_float_binding: %d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
