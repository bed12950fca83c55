/*
 * test_rsc_binding.cpp -- TEST INFRASTRUCTURE.  Drop-in check of the rank-select compressed sparse vector path at the
 * bm::bvector<> level: the UNMODIFIED reference (bm::sparse_vector_scanner<rsc_sparse_vector<unsigned>>,
 * bm::rank_compressor<bvector<>>; headers from the reference tree) against bm::b200::scanner<rsc_sparse_vector<unsigned>> and
 * bm::b200::rank_compressor (bitmagic_b200/include/bmb200_scanner.hpp, which talks to libbmb200.so).
 * Parity criterion = the reference's own: compare() == 0 and equal count().  Built by oracle/rsc.mk into oracle/_ref/.
 */
#include <cstdio>
#include <cstdlib>
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
typedef bm::sparse_vector<unsigned, bvect> svect;
typedef bm::rsc_sparse_vector<unsigned, svect> rsc_vect;
static int g_fail = 0, g_checks = 0;
#define CHECK(cond, ...) do { ++g_checks; if (!(cond)) { ++g_fail; std::printf("FAIL %s:%d: ", __FILE__, __LINE__); std::printf(__VA_ARGS__); std::printf("\n"); } } while (0)

// a nullable vector of n elements: NOT-NULL runs (FULL and GAP blocks of NN), an iid region (BIT blocks), a NULL superblock gap
static void make_rsc(rsc_vect& rsc, std::mt19937_64& rng, uint64_t n, double nn_density, unsigned max_value)
{
    svect sv(bm::use_null);
    sv.resize((svect::size_type)n);
    std::uniform_real_distribution<double> u(0.0, 1.0);
    std::uniform_int_distribution<unsigned> val(0, max_value);
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t nb = i >> 16;
        bool nn;
        if (nb % 7 == 1) nn = true;                                  // FULL blocks of NN
        else if (nb % 7 == 3) nn = ((i >> 9) & 3u) == 0u;            // runs: a GAP block of NN
        else if (nb >= 260 && nb < 520) nn = false;                  // a NULL superblock
        else nn = u(rng) < nn_density;
        if (nn) sv.set((svect::size_type)i, val(rng));
    }
    BM_DECLARE_TEMP_BLOCK(tb)
    sv.optimize(tb);
    rsc.load_from(sv);
    rsc.sync();
}

template<class Fn>
static void each_pred(Fn fn)
{
    for (int pred = BMB200_SCAN_EQ; pred <= BMB200_SCAN_RANGE; ++pred) fn(pred);
}

static void ref_search(bm::sparse_vector_scanner<rsc_vect>& sc, const rsc_vect& v, int pred, unsigned a, unsigned b, bvect& out)
{
    switch (pred) {
    case BMB200_SCAN_EQ: sc.find_eq(v, a, out); break;
    case BMB200_SCAN_GT: sc.find_gt(v, a, out); break;
    case BMB200_SCAN_GE: sc.find_ge(v, a, out); break;
    case BMB200_SCAN_LT: sc.find_lt(v, a, out); break;
    case BMB200_SCAN_LE: sc.find_le(v, a, out); break;
    default: sc.find_range(v, a, b, out); break;
    }
}

static void gpu_search(bm::b200::scanner<rsc_vect>& sc, int pred, unsigned a, unsigned b, bvect& out)
{
    switch (pred) {
    case BMB200_SCAN_EQ: sc.find_eq(a, out); break;
    case BMB200_SCAN_GT: sc.find_gt(a, out); break;
    case BMB200_SCAN_GE: sc.find_ge(a, out); break;
    case BMB200_SCAN_LT: sc.find_lt(a, out); break;
    case BMB200_SCAN_LE: sc.find_le(a, out); break;
    default: sc.find_range(a, b, out); break;
    }
}

#ifdef BM64ADDR
// ---- BM64ADDR: an rsc vector whose logical size passes 2^32 (NOT-NULL elements around it), and rank compression where count(NN)
// passes 2^32, so compressed positions do too ----
static void check_past_2_32(bm::b200::context& ctx, std::mt19937_64& rng)
{
    const uint64_t B = 65536u, G = uint64_t(1) << 32;
    {
        svect sv(bm::use_null);
        sv.resize((svect::size_type)(G + 3 * B + 17));
        for (uint64_t i = G - 2 * B; i < G + 3 * B + 17; ++i) {
            const uint64_t nb = i >> 16;
            const bool nn = nb == 65535 ? true : nb == 65537 ? ((i >> 9) & 3u) == 0u : rng() % 3 == 0;
            if (nn) sv.set((svect::size_type)i, unsigned(rng() % 500));
        }
        for (uint64_t i = 0; i < 2000; ++i) sv.set((svect::size_type)(i * 5), unsigned(i % 40));
        { BM_DECLARE_TEMP_BLOCK(tb) sv.optimize(tb); }
        rsc_vect rsc;
        rsc.load_from(sv);
        rsc.sync();
        bm::sparse_vector_scanner<rsc_vect> ref_sc;
        bm::b200::scanner<rsc_vect> sc(ctx, rsc);
        const unsigned vals[][2] = {{0u, 0u}, {7u, 30u}, {250u, 100u}, {499u, 499u}, {500u, 600u}};
        each_pred([&](int pred) {
            for (const auto& v : vals) {
                bvect r, g;
                ref_search(ref_sc, rsc, pred, v[0], v[1], r);
                gpu_search(sc, pred, v[0], v[1], g);
                CHECK(r.compare(g) == 0 && r.count() == g.count(), "64: rsc size 2^32+3*65536+17 pred=%d value=%u/%u: count ref %llu gpu %llu",
                      pred, v[0], v[1], (unsigned long long)r.count(), (unsigned long long)g.count());
            }
        });
    }
    {   // index vector: 65537 FULL blocks (count 2^32 + 65536), then a bit-block, a GAP block and a sparse tail at block 69000
        bvect idx, src;
        idx.set_range(0, (bvect::size_type)(G + B - 1));
        for (uint64_t p = G + B; p < G + 2 * B; p += 1 + rng() % 5) idx.set_bit((bvect::size_type)p);
        for (uint64_t p = G + 2 * B + 7; p < G + 3 * B; p += 700 + rng() % 300) idx.set_range((bvect::size_type)p, (bvect::size_type)(p + 200));
        for (uint64_t k = 0; k < 50; ++k) idx.set_bit((bvect::size_type)(69000 * B + k * 977));
        { BM_DECLARE_TEMP_BLOCK(tb) idx.optimize(tb); }
        // source: a subset of idx in every kind of index block, on both sides of 2^32
        for (uint64_t p = 3; p < 2 * B; p += 1 + rng() % 400) src.set_bit((bvect::size_type)p);
        for (uint64_t p = G - 3 * B; p < G + B; p += 1 + rng() % 900) src.set_bit((bvect::size_type)p);
        src.set_bit((bvect::size_type)(G - 1)); src.set_bit((bvect::size_type)G);
        bvect in_idx; in_idx.set_range((bvect::size_type)(G + B), (bvect::size_type)(70000 * B - 1)); in_idx &= idx;
        for (bvect::enumerator en = in_idx.first(); en.valid(); ++en) if (rng() % 3 == 0) src.set_bit(*en);
        bm::rank_compressor<bvect> ref_rc;
        bm::b200::rank_compressor<bvect> rc(ctx);
        bvect rt, gt, rd, gd;
        ref_rc.compress(rt, idx, src); rc.compress(gt, idx, src);
        bvect::size_type last = 0;
        CHECK(rt.find_reverse(last) && uint64_t(last) >= G + B, "64: compressed positions pass 2^32 (last %llu)", (unsigned long long)last);
        CHECK(rt.compare(gt) == 0 && rt.count() == gt.count(), "64: compress, count(NN) > 2^32: count ref %llu gpu %llu",
              (unsigned long long)rt.count(), (unsigned long long)gt.count());
        ref_rc.decompress(rd, idx, rt); rc.decompress(gd, idx, rt);
        CHECK(rd.compare(gd) == 0 && rd.count() == gd.count() && rd.compare(src) == 0, "64: decompress, count(NN) > 2^32");
    }
}
#endif

int main()
{
    std::mt19937_64 rng(20261015);
    bm::b200::context ctx(0);
#ifdef BM64ADDR
    check_past_2_32(ctx, rng);
#endif
    struct Case { uint64_t n; double density; unsigned max_value; } cases[] = {
        {600u * 65536u + 4321u, 0.3, 1000u}, {3u * 65536u, 1.0, 70000u}, {100000u, 0.0, 5u}, {0u, 0.5, 9u}};
    for (const Case& cs : cases) {
        rsc_vect rsc;
        make_rsc(rsc, rng, cs.n, cs.density, cs.max_value);
        bm::sparse_vector_scanner<rsc_vect> ref_sc;
        bm::b200::scanner<rsc_vect> sc(ctx, rsc);
        const unsigned vals[][2] = {{0u, 0u}, {1u, 7u}, {cs.max_value / 2u, cs.max_value / 3u}, {cs.max_value, 0u}, {cs.max_value + 1u, cs.max_value + 9u}};
        each_pred([&](int pred) {
            for (const auto& v : vals) {
                bvect r, g;
                ref_search(ref_sc, rsc, pred, v[0], v[1], r);
                gpu_search(sc, pred, v[0], v[1], g);
                CHECK(r.compare(g) == 0 && r.count() == g.count(), "n=%llu pred=%d value=%u/%u: count ref %llu gpu %llu",
                      (unsigned long long)cs.n, pred, v[0], v[1], (unsigned long long)r.count(), (unsigned long long)g.count());
            }
            // batched and count-only forms
            std::vector<uint64_t> bv = pred == BMB200_SCAN_RANGE ? std::vector<uint64_t>{2, 40, 300, 10, 0, 0} : std::vector<uint64_t>{0, 3, 77, 999, 5};
            std::vector<bvect> outs; std::vector<bvect::size_type> counts;
            sc.find_batch(pred, bv, outs); sc.count_batch(pred, bv, counts);
            const size_t nv = outs.size();
            for (size_t k = 0; k < nv; ++k) {
                bvect r;
                if (pred == BMB200_SCAN_RANGE) ref_search(ref_sc, rsc, pred, (unsigned)bv[2 * k], (unsigned)bv[2 * k + 1], r);
                else ref_search(ref_sc, rsc, pred, (unsigned)bv[k], 0u, r);
                CHECK(r.compare(outs[k]) == 0 && r.count() == counts[k], "batch n=%llu pred=%d k=%zu", (unsigned long long)cs.n, pred, k);
            }
        });
        // rank compression on the vector's own NN: a subset of NN (decompressed search result) round-trips
        const bvect& nn = *rsc.get_null_bvector();
        bvect srcl;
        ref_search(ref_sc, rsc, BMB200_SCAN_LT, cs.max_value / 2u, 0u, srcl);
        bm::rank_compressor<bvect> ref_rc;
        bm::b200::rank_compressor<bvect> rc(ctx);
        bvect rt, gt, rd, gd;
        ref_rc.compress(rt, nn, srcl); rc.compress(gt, nn, srcl);
        CHECK(rt.compare(gt) == 0 && rt.count() == gt.count(), "compress n=%llu: count ref %llu gpu %llu",
              (unsigned long long)cs.n, (unsigned long long)rt.count(), (unsigned long long)gt.count());
        ref_rc.decompress(rd, nn, rt); rc.decompress(gd, nn, rt);
        CHECK(rd.compare(gd) == 0 && rd.count() == gd.count() && rd.compare(srcl) == 0, "decompress n=%llu", (unsigned long long)cs.n);
    }
    std::printf("test_rsc_binding: %d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
