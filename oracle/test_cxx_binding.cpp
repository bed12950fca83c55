/*
 * test_cxx_binding.cpp -- TEST INFRASTRUCTURE.  Drop-in check at the bm::bvector<> level:
 * the UNMODIFIED reference (bm::aggregator, bvector::build_rs_index; headers from /root/reference/src)
 * against bm::b200::aggregator / bm::b200::build_rs_index (bitmagic_b200/include/bmb200_aggregator.hpp,
 * which talks to libbmb200.so).  Parity criterion = the reference's own: compare()==0, equal count(),
 * equal calc_stat block kinds under opt_compress, equal rs_index fields and query answers
 * (tests/stress/t.cpp:10887-10921, :2658-2885, :4975-5090).  Built by oracle/Makefile into oracle/_ref/.
 */
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>
#include <memory>

#include "bm.h"
#include "bmaggregator.h"
#include "bmserial.h"
#include "bmb200_aggregator.hpp"
#include "bmb200_scanner.hpp"

typedef bm::bvector<> bvect;
static int g_fail = 0, g_checks = 0;
#define CHECK(cond, ...) do { ++g_checks; if (!(cond)) { ++g_fail; std::printf("FAIL %s:%d: ", __FILE__, __LINE__); std::printf(__VA_ARGS__); std::printf("\n"); } } while (0)

static void fill(bvect& bv, std::mt19937_64& rng, unsigned n_bits, double density, bool ranges)
{
    std::geometric_distribution<unsigned> skip(density);
    for (uint64_t p = skip(rng); p < n_bits; p += 1 + skip(rng)) bv.set_bit_no_check((bvect::size_type)p);
    if (ranges) {
        bv.set_range(70000, 70000 + 200000);            // spans whole blocks -> FULL blocks after optimize
        bv.set_range(n_bits / 2, n_bits / 2 + 300);
    }
}

#ifdef BM64ADDR
// ---- BM64ADDR: vectors past 2^32 bits.  Their blocks straddle columns 65535 / 65536 (bit 2^32) and reach block 69999, so every
// upload holds ~70 000 columns; a default-constructed vector is 2^48 - 1 bits long, which the binding must not upload whole ----
static const uint64_t B = 65536u, G = uint64_t(1) << 32;

// shape 0: random bits in a few block spans; 1: plus a run of FULL blocks across 2^32; 2: plus the two bits around 2^32;
// 3: GAP-friendly runs only
static void fill64(bvect& bv, std::mt19937_64& rng, double density, int shape)
{
    const uint64_t spans[][2] = {{0, 2}, {65531, 65541}, {66600, 66601}, {69996, 70000}};
    std::geometric_distribution<unsigned> skip(density);
    if (shape != 3)
        for (const auto& s : spans)
            for (uint64_t p = s[0] * B + skip(rng); p < s[1] * B; p += 1 + skip(rng)) bv.set_bit_no_check((bvect::size_type)p);
    if (shape == 1) bv.set_range(G - 3 * B - 77, G + 2 * B + 500);
    if (shape == 2) { bv.set_bit(G - 1); bv.set_bit(G); bv.set_bit(70000 * B - 1); }
    if (shape == 3)
        for (uint64_t p = 65533 * B + 11; p < 65540 * B; p += 4099 + (rng() % 2000)) bv.set_range(p, p + (rng() % 300));
}

static bool same_kinds(const bvect& a, const bvect& b)
{
    bvect::statistics s1, s2; a.calc_stat(&s1); b.calc_stat(&s2);
    return s1.bit_blocks == s2.bit_blocks && s1.gap_blocks == s2.gap_blocks;
}

static void check_past_2_32(bm::b200::context& ctx, std::mt19937_64& rng)
{
    std::vector<std::unique_ptr<bvect>> vs;
    for (int k = 0; k < 10; ++k) {
        vs.emplace_back(new bvect());
        fill64(*vs.back(), rng, k < 6 ? 0.6 / (k + 1) : 0.02, k % 4);
        if (k >= 4) { BM_DECLARE_TEMP_BLOCK(tb) vs.back()->optimize(tb, bvect::opt_compress); }
    }
    std::vector<const bvect*> all; for (auto& v : vs) all.push_back(v.get());
    for (int opt = 0; opt < 2; ++opt) {
        const bvect::optmode om = opt ? bvect::opt_compress : bvect::opt_none;
        bm::aggregator<bvect> ref; ref.set_optimization(om);
        bm::b200::aggregator<bvect> gpu(ctx); gpu.set_optimization(om);
        for (size_t n : {size_t(2), size_t(5), all.size()}) {
            bvect r, g;
            ref.combine_or(r, all.data(), n); gpu.combine_or(g, all.data(), n);
            CHECK(r.compare(g) == 0 && r.count() == g.count() && (!opt || same_kinds(r, g)), "64: combine_or n=%zu opt=%d (%llu vs %llu bits)",
                  n, opt, (unsigned long long)r.count(), (unsigned long long)g.count());
            ref.combine_and(r, all.data(), n); gpu.combine_and(g, all.data(), n);
            CHECK(r.compare(g) == 0 && r.count() == g.count(), "64: combine_and n=%zu opt=%d", n, opt);
        }
        for (size_t na : {size_t(1), size_t(2)}) {
            bvect r, g;
            bool f1 = ref.combine_and_sub(r, all.data(), na, all.data() + na, all.size() - na, false);
            bool f2 = gpu.combine_and_sub(g, all.data(), na, all.data() + na, all.size() - na, false);
            CHECK(f1 == f2 && r.compare(g) == 0 && r.count() == g.count() && same_kinds(r, g), "64: combine_and_sub na=%zu opt=%d", na, opt);
            CHECK(gpu.count_and_sub(all.data(), na, all.data() + na, all.size() - na) == r.count(), "64: count_and_sub na=%zu", na);
        }
        for (size_t n : {size_t(1), size_t(2), size_t(3)}) {     // dense sources: the carry crosses column 65535 -> 65536
            const bvect* sh[3] = {all[1], all[0], all[2]};
            bvect r, g;
            bool f1 = ref.combine_shift_right_and(r, sh, n, false), f2 = gpu.combine_shift_right_and(g, sh, n, false);
            CHECK(f1 == f2 && r.compare(g) == 0 && r.count() == g.count(), "64: combine_shift_right_and n=%zu opt=%d (%llu vs %llu bits)",
                  n, opt, (unsigned long long)r.count(), (unsigned long long)g.count());
        }
    }
    {   // find_first_and_sub: answers past 2^32, with and without range hints above 2^32, uploaded and resident
        bvect a1, a2, s1;
        a1.set_range(G + 5 * B + 100, G + 5 * B + 4000); a1.set_range(G - 20, G + 10); a1.set_bit(3 * B);
        a2.set_range(G + 5 * B + 300, G + 6 * B); a2.set_range(G - 5, G + 3);
        s1.set_range(G - 30, G - 1); s1.set_bit(3 * B);
        bm::b200::device_set<bvect> ds(ctx);
        std::vector<const bvect*> mem = {&a1, &a2, &s1, all[0], all[1], all[2]};
        ds.assign(mem.data(), mem.size());
        std::vector<std::vector<const bvect*>> ands = {{&a1, &a2}, {all[0], all[1]}, {all[2]}};
        std::vector<std::vector<const bvect*>> subs = {{}, {&s1}, {all[2]}};
        struct Hint { bool on; uint64_t from, to; };
        const Hint hints[] = {{false, 0, 0}, {true, G - 3 * B, G + 9 * B}, {true, G + 1, G + 2 * B + 17}, {true, G + 5 * B + 250, G + 5 * B + 3999},
                              {true, G + 5 * B + 4001, G + 5 * B + 9000}, {true, 65535 * B + 5, 65535 * B + 65535}, {true, 69990 * B, 70000 * B - 1}};
        bm::aggregator<bvect> ref; bm::b200::aggregator<bvect> gpu(ctx);
        for (int resident = 0; resident < 2; ++resident) {
            gpu.set_device_set(resident ? &ds : nullptr);
            for (const Hint& h : hints)
                for (size_t x = 0; x < ands.size(); ++x) for (size_t y = 0; y < subs.size(); ++y) {
                    ref.reset_range_hint(); gpu.reset_range_hint();
                    if (h.on) { bool r1 = ref.set_range_hint(h.from, h.to), r2 = gpu.set_range_hint(h.from, h.to); CHECK(r1 == r2, "64: set_range_hint return"); }
                    bvect::size_type i1 = 0, i2 = 0;
                    bool f1 = ref.find_first_and_sub(i1, ands[x].data(), ands[x].size(), subs[y].empty() ? 0 : subs[y].data(), subs[y].size());
                    bool f2 = gpu.find_first_and_sub(i2, ands[x].data(), ands[x].size(), subs[y].empty() ? 0 : subs[y].data(), subs[y].size());
                    CHECK(f1 == f2 && (!f1 || i1 == i2), "64: find_first_and_sub and=%zu sub=%zu hint=[%llu,%llu] resident=%d: ref %d@%llu vs %d@%llu",
                          x, y, (unsigned long long)h.from, (unsigned long long)h.to, resident, (int)f1, (unsigned long long)i1, (int)f2, (unsigned long long)i2);
                }
        }
        bvect::size_type i1 = 0, i2 = 0;
        ref.reset_range_hint(); gpu.reset_range_hint(); gpu.set_device_set(nullptr);
        const bvect* aa[2] = {&a1, &a2};
        bool f1 = ref.find_first_and_sub(i1, aa, 2, 0, 0), f2 = gpu.find_first_and_sub(i2, aa, 2, 0, 0);
        CHECK(f1 && f2 && i1 == i2 && i2 == G - 5, "64: find_first_and_sub straddling 2^32: %llu", (unsigned long long)i2);
    }
    {   // 3-operand ops, bits and block kinds
        std::vector<const bvect*> ops = {all[0], all[1], all[3], all[5], all[6], all[7]};
        for (int opt = 0; opt < 2; ++opt) {
            const bvect::optmode om = opt ? bvect::opt_compress : bvect::opt_none;
            for (size_t x = 0; x < ops.size(); ++x) for (size_t y = 0; y < ops.size(); ++y) {
                if (x == y) continue;
                for (int op = 0; op < 4; ++op) {
                    bvect t1, t2;
                    switch (op) {
                    case 0: t1.bit_and(*ops[x], *ops[y], om); bm::b200::bit_and(ctx, t2, *ops[x], *ops[y], om); break;
                    case 1: t1.bit_or (*ops[x], *ops[y], om); bm::b200::bit_or (ctx, t2, *ops[x], *ops[y], om); break;
                    case 2: t1.bit_sub(*ops[x], *ops[y], om); bm::b200::bit_sub(ctx, t2, *ops[x], *ops[y], om); break;
                    default: t1.bit_xor(*ops[x], *ops[y], om); bm::b200::bit_xor(ctx, t2, *ops[x], *ops[y], om); break;
                    }
                    CHECK(t1.compare(t2) == 0 && t1.count() == t2.count() && same_kinds(t1, t2), "64: binop %d (%zu,%zu) opt=%d", op, x, y, opt);
                }
            }
        }
    }
    {   // pipeline with an OR target
        bm::aggregator<bvect> ref; bm::b200::aggregator<bvect> gpu(ctx);
        bm::aggregator<bvect>::pipeline<bm::agg_opt_bvect_and_counts> rp;
        bm::b200::pipeline<bvect> gp(ctx);
        bvect or_ref, or_gpu; or_ref.init(); or_gpu.init();
        rp.set_or_target(&or_ref); gp.set_or_target(&or_gpu);
        for (int g = 0; g < 6; ++g) {
            auto* a1 = rp.add(); auto* a2 = gp.add();
            for (int k = 0; k < 1 + g % 2; ++k) { a1->add(all[(g + k) % 10], 0); a2->add(all[(g + k) % 10], 0); }
            for (int k = 0; k < g % 3; ++k) { a1->add(all[(g * 3 + k + 4) % 10], 1); a2->add(all[(g * 3 + k + 4) % 10], 1); }
        }
        rp.complete(); gp.complete();
        ref.combine_and_sub(rp); gpu.combine_and_sub(gp);
        auto& r1 = rp.get_bv_res_vector(); auto& c1 = rp.get_bv_count_vector();
        auto& r2 = gp.get_bv_res_vector(); auto& c2 = gp.get_bv_count_vector();
        CHECK(r1.size() == r2.size() && c1.size() == c2.size(), "64: pipeline sizes");
        for (size_t g = 0; g < r2.size() && g < r1.size(); ++g) {
            CHECK((uint64_t)c1[g] == (uint64_t)c2[g] && (r1[g] == 0) == (r2[g] == 0) && (!r1[g] || !r2[g] || r1[g]->compare(*r2[g]) == 0), "64: pipeline g=%zu", g);
        }
        CHECK(or_ref.compare(or_gpu) == 0, "64: pipeline OR target");
    }
    {   // resident device_set, and a shard of columns [65530, 65540) around 2^32
        bm::b200::device_set<bvect> ds(ctx);
        ds.assign(all.data(), all.size());
        CHECK(ds.n_blocks() == 70000u, "64: device_set columns %u (want 70000)", ds.n_blocks());
        bm::aggregator<bvect> ref; ref.set_optimization(bvect::opt_compress);
        bm::b200::aggregator<bvect> gpu(ctx); gpu.set_optimization(bvect::opt_compress); gpu.set_device_set(&ds);
        bvect r, g;
        ref.combine_or(r, all.data(), all.size()); gpu.combine_or(g, all.data(), all.size());
        CHECK(r.compare(g) == 0 && same_kinds(r, g), "64: resident combine_or");
        bool f1 = ref.combine_and_sub(r, all.data(), 2, all.data() + 2, all.size() - 2, false);
        bool f2 = gpu.combine_and_sub(g, all.data(), 2, all.data() + 2, all.size() - 2, false);
        CHECK(f1 == f2 && r.compare(g) == 0, "64: resident combine_and_sub");
        bm::b200::device_set<bvect> sh(ctx);
        sh.assign(all.data(), all.size(), 65530, 65540);
        bm::b200::aggregator<bvect> g2(ctx); g2.set_optimization(bvect::opt_compress); g2.set_device_set(&sh);
        ref.combine_or(r, all.data(), all.size()); g2.combine_or(g, all.data(), all.size());
        bvect mask; mask.set_range(65530 * B, 65540 * B - 1);
        r &= mask;
        CHECK(r.compare(g) == 0 && r.count() == g.count(), "64: shard [65530,65540)");
    }
    // rs_index built on the GPU, queried by the reference's count_to / select past 2^32
    for (int k : {0, 1, 2, 7}) {
        const bvect& bv = *all[k];
        bvect::rs_index_type rs_ref, rs_gpu;
        bv.build_rs_index(&rs_ref);
        bm::b200::build_rs_index(ctx, bv, &rs_gpu);
        CHECK(rs_ref.count() == rs_gpu.count(), "64: rs count k=%d", k);
        bool q = true;
        const uint64_t fixed[] = {0, G - 1, G, G + 1, 65536 * B + 65535, 66600 * B + 3, 70000 * B - 1, 70000 * B, 80000 * B};
        for (int i = 0; i < 20000; ++i) {
            bvect::size_type p = i < 9 ? (bvect::size_type)fixed[i] : (bvect::size_type)(i % 2 ? G - 6 * B + rng() % (12 * B) : rng() % (70000 * B));
            q &= bv.count_to(p, rs_gpu) == bv.count_to(p, rs_ref);
            bvect::size_type r = (bvect::size_type)(rng() % (rs_ref.count() + 2)), p1 = 0, p2 = 0;
            bool f1 = bv.select(r, p1, rs_ref), f2 = bv.select(r, p2, rs_gpu);
            q &= (f1 == f2) && (!f1 || p1 == p2);
        }
        CHECK(q, "64: rank/select with the GPU-built index k=%d", k);
    }
    // sparse_vector<unsigned> of more than 2^32 elements: values around 2^32, plain (universe [0, size)) and nullable
    for (int nullable = 0; nullable < 2; ++nullable) {
        typedef bm::sparse_vector<unsigned, bvect> svect;
        svect sv(nullable ? bm::use_null : bm::no_null);
        sv.resize((svect::size_type)(G + 2 * B + 99));
        for (uint64_t i = G - 2 * B + 5; i < G + 2 * B + 99; ++i) {
            if (nullable && rng() % 7 == 0) continue;
            unsigned v = rng() % 3 == 0 ? 0u : unsigned(rng() % 900);
            if (i >= G - 300 && i < G + 700) v = 55;
            sv.set((svect::size_type)i, v);
        }
        for (uint64_t i = 0; i < 3000; ++i) sv.set((svect::size_type)(i * 7), unsigned(i % 60));
        { BM_DECLARE_TEMP_BLOCK(tb) sv.optimize(tb); }
        bm::sparse_vector_scanner<svect> ref_sc;
        bm::b200::scanner<svect> gpu_sc(ctx, sv);
        for (unsigned v : {0u, 55u, 899u, 1000u}) {
            bvect a, b;
            ref_sc.find_eq(sv, v, a); gpu_sc.find_eq(v, b); CHECK(a.compare(b) == 0 && a.count() == b.count(), "64: scanner find_eq(%u) nullable=%d", v, nullable);
            ref_sc.find_gt(sv, v, a); gpu_sc.find_gt(v, b); CHECK(a.compare(b) == 0, "64: scanner find_gt(%u) nullable=%d", v, nullable);
            ref_sc.find_le(sv, v, a); gpu_sc.find_le(v, b); CHECK(a.compare(b) == 0 && a.count() == b.count(), "64: scanner find_le(%u) nullable=%d", v, nullable);
            ref_sc.find_range(sv, v / 2, v, a); gpu_sc.find_range(v / 2, v, b); CHECK(a.compare(b) == 0, "64: scanner find_range(%u) nullable=%d", v, nullable);
        }
        std::vector<uint64_t> vals = {7, 55, 0};
        std::vector<bvect> outs; std::vector<bvect::size_type> cnts;
        gpu_sc.find_batch(BMB200_SCAN_EQ, vals, outs); gpu_sc.count_batch(BMB200_SCAN_EQ, vals, cnts);
        for (size_t k = 0; k < vals.size(); ++k) {
            bvect a; ref_sc.find_eq(sv, (unsigned)vals[k], a);
            CHECK(a.compare(outs[k]) == 0 && a.count() == cnts[k], "64: scanner batch eq k=%zu nullable=%d", k, nullable);
        }
    }
    // serialization BLOBs of these vectors (64-bit stream headers, blocks past 65535), decoded and aggregated on the GPU
    for (unsigned level : {2u, 6u}) {
        std::vector<bm::serializer<bvect>::buffer> bufs(all.size());
        for (size_t k = 0; k < all.size(); ++k) { bm::serializer<bvect> ser; ser.set_compression_level(level); ser.serialize(*all[k], bufs[k]); }
        bm::aggregator<bvect> ref; ref.set_optimization(bvect::opt_compress);
        // the sources' own size (2^48 - 1: default vectors) and the bound of their bits, which a BLOB reader has to be told
        bm::b200::blob_aggregator<bvect> gpu(ctx, all[0]->size(), (bvect::size_type)(70000 * B)); gpu.set_optimization(bvect::opt_compress);
        for (size_t k = 0; k < all.size(); ++k) gpu.add(bufs[k].data(), bufs[k].size(), k < 2 ? 0 : 1);
        bvect r, g;
        bool f1 = ref.combine_and_sub(r, all.data(), 2, all.data() + 2, all.size() - 2, false), f2 = gpu.combine_and_sub(g);
        CHECK(f1 == f2 && r.compare(g) == 0 && r.count() == g.count(), "64: blob combine_and_sub level=%u", level);
        gpu.reset();
        for (size_t k = 0; k < all.size(); ++k) gpu.add(bufs[k].data(), bufs[k].size());
        ref.combine_or(r, all.data(), all.size()); gpu.combine_or(g);
        CHECK(r.compare(g) == 0 && r.count() == g.count() && r.size() == g.size(), "64: blob combine_or level=%u", level);
    }
    {   // without an extent, a default vector's size needs 2^32 columns: refused, not truncated to 0
        bool refused = false;
        try { bm::b200::blob_aggregator<bvect> gpu(ctx, bvect().size()); } catch (const std::length_error&) { refused = true; }
        CHECK(refused, "64: blob_aggregator of size 2^48 - 1 without an extent");
    }
    bmb200_ctx_trim(ctx.get());
}
#endif

int main()
{
    std::mt19937_64 rng(20260923);
    const unsigned n_bits = 40u * 65536u + 12345u;
    bm::b200::context ctx(0);
    std::vector<std::unique_ptr<bvect>> vs;
    for (int k = 0; k < 24; ++k) {
        vs.emplace_back(new bvect());
        fill(*vs.back(), rng, n_bits, 0.4 / (k + 1), k % 5 == 3);
        if (k >= 6) { BM_DECLARE_TEMP_BLOCK(tb) vs.back()->optimize(tb, bvect::opt_compress); }
    }
    std::vector<const bvect*> all; for (auto& v : vs) all.push_back(v.get());

    for (int opt = 0; opt < 2; ++opt) {
        bvect::optmode om = opt ? bvect::opt_compress : bvect::opt_none;
        bm::aggregator<bvect> ref; ref.set_optimization(om);
        bm::b200::aggregator<bvect> gpu(ctx); gpu.set_optimization(om);
        for (size_t n : {size_t(1), size_t(2), size_t(7), all.size()}) {
            bvect t_ref, t_gpu;
            ref.combine_or(t_ref, all.data(), n); gpu.combine_or(t_gpu, all.data(), n);
            CHECK(t_ref.compare(t_gpu) == 0, "combine_or n=%zu opt=%d", n, opt);
            CHECK(t_ref.count() == t_gpu.count(), "combine_or count n=%zu", n);
            if (opt) { bvect::statistics s1, s2; t_ref.calc_stat(&s1); t_gpu.calc_stat(&s2);
                       CHECK(s1.bit_blocks == s2.bit_blocks && s1.gap_blocks == s2.gap_blocks, "combine_or kinds n=%zu (%zu/%zu vs %zu/%zu)", n, (size_t)s1.bit_blocks, (size_t)s1.gap_blocks, (size_t)s2.bit_blocks, (size_t)s2.gap_blocks); }
            ref.combine_and(t_ref, all.data(), n); gpu.combine_and(t_gpu, all.data(), n);
            CHECK(t_ref.compare(t_gpu) == 0, "combine_and n=%zu opt=%d", n, opt);
        }
        for (size_t na : {size_t(1), size_t(2), size_t(3)}) {
            bvect t_ref, t_gpu;
            bool f1 = ref.combine_and_sub(t_ref, all.data(), na, all.data() + na, all.size() - na, false);
            bool f2 = gpu.combine_and_sub(t_gpu, all.data(), na, all.data() + na, all.size() - na, false);
            CHECK(f1 == f2, "combine_and_sub found na=%zu", na);
            CHECK(t_ref.compare(t_gpu) == 0, "combine_and_sub na=%zu", na);
            bvect::statistics s1, s2; t_ref.calc_stat(&s1); t_gpu.calc_stat(&s2);
            CHECK(s1.bit_blocks == s2.bit_blocks && s1.gap_blocks == s2.gap_blocks, "combine_and_sub kinds na=%zu", na);
            CHECK(gpu.count_and_sub(all.data(), na, all.data() + na, all.size() - na) == t_ref.count(), "count_and_sub na=%zu", na);
        }
    }
    {   // residency: bm::b200::device_set uploaded once, then every call whose sources are members runs on the device copy
        bm::b200::device_set<bvect> ds(ctx);
        ds.assign(all.data(), all.size());
        CHECK(ds.resident() && ds.size() == all.size() && !ds.stale(), "device_set assign");
        CHECK(ds.index_of(all[5]) == 5 && ds.index_of(nullptr) < 0, "device_set index_of");
        bm::aggregator<bvect> ref; ref.set_optimization(bvect::opt_compress);
        bm::b200::aggregator<bvect> gpu(ctx); gpu.set_optimization(bvect::opt_compress); gpu.set_device_set(&ds);
        for (int rep = 0; rep < 3; ++rep) {                   // repeated calls recycle the result buffers
            for (size_t n : {size_t(2), size_t(9), all.size()}) {
                bvect t_ref, t_gpu;
                ref.combine_or(t_ref, all.data() + rep, n - rep); gpu.combine_or(t_gpu, all.data() + rep, n - rep);
                CHECK(t_ref.compare(t_gpu) == 0 && t_ref.count() == t_gpu.count(), "resident combine_or n=%zu rep=%d", n, rep);
                bvect::statistics s1, s2; t_ref.calc_stat(&s1); t_gpu.calc_stat(&s2);
                CHECK(s1.bit_blocks == s2.bit_blocks && s1.gap_blocks == s2.gap_blocks, "resident combine_or kinds n=%zu", n);
            }
            bvect t_ref, t_gpu;
            bool f1 = ref.combine_and_sub(t_ref, all.data(), 2, all.data() + 2 + rep, all.size() - 2 - rep, false);
            bool f2 = gpu.combine_and_sub(t_gpu, all.data(), 2, all.data() + 2 + rep, all.size() - 2 - rep, false);
            CHECK(f1 == f2 && t_ref.compare(t_gpu) == 0, "resident combine_and_sub rep=%d", rep);
            CHECK(gpu.count_and_sub(all.data(), 2, all.data() + 2, all.size() - 2) == [&]{ bvect t; ref.combine_and_sub(t, all.data(), 2, all.data() + 2, all.size() - 2, false); return t.count(); }(), "resident count_and_sub");
        }
        {   // a source that is NOT a member: the call falls back to its own upload, same answer
            bvect extra; fill(extra, rng, n_bits, 0.01, false);
            const bvect* mix[3] = {all[0], &extra, all[7]};
            bvect t_ref, t_gpu; ref.combine_or(t_ref, mix, 3); gpu.combine_or(t_gpu, mix, 3);
            CHECK(t_ref.compare(t_gpu) == 0, "non-member source falls back to upload");
        }
        {   // a shard of the block range: result holds those blocks only (what one rank of a sharded aggregation sees)
            bm::b200::device_set<bvect> sh(ctx);
            sh.assign(all.data(), all.size(), 10, 30);
            bm::b200::aggregator<bvect> g2(ctx); g2.set_optimization(bvect::opt_compress); g2.set_device_set(&sh);
            bvect t_ref, t_gpu; ref.combine_or(t_ref, all.data(), all.size()); g2.combine_or(t_gpu, all.data(), all.size());
            bvect mask; mask.set_range(10u * 65536u, 30u * 65536u - 1u);
            t_ref &= mask;
            CHECK(t_ref.compare(t_gpu) == 0, "shard [10,30): result restricted to the shard's blocks");
        }
        vs[3]->resize(n_bits + 70000);                        // the O(1) stamp notices a resize
        CHECK(ds.stale(), "device_set stale() after resize");
        vs[3]->resize(n_bits);
    }
    {   // bvectors on the page-locked slab allocator (bmb200_alloc.hpp): >= 64 sources go up by slab DMA + device gather
        typedef bm::b200::slab_bvector sbv;
        std::vector<std::unique_ptr<sbv>> ss; std::vector<const sbv*> sp;
        std::mt19937_64 r2(777);
        for (int k = 0; k < 80; ++k) {
            ss.emplace_back(new sbv());
            std::geometric_distribution<unsigned> skip(0.3 / (k + 1));
            for (uint64_t p = skip(r2); p < n_bits; p += 1 + skip(r2)) ss.back()->set_bit_no_check((sbv::size_type)p);
            if (k % 5 == 3) ss.back()->set_range(70000, 270000);
            if (k >= 10) { BM_DECLARE_TEMP_BLOCK(tb) ss.back()->optimize(tb, sbv::opt_compress); }
            sp.push_back(ss.back().get());
        }
        CHECK(bm::b200::slab_heap::instance().slab_count() >= 1, "slab heap in use");
        bm::aggregator<sbv> ref; ref.set_optimization(sbv::opt_compress);
        bm::b200::aggregator<sbv> gpu(ctx); gpu.set_optimization(sbv::opt_compress);
        {   // cold calls: every call uploads (80 sources: slab road; 9 sources: packing road)
            for (size_t n : {size_t(9), sp.size()}) {
                sbv t_ref, t_gpu; ref.combine_or(t_ref, sp.data(), n); gpu.combine_or(t_gpu, sp.data(), n);
                CHECK(t_ref.compare(t_gpu) == 0 && t_ref.count() == t_gpu.count(), "slab_bvector cold combine_or n=%zu", n);
            }
            sbv t_ref, t_gpu;
            bool f1 = ref.combine_and_sub(t_ref, sp.data(), 2, sp.data() + 2, sp.size() - 2, false);
            bool f2 = gpu.combine_and_sub(t_gpu, sp.data(), 2, sp.data() + 2, sp.size() - 2, false);
            CHECK(f1 == f2 && t_ref.compare(t_gpu) == 0, "slab_bvector cold combine_and_sub");
        }
        bm::b200::device_set<sbv> ds(ctx);
        ds.assign(sp.data(), sp.size());
        gpu.set_device_set(&ds);
        for (int rep = 0; rep < 2; ++rep) {
            sbv t_ref, t_gpu;
            ref.combine_or(t_ref, sp.data() + rep, sp.size() - rep); gpu.combine_or(t_gpu, sp.data() + rep, sp.size() - rep);
            CHECK(t_ref.compare(t_gpu) == 0, "slab_bvector resident combine_or rep=%d", rep);
            sbv::statistics s1, s2; t_ref.calc_stat(&s1); t_gpu.calc_stat(&s2);
            CHECK(s1.bit_blocks == s2.bit_blocks && s1.gap_blocks == s2.gap_blocks, "slab_bvector resident kinds rep=%d", rep);
            bool f1 = ref.combine_and_sub(t_ref, sp.data(), 3, sp.data() + 3 + rep, sp.size() - 3 - rep, false);
            bool f2 = gpu.combine_and_sub(t_gpu, sp.data(), 3, sp.data() + 3 + rep, sp.size() - 3 - rep, false);
            CHECK(f1 == f2 && t_ref.compare(t_gpu) == 0, "slab_bvector resident combine_and_sub rep=%d", rep);
        }
        ds.release();
        bmb200_ctx_trim(ctx.get());
    }
    {   // find_first_and_sub + set_range_hint (src/bmaggregator.h:961-994, 1457-1549): same index / same "found" as the reference,
        // without a hint, with a multi-block hint (block range only) and with a one-block hint (block masked by the range)
        bm::aggregator<bvect> ref; bm::b200::aggregator<bvect> gpu(ctx);
        bm::b200::device_set<bvect> ds(ctx); ds.assign(all.data(), all.size());
        bvect lone_a, lone_b, lone_s;                        // sparse trees: hits far from bit 0, SUB group with a short extent
        // (no block where EVERY AND source is FULL and the SUB group is empty: there the reference returns ~0 as digest without writing
        //  its temp block, src/bmaggregator.h:1752-1759, and find_first_and_sub then reads the first bit of a stale block)
        lone_a.set_range(5u * 65536u + 100u, 5u * 65536u + 4000u); lone_a.set_range(30u * 65536u + 10u, 30u * 65536u + 70000u);
        lone_b.set_range(5u * 65536u + 300u, 31u * 65536u); lone_s.set_range(5u * 65536u, 5u * 65536u + 999u); lone_s.set_bit(2u * 65536u + 7u);
        std::vector<std::vector<const bvect*>> ands = {{all[0], all[1]}, {all[0], all[1], all[2], all[3]}, {all[7]}, {all[20], all[21]}, {&lone_a, &lone_b}};
        std::vector<std::vector<const bvect*>> subs = {{}, {all[4]}, {all[5], all[9], all[13]}, {&lone_s}, {all[0]}};
        struct Hint { bool on; unsigned from, to; };
        const Hint hints[] = {{false, 0, 0}, {true, 3u * 65536u + 17u, 9u * 65536u + 5u}, {true, 65536u * 5u + 500u, 65536u * 5u + 3500u},
                              {true, 65536u * 30u + 60000u, 65536u * 33u}, {true, 70010u, 70020u}, {true, 65536u * 39u, n_bits - 1u}};
        for (int resident = 0; resident < 2; ++resident) {
            gpu.set_device_set(resident ? &ds : nullptr);
            for (const Hint& h : hints)
                for (size_t x = 0; x < ands.size(); ++x) for (size_t y = 0; y < subs.size(); ++y) {
                    if (resident && (x == 4 || y == 3)) continue;          // the lone vectors are not members of ds: that is the upload road, covered above
                    ref.reset_range_hint(); gpu.reset_range_hint();
                    if (h.on) { bool r1 = ref.set_range_hint(h.from, h.to), r2 = gpu.set_range_hint(h.from, h.to); CHECK(r1 == r2, "set_range_hint return"); }
                    bvect::size_type i1 = 0, i2 = 0;
                    bool f1 = ref.find_first_and_sub(i1, ands[x].data(), ands[x].size(), subs[y].empty() ? 0 : subs[y].data(), subs[y].size());
                    bool f2 = gpu.find_first_and_sub(i2, ands[x].data(), ands[x].size(), subs[y].empty() ? 0 : subs[y].data(), subs[y].size());
                    CHECK(f1 == f2 && (!f1 || i1 == i2), "find_first_and_sub and=%zu sub=%zu hint=%d[%u,%u] resident=%d: ref %d@%u vs %d@%u",
                          x, y, (int)h.on, h.from, h.to, resident, (int)f1, (unsigned)i1, (int)f2, (unsigned)i2);
                }
        }
        ref.reset_range_hint(); gpu.reset_range_hint(); gpu.set_device_set(nullptr);
        for (int k = 0; k < 2; ++k) { ref.add(all[k]); gpu.add(all[k]); } ref.add(all[4], 1); gpu.add(all[4], 1);
        bvect::size_type i1 = 0, i2 = 0; bool f1 = ref.find_first_and_sub(i1), f2 = gpu.find_first_and_sub(i2);
        CHECK(f1 == f2 && i1 == i2, "member find_first_and_sub");
    }
    {   // member forms with add()/reset(), as samples/bvsample16/sample16.cpp uses them
        bm::aggregator<bvect> ref; bm::b200::aggregator<bvect> gpu(ctx);
        for (int k = 0; k < 3; ++k) { ref.add(all[k]); gpu.add(all[k]); }
        for (int k = 10; k < 16; ++k) { ref.add(all[k], 1); gpu.add(all[k], 1); }
        bvect a, b; ref.combine_or(a); gpu.combine_or(b); CHECK(a.compare(b) == 0, "member combine_or");
        ref.combine_and(a); gpu.combine_and(b); CHECK(a.compare(b) == 0, "member combine_and");
        bool f1 = ref.combine_and_sub(a), f2 = gpu.combine_and_sub(b);
        CHECK(f1 == f2 && a.compare(b) == 0, "member combine_and_sub");
    }
    {   // SHIFT-R-AND (tests/stress/t.cpp AggregatorTest shift-and cases): dense sources so a few steps survive
        std::vector<std::unique_ptr<bvect>> ds; std::vector<const bvect*> dp;
        for (int k = 0; k < 6; ++k) {
            ds.emplace_back(new bvect()); fill(*ds.back(), rng, n_bits, 0.7, k % 2 == 1);
            ds.back()->set_bit(n_bits - 1); ds.back()->set_bit(65535); ds.back()->set_bit(65536);
            if (k >= 3) { BM_DECLARE_TEMP_BLOCK(tb) ds.back()->optimize(tb, bvect::opt_compress); }
            dp.push_back(ds.back().get());
        }
        for (int opt = 0; opt < 2; ++opt)
            for (size_t n : {size_t(1), size_t(2), size_t(4), size_t(6)}) {
                bm::aggregator<bvect> ref; bm::b200::aggregator<bvect> gpu(ctx);
                ref.set_optimization(opt ? bvect::opt_compress : bvect::opt_none); gpu.set_optimization(opt ? bvect::opt_compress : bvect::opt_none);
                bvect a, b;
                bool f1 = ref.combine_shift_right_and(a, dp.data(), n, false), f2 = gpu.combine_shift_right_and(b, dp.data(), n, false);
                CHECK(f1 == f2 && a.compare(b) == 0 && a.count() == b.count(), "combine_shift_right_and n=%zu opt=%d (%u vs %u bits)", n, opt, (unsigned)a.count(), (unsigned)b.count());
            }
    }
    {   // 3-operand ops: bits AND block kinds (calc_stat) for every pairing of block kinds and both opt modes.
        // all[0..5] hold bit-blocks (not optimized), all[6..] are optimize()d (GAP / FULL / NULL / bit), k % 5 == 3 have FULL ranges
        bvect sparse_a, sparse_b, inv;                        // GAP x GAP with disjoint, nested and identical runs; an almost-full vector
        for (unsigned p = 100; p < n_bits; p += 997) { sparse_a.set_bit(p); sparse_a.set_bit(p + 1); }
        for (unsigned p = 101; p < n_bits; p += 1499) sparse_b.set_range(p, p + 40);
        inv.set_range(0, n_bits - 1); for (unsigned p = 5; p < n_bits; p += 7919) inv.clear_bit(p);
        { BM_DECLARE_TEMP_BLOCK(tb) sparse_a.optimize(tb); sparse_b.optimize(tb); inv.optimize(tb); }
        std::vector<const bvect*> ops = {all[0], all[3], all[7], all[8], all[13], all[20], &sparse_a, &sparse_b, &inv};
        for (int opt = 0; opt < 2; ++opt) {
            bvect::optmode om = opt ? bvect::opt_compress : bvect::opt_none;
            for (size_t x = 0; x < ops.size(); ++x) for (size_t y = 0; y < ops.size(); ++y) {
                if (x == y) continue;
                for (int op = 0; op < 4; ++op) {
                    bvect t1, t2;
                    switch (op) {
                    case 0: t1.bit_and(*ops[x], *ops[y], om); bm::b200::bit_and(ctx, t2, *ops[x], *ops[y], om); break;
                    case 1: t1.bit_or (*ops[x], *ops[y], om); bm::b200::bit_or (ctx, t2, *ops[x], *ops[y], om); break;
                    case 2: t1.bit_sub(*ops[x], *ops[y], om); bm::b200::bit_sub(ctx, t2, *ops[x], *ops[y], om); break;
                    default: t1.bit_xor(*ops[x], *ops[y], om); bm::b200::bit_xor(ctx, t2, *ops[x], *ops[y], om); break;
                    }
                    bvect::statistics s1, s2; t1.calc_stat(&s1); t2.calc_stat(&s2);
                    CHECK(t1.compare(t2) == 0 && t1.count() == t2.count(), "binop %d (%zu,%zu) opt=%d: bits", op, x, y, opt);
                    CHECK(s1.bit_blocks == s2.bit_blocks && s1.gap_blocks == s2.gap_blocks, "binop %d (%zu,%zu) opt=%d: kinds ref %zu bit / %zu gap, b200 %zu bit / %zu gap",
                          op, x, y, opt, (size_t)s1.bit_blocks, (size_t)s1.gap_blocks, (size_t)s2.bit_blocks, (size_t)s2.gap_blocks);
                }
            }
        }
        bvect t1, t2;
        t1.bit_and(*all[0], *all[9], bvect::opt_none); bm::b200::bit_and(ctx, t2, *all[0], *all[9]); CHECK(t1.compare(t2) == 0, "bit_and");
        t1.bit_or(*all[2], *all[20], bvect::opt_none); bm::b200::bit_or(ctx, t2, *all[2], *all[20]); CHECK(t1.compare(t2) == 0, "bit_or");
        t1.bit_sub(*all[1], *all[3], bvect::opt_none); bm::b200::bit_sub(ctx, t2, *all[1], *all[3]); CHECK(t1.compare(t2) == 0, "bit_sub");
    }
    {   // pipeline: many argument groups over shared vectors (tests/stress/t.cpp:10383-10640)
        bm::aggregator<bvect> ref; bm::b200::aggregator<bvect> gpu(ctx);
        bm::aggregator<bvect>::pipeline<bm::agg_opt_bvect_and_counts> rp;
        bm::b200::pipeline<bvect> gp(ctx);
        bvect or_ref, or_gpu; or_ref.init(); or_gpu.init();
        rp.set_or_target(&or_ref); gp.set_or_target(&or_gpu);
        for (int g = 0; g < 12; ++g) {
            auto* a1 = rp.add(); auto* a2 = gp.add();
            int na = 1 + g % 3, ns = (g * 5) % 9;
            for (int k = 0; k < na; ++k) { a1->add(all[(g + k) % 24], 0); a2->add(all[(g + k) % 24], 0); }
            for (int k = 0; k < ns; ++k) { a1->add(all[(g * 7 + k + 3) % 24], 1); a2->add(all[(g * 7 + k + 3) % 24], 1); }
        }
        rp.complete(); gp.complete();
        ref.combine_and_sub(rp); gpu.combine_and_sub(gp);
        auto& r1 = rp.get_bv_res_vector(); auto& c1 = rp.get_bv_count_vector();
        auto& r2 = gp.get_bv_res_vector(); auto& c2 = gp.get_bv_count_vector();
        CHECK(r1.size() == r2.size() && c1.size() == c2.size(), "pipeline sizes");
        for (size_t g = 0; g < r2.size(); ++g) {
            CHECK((size_t)c1[g] == (size_t)c2[g], "pipeline count g=%zu", g);
            CHECK((r1[g] == 0) == (r2[g] == 0), "pipeline null-ness g=%zu", g);
            if (r1[g] && r2[g]) CHECK(r1[g]->compare(*r2[g]) == 0, "pipeline result g=%zu", g);
        }
        CHECK(or_ref.compare(or_gpu) == 0, "pipeline OR target");
    }
    {   // bit_or_and / merge (src/bm.h:6283,5883)
        bvect t1(*all[5]), t2(*all[5]);
        t1.bit_or_and(*all[0], *all[7]); bm::b200::bit_or_and(ctx, t2, *all[0], *all[7]); CHECK(t1.compare(t2) == 0, "bit_or_and");
        bvect m1(*all[2]), m2(*all[2]), s1(*all[13]), s2(*all[13]);
        m1.merge(s1); bm::b200::merge(ctx, m2, s2); CHECK(m1.compare(m2) == 0 && m1.count() == m2.count(), "merge");
    }
    {   bvect t1, t2;
        t1.bit_xor(*all[4], *all[11], bvect::opt_none); bm::b200::bit_xor(ctx, t2, *all[4], *all[11]); CHECK(t1.compare(t2) == 0, "bit_xor");
    }
    // rs_index built on the GPU, consumed by the reference's own count_to / select
    for (int k : {0, 3, 8, 23}) {
        const bvect& bv = *all[k];
        bvect::rs_index_type rs_ref, rs_gpu;
        bv.build_rs_index(&rs_ref);
        bm::b200::build_rs_index(ctx, bv, &rs_gpu);
        CHECK(rs_ref.count() == rs_gpu.count(), "rs count k=%d", k);
        unsigned nb_tot = (n_bits >> 16) + 1;
        bool same = true;
        for (unsigned nb = 0; nb < nb_tot; ++nb)
            same &= rs_ref.count(nb) == rs_gpu.count(nb) && rs_ref.rcount(nb) == rs_gpu.rcount(nb) &&
                    (rs_ref.count(nb) == 0 || rs_ref.sub_count(nb) == rs_gpu.sub_count(nb));
        CHECK(same, "rs fields k=%d", k);
        bool q = true;
        for (int i = 0; i < 20000; ++i) {
            bvect::size_type p = (bvect::size_type)(rng() % n_bits);
            q &= bv.count_to(p, rs_gpu) == bv.count_to(p, rs_ref);
            bvect::size_type r = (bvect::size_type)(rng() % (rs_ref.count() + 2)), p1 = 0, p2 = 0;
            bool f1 = bv.select(r, p1, rs_ref), f2 = bv.select(r, p2, rs_gpu);
            q &= (f1 == f2) && (!f1 || p1 == p2);
        }
        CHECK(q, "rank/select through the reference with the GPU-built index k=%d", k);
    }
    // sparse_vector_scanner vs bm::b200::scanner on real bm::sparse_vector<unsigned> objects (plain and nullable)
    for (int nullable = 0; nullable < 2; ++nullable) {
        typedef bm::sparse_vector<unsigned, bvect> svect;
        svect sv(nullable ? bm::use_null : bm::no_null);
        const unsigned n = 5u * 65536u + 777u;
        sv.resize(n);
        for (unsigned i = 0; i < n; ++i) {
            if (nullable && rng() % 9 == 0) continue;
            unsigned v = (rng() % 3 == 0) ? 0u : unsigned(rng() % 3000);
            if (i > 100000 && i < 104000) v = 55;
            if (rng() % 1500 == 0) v |= 1u << 18;
            sv.set(i, v);
        }
        { BM_DECLARE_TEMP_BLOCK(tb) sv.optimize(tb); }
        bm::sparse_vector_scanner<svect> ref_sc;
        bm::b200::scanner<svect> gpu_sc(ctx, sv);
        for (unsigned v : {0u, 1u, 55u, 2999u, 3000u, (1u << 18) + 5u, 1u << 25}) {
            bvect a, b;
            ref_sc.find_eq(sv, v, a); gpu_sc.find_eq(v, b); CHECK(a.compare(b) == 0, "scanner find_eq(%u) nullable=%d", v, nullable);
            ref_sc.find_gt(sv, v, a); gpu_sc.find_gt(v, b); CHECK(a.compare(b) == 0, "scanner find_gt(%u) nullable=%d", v, nullable);
            ref_sc.find_ge(sv, v, a); gpu_sc.find_ge(v, b); CHECK(a.compare(b) == 0, "scanner find_ge(%u) nullable=%d", v, nullable);
            ref_sc.find_lt(sv, v, a); gpu_sc.find_lt(v, b); CHECK(a.compare(b) == 0, "scanner find_lt(%u) nullable=%d", v, nullable);
            ref_sc.find_le(sv, v, a); gpu_sc.find_le(v, b); CHECK(a.compare(b) == 0, "scanner find_le(%u) nullable=%d", v, nullable);
            ref_sc.find_range(sv, v / 2, v, a); gpu_sc.find_range(v / 2, v, b); CHECK(a.compare(b) == 0, "scanner find_range(%u,%u) nullable=%d", v / 2, v, nullable);
        }
        { bvect a, b; ref_sc.find_nonzero(sv, a); gpu_sc.find_nonzero(b); CHECK(a.compare(b) == 0, "scanner find_nonzero nullable=%d", nullable);
          ref_sc.find_zero(sv, a); gpu_sc.find_zero(b); CHECK(a.compare(b) == 0, "scanner find_zero nullable=%d", nullable); }
        std::vector<uint64_t> vals = {7, 55, 0, 2500, 99999};
        std::vector<bvect> outs; std::vector<bvect::size_type> cnts;
        gpu_sc.find_batch(BMB200_SCAN_EQ, vals, outs); gpu_sc.count_batch(BMB200_SCAN_EQ, vals, cnts);
        for (size_t k = 0; k < vals.size(); ++k) {
            bvect a; ref_sc.find_eq(sv, (unsigned)vals[k], a);
            CHECK(a.compare(outs[k]) == 0 && a.count() == cnts[k], "scanner batch eq k=%zu nullable=%d", k, nullable);
        }
    }
    // ---- operands as serialization BLOBs (bm::serializer<>, every compression level, with and without bookmarks): decoded on the
    // GPU and aggregated there (bm::b200::blob_aggregator) == bm::deserialize + bm::aggregator on the host
    for (unsigned level = 0; level <= 6; ++level) {
        for (int bookmarks = 0; bookmarks < 2; ++bookmarks) {
            if (bookmarks && level != 2 && level != 6) continue;
            std::vector<bm::serializer<bvect>::buffer> bufs(all.size());
            for (size_t k = 0; k < all.size(); ++k) {
                bm::serializer<bvect> ser; ser.set_compression_level(level);
                if (bookmarks) ser.set_bookmarks(true, 8);
                ser.serialize(*all[k], bufs[k]);
            }
            bm::aggregator<bvect> ref; ref.set_optimization(bvect::opt_compress);
            bm::b200::blob_aggregator<bvect> gpu(ctx, n_bits); gpu.set_optimization(bvect::opt_compress);
            // the host side of the comparison goes through bm::deserialize, like an application holding BLOBs would
            std::vector<std::unique_ptr<bvect>> back;
            for (size_t k = 0; k < all.size(); ++k) { back.emplace_back(new bvect()); bm::deserialize(*back.back(), bufs[k].data()); }
            std::vector<const bvect*> bp; for (auto& v : back) bp.push_back(v.get());
            for (size_t k = 0; k < all.size(); ++k) gpu.add(bufs[k].data(), bufs[k].size(), k < 3 ? 0 : 1);
            bvect t_ref, t_gpu;
            bool f_ref = ref.combine_and_sub(t_ref, bp.data(), 3, bp.data() + 3, bp.size() - 3, false);
            bool f_gpu = gpu.combine_and_sub(t_gpu);
            CHECK(f_ref == f_gpu && t_ref.compare(t_gpu) == 0 && t_ref.count() == t_gpu.count(), "blob combine_and_sub level=%u bookmarks=%d", level, bookmarks);
            gpu.reset();
            for (size_t k = 0; k < all.size(); ++k) gpu.add(bufs[k].data(), bufs[k].size());
            ref.combine_or(t_ref, bp.data(), bp.size()); gpu.combine_or(t_gpu);
            CHECK(t_ref.compare(t_gpu) == 0 && t_ref.count() == t_gpu.count(), "blob combine_or level=%u bookmarks=%d", level, bookmarks);
        }
    }
#ifdef BM64ADDR
    check_past_2_32(ctx, rng);
#endif
    std::printf("%s: %d checks, %d failed\n", g_fail ? "FAILED" : "OK", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
