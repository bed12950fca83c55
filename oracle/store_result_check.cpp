/*
 * store_result_check.cpp -- TEST INFRASTRUCTURE.  bm::b200::detail::store_result (the binding's result materialisation: recycles the
 * target's blocks in place, several host threads over disjoint top-level sub-trees) against a fresh build of the same result:
 * random kind mixes, changing sizes / block ranges / shard offsets from call to call into ONE target.  Host code only (no GPU needed);
 * built by oracle/Makefile into oracle/_ref/ because it needs the reference headers.
 */
#include <cstdio>
#include <random>
#include <vector>
#include "bm.h"
#include "bmaggregator.h"
#include "bmb200_aggregator.hpp"
typedef bm::bvector<> bvect;
int main()
{
    std::mt19937 rng(7);
    bvect target; int fails = 0;
#ifdef BM64ADDR
    // the binding's upload extent (bm::b200::detail::extent_of): populated blocks up to the last set bit, capped by size(), never
    // truncated to 32 bits; a vector whose last block is column 2^32 - 1 needs 2^32 columns and is refused
    {
        const uint64_t G = uint64_t(1) << 32;
        auto extent_with = [](uint64_t bit) { bvect bv; bv.set((bvect::size_type)bit); return (uint64_t)bm::b200::detail::extent_of(bv); };
        bvect empty, sized(1000), none(0);
        struct { const char* what; uint64_t got, want; } cases[] = {
            {"default vector", bm::b200::detail::extent_of(empty), 1}, {"size 1000", bm::b200::detail::extent_of(sized), 1},
            {"size 0", bm::b200::detail::extent_of(none), 0}, {"bit 2^32 - 1", extent_with(G - 1), 65536},
            {"bit 2^32", extent_with(G), 65537}, {"bit 2^33", extent_with(2 * G), 131073},
            {"bit 2^32 + 65535", extent_with(G + 65535), 65537}, {"bit 2^32 + 65536", extent_with(G + 65536), 65538},
            {"default size in blocks", bm::b200::detail::size_blocks(empty.size()), G}};
        for (const auto& c : cases)
            if (c.got != c.want) { ++fails; std::printf("extent %s: %llu, want %llu\n", c.what, (unsigned long long)c.got, (unsigned long long)c.want); }
        bool refused = false;
        try { extent_with(empty.size() - 1); } catch (const std::length_error&) { refused = true; }
        if (!refused) { ++fails; std::printf("extent of a bit in block 2^32 - 1 was not refused\n"); }
        refused = false;
        try { bm::b200::detail::column_count(G, "column_count"); } catch (const std::length_error&) { refused = true; }
        if (!refused || bm::b200::detail::column_count(G - 1, "column_count") != G - 1) { ++fails; std::printf("column_count(2^32) not refused\n"); }
    }
#endif
    for (int it = 0; it < 60; ++it) {
        const uint32_t n_cols = (it % 3 == 0) ? 2400 : (it % 3 == 1 ? 700 : 2048 + 256 * (it % 5));
#ifdef BM64ADDR
        // shard offsets past 2^32 bits: top-level index >= 256, one of them straddling top-level entries 255 / 256
        const uint32_t nb_off = (it % 4 == 3) ? 100 : (it % 4 == 2 ? 65536u + 300u : (it % 4 == 1 ? 65536u - 600u : 0));
#else
        const uint32_t nb_off = (it % 4 == 3) ? 100 : 0;
#endif
        std::vector<uint8_t> kind(n_cols); std::vector<uint64_t> off(n_cols);
        std::vector<uint16_t> gaps; std::vector<uint32_t> bits;
        const int mode = it % 6;
        for (uint32_t c = 0; c < n_cols; ++c) {
            unsigned r = rng() % 100;
            unsigned k = mode == 5 ? BMB200_BLK_FULL : r < 25 ? BMB200_BLK_NULL : r < 35 ? BMB200_BLK_FULL : r < 55 ? BMB200_BLK_BIT : BMB200_BLK_GAP;
            if (mode == 4 && (c >> 8) % 2) k = BMB200_BLK_NULL;       // whole top-level blocks empty
            kind[c] = (uint8_t)k;
            if (k == BMB200_BLK_BIT) { off[c] = bits.size() / 2048; for (int w = 0; w < 2048; ++w) bits.push_back(rng()); }
            else if (k == BMB200_BLK_GAP) {
                off[c] = gaps.size();
                uint32_t runs = 1 + rng() % (it % 2 ? 1270 : 200); std::vector<uint16_t> g(runs + 1);
                uint32_t pos = rng() % 20;
                for (uint32_t q = 1; q < runs; ++q) { g[q] = (uint16_t)pos; pos += 1 + rng() % 45; }
                g[runs] = 65535; g[0] = (uint16_t)((runs << 3) | (rng() & 1));
                gaps.insert(gaps.end(), g.begin(), g.end()); while (gaps.size() % 8) gaps.push_back(0);
            }
        }
        bvect::size_type sz = (bvect::size_type)((it % 7 == 6 ? 3000u : 2700u) * 65536u - 1);
        if (nb_off >= 65536u - 600u) sz = (bvect::size_type)((uint64_t(nb_off) + n_cols + (it % 7 == 6 ? 5u : 0u)) * 65536u - 1u);
        bvect fresh;
        bm::b200::detail::store_result(fresh, sz, n_cols, kind.data(), off.data(), bits.data(), gaps.data(), nb_off);
        bm::b200::detail::store_result(target, sz, n_cols, kind.data(), off.data(), bits.data(), gaps.data(), nb_off);
        bvect::statistics a, b; fresh.calc_stat(&a); target.calc_stat(&b);
        bool ok = fresh.compare(target) == 0 && a.bit_blocks == b.bit_blocks && a.gap_blocks == b.gap_blocks && fresh.count() == target.count() && fresh.size() == target.size();
        if (!ok) { ++fails; std::printf("iteration %d differs (%zu/%zu vs %zu/%zu)\n", it, (size_t)a.bit_blocks, (size_t)a.gap_blocks, (size_t)b.bit_blocks, (size_t)b.gap_blocks); }
    }
    std::printf("%s: %d failures\n", fails ? "FAILED" : "OK", fails);
    return fails != 0;
}
