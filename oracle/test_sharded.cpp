/*
 * test_sharded.cpp -- TEST INFRASTRUCTURE.  bm::b200::sharded_aggregator<bm::bvector<>> (one process per GPU, block-range shards,
 * ONE ncclAllGather of per-column popcounts behind bmb200_exchange_popcounts) against bm::aggregator on the full vectors.
 *   usage: test_sharded <rank> <nranks> <id-file>      (rank r uses GPU r; rank 0 writes the 128-byte communicator id to <id-file>)
 * Every rank builds the same seeded vectors, keeps only its shard on its GPU, and checks: its target == the reference result
 * restricted to its block range, count() == the reference cardinality, block_popcounts() == the reference's per-block counts.
 */
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <memory>
#include <random>
#include <thread>
#include <vector>

#include "bm.h"
#include "bmaggregator.h"
#include "bmb200_aggregator.hpp"

typedef bm::bvector<> bvect;
static int g_fail = 0, g_checks = 0;
#define CHECK(cond, ...) do { ++g_checks; if (!(cond)) { ++g_fail; std::printf("FAIL %s:%d: ", __FILE__, __LINE__); std::printf(__VA_ARGS__); std::printf("\n"); } } while (0)

int main(int argc, char** argv)
{
    if (argc < 4) { std::printf("usage: %s rank nranks idfile\n", argv[0]); return 2; }
    const int rank = std::atoi(argv[1]), nranks = std::atoi(argv[2]);
    const char* idfile = argv[3];
    char id[BMB200_COMM_ID_BYTES];
    if (rank == 0) {
        bm::b200::sharded_aggregator<bvect>::unique_id(id);
        std::ofstream f(std::string(idfile) + ".tmp", std::ios::binary); f.write(id, sizeof id); f.close();
        std::rename((std::string(idfile) + ".tmp").c_str(), idfile);
    } else {
        for (int tries = 0; tries < 600; ++tries) {
            std::ifstream f(idfile, std::ios::binary);
            if (f && f.read(id, sizeof id)) break;
            std::this_thread::sleep_for(std::chrono::milliseconds(100));
            if (tries == 599) { std::printf("rank %d: no communicator id\n", rank); return 3; }
        }
    }
    const unsigned n_blocks = 256u * 2u * (unsigned)nranks + 256u;          // ragged: one rank gets an extra superblock
    const unsigned n_bits = n_blocks * 65536u - 777u;
    std::mt19937_64 rng(4242);
    std::vector<std::unique_ptr<bvect>> vs;
    for (int k = 0; k < 12; ++k) {
        vs.emplace_back(new bvect());
        vs.back()->resize(n_bits);                          // (a default bvector spans 2^32 - 1 bits = 65536 blocks)
        std::geometric_distribution<unsigned> skip(0.002 / (k + 1));
        for (uint64_t p = skip(rng); p < n_bits; p += 1 + skip(rng)) vs.back()->set_bit_no_check((bvect::size_type)p);
        if (k % 4 == 1) vs.back()->set_range(65536u * 300u, 65536u * 302u + 99u);
        if (k >= 3) { BM_DECLARE_TEMP_BLOCK(tb) vs.back()->optimize(tb, bvect::opt_compress); }
    }
    std::vector<const bvect*> all; for (auto& v : vs) all.push_back(v.get());

    bm::b200::context ctx(rank);
    bm::b200::sharded_aggregator<bvect> sh(ctx, nranks, rank, id);
    sh.set_optimization(bvect::opt_compress);
    sh.assign(all.data(), all.size());
    const uint32_t from = sh.shard_from(), to = sh.shard_to();
    bvect mask; mask.set_range((bvect::size_type)from * 65536u, (bvect::size_type)((uint64_t)to * 65536ull - 1ull));

    bm::aggregator<bvect> ref; ref.set_optimization(bvect::opt_compress);
    for (int pass = 0; pass < 2; ++pass) {
        bvect t_ref, t_gpu;
        if (pass == 0) { ref.combine_or(t_ref, all.data(), all.size()); sh.combine_or(t_gpu, all.data(), all.size()); }
        else { ref.combine_and_sub(t_ref, all.data(), 2, all.data() + 2, all.size() - 2, false); sh.combine_and_sub(t_gpu, all.data(), 2, all.data() + 2, all.size() - 2); }
        CHECK(sh.count() == (uint64_t)t_ref.count(), "pass %d: global count %llu vs %llu", pass, (unsigned long long)sh.count(), (unsigned long long)t_ref.count());
        const std::vector<uint32_t>& pop = sh.block_popcounts();
        CHECK(pop.size() == n_blocks, "pass %d: popcount vector size", pass);
        unsigned bad = 0;
        for (unsigned nb = 0; nb < n_blocks && nb < pop.size(); ++nb) {
            bvect::size_type lo = (bvect::size_type)nb * 65536u, hi = lo + 65535u; if (hi >= n_bits) hi = n_bits - 1;
            if (pop[nb] != (uint32_t)t_ref.count_range(lo, hi)) ++bad;
        }
        CHECK(bad == 0, "pass %d: %u per-block popcounts differ", pass, bad);
        bvect shard_ref(t_ref); shard_ref &= mask;
        CHECK(shard_ref.compare(t_gpu) == 0, "pass %d: rank %d target != reference restricted to blocks [%u, %u)", pass, rank, from, to);
    }
    std::printf("%s: rank %d/%d blocks [%u, %u): %d checks, %d failed; exchange mode %d (1 = ncclAllGather)\n",
                g_fail ? "FAILED" : "OK", rank, nranks, from, to, g_checks, g_fail, sh.exchange_mode());
    return g_fail ? 1 : 0;
}
