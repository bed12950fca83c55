/*
 * test_str_binding.cpp -- TEST INFRASTRUCTURE.  Drop-in check of the string scanner at the bm::bvector<> level: the
 * UNMODIFIED reference's bm::sparse_vector_scanner<> (headers from the reference tree) against bm::b200::scanner<>
 * (bitmagic_b200/include/bmb200_scanner.hpp, which talks to libbmb200.so) on real str_sparse_vector<char, bvector<>, 32>:
 * plain, nullable and remap()ed; find_eq_str, find_eq_str_prefix, find_eq_str(pos), and the batched forms against the
 * reference's pipeline (results and counts).  Parity criterion = the reference's own: compare() == 0, equal count() and the
 * same return value.  Built by oracle/str.mk into oracle/_ref/.
 *
 * Queries stay where the reference defines an answer (DESIGN.md §3.5c): for a remapped vector no query longer than
 * effective_max_str() - 1 and no byte >= 0x80, and no empty string: the reference answers it with find_zero, which ORs only
 * effective_slices() planes, 1 for a string vector (the product returns the elements whose planes are all 0).
 */
#include <cstdio>
#include <cstdint>
#include <random>
#include <string>
#include <vector>

#include "bm.h"
#include "bmstrsparsevec.h"
#include "bmsparsevec_algo.h"
#include "bmb200_aggregator.hpp"
#include "bmb200_scanner.hpp"

typedef bm::bvector<> bvect;
typedef bm::str_sparse_vector<char, bvect, 32> str_svect;
static int g_fail = 0, g_checks = 0;
#define CHECK(cond, ...) do { ++g_checks; if (!(cond)) { ++g_fail; std::printf("FAIL %s:%d: ", __FILE__, __LINE__); std::printf(__VA_ARGS__); std::printf("\n"); } } while (0)

// a dictionary of words over a small alphabet (shared prefixes), long runs of one word (GAP / FULL planes), NULLs
static std::vector<std::string> words(std::mt19937_64& rng, size_t n)
{
    std::vector<std::string> w;
    std::uniform_int_distribution<int> len(1, 14), ch(0, 5);
    const char alpha[] = "abcxyz";
    for (size_t k = 0; k < n; ++k) {
        std::string s; const int l = len(rng);
        for (int i = 0; i < l; ++i) s.push_back(alpha[ch(rng)]);
        w.push_back(s);
    }
    return w;
}

static void fill(str_svect& sv, std::mt19937_64& rng, uint64_t n, bool nullable, const std::vector<std::string>& dict)
{
    std::uniform_int_distribution<size_t> pick(0, dict.size() - 1);
    std::uniform_real_distribution<double> u(0.0, 1.0);
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t nb = i >> 16;
        if (nullable && (nb % 3 == 2 || u(rng) < 0.2)) { sv.push_back_null(); continue; }
        if (nb % 3 == 1) sv.push_back(dict[((i >> 12) & 1u)].c_str());          // long runs of two words
        else if (i % 777 == 5) sv.push_back("");
        else sv.push_back(dict[pick(rng)].c_str());
    }
}

static void check_vector(bm::b200::context& ctx, const str_svect& sv, const char* what, const std::vector<std::string>& all)
{
    std::vector<std::string> queries;
    for (const auto& q : all) if (!q.empty() && (!sv.is_remap() || q.size() < sv.effective_max_str())) queries.push_back(q);
    bm::sparse_vector_scanner<str_svect> ref_sc;
    bm::b200::scanner<str_svect> sc(ctx, sv);
    for (const auto& q : queries) {
        bvect r, g;
        bool fr = ref_sc.find_eq_str(sv, q.c_str(), r), fg = sc.find_eq_str(q.c_str(), g);
        CHECK(fr == fg && r.compare(g) == 0 && r.count() == g.count(), "%s find_eq_str(\"%s\"): ref %d/%llu gpu %d/%llu", what, q.c_str(),
              (int)fr, (unsigned long long)r.count(), (int)fg, (unsigned long long)g.count());
        bvect rp, gp;
        fr = ref_sc.find_eq_str_prefix(sv, q.c_str(), rp); fg = sc.find_eq_str_prefix(q.c_str(), gp);
        CHECK(fr == fg && rp.compare(gp) == 0 && rp.count() == gp.count(), "%s find_eq_str_prefix(\"%s\"): ref %llu gpu %llu", what,
              q.c_str(), (unsigned long long)rp.count(), (unsigned long long)gp.count());
        str_svect::size_type pr = 0, pg = 0;
        fr = ref_sc.find_eq_str(sv, q.c_str(), pr); fg = sc.find_eq_str(q.c_str(), pg);
        CHECK(fr == fg && (!fr || pr == pg), "%s find_eq_str(\"%s\", pos): ref %d@%llu gpu %d@%llu", what, q.c_str(), (int)fr,
              (unsigned long long)pr, (int)fg, (unsigned long long)pg);
    }
    // the batched forms against the reference's pipeline
    const std::vector<std::string>& batch = queries;
    bm::sparse_vector_scanner<str_svect>::pipeline<bm::agg_opt_bvect_and_counts> pipe(sv);
    for (const auto& q : batch) pipe.add(q.c_str());
    pipe.complete();
    ref_sc.find_eq_str(pipe);
    std::vector<bvect> outs; std::vector<bvect::size_type> counts;
    sc.find_eq_str_batch(batch, outs); sc.count_eq_str_batch(batch, counts);
    for (size_t k = 0; k < batch.size(); ++k) {
        const bvect* r = pipe.get_bv_res_vector()[k];
        bvect empty;
        const bvect& rr = r ? *r : empty;
        CHECK(rr.compare(outs[k]) == 0 && rr.count() == counts[k] && (bvect::size_type)pipe.get_bv_count_vector()[k] == counts[k],
              "%s batch \"%s\": ref %llu gpu %llu / %llu", what, batch[k].c_str(), (unsigned long long)rr.count(),
              (unsigned long long)outs[k].count(), (unsigned long long)counts[k]);
    }
}

int main()
{
    std::mt19937_64 rng(20261017);
    bm::b200::context ctx(0);
    const std::vector<std::string> dict = words(rng, 300);
    const uint64_t sizes[] = {3u * 65536u + 123u, 1000u, 0u};
    char what[96];
    for (uint64_t n : sizes)
        for (int nullable = 0; nullable < 2; ++nullable)
            for (int remap = 0; remap < 2; ++remap) {
                str_svect sv(nullable ? bm::use_null : bm::no_null);
                fill(sv, rng, n, nullable != 0, dict);
                if (remap) sv.remap();
                BM_DECLARE_TEMP_BLOCK(tb)
                sv.optimize(tb);
                std::vector<std::string> q = {"a", "ab", "abc", "zzzzzzzzzzzzzz", "q", "x", "xyzab"};
                for (int k = 0; k < 12; ++k) q.push_back(dict[(size_t)k * 7 % dict.size()]);
                for (int k = 0; k < 4; ++k) q.push_back(dict[(size_t)k].substr(0, 2));          // prefixes of stored words
                if (!remap) { q.push_back("ab\xc3\xa9"); q.push_back(dict[0] + "abcabcabcabcabcabcabc"); }
                std::snprintf(what, sizeof(what), "n=%llu nullable=%d remap=%d", (unsigned long long)n, nullable, remap);
                check_vector(ctx, sv, what, q);
            }
    std::printf("test_str_binding: %d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
