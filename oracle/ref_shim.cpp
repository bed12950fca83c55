/*
 * ref_shim.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * extern "C" wrapper around the UNMODIFIED reference (tlk00/BitMagic headers included from
 * /root/reference/src where they lie; nothing is copied).  Built by oracle/Makefile into
 * oracle/_ref/libbmref.so (32-bit addressing) and oracle/_ref/libbmref64.so (-DBM64ADDR) with the
 * reference's own AVX2 flags (-DBMAVX2OPT -march=skylake, reference CMakeLists.txt:91).
 *
 * Used to (1) pin oracle/bm_oracle.c, (2) generate tests/golden fixtures, (3) serve as the
 * "reference" CPU baseline in bench.py.  Never linked into the product.
 *
 * Data crosses the wrapper in the packed column-major format of include/bmb200.h: each call
 * rebuilds real bm::bvector<> objects from the packed set (blocks_manager::copy_bit_block /
 * allocate_gap_block / set_block_ptr), runs the reference entry point, and walks the result's
 * block tree back out.
 */
#include <cstdint>
#include <cstring>
#include <vector>
#include <memory>
#include <thread>
#include <chrono>
#include <algorithm>
#include <malloc.h>

#include "bm.h"
#include "bmaggregator.h"
#include "bmalgo.h"
#include "bmrs.h"
#include "bmserial.h"
#include "bmsparsevec.h"
#include "bmsparsevec_algo.h"

#include "../include/bmb200.h"

typedef bm::bvector<> bvect;

namespace {

inline uint32_t set_desc(const bmb200_packed_set* s, uint32_t v, uint32_t nb)
{ return s->desc[(size_t)nb * s->n_vec + v]; }
inline const uint32_t* set_bit_ptr(const bmb200_packed_set* s, uint32_t nb, uint32_t rel)
{ return s->bit_pool + (s->bit_base[nb] + rel) * (size_t)BMB200_BLOCK_WORDS; }
inline const uint16_t* set_gap_ptr(const bmb200_packed_set* s, uint32_t nb, uint32_t rel)
{ return s->gap_pool + (s->gap_base[nb] + (rel & BMB200_DESC_REL_MASK)) * (size_t)BMB200_GAP_UNIT_WORDS + (rel >> 29); }

/* vector `v`, block columns [nb_from, nb_to) of the packed set -> a real bvector whose block 0 is nb_from */
void build_bvector(const bmb200_packed_set* s, uint32_t v, uint32_t nb_from, uint32_t nb_to, bvect& bv)
{
    bv.clear(true);
    uint64_t bits = (uint64_t)(nb_to - nb_from) * 65536ull;
    if (bits > (uint64_t)bm::id_max) bits = bm::id_max;
    bv.resize((bvect::size_type)bits);
    bv.init();
    bvect::blocks_manager_type& bman = bv.get_blocks_manager();
    BM_DECLARE_TEMP_BLOCK(tb)   /* SIMD-aligned staging: packed arenas are only 4-byte aligned on the host */
    for (uint32_t nb = nb_from; nb < nb_to; ++nb)
    {
        uint32_t d = set_desc(s, v, nb);
        uint32_t kind = d & 3u, rel = d >> 2;
        if (kind == BMB200_BLK_NULL) continue;
        uint32_t lnb = nb - nb_from;
        unsigned i = lnb >> 8, j = lnb & 255u;
        bman.reserve_top_blocks(i + 1);
        bman.check_alloc_top_subblock(i);
        if (kind == BMB200_BLK_FULL)
            bman.set_block_ptr(i, j, FULL_BLOCK_FAKE_ADDR);
        else if (kind == BMB200_BLK_BIT)
        {
            std::memcpy(tb.begin(), set_bit_ptr(s, nb, rel), BMB200_BLOCK_BYTES);
            bman.copy_bit_block(i, j, tb.begin());
        }
        else
        {
            const bm::gap_word_t* g = set_gap_ptr(s, nb, rel);
            unsigned len = bm::gap_length(g) - 1;
            int level = bm::gap_calc_level(len, bman.glen());
            bm::gap_word_t* gb = bman.allocate_gap_block(unsigned(level), g);
            bman.set_block_ptr(i, j, (bm::word_t*)BMPTR_SETBIT0(gb));
        }
    }
}

/* walk a bvector's block tree into per-column outputs */
void export_bvector(const bvect& bv, uint32_t n_cols,
                    uint8_t* kind, uint32_t* popcnt, uint32_t* blocks, uint16_t* gaps)
{
    const bvect::blocks_manager_type& bman = bv.get_blocks_manager();
    BM_DECLARE_TEMP_BLOCK(tb)   /* the reference's block functions need SIMD-aligned destinations */
    for (uint32_t c = 0; c < n_cols; ++c)
    {
        unsigned i = c >> 8, j = c & 255u;
        const bm::word_t* blk = 0;
        if (bman.is_init() && i < bman.top_block_size())
            blk = bman.get_block_ptr(i, j);
        uint8_t kd; uint32_t pc = 0;
        uint32_t* bout = blocks ? blocks + (size_t)c * BMB200_BLOCK_WORDS : 0;
        uint16_t* gout = gaps ? gaps + (size_t)c * BMB200_GAP_MAX_WORDS : 0;
        if (gout) std::memset(gout, 0, sizeof(uint16_t) * BMB200_GAP_MAX_WORDS);
        if (!blk) { kd = BMB200_BLK_NULL; if (bout) std::memset(bout, 0, BMB200_BLOCK_BYTES); }
        else if (blk == FULL_BLOCK_FAKE_ADDR || blk == FULL_BLOCK_REAL_ADDR)
        { kd = BMB200_BLK_FULL; pc = 65536; if (bout) std::memset(bout, 0xFF, BMB200_BLOCK_BYTES); }
        else if (BM_IS_GAP(blk))
        {
            const bm::gap_word_t* g = BMGAP_PTR(blk);
            kd = BMB200_BLK_GAP; pc = bm::gap_bit_count_unr(g);
            if (bout) { bm::gap_convert_to_bitset(tb.begin(), g); std::memcpy(bout, tb.begin(), BMB200_BLOCK_BYTES); }
            if (gout) std::memcpy(gout, g, sizeof(uint16_t) * bm::gap_length(g));
        }
        else
        {
            kd = BMB200_BLK_BIT; pc = bm::bit_block_count(blk);
            if (bout) std::memcpy(bout, blk, BMB200_BLOCK_BYTES);
        }
        if (kind) kind[c] = kd;
        if (popcnt) popcnt[c] = pc;
    }
}

struct Built {
    std::vector<std::unique_ptr<bvect>> own;
    std::vector<const bvect*> g0, g1;
};

void build_groups(const bmb200_packed_set* s, const bmb200_agg_args* a, uint32_t nb_from, uint32_t nb_to, Built& b)
{
    std::vector<int> slot(s->n_vec, -1);
    auto get = [&](uint32_t v) -> const bvect* {
        if (slot[v] < 0) {
            b.own.emplace_back(new bvect());
            build_bvector(s, v, nb_from, nb_to, *b.own.back());
            slot[v] = (int)b.own.size() - 1;
        }
        return b.own[slot[v]].get();
    };
    for (uint32_t k = 0; k < a->n0; ++k) b.g0.push_back(get(a->group0[k]));
    if (a->op == BMB200_OP_AND_SUB)
        for (uint32_t k = 0; k < a->n1; ++k) b.g1.push_back(get(a->group1[k]));
}

/* run one reference aggregation; target is replaced */
bool run_op(bm::aggregator<bvect>& agg, const bmb200_agg_args* a, const Built& b, bvect& target)
{
    bool any = false;
    agg.set_optimization((a->flags & BMB200_F_OPT_COMPRESS) ? bvect::opt_compress : bvect::opt_none);
    switch (a->op)
    {
    case BMB200_OP_OR:
        agg.combine_or(target, b.g0.data(), b.g0.size());
        any = target.any();
        break;
    case BMB200_OP_AND:
        agg.combine_and(target, b.g0.data(), b.g0.size());
        any = target.any();
        break;
    case BMB200_OP_AND_SUB:
        any = agg.combine_and_sub(target, b.g0.data(), b.g0.size(),
                                  b.g1.empty() ? 0 : b.g1.data(), b.g1.size(), false);
        break;
    case BMB200_OP_SHIFT_R_AND:
        any = agg.combine_shift_right_and(target, b.g0.data(), b.g0.size(), false);
        break;
    case BMB200_OP_XOR:
        target.clear(true);
        if (!b.g0.empty()) {
            target = *b.g0[0];
            for (size_t k = 1; k < b.g0.size(); ++k) target.bit_xor(*b.g0[k]);
        }
        any = target.any();
        break;
    default: break;
    }
    return any;
}

} // namespace

extern "C" {

int ref_is_64(void)
{
#ifdef BM64ADDR
    return 1;
#else
    return 0;
#endif
}

const char* ref_simd(void)
{
#if defined(BMAVX512OPT)
    return "avx512";
#elif defined(BMAVX2OPT)
    return "avx2";
#elif defined(BMSSE42OPT)
    return "sse4.2";
#else
    return "scalar";
#endif
}

/* aggregator::combine_or / combine_and / combine_and_sub (src/bmaggregator.h:1101,1126,1162) or
 * chained bvector::bit_xor (src/bm.h:6572) on the real reference; outputs per column like orc_aggregate */
int ref_aggregate(const bmb200_packed_set* s, const bmb200_agg_args* a,
                  uint8_t* kind, uint32_t* popcnt, uint32_t* blocks, uint16_t* gaps, int* any_out)
{
    try {
        uint32_t nb_to = a->nb_to ? a->nb_to : s->n_blocks;
        Built b; build_groups(s, a, a->nb_from, nb_to, b);
        bvect target;
        bm::aggregator<bvect> agg;
        bool any = run_op(agg, a, b, target);
        if (any_out) *any_out = any ? 1 : 0;
        export_bvector(target, nb_to - a->nb_from, kind, popcnt, blocks, gaps);
        return 0;
    } catch (...) { return 1; }
}

/* "horizontal" (sequential 2-operand) path the reference's own stress tests use as their oracle:
 * combine_or_horizontal / combine_and_sub_horizontal src/bmaggregator.h:2407-2474 */
int ref_aggregate_horizontal(const bmb200_packed_set* s, const bmb200_agg_args* a,
                             uint8_t* kind, uint32_t* popcnt, uint32_t* blocks)
{
    try {
        uint32_t nb_to = a->nb_to ? a->nb_to : s->n_blocks;
        Built b; build_groups(s, a, a->nb_from, nb_to, b);
        bvect target;
        bm::aggregator<bvect> agg;
        switch (a->op) {
        case BMB200_OP_OR:  agg.combine_or_horizontal(target, b.g0.data(), b.g0.size()); break;
        case BMB200_OP_AND: agg.combine_and_horizontal(target, b.g0.data(), b.g0.size()); break;
        case BMB200_OP_AND_SUB:
            agg.combine_and_sub_horizontal(target, b.g0.data(), b.g0.size(),
                                           b.g1.empty() ? 0 : b.g1.data(), b.g1.size());
            break;
        default: return 2;
        }
        export_bvector(target, nb_to - a->nb_from, kind, popcnt, blocks, 0);
        return 0;
    } catch (...) { return 1; }
}

/* bvector 3-operand ops (src/bm.h:1745-1850): t.bit_and(a,b,opt) etc.; op: 0 OR 1 AND 2 SUB 3 XOR; false for any other op */
static bool run_binop(const bmb200_packed_set* s, int op, uint32_t va, uint32_t vb, int compress, bvect& t)
{
    bvect a, b;
    build_bvector(s, va, 0, s->n_blocks, a);
    build_bvector(s, vb, 0, s->n_blocks, b);
    bvect::optmode om = compress ? bvect::opt_compress : bvect::opt_none;
    switch (op) {
    case 0: t.bit_or(a, b, om); return true;
    case 1: t.bit_and(a, b, om); return true;
    case 2: t.bit_sub(a, b, om); return true;
    case 3: t.bit_xor(a, b, om); return true;
    default: return false;
    }
}

int ref_binop(const bmb200_packed_set* s, int op, uint32_t va, uint32_t vb, int compress,
              uint8_t* kind, uint32_t* popcnt, uint32_t* blocks, uint64_t* count_out)
{
    try {
        bvect t;
        if (!run_binop(s, op, va, vb, compress, t)) return 2;
        if (count_out) *count_out = t.count();
        export_bvector(t, s->n_blocks, kind, popcnt, blocks, 0);
        return 0;
    } catch (...) { return 1; }
}

/* ref_binop with the GAP words of the result as well (header with its capacity level + run ends, zero-filled past the
 * block), so that the block kinds and GAP levels the two-operand ops store can be compared word for word */
int ref_binop_gaps(const bmb200_packed_set* s, int op, uint32_t va, uint32_t vb, int compress,
                   uint8_t* kind, uint32_t* popcnt, uint32_t* blocks, uint16_t* gaps)
{
    try {
        bvect t;
        if (!run_binop(s, op, va, vb, compress, t)) return 2;
        export_bvector(t, s->n_blocks, kind, popcnt, blocks, gaps);
        return 0;
    } catch (...) { return 1; }
}

/* bm::count_and / count_or / count_sub / count_xor (src/bmalgo.h:48-51) */
int ref_count_op(const bmb200_packed_set* s, int op, uint32_t va, uint32_t vb, uint64_t* out)
{
    try {
        bvect a, b;
        build_bvector(s, va, 0, s->n_blocks, a);
        build_bvector(s, vb, 0, s->n_blocks, b);
        switch (op) {
        case 0: *out = bm::count_or(a, b); break;
        case 1: *out = bm::count_and(a, b); break;
        case 2: *out = bm::count_sub(a, b); break;
        case 3: *out = bm::count_xor(a, b); break;
        default: return 2;
        }
        return 0;
    } catch (...) { return 1; }
}

/* bvector::optimize(opt_compress) on one vector of the set (src/bm.h:3667) -> per-column kinds + data */
int ref_optimize(const bmb200_packed_set* s, uint32_t v,
                 uint8_t* kind, uint32_t* popcnt, uint32_t* blocks, uint16_t* gaps)
{
    try {
        bvect a;
        build_bvector(s, v, 0, s->n_blocks, a);
        BM_DECLARE_TEMP_BLOCK(tb)
        a.optimize(tb, bvect::opt_compress);
        export_bvector(a, s->n_blocks, kind, popcnt, blocks, gaps);
        return 0;
    } catch (...) { return 1; }
}

/* build_rs_index (src/bm.h:2531) and read every field back through the public rs_index accessors
 * (count / rcount / sub_count / get_super_block_rcount, src/bmrs.h:324-384,398-460) */
int ref_rs_build(const bmb200_packed_set* s, uint32_t v,
                 uint32_t* bcount, uint64_t* sub_count, uint64_t* sb_count, uint64_t* total)
{
    try {
        bvect a;
        build_bvector(s, v, 0, s->n_blocks, a);
        bvect::rs_index_type rs;
        a.build_rs_index(&rs);
        uint32_t nsb = (s->n_blocks + 255u) / 256u;
        if (sb_count) {
            sb_count[0] = 0;
            for (uint32_t i = 0; i < nsb; ++i) sb_count[i + 1] = rs.get_super_block_rcount(i);
        }
        for (uint32_t nb = 0; nb < s->n_blocks; ++nb) {
            if (bcount) bcount[nb] = rs.count(nb);
            if (sub_count) sub_count[nb] = rs.sub_count(nb);
        }
        if (total) *total = rs.count();
        return 0;
    } catch (...) { return 1; }
}

/* count_to (src/bm.h:3120) and select (src/bm.h:5350) with the reference's own rs_index */
int ref_rank_select(const bmb200_packed_set* s, uint32_t v,
                    const uint64_t* pos, uint64_t n_pos, uint64_t* rank_out,
                    const uint64_t* rank, uint64_t n_rank, uint64_t* pos_out, uint8_t* found,
                    double* sec_build, double* sec_rank, double* sec_select)
{
    try {
        bvect a;
        build_bvector(s, v, 0, s->n_blocks, a);
        bvect::rs_index_type rs;
        auto t0 = std::chrono::steady_clock::now();
        a.build_rs_index(&rs);
        auto t1 = std::chrono::steady_clock::now();
        for (uint64_t q = 0; q < n_pos; ++q) {
            uint64_t p = pos[q];
            if (p >= (uint64_t)bm::id_max) p = bm::id_max - 1;
            rank_out[q] = a.count_to((bvect::size_type)p, rs);
        }
        auto t2 = std::chrono::steady_clock::now();
        for (uint64_t q = 0; q < n_rank; ++q) {
            bvect::size_type p = 0;
            bool f = a.select((bvect::size_type)rank[q], p, rs);
            found[q] = f ? 1 : 0; pos_out[q] = f ? (uint64_t)p : 0;
        }
        auto t3 = std::chrono::steady_clock::now();
        if (sec_build)  *sec_build  = std::chrono::duration<double>(t1 - t0).count();
        if (sec_rank)   *sec_rank   = std::chrono::duration<double>(t2 - t1).count();
        if (sec_select) *sec_select = std::chrono::duration<double>(t3 - t2).count();
        return 0;
    } catch (...) { return 1; }
}

/*
 * aggregator::pipeline (src/bmaggregator.h:222-341) executed by combine_and_sub(TPipe&) (:1291-1453) on the real
 * reference, options agg_opt_bvect_and_counts: per-group result vectors + counts, optional OR target.
 * members/offsets as in bmb200_batch_args.  Outputs: counts[n_groups]; kind/popcnt/blocks for n_groups*n_blocks
 * columns (group-major); or_kind/or_blocks for the OR target (n_blocks columns) when want_or != 0.
 */
int ref_pipeline(const bmb200_packed_set* s, uint32_t n_groups, const uint32_t* members, const uint32_t* offsets, int want_or,
                 uint64_t* counts, uint8_t* kind, uint32_t* popcnt, uint32_t* blocks, uint8_t* or_kind, uint32_t* or_blocks)
{
    try {
        std::vector<std::unique_ptr<bvect>> own(s->n_vec);
        auto get = [&](uint32_t v) -> const bvect* {
            if (!own[v]) { own[v].reset(new bvect()); build_bvector(s, v, 0, s->n_blocks, *own[v]); }
            return own[v].get();
        };
        bm::aggregator<bvect> agg;
        bm::aggregator<bvect>::pipeline<bm::agg_opt_bvect_and_counts> pipe;
        bvect bv_or;
        if (want_or) { bv_or.init(); pipe.set_or_target(&bv_or); }
        for (uint32_t g = 0; g < n_groups; ++g) {
            bm::aggregator<bvect>::arg_groups* args = pipe.add();
            for (uint32_t k = offsets[2 * g]; k < offsets[2 * g + 1]; ++k) args->add(get(members[k]), 0);
            for (uint32_t k = offsets[2 * g + 1]; k < offsets[2 * g + 2]; ++k) args->add(get(members[k]), 1);
        }
        pipe.complete();
        agg.combine_and_sub(pipe);
        auto& res = pipe.get_bv_res_vector();
        auto& cnt = pipe.get_bv_count_vector();
        for (uint32_t g = 0; g < n_groups; ++g) {
            if (counts) counts[g] = (uint64_t)cnt[g];
            const bvect* bv = res[g];
            size_t o = (size_t)g * s->n_blocks;
            if (bv) export_bvector(*bv, s->n_blocks, kind ? kind + o : 0, popcnt ? popcnt + o : 0,
                                   blocks ? blocks + o * BMB200_BLOCK_WORDS : 0, 0);
            else {
                if (kind) std::memset(kind + o, 0, s->n_blocks);
                if (popcnt) std::memset(popcnt + o, 0, sizeof(uint32_t) * s->n_blocks);
                if (blocks) std::memset(blocks + o * BMB200_BLOCK_WORDS, 0, (size_t)s->n_blocks * BMB200_BLOCK_BYTES);
            }
        }
        if (want_or) export_bvector(bv_or, s->n_blocks, or_kind, 0, or_blocks, 0);
        return 0;
    } catch (...) { return 1; }
}

/*
 * bm::sparse_vector<unsigned, bvector<>> + bm::sparse_vector_scanner<> (src/bmsparsevec.h, src/bmsparsevec_algo.h:1083-1182)
 * on the real reference.  values[n] (+ optional nulls[n] != 0 => set_null) -> optimize()d sparse vector.
 *   ref_sv_planes: the vector's own bit-planes (get_slice(j), j < effective_slices()) and, last, the searchable
 *                  universe (NOT-NULL plane of a nullable vector, else [0, n)) as per-column kind / blocks / GAP words,
 *                  (n_planes + 1) * n_cols columns, plane-major -- the GPU scan runs on exactly these blocks.
 *   ref_sv_scan:   pred = BMB200_SCAN_*; one result vector per search value (RANGE: (lo, hi) pairs), value-major.
 */
typedef bm::sparse_vector<unsigned, bvect> svect;

static void build_sv(svect& sv, const uint32_t* values, const uint8_t* nulls, uint64_t n)
{
    sv.resize((svect::size_type)n);
    for (uint64_t i = 0; i < n; ++i) {
        if (nulls && nulls[i]) continue;             /* stays NULL (resize(.., set_null)) */
        sv.set((svect::size_type)i, values[i]);
    }
    BM_DECLARE_TEMP_BLOCK(tb)
    sv.optimize(tb);
}

int ref_sv_planes(const uint32_t* values, const uint8_t* nulls, uint64_t n, uint32_t n_cols, uint32_t max_planes,
                  uint32_t* n_planes_out, uint8_t* kind, uint32_t* blocks, uint16_t* gaps)
{
    try {
        svect sv(nulls ? bm::use_null : bm::no_null);
        build_sv(sv, values, nulls, n);
        unsigned np = sv.effective_slices();
        while (np > 1 && !sv.get_slice(np - 1)) --np;           /* trailing absent planes carry no bits */
        if (np > max_planes) return 3;
        *n_planes_out = np;
        bvect empty;
        for (unsigned j = 0; j <= np; ++j) {
            const bvect* bv;
            bvect uni;
            if (j < np) bv = sv.get_slice(j);
            else if (nulls) bv = sv.get_null_bvector();
            else { if (n) uni.set_range(0, (bvect::size_type)(n - 1)); uni.optimize(); bv = &uni; }
            size_t o = (size_t)j * n_cols;
            export_bvector(bv ? *bv : empty, n_cols, kind + o, 0, blocks + o * BMB200_BLOCK_WORDS, gaps + o * BMB200_GAP_MAX_WORDS);
        }
        return 0;
    } catch (...) { return 1; }
}

int ref_sv_scan(const uint32_t* values, const uint8_t* nulls, uint64_t n, int pred, const uint32_t* search, uint32_t n_search,
                uint32_t n_cols, uint64_t* counts, uint8_t* kind, uint32_t* popcnt, uint32_t* blocks)
{
    try {
        svect sv(nulls ? bm::use_null : bm::no_null);
        build_sv(sv, values, nulls, n);
        bm::sparse_vector_scanner<svect> scanner;
        for (uint32_t k = 0; k < n_search; ++k) {
            bvect bv;
            switch (pred) {
            case BMB200_SCAN_EQ: scanner.find_eq(sv, search[k], bv); break;
            case BMB200_SCAN_GT: scanner.find_gt(sv, search[k], bv); break;
            case BMB200_SCAN_GE: scanner.find_ge(sv, search[k], bv); break;
            case BMB200_SCAN_LT: scanner.find_lt(sv, search[k], bv); break;
            case BMB200_SCAN_LE: scanner.find_le(sv, search[k], bv); break;
            case BMB200_SCAN_RANGE: scanner.find_range(sv, search[2 * k], search[2 * k + 1], bv); break;
            default: return 2;
            }
            if (counts) counts[k] = (uint64_t)bv.count();
            size_t o = (size_t)k * n_cols;
            export_bvector(bv, n_cols, kind ? kind + o : 0, popcnt ? popcnt + o : 0, blocks ? blocks + o * BMB200_BLOCK_WORDS : 0, 0);
        }
        return 0;
    } catch (...) { return 1; }
}

/*
 * bm::serializer<> / bm::deserialize (src/bmserial.h) on the real reference.
 *   ref_serialize:   vector v of the packed set -> BLOB at the given compression level (serializer::set_compression_level,
 *                    :1454), default header (byte order + GAP levels).  *size = bytes written (<= cap).
 *   ref_deserialize: BLOB -> bvector (bm::deserialize, :4152) -> per-column kind / popcount / bits / GAP words.
 */
int ref_serialize(const bmb200_packed_set* s, uint32_t v, int level, unsigned char* out, uint64_t cap, uint64_t* size)
{
    try {
        bvect bv; build_bvector(s, v, 0, s->n_blocks, bv);
        bm::serializer<bvect> ser;
        ser.set_compression_level((unsigned)level);
        bm::serializer<bvect>::buffer buf;
        ser.serialize(bv, buf);
        if (buf.size() > cap) return 3;
        std::memcpy(out, buf.data(), buf.size());
        *size = buf.size();
        return 0;
    } catch (...) { return 1; }
}

/* same with serializer::set_bookmarks(true, interval) (src/bmserial.h:1487): skip marks every `interval` blocks */
int ref_serialize_bookmarks(const bmb200_packed_set* s, uint32_t v, int level, uint32_t interval, unsigned char* out, uint64_t cap, uint64_t* size)
{
    try {
        bvect bv; build_bvector(s, v, 0, s->n_blocks, bv);
        bm::serializer<bvect> ser;
        ser.set_compression_level((unsigned)level);
        ser.set_bookmarks(true, interval);
        bm::serializer<bvect>::buffer buf;
        ser.serialize(bv, buf);
        if (buf.size() > cap) return 3;
        std::memcpy(out, buf.data(), buf.size());
        *size = buf.size();
        return 0;
    } catch (...) { return 1; }
}

int ref_deserialize(const unsigned char* blob, uint32_t n_cols, uint8_t* kind, uint32_t* popcnt, uint32_t* blocks, uint16_t* gaps)
{
    try {
        bvect bv;
        bm::deserialize(bv, blob);
        export_bvector(bv, n_cols, kind, popcnt, blocks, gaps);
        return 0;
    } catch (...) { return 1; }
}

/* wall time (seconds, best of `repeats`) of the n_search scanner calls alone -- the vector is built and optimize()d
 * before the clock starts; total = sum of result cardinalities */
int ref_sv_time_scan(const uint32_t* values, const uint8_t* nulls, uint64_t n, int pred, const uint32_t* search, uint32_t n_search,
                     int repeats, double* best_sec, uint64_t* total)
{
    try {
        svect sv(nulls ? bm::use_null : bm::no_null);
        build_sv(sv, values, nulls, n);
        bm::sparse_vector_scanner<svect> scanner;
        double best = 1e30; uint64_t tot = 0;
        for (int r = 0; r < repeats; ++r) {
            tot = 0;
            auto t0 = std::chrono::steady_clock::now();
            for (uint32_t k = 0; k < n_search; ++k) {
                bvect bv;
                switch (pred) {
                case BMB200_SCAN_EQ: scanner.find_eq(sv, search[k], bv); break;
                case BMB200_SCAN_GT: scanner.find_gt(sv, search[k], bv); break;
                case BMB200_SCAN_GE: scanner.find_ge(sv, search[k], bv); break;
                case BMB200_SCAN_LT: scanner.find_lt(sv, search[k], bv); break;
                case BMB200_SCAN_LE: scanner.find_le(sv, search[k], bv); break;
                case BMB200_SCAN_RANGE: scanner.find_range(sv, search[2 * k], search[2 * k + 1], bv); break;
                default: return 2;
                }
                tot += (uint64_t)bv.count();
            }
            double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            if (sec < best) best = sec;
        }
        *best_sec = best; *total = tot;
        return 0;
    } catch (...) { return 1; }
}

/*
 * CPU baseline timing.  The reference aggregator is single-threaded; for an all-cores figure each of
 * `threads` workers owns its own bm::aggregator and its own copy of the inputs restricted to a
 * contiguous range of block columns (BASELINE.md section 3).  Columns [nb_from, nb_to) are split evenly.
 * Returns the best-of-`repeats` wall time (seconds) for ONE pass over all the columns, and the total
 * popcount of the result (so the work cannot be optimised away).
 */
int ref_time_aggregate(const bmb200_packed_set* s, const bmb200_agg_args* a,
                       int threads, int repeats, double* best_sec, uint64_t* total_bits)
{
    try {
        uint32_t nb_to = a->nb_to ? a->nb_to : s->n_blocks;
        uint32_t ncols = nb_to - a->nb_from;
        if (threads < 1) threads = 1;
        if ((uint32_t)threads > ncols) threads = (int)ncols;
        std::vector<Built> built(threads);
        std::vector<uint32_t> lo(threads), hi(threads);
        for (int t = 0; t < threads; ++t) {
            lo[t] = a->nb_from + (uint32_t)((uint64_t)ncols * t / threads);
            hi[t] = a->nb_from + (uint32_t)((uint64_t)ncols * (t + 1) / threads);
        }
        {   /* input construction is setup, not timed; done in parallel */
            std::vector<std::thread> th;
            for (int t = 0; t < threads; ++t)
                th.emplace_back([&, t]() { build_groups(s, a, lo[t], hi[t], built[t]); });
            for (auto& x : th) x.join();
        }
        double best = 1e30; uint64_t tot = 0;
        for (int r = 0; r < repeats; ++r) {
            std::vector<uint64_t> cnt(threads, 0);
            auto t0 = std::chrono::steady_clock::now();
            std::vector<std::thread> th;
            for (int t = 0; t < threads; ++t)
                th.emplace_back([&, t]() {
                    bm::aggregator<bvect> agg;
                    bvect target;
                    run_op(agg, a, built[t], target);
                    cnt[t] = target.count();
                });
            for (auto& x : th) x.join();
            auto t1 = std::chrono::steady_clock::now();
            double sec = std::chrono::duration<double>(t1 - t0).count();
            if (sec < best) best = sec;
            tot = 0; for (auto c : cnt) tot += c;
        }
        if (best_sec) *best_sec = best;
        if (total_bits) *total_bits = tot;
        return 0;
    } catch (...) { return 1; }
}

/*
 * Persistent timing / parity job: the bvectors are built ONCE (per worker: its contiguous range of block columns of every
 * source vector), every ref_job_run pass runs the reference aggregator on all workers, and ref_job_export walks the
 * result of the last pass into per-column kind / popcount / digest (calc_block_digest0, src/bmfunc.h:1239) / GAP length.
 * Workers = T = `threads` (BASELINE.md section 3: one bm::aggregator per thread over a contiguous range of block indices).
 */
struct RefJob {
    bmb200_agg_args a;
    std::vector<uint32_t> g0, g1;
    std::vector<Built> built;
    std::vector<uint32_t> lo, hi;
    std::vector<std::unique_ptr<bvect>> target;
    uint32_t nb_from = 0, ncols = 0;
};

void* ref_job_create(const bmb200_packed_set* s, const bmb200_agg_args* a, int threads)
{
    try {
        /* the workers build ~13 GB of 8 KB / sub-KB blocks through malloc at the same time: let every malloc arena grow in 64 MB
         * steps instead of 128 KB ones (each step is an mprotect under the process-wide mmap lock, which also stalls page faults) */
        mallopt(M_TOP_PAD, 64 << 20);
        std::unique_ptr<RefJob> j(new RefJob());
        j->a = *a;
        j->g0.assign(a->group0, a->group0 + a->n0); j->a.group0 = j->g0.data();
        if (a->op == BMB200_OP_AND_SUB && a->n1) { j->g1.assign(a->group1, a->group1 + a->n1); j->a.group1 = j->g1.data(); }
        else { j->a.group1 = 0; j->a.n1 = 0; }
        uint32_t nb_to = a->nb_to ? a->nb_to : s->n_blocks;
        j->nb_from = a->nb_from; j->ncols = nb_to - a->nb_from;
        if (threads < 1) threads = 1;
        if ((uint32_t)threads > j->ncols) threads = (int)j->ncols;
        j->built.resize(threads); j->lo.resize(threads); j->hi.resize(threads); j->target.resize(threads);
        /* whole 256-block superblocks per worker whenever there are at least `threads` of them: the reference walks all 256
         * sub-blocks of every top-level block it touches (src/bmaggregator.h:1565-1566), so a finer split makes it do extra work */
        const uint32_t nsb = j->ncols / 256u;
        const bool aligned = (j->ncols % 256u == 0) && nsb >= (uint32_t)threads;
        for (int t = 0; t < threads; ++t) {
            if (aligned) { j->lo[t] = a->nb_from + 256u * (uint32_t)((uint64_t)nsb * t / threads); j->hi[t] = a->nb_from + 256u * (uint32_t)((uint64_t)nsb * (t + 1) / threads); }
            else { j->lo[t] = a->nb_from + (uint32_t)((uint64_t)j->ncols * t / threads); j->hi[t] = a->nb_from + (uint32_t)((uint64_t)j->ncols * (t + 1) / threads); }
            j->target[t].reset(new bvect());
        }
        std::vector<std::thread> th;
        RefJob* jp = j.get();
        for (int t = 0; t < threads; ++t)
            th.emplace_back([jp, s, t]() { build_groups(s, &jp->a, jp->lo[t], jp->hi[t], jp->built[t]); });
        for (auto& x : th) x.join();
        return j.release();
    } catch (...) { return 0; }
}

int ref_job_threads(void* job) { return job ? (int)((RefJob*)job)->built.size() : 0; }

/* one timed pass per repeat: all workers run the reference entry point on their range; sec[r] = wall time of pass r */
int ref_job_run(void* job, int repeats, double* sec, uint64_t* total_bits)
{
    if (!job) return 2;
    try {
        RefJob* j = (RefJob*)job;
        const int T = (int)j->built.size();
        uint64_t tot = 0;
        for (int r = 0; r < repeats; ++r) {
            std::vector<uint64_t> cnt(T, 0);
            auto t0 = std::chrono::steady_clock::now();
            std::vector<std::thread> th;
            for (int t = 0; t < T; ++t)
                th.emplace_back([j, &cnt, t]() {
                    bm::aggregator<bvect> agg;
                    run_op(agg, &j->a, j->built[t], *j->target[t]);
                    cnt[t] = j->target[t]->count();
                });
            for (auto& x : th) x.join();
            auto t1 = std::chrono::steady_clock::now();
            if (sec) sec[r] = std::chrono::duration<double>(t1 - t0).count();
            tot = 0; for (auto c : cnt) tot += c;
        }
        if (total_bits) *total_bits = tot;
        return 0;
    } catch (...) { return 1; }
}

int ref_job_export(void* job, uint8_t* kind, uint32_t* popcnt, uint64_t* digest, uint32_t* gap_len)
{
    if (!job) return 2;
    try {
        RefJob* j = (RefJob*)job;
        const int T = (int)j->built.size();
        std::vector<std::thread> th;
        for (int t = 0; t < T; ++t)
            th.emplace_back([=]() {
                const bvect& bv = *j->target[t];
                const bvect::blocks_manager_type& bman = bv.get_blocks_manager();
                BM_DECLARE_TEMP_BLOCK(tb)
                for (uint32_t c = j->lo[t]; c < j->hi[t]; ++c)
                {
                    uint32_t lc = c - j->lo[t], oc = c - j->nb_from;
                    unsigned i = lc >> 8, jj = lc & 255u;
                    const bm::word_t* blk = 0;
                    if (bman.is_init() && i < bman.top_block_size()) blk = bman.get_block_ptr(i, jj);
                    uint8_t kd; uint32_t pc = 0, gl = 0; uint64_t dg = 0;
                    if (!blk) kd = BMB200_BLK_NULL;
                    else if (blk == FULL_BLOCK_FAKE_ADDR || blk == FULL_BLOCK_REAL_ADDR) { kd = BMB200_BLK_FULL; pc = 65536; dg = ~0ull; }
                    else if (BM_IS_GAP(blk)) {
                        const bm::gap_word_t* g = BMGAP_PTR(blk);
                        kd = BMB200_BLK_GAP; pc = bm::gap_bit_count_unr(g); gl = bm::gap_length(g) - 1;
                        bm::gap_convert_to_bitset(tb.begin(), g); dg = bm::calc_block_digest0(tb.begin());
                    }
                    else { kd = BMB200_BLK_BIT; pc = bm::bit_block_count(blk); dg = bm::calc_block_digest0(blk); }
                    if (kind) kind[oc] = kd;
                    if (popcnt) popcnt[oc] = pc;
                    if (digest) digest[oc] = dg;
                    if (gap_len) gap_len[oc] = gl;
                }
            });
        for (auto& x : th) x.join();
        return 0;
    } catch (...) { return 1; }
}

void ref_job_free(void* job) { delete (RefJob*)job; }

} // extern "C"
