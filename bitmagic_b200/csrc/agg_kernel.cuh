// agg_kernel.cuh -- N-way block-column aggregation kernel (OR / AND / AND-SUB / XOR) for sm_90a.
//
// Replaces, for one block column (i,j) per CTA iteration, the reference's
//   sort_input_blocks_or/_and      src/bmaggregator.h:2278-2366   (classification pass, ordered compaction)
//   process_bit_blocks_or/_and/_sub src/bmaggregator.h:1924-2205  (bit phase, register accumulator)
//   process_gap_blocks_or/_and/_sub src/bmaggregator.h:1808-1890  (GAP phase, run scatter into smem)
//   bit_block_count / calc_block_digest0 / bit_block_calc_change  src/bmfunc.h:5808,1239,6040 (epilogue)
//   the classification half of opt_copy_bit_block                 src/bmblocks.h:1355-1409
//
// Layout / mapping:
//   * persistent CTAs (grid = SMs x 2) pull block columns from an atomic counter (claimed one column ahead), so
//     skewed columns (NULL / GAP / bit mixes) balance themselves;
//   * 512 threads own the 8 KB accumulator in registers: thread t holds words [4t, 4t+4) as one uint4,
//     every source bit-block is consumed with one coalesced 128-bit streaming load per thread,
//     4 blocks in flight per thread (32 KB per CTA);
//   * GAP sources are never expanded on their own.  The column's GAP segment is contiguous in the arena
//     (column-major layout), so it is streamed with cp.async.bulk (TMA) into a 64 KB shared-memory ring tracked
//     by mbarriers -- without a single LSU global load.
//     The bit phase runs first and is folded into an 8 KB "live" mask L in shared memory; GAP runs then only
//     ever CLEAR bits of L (red.shared.and), so a run whose word of L is already dead costs one shared load
//     and no atomic (the reference gets the same effect from its digest, src/bmfunc.h:7615):
//         OR      : L = ~U,      selected runs = 1-runs,                       R = ~L
//         AND-SUB : L = P & ~U,  selected runs = 0-runs of AND-group GAPs and
//                                                1-runs of SUB-group GAPs,     R = L
//         XOR     : L = X,       runs are XOR-ed in (red.shared.xor),          R = L
//     Two consumers of the ring:
//       - FLAT (OR sources / SUB group): when every GAP block of the streamed window belongs to the list and is
//         stored in the BMB200_DESC_GAP_FLAT form, the window is just an array of aligned (prev_end, end) u16
//         pairs -- headers, pads and tail fill decode to empty runs.  The ring is cut into two private 2 KB slots
//         per warp (one mbarrier each); warps claim 4 KB pieces of the window from a shared counter, refill their
//         own slots and eat them with 128-bit shared loads, 4 runs per load: no per-block bookkeeping, no
//         cross-warp hand-off;
//       - per block (AND-group GAPs, XOR, subsets of the pool, raw GAP layout): 16 KB chunks in a 4-stage ring,
//         16 lanes share one GAP block, the warp that finishes a chunk last re-arms its stage (no producer warp).
//     Unsorted / sparse member lists fall back to per-block gathers from global memory.
//   * epilogue fuses popcount, 64-wave digest, run count and the result-kind decision.
#pragma once
#include "common.cuh"
#include "coverage_kernel.cuh"
#include <type_traits>

namespace bmb200 {

constexpr int kAggThreads = 512;
constexpr int kAggWarps   = kAggThreads / 32;
constexpr int kAggChunk   = 1024;   // group members classified per pass (AND-SUB)
constexpr int kAggChunkWide = 1408; // ... in the one-group kernels (OR / AND / XOR)

constexpr int      kCtasPerSm     = 2;                             // resident CTAs per SM agg_kernel is shaped for (64 registers)
constexpr int      kBitUnroll     = 4;                             // bit-blocks in flight per thread
constexpr uint32_t kLanesPerBlock = 16;                            // lanes that share one GAP block in the streamed scatter
constexpr uint32_t kGroupsPerWarp = 32u / kLanesPerBlock;          // `lane` below = lane inside its group
constexpr uint32_t kVarSleepNs    = 64;                            // back-off of an mbarrier wait
constexpr int      kGapStages     = 4;
constexpr uint32_t kGapChunkBytes = 16384;
constexpr uint32_t kRingBytes     = kGapStages * kGapChunkBytes;   // 64 KB; offsets wrap by modulo
constexpr uint32_t kGapMaxBytes   = 2560;                          // gap_max_buff_len * 2
constexpr uint32_t kRingTail      = kGapMaxBytes + 512;           // tail mirror (+ over-read slack of one 64-run step)
constexpr size_t   kAggRingSmem   = kRingBytes + kRingTail;       // blocks never wrap
// dynamic shared memory of agg_kernel: [pad to the next 8 KB boundary of the shared WINDOW][live mask L, 8 KB][ring + tail].
// L must be 8 KB aligned in window addresses (flat_quad forms word addresses with one and-or); static shared memory starts at
// window offset = the driver's reserved bytes (1 KB on sm_90), so the pad depends on the kernel's static size -- the host
// computes it (agg_dyn_smem) and the kernel re-derives the position from the real address.
constexpr uint32_t kLiveAlign     = 8192u;
__host__ inline size_t agg_dyn_smem(size_t static_bytes, size_t reserved_bytes, size_t ring_bytes = kAggRingSmem)
{
    const size_t start = reserved_bytes + static_bytes;                   // window offset of the dynamic region (before its own alignment)
    const size_t start_al = (start + 127) & ~(size_t)127;
    const size_t k_at = (start_al + kLiveAlign - 1) & ~(size_t)(kLiveAlign - 1);
    return (k_at - start) + kLiveAlign + ring_bytes + 128;
}
// FLAT consumer: the ring is cut into one private slot per warp; warp w streams chunks w, w+16, ... of the window through
// its own slot and its own mbarrier -- no cross-warp hand-off, the per-chunk overhead is paid once per slot, not 16 times
constexpr uint32_t kFlatSlots     = 2u;                                      // barriers per warp (the most slots a warp's region is cut into)
constexpr uint32_t kFlatWarpBytes = kRingBytes / kAggWarps;                  // 4 KB of the 64 KB ring per warp
static_assert(kFlatWarpBytes % 2048u == 0, "a warp's ring region is cut into 1 or 2 slots of whole KB");
// The region is used as TWO 2 KB slots (one fills while the other is consumed) or as ONE 4 KB slot, chosen per window: the per-slot
// control code (claim, mbarrier wait, refill) is ~18 % of the GAP-phase instructions with 2 KB slots, so long windows (config 5: 2.7 MB
// per column) take 4 KB pieces; short ones (config 3: ~0.4 MB per column = 6 pieces per warp) keep 2 KB pieces, whose finer claim
// granularity balances the 16 warps better.
constexpr uint32_t kFlatBigWindow = 640u << 10;                              // >= 10 pieces of 4 KB for each of the 16 warps

struct AggParams {
    SetView   set;
    const uint32_t* group;     // device: member vector ids of all argument groups, concatenated
    const uint32_t* goff;      // device [2*n_groups+1]: group g = members [goff[2g], goff[2g+1]) (group0) + [goff[2g+1], goff[2g+2]) (group1)
    uint32_t  n_groups;        // 1 for a plain aggregate, > 1 for a pipeline batch
    uint32_t  nb_from, n_cols;
    uint32_t  compress;        // classify like opt_copy_bit_block(opt_compress)
    uint32_t  store_blocks;    // 0 = counts only
    uint32_t  gap_mode;        // 0 = auto (stream when sorted), 1 = always gather
    uint32_t  dyn_bytes;       // dynamic shared memory the launch was given (checked against the aligned layout)
    uint32_t  binary;          // 0 = aggregator semantics; 1 + BINOP_* = two-operand bvector op (result kinds follow combine_operation_block_*)
    uint64_t  gap_pool_bytes;  // readable bytes of gap_pool (including the allocation slack)
    uint32_t* blocks;          // [n_cols][2048]
    uint32_t* popcnt;          // [n_cols]
    uint64_t* digest;          // [n_cols]
    uint32_t* nruns;           // [n_cols]
    uint8_t*  kind;            // [n_cols]
    uint16_t* gaps;            // [n_cols][1280] GAP form of the columns classified GAP (compress mode), else null
    unsigned long long* total; // [n_groups] sum of popcounts per argument group
    uint32_t* or_blocks;       // [n_cols][2048] OR of every group's result (pipeline set_or_target), or null
    uint32_t* work_counter;    // zeroed before launch
};

// flag bits collected while classifying
constexpr uint32_t kFlNull0 = 1u;   // a NULL block in group0
constexpr uint32_t kFlFull0 = 2u;   // a FULL block in group0
constexpr uint32_t kFlFull1 = 4u;   // a FULL block in group1 (SUB)
constexpr uint32_t kRelMask = BMB200_DESC_REL_MASK;   // list entries are desc >> 2: unit in the low 28 bits, FLAT in bit 28, pad in bit 29
constexpr uint32_t kEntFlat = BMB200_DESC_GAP_FLAT >> 2;
constexpr uint32_t kFlatMinBlocks = 16u;              // shorter lists take the per-block path

// ---- mbarrier / bulk-copy primitives (PTX; SASS: SYNCS.*, UBLKCP) ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
// The raw forms take 32-bit shared-window addresses (callers that keep them in registers); the others convert a generic pointer.
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) { mbar_arrive_expect_tx(smem_u32(bar), bytes); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "nanosleep.u32 %2;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t}\n" :: "r"(bar), "r"(parity), "n"(kVarSleepNs) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) { mbar_wait(smem_u32(bar), parity); }
__device__ __forceinline__ uint32_t atoms_add(uint32_t a, uint32_t v)
{
    uint32_t old; asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(a), "r"(v) : "memory"); return old;
}
__device__ __forceinline__ void sts32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void bulk_g2s(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_dst), "l"(gsrc), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar)
{
    bulk_g2s(smem_u32(smem_dst), gsrc, bytes, smem_u32(bar));
}
__device__ __forceinline__ void fence_proxy_async()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar, uint32_t count = 1u)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
// Block barrier over the NT threads that compute a column: the whole CTA (__syncthreads) in agg_kernel, named barrier 1
// over the consumer warps in agg_pipe_kernel (PIPE), whose producer warp never joins it.
template <bool PIPE, int NT = kAggThreads>
__device__ __forceinline__ void agg_sync()
{
    if (PIPE) asm volatile("bar.sync 1, %0;" :: "n"(NT) : "memory");
    else      __syncthreads();
}

// raw 32-bit shared-window addresses keep the scatter loop free of generic->shared conversions
__device__ __forceinline__ uint32_t lds32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t lds16(uint32_t a) { uint16_t v; asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(a)); return (uint32_t)v; }
__device__ __forceinline__ uint4 lds128(uint32_t a)
{
    uint4 v; asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a)); return v;
}
__device__ __forceinline__ void reds_and(uint32_t a, uint32_t v) { asm volatile("red.shared.and.b32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void reds_xor(uint32_t a, uint32_t v) { asm volatile("red.shared.xor.b32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
// mask of `width` bits starting at bit `pos` (pos < 32; bits beyond bit 31 are dropped) -- SASS BMSK
__device__ __forceinline__ uint32_t bmsk(uint32_t pos, uint32_t width)
{
    uint32_t m; asm("bmsk.clamp.b32 %0, %1, %2;" : "=r"(m) : "r"(pos), "r"(width)); return m;
}

template <int OP>
__device__ __forceinline__ void acc_apply0(uint4& a, const uint4& v)
{
    if (OP == BMB200_OP_OR)       { a.x |= v.x; a.y |= v.y; a.z |= v.z; a.w |= v.w; }
    else if (OP == BMB200_OP_XOR) { a.x ^= v.x; a.y ^= v.y; a.z ^= v.z; a.w ^= v.w; }
    else                          { a.x &= v.x; a.y &= v.y; a.z &= v.z; a.w &= v.w; }
}
__device__ __forceinline__ void acc_or(uint4& a, const uint4& v)
{
    a.x |= v.x; a.y |= v.y; a.z |= v.z; a.w |= v.w;
}

// stream `n` bit-blocks of this column (indices in lst[], relative to the column's bit segment)
template <int OP, bool ROLE1>
__device__ __forceinline__ void bit_phase(const uint4* __restrict__ seg, const uint32_t* lst, uint32_t n, uint4& acc)
{
    const uint4 ident = (!ROLE1 && (OP == BMB200_OP_AND || OP == BMB200_OP_AND_SUB))
                            ? make_uint4(~0u, ~0u, ~0u, ~0u) : make_uint4(0u, 0u, 0u, 0u);
    for (uint32_t i = 0; i < n; i += kBitUnroll) {
        uint4 v[kBitUnroll];
#pragma unroll
        for (int u = 0; u < kBitUnroll; ++u) {
            if (i + u < n) v[u] = ld_stream_v4(seg + (size_t)lst[i + u] * (kBlockWords / 4));
            else           v[u] = ident;
        }
#pragma unroll
        for (int u = 0; u < kBitUnroll; ++u) {
            if (ROLE1) acc_or(acc, v[u]); else acc_apply0<OP>(acc, v[u]);
        }
    }
}

// apply one run [s, e] (inclusive bit positions) to the live mask L (Ls = its shared-window address):
// clear the bits (OR / AND / AND-SUB) or flip them (XOR)
template <bool XOR>
__device__ __forceinline__ void apply_word(uint32_t a, uint32_t m)
{
    if (XOR) reds_xor(a, m); else reds_and(a, ~m);
}
template <bool XOR>
__device__ __forceinline__ void apply_run(uint32_t Ls, uint32_t s, uint32_t e)
{
    const uint32_t ws = s >> 5, we = e >> 5;
    const uint32_t m0 = 0xffffffffu << (s & 31u);
    const uint32_t m1 = 0xffffffffu >> (31u - (e & 31u));
    if (ws == we) {
        apply_word<XOR>(Ls + ws * 4u, m0 & m1);
    } else {
        apply_word<XOR>(Ls + ws * 4u, m0);
        apply_word<XOR>(Ls + we * 4u, m1);
        for (uint32_t w = ws + 1; w < we; ++w) apply_word<XOR>(Ls + w * 4u, 0xffffffffu);
    }
}

// FLAT consumer: one aligned u32 of a flat window = (prev_end, end) of a 1-run, or a header / pad / fill pair
// (prev_end >= end: nothing to do).  Four pairs per call, branch-free on the common path: the mask of an empty
// pair is 0, the atomic is predicated, and only runs that continue past their first word take the slow branch.
// TEST: look at the word of L first -- bits only ever get cleared, so a stale read can only cause a redundant
// atomic, never a missed one.
__device__ __forceinline__ void reds_and_if(uint32_t a, uint32_t v, uint32_t cond)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\t@p red.shared.and.b32 [%0], %1;\n\t}"
                 :: "r"(a), "r"(v), "r"(cond) : "memory");
}
__device__ __forceinline__ void flat_pair_tail(uint32_t Ls, uint32_t w)   // words after the first of a long run
{
    const uint32_t lo = w & 0xffffu, hi = w >> 16;
    if (lo >= hi) return;
    const uint32_t s = lo + 1u, sb = s & 31u, wd = hi - lo;
    if (sb + wd <= 32u) return;
    uint32_t rem = sb + wd - 32u;
    uint32_t a = Ls + ((s >> 5) << 2) + 4u;
    for (; rem >= 32u; rem -= 32u, a += 4u) reds_and(a, 0u);
    if (rem) reds_and(a, 0xffffffffu << rem);
}
__device__ __noinline__ void flat_quad_tail(uint32_t Ls, const uint4 q)   // rare: some run of the quad continues past its first word
{
    flat_pair_tail(Ls, q.x); flat_pair_tail(Ls, q.y); flat_pair_tail(Ls, q.z); flat_pair_tail(Ls, q.w);
}
// Pair decode: hi - lo by one dp2a, word address by one and-or (L is 8 KB aligned).
// hi16(w) - lo16(w) in one instruction: dp2a.lo = c + lo16(a) * sbyte0(b) + hi16(a) * sbyte1(b) with b = (+1, -1)   (SASS IDP.2A)
__device__ __forceinline__ int pair_width(uint32_t w)
{
    int d; asm("dp2a.lo.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(w), "r"(0x000001ffu), "r"(0)); return d;
}
// ((x & 0x1ffc) | base): one LOP3 (base = shared address of L, 8 KB aligned, so the OR is the add)
__device__ __forceinline__ uint32_t and_or(uint32_t x, uint32_t msk, uint32_t base)
{
    uint32_t r; asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(r) : "r"(x), "r"(msk), "r"(base)); return r;
}
// MODE 0: L is mostly alive -- every run goes straight to its (predicated) atomic.  MODE 1: test-first.
// (A third form that OR-ed the four hit tests of a quad behind ONE branch was slower on C5 and dropped: the
// extra divergence costs more than the skipped instructions.)
template <int MODE>
__device__ __forceinline__ void flat_quad(uint32_t Ls, const uint4& q)
{
    constexpr bool TEST = MODE != 0;
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
    uint32_t a[4], m[4], nm[4], reach = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const uint32_t t = w[i] + 1u;                                         // low half = run start s = lo + 1 (s == 65536 wraps to 0: pad / terminator, mask 0)
        const uint32_t sb = t & 31u;
        const uint32_t wd = (uint32_t)max(pair_width(w[i]), 0);               // wd == 0: no run
        m[i] = bmsk(sb, wd);
        nm[i] = ~m[i];
        a[i] = and_or(t >> 3, 0x1ffcu, Ls);
        reach = max(reach, sb + wd);
    }
    if (TEST) {
        uint32_t v[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) v[i] = lds32(a[i]) & m[i];
#pragma unroll
        for (int i = 0; i < 4; ++i) reds_and_if(a[i], nm[i], v[i]);
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) reds_and_if(a[i], nm[i], m[i]);
    }
    if (reach > 32u) flat_quad_tail(Ls, q);
}

// Singles of the run-list companion (runlist_kernel.cuh): one word unit per 128-bit load, 23 five-bit offsets inside one word of L
// OR-ed into one mask, one atomic per unit.  The units are dealt out by bank, so a warp's atomic is one shared-memory wavefront in a
// part's full rounds.
__device__ __forceinline__ void sgl_unit(uint32_t Ls, const uint4& q)
{
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
    uint32_t m = 0;
#pragma unroll
    for (int f = 0; f < 23; ++f) m |= 1u << ((w[f / 6] >> (5 * (f % 6))) & 31u);
    const uint32_t word = (q.x >> 30) | ((q.y >> 30) << 2) | ((q.z >> 30) << 4) | ((q.w >> 25) << 6);
    reds_and(Ls + 4u * word, ~m);
}

// One slot of the FLAT window (bytes = what the bulk copy delivered, a multiple of 16; src = slot address + lane * 16): every lane eats
// 4 runs per 128-bit load, 1 KB of the slot per step.  Deliberately ONE out-of-line copy per kernel: inlined into both slot
// branches of the consumer (and unrolled) the sweep alone was ~50 KB of SASS, more than the instruction cache of an SM
// sub-partition holds -- ncu showed `no_instruction` as the top stall of the GAP phase.  SGL: the stage holds companion singles.
template <int MODE, bool SGL = false>
__device__ __forceinline__ void flat_sweep_mode(uint32_t Ls, uint32_t src, uint32_t bytes, uint32_t lane_off)
{
    auto eat = [&](const uint4& q) { if (SGL) sgl_unit(Ls, q); else flat_quad<MODE>(Ls, q); };
    uint32_t h = 0;
#pragma unroll 1
    for (; h + 1024u <= bytes; h += 1024u) {
        const uint4 qa = lds128(src + h), qb = lds128(src + h + 512u);
        eat(qa); eat(qb);
    }
    if (h + lane_off < bytes)        { const uint4 qa = lds128(src + h);        eat(qa); }     // last, partial KB of the window
    if (h + 512u + lane_off < bytes) { const uint4 qb = lds128(src + h + 512u); eat(qb); }
}
__device__ __noinline__ void flat_sweep_fn(uint32_t Ls, uint32_t src, uint32_t bytes, uint32_t lane_off, uint32_t mode)
{
    if (mode) flat_sweep_mode<1>(Ls, src, bytes, lane_off); else flat_sweep_mode<0>(Ls, src, bytes, lane_off);
}
__device__ __noinline__ void sgl_sweep_fn(uint32_t Ls, uint32_t src, uint32_t bytes, uint32_t lane_off)
{
    flat_sweep_mode<0, true>(Ls, src, bytes, lane_off);
}
// The sweep's form for one column, re-sampled before each piece until it switches (warp-uniform): a 1024-bit sample of L (piece
// number c varies the sample); below 25 % alive the test-first form wins (one shared load, rarely an atomic).  Bits of L only ever
// get cleared, so the switch is one-way per column.
__device__ __forceinline__ void flat_update_mode(uint32_t& mode, uint32_t Ls, uint32_t lane, uint32_t c)
{
    if (mode == 0u) {
        const uint32_t smp = lds32(Ls + (((lane * 65u + c * 7u) & (kBlockWords - 1u)) << 2));
        mode = __reduce_add_sync(0xffffffffu, (uint32_t)__popc(smp)) < 256u ? 1u : 0u;
    }
}

// GAP format (src/bmfunc.h:1696-1725): buf[0] = header (bit0 first-run value, len = hdr>>3),
// buf[k] k=1..len inclusive run ends; run k = (buf[k-1], buf[k]], value = first ^ ((k-1)&1).
// Selected runs (value == want), one per lane:
//   first == want : k = 2j+1, start = j ? buf[2j]+1 : 0 , end = buf[2j+1]      j < (len+1)/2
//   first != want : k = 2j+2, start = buf[2j+1]+1       , end = buf[2j+2]      j <  len/2

// one warp, GAP block resident in shared memory at byte address `ba` (16-byte aligned, contiguous thanks to
// the tail mirror); hdr = its header word.  Two runs per lane and step: one 64-bit load brings
// buf[4t..4t+3]; the straddling run of the "first != want" case takes buf[4t+4] from the next lane.
// `ba` = shared address of the block's 16-byte unit, `pad` = 1 when the block sits behind one u16 of lead padding
// (BMB200_DESC_GAP_PAD).  The (start,end) pair of selected run j lives at A0 + 4j with
//   A0 = &buf[0] when first == want (runs k = 2j+1), &buf[1] otherwise (runs k = 2j+2);
// packers choose the pad so that A0 is 4-byte aligned for the 1-runs: one 32-bit load per run.
template <bool XOR>
__device__ __forceinline__ void gap_scatter_ring(uint32_t Ks, uint32_t ba, uint32_t pad, uint32_t want, int lane)
{
    const uint32_t h = ba + 2u * pad;
    const uint32_t hdr = lds16(h);
    const uint32_t len = hdr >> 3;
    const bool odd = ((hdr & 1u) == want);
    const uint32_t nsel = odd ? (len + 1u) >> 1 : len >> 1;
    const uint32_t A0 = h + (odd ? 0u : 2u);
    // two scatter steps per loop trip: both loads are issued before the first red
    if ((A0 & 2u) == 0u) {
        for (uint32_t j = lane; j < nsel; j += 2u * kLanesPerBlock) {
            const uint32_t a = A0 + 4u * j;
            const bool v1 = (j + kLanesPerBlock < nsel);
            const uint32_t w0 = lds32(a);
            const uint32_t w1 = v1 ? lds32(a + 4u * kLanesPerBlock) : 0u;
            apply_run<XOR>(Ks, (odd && j == 0u) ? 0u : (w0 & 0xffffu) + 1u, w0 >> 16);
            if (v1) apply_run<XOR>(Ks, (w1 & 0xffffu) + 1u, w1 >> 16);
        }
    } else {
        for (uint32_t j = lane; j < nsel; j += 2u * kLanesPerBlock) {
            const uint32_t a = A0 + 4u * j;
            const bool v1 = (j + kLanesPerBlock < nsel);
            const uint32_t s0 = lds16(a), e0 = lds16(a + 2u);
            const uint32_t s1 = v1 ? lds16(a + 4u * kLanesPerBlock) : 0u, e1 = v1 ? lds16(a + 4u * kLanesPerBlock + 2u) : 0u;
            apply_run<XOR>(Ks, (odd && j == 0u) ? 0u : s0 + 1u, e0);
            if (v1) apply_run<XOR>(Ks, s1 + 1u, e1);
        }
    }
}

// one warp, GAP block read straight from global memory (fallback for unsorted / sparse member lists);
// g = &buf[0] (lead pad already skipped)
template <bool XOR>
__device__ __forceinline__ void gap_scatter_gather(uint32_t Ks, const uint16_t* __restrict__ g, uint32_t want, int lane)
{
    const uint32_t hdr = g[0];
    const uint32_t len = hdr >> 3;
    const bool odd = ((hdr & 1u) == want);
    const uint32_t nsel = odd ? (len + 1u) >> 1 : len >> 1;
    const uint16_t* a0 = g + (odd ? 0 : 1);
    for (uint32_t j = lane; j < nsel; j += 32) {
        const uint32_t sv = a0[2u * j], ev = a0[2u * j + 1u];
        apply_run<XOR>(Ks, (odd && j == 0u) ? 0u : sv + 1u, ev);
    }
}

// ---- two-operand bvector ops (bvector::bit_or / bit_and / bit_xor / bit_sub, src/bm.h:5973,6185,6072,6403) ----
// The reference decides the KIND of every result block from the kinds of the two argument blocks
// (combine_operation_block_or/_and/_xor/_sub, src/bm.h:6945,7100,7018,7285): a NULL / FULL argument clones the other block
// (a GAP block stays GAP, a bit-block stays a bit-block), GAP x GAP is merged into a GAP block (gap_buff_op, src/bmfunc.h:3747),
// GAP x bit and bit x bit produce a bit-block that only opt_compress re-classifies (optimize_bit_block, src/bmblocks.h:1414),
// with op-specific all-zero / all-one checks.  binop_rule() is that table; finish_block() applies it.
constexpr uint32_t BINOP_OR = 0u, BINOP_AND = 1u, BINOP_SUB = 2u, BINOP_XOR = 3u;
constexpr uint32_t kRuleComputed = 1u, kRuleCloneBit = 2u, kRuleCloneGap = 3u;   // bits 0-1
constexpr uint32_t kRuleZchk = 4u, kRuleOchk = 8u, kRuleFull = 16u, kRuleMerge = 32u;
__host__ __device__ __forceinline__ uint32_t binop_clone(uint32_t k)
{   // clone_assign_block (src/bmblocks.h:893): FULL stays FULL, a GAP block is copied as GAP (all-zero -> NULL, all-one -> FULL), a bit-block verbatim
    return k == BMB200_BLK_FULL ? kRuleFull : k == BMB200_BLK_GAP ? kRuleCloneGap : kRuleCloneBit;
}
__host__ __device__ __forceinline__ uint32_t binop_rule(uint32_t op, uint32_t ka, uint32_t kb)
{
    const uint32_t N = BMB200_BLK_NULL, F = BMB200_BLK_FULL, B = BMB200_BLK_BIT, G = BMB200_BLK_GAP;
    if (ka == G && kb == G) return kRuleMerge;
    switch (op) {
    case BINOP_OR:
        if (ka == N) return binop_clone(kb);
        if (kb == N) return binop_clone(ka);
        if (ka == F || kb == F) return kRuleFull;
        return (ka == B && kb == B) ? (kRuleComputed | kRuleOchk) : kRuleComputed;        // bit_block_or_2way reports all-ones; gap_add_to_bitset does not
    case BINOP_AND:
        if (ka == N || kb == N) return kRuleComputed | kRuleZchk;                        // (the kernel's NULL short-circuit answers first)
        if (ka == F) return binop_clone(kb);
        if (kb == F) return binop_clone(ka);
        return kRuleComputed | kRuleZchk;                                                // bit_is_all_zero / digest == 0
    case BINOP_XOR:
        if (ka == N) return binop_clone(kb);
        if (kb == N) return binop_clone(ka);
        if (ka == F && kb == F) return kRuleComputed | kRuleZchk;                        // 1 ^ 1: nothing stored
        if (ka == F) return kb == G ? kRuleCloneGap : kRuleCloneBit;                     // inverted clone keeps the kind
        if (kb == F) return ka == G ? kRuleCloneGap : kRuleCloneBit;
        return (ka == B && kb == B) ? (kRuleComputed | kRuleZchk) : kRuleComputed;       // only bit_block_xor_2way checks for zero
    default: /* BINOP_SUB: a - b */
        if (kb == N) return binop_clone(ka);
        if (ka == N || kb == F) return kRuleComputed | kRuleZchk;                        // (short-circuited to NULL by the kernel)
        if (ka == F) return kb == G ? kRuleComputed : (kRuleComputed | kRuleZchk);       // FULL is treated as a real all-ones bit-block
        if (ka == B && kb == G) return kRuleComputed;                                    // clone + gap_sub_to_bitset: no zero check
        return kRuleComputed | kRuleZchk;
    }
}

// Epilogue shared by agg_kernel, agg_pipe_kernel and finalize_blocks_kernel: R = this thread's WPT words of the result block, held by
// NT = 2048 / WPT threads as WPT / 4 quarters of uint4: R[h] = words [4 (h NT + tid), 4 (h NT + tid) + 4) -- one uint4 per thread for
// the 512-thread kernels, two for the 256 consumer threads of agg_pipe_kernel (so every LDS.128 / store of a quarter is conflict-free
// and coalesced).  state: 0 = nothing stored, 1 = FULL, 2 = computed block.  Fuses bit_block_count, calc_block_digest0,
// bit_block_calc_change, the opt_copy_bit_block classification and its bit_to_gap branch
// (src/bmfunc.h:5808,1239,6040,5540; src/bmblocks.h:1355-1409).
template <int N> struct Quads { uint4 q[N]; };     // a thread's words of a result block (finish_block)
template <bool EMPTY_DIGEST_IS_NULL, bool PIPE = false, int WPT = 4>
__device__ __forceinline__ void finish_block(const AggParams& p, uint32_t col, uint32_t colx, uint32_t grp, const Quads<WPT / 4> Rv,
                                             int state, uint32_t* K, uint32_t* s_pc, uint32_t* s_tr, uint32_t* s_dg, uint32_t rule = 0u)
{
    static_assert(WPT == 4 || WPT == 8, "a thread holds one or two uint4 of the result block");
    constexpr int H = WPT / 4, NT = (int)kBlockWords / WPT, NW = NT / 32;
    const uint4 (&R)[H] = Rv.q;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint4* K4 = reinterpret_cast<uint4*>(K);
    // popcount, digest (4 waves per warp and quarter: 8 threads x 4 words = one 32-word wave), run ends
    uint32_t dg4 = 0, pc = 0;    // dg4 bit 4h + q = wave q of this warp's quarter h is not empty
#pragma unroll
    for (int h = 0; h < H; ++h) {
        K4[h * NT + tid] = R[h];     // reuse K so each thread can see its right neighbour's first word
        const uint32_t nz = (R[h].x | R[h].y | R[h].z | R[h].w) != 0u;
        const uint32_t bal = __ballot_sync(0xffffffffu, nz);
#pragma unroll
        for (int q = 0; q < 4; ++q) if ((bal >> (8 * q)) & 0xffu) dg4 |= (1u << (4 * h + q));
        pc += popc4(R[h]);
    }
    pc = warp_sum(pc);
    agg_sync<PIPE, NT>();
    // x has a bit at every position p whose successor differs (bit_block_calc_change src/bmfunc.h:6040 counts
    // them; bit_block_to_gap src/bmfunc.h:5540 emits them as run ends); bit 65535 has no successor
    uint32_t x[H][4], cnt[H];
#pragma unroll
    for (int h = 0; h < H; ++h) {
        const uint4 r = R[h];
        const uint32_t nxt = (h < H - 1 || tid + 1 < NT) ? (K[4 * (h * NT + tid) + 4] & 1u) : (r.w >> 31);
        x[h][0] = r.x ^ ((r.x >> 1) | (r.y << 31)); x[h][1] = r.y ^ ((r.y >> 1) | (r.z << 31));
        x[h][2] = r.z ^ ((r.z >> 1) | (r.w << 31)); x[h][3] = r.w ^ ((r.w >> 1) | (nxt << 31));
        cnt[h] = __popc(x[h][0]) + __popc(x[h][1]) + __popc(x[h][2]) + __popc(x[h][3]);
    }
    // inclusive warp scan of the run-end counts; with two quarters both are scanned at once, quarter 1 in the high 16 bits
    // (a quarter has at most 32768 run ends, so the low field never carries)
    uint32_t inc = H == 1 ? cnt[0] : cnt[0] | (cnt[H - 1] << 16);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) s_tr[warp] = inc;
    if (lane == 0) { s_pc[warp] = pc; s_dg[warp] = dg4; }
    agg_sync<PIPE, NT>();
    uint32_t tpc = 0, ttr = 0, woff = 0; uint64_t dg = 0;
#pragma unroll
    for (int w = 0; w < NW; ++w) {
        const uint32_t t = s_tr[w];
        tpc += s_pc[w]; ttr += t; if (w < warp) woff += t;
        if (H == 1) dg |= (uint64_t)s_dg[w] << (4 * w);
        else        dg |= ((uint64_t)(s_dg[w] & 0xfu) << (4 * w)) | ((uint64_t)(s_dg[w] >> 4) << (4 * NW + 4 * w));
    }
    const uint32_t runs = H == 1 ? ttr + 1u : (ttr & 0xffffu) + (ttr >> 16) + 1u;

    // result kind: aggregator stores nothing when the AND/SUB/XOR digest is empty; otherwise
    // copy_bit_block (opt_none) or the opt_copy_bit_block classification (src/bmblocks.h:1355-1409)
    uint32_t kd;
    if (state == 0) kd = BMB200_BLK_NULL;
    else if (state == 1) kd = BMB200_BLK_FULL;
    else if (rule) {                     // two-operand bvector op: the kind follows the argument kinds (binop_rule)
        const uint32_t mode = rule & 3u;
        if (rule & kRuleFull) kd = BMB200_BLK_FULL;
        else if (mode == kRuleCloneBit) kd = BMB200_BLK_BIT;
        else if (mode == kRuleCloneGap) kd = tpc == 0u ? BMB200_BLK_NULL : tpc == 65536u ? BMB200_BLK_FULL : BMB200_BLK_GAP;
        else if ((rule & kRuleZchk) && tpc == 0u) kd = BMB200_BLK_NULL;
        else if ((rule & kRuleOchk) && tpc == 65536u) kd = BMB200_BLK_FULL;
        else if (!p.compress) kd = BMB200_BLK_BIT;
        else if (runs == 1u) kd = tpc ? BMB200_BLK_FULL : BMB200_BLK_NULL;      // optimize_bit_block
        else if (runs < BMB200_GAP_THRESHOLD) kd = BMB200_BLK_GAP;
        else kd = BMB200_BLK_BIT;
    }
    else if (EMPTY_DIGEST_IS_NULL && dg == 0) kd = BMB200_BLK_NULL;
    else if (!p.compress) kd = BMB200_BLK_BIT;
    else if (runs == 1u) kd = tpc ? BMB200_BLK_FULL : BMB200_BLK_NULL;
    else if (runs < BMB200_GAP_THRESHOLD) kd = BMB200_BLK_GAP;
    else kd = BMB200_BLK_BIT;

    if (p.or_blocks && kd != BMB200_BLK_NULL) {      // pipeline OR target: union of all group results of this column
#pragma unroll
        for (int h = 0; h < H; ++h) {
            uint32_t* ob = p.or_blocks + (size_t)colx * kBlockWords + 4u * (h * NT + tid);
            if (R[h].x) atomicOr(ob + 0, R[h].x);
            if (R[h].y) atomicOr(ob + 1, R[h].y);
            if (R[h].z) atomicOr(ob + 2, R[h].z);
            if (R[h].w) atomicOr(ob + 3, R[h].w);
        }
    }
    if (p.store_blocks && kd == BMB200_BLK_BIT) {
#pragma unroll
        for (int h = 0; h < H; ++h)
            st_stream_v4(reinterpret_cast<uint4*>(p.blocks) + (size_t)col * (kBlockWords / 4) + h * NT + tid, R[h]);
    }
    if (p.store_blocks && kd == BMB200_BLK_GAP) {
        // bit -> GAP fused here (the bit_to_gap branch of opt_copy_bit_block): run ends in order, header last
        uint16_t* gout = p.gaps + (size_t)col * kGapMax;
#pragma unroll
        for (int h = 0; h < H; ++h) {
            uint32_t off = H == 1 ? 1u + woff + inc - cnt[0]
                         : h == 0 ? 1u + (woff & 0xffffu) + (inc & 0xffffu) - cnt[0]
                                  : 1u + (ttr & 0xffffu) + (woff >> 16) + (inc >> 16) - cnt[h];
            const uint32_t base = 128u * (h * NT + tid);
            uint32_t m;
            m = x[h][0]; while (m) { const uint32_t b = __ffs(m) - 1u; m &= m - 1u; gout[off++] = (uint16_t)(base + b); }
            m = x[h][1]; while (m) { const uint32_t b = __ffs(m) - 1u; m &= m - 1u; gout[off++] = (uint16_t)(base + 32u + b); }
            m = x[h][2]; while (m) { const uint32_t b = __ffs(m) - 1u; m &= m - 1u; gout[off++] = (uint16_t)(base + 64u + b); }
            m = x[h][3]; while (m) { const uint32_t b = __ffs(m) - 1u; m &= m - 1u; gout[off++] = (uint16_t)(base + 96u + b); }
        }
        if (tid == 0) {
            const uint32_t lvl = runs <= 124u ? 0u : runs <= 252u ? 1u : runs <= 508u ? 2u : 3u;   // gap_calc_level src/bmfunc.h:5418
            gout[runs] = 65535u;
            gout[0] = (uint16_t)((R[0].x & 1u) | (lvl << 1) | (runs << 3));
        }
    }
    if (tid == 0) {
        p.popcnt[col] = tpc;
        p.digest[col] = dg;
        p.nruns[col]  = runs;
        p.kind[col]   = (uint8_t)kd;
        if (tpc) atomicAdd(p.total + grp, (unsigned long long)tpc);
    }
}
template <bool EMPTY_DIGEST_IS_NULL, bool PIPE = false>
__device__ __forceinline__ void finish_block(const AggParams& p, uint32_t col, uint32_t colx, uint32_t grp, uint4 R, int state,
                                             uint32_t* K, uint32_t* s_pc, uint32_t* s_tr, uint32_t* s_dg, uint32_t rule = 0u)
{
    finish_block<EMPTY_DIGEST_IS_NULL, PIPE, 4>(p, col, colx, grp, Quads<1>{{R}}, state, K, s_pc, s_tr, s_dg, rule);
}

// AND / AND-SUB result state (0 = NULL, 1 = FULL, 2 = computed): an AND-group NULL block, an empty AND group or a SUB-group FULL
// block empties the column; an AND group of FULL blocks only, with no SUB group (AND-SUB), fills it
template <int OP>
__device__ __forceinline__ int and_state(uint32_t flags, uint32_t tot_bit0, uint32_t tot_gap0, uint32_t n0, uint32_t n1)
{
    if ((flags & kFlNull0) || n0 == 0) return 0;
    if (flags & kFlFull1) return 0;
    if (tot_bit0 + tot_gap0 == 0 && (OP == BMB200_OP_AND || n1 == 0)) return 1;
    return 2;
}

template <int OP>
__global__ void __launch_bounds__(kAggThreads, kCtasPerSm) agg_kernel(const AggParams p)
{
    // members classified per pass: the AND-SUB kernel keeps three lists (static smem must stay below the 16 KB boundary the live mask
    // sits on), the one-group kernels use the room for longer lists -- a 4096-member OR (config 5) takes 3 passes instead of 4, and
    // every pass costs a classification, a window check over the descriptor row and two block barriers
    constexpr int kChunkN = (OP == BMB200_OP_AND_SUB) ? kAggChunk : kAggChunkWide;
    constexpr int kMaxChunksN = (kChunkN * 4096) / (int)kGapChunkBytes + 4;      // streamed only when span <= n * 4096
    extern __shared__ __align__(128) uint8_t dyn_smem[];
    // the live mask L (see the header comment) sits at the first 8 KB boundary of the shared window inside the dynamic region, the ring behind it
    const uint32_t dyn_s = smem_u32(dyn_smem);
    const uint32_t k_off = ((dyn_s + kLiveAlign - 1u) & ~(kLiveAlign - 1u)) - dyn_s;
    if (k_off + kLiveAlign + (uint32_t)kAggRingSmem > p.dyn_bytes) __trap();       // host and kernel disagree about the layout
    uint32_t* K = reinterpret_cast<uint32_t*>(dyn_smem + k_off);
    uint32_t* ring = reinterpret_cast<uint32_t*>(dyn_smem + k_off + kLiveAlign);

    __shared__ uint32_t lst_bit0[kChunkN];
    __shared__ uint32_t lst_bit1[kChunkN];
    __shared__ uint32_t lst_gap[kChunkN];      // group0 GAPs from the front, group1 GAPs from the back (both in member order)
    __shared__ uint32_t s_cfirst[kMaxChunksN];    // first list entry starting in each ring chunk
    __shared__ __align__(8) uint64_t s_full[kGapStages];
    __shared__ uint32_t s_done[kGapStages];
    __shared__ __align__(8) uint64_t s_wfull[kAggWarps * kFlatSlots];   // FLAT consumer: one "slot filled" barrier per private slot
    __shared__ uint32_t s_flat_next;             // next unclaimed chunk of the flat window
    __shared__ uint2 s_wpk[2][kAggWarps];        // per-warp counts of the ordered compaction, packed (bit0 | bit1<<16, gap0 | gap1<<16); one buffer per trip
    __shared__ uint32_t s_stat[4];               // flags, total nbit0, total ngap0, nfull0
    __shared__ uint32_t s_flat[3];               // GAP blocks inside the flat window, first unit behind it, non-FLAT members
    __shared__ uint32_t s_col, s_gap_next;
    __shared__ uint32_t s_pc[kAggWarps], s_tr[kAggWarps], s_dg[kAggWarps];

    constexpr bool kIsXor = (OP == BMB200_OP_XOR);
    constexpr bool kIsAnd = (OP == BMB200_OP_AND || OP == BMB200_OP_AND_SUB);
    constexpr int  kFlatList = (OP == BMB200_OP_OR) ? 0 : (OP == BMB200_OP_AND_SUB) ? 1 : -1;   // the list of 1-run sources

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t M = p.set.n_vec;
    uint4* K4 = reinterpret_cast<uint4*>(K);
    // opaque copies: keeps the shared-window base addresses in registers instead of re-deriving them
    // (S2UR SR_CgaCtaId + LEA) inside the scatter loop
    uint32_t Ks, ring_s;
    asm volatile("mov.u32 %0, %1;" : "=r"(Ks) : "r"(smem_u32(K)));
    asm volatile("mov.u32 %0, %1;" : "=r"(ring_s) : "r"(smem_u32(ring)));
    uint32_t done_s, wfull_s, flat_next_s;
    asm volatile("mov.u32 %0, %1;" : "=r"(flat_next_s) : "r"(smem_u32(&s_flat_next)));
    asm volatile("mov.u32 %0, %1;" : "=r"(done_s) : "r"(smem_u32(s_done)));
    asm volatile("mov.u32 %0, %1;" : "=r"(wfull_s) : "r"(smem_u32(&s_wfull[warp * kFlatSlots])));
    uint32_t wphase = 0;     // bit k = phase of this warp's slot k barrier
    uint32_t wchunk[kFlatSlots];   // chunk in flight / resident in slot k (warp-uniform)
    uint32_t gseq = 0;       // chunks streamed so far by this CTA: chunk g lives in stage g % S, its mbarrier phase is (g / S) & 1

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < kGapStages; ++s) mbar_init(&s_full[s], 1u);
#pragma unroll
        for (int w = 0; w < kAggWarps * (int)kFlatSlots; ++w) mbar_init(&s_wfull[w], 1u);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // work items are claimed one iteration ahead: the round trip of the global atomic hides behind the current column
    uint32_t next_item = 0;
    if (tid == 0) next_item = atomicAdd(p.work_counter, 1u);
    __syncthreads();

    for (;;) {
        if (tid == 0) s_col = next_item;
        __syncthreads();
        const uint32_t item = s_col;
        if (item >= p.n_cols * p.n_groups) break;
        if (tid == 0) next_item = atomicAdd(p.work_counter, 1u);
        // groups of one column are adjacent work items: concurrently running CTAs share the column's source blocks in L2
        const uint32_t colx = item / p.n_groups, grp = item - colx * p.n_groups;
        const uint32_t col = grp * p.n_cols + colx;          // output slot (group-major)
        const uint32_t nb = p.nb_from + colx;
        const uint32_t gb0 = p.goff[2u * grp], gb1 = p.goff[2u * grp + 1u], gb2 = p.goff[2u * grp + 2u];
        const uint32_t n0 = gb1 - gb0, n1 = (OP == BMB200_OP_AND_SUB) ? gb2 - gb1 : 0u;
        const uint32_t ntot = n0 + n1;
        const uint32_t* gmem = p.group + gb0;
        uint32_t rule = 0u;
        if (p.binary) {                  // two-operand op: members 0 and 1 are the arguments (a, b)
            const uint32_t* dr = p.set.desc + (size_t)nb * M;
            rule = binop_rule(p.binary - 1u, dr[gmem[0]] & 3u, dr[gmem[1]] & 3u);
            if (rule & kRuleMerge) {     // GAP x GAP was merged by gap_merge_kernel, unless the merged block outgrew the GAP format (kind 0xFF)
                if (p.kind[col] != 0xffu) { __syncthreads(); continue; }    // (barrier: nobody may still be reading s_col when thread 0 rewrites it)
                rule = kRuleComputed;    // convert_gap2bitset: a bit-block, never re-classified
            }
        }

        // live mask: everything alive (nothing covered yet / every bit still a candidate); XOR starts from zero
        K4[tid] = kIsXor ? make_uint4(0u, 0u, 0u, 0u) : make_uint4(~0u, ~0u, ~0u, ~0u);
        if (tid < 4) s_stat[tid] = 0u;
        uint4 acc0 = kIsAnd ? make_uint4(~0u, ~0u, ~0u, ~0u) : make_uint4(0u, 0u, 0u, 0u);
        uint4 acc1 = make_uint4(0u, 0u, 0u, 0u);   // union of SUB-group bit-blocks
        uint32_t flat_mode = 0;                    // FLAT consumer form of this column (warp-uniform, one-way): 0 = atomics, 1 = test-first

        const uint32_t* drow = p.set.desc + (size_t)nb * M;
        const uint4* bseg = reinterpret_cast<const uint4*>(p.set.bit_pool)
                            + p.set.bit_base[nb] * (size_t)(kBlockWords / 4) + tid;
        const uint64_t gseg_unit = p.set.gap_base[nb];
        const uint16_t* gseg = p.set.gap_pool + gseg_unit * (size_t)kGapUnit;
        const uint64_t gseg_avail = p.gap_pool_bytes - gseg_unit * 16ull;   // readable bytes from gseg on
        if (ntot == 0) __syncthreads();

        for (uint32_t cs = 0; cs < ntot; cs += kChunkN) {
            if (tid == 0) { s_gap_next = 0u; s_flat_next = 0u; s_flat[0] = 0u; s_flat[1] = 0xffffffffu; s_flat[2] = 0u; }
            // ---- classification (sort_input_blocks_*): order-preserving compaction into 4 lists ----
            // per trip: 4 ballots, one packed count pair per warp, ONE block barrier, then every warp scans the 16 warp
            // counts with shuffles; the running list lengths stay in (uniform) registers
            const uint32_t ce = min(cs + (uint32_t)kChunkN, ntot);
            uint32_t fl = 0, nfull0 = 0, nonflat = 0;
            uint32_t run01 = 0, run23 = 0;                       // nbit0 | nbit1 << 16, ngap0 | ngap1 << 16 so far
            int trip = 0;
            for (uint32_t kb = cs; kb < ce; kb += kAggThreads, trip ^= 1) {   // uniform trip count (<= 3)
                const uint32_t k = kb + tid;
                uint32_t kind = 0xffu, rel = 0; bool g1 = false;
                if (k < ce) {
                    const uint32_t d = drow[gmem[k]];
                    kind = d & 3u; rel = d >> 2; g1 = (k >= n0);
                }
                const bool c0 = (kind == BMB200_BLK_BIT) && !g1, c1 = (kind == BMB200_BLK_BIT) && g1;
                const bool c2 = (kind == BMB200_BLK_GAP) && !g1, c3 = (kind == BMB200_BLK_GAP) && g1;
                if (kind == BMB200_BLK_NULL && !g1) fl |= kFlNull0;
                if (kind == BMB200_BLK_FULL) { if (g1) fl |= kFlFull1; else { fl |= kFlFull0; ++nfull0; } }
                if ((kFlatList == 0 ? c2 : c3) && !(rel & kEntFlat)) nonflat = 1u;
                const uint32_t lt = (1u << lane) - 1u;
                const uint32_t m0 = __ballot_sync(0xffffffffu, c0), m1 = __ballot_sync(0xffffffffu, c1);
                const uint32_t m2 = __ballot_sync(0xffffffffu, c2), m3 = __ballot_sync(0xffffffffu, c3);
                if (lane == 0) s_wpk[trip][warp] = make_uint2(__popc(m0) | (__popc(m1) << 16), __popc(m2) | (__popc(m3) << 16));
                __syncthreads();
                uint2 x = (lane < kAggWarps) ? s_wpk[trip][lane] : make_uint2(0u, 0u);
#pragma unroll
                for (int o = 1; o < kAggWarps; o <<= 1) {        // inclusive scan over the warps (16-bit fields never overflow: <= 1024)
                    const uint32_t y0 = __shfl_up_sync(0xffffffffu, x.x, o), y1 = __shfl_up_sync(0xffffffffu, x.y, o);
                    if (lane >= o) { x.x += y0; x.y += y1; }
                }
                const uint32_t t01 = __shfl_sync(0xffffffffu, x.x, kAggWarps - 1), t23 = __shfl_sync(0xffffffffu, x.y, kAggWarps - 1);
                uint32_t e01 = __shfl_sync(0xffffffffu, x.x, (warp + 31) & 31), e23 = __shfl_sync(0xffffffffu, x.y, (warp + 31) & 31);
                if (warp == 0) { e01 = 0u; e23 = 0u; }
                e01 += run01; e23 += run23;
                if (c0) lst_bit0[(e01 & 0xffffu) + __popc(m0 & lt)] = rel;
                if (c1) lst_bit1[(e01 >> 16) + __popc(m1 & lt)] = rel;
                if (c2) lst_gap[(e23 & 0xffffu) + __popc(m2 & lt)] = rel;
                if (c3) lst_gap[kChunkN - 1 - ((e23 >> 16) + __popc(m3 & lt))] = rel;
                run01 += t01; run23 += t23;
            }
            fl = __reduce_or_sync(0xffffffffu, fl);
            nfull0 = warp_sum(nfull0);
            nonflat = __reduce_or_sync(0xffffffffu, nonflat);
            if (lane == 0) { if (fl) atomicOr(&s_stat[0], fl); if (nfull0) atomicAdd(&s_stat[3], nfull0); if (nonflat) s_flat[2] = 1u; }
            const uint32_t nbit0 = run01 & 0xffffu, nbit1 = run01 >> 16, ngap0 = run23 & 0xffffu, ngap1 = run23 >> 16;
            if (tid == 0) { s_stat[1] += nbit0; s_stat[2] += ngap0; }
            __syncthreads();

            // ---- GAP lists: decide flat / stream / gather (uniform), set up the first streamed pass ----
            // pass 0 = group0 list (front), pass 1 = group1 list (back, read reversed so it is in member order)
            const uint32_t want0 = kIsAnd ? 0u : 1u;
            bool ok0 = false, ok1 = false;                      // list q is streamed per block (else gathered)
            bool flat = false;                                  // list kFlatList is streamed flat
            uint32_t lo0 = 0, lo1 = 0, wb0 = 0, wb1 = 0, nc0 = 0, nc1 = 0;   // window start unit, bytes, chunks
            {
                int bad0 = 0, bad1 = 0;
                for (uint32_t i = tid; i + 1 < ngap0; i += kAggThreads) bad0 |= !((lst_gap[i] & kRelMask) < (lst_gap[i + 1] & kRelMask));
                for (uint32_t i = tid; i + 1 < ngap1; i += kAggThreads)
                    bad1 |= !((lst_gap[kChunkN - 1 - i] & kRelMask) < (lst_gap[kChunkN - 2 - i] & kRelMask));
                // NB: __syncthreads_or returns a predicate, not a bitwise OR -> one vote per list
                const bool sorted0 = !__syncthreads_or(bad0), sorted1 = !__syncthreads_or(bad1);
                // FLAT window: the units [lo, end) hold exactly the list's GAP blocks, all in FLAT form
                if (kFlatList >= 0 && p.gap_mode == 0u) {
                    const uint32_t nq = kFlatList ? ngap1 : ngap0;
                    const bool sortedq = kFlatList ? sorted1 : sorted0;
                    if (nq >= kFlatMinBlocks && sortedq && !s_flat[2] && M <= 8u * nq + 1024u) {   // uniform
                        const uint32_t lo = (kFlatList ? lst_gap[kChunkN - 1] : lst_gap[0]) & kRelMask;
                        const uint32_t hi = (kFlatList ? lst_gap[kChunkN - nq] : lst_gap[nq - 1]) & kRelMask;
                        uint32_t c = 0, e = (uint32_t)(p.set.gap_base[nb + 1] - gseg_unit);
                        for (uint32_t v = tid; v < M; v += kAggThreads) {
                            const uint32_t d = drow[v];
                            if ((d & 3u) == BMB200_BLK_GAP) {
                                const uint32_t u = (d >> 2) & kRelMask;
                                if (u >= lo && u <= hi) ++c; else if (u > hi) e = min(e, u);
                            }
                        }
                        c = warp_sum(c); e = __reduce_min_sync(0xffffffffu, e);
                        if (lane == 0) { if (c) atomicAdd(&s_flat[0], c); atomicMin(&s_flat[1], e); }
                        __syncthreads();
                        const uint32_t end = s_flat[1];
                        if (s_flat[0] == nq && end > hi) {
                            flat = true;
                            const uint32_t w = (end - lo) * 16u;
                            if (kFlatList) { lo1 = lo; wb1 = w; nc1 = (w + kGapChunkBytes - 1u) / kGapChunkBytes; }
                            else           { lo0 = lo; wb0 = w; nc0 = (w + kGapChunkBytes - 1u) / kGapChunkBytes; }
                        }
                    }
                }
                auto plan = [&](uint32_t n, bool sorted, uint32_t lo, uint32_t hi, bool& ok, uint32_t& wlo, uint32_t& wb, uint32_t& nc) {
                    if (n == 0 || p.gap_mode == 1u || !sorted) return;
                    const uint64_t span = (uint64_t)(hi - lo) * 16ull + kGapMaxBytes;
                    if (span > (uint64_t)n * 4096ull) return;                    // sparse subset: gather instead
                    const uint64_t avail = (gseg_avail - (uint64_t)lo * 16ull) & ~15ull;
                    const uint64_t w = span < avail ? span : avail;
                    ok = true; wlo = lo; wb = (uint32_t)w; nc = (uint32_t)((w + kGapChunkBytes - 1) / kGapChunkBytes);
                };
                if (ngap0 && !(flat && kFlatList == 0)) plan(ngap0, sorted0, lst_gap[0] & kRelMask, lst_gap[ngap0 - 1] & kRelMask, ok0, lo0, wb0, nc0);
                if (ngap1 && !(flat && kFlatList == 1)) plan(ngap1, sorted1, lst_gap[kChunkN - 1] & kRelMask, lst_gap[kChunkN - ngap1] & kRelMask, ok1, lo1, wb1, nc1);
            }
            auto issue_fill = [&](uint32_t wlo, uint32_t wbytes, uint32_t c, bool mirror) {   // one thread: arm the stage of chunk c, start the copy
                const uint32_t s = (gseq + c) % kGapStages;
                const uint32_t off = c * kGapChunkBytes;
                const uint32_t bytes = min(kGapChunkBytes, wbytes - off);
                const uint32_t extra = (s || !mirror) ? 0u : min(kGapMaxBytes, bytes);   // stage 0 is mirrored behind the ring
                const uint8_t* src = reinterpret_cast<const uint8_t*>(gseg) + (size_t)wlo * 16u + off;
                mbar_arrive_expect_tx(&s_full[s], bytes + extra);
                bulk_g2s(reinterpret_cast<uint8_t*>(ring) + s * kGapChunkBytes, src, bytes, &s_full[s]);
                if (extra) bulk_g2s(reinterpret_cast<uint8_t*>(ring) + kRingBytes, src, extra, &s_full[s]);
            };
            // FLAT: warps claim pieces of the window from a shared counter (one claim = kFlatSlots consecutive chunks, one per
            // private slot) and pull them through their slots
            auto flat_big = [&](uint32_t wbytes) -> bool {       // uniform: one 4 KB slot per warp instead of two 2 KB slots
                return wbytes >= kFlatBigWindow;
            };
            auto flat_claim = [&](auto S) -> uint32_t {          // whole warp; returns the first chunk of the claimed piece (S chunks)
                uint32_t c = 0;
                if (lane == 0) c = atoms_add(flat_next_s, 1u) * decltype(S)::value;   // raw atom.shared: no warp-aggregation code around a one-lane atomic
                return __shfl_sync(0xffffffffu, c, 0);
            };
            auto flat_fill = [&](auto S, uint32_t wlo, uint32_t wbytes, uint32_t c, uint32_t k) {   // whole warp: chunk c -> slot k (caller checked c < nfc)
                constexpr uint32_t kChunk = kFlatWarpBytes / decltype(S)::value;
                if (lane == 0) {
                    const uint32_t off = c * kChunk;
                    const uint32_t bytes = min(kChunk, wbytes - off);
                    const uint32_t bar = wfull_s + 8u * k;
                    fence_proxy_async();
                    mbar_arrive_expect_tx(bar, bytes);
                    bulk_g2s(ring_s + (uint32_t)warp * kFlatWarpBytes + k * kChunk,
                             reinterpret_cast<const uint8_t*>(gseg) + (size_t)wlo * 16u + off, bytes, bar);
                }
            };
            auto flat_setup = [&](auto S, uint32_t wlo, uint32_t wbytes) {
                constexpr uint32_t kS = decltype(S)::value, kChunk = kFlatWarpBytes / kS;
                const uint32_t nfc = (wbytes + kChunk - 1u) / kChunk;
                const uint32_t c0 = flat_claim(S);
#pragma unroll
                for (uint32_t k = 0; k < kS; ++k) { wchunk[k] = c0 + k; if (c0 + k < nfc) flat_fill(S, wlo, wbytes, c0 + k, k); }
            };
            auto stream_setup = [&](int q, bool isflat) {               // all threads; ends with a block barrier
                const uint32_t n = q ? ngap1 : ngap0, wlo = q ? lo1 : lo0, nc = q ? nc1 : nc0, wbytes = q ? wb1 : wb0;
                if (isflat) {      // the ring is idle here (block barrier at the end of the previous pass / column)
                    if (flat_big(wbytes)) flat_setup(std::integral_constant<uint32_t, 1u>{}, wlo, wbytes);
                    else                  flat_setup(std::integral_constant<uint32_t, 2u>{}, wlo, wbytes);
                    return;
                }
                {
                    for (uint32_t i = tid; i < n; i += kAggThreads) {
                        const uint32_t ei = (q ? lst_gap[kChunkN - 1 - i] : lst_gap[i]) & kRelMask;
                        const uint32_t ci = ((ei - wlo) * 16u) / kGapChunkBytes;
                        int cp = -1;
                        if (i) { const uint32_t ep = (q ? lst_gap[kChunkN - i] : lst_gap[i - 1]) & kRelMask; cp = (int)(((ep - wlo) * 16u) / kGapChunkBytes); }
                        for (int c = cp + 1; c <= (int)ci; ++c) s_cfirst[c] = i;
                        if (i == n - 1) for (uint32_t c = ci + 1; c <= nc; ++c) s_cfirst[c] = n;
                    }
                }
                if (tid < kGapStages) s_done[tid] = 0u;
                __syncthreads();
                if (tid == 0) {
                    fence_proxy_async();
                    const uint32_t pre = min((uint32_t)kGapStages, nc);
                    for (uint32_t c = 0; c < pre; ++c) issue_fill(wlo, wbytes, c, !isflat);
                }
            };
            auto stage_release = [&](uint32_t s, uint32_t r, uint32_t nc, uint32_t wlo, uint32_t wbytes, bool mirror) {   // per warp, after its share of chunk r
                __syncwarp();
                if (lane == 0) {
                    __threadfence_block();
                    const uint32_t old = atoms_add(done_s + 4u * s, 1u);
                    if (old == kAggWarps - 1) {          // last warp out re-arms the stage
                        sts32(done_s + 4u * s, 0u);      // nobody touches the counter again before the refill has landed
                        if (r + kGapStages < nc) { __threadfence_block(); fence_proxy_async(); issue_fill(wlo, wbytes, r + kGapStages, mirror); }
                    }
                }
            };
            auto stream_consume = [&](int q, uint32_t want) {   // per warp, no block barriers inside
                const uint32_t wlo = q ? lo1 : lo0, nc = q ? nc1 : nc0, wbytes = q ? wb1 : wb0;
                const uint32_t rot = (gseq % kGapStages) * kGapChunkBytes;      // ring offset of the window start
                mbar_wait(&s_full[gseq % kGapStages], (gseq / kGapStages) & 1u);
                for (uint32_t r = 0; r < nc; ++r) {
                    const uint32_t s = (gseq + r) % kGapStages;
                    if (r + 1 < nc) {                 // blocks starting in chunk r may spill into chunk r+1
                        const uint32_t g1 = gseq + r + 1;
                        mbar_wait(&s_full[g1 % kGapStages], (g1 / kGapStages) & 1u);
                    }
                    {   // block i always goes to slot i % (16 * groups): the per-round remainders rotate over the slots
                        constexpr uint32_t kSlots = kAggWarps * kGroupsPerWarp;
                        const uint32_t slot = (uint32_t)warp * kGroupsPerWarp + ((uint32_t)lane / kLanesPerBlock);
                        const int sub = lane & (int)(kLanesPerBlock - 1u);
                        const uint32_t ibeg = s_cfirst[r], iend = s_cfirst[r + 1];
                        for (uint32_t i = ibeg + ((slot - ibeg) & (kSlots - 1u)); i < iend; i += kSlots) {
                            const uint32_t ent = q ? lst_gap[kChunkN - 1 - i] : lst_gap[i];
                            const uint32_t ba = ring_s + (rot + ((ent & kRelMask) - wlo) * 16u) % kRingBytes;
                            gap_scatter_ring<kIsXor>(Ks, ba, ent >> 29, want, sub);
                        }
                    }
                    stage_release(s, r, nc, wlo, wbytes, true);
                }
                gseq += nc;
            };
            auto flat_consume_s = [&](auto S, uint32_t wlo, uint32_t wbytes) {   // per warp, no cross-warp synchronisation at all
                constexpr uint32_t kS = decltype(S)::value, kChunk = kFlatWarpBytes / kS;
                const uint32_t nfc = (wbytes + kChunk - 1u) / kChunk;
                for (;;) {
                    if (wchunk[0] >= nfc) break;                 // chunks of a piece are consecutive: slot 0 empty = nothing left
#pragma unroll
                    for (uint32_t k = 0; k < kS; ++k) {
                        const uint32_t c = wchunk[k];
                        if (c < nfc) {
                            mbar_wait(wfull_s + 8u * k, (wphase >> k) & 1u); wphase ^= 1u << k;
                            const uint32_t bytes = min(kChunk, wbytes - c * kChunk);
                            flat_update_mode(flat_mode, Ks, (uint32_t)lane, c);
                            flat_sweep_fn(Ks, ring_s + (uint32_t)warp * kFlatWarpBytes + k * kChunk + (uint32_t)lane * 16u, bytes, (uint32_t)lane * 16u, flat_mode);
                            __syncwarp();
                        }
                        // slot k is free: the next piece is claimed when slot 0 frees up, its chunk k goes into slot k
                        const uint32_t cn = (k == 0) ? flat_claim(S) : wchunk[0] + k;
                        wchunk[k] = cn;
                        if (cn < nfc) flat_fill(S, wlo, wbytes, cn, k);
                    }
                }
            };
            auto flat_consume = [&](int q) {
                const uint32_t wlo = q ? lo1 : lo0, wbytes = q ? wb1 : wb0;
                if (flat_big(wbytes)) flat_consume_s(std::integral_constant<uint32_t, 1u>{}, wlo, wbytes);
                else                  flat_consume_s(std::integral_constant<uint32_t, 2u>{}, wlo, wbytes);
            };
            auto gather_pass = [&](int q, uint32_t want) {       // per warp; dynamic block distribution
                const uint32_t n = q ? ngap1 : ngap0;
                for (;;) {
                    uint32_t g = 0;
                    if (lane == 0) g = atomicAdd(&s_gap_next, 1u);
                    g = __shfl_sync(0xffffffffu, g, 0);
                    if (g >= n) break;
                    const uint32_t ent = q ? lst_gap[kChunkN - 1 - g] : lst_gap[g];
                    gap_scatter_gather<kIsXor>(Ks, gseg + (size_t)(ent & kRelMask) * kGapUnit + (ent >> 29), want, lane);
                }
            };

            // the first streamed list starts landing in the ring while the bit-blocks stream through registers
            const bool flat0 = flat && kFlatList == 0, flat1 = flat && kFlatList == 1;
            const bool str0 = ok0 || flat0, str1 = ok1 || flat1;
            const int first_q = flat ? kFlatList : (ok0 ? 0 : (ok1 ? 1 : -1));
            if (first_q >= 0) stream_setup(first_q, flat);

            // ---- bit phase: registers <- streamed bit-blocks, then folded into the live mask ----
            bit_phase<OP, false>(bseg, lst_bit0, nbit0, acc0);
            if (OP == BMB200_OP_AND_SUB) bit_phase<OP, true>(bseg, lst_bit1, nbit1, acc1);
            {
                uint4 l = K4[tid];
                if (kIsXor)      { l.x ^= acc0.x; l.y ^= acc0.y; l.z ^= acc0.z; l.w ^= acc0.w; acc0 = make_uint4(0u, 0u, 0u, 0u); }
                else if (kIsAnd) { l.x &= acc0.x & ~acc1.x; l.y &= acc0.y & ~acc1.y; l.z &= acc0.z & ~acc1.z; l.w &= acc0.w & ~acc1.w; }
                else             { l.x &= ~acc0.x; l.y &= ~acc0.y; l.z &= ~acc0.z; l.w &= ~acc0.w; }
                K4[tid] = l;
            }
            __syncthreads();

            // ---- GAP phase: runs clear (XOR: flip) bits of the live mask ----
            if (flat) {
                // a FLAT block without lead pad starts with a 1-run whose pair slot holds the header: the flat pass
                // clears at most a suffix of (0 .. buf[1]); clear the whole run here
                const uint32_t n = kFlatList ? ngap1 : ngap0;
                for (uint32_t i = tid; i < n; i += kAggThreads) {
                    const uint32_t ent = kFlatList ? lst_gap[kChunkN - 1 - i] : lst_gap[i];
                    if (!(ent >> 29)) apply_run<false>(Ks, 0u, gseg[(size_t)(ent & kRelMask) * kGapUnit + 1u]);
                }
                flat_consume(kFlatList);
            } else if (first_q >= 0) stream_consume(first_q, first_q ? 1u : want0);
            {
                const int second_q = (first_q == 0 && str1) ? 1 : (first_q == 1 && str0 ? 0 : -1);
                if (second_q >= 0) {
                    __syncthreads();                     // ring and s_cfirst are reused by the second list
                    stream_setup(second_q, false);
                    stream_consume(second_q, second_q ? 1u : want0);
                }
            }
            if (ngap0 && !str0) gather_pass(0, want0);
            if (ngap1 && !str1) {
                if (ngap0 && !str0) { __syncthreads(); if (tid == 0) s_gap_next = 0u; __syncthreads(); }
                gather_pass(1, 1u);
            }
            __syncthreads();
        }

        // ---- epilogue ----
        const uint32_t flags = s_stat[0], tot_bit0 = s_stat[1], tot_gap0 = s_stat[2], tot_full0 = s_stat[3];
        const uint4 k4 = K4[tid];
        uint4 R;
        int state;   // 0 = NULL (nothing stored), 1 = FULL, 2 = computed block R
        if (OP == BMB200_OP_OR) {
            if (flags & kFlFull0) state = 1;
            else if (tot_bit0 + tot_gap0 == 0) state = 0;
            else {
                state = 2;
                // all-ones is only detected inside the bit-block OR calls (>= 2 bit sources), :1948-1957
                const int ones = __syncthreads_and((acc0.x & acc0.y & acc0.z & acc0.w) == 0xffffffffu);
                if (ones && tot_bit0 >= 2) state = 1;
            }
            R = make_uint4(~k4.x, ~k4.y, ~k4.z, ~k4.w);
        } else if (OP == BMB200_OP_XOR) {
            state = (tot_bit0 + tot_gap0 + tot_full0) ? 2 : 0;
            const uint32_t inv = (tot_full0 & 1u) ? 0xffffffffu : 0u;
            R = make_uint4(k4.x ^ inv, k4.y ^ inv, k4.z ^ inv, k4.w ^ inv);
        } else {
            state = and_state<OP>(flags, tot_bit0, tot_gap0, n0, n1);
            R = k4;
        }
        if (state == 0) R = make_uint4(0u, 0u, 0u, 0u);
        if (state == 1) R = make_uint4(~0u, ~0u, ~0u, ~0u);

        finish_block<OP != BMB200_OP_OR>(p, col, colx, grp, R, state, K, s_pc, s_tr, s_dg, rule);
    }
}

// ---- whole-set AND-SUB: a producer warp streams every column through a shared-memory stage ring ----
//
// When the argument is ONE AND-SUB group whose group0 + group1 name every vector of the set exactly once,
// every block of column nb is needed: its bit-blocks are the contiguous run bit_pool[bit_base[nb] .. bit_base[nb+1]) and its GAP
// blocks the contiguous units gap_pool[gap_base[nb] .. gap_base[nb+1]).  No member list has to be resolved before the bytes can be
// requested, so one producer warp streams columns back to back with cp.async.bulk into a ring of 8 KB stages (full / empty mbarrier
// per stage) and HBM keeps ~kPipeStages x 8 KB per CTA in flight across column boundaries, while 8 consumer warps classify the
// column from its descriptor row, fold the staged bit-blocks (stage j = bit-block j of the segment) and sweep the staged GAP segment
// in FLAT form.  Two CTAs are resident per SM: the phases of a column are limited by different resources (the bit phase by HBM,
// the companion sweep by shared-memory issue, classification and epilogue by barriers and latency), so while one CTA sweeps or
// finishes a column, the other's ring keeps the SM's share of HBM busy.  A column whose GAP blocks are not all FLAT SUB-group blocks (raw GAP form, GAP blocks in the AND group) releases
// its GAP stages unread and applies its GAP blocks straight from global memory.  With the run-list companion (RunLists, passed only
// when the AND group holds no GAP block) the producer streams the column's companion singles and long runs in place of its GAP segment:
// part A (the GAP blocks' runs), or A + B (also the runs of the listed bit-blocks, which it then does not stream) when the AND group
// holds no listed bit-block either.  A column whose streamed part has a union mask (RunLists::un_slot) streams that 8 KB mask
// instead, as one more bit stage that the consumers fold as a SUB-group bit-block: no companion stages, no sweep.
// Protocol (no wait can outlive the producer): the producer warp plans column i + 1 (claim, bases, listed flags) right after it has
// issued column i's first stage, and publishes (item, #bit stages, GAP bytes, first stage, plan) once a queue slot is free and
// column i's last stage is issued; after the last column it publishes an end marker.  Consumers read every queue entry, copy it out
// and free its slot, and wait for exactly the stages it announces: every warp waits for every bit stage (two 16-byte words per
// thread); GAP or companion stage g of the column goes to the kPipeGroup warps of group g % kPipeGroups, each sweeping its
// kPipeSlice bytes of it.  Every waiter arrives once on the stage's empty barrier, for kPipeWarps / (its waiters) warps, so a stage
// is free as soon as its slowest slice is done and the rest of the ring stays requested.  With part B the entry's bit stages are the
// column's unlisted bit-blocks in order.  With the companion the plan names the AND-group stages (PipeCol) and the consumers skip
// the descriptor row; a column with no companion stage to sweep (a union column) goes from the bit phase straight to the epilogue.
// Parity waits are sound because every waiter has waited for every earlier fill of the stage: fills of earlier columns all
// completed before the column barriers the waiter has passed, and within a column a ring slot is reused only by bit stages,
// which every warp waits for, or by GAP stages of the same warp group (kPipeStages = 12 is a multiple of kPipeGroups = 4).
constexpr int      kPipeCtasPerSm = 2;                     // resident CTAs per SM the kernel is shaped for (<= 112 registers)
constexpr int      kPipeConsumers = 256;                   // consumer threads: 8 words of L per thread, as two uint4
constexpr int      kPipeWarps   = kPipeConsumers / 32;
constexpr int      kPipeWpt     = (int)kBlockWords / kPipeConsumers;
constexpr int      kPipeStages  = 12;                      // 96 KB of stages per CTA: with L and the static part 112 KB, so two CTAs fill the SM's 228 KB
constexpr uint32_t kPipeStage   = 8192u;
constexpr uint32_t kPipeGroup   = 2u;                      // consumer warps that share one GAP or companion stage (DESIGN §3.1a)
constexpr uint32_t kPipeGroups  = kPipeWarps / kPipeGroup; // GAP stage g of a column goes to warp group g % kPipeGroups
constexpr uint32_t kPipeSlice   = kPipeStage / kPipeGroup; // bytes of such a stage each warp of its group sweeps
constexpr int      kPipeQueue   = 2;                       // columns claimed ahead of the consumers (more would unbalance the tail)
constexpr uint32_t kPipeMaxVec  = 4096u;                   // role table size: larger sets take agg_kernel
constexpr int      kPipePerThr  = (int)kPipeMaxVec / kPipeConsumers;
constexpr uint32_t kPipeMaxAndGap = 64u;                   // AND-group GAP blocks per column the FLAT path takes (more: in-place reads)
constexpr uint32_t kPipeThreads = kPipeConsumers + 32u;    // 8 consumer warps + 1 producer warp
static_assert(kPipeStages % kPipeGroups == 0, "a ring slot must go to the same warp group each time a column reuses it");
// The coverage instantiation streams bit stages only (every warp waits for every stage, so any ring depth keeps the parity waits
// sound) and at most n0 + 1 of them per column (3 on C3).  A shallower ring lets a third CTA per SM keep one more column's
// fixed per-column work (queue hand-off, fold, finish_block) in flight; at three CTAs the register cap is 72.
constexpr int      kCovCtasPerSm = 3;
constexpr int      kCovStages    = 6;
constexpr size_t pipe_ring_smem(bool cov) { return (size_t)(cov ? kCovStages : kPipeStages) * kPipeStage; }
static_assert(kPipeWpt == 8 && kPipeStage == 2u * 16u * kPipeConsumers, "a bit stage is two LDS.128 per consumer thread");

// *bad |= 1 when a GAP block of the set is not in the BMB200_DESC_GAP_FLAT form (agg_pipe_kernel sweeps SUB-group blocks as FLAT pairs)
__global__ void desc_flat_check_kernel(const uint32_t* __restrict__ desc, size_t n, uint32_t* bad)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t d = desc[i];
        if ((d & 3u) == BMB200_BLK_GAP && !(d & BMB200_DESC_GAP_FLAT)) { atomicOr(bad, 1u); return; }
    }
}

// The run-list companion of the set's GAP blocks and sparse bit-blocks (runlist_kernel.cuh), or all null.  The host passes it only
// when no GAP block of the set belongs to the AND group; the kernel then streams each column's singles and long runs in place of its
// GAP segment: part A only (listed null), or A + B (listed set: then no listed bit-block belongs to the AND group either).
struct RunLists {
    const uint64_t* sgl_base;   // [n_blocks+1] word units of sgl
    const uint64_t* lr_base;    // [n_blocks+1] 16-byte units of lr
    const uint64_t* sgl_mid;    // [n_blocks] end of column nb's part A singles = start of its part B
    const uint64_t* lr_mid;     // [n_blocks] ... long runs
    const uint4* sgl;           // singles: word units (runlist_kernel.cuh)
    const uint32_t* lr;         // long runs: FLAT pairs
    const uint32_t* listed;     // bit i: bit-block i of bit_pool is in part B and not streamed; null = stream part A only
    const uint32_t* un_slot;    // [n_blocks][2]: un_pool slot of the column's U_A / U_AB, ~0 = stream that part packed
    const uint32_t* un_pool;    // [slots][2048]: the union of the part's runs, streamed as one SUB-group bit stage
    const uint16_t* full_cnt;   // [n_blocks]: vectors whose block in column nb is FULL
};
constexpr uint32_t kPipeLstWords = kPipeMaxVec / 32u;       // listed flags of one column's bit-blocks

// The coverage plane GT_n0 of the set for this call's AND-group size (coverage_kernel.cuh), or all null.  The host passes it only
// when no GAP block of the set belongs to the AND group; the kernel then streams each column's AND-group bit-blocks and the
// column's plane slot (unless kCovZero), folded as a SUB-group bit-block, and nothing else.
struct Coverage {
    const uint32_t* slot;       // [n_blocks]: pool slot of column nb's plane, kCovZero or kCovOne
    const uint32_t* pool;       // [slots][2048]
};

// One column as the producer warp plans it (every lane holds the same values except the AND-member fields).  With the companion
// the plan also decides what the consumers would otherwise learn from the column's descriptor row: which streamed stages are
// AND-group bit-blocks (their stream indices, published sorted), how many there are and the result state.
struct PipeCol {
    uint32_t item;               // ~0 = no column left
    uint32_t nstr, nlst, un;     // streamed bit-blocks, listed ones (not streamed), 1 = the companion part is a union mask
    uint32_t gbytes, lbytes;     // GAP segment or companion singles bytes, companion long-run bytes
    const uint8_t *bsrc, *gsrc, *lsrc;
    uint32_t ka, kb;             // stream index of AND member lane / lane + 32 when it is a bit-block, else ~0
    uint32_t ra, rb;             // ... its position in the sorted index list
    uint32_t rela, relb;         // ... with coverage: its block index in the column's bit segment (streamed in place)
    uint32_t nb0, state;         // AND-group bit-blocks; 0 = NULL, 1 = FULL, 2 = computed (and_state)
};

// COV: the call streams the coverage plane cv (else cv is null).  A template parameter, so the companion and segment paths compile
// as they would without it.
template <bool COV>
__global__ void __launch_bounds__(kPipeThreads, COV ? kCovCtasPerSm : kPipeCtasPerSm) agg_pipe_kernel(const AggParams p, const RunLists rl, const Coverage cv)
{
    constexpr int OP = BMB200_OP_AND_SUB;
    constexpr int NS = COV ? kCovStages : kPipeStages;    // ring stages
    extern __shared__ __align__(128) uint8_t dyn_smem[];
    const uint32_t dyn_s = smem_u32(dyn_smem);
    const uint32_t k_off = ((dyn_s + kLiveAlign - 1u) & ~(kLiveAlign - 1u)) - dyn_s;
    if (k_off + kLiveAlign + (uint32_t)NS * kPipeStage > p.dyn_bytes) __trap();     // host and kernel disagree about the layout
    uint32_t* K = reinterpret_cast<uint32_t*>(dyn_smem + k_off);
    uint8_t* ring = dyn_smem + k_off + kLiveAlign;

    __shared__ __align__(8) uint64_t s_full[NS], s_empty[NS], s_qfull[kPipeQueue], s_qempty[kPipeQueue];
    __shared__ uint4 s_q[kPipeQueue];                       // (item | ~0 = end, bit stages, GAP or companion singles bytes, first stage)
    __shared__ uint32_t s_qlr[kPipeQueue];                  // companion long-run bytes (0 without the companion)
    __shared__ uint32_t s_qpl[kPipeQueue];                  // companion plan: AND-group bit-blocks | result state << 16
    __shared__ uint16_t s_qidx[kPipeQueue][kPipeMaxAndGap]; // ... their stream indices, ascending
    __shared__ uint32_t s_lst[2][kPipeLstWords];            // producer, with part B: bit j = bit-block j of the column is listed
    __shared__ uint32_t s_lrk[kPipeLstWords];               // ... listed bit-blocks in words < w of the column being planned
    __shared__ uint32_t s_g1[kPipeMaxVec / 32];             // vector -> member of group1 (AND-SUB)
    __shared__ uint32_t s_brole[2][kPipeMaxVec / 32];       // bit-block j of the column -> group1, one buffer per column parity
    __shared__ uint32_t s_st[2][6];                         // flags, bit0, gap0, AND-group GAP blocks, non-FLAT, first GAP unit
    __shared__ uint2 s_ag[2][kPipeMaxAndGap];               // AND-group GAP blocks of the column: (descriptor, end of its last 16-byte unit)
    __shared__ uint32_t s_pc[kPipeWarps], s_tr[kPipeWarps], s_dg[kPipeWarps];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t M = p.set.n_vec;
    const uint32_t n0 = p.goff[1], n1 = p.goff[2] - p.goff[1];
    const bool planned = COV || rl.sgl_base != nullptr;     // the producer's plan replaces the classification
    if (tid == 0) {
        for (int s = 0; s < NS; ++s) { mbar_init(&s_full[s], 1u); mbar_init(&s_empty[s], kPipeWarps); }
        for (int q = 0; q < kPipeQueue; ++q) { mbar_init(&s_qfull[q], 1u); mbar_init(&s_qempty[q], kPipeWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (uint32_t i = tid; i < kPipeMaxVec / 32; i += kPipeThreads) { s_g1[i] = 0u; s_brole[0][i] = 0u; }
    if (tid < 12) (&s_st[0][0])[tid] = (tid % 6 == 5) ? ~0u : 0u;
    __syncthreads();
    if (!planned)                                           // the descriptor-row classification's role table
        for (uint32_t k = n0 + tid; k < n0 + n1; k += kPipeThreads) { const uint32_t v = p.group[k]; atomicOr(&s_g1[v >> 5], 1u << (v & 31u)); }
    __syncthreads();                                        // the last CTA-wide barrier: the producer warp leaves below

    if (warp == kPipeWarps) {                               // ---- producer warp ----
        // AND-group members lane and lane + 32 (the companion plan looks only at them; whole_set() allows at most 64)
        const uint32_t ma = (uint32_t)lane < n0 ? p.group[lane] : ~0u, mb = (uint32_t)lane + 32u < n0 ? p.group[lane + 32] : ~0u;
        // Claims the next column and plans it; its listed flags go to s_lst[par].  Three dependent round trips (claim, bases and
        // AND-member descriptors, listed words), all taken while the previous column's stages are in flight.
        auto plan = [&](uint32_t par) {
            PipeCol c{};
            uint32_t item = 0;
            if (lane == 0) item = atomicAdd(p.work_counter, 1u);
            c.item = __shfl_sync(0xffffffffu, item, 0);
            if (c.item >= p.n_cols) { c.item = ~0u; return c; }
            const uint32_t nb = p.nb_from + c.item;
            const uint64_t b0 = p.set.bit_base[nb];
            const uint32_t nbit = (uint32_t)(p.set.bit_base[nb + 1] - b0);
            c.bsrc = reinterpret_cast<const uint8_t*>(p.set.bit_pool + b0 * kBlockWords);
            c.ka = c.kb = ~0u;
            if (COV) {          // coverage: the AND members' bit-blocks (stream index = rank among them), then the plane
                const uint32_t* drow = p.set.desc + (size_t)nb * M;
                const uint32_t da = ma != ~0u ? drow[ma] : 0u, db = mb != ~0u ? drow[mb] : 0u;
                const uint32_t cs = cv.slot[nb];
                const bool ba = ma != ~0u && (da & 3u) == BMB200_BLK_BIT, bb = mb != ~0u && (db & 3u) == BMB200_BLK_BIT;
                const uint32_t mba = __ballot_sync(0xffffffffu, ba), mbb = __ballot_sync(0xffffffffu, bb);
                const uint32_t null0 = __ballot_sync(0xffffffffu, (ma != ~0u && (da & 3u) == BMB200_BLK_NULL) ||
                                                                  (mb != ~0u && (db & 3u) == BMB200_BLK_NULL));
                c.nb0 = __popc(mba) + __popc(mbb);
                c.state = (null0 || n0 == 0u || cs == kCovOne) ? 0u : (c.nb0 == 0u && n1 == 0u) ? 1u : 2u;
                if (c.state == 0u) { c.nb0 = 0u; return c; }                 // a NULL result streams nothing
                const uint32_t lt = (1u << lane) - 1u;
                if (ba) { c.ka = c.ra = __popc(mba & lt); c.rela = (da >> 2) & kRelMask; }
                if (bb) { c.kb = c.rb = __popc(mba) + __popc(mbb & lt); c.relb = (db >> 2) & kRelMask; }
                c.nstr = c.nb0;
                if (cs != kCovZero) {
                    c.un = 1u; c.gbytes = kPipeStage;
                    c.gsrc = reinterpret_cast<const uint8_t*>(cv.pool + (size_t)cs * kBlockWords);
                }
                return c;
            }
            // behind the bit-blocks: the GAP segment (gsrc, gbytes), or the companion's singles (gsrc, gbytes) and long runs (lsrc, lbytes)
            if (rl.sgl_base) {
                const uint32_t* drow = p.set.desc + (size_t)nb * M;
                const uint32_t da = ma != ~0u ? drow[ma] : 0u, db = mb != ~0u ? drow[mb] : 0u;
                const uint32_t nfull = rl.full_cnt[nb];
                const uint64_t s0 = rl.sgl_base[nb], l0 = rl.lr_base[nb];
                const uint64_t s1 = rl.listed ? rl.sgl_base[nb + 1] : rl.sgl_mid[nb], l1 = rl.listed ? rl.lr_base[nb + 1] : rl.lr_mid[nb];
                const uint32_t us = rl.un_slot[2u * nb + (rl.listed ? 1u : 0u)];
                c.gbytes = (uint32_t)((s1 - s0) * 16u); c.lbytes = (uint32_t)((l1 - l0) * 16u);
                c.gsrc = reinterpret_cast<const uint8_t*>(rl.sgl + s0); c.lsrc = reinterpret_cast<const uint8_t*>(rl.lr + l0 * 4u);
                if (rl.listed) {        // the column's listed flags (bit j = bit-block j) and their running counts, 32 words per step
                    const uint32_t* lw = rl.listed + (b0 >> 5);
                    const uint32_t sh = (uint32_t)b0 & 31u, nw = (nbit + 31u) / 32u;
                    for (uint32_t w0 = 0; w0 < nw; w0 += 32u) {
                        const uint32_t w = w0 + (uint32_t)lane;
                        uint32_t f = w < nw ? __funnelshift_r(lw[w], lw[w + 1u], sh) : 0u;
                        if (32u * w + 32u > nbit) f &= (1u << (nbit & 31u)) - 1u;
                        uint32_t x = __popc(f);
#pragma unroll
                        for (uint32_t o = 1; o < 32u; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if ((uint32_t)lane >= o) x += y; }
                        if (w < nw) { s_lst[par][w] = f; s_lrk[w] = c.nlst + x - __popc(f); }
                        c.nlst += __shfl_sync(0xffffffffu, x, 31);
                    }
                    __syncwarp();
                }
                // a union mask stands for the part: one 8 KB stage behind the streamed bit-blocks, folded as a SUB-group bit-block
                if (us != ~0u) {
                    c.un = 1u; c.lbytes = 0u; c.gbytes = kPipeStage;
                    c.gsrc = reinterpret_cast<const uint8_t*>(rl.un_pool + (size_t)us * kBlockWords);
                }
                // AND members: stream index of a bit-block = rel minus the listed blocks below it (an AND member is never listed:
                // use_run_lists streams part B only then); NULL and FULL members decide the state; the companion rule leaves no GAP
                auto key = [&](uint32_t m, uint32_t d) -> uint32_t {
                    if (m == ~0u || (d & 3u) != BMB200_BLK_BIT) return ~0u;
                    uint32_t j = (d >> 2) & kRelMask;
                    if (rl.listed) j -= s_lrk[j >> 5] + __popc(s_lst[par][j >> 5] & ((1u << (j & 31u)) - 1u));
                    return j;
                };
                c.ka = key(ma, da); c.kb = key(mb, db);
                const uint32_t null0 = __ballot_sync(0xffffffffu, (ma != ~0u && (da & 3u) == BMB200_BLK_NULL) ||
                                                                  (mb != ~0u && (db & 3u) == BMB200_BLK_NULL));
                const uint32_t full0 = __popc(__ballot_sync(0xffffffffu, ma != ~0u && (da & 3u) == BMB200_BLK_FULL)) +
                                       __popc(__ballot_sync(0xffffffffu, mb != ~0u && (db & 3u) == BMB200_BLK_FULL));
                c.nb0 = __popc(__ballot_sync(0xffffffffu, c.ka != ~0u)) + __popc(__ballot_sync(0xffffffffu, c.kb != ~0u));
                c.state = (null0 || n0 == 0u || nfull > full0) ? 0u : (c.nb0 == 0u && n1 == 0u) ? 1u : 2u;   // nfull > full0: a SUB block is FULL
                for (uint32_t k = 0; k < n0; ++k) {               // sorted position: the indices are distinct, ~0 sorts last
                    const uint32_t x = __shfl_sync(0xffffffffu, k < 32u ? c.ka : c.kb, k & 31u);
                    c.ra += x < c.ka; c.rb += x < c.kb;
                }
            } else {
                const uint64_t g0 = p.set.gap_base[nb];
                c.gbytes = (uint32_t)((p.set.gap_base[nb + 1] - g0) * 16u);
                c.gsrc = reinterpret_cast<const uint8_t*>(p.set.gap_pool + g0 * kGapUnit);
            }
            c.nstr = nbit - c.nlst;
            return c;
        };
        // With the companion, column i's plan is made right after column i - 1's first stage is issued and published after its
        // last: no global round trip separates the two columns' stages.  The GAP-segment path plans after the last stage, as its
        // columns are long enough to hide the round trips and a column claimed a whole column early unbalances the tail.  The
        // first trip streams nothing and plans column 0.
        PipeCol cur{};
        uint32_t seq = 0;
        for (uint32_t qi = 0;; ++qi) {
            const uint32_t par = qi & 1u, ng = cur.nstr + (cur.gbytes + kPipeStage - 1u) / kPipeStage;
            const uint32_t ns = ng + (cur.lbytes + kPipeStage - 1u) / kPipeStage, jp = planned ? 0u : max(ns, 1u) - 1u;
            PipeCol nxt;
            for (uint32_t j = 0, jb = 0; j < max(ns, 1u); ++j) {
                if (j < ns) {
                    const uint32_t s = seq % NS;
                    if (j < cur.nstr && cur.nlst)                // the next unlisted bit-block
                        while ((s_lst[par ^ 1u][jb >> 5] >> (jb & 31u)) & 1u) ++jb;
                    mbar_wait(&s_empty[s], ((seq / NS) & 1u) ^ 1u);
                    uint32_t bytes; const uint8_t* src;
                    if (COV && j < cur.nstr) {                   // coverage: AND member with stream index j, in place
                        const uint32_t ha = __ballot_sync(0xffffffffu, cur.ka == j), hb = __ballot_sync(0xffffffffu, cur.kb == j);
                        const uint32_t rel = ha ? __shfl_sync(0xffffffffu, cur.rela, __ffs(ha) - 1) : __shfl_sync(0xffffffffu, cur.relb, __ffs(hb) - 1);
                        bytes = kPipeStage; src = cur.bsrc + (size_t)rel * kPipeStage;
                    }
                    else if (j < cur.nstr) { bytes = kPipeStage; src = cur.bsrc + (size_t)jb++ * kPipeStage; }
                    else if (j < ng)  { const uint32_t o = (j - cur.nstr) * kPipeStage; bytes = min(kPipeStage, cur.gbytes - o); src = cur.gsrc + o; }
                    else              { const uint32_t o = (j - ng) * kPipeStage;       bytes = min(kPipeStage, cur.lbytes - o); src = cur.lsrc + o; }
                    if (lane == 0) {
                        mbar_arrive_expect_tx(&s_full[s], bytes);
                        bulk_g2s(ring + (size_t)s * kPipeStage, src, bytes, &s_full[s]);
                    }
                    ++seq;
                }
                if (j == jp) nxt = plan(par);
            }
            const uint32_t qs = qi % kPipeQueue;
            mbar_wait(&s_qempty[qs], ((qi / kPipeQueue) & 1u) ^ 1u);
            if (nxt.item == ~0u) {
                if (lane == 0) { s_q[qs] = make_uint4(~0u, 0u, 0u, 0u); mbar_arrive(&s_qfull[qs]); }
                return;
            }
            if (nxt.ka != ~0u) s_qidx[qs][nxt.ra] = (uint16_t)nxt.ka;
            if (nxt.kb != ~0u) s_qidx[qs][nxt.rb] = (uint16_t)nxt.kb;
            if (lane == 0) {
                s_q[qs] = make_uint4(nxt.item, nxt.nstr + nxt.un, nxt.un ? 0u : nxt.gbytes, seq);
                s_qlr[qs] = nxt.lbytes; s_qpl[qs] = nxt.nb0 | (nxt.state << 16);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&s_qfull[qs]);
            cur = nxt;
        }
    }

    // ---- consumers: tid < kPipeConsumers; thread t holds words [4t, 4t + 4) and [4 (t + 256), 4 (t + 256) + 4) of L ----
    uint4* K4 = reinterpret_cast<uint4*>(K);
    uint32_t Ks, ring_s;
    asm volatile("mov.u32 %0, %1;" : "=r"(Ks) : "r"(smem_u32(K)));
    asm volatile("mov.u32 %0, %1;" : "=r"(ring_s) : "r"(smem_u32(ring)));
    constexpr int H = kPipeWpt / 4;
    for (uint32_t qi = 0;; ++qi) {
        const uint32_t b = qi & 1u, qs = qi % kPipeQueue;
        if (!planned) {
            if (tid < 6) s_st[b ^ 1u][tid] = (tid == 5) ? ~0u : 0u;      // next column's counters (nobody reads them any more)
            if (tid < (int)(kPipeMaxVec / 32)) s_brole[b ^ 1u][tid] = 0u;
        }
        mbar_wait(&s_qfull[qs], (qi / kPipeQueue) & 1u);
        const uint4 e = s_q[qs];
        if (e.x == ~0u) break;
        const uint32_t item = e.x, nbit = e.y, gbytes = e.z, seq0 = e.w;
        const uint32_t lbytes = s_qlr[qs], pl = s_qpl[qs], pnb0 = pl & 0xffffu;
        // the plan's AND stream indices, entries lane and lane + 32 (copied out, so the slot is free for the producer right away)
        const uint32_t ia = (uint32_t)lane < pnb0 ? s_qidx[qs][lane] : ~0u, ib = (uint32_t)lane + 32u < pnb0 ? s_qidx[qs][lane + 32] : ~0u;
        __syncwarp();
        if (lane == 0) mbar_arrive(&s_qempty[qs]);
        const uint32_t nb = p.nb_from + item;
        const uint32_t* drow = p.set.desc + (size_t)nb * M;
        const uint16_t* gseg = p.set.gap_pool + p.set.gap_base[nb] * (size_t)kGapUnit;
        int state = (int)(pl >> 16);
        uint32_t nag = 0;
        bool flat = false;
        uint32_t lead = 0;

        // ---- classification by vector (every vector is a member: no member list to resolve); vector tid + 256 i is trip i ----
        // The descriptors are dropped after it: the rare paths behind the bit phase re-read the row.  `lead` keeps the one fact
        // the FLAT path needs from it, bit i = trip i's vector is a SUB-group GAP block without lead pad.
        if (!planned) {
        uint32_t fl = 0, nb0 = 0, ng0 = 0, nonflat = 0, lo = ~0u;
        {
            uint32_t dv[kPipePerThr];
#pragma unroll
            for (int i = 0; i < kPipePerThr; ++i) {
                const uint32_t v = (uint32_t)tid + (uint32_t)i * kPipeConsumers;
                dv[i] = v < M ? drow[v] : BMB200_BLK_NULL;
            }
#pragma unroll
            for (int i = 0; i < kPipePerThr; ++i) {
                const uint32_t v = (uint32_t)tid + (uint32_t)i * kPipeConsumers;
                if (v >= M) continue;
                const uint32_t d = dv[i], kind = d & 3u;
                const bool g1 = (s_g1[v >> 5] >> (v & 31u)) & 1u;
                if (kind == BMB200_BLK_BIT) {
                    if (g1) {                                             // without the companion, stage j is bit-block j
                        const uint32_t j = (d >> 2) & (kPipeMaxVec - 1u);
                        atomicOr(&s_brole[b][j >> 5], 1u << (j & 31u));
                    } else {
                        ++nb0;
                    }
                } else if (kind == BMB200_BLK_GAP) {
                    const uint32_t u = (d >> 2) & kRelMask;
                    if (g1) {
                        if (!((d >> 2) & kEntFlat)) nonflat = 1u;         // the FLAT sweep reads SUB-group blocks in FLAT form only
                        if (!(d >> 31)) lead |= 1u << i;
                    } else {                                              // AND group: listed, applied from global memory and blanked in the stage
                        ++ng0;
                        const uint32_t k = atomicAdd(&s_st[b][3], 1u);
                        if (k < kPipeMaxAndGap) s_ag[b][k] = make_uint2(d, (u * 16u + 2u * (d >> 31) + 2u * ((gseg[(size_t)u * kGapUnit + (d >> 31)] >> 3) + 1u) + 15u) & ~15u);
                        else nonflat = 1u;
                    }
                    lo = min(lo, u);
                } else if (kind == BMB200_BLK_NULL) {
                    if (!g1) fl |= kFlNull0;
                } else {
                    fl |= g1 ? kFlFull1 : kFlFull0;
                }
            }
        }
        fl = __reduce_or_sync(0xffffffffu, fl); nonflat = __reduce_or_sync(0xffffffffu, nonflat); lo = __reduce_min_sync(0xffffffffu, lo);
        nb0 = warp_sum(nb0); ng0 = warp_sum(ng0);
        if (lane == 0) {
            if (fl) atomicOr(&s_st[b][0], fl);
            if (nb0) atomicAdd(&s_st[b][1], nb0);
            if (ng0) atomicAdd(&s_st[b][2], ng0);
            if (nonflat) s_st[b][4] = 1u;
            if (lo != ~0u) atomicMin(&s_st[b][5], lo);
        }
        agg_sync<true, kPipeConsumers>();
        // FLAT: the whole GAP segment is a flat window of 1-run sources (headers, pads and tail fill decode to empty runs)
        flat = s_st[b][4] == 0u && s_st[b][5] == 0u;
        nag = s_st[b][3];                                        // <= kPipeMaxAndGap when flat
        state = and_state<OP>(s_st[b][0], s_st[b][1], s_st[b][2], n0, n1);
        }

        // ---- bit phase: stage j = bit-block j of the column, two LDS.128 per thread ----
        // Planned: stage j is an AND-group bit-block when it is the plan's next index (ascending); every other stage is SUB.
        uint4 acc0[H], acc1[H];
#pragma unroll
        for (int h = 0; h < H; ++h) { acc0[h] = make_uint4(~0u, ~0u, ~0u, ~0u); acc1[h] = make_uint4(0u, 0u, 0u, 0u); }
        uint32_t na = 0, and_j = __shfl_sync(0xffffffffu, ia, 0);
        for (uint32_t j = 0; j < nbit; ++j) {
            const uint32_t sq = seq0 + j, s = sq % NS;
            mbar_wait(&s_full[s], (sq / NS) & 1u);
            uint4 v[H];
#pragma unroll
            for (int h = 0; h < H; ++h) v[h] = lds128(ring_s + s * kPipeStage + (uint32_t)(h * kPipeConsumers + tid) * 16u);
            bool sub;
            if (planned) {
                sub = j != and_j;
                if (!sub) { ++na; and_j = __shfl_sync(0xffffffffu, na < 32u ? ia : ib, na & 31u); }
            } else {
                sub = (s_brole[b][j >> 5] >> (j & 31u)) & 1u;
            }
#pragma unroll
            for (int h = 0; h < H; ++h) { if (sub) acc_or(acc1[h], v[h]); else acc_apply0<OP>(acc0[h], v[h]); }
            __syncwarp();
            if (lane == 0) mbar_arrive(&s_empty[s]);
        }
        // the GAP phase's stages: the GAP segment, or the companion's singles and long-run stages (none on a union column)
        const uint32_t ngs = (gbytes + kPipeStage - 1u) / kPipeStage, nst = ngs + (lbytes + kPipeStage - 1u) / kPipeStage;
        Quads<H> R;
        if (planned && nst == 0u) {      // nothing to sweep: the folded registers are the result, no live mask and no GAP-phase barriers
#pragma unroll
            for (int h = 0; h < H; ++h)
                R.q[h] = state == 0 ? make_uint4(0u, 0u, 0u, 0u) : state == 1 ? make_uint4(~0u, ~0u, ~0u, ~0u)
                       : make_uint4(acc0[h].x & ~acc1[h].x, acc0[h].y & ~acc1[h].y, acc0[h].z & ~acc1[h].z, acc0[h].w & ~acc1[h].w);
            finish_block<true, true, kPipeWpt>(p, item, item, 0u, R, state, K, s_pc, s_tr, s_dg);
            continue;
        }
        // live mask L = AND of the AND-group bit-blocks minus the SUB-group ones (every bit a candidate without bit-blocks)
#pragma unroll
        for (int h = 0; h < H; ++h)
            K4[h * kPipeConsumers + tid] = make_uint4(acc0[h].x & ~acc1[h].x, acc0[h].y & ~acc1[h].y, acc0[h].z & ~acc1[h].z, acc0[h].w & ~acc1[h].w);
        agg_sync<true, kPipeConsumers>();

        // ---- GAP phase: GAP stage g goes to warp group g % kPipeGroups; a warp sweeps bytes [wlo, wlo + kPipeSlice) of it ----
        const uint32_t grp = (uint32_t)warp / kPipeGroup, wlo = ((uint32_t)warp % kPipeGroup) * kPipeSlice;
        if (planned) {
            // run-list companion: every GAP block is a SUB-group block, so the phase clears the column's singles (stages 0 .. ngs-1)
            // and long runs (the stages behind them) from L; no lead-pad repair, no AND-group blocks
            uint32_t flat_mode = 0;
            for (uint32_t g = grp; g < nst; g += kPipeGroups) {
                const uint32_t sq = seq0 + nbit + g, s = sq % NS;
                const bool sgl = g < ngs;
                const uint32_t bytes = sgl ? min(kPipeStage, gbytes - g * kPipeStage) : min(kPipeStage, lbytes - (g - ngs) * kPipeStage);
                const uint32_t src = ring_s + s * kPipeStage + wlo + (uint32_t)lane * 16u, sb = bytes > wlo ? bytes - wlo : 0u;
                mbar_wait(&s_full[s], (sq / NS) & 1u);
                if (sgl) {
                    sgl_sweep_fn(Ks, src, min(kPipeSlice, sb), (uint32_t)lane * 16u);                      // a partial last stage
                } else {                                                                                   // leaves later slices empty
                    flat_update_mode(flat_mode, Ks, (uint32_t)lane, g);
                    flat_sweep_fn(Ks, src, min(kPipeSlice, sb), (uint32_t)lane * 16u, flat_mode);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&s_empty[s], kPipeGroups);
            }
        } else if (flat) {
            // a FLAT SUB-group block without lead pad starts with a 1-run whose pair slot holds the header: clear that whole run here
            for (uint32_t m = lead; m; m &= m - 1u) {
                const uint32_t v = (uint32_t)tid + (uint32_t)(__ffs(m) - 1) * kPipeConsumers;
                apply_run<false>(Ks, 0u, gseg[(size_t)((drow[v] >> 2) & kRelMask) * kGapUnit + 1u]);
            }
            for (uint32_t i = (uint32_t)warp; i < nag; i += kPipeWarps) {  // AND-group GAP blocks: their 0-runs, read in place
                const uint32_t d = s_ag[b][i].x;
                gap_scatter_gather<false>(Ks, gseg + (size_t)((d >> 2) & kRelMask) * kGapUnit + (d >> 31), 0u, lane);
            }
            uint32_t flat_mode = 0;
            for (uint32_t g = grp; g < ngs; g += kPipeGroups) {
                const uint32_t sq = seq0 + nbit + g, s = sq % NS;
                const uint32_t st0 = g * kPipeStage, bytes = min(kPipeStage, gbytes - st0), sb = bytes > wlo ? bytes - wlo : 0u;
                mbar_wait(&s_full[s], (sq / NS) & 1u);
                if (nag) {   // blank the AND-group bytes of this warp's slice: as zero pairs the sweep reads no run in them
                    const uint32_t w0 = st0 + wlo, w1 = w0 + min(kPipeSlice, sb);
                    for (uint32_t i = 0; i < nag; ++i) {
                        const uint2 a = s_ag[b][i];
                        const uint32_t bs = max(((a.x >> 2) & kRelMask) * 16u, w0), be = min(a.y, w1);
                        for (uint32_t x = bs + 2u * (uint32_t)lane; x < be; x += 64u)
                            asm volatile("st.shared.u16 [%0], %1;" :: "r"(ring_s + s * kPipeStage + (x - st0)), "h"((uint16_t)0) : "memory");
                    }
                    fence_proxy_async();     // generic writes before the stage is refilled by the async proxy
                    __syncwarp();
                }
                flat_update_mode(flat_mode, Ks, (uint32_t)lane, g);
                flat_sweep_fn(Ks, ring_s + s * kPipeStage + wlo + (uint32_t)lane * 16u, min(kPipeSlice, sb), (uint32_t)lane * 16u, flat_mode);
                __syncwarp();
                if (lane == 0) mbar_arrive(&s_empty[s], kPipeGroups);
            }
        } else {
            for (uint32_t g = 0; g < ngs; ++g) {                      // release the staged segment unread
                const uint32_t sq = seq0 + nbit + g, s = sq % NS;
                mbar_wait(&s_full[s], (sq / NS) & 1u);
                if (lane == 0) mbar_arrive(&s_empty[s]);
            }
            for (int i = 0; i < kPipePerThr; ++i) {                   // this warp's 32 vectors of trip i, one GAP block at a time
                const uint32_t v = (uint32_t)tid + (uint32_t)i * kPipeConsumers;
                const uint32_t dv = v < M ? drow[v] : BMB200_BLK_NULL;
                uint32_t m = __ballot_sync(0xffffffffu, (dv & 3u) == BMB200_BLK_GAP);
                while (m) {
                    const int l = __ffs(m) - 1; m &= m - 1u;
                    const uint32_t d = __shfl_sync(0xffffffffu, dv, l);
                    const uint32_t vl = v - (uint32_t)lane + (uint32_t)l;
                    const uint32_t want = (s_g1[vl >> 5] >> (vl & 31u)) & 1u;   // AND group: 0-runs, SUB group: 1-runs
                    gap_scatter_gather<false>(Ks, gseg + (size_t)((d >> 2) & kRelMask) * kGapUnit + (d >> 31), want, lane);
                }
            }
        }
        agg_sync<true, kPipeConsumers>();

        // ---- epilogue ----
#pragma unroll
        for (int h = 0; h < H; ++h)
            R.q[h] = state == 0 ? make_uint4(0u, 0u, 0u, 0u) : state == 1 ? make_uint4(~0u, ~0u, ~0u, ~0u) : K4[h * kPipeConsumers + tid];
        finish_block<true, true, kPipeWpt>(p, item, item, 0u, R, state, K, s_pc, s_tr, s_dg);
    }
}


// OR target of a pipeline batch: the per-column union was accumulated with global red.or by agg_kernel; this kernel
// only runs the epilogue (counts, digest, kind, bit->GAP) over those blocks.  One CTA per column, grid-stride.
__global__ void __launch_bounds__(kAggThreads, kCtasPerSm) finalize_blocks_kernel(const AggParams p, const uint32_t* __restrict__ src)
{
    __shared__ __align__(16) uint32_t K[kBlockWords];
    __shared__ uint32_t s_pc[kAggWarps], s_tr[kAggWarps], s_dg[kAggWarps];
    for (uint32_t col = blockIdx.x; col < p.n_cols; col += gridDim.x) {
        const uint4 R = reinterpret_cast<const uint4*>(src)[(size_t)col * (kBlockWords / 4) + threadIdx.x];
        finish_block<true>(p, col, col, 0u, R, 2, K, s_pc, s_tr, s_dg);
        __syncthreads();
    }
}

}  // namespace bmb200
