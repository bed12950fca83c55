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
// Block barrier over the kAggThreads threads that compute a column: the whole CTA (__syncthreads) in agg_kernel, named barrier 1
// over the consumer warps in agg_pipe_kernel (PIPE), whose producer warp never joins it.
template <bool PIPE>
__device__ __forceinline__ void agg_sync()
{
    if (PIPE) asm volatile("bar.sync 1, %0;" :: "n"(kAggThreads) : "memory");
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

// Singles of the run-list companion (runlist_kernel.cuh): eight u16 bit positions per 128-bit load, one bit each.
// MODE 0: one atomic per position.  MODE 1: test-first, as in flat_quad.
template <int MODE>
__device__ __forceinline__ void sgl_oct(uint32_t Ls, const uint4& q)
{
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
    uint32_t a[8], m[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        a[2 * i]     = and_or(w[i] >> 3, 0x1ffcu, Ls);  m[2 * i]     = 1u << (w[i] & 31u);
        a[2 * i + 1] = and_or(w[i] >> 19, 0x1ffcu, Ls); m[2 * i + 1] = 1u << ((w[i] >> 16) & 31u);
    }
    if (MODE) {
        uint32_t v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = lds32(a[i]) & m[i];
#pragma unroll
        for (int i = 0; i < 8; ++i) reds_and_if(a[i], ~m[i], v[i]);
    } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) reds_and(a[i], ~m[i]);
    }
}

// One slot of the FLAT window (bytes = what the bulk copy delivered, a multiple of 16; src = slot address + lane * 16): every lane eats
// 4 runs per 128-bit load, 1 KB of the slot per step.  Deliberately ONE out-of-line copy per kernel: inlined into both slot
// branches of the consumer (and unrolled) the sweep alone was ~50 KB of SASS, more than the instruction cache of an SM
// sub-partition holds -- ncu showed `no_instruction` as the top stall of the GAP phase.  SGL: the stage holds companion singles.
template <int MODE, bool SGL = false>
__device__ __forceinline__ void flat_sweep_mode(uint32_t Ls, uint32_t src, uint32_t bytes, uint32_t lane_off)
{
    auto eat = [&](const uint4& q) { if (SGL) sgl_oct<MODE>(Ls, q); else flat_quad<MODE>(Ls, q); };
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
__device__ __noinline__ void sgl_sweep_fn(uint32_t Ls, uint32_t src, uint32_t bytes, uint32_t lane_off, uint32_t mode)
{
    if (mode) flat_sweep_mode<1, true>(Ls, src, bytes, lane_off); else flat_sweep_mode<0, true>(Ls, src, bytes, lane_off);
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

// Epilogue shared by agg_kernel, agg_pipe_kernel and finalize_blocks_kernel: R = this thread's 4 words of the result block.
// state: 0 = nothing stored, 1 = FULL, 2 = computed block.  Fuses bit_block_count, calc_block_digest0,
// bit_block_calc_change, the opt_copy_bit_block classification and its bit_to_gap branch
// (src/bmfunc.h:5808,1239,6040,5540; src/bmblocks.h:1355-1409).
template <bool EMPTY_DIGEST_IS_NULL, bool PIPE = false>
__device__ __forceinline__ void finish_block(const AggParams& p, uint32_t col, uint32_t colx, uint32_t grp, uint4 R, int state,
                                             uint32_t* K, uint32_t* s_pc, uint32_t* s_tr, uint32_t* s_dg, uint32_t rule = 0u)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint4* K4 = reinterpret_cast<uint4*>(K);
    // popcount, digest (4 waves per warp: 8 threads x 4 words = one 32-word wave), run ends
    K4[tid] = R;                 // reuse K so each thread can see its right neighbour's first word
    const uint32_t nz = (R.x | R.y | R.z | R.w) != 0u;
    const uint32_t bal = __ballot_sync(0xffffffffu, nz);
    uint32_t dg4 = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) if ((bal >> (8 * q)) & 0xffu) dg4 |= (1u << q);
    uint32_t pc = warp_sum(popc4(R));
    agg_sync<PIPE>();
    // x has a bit at every position p whose successor differs (bit_block_calc_change src/bmfunc.h:6040 counts
    // them; bit_block_to_gap src/bmfunc.h:5540 emits them as run ends); bit 65535 has no successor
    const uint32_t nxt = (tid + 1 < kAggThreads) ? (K[4 * tid + 4] & 1u) : (R.w >> 31);
    const uint32_t x0 = R.x ^ ((R.x >> 1) | (R.y << 31)), x1 = R.y ^ ((R.y >> 1) | (R.z << 31));
    const uint32_t x2 = R.z ^ ((R.z >> 1) | (R.w << 31)), x3 = R.w ^ ((R.w >> 1) | (nxt << 31));
    const uint32_t cnt = __popc(x0) + __popc(x1) + __popc(x2) + __popc(x3);
    uint32_t inc = cnt;          // inclusive warp scan of the run-end counts
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) s_tr[warp] = inc;
    if (lane == 0) { s_pc[warp] = pc; s_dg[warp] = dg4; }
    agg_sync<PIPE>();
    uint32_t tpc = 0, ttr = 0, woff = 0; uint64_t dg = 0;
#pragma unroll
    for (int w = 0; w < kAggWarps; ++w) {
        const uint32_t t = s_tr[w];
        tpc += s_pc[w]; ttr += t; if (w < warp) woff += t;
        dg |= (uint64_t)s_dg[w] << (4 * w);
    }
    const uint32_t runs = ttr + 1u;

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
        uint32_t* ob = p.or_blocks + (size_t)colx * kBlockWords + 4u * tid;
        if (R.x) atomicOr(ob + 0, R.x);
        if (R.y) atomicOr(ob + 1, R.y);
        if (R.z) atomicOr(ob + 2, R.z);
        if (R.w) atomicOr(ob + 3, R.w);
    }
    if (p.store_blocks && kd == BMB200_BLK_BIT)
        st_stream_v4(reinterpret_cast<uint4*>(p.blocks) + (size_t)col * (kBlockWords / 4) + tid, R);
    if (p.store_blocks && kd == BMB200_BLK_GAP) {
        // bit -> GAP fused here (the bit_to_gap branch of opt_copy_bit_block): run ends in order, header last
        uint16_t* gout = p.gaps + (size_t)col * kGapMax;
        uint32_t off = 1u + woff + inc - cnt;
        const uint32_t base = 128u * tid;
        uint32_t m;
        m = x0; while (m) { const uint32_t b = __ffs(m) - 1u; m &= m - 1u; gout[off++] = (uint16_t)(base + b); }
        m = x1; while (m) { const uint32_t b = __ffs(m) - 1u; m &= m - 1u; gout[off++] = (uint16_t)(base + 32u + b); }
        m = x2; while (m) { const uint32_t b = __ffs(m) - 1u; m &= m - 1u; gout[off++] = (uint16_t)(base + 64u + b); }
        m = x3; while (m) { const uint32_t b = __ffs(m) - 1u; m &= m - 1u; gout[off++] = (uint16_t)(base + 96u + b); }
        if (tid == 0) {
            const uint32_t lvl = runs <= 124u ? 0u : runs <= 252u ? 1u : runs <= 508u ? 2u : 3u;   // gap_calc_level src/bmfunc.h:5418
            gout[runs] = 65535u;
            gout[0] = (uint16_t)((R.x & 1u) | (lvl << 1) | (runs << 3));
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
// per stage) and HBM keeps ~kPipeStages x 8 KB per SM in flight across column boundaries, while 16 consumer warps classify the
// column from its descriptor row, fold the staged bit-blocks (stage j = bit-block j of the segment) and sweep the staged GAP segment
// in FLAT form.  A column whose GAP blocks are not all FLAT SUB-group blocks (raw GAP form, GAP blocks in the AND group) releases
// its GAP stages unread and applies its GAP blocks straight from global memory.  With the run-list companion (RunLists, passed only
// when the AND group holds no GAP block) the producer streams the column's companion singles and long runs in place of its GAP segment:
// part A (the GAP blocks' runs), or A + B (also the runs of the listed bit-blocks, which it then does not stream) when the AND group
// holds no listed bit-block either.
// Protocol (no wait can outlive the producer): the producer claims a column only when a queue slot is free, publishes (item, #bit
// stages, GAP bytes, first stage) and then issues all of the column's stages in order, each after its empty barrier; after the last
// column it publishes an end marker.  Consumers read every queue entry, wait for exactly the stages the entry announces and release
// each of them exactly once (bit stage: every warp arrives; GAP stage: its one reader arrives for all 16).  They free the queue slot
// once the column is classified, because classification reads the column's listed flags that the producer staged with the entry.
// With part B the entry's bit stages are the column's unlisted bit-blocks in order; stage j is the j-th of them.
// Parity waits are only sound when the waiter has seen the stage's previous fill complete.  Bit stages (streamed ones only, with
// part B) are still waited for by every warp in order; GAP or companion stage g still goes to warp g % 16, so with a ring of a
// multiple of 16 stages the previous fill of each stage a warp waits for was one of its own GAP stages, or a bit stage / an earlier
// column that every warp has finished.
constexpr int      kPipeStages  = 16;                      // 128 KB of stages
constexpr uint32_t kPipeStage   = 8192u;
constexpr int      kPipeQueue   = 2;                       // columns claimed ahead of the consumers (more would unbalance the tail)
constexpr uint32_t kPipeMaxVec  = 4096u;                   // role table size: larger sets take agg_kernel
constexpr int      kPipePerThr  = (int)kPipeMaxVec / kAggThreads;
constexpr uint32_t kPipeMaxAndGap = 64u;                   // AND-group GAP blocks per column the FLAT path takes (more: in-place reads)
constexpr uint32_t kPipeThreads = kAggThreads + 32u;       // 16 consumer warps + 1 producer warp
constexpr size_t   kPipeRingSmem = (size_t)kPipeStages * kPipeStage;
static_assert(kPipeStages % kAggWarps == 0, "GAP stage g is consumed by warp g % 16: the ring must hold a multiple of 16 stages");

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
    const uint64_t* sgl_base;   // [n_blocks+1] 16-byte units of sgl
    const uint64_t* lr_base;    // [n_blocks+1] 16-byte units of lr
    const uint64_t* sgl_mid;    // [n_blocks] end of column nb's part A singles = start of its part B
    const uint64_t* lr_mid;     // [n_blocks] ... long runs
    const uint16_t* sgl;        // singles: u16 bit positions
    const uint32_t* lr;         // long runs: FLAT pairs
    const uint32_t* listed;     // bit i: bit-block i of bit_pool is in part B and not streamed; null = stream part A only
};
constexpr uint32_t kPipeLstWords = kPipeMaxVec / 32u;       // listed flags of one column's bit-blocks

__global__ void __launch_bounds__(kPipeThreads, 1) agg_pipe_kernel(const AggParams p, const RunLists rl)
{
    constexpr int OP = BMB200_OP_AND_SUB;
    extern __shared__ __align__(128) uint8_t dyn_smem[];
    const uint32_t dyn_s = smem_u32(dyn_smem);
    const uint32_t k_off = ((dyn_s + kLiveAlign - 1u) & ~(kLiveAlign - 1u)) - dyn_s;
    if (k_off + kLiveAlign + (uint32_t)kPipeRingSmem > p.dyn_bytes) __trap();     // host and kernel disagree about the layout
    uint32_t* K = reinterpret_cast<uint32_t*>(dyn_smem + k_off);
    uint8_t* ring = dyn_smem + k_off + kLiveAlign;

    __shared__ __align__(8) uint64_t s_full[kPipeStages], s_empty[kPipeStages], s_qfull[kPipeQueue], s_qempty[kPipeQueue];
    __shared__ uint4 s_q[kPipeQueue];                       // (item | ~0 = end, bit stages, GAP or companion singles bytes, first stage)
    __shared__ uint32_t s_qlr[kPipeQueue];                  // companion long-run bytes (0 without the companion)
    __shared__ uint32_t s_lst[kPipeQueue][kPipeLstWords];   // with part B: bit j = the column's bit-block j is listed
    __shared__ uint32_t s_lrk[kPipeQueue][kPipeLstWords];   // ... listed bit-blocks in words < w
    __shared__ uint32_t s_g1[kPipeMaxVec / 32];             // vector -> member of group1 (AND-SUB)
    __shared__ uint32_t s_brole[2][kPipeMaxVec / 32];       // bit-block j of the column -> group1, one buffer per column parity
    __shared__ uint32_t s_st[2][6];                         // flags, bit0, gap0, AND-group GAP blocks, non-FLAT, first GAP unit
    __shared__ uint2 s_ag[2][kPipeMaxAndGap];               // AND-group GAP blocks of the column: (descriptor, end of its last 16-byte unit)
    __shared__ uint32_t s_pc[kAggWarps], s_tr[kAggWarps], s_dg[kAggWarps];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t M = p.set.n_vec;
    const uint32_t n0 = p.goff[1], n1 = p.goff[2] - p.goff[1];
    if (tid == 0) {
        for (int s = 0; s < kPipeStages; ++s) { mbar_init(&s_full[s], 1u); mbar_init(&s_empty[s], kAggWarps); }
        for (int q = 0; q < kPipeQueue; ++q) { mbar_init(&s_qfull[q], 1u); mbar_init(&s_qempty[q], kAggWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (uint32_t i = tid; i < kPipeMaxVec / 32; i += kPipeThreads) { s_g1[i] = 0u; s_brole[0][i] = 0u; }
    if (tid < 12) (&s_st[0][0])[tid] = (tid % 6 == 5) ? ~0u : 0u;
    __syncthreads();
    for (uint32_t k = n0 + tid; k < n0 + n1; k += kPipeThreads) { const uint32_t v = p.group[k]; atomicOr(&s_g1[v >> 5], 1u << (v & 31u)); }
    __syncthreads();                                        // the last CTA-wide barrier: the producer warp leaves below

    if (warp == kAggWarps) {                                // ---- producer (one lane) ----
        if (lane != 0) return;
        uint32_t seq = 0;
        for (uint32_t qi = 0;; ++qi) {
            const uint32_t qs = qi % kPipeQueue;
            mbar_wait(&s_qempty[qs], ((qi / kPipeQueue) & 1u) ^ 1u);
            const uint32_t item = atomicAdd(p.work_counter, 1u);
            if (item >= p.n_cols) { s_q[qs] = make_uint4(~0u, 0u, 0u, 0u); mbar_arrive(&s_qfull[qs]); return; }
            const uint32_t nb = p.nb_from + item;
            const uint64_t b0 = p.set.bit_base[nb];
            const uint32_t nbit = (uint32_t)(p.set.bit_base[nb + 1] - b0);
            // behind the bit-blocks: the GAP segment (gsrc, gbytes), or the companion's singles (gsrc, gbytes) and long runs (lsrc, lbytes)
            uint32_t gbytes, lbytes = 0, nlst = 0;
            const uint8_t *gsrc, *lsrc = nullptr;
            if (rl.sgl_base) {
                const uint64_t s0 = rl.sgl_base[nb], l0 = rl.lr_base[nb];
                const uint64_t s1 = rl.listed ? rl.sgl_base[nb + 1] : rl.sgl_mid[nb], l1 = rl.listed ? rl.lr_base[nb + 1] : rl.lr_mid[nb];
                gbytes = (uint32_t)((s1 - s0) * 16u); lbytes = (uint32_t)((l1 - l0) * 16u);
                gsrc = reinterpret_cast<const uint8_t*>(rl.sgl + s0 * 8u); lsrc = reinterpret_cast<const uint8_t*>(rl.lr + l0 * 4u);
                if (rl.listed) {        // stage the column's listed flags (bit j = bit-block j) and their running counts for everyone
                    const uint32_t* lw = rl.listed + (b0 >> 5);
                    const uint32_t sh = (uint32_t)b0 & 31u, nw = (nbit + 31u) / 32u;
                    uint32_t r = lw[0];
#pragma unroll 4
                    for (uint32_t w = 0; w < nw; ++w) {
                        const uint32_t r1 = lw[w + 1u];
                        uint32_t f = __funnelshift_r(r, r1, sh);
                        if (32u * w + 32u > nbit) f &= (1u << (nbit & 31u)) - 1u;
                        s_lst[qs][w] = f; s_lrk[qs][w] = nlst; nlst += __popc(f); r = r1;
                    }
                }
            } else {
                const uint64_t g0 = p.set.gap_base[nb];
                gbytes = (uint32_t)((p.set.gap_base[nb + 1] - g0) * 16u);
                gsrc = reinterpret_cast<const uint8_t*>(p.set.gap_pool + g0 * kGapUnit);
            }
            const uint32_t nstr = nbit - nlst;                   // streamed bit-blocks
            s_q[qs] = make_uint4(item, nstr, gbytes, seq); s_qlr[qs] = lbytes;
            mbar_arrive(&s_qfull[qs]);
            const uint8_t* bsrc = reinterpret_cast<const uint8_t*>(p.set.bit_pool + b0 * kBlockWords);
            const uint32_t ng = nstr + (gbytes + kPipeStage - 1u) / kPipeStage, ns = ng + (lbytes + kPipeStage - 1u) / kPipeStage;
            for (uint32_t j = 0, jb = 0; j < ns; ++j, ++seq) {
                const uint32_t s = seq % kPipeStages;
                if (j < nstr && nlst)                            // the next unlisted bit-block
                    while ((s_lst[qs][jb >> 5] >> (jb & 31u)) & 1u) ++jb;
                mbar_wait(&s_empty[s], ((seq / kPipeStages) & 1u) ^ 1u);
                uint32_t bytes; const uint8_t* src;
                if (j < nstr)    { bytes = kPipeStage; src = bsrc + (size_t)jb++ * kPipeStage; }
                else if (j < ng) { const uint32_t o = (j - nstr) * kPipeStage; bytes = min(kPipeStage, gbytes - o); src = gsrc + o; }
                else             { const uint32_t o = (j - ng) * kPipeStage;   bytes = min(kPipeStage, lbytes - o); src = lsrc + o; }
                mbar_arrive_expect_tx(&s_full[s], bytes);
                bulk_g2s(ring + (size_t)s * kPipeStage, src, bytes, &s_full[s]);
            }
        }
    }

    // ---- consumers: tid < kAggThreads ----
    uint4* K4 = reinterpret_cast<uint4*>(K);
    uint32_t Ks, ring_s;
    asm volatile("mov.u32 %0, %1;" : "=r"(Ks) : "r"(smem_u32(K)));
    asm volatile("mov.u32 %0, %1;" : "=r"(ring_s) : "r"(smem_u32(ring)));
    for (uint32_t qi = 0;; ++qi) {
        const uint32_t b = qi & 1u, qs = qi % kPipeQueue;
        K4[tid] = make_uint4(~0u, ~0u, ~0u, ~0u);           // live mask: every bit still a candidate
        if (tid < 6) s_st[b ^ 1u][tid] = (tid == 5) ? ~0u : 0u;          // next column's counters (nobody reads them any more)
        if (tid < (int)(kPipeMaxVec / 32)) s_brole[b ^ 1u][tid] = 0u;
        mbar_wait(&s_qfull[qs], (qi / kPipeQueue) & 1u);
        const uint4 e = s_q[qs];
        const uint32_t lbytes = s_qlr[qs];
        if (e.x == ~0u) break;
        const uint32_t item = e.x, nbit = e.y, gbytes = e.z, seq0 = e.w;
        const uint32_t nb = p.nb_from + item;
        const uint32_t* drow = p.set.desc + (size_t)nb * M;
        const uint16_t* gseg = p.set.gap_pool + p.set.gap_base[nb] * (size_t)kGapUnit;

        // ---- classification by vector (every vector is a member: no member list to resolve) ----
        uint32_t dv[kPipePerThr];
        uint32_t fl = 0, nb0 = 0, ng0 = 0, nonflat = 0, lo = ~0u;
#pragma unroll
        for (int i = 0; i < kPipePerThr; ++i) {
            const uint32_t v = (uint32_t)tid + (uint32_t)i * kAggThreads;
            dv[i] = v < M ? drow[v] : BMB200_BLK_NULL;
        }
#pragma unroll
        for (int i = 0; i < kPipePerThr; ++i) {
            const uint32_t v = (uint32_t)tid + (uint32_t)i * kAggThreads;
            if (v >= M) continue;
            const uint32_t d = dv[i], kind = d & 3u;
            const bool g1 = (s_g1[v >> 5] >> (v & 31u)) & 1u;
            if (kind == BMB200_BLK_BIT) {
                // role by streamed index: rel minus the listed blocks below it (a listed block is a SUB-group block, never streamed)
                if (g1) {
                    uint32_t j = (d >> 2) & (kPipeMaxVec - 1u);
                    if (rl.listed) {
                        const uint32_t f = s_lst[qs][j >> 5], below = f & ((1u << (j & 31u)) - 1u);
                        if ((f >> (j & 31u)) & 1u) continue;
                        j -= s_lrk[qs][j >> 5] + __popc(below);
                    }
                    atomicOr(&s_brole[b][j >> 5], 1u << (j & 31u));
                } else {
                    ++nb0;
                }
            } else if (kind == BMB200_BLK_GAP) {
                const uint32_t u = (d >> 2) & kRelMask;
                if (g1) {
                    if (!((d >> 2) & kEntFlat)) nonflat = 1u;         // the FLAT sweep reads SUB-group blocks in FLAT form only
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
        fl = __reduce_or_sync(0xffffffffu, fl); nonflat = __reduce_or_sync(0xffffffffu, nonflat); lo = __reduce_min_sync(0xffffffffu, lo);
        nb0 = warp_sum(nb0); ng0 = warp_sum(ng0);
        if (lane == 0) {
            if (fl) atomicOr(&s_st[b][0], fl);
            if (nb0) atomicAdd(&s_st[b][1], nb0);
            if (ng0) atomicAdd(&s_st[b][2], ng0);
            if (nonflat) s_st[b][4] = 1u;
            if (lo != ~0u) atomicMin(&s_st[b][5], lo);
        }
        agg_sync<true>();
        if (lane == 0) mbar_arrive(&s_qempty[qs]);               // the entry and its listed flags are read: the slot may be refilled
        // FLAT: the whole GAP segment is a flat window of 1-run sources (headers, pads and tail fill decode to empty runs)
        const bool flat = s_st[b][4] == 0u && s_st[b][5] == 0u;
        const uint32_t nag = s_st[b][3];                         // <= kPipeMaxAndGap when flat

        // ---- bit phase: stage j = bit-block j of the column ----
        uint4 acc0 = make_uint4(~0u, ~0u, ~0u, ~0u);
        uint4 acc1 = make_uint4(0u, 0u, 0u, 0u);
        for (uint32_t j = 0; j < nbit; ++j) {
            const uint32_t sq = seq0 + j, s = sq % kPipeStages;
            mbar_wait(&s_full[s], (sq / kPipeStages) & 1u);
            const uint4 v = lds128(ring_s + s * kPipeStage + (uint32_t)tid * 16u);
            if ((s_brole[b][j >> 5] >> (j & 31u)) & 1u) acc_or(acc1, v); else acc_apply0<OP>(acc0, v);
            __syncwarp();
            if (lane == 0) mbar_arrive(&s_empty[s]);
        }
        {
            uint4 l = K4[tid];
            l.x &= acc0.x & ~acc1.x; l.y &= acc0.y & ~acc1.y; l.z &= acc0.z & ~acc1.z; l.w &= acc0.w & ~acc1.w;
            K4[tid] = l;
        }
        agg_sync<true>();

        // ---- GAP phase: GAP stage g belongs to warp g % 16 ----
        const uint32_t ngs = (gbytes + kPipeStage - 1u) / kPipeStage;
        if (rl.sgl_base) {
            // run-list companion: every GAP block is a SUB-group block, so the phase clears the column's singles (stages 0 .. ngs-1)
            // and long runs (the stages behind them) from L; no lead-pad repair, no AND-group blocks
            const uint32_t nst = ngs + (lbytes + kPipeStage - 1u) / kPipeStage;
            uint32_t flat_mode = 0;
            for (uint32_t g = (uint32_t)warp; g < nst; g += kAggWarps) {
                const uint32_t sq = seq0 + nbit + g, s = sq % kPipeStages;
                const uint32_t src = ring_s + s * kPipeStage + (uint32_t)lane * 16u;
                mbar_wait(&s_full[s], (sq / kPipeStages) & 1u);
                flat_update_mode(flat_mode, Ks, (uint32_t)lane, g);
                if (g < ngs) sgl_sweep_fn(Ks, src, min(kPipeStage, gbytes - g * kPipeStage), (uint32_t)lane * 16u, flat_mode);
                else         flat_sweep_fn(Ks, src, min(kPipeStage, lbytes - (g - ngs) * kPipeStage), (uint32_t)lane * 16u, flat_mode);
                __syncwarp();
                if (lane == 0) mbar_arrive(&s_empty[s], kAggWarps);
            }
        } else if (flat) {
            // a FLAT SUB-group block without lead pad starts with a 1-run whose pair slot holds the header: clear that whole run here
#pragma unroll
            for (int i = 0; i < kPipePerThr; ++i) {
                const uint32_t d = dv[i], v = (uint32_t)tid + (uint32_t)i * kAggThreads;
                if (v < M && (d & 3u) == BMB200_BLK_GAP && !(d >> 31) && ((s_g1[v >> 5] >> (v & 31u)) & 1u))
                    apply_run<false>(Ks, 0u, gseg[(size_t)((d >> 2) & kRelMask) * kGapUnit + 1u]);
            }
            for (uint32_t i = (uint32_t)warp; i < nag; i += kAggWarps) {   // AND-group GAP blocks: their 0-runs, read in place
                const uint32_t d = s_ag[b][i].x;
                gap_scatter_gather<false>(Ks, gseg + (size_t)((d >> 2) & kRelMask) * kGapUnit + (d >> 31), 0u, lane);
            }
            uint32_t flat_mode = 0;
            for (uint32_t g = (uint32_t)warp; g < ngs; g += kAggWarps) {
                const uint32_t sq = seq0 + nbit + g, s = sq % kPipeStages;
                mbar_wait(&s_full[s], (sq / kPipeStages) & 1u);
                if (nag) {   // blank the staged bytes of AND-group blocks: as zero pairs the sweep reads no run in them
                    const uint32_t st0 = g * kPipeStage, st1 = st0 + min(kPipeStage, gbytes - st0);
                    for (uint32_t i = 0; i < nag; ++i) {
                        const uint2 a = s_ag[b][i];
                        const uint32_t bs = max(((a.x >> 2) & kRelMask) * 16u, st0), be = min(a.y, st1);
                        for (uint32_t x = bs + 2u * (uint32_t)lane; x < be; x += 64u)
                            asm volatile("st.shared.u16 [%0], %1;" :: "r"(ring_s + s * kPipeStage + (x - st0)), "h"((uint16_t)0) : "memory");
                    }
                    fence_proxy_async();     // generic writes before the stage is refilled by the async proxy
                    __syncwarp();
                }
                flat_update_mode(flat_mode, Ks, (uint32_t)lane, g);
                flat_sweep_fn(Ks, ring_s + s * kPipeStage + (uint32_t)lane * 16u, min(kPipeStage, gbytes - g * kPipeStage), (uint32_t)lane * 16u, flat_mode);
                __syncwarp();
                if (lane == 0) mbar_arrive(&s_empty[s], kAggWarps);
            }
        } else {
            for (uint32_t g = (uint32_t)warp; g < ngs; g += kAggWarps) {      // release the staged segment unread
                const uint32_t sq = seq0 + nbit + g, s = sq % kPipeStages;
                mbar_wait(&s_full[s], (sq / kPipeStages) & 1u);
                if (lane == 0) mbar_arrive(&s_empty[s], kAggWarps);
            }
#pragma unroll
            for (int i = 0; i < kPipePerThr; ++i) {            // this warp's 32 vectors of trip i, one GAP block at a time
                const uint32_t v = (uint32_t)tid + (uint32_t)i * kAggThreads;
                uint32_t m = __ballot_sync(0xffffffffu, v < M && (dv[i] & 3u) == BMB200_BLK_GAP);
                while (m) {
                    const int l = __ffs(m) - 1; m &= m - 1u;
                    const uint32_t d = __shfl_sync(0xffffffffu, dv[i], l);
                    const uint32_t vl = v - (uint32_t)lane + (uint32_t)l;
                    const uint32_t want = (s_g1[vl >> 5] >> (vl & 31u)) & 1u;   // AND group: 0-runs, SUB group: 1-runs
                    gap_scatter_gather<false>(Ks, gseg + (size_t)((d >> 2) & kRelMask) * kGapUnit + (d >> 31), want, lane);
                }
            }
        }
        agg_sync<true>();

        // ---- epilogue ----
        const int state = and_state<OP>(s_st[b][0], s_st[b][1], s_st[b][2], n0, n1);
        const uint4 R = state == 0 ? make_uint4(0u, 0u, 0u, 0u) : state == 1 ? make_uint4(~0u, ~0u, ~0u, ~0u) : K4[tid];
        finish_block<true, true>(p, item, item, 0u, R, state, K, s_pc, s_tr, s_dg);
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
