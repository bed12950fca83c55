// coverage_kernel.cuh -- the coverage planes of a set (built once per set and AND-group size, streamed by agg_pipe_kernel).
//
// For a bit x of column nb let cnt(x) be the number of vectors whose block nb holds x (FULL blocks hold every bit, NULL blocks
// none, GAP blocks their 1-runs).  The coverage plane of n0 is GT_n0 = { x : cnt(x) > n0 }.  In a whole-set AND-SUB call every
// vector is in exactly one group, so for x in AND(group0), with n0 = |group0|, cnt(x) = n0 + |{v in group1 : x in v}|, and
//     AND(group0) & ~OR(group1)  ==  AND(group0) & ~GT_n0.
// GT_n0 depends only on the set and n0, so one plane serves every such call whose AND group has n0 members, over any column range:
// the kernel streams the AND members' bit-blocks and the plane, and folds the plane as a SUB-group bit-block.
// Storage: slot[nb] = the pool slot (8 KB) holding column nb's plane, or kCovZero (no bit has cnt > n0) / kCovOne (every bit has).
#pragma once
#include "runlist_kernel.cuh"

namespace bmb200 {

constexpr uint32_t kCovZero   = ~0u;          // slot sentinel: the column's plane is empty (no SUB-group stage)
constexpr uint32_t kCovOne    = ~0u - 1u;     // ... the plane is full (the result column is NULL)
constexpr uint32_t kCovHalf   = 32768u;       // bits of a column whose GAP coverage one pass counts in shared memory
constexpr size_t   kCovSmem   = kCovHalf * 4u;
constexpr int      kCovWpt    = (int)kBlockWords / kRlThreads;   // words t + 512 k of the column, k < 4, per thread
constexpr int      kCovPlanes = 7;            // bit-sliced bit-block counts to 127, then sticky: > 64 >= n0 either way
static_assert(kCovHalf == 16u * kBlockWords && kCovWpt == 4, "each half of a column is words t + 512 k of two k per thread");

// One CTA per column: cnt(x) = (bit-blocks holding x) + (GAP 1-runs covering x) + (FULL blocks), compared with n0.
//   bit-blocks: per-thread bit-sliced saturating counters over the thread's 4 words;
//   GAP blocks: a difference array (+1 at s, -1 at e + 1, modulo 2^32) over one half of the column at a time, prefix-summed;
//   FULL blocks: a count per column.
// tot[0] hands out pool slots, tot[1] counts kCovOne columns (both zeroed before the launch).  pool has a slot for every column.
__global__ void __launch_bounds__(kRlThreads) cov_kernel(const SetView v, uint32_t n0, uint32_t* __restrict__ slot,
                                                         uint32_t* __restrict__ pool, unsigned long long* __restrict__ tot)
{
    extern __shared__ uint32_t D[];                             // [kCovHalf]
    __shared__ uint32_t s_w[kRlWarps], s_slot;
    const uint32_t nb = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31u;
    const uint32_t M = v.n_vec;
    const uint32_t* drow = v.desc + (size_t)nb * M;
    uint32_t nfull = 0;
    for (uint32_t x0 = 0; x0 < M; x0 += kRlThreads)
        nfull += __syncthreads_count(x0 + tid < M && (drow[x0 + tid] & 3u) == BMB200_BLK_FULL);
    if (nfull > n0) {
        if (tid == 0) { slot[nb] = kCovOne; atomicAdd(&tot[1], 1ull); }
        return;
    }
    const uint32_t T = n0 - nfull;                              // a bit is in the plane when its other blocks count more than T

    uint32_t c[kCovWpt][kCovPlanes], o[kCovWpt];
#pragma unroll
    for (int k = 0; k < kCovWpt; ++k) {
        o[k] = 0u;
#pragma unroll
        for (int p = 0; p < kCovPlanes; ++p) c[k][p] = 0u;
    }
    const uint64_t b0 = v.bit_base[nb];
    const uint32_t nbit = (uint32_t)(v.bit_base[nb + 1] - b0);
#pragma unroll 2
    for (uint32_t j = 0; j < nbit; ++j) {
        const uint32_t* blk = v.bit_pool + (b0 + j) * kBlockWords + tid;
        uint32_t x[kCovWpt];
#pragma unroll
        for (int k = 0; k < kCovWpt; ++k) x[k] = ld_nc_u32(blk + k * kRlThreads);
#pragma unroll
        for (int k = 0; k < kCovWpt; ++k) {
            uint32_t cy = x[k];
#pragma unroll
            for (int p = 0; p < kCovPlanes; ++p) { const uint32_t t = c[k][p] & cy; c[k][p] ^= cy; cy = t; }
            o[k] |= cy;
        }
    }

    uint32_t r[kCovWpt];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const uint32_t lo = (uint32_t)h * kCovHalf, hi = lo + kCovHalf - 1u;
        for (uint32_t i = tid; i < kCovHalf; i += kRlThreads) D[i] = 0u;
        __syncthreads();
        rl_gap_blocks(v, nb, warp, lane, nullptr, [&](const uint16_t* g) {
            const uint32_t hdr = g[0], n = gap_ones(hdr);
            for (uint32_t j = lane; j < n; j += 32u) {
                uint32_t s, e;
                gap_one_run(g, hdr, j, s, e);
                s = max(s, lo);
                if (s > min(e, hi)) continue;
                atomicAdd(&D[s - lo], 1u);
                if (e < hi) atomicAdd(&D[e + 1u - lo], ~0u);
            }
        });
        __syncthreads();
        // inclusive prefix sum: warp w takes entries [w * span, (w + 1) * span), 32 consecutive per step
        constexpr uint32_t span = kCovHalf / kRlWarps;
        uint32_t* Dw = D + warp * span;
        uint32_t sum = 0;
        for (uint32_t i = lane; i < span; i += 32u) sum += Dw[i];
        sum = warp_sum(sum);
        if (lane == 0) s_w[warp] = sum;
        __syncthreads();
        uint32_t carry = 0;
        for (uint32_t w = 0; w < warp; ++w) carry += s_w[w];
        for (uint32_t i = lane; i < span; i += 32u) {
            const uint32_t x = Dw[i];
            uint32_t t;
            Dw[i] = carry + warp_excl_scan(x, lane, t) + x;
            carry += t;
        }
        __syncthreads();
        // the warp's words 32 warp + 512 k + l, k = 2h, 2h + 1: lane l tests bit l of each word, so the reads of D are
        // conflict-free, and the word's owner keeps the ballot
#pragma unroll
        for (int k = 2 * h; k < 2 * h + 2; ++k) {
            const uint32_t w0 = 32u * warp + (uint32_t)k * kRlThreads;
            uint32_t mine = 0;
            for (uint32_t j = 0; j < 32u; ++j) {
                uint32_t b = 0;
#pragma unroll
                for (int p = 0; p < kCovPlanes; ++p) b |= ((__shfl_sync(0xffffffffu, c[k][p], j) >> lane) & 1u) << p;
                const bool ov = (__shfl_sync(0xffffffffu, o[k], j) >> lane) & 1u;
                const uint32_t m = __ballot_sync(0xffffffffu, ov || b + D[32u * (w0 + j) + lane - lo] > T);
                if (lane == j) mine = m;
            }
            r[k] = mine;
        }
        __syncthreads();                                        // D is zeroed again for the next half
    }

    bool any = false, all = true;
#pragma unroll
    for (int k = 0; k < kCovWpt; ++k) { any |= r[k] != 0u; all &= r[k] == ~0u; }
    any = __syncthreads_or(any); all = __syncthreads_and(all);
    if (all || !any) {
        if (tid == 0) { slot[nb] = all ? kCovOne : kCovZero; if (all) atomicAdd(&tot[1], 1ull); }
        return;
    }
    if (tid == 0) { s_slot = (uint32_t)atomicAdd(&tot[0], 1ull); slot[nb] = s_slot; }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kCovWpt; ++k) pool[(size_t)s_slot * kBlockWords + tid + (uint32_t)k * kRlThreads] = r[k];
}

}  // namespace bmb200
