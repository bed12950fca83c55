// column_walk.cuh -- what the kernels that walk the blocks of one block column share (sm_90a): a block as one thread's four
// words, the batched block loader with its GAP expansion, and the work-item claim.  GAP descriptors are decoded by
// gap_block_addr / gap_block_ptr (common.cuh).
// Used by the scans (scan_kernel.cuh, str_scan_kernel.cuh, scan_in_kernel.cuh), the mismatch and SHIFT-RIGHT-AND kernels and
// the rank compression kernels (rank_kernel.cuh).  agg_kernel.cuh keeps its own copies.
#pragma once
#include "agg_kernel.cuh"

namespace bmb200 {

// selected (1-) runs of one GAP block straight from global memory into the zeroed mask, all 512 threads
__device__ __forceinline__ void gap_expand_block(uint32_t Ks, const uint16_t* __restrict__ g, int tid)
{
    const uint32_t hdr = g[0];
    const uint32_t len = hdr >> 3;
    const bool odd = (hdr & 1u) != 0u;                       // first run is a 1-run
    const uint32_t nsel = odd ? (len + 1u) >> 1 : len >> 1;
    const uint16_t* a0 = g + (odd ? 0 : 1);
    for (uint32_t j = tid; j < nsel; j += kAggThreads) {
        const uint32_t sv = a0[2u * j], ev = a0[2u * j + 1u];
        apply_run<true>(Ks, (odd && j == 0u) ? 0u : sv + 1u, ev);   // runs of one block are disjoint: XOR into zeros == OR
    }
}

// a NULL, FULL or bit block as this thread's 4 words; bseg = the column's bit segment + threadIdx.x.  A GAP block reads as zeros.
__device__ __forceinline__ uint4 block_now(const uint4* bseg, uint32_t d)
{
    const uint32_t kind = d & 3u;
    if (kind == BMB200_BLK_BIT) return ld_stream_v4(bseg + (size_t)(d >> 2) * (kBlockWords / 4));
    return kind == BMB200_BLK_FULL ? make_uint4(~0u, ~0u, ~0u, ~0u) : make_uint4(0u, 0u, 0u, 0u);
}

// The blocks d[0..N) of one column as this thread's words P[0..N).  The NULL / FULL / bit loads are issued together; the GAP
// blocks are expanded into the 8 KB shared buffers K[u] and share one sequence of zero, barrier, expand, barrier, read,
// barrier (the last one because the next call rewrites the buffers).  d[] is the same for every thread, so when no block is
// GAP the whole CTA skips the barriers.
template <int N>
__device__ __forceinline__ void load_blocks(const uint32_t (&d)[N], uint4 (&P)[N], const uint4* bseg, const uint16_t* gseg,
                                            uint32_t (*K)[kBlockWords])
{
    const int tid = threadIdx.x;
    bool any_gap = false;
#pragma unroll
    for (int u = 0; u < N; ++u) {
        P[u] = block_now(bseg, d[u]);
        any_gap |= (d[u] & 3u) == BMB200_BLK_GAP;
    }
    if (!any_gap) return;
#pragma unroll
    for (int u = 0; u < N; ++u)
        if ((d[u] & 3u) == BMB200_BLK_GAP) reinterpret_cast<uint4*>(K[u])[tid] = make_uint4(0u, 0u, 0u, 0u);
    __syncthreads();
#pragma unroll
    for (int u = 0; u < N; ++u)
        if ((d[u] & 3u) == BMB200_BLK_GAP) gap_expand_block(smem_u32(K[u]), gap_block_ptr(gseg, d[u]), tid);
    __syncthreads();
#pragma unroll
    for (int u = 0; u < N; ++u)
        if ((d[u] & 3u) == BMB200_BLK_GAP) P[u] = reinterpret_cast<const uint4*>(K[u])[tid];
    __syncthreads();
}

// Work items are claimed one CTA at a time from a device counter.  Thread 0 claims the next item while the CTA works on the
// current one, and next() publishes it to every thread through s_item between two barriers (the first one also ends every
// thread's use of the previous item).  `stop` runs on thread 0 before publication; when it returns true the CTA gets `limit`
// instead, which ends its claim loop.  The caller leaves its loop at the first item >= limit.
struct NoStop {
    __device__ __forceinline__ bool operator()(uint32_t) const { return false; }
};
struct WorkClaim {
    uint32_t ahead;                                          // thread 0: the item claimed ahead

    __device__ __forceinline__ explicit WorkClaim(uint32_t* counter) : ahead(threadIdx.x == 0 ? atomicAdd(counter, 1u) : 0u) {}

    template <class Stop = NoStop>
    __device__ __forceinline__ uint32_t next(uint32_t* counter, uint32_t& s_item, uint32_t limit, Stop stop = Stop())
    {
        __syncthreads();
        if (threadIdx.x == 0) s_item = stop(ahead) ? limit : ahead;
        __syncthreads();
        const uint32_t item = s_item;
        if (threadIdx.x == 0 && item < limit) ahead = atomicAdd(counter, 1u);
        return item;
    }
};

}  // namespace bmb200
