// gap_expand.cuh -- one GAP block expanded into a zeroed 8 KB shared mask by all threads of a CTA (sm_90a).
// Shared by the bit-sliced scan (scan_kernel.cuh) and the rank compression kernels (rank_kernel.cuh).
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

}  // namespace bmb200
