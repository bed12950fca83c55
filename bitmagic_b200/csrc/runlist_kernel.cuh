// runlist_kernel.cuh -- the run-list companion of a set's GAP blocks (built once per set, streamed by agg_pipe_kernel).
//
// For a whole-set AND-SUB whose AND group holds no GAP block, every GAP block of the set is a SUB-group block: the GAP phase only
// clears the union of all GAP 1-runs of the column from the live mask, so block identity and order do not matter.  The companion
// re-encodes those 1-runs per column nb in two parts, each padded to whole 16-byte units:
//   singles   sgl_pool units [sgl_base[nb], sgl_base[nb+1]): one u16 bit position per 1-run of length 1, padded with repeats of
//             the part's last entry (clearing a bit twice is harmless);
//   long runs lr_pool units  [lr_base[nb],  lr_base[nb+1]):  one FLAT pair (s - 1 | e << 16) per 1-run [s, e] with e > s, padded
//             with (0, 0) = no run.  A long run from bit 0 is stored as the single 0 plus the pair (0, e).
// At C3's densities (<= 1 %) almost every 1-run is a single bit: 2 bytes instead of the 4 of a FLAT pair.
// The build decodes every GAP block from its header, so FLAT and raw-form sets both have a companion.
#pragma once
#include "common.cuh"

namespace bmb200 {

constexpr int kRlThreads = 512;
constexpr int kRlWarps   = kRlThreads / 32;

// One warp decodes the GAP block at g (= &buf[0], lead pad already skipped) and appends its 1-runs in order: singles to sout[ns..),
// long-run pairs to lout[nl..) (WRITE), or only counts them.  ns / nl are warp-uniform running counts.
template <bool WRITE>
__device__ __forceinline__ void rl_block(const uint16_t* __restrict__ g, uint32_t lane, uint32_t& ns, uint32_t& nl,
                                         uint16_t* sout, uint32_t* lout)
{
    const uint32_t hdr = g[0], len = hdr >> 3, first = hdr & 1u;
    const uint32_t nsel = first ? (len + 1u) >> 1 : len >> 1;      // 1-runs: k = 2j+1 (first run is 1) or 2j+2
    const uint32_t lt = (1u << lane) - 1u;
    for (uint32_t j0 = 0; j0 < nsel; j0 += 32u) {
        const uint32_t j = j0 + lane;
        uint32_t s = 0, e = 0;
        const bool ok = j < nsel;
        if (ok) {
            const uint32_t k = 2u * j + (first ? 1u : 2u);
            s = (k == 1u) ? 0u : g[k - 1u] + 1u;
            e = g[k];
        }
        const bool sg = ok && (s == e || s == 0u), lg = ok && e > s;
        const uint32_t bs = __ballot_sync(0xffffffffu, sg), bl = __ballot_sync(0xffffffffu, lg);
        if (WRITE) {
            if (sg) sout[ns + __popc(bs & lt)] = (uint16_t)s;
            if (lg) lout[nl + __popc(bl & lt)] = (s ? s - 1u : 0u) | (e << 16);
        }
        ns += __popc(bs); nl += __popc(bl);
    }
}

// Warp w of a column takes vectors [w * per, (w + 1) * per): its runs land in vector order behind those of warps < w.
template <bool WRITE>
__device__ __forceinline__ void rl_column(const SetView v, uint32_t nb, uint32_t warp, uint32_t lane, uint32_t& ns, uint32_t& nl,
                                          uint16_t* sout, uint32_t* lout)
{
    const uint32_t M = v.n_vec, per = (M + kRlWarps - 1u) / kRlWarps;
    const uint32_t* drow = v.desc + (size_t)nb * M;
    const uint16_t* gseg = v.gap_pool + v.gap_base[nb] * (size_t)kGapUnit;
    for (uint32_t v0 = warp * per; v0 < min(M, (warp + 1u) * per); v0 += 32u) {
        const uint32_t x = v0 + lane;
        const uint32_t d = (x < min(M, (warp + 1u) * per)) ? drow[x] : BMB200_BLK_NULL;
        uint32_t m = __ballot_sync(0xffffffffu, (d & 3u) == BMB200_BLK_GAP);
        while (m) {
            const int l = __ffs(m) - 1; m &= m - 1u;
            const uint32_t dl = __shfl_sync(0xffffffffu, d, l);
            rl_block<WRITE>(gseg + (size_t)((dl >> 2) & BMB200_DESC_REL_MASK) * kGapUnit + (dl >> 31), lane, ns, nl, sout, lout);
        }
    }
}

// pass 1, one CTA per column: per-warp counts wcnt[nb][w] = (singles, long runs), and the column's part sizes in 16-byte units
__global__ void __launch_bounds__(kRlThreads) rl_count_kernel(const SetView v, uint2* __restrict__ wcnt, uint64_t* __restrict__ sgl_units,
                                                              uint64_t* __restrict__ lr_units)
{
    __shared__ uint2 s_c[kRlWarps];
    const uint32_t nb = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    uint32_t ns = 0, nl = 0;
    rl_column<false>(v, nb, warp, lane, ns, nl, nullptr, nullptr);
    if (lane == 0) { s_c[warp] = make_uint2(ns, nl); wcnt[(size_t)nb * kRlWarps + warp] = make_uint2(ns, nl); }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t ts = 0, tl = 0;
        for (int w = 0; w < kRlWarps; ++w) { ts += s_c[w].x; tl += s_c[w].y; }
        sgl_units[nb] = (ts + 7u) / 8u;
        lr_units[nb] = (tl + 3u) / 4u;
    }
}

// pass 2, one CTA per column: every warp decodes its vectors again, straight into its slots of the two parts, then the pads
__global__ void __launch_bounds__(kRlThreads) rl_write_kernel(const SetView v, const uint2* __restrict__ wcnt,
                                                              const uint64_t* __restrict__ sgl_base, const uint64_t* __restrict__ lr_base,
                                                              uint16_t* __restrict__ sgl, uint32_t* __restrict__ lr)
{
    const uint32_t nb = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    uint16_t* sout = sgl + sgl_base[nb] * 8u;
    uint32_t* lout = lr + lr_base[nb] * 4u;
    const uint32_t scap = (uint32_t)(sgl_base[nb + 1] - sgl_base[nb]) * 8u, lcap = (uint32_t)(lr_base[nb + 1] - lr_base[nb]) * 4u;
    uint32_t ns = 0, nl = 0, ts = 0, tl = 0;
    for (uint32_t w = 0; w < (uint32_t)kRlWarps; ++w) {
        const uint2 c = wcnt[(size_t)nb * kRlWarps + w];
        if (w < warp) { ns += c.x; nl += c.y; }
        ts += c.x; tl += c.y;
    }
    rl_column<true>(v, nb, warp, lane, ns, nl, sout, lout);
    __syncthreads();                                     // the part's last single is written before it is repeated
    for (uint32_t i = ts + threadIdx.x; i < scap; i += kRlThreads) sout[i] = sout[ts - 1u];
    for (uint32_t i = tl + threadIdx.x; i < lcap; i += kRlThreads) lout[i] = 0u;
}

// bits[v >> 5] bit (v & 31) = vector v holds a GAP block in some column (bits zeroed before the launch); grid (vector tiles, column slices)
__global__ void __launch_bounds__(256) gap_vectors_kernel(const uint32_t* __restrict__ desc, uint32_t n_vec, uint32_t n_blocks,
                                                          uint32_t* __restrict__ bits)
{
    const uint32_t x = blockIdx.x * 256u + threadIdx.x;
    bool gap = false;
    if (x < n_vec)
        for (uint32_t nb = blockIdx.y; nb < n_blocks && !gap; nb += gridDim.y) gap = (desc[(size_t)nb * n_vec + x] & 3u) == BMB200_BLK_GAP;
    const uint32_t m = __ballot_sync(0xffffffffu, gap);
    if ((threadIdx.x & 31u) == 0 && m) atomicOr(&bits[x >> 5], m);
}

}  // namespace bmb200
