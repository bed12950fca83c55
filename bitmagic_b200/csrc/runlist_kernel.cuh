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
// Those runs are part A of each column.  Part B lists, in the same encoding, the 1-runs of every sparse bit-block (a *listed*
// block: its list takes at most kListBitMax bytes).  A SUB-group bit-block only clears its 1-bits from the live mask, exactly as
// a GAP block's runs do, so a call whose AND group holds no listed block streams A + B and skips the listed 8 KB blocks.
// Per column, A's and B's singles are adjacent in sgl_pool ([sgl_base, sgl_mid) then [sgl_mid, sgl_base[nb+1])), and so are
// their long runs in lr_pool; each part is padded on its own.  listed: bit i = bit-block i of bit_pool is in part B.
#pragma once
#include "common.cuh"

namespace bmb200 {

constexpr int kRlThreads = 512;
constexpr int kRlWarps   = kRlThreads / 32;
// A bit-block is listed when 2 x singles + 4 x long runs <= kListBitMax bytes.  Every listed run is one more position for the
// consumers to sweep, so a larger threshold streams fewer bytes but sweeps more.  On C3 (H100 80GB HBM3, 400 W, DESIGN §6) the
// whole-set AND-SUB took 3.26 / 3.07 / 3.20 / 3.56 / 3.80 ms at 2048 / 3072 / 4096 / 6144 / 8192: 3072 is the fastest.
constexpr uint32_t kListBitMax = 3072u;

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

__device__ __forceinline__ uint32_t warp_excl_scan(uint32_t v, uint32_t lane, uint32_t& total)
{
    uint32_t x = v;
#pragma unroll
    for (uint32_t o = 1; o < 32u; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    total = __shfl_sync(0xffffffffu, x, 31);
    return x - v;
}

// One warp lists the 1-runs of the bit-block at w in bit order, 32 consecutive words per step, in part A's encoding: singles to
// sout[ns..), long-run pairs to lout16[2 nl..) (WRITE), or only counts them.  A pair is written as its two u16 halves: the lane
// holding the k-th long-run start writes s - 1 (0 for a run from bit 0), the lane holding the k-th long-run end writes e, so a
// run that crosses words or steps needs no pairing.  ns / nl are warp-uniform running counts.
template <bool WRITE>
__device__ __forceinline__ void rl_bit_block(const uint32_t* __restrict__ w, uint32_t lane, uint32_t& ns, uint32_t& nl,
                                             uint16_t* sout, uint16_t* lout16)
{
    uint32_t cs = 0, cl = 0, ne = nl;
#pragma unroll 4
    for (uint32_t i = lane; i < kBlockWords; i += 32u) {
        const uint32_t x = w[i];
        uint32_t pv = __shfl_up_sync(0xffffffffu, x, 1), nx = __shfl_down_sync(0xffffffffu, x, 1);
        if (lane == 0u)  pv = i ? w[i - 1u] : 0u;                           // the bits around the block are 0
        if (lane == 31u) nx = i + 1u < kBlockWords ? w[i + 1u] : 0u;
        const uint32_t S = x & ~((x << 1) | (pv >> 31)), E = x & ~((x >> 1) | (nx << 31));   // first / last bits of the 1-runs
        const uint32_t ls = S & ~E, le = E & ~S;                                              // ... of the long runs
        const uint32_t sm = (S & E) | (i == 0u ? ls & 1u : 0u);            // singles; a long run from bit 0 adds the single 0
        if (WRITE) {
            uint32_t ts, tl, te;
            uint32_t os = ns + warp_excl_scan(__popc(sm), lane, ts), ol = nl + warp_excl_scan(__popc(ls), lane, tl);
            uint32_t oe = ne + warp_excl_scan(__popc(le), lane, te);
            for (uint32_t m = sm; m; m &= m - 1u) sout[os++] = (uint16_t)(32u * i + (uint32_t)__ffs(m) - 1u);
            for (uint32_t m = ls; m; m &= m - 1u) {
                const uint32_t s = 32u * i + (uint32_t)__ffs(m) - 1u;
                lout16[2u * ol++] = (uint16_t)(s ? s - 1u : 0u);
            }
            for (uint32_t m = le; m; m &= m - 1u) lout16[2u * oe++ + 1u] = (uint16_t)(32u * i + (uint32_t)__ffs(m) - 1u);
            ns += ts; nl += tl; ne += te;
        } else {
            cs += __popc(sm); cl += __popc(ls);
        }
    }
    if (!WRITE) { ns += warp_sum(cs); nl += warp_sum(cl); }
}

// Part B of column nb: warp w takes the column's bit-blocks [w * per, (w + 1) * per), so their runs land in bit_pool order behind
// those of warps < w.  The count pass (!WRITE) measures every block, lists those within kListBitMax bytes (sets their flag, counts
// them in nlst) and counts their runs; the write pass lists the flagged blocks again.
template <bool WRITE>
__device__ __forceinline__ void rl_bits(const SetView v, uint32_t nb, uint32_t warp, uint32_t lane, uint32_t& ns, uint32_t& nl,
                                        uint32_t& nlst, uint32_t* listed, uint16_t* sout, uint16_t* lout16)
{
    const uint64_t b0 = v.bit_base[nb];
    const uint32_t n = (uint32_t)(v.bit_base[nb + 1] - b0), per = (n + kRlWarps - 1u) / kRlWarps;
    for (uint32_t j = warp * per; j < min(n, (warp + 1u) * per); ++j) {
        const uint64_t i = b0 + j;
        const uint32_t* blk = v.bit_pool + i * kBlockWords;
        if (WRITE) {
            if ((listed[i >> 5] >> (i & 31u)) & 1u) rl_bit_block<true>(blk, lane, ns, nl, sout, lout16);
        } else {
            uint32_t s = 0, l = 0;
            rl_bit_block<false>(blk, lane, s, l, nullptr, nullptr);
            if (2u * s + 4u * l <= kListBitMax) {
                ns += s; nl += l; ++nlst;
                if (lane == 0u) atomicOr(&listed[i >> 5], 1u << (i & 31u));
            }
        }
    }
}

// pass 1, one CTA per column: per-warp counts wcnt[nb][w] = (singles, long runs) of part A and wcnt[nb][kRlWarps + w] of part B,
// the listed flags (zeroed before the launch), the column's A + B sizes in 16-byte units, and the set's totals
// tot = (A singles units, A long-run units, B singles units, B long-run units, listed blocks), zeroed before the launch
__global__ void __launch_bounds__(kRlThreads) rl_count_kernel(const SetView v, uint2* __restrict__ wcnt, uint64_t* __restrict__ sgl_units,
                                                              uint64_t* __restrict__ lr_units, uint32_t* __restrict__ listed,
                                                              unsigned long long* __restrict__ tot)
{
    __shared__ uint2 s_c[2 * kRlWarps];
    __shared__ uint32_t s_n[kRlWarps];
    const uint32_t nb = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    uint32_t ns = 0, nl = 0, bs = 0, bl = 0, nlst = 0;
    rl_column<false>(v, nb, warp, lane, ns, nl, nullptr, nullptr);
    rl_bits<false>(v, nb, warp, lane, bs, bl, nlst, listed, nullptr, nullptr);
    if (lane == 0) {
        s_c[warp] = make_uint2(ns, nl); s_c[kRlWarps + warp] = make_uint2(bs, bl); s_n[warp] = nlst;
        wcnt[(size_t)nb * 2 * kRlWarps + warp] = make_uint2(ns, nl); wcnt[(size_t)nb * 2 * kRlWarps + kRlWarps + warp] = make_uint2(bs, bl);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t ts = 0, tl = 0, tbs = 0, tbl = 0, tn = 0;
        for (int w = 0; w < kRlWarps; ++w) {
            ts += s_c[w].x; tl += s_c[w].y; tbs += s_c[kRlWarps + w].x; tbl += s_c[kRlWarps + w].y; tn += s_n[w];
        }
        const uint32_t u[5] = {(ts + 7u) / 8u, (tl + 3u) / 4u, (tbs + 7u) / 8u, (tbl + 3u) / 4u, tn};
        sgl_units[nb] = u[0] + u[2];
        lr_units[nb] = u[1] + u[3];
#pragma unroll
        for (int k = 0; k < 5; ++k) if (u[k]) atomicAdd(&tot[k], (unsigned long long)u[k]);
    }
}

// pass 2, one CTA per column: every warp decodes its GAP blocks and lists its flagged bit-blocks again, straight into its slots of
// the column's parts (A at the column's bases, B at its mids), then the pads
__global__ void __launch_bounds__(kRlThreads) rl_write_kernel(const SetView v, const uint2* __restrict__ wcnt,
                                                              const uint64_t* __restrict__ sgl_base, const uint64_t* __restrict__ lr_base,
                                                              const uint32_t* __restrict__ listed, uint16_t* __restrict__ sgl,
                                                              uint32_t* __restrict__ lr, uint64_t* __restrict__ sgl_mid,
                                                              uint64_t* __restrict__ lr_mid)
{
    const uint32_t nb = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    uint32_t ns = 0, nl = 0, ts = 0, tl = 0, bs = 0, bl = 0, tbs = 0, tbl = 0, nlst = 0;
    for (uint32_t w = 0; w < (uint32_t)kRlWarps; ++w) {
        const uint2 c = wcnt[(size_t)nb * 2 * kRlWarps + w], cb = wcnt[(size_t)nb * 2 * kRlWarps + kRlWarps + w];
        if (w < warp) { ns += c.x; nl += c.y; bs += cb.x; bl += cb.y; }
        ts += c.x; tl += c.y; tbs += cb.x; tbl += cb.y;
    }
    const uint32_t scap = (ts + 7u) / 8u * 8u, lcap = (tl + 3u) / 4u * 4u, bscap = (tbs + 7u) / 8u * 8u, blcap = (tbl + 3u) / 4u * 4u;
    uint16_t* sout = sgl + sgl_base[nb] * 8u;
    uint32_t* lout = lr + lr_base[nb] * 4u;
    uint16_t* bsout = sout + scap;
    uint32_t* blout = lout + lcap;
    rl_column<true>(v, nb, warp, lane, ns, nl, sout, lout);
    rl_bits<true>(v, nb, warp, lane, bs, bl, nlst, const_cast<uint32_t*>(listed), bsout, reinterpret_cast<uint16_t*>(blout));
    if (threadIdx.x == 0) { sgl_mid[nb] = sgl_base[nb] + scap / 8u; lr_mid[nb] = lr_base[nb] + lcap / 4u; }
    __syncthreads();                                     // a part's last single is written before it is repeated
    for (uint32_t i = ts + threadIdx.x; i < scap; i += kRlThreads) sout[i] = sout[ts - 1u];
    for (uint32_t i = tl + threadIdx.x; i < lcap; i += kRlThreads) lout[i] = 0u;
    for (uint32_t i = tbs + threadIdx.x; i < bscap; i += kRlThreads) bsout[i] = bsout[tbs - 1u];
    for (uint32_t i = tbl + threadIdx.x; i < blcap; i += kRlThreads) blout[i] = 0u;
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

// bits[v >> 5] bit (v & 31) = vector v holds a listed bit-block in some column (bits zeroed before the launch); grid as above
__global__ void __launch_bounds__(256) listed_vectors_kernel(const uint32_t* __restrict__ desc, const uint64_t* __restrict__ bit_base,
                                                             const uint32_t* __restrict__ listed, uint32_t n_vec, uint32_t n_blocks,
                                                             uint32_t* __restrict__ bits)
{
    const uint32_t x = blockIdx.x * 256u + threadIdx.x;
    bool hit = false;
    if (x < n_vec)
        for (uint32_t nb = blockIdx.y; nb < n_blocks && !hit; nb += gridDim.y) {
            const uint32_t d = desc[(size_t)nb * n_vec + x];
            if ((d & 3u) != BMB200_BLK_BIT) continue;
            const uint64_t i = bit_base[nb] + ((d >> 2) & BMB200_DESC_REL_MASK);
            hit = (listed[i >> 5] >> (i & 31u)) & 1u;
        }
    const uint32_t m = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31u) == 0 && m) atomicOr(&bits[x >> 5], m);
}

}  // namespace bmb200
