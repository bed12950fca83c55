// aux_kernels.cuh -- result post-step (bit -> GAP), rs_index build + block-scan, batched rank/select,
// and the synthetic-set generator.  sm_90a only.
#pragma once
#include "common.cuh"

namespace bmb200 {

// ---------------------------------------------------------------------------------------------
// bit-block (in shared memory) -> GAP block.  Restates bit_block_to_gap (src/bmfunc.h:5540-5617) as
// "find every position p with bit[p] != bit[p+1], prefix-scan the per-thread counts, write the
// run ends in order".  256 threads, thread t owns words [8t, 8t+8).  Returns len (number of runs);
// out[0] = header with the capacity level set like allocate_gap_block (src/bmblocks.h:1902-1921).
// ---------------------------------------------------------------------------------------------
constexpr int kPostThreads = 256;

__device__ __forceinline__ uint32_t gap_level_for(uint32_t len)
{   // gap_calc_level src/bmfunc.h:5418 with the default table {128,256,512,1280}
    return len <= 124u ? 0u : len <= 252u ? 1u : len <= 508u ? 2u : 3u;
}

// s_blk: 2048 words in smem (+1 readable pad word not required), s_scan: 8 words, out: >= len+1 u16
__device__ uint32_t block_to_gap_256(const uint32_t* s_blk, uint32_t* s_scan, uint16_t* out, uint32_t max_len)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t x[8]; uint32_t cnt = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const uint32_t wi = 8u * tid + i;
        const uint32_t w = s_blk[wi];
        const uint32_t nxt = (wi + 1 < kBlockWords) ? (s_blk[wi + 1] & 1u) : (w >> 31);  // last bit: no successor
        x[i] = w ^ ((w >> 1) | (nxt << 31));
        cnt += __popc(x[i]);
    }
    // exclusive scan of cnt over 256 threads
    uint32_t inc = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) s_scan[warp] = inc;
    __syncthreads();
    uint32_t woff = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kPostThreads / 32; ++w) { const uint32_t v = s_scan[w]; if (w < warp) woff += v; total += v; }
    uint32_t off = woff + inc - cnt;          // run ends before this thread
    const uint32_t len = total + 1u;          // + the final run end 65535
    if (len <= max_len) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            uint32_t m = x[i];
            const uint32_t base = (8u * tid + i) * 32u;
            while (m) { const uint32_t b = __ffs(m) - 1u; m &= m - 1u; out[1u + off++] = (uint16_t)(base + b); }
        }
        if (tid == 0) {
            out[len] = 65535u;
            out[0] = (uint16_t)((s_blk[0] & 1u) | (gap_level_for(len) << 1) | (len << 3));
        }
    }
    __syncthreads();
    return len;
}

// result post-step: columns whose kind is GAP get their stored bit-block converted (opt_copy_bit_block's
// bit_to_gap branch, src/bmblocks.h:1389-1403).  gaps: [n_cols][1280] u16.
__global__ void __launch_bounds__(kPostThreads) result_to_gap_kernel(const uint32_t* __restrict__ blocks,
                                                                     const uint8_t* __restrict__ kind,
                                                                     uint16_t* __restrict__ gaps, uint32_t n_cols)
{
    __shared__ __align__(16) uint32_t s_blk[kBlockWords];
    __shared__ uint32_t s_scan[8];
    for (uint32_t col = blockIdx.x; col < n_cols; col += gridDim.x) {
        if (kind[col] != BMB200_BLK_GAP) continue;
        const uint4* src = reinterpret_cast<const uint4*>(blocks + (size_t)col * kBlockWords);
        uint4* dst = reinterpret_cast<uint4*>(s_blk);
        dst[threadIdx.x] = src[threadIdx.x];
        dst[threadIdx.x + kPostThreads] = src[threadIdx.x + kPostThreads];
        __syncthreads();
        block_to_gap_256(s_blk, s_scan, gaps + (size_t)col * kGapMax, kGapMax - 1u);
    }
}

// compaction of an optimized result into per-vector flat form: off[c] computed on the host from kinds
// and gap lengths; this kernel only moves data.  bits_out: compacted BIT blocks, gaps_out: compacted GAPs.
__global__ void __launch_bounds__(256) result_compact_kernel(const uint32_t* __restrict__ blocks,
                                                             const uint16_t* __restrict__ gaps,
                                                             const uint8_t* __restrict__ kind,
                                                             const uint64_t* __restrict__ off,
                                                             uint32_t* __restrict__ bits_out,
                                                             uint16_t* __restrict__ gaps_out, uint32_t n_cols)
{
    for (uint32_t col = blockIdx.x; col < n_cols; col += gridDim.x) {
        const uint32_t kd = kind[col];
        if (kd == BMB200_BLK_BIT) {
            const uint4* src = reinterpret_cast<const uint4*>(blocks + (size_t)col * kBlockWords);
            uint4* dst = reinterpret_cast<uint4*>(bits_out + off[col] * (size_t)kBlockWords);
            dst[threadIdx.x] = src[threadIdx.x];
            dst[threadIdx.x + 256] = src[threadIdx.x + 256];
        } else if (kd == BMB200_BLK_GAP) {
            const uint16_t* src = gaps + (size_t)col * kGapMax;
            uint16_t* dst = gaps_out + off[col];
            const uint32_t n = (uint32_t)(src[0] >> 3) + 1u;
            const uint32_t npad = (n + kGapUnit - 1u) / kGapUnit * kGapUnit;
            for (uint32_t i = threadIdx.x; i < npad; i += 256) dst[i] = (i < n) ? src[i] : (uint16_t)0;
        }
    }
}

// bmb200_set_upload_slabs: the host slabs were copied to the device as they lie (mirror); this kernel moves every real block from
// its place in the mirror (src[nb][v], 32-byte units) to its place in the column-major arena -- the device-side twin of
// host_pack.hpp's pack_column, same FLAT form (lead pad 0xFFFF iff the first run is 0, zeros up to the next 16-byte unit).
// One warp per block: 8 KB = 16 x 128-bit per lane; a GAP block without lead pad is a straight 128-bit copy (the mirror keeps
// the allocator's 32-byte alignment), one with lead pad shifts by one u16 through 16-bit loads.
// HBM bytes: every stored byte is read once and written once (+ 8 B of descriptor / source per block).
__global__ void __launch_bounds__(256) slab_gather_kernel(SetView set, const uint8_t* __restrict__ mirror,
                                                          const uint32_t* __restrict__ src)
{
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    for (uint32_t nb = blockIdx.x; nb < set.n_blocks; nb += gridDim.x) {
        const uint32_t* drow = set.desc + (size_t)nb * set.n_vec;
        const uint32_t* srow = src + (size_t)nb * set.n_vec;
        uint4* bit_dst = reinterpret_cast<uint4*>(const_cast<uint32_t*>(set.bit_pool) + set.bit_base[nb] * (size_t)kBlockWords);
        uint16_t* gap_dst = const_cast<uint16_t*>(set.gap_pool) + set.gap_base[nb] * (size_t)kGapUnit;
        for (uint32_t v = warp; v < set.n_vec; v += 8u) {
            const uint32_t d = drow[v], kd = d & 3u;
            if (kd == BMB200_BLK_BIT) {
                const uint4* in = reinterpret_cast<const uint4*>(mirror + (size_t)srow[v] * 32u);
                uint4* out = bit_dst + (size_t)((d >> 2) & BMB200_DESC_REL_MASK) * (kBlockWords / 4u);
                uint4 r[16];
#pragma unroll
                for (uint32_t k = 0; k < 16; ++k) r[k] = ld_stream_v4(in + lane + 32u * k);
#pragma unroll
                for (uint32_t k = 0; k < 16; ++k) out[lane + 32u * k] = r[k];
            } else if (kd == BMB200_BLK_GAP) {
                const uint16_t* in = reinterpret_cast<const uint16_t*>(mirror + (size_t)srow[v] * 32u);
                uint16_t* out = gap_dst + (size_t)((d >> 2) & BMB200_DESC_REL_MASK) * kGapUnit;
                const uint32_t words = (uint32_t)(in[0] >> 3) + 1u, pad = d >> 31;
                const uint32_t units = (words + pad + kGapUnit - 1u) / kGapUnit;
                if (!pad) {
                    for (uint32_t u = lane; u < units; u += 32u) {
                        uint4 q = reinterpret_cast<const uint4*>(in)[u];          // the last unit may read past the block: still inside the mirror (slack)
                        const uint32_t keep = words - u * kGapUnit;               // valid u16 in this unit (>= 1)
                        if (keep < kGapUnit) {
                            uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
                            for (uint32_t k = 0; k < 4; ++k) {
                                const uint32_t lo = 2u * k < keep ? 0xffffu : 0u, hi = 2u * k + 1u < keep ? 0xffff0000u : 0u;
                                w[k] &= lo | hi;
                            }
                            q = make_uint4(w[0], w[1], w[2], w[3]);
                        }
                        reinterpret_cast<uint4*>(out)[u] = q;
                    }
                } else {
                    for (uint32_t u = lane; u < units; u += 32u) {
                        uint32_t w[4];
#pragma unroll
                        for (uint32_t k = 0; k < 4; ++k) {
                            const uint32_t i0 = u * kGapUnit + 2u * k, i1 = i0 + 1u;      // output positions; input = position - 1
                            const uint32_t a = i0 == 0 ? 0xffffu : (i0 - 1u < words ? (uint32_t)in[i0 - 1u] : 0u);
                            const uint32_t b = i1 - 1u < words ? (uint32_t)in[i1 - 1u] : 0u;
                            w[k] = a | (b << 16);
                        }
                        reinterpret_cast<uint4*>(out)[u] = make_uint4(w[0], w[1], w[2], w[3]);
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// rs_index build (bvector::build_rs_index src/bm.h:2531-2660): one warp per block computes
//   bcount, first = bits in [0,21824], second = bits in (21824,43648], aux0, aux1
// bit-block : aux0/aux1 = bits in [0,32736] / [0,54560]              (src/bm.h:2626-2641)
// GAP block : aux = (gap_bfind(border+1) << 1) | is_set               (src/bm.h:2601-2625)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cnt_le(uint32_t w, uint32_t wi, uint32_t B)
{   // bits of word wi (bit positions 32*wi .. 32*wi+31) at positions <= B
    const uint32_t bw = B >> 5;
    if (wi < bw) return __popc(w);
    if (wi > bw) return 0u;
    return __popc(w & (0xffffffffu >> (31u - (B & 31u))));
}

// Device-private FINE index next to the reference-format fields (which stay exactly what rs_index::register_super_block
// receives): per block 128 entries, one per 512-bit window k:  bits 0..15 = ones in [0, 512k), bits 16..31 (GAP blocks) = index of
// the run that holds bit 512k (gap_bfind(512k)); plus 8 pivots (the entries of k = 0, 16, .., 112) for the two-level search of
// select.  The reference's anchors (rs3 borders, src/bmconst.h:120-124) bound a count_to scan to ~170 words = 11 sectors; with the
// fine index a query touches one 64-byte window of the block (2 sectors) -- what a sector-granular random-access bound asks for.
constexpr uint32_t kRsWin = 128u;           // 512-bit windows per block
constexpr uint32_t kRsPiv = 8u;             // pivots per block (every 16th window)
constexpr uint32_t kRsRowPiv = 16u;         // pivots per superblock row (every 16th block)

__global__ void __launch_bounds__(256) rs_block_kernel(const SetView set, uint32_t vec,
                                                       uint32_t* __restrict__ bcount,
                                                       uint64_t* __restrict__ sub_count,
                                                       uint32_t* __restrict__ fine, uint32_t* __restrict__ fine_piv)
{
    // GAP blocks: the whole block is staged in shared memory with 128-bit loads (it is at most 2.5 KB), a prefix of the ones per run is
    // built next to it, and everything the index needs -- the two rs3 borders and the 128 fine windows -- is then ONE binary search
    // each over the staged run ends (130 searches per block, 4-5 per lane) instead of per-run work with shared atomics
    __shared__ __align__(16) uint16_t s_raw[8][1296];
    __shared__ uint16_t s_pfx[8][1288];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const uint32_t warps_total = gridDim.x * (blockDim.x >> 5);
    for (uint32_t nb = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); nb < set.n_blocks; nb += warps_total) {
        const uint32_t d = set.desc[(size_t)nb * set.n_vec + vec];
        const uint32_t kd = d & 3u, rel = d >> 2;
        uint32_t tot = 0, le0 = 0, le1 = 0, a0 = 0, a1 = 0;
        uint32_t* fout = fine + (size_t)nb * kRsWin;
        if (kd == BMB200_BLK_GAP) {
            const auto [unit, pad] = gap_block_addr(set.gap_pool + set.gap_base[nb] * (size_t)kGapUnit, d);
            const uint32_t hdr = unit[pad], len = hdr >> 3, first = hdr & 1u;
            __syncwarp();
            {
                const uint4* src = reinterpret_cast<const uint4*>(unit);
                const uint32_t nvec = (len + 1u + pad + 7u) >> 3;
                for (uint32_t v = lane; v < nvec; v += 32u) reinterpret_cast<uint4*>(s_raw[wib])[v] = ld_stream_v4(src + v);
            }
            __syncwarp();
            const uint16_t* E = s_raw[wib] + pad;            // E[0] = header, E[1 .. len] = run ends
            uint16_t* P = s_pfx[wib];                        // P[k] = ones in runs 1 .. k (fits 16 bits for every k < len)
            uint32_t carry = 0;
            for (uint32_t base = 1u; base <= len; base += 256u) {        // 8 consecutive runs per lane and trip
                const uint32_t k0 = base + 8u * (uint32_t)lane;
                uint32_t prev = (k0 == 1u || k0 > len) ? 0xffffffffu : (uint32_t)E[k0 - 1u];      // run 1 starts at bit 0
                uint32_t loc[8], sum = 0;
#pragma unroll
                for (uint32_t q = 0; q < 8u; ++q) {
                    const uint32_t k = k0 + q;
                    if (k <= len) { const uint32_t e = E[k]; if (first ^ ((k - 1u) & 1u)) sum += e - prev; prev = e; }
                    loc[q] = sum;
                }
                uint32_t x = sum;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
                const uint32_t before = carry + x - sum;
#pragma unroll
                for (uint32_t q = 0; q < 8u; ++q) if (k0 + q <= len) P[k0 + q] = (uint16_t)(before + loc[q]);
                carry += __shfl_sync(0xffffffffu, x, 31);
            }
            if (lane == 0) P[0] = 0;
            tot = carry;
            __syncwarp();
            // 130 searches: the 128 window starts 512 t, then the two rs3 borders (positions B0 + 1 and B1 + 1)
            for (uint32_t t = lane; t < kRsWin + 2u; t += 32u) {
                const uint32_t b = t < kRsWin ? (t << 9) : (t == kRsWin ? kRs3B0 + 1u : kRs3B1 + 1u);
                uint32_t lo = 1u, hi = len;                              // first run j with E[j] >= b: the run that holds bit b (gap_bfind, src/bmfunc.h:1844)
                while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if ((uint32_t)E[mid] < b) lo = mid + 1u; else hi = mid; }
                const uint32_t j = lo, sj = (j == 1u) ? 0u : (uint32_t)E[j - 1u] + 1u, val = first ^ ((j - 1u) & 1u);
                const uint32_t ob = (uint32_t)P[j - 1u] + ((val && b > sj) ? b - sj : 0u);      // ones in [0, b)
                if (t < kRsWin) {
                    fout[t] = ob | (j << 16);
                    if ((t & 15u) == 0u) fine_piv[(size_t)nb * kRsPiv + (t >> 4)] = ob;
                } else if (t == kRsWin) { le0 = ob; a0 = (j << 1) | val; }
                else { le1 = ob; a1 = (j << 1) | val; }
            }
            // t = 128 ran on lane 0, t = 129 on lane 1
            le1 = __shfl_sync(0xffffffffu, le1, 1); a1 = __shfl_sync(0xffffffffu, a1, 1);
            __syncwarp();
        } else if (kd != BMB200_BLK_NULL) {
            if (kd == BMB200_BLK_BIT) {
                // 16 coalesced 512-byte warp loads per block, all issued before the popcounts (8 KB in flight per warp)
                const uint4* b4 = reinterpret_cast<const uint4*>(set.bit_pool + (set.bit_base[nb] + rel) * (size_t)kBlockWords);
                uint4 v[16];
#pragma unroll
                for (int it = 0; it < 16; ++it) v[it] = ld_stream_v4(b4 + it * 32 + lane);
                uint32_t carry = 0;                        // ones before the 8 windows of this iteration (warp-uniform)
#pragma unroll
                for (int it = 0; it < 16; ++it) {
                    const uint32_t wi = (uint32_t)(it * 32 + lane) * 4u;
                    const uint32_t w4[4] = {v[it].x, v[it].y, v[it].z, v[it].w};
                    uint32_t p4 = 0;
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const uint32_t w = w4[q];
                        p4 += __popc(w);
                        le0 += cnt_le(w, wi + q, kRs3B0);   le1 += cnt_le(w, wi + q, kRs3B1);
                        a0  += cnt_le(w, wi + q, kRs3B0_1); a1  += cnt_le(w, wi + q, kRs3B1_1);
                    }
                    tot += p4;
                    // fine index: 4 adjacent lanes = one 512-bit window (window it*8 + lane/4); exclusive scan over the 8 windows
                    uint32_t ws = p4 + __shfl_xor_sync(0xffffffffu, p4, 1);
                    ws += __shfl_xor_sync(0xffffffffu, ws, 2);
                    uint32_t x = ws;
#pragma unroll
                    for (int sft = 4; sft < 32; sft <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, sft); if (lane >= sft) x += y; }
                    const uint32_t before = carry + x - ws;
                    if ((lane & 3) == 0) {
                        const uint32_t k = (uint32_t)it * 8u + ((uint32_t)lane >> 2);
                        fout[k] = before;
                        if ((k & 15u) == 0u) fine_piv[(size_t)nb * kRsPiv + (k >> 4)] = before;
                    }
                    carry += __shfl_sync(0xffffffffu, x, 31);
                }
            } else {   // FULL block: an all-ones block, like BLOCK_ADDR_SAN in src/bm.h:2628
                for (uint32_t wi = lane; wi < kBlockWords; wi += 32) {
                    tot += 32u;
                    le0 += cnt_le(0xffffffffu, wi, kRs3B0);   le1 += cnt_le(0xffffffffu, wi, kRs3B1);
                    a0  += cnt_le(0xffffffffu, wi, kRs3B0_1); a1  += cnt_le(0xffffffffu, wi, kRs3B1_1);
                }
            }
            tot = warp_sum(tot); le0 = warp_sum(le0); le1 = warp_sum(le1); a0 = warp_sum(a0); a1 = warp_sum(a1);
        }
        if (lane == 0) {
            const uint32_t firstc = le0, secondc = le1 - le0;
            bcount[nb] = tot;
            sub_count[nb] = (uint64_t)(firstc | (secondc << 16)) | ((uint64_t)a0 << 32) | ((uint64_t)a1 << 48);
        }
    }
}

// block-scan, level 1: one CTA per 256-block superblock -> running counts inside the superblock
// (rs_index::register_super_block src/bmrs.h:688-715) and the superblock total
__global__ void __launch_bounds__(256) rs_scan_rows_kernel(const uint32_t* __restrict__ bcount, uint32_t n_blocks,
                                                           uint32_t* __restrict__ row_cum, uint64_t* __restrict__ sb_tot,
                                                           uint32_t* __restrict__ row_piv)
{
    __shared__ uint32_t s_w[8];
    const uint32_t sb = blockIdx.x, nb = sb * 256u + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t c = (nb < n_blocks) ? bcount[nb] : 0u;
    uint32_t inc = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) s_w[warp] = inc;
    __syncthreads();
    uint32_t woff = 0, total = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) { const uint32_t v = s_w[w]; if (w < warp) woff += v; total += v; }
    row_cum[nb] = woff + inc;                              // padded to whole superblocks: entries past n_blocks repeat the total
    if ((threadIdx.x & 15) == 15) row_piv[sb * kRsRowPiv + (threadIdx.x >> 4)] = woff + inc;     // inclusive count at the end of each group of 16 blocks
    if (threadIdx.x == 0) sb_tot[sb] = total;
}

// block-scan, level 2: running totals over superblocks (sblock_count_, src/bmrs.h:586-620); one CTA
__global__ void __launch_bounds__(1024) rs_scan_sb_kernel(const uint64_t* __restrict__ sb_tot, uint32_t nsb,
                                                          uint64_t* __restrict__ sb_cum)
{
    __shared__ uint64_t s_w[32];
    __shared__ uint64_t s_carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) { s_carry = 0; sb_cum[0] = 0; }
    __syncthreads();
    for (uint32_t base = 0; base < nsb; base += 1024u) {
        const uint32_t i = base + threadIdx.x;
        const uint64_t c = (i < nsb) ? sb_tot[i] : 0ull;
        uint64_t inc = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint64_t y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
        if (lane == 31) s_w[warp] = inc;
        __syncthreads();
        uint64_t woff = 0, total = 0;
        for (int w = 0; w < 32; ++w) { const uint64_t v = s_w[w]; if (w < warp) woff += v; total += v; }
        const uint64_t carry = s_carry;
        if (i < nsb) sb_cum[i + 1] = carry + woff + inc;
        __syncthreads();
        if (threadIdx.x == 0) s_carry = carry + total;
        __syncthreads();
    }
}

struct RsView {
    SetView set;
    uint32_t vec;
    uint32_t nsb;
    const uint32_t* bcount;     // [n_blocks]
    const uint64_t* sub_count;  // [n_blocks]
    const uint32_t* row_cum;    // [nsb * 256] inclusive running count inside the superblock (padded with the total)
    const uint64_t* sb_cum;     // [nsb+1]
    const uint32_t* fine;       // [n_blocks][128]   ones before window k | run index << 16
    const uint32_t* fine_piv;   // [n_blocks][8]     ones before window 16 q
    const uint32_t* row_piv;    // [nsb][16]         inclusive count at block 16 q + 15 of the superblock
};

// 1-bits of a GAP block in [from, to], scanning from run index k (run k must contain `from`)
__device__ __forceinline__ uint32_t gap_count_from(const uint16_t* __restrict__ g, uint32_t k, uint32_t from, uint32_t to)
{
    const uint32_t first = g[0] & 1u;
    uint32_t c = 0, s = from;
    for (;; ++k) {
        const uint32_t e = g[k];
        const uint32_t v = first ^ ((k - 1u) & 1u);
        if (e >= to) { if (v) c += to - s + 1u; break; }
        if (v) c += e - s + 1u;
        s = e + 1u;
    }
    return c;
}
__device__ __forceinline__ uint4 ld_nc_v4(const uint4* p)
{
    uint4 r; asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p)); return r;
}
// how many of the 4 words are < x
__device__ __forceinline__ uint32_t cnt_lt4(const uint4& v, uint32_t x) { return (v.x < x) + (v.y < x) + (v.z < x) + (v.w < x); }
__device__ __forceinline__ uint32_t cnt_lt4_lo16(const uint4& v, uint32_t x)
{ return ((v.x & 0xffffu) < x) + ((v.y & 0xffffu) < x) + ((v.z & 0xffffu) < x) + ((v.w & 0xffffu) < x); }

// inclusive rank, bvector::count_to src/bm.h:3120-3167.  One thread per query; per query: superblock total (cached), one
// row entry, the descriptor, ONE fine-index entry and at most one 64-byte window of the block (128-bit loads).
__global__ void __launch_bounds__(256) rs_rank_kernel(const RsView rs, const uint64_t* __restrict__ pos, uint64_t n,
                                                      uint64_t* __restrict__ out)
{
    for (uint64_t q = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; q < n; q += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t p = pos[q];
        const uint64_t nb64 = p >> 16;
        if (nb64 >= rs.set.n_blocks) { out[q] = rs.sb_cum[rs.nsb]; continue; }
        const uint32_t nb = (uint32_t)nb64, in = (uint32_t)(p & 0xffffu);
        uint64_t r = rs.sb_cum[nb >> 8] + ((nb & 255u) ? rs.row_cum[nb - 1] : 0u);
        const uint32_t d = rs.set.desc[(size_t)nb * rs.set.n_vec + rs.vec];
        const uint32_t kd = d & 3u, rel = d >> 2;
        if (kd == BMB200_BLK_FULL) r += in + 1u;
        else if (kd != BMB200_BLK_NULL) {
            const uint32_t k = in >> 9, f = rs.fine[(size_t)nb * kRsWin + k];
            uint32_t c = f & 0xffffu;
            if (kd == BMB200_BLK_BIT) {
                const uint4* w4 = reinterpret_cast<const uint4*>(rs.set.bit_pool + (rs.set.bit_base[nb] + rel) * (size_t)kBlockWords + 16u * k);
                const uint32_t wt = (in >> 5) & 15u;                        // word of `in` inside the window
                const uint32_t last = 0xffffffffu >> (31u - (in & 31u));   // bits <= in of that word
#pragma unroll
                for (uint32_t i = 0; i < 4; ++i) {
                    if (4u * i > wt) break;
                    const uint4 v = ld_nc_v4(w4 + i);
                    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                    for (uint32_t j = 0; j < 4; ++j) {
                        const uint32_t wi = 4u * i + j;
                        c += __popc(w[j] & (wi < wt ? 0xffffffffu : wi == wt ? last : 0u));
                    }
                }
            } else {
                const uint16_t* g = gap_block_ptr(rs.set.gap_pool + rs.set.gap_base[nb] * (size_t)kGapUnit, d);
                c += gap_count_from(g, f >> 16, k << 9, in);
            }
            r += c;
        }
        out[q] = r;
    }
}

// 1-based select, bvector::select src/bm.h:5350-5385 (rs_index::find src/bmrs.h:398-460, bit_find_rank src/bmfunc.h:9673-9768;
// word select via __fns instead of PDEP, src/bmbmi2.h:56-71).  One thread per query; every level below the superblock is a
// two-level search over 128-bit loads (16 pivots -> 16 entries), no dependent binary-search chains, then one 64-byte window.
__global__ void __launch_bounds__(256) rs_select_kernel(const RsView rs, const uint64_t* __restrict__ rank, uint64_t n,
                                                        uint64_t* __restrict__ pos, uint8_t* __restrict__ found)
{
    const uint64_t total = rs.sb_cum[rs.nsb];
    for (uint64_t q = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; q < n; q += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = rank[q];
        if (r == 0 || r > total) { found[q] = 0; pos[q] = 0; continue; }
        // smallest superblock i with sb_cum[i+1] >= r (the table is small and shared by every query: cache-resident)
        uint32_t lo = 0, hi = rs.nsb - 1u;
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (rs.sb_cum[mid + 1] < r) lo = mid + 1; else hi = mid; }
        const uint32_t sb = lo;
        uint32_t rr = (uint32_t)(r - rs.sb_cum[sb]);
        // block inside the superblock: group of 16 by the pivots, then the block by the group's 16 running counts
        const uint4* pv = reinterpret_cast<const uint4*>(rs.row_piv + (size_t)sb * kRsRowPiv);
        const uint4 p0 = ld_nc_v4(pv), p1 = ld_nc_v4(pv + 1), p2 = ld_nc_v4(pv + 2), p3 = ld_nc_v4(pv + 3);
        const uint32_t grp = cnt_lt4(p0, rr) + cnt_lt4(p1, rr) + cnt_lt4(p2, rr) + cnt_lt4(p3, rr);       // < 16: rr <= superblock total
        const uint4* rc = reinterpret_cast<const uint4*>(rs.row_cum + (size_t)sb * 256u + 16u * grp);
        const uint4 c0 = ld_nc_v4(rc), c1 = ld_nc_v4(rc + 1), c2 = ld_nc_v4(rc + 2), c3 = ld_nc_v4(rc + 3);
        const uint32_t j = cnt_lt4(c0, rr) + cnt_lt4(c1, rr) + cnt_lt4(c2, rr) + cnt_lt4(c3, rr);
        const uint32_t ce[16] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w, c2.x, c2.y, c2.z, c2.w, c3.x, c3.y, c3.z, c3.w};
        const uint32_t pe[16] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w, p2.x, p2.y, p2.z, p2.w, p3.x, p3.y, p3.z, p3.w};
        uint32_t prev = 0;
        if (j) {
#pragma unroll
            for (int i = 0; i < 15; ++i) if ((uint32_t)i + 1u == j) prev = ce[i];
        } else if (grp) {
#pragma unroll
            for (int i = 0; i < 15; ++i) if ((uint32_t)i + 1u == grp) prev = pe[i];
        }
        const uint32_t nb = sb * 256u + 16u * grp + j;
        rr -= prev;                                                        // rank inside the block, 1-based
        const uint32_t d = rs.set.desc[(size_t)nb * rs.set.n_vec + rs.vec];
        const uint32_t kd = d & 3u, rel = d >> 2;
        uint32_t bit = 0;
        if (kd == BMB200_BLK_FULL) bit = rr - 1u;
        else {
            // window: last k with (ones before window k) < rr -- 8 pivots, then the group's 16 entries
            const uint4* fp = reinterpret_cast<const uint4*>(rs.fine_piv + (size_t)nb * kRsPiv);
            const uint4 f0 = ld_nc_v4(fp), f1 = ld_nc_v4(fp + 1);
            const uint32_t g8 = cnt_lt4(f0, rr) + cnt_lt4(f1, rr) - 1u;   // pivot 0 is 0 < rr
            const uint4* fe = reinterpret_cast<const uint4*>(rs.fine + (size_t)nb * kRsWin + 16u * g8);
            const uint4 e0 = ld_nc_v4(fe), e1 = ld_nc_v4(fe + 1), e2 = ld_nc_v4(fe + 2), e3 = ld_nc_v4(fe + 3);
            const uint32_t kk = cnt_lt4_lo16(e0, rr) + cnt_lt4_lo16(e1, rr) + cnt_lt4_lo16(e2, rr) + cnt_lt4_lo16(e3, rr) - 1u;
            const uint32_t ee[16] = {e0.x, e0.y, e0.z, e0.w, e1.x, e1.y, e1.z, e1.w, e2.x, e2.y, e2.z, e2.w, e3.x, e3.y, e3.z, e3.w};
            uint32_t ent = ee[0];
#pragma unroll
            for (int i = 1; i < 16; ++i) if ((uint32_t)i == kk) ent = ee[i];
            const uint32_t k = 16u * g8 + kk;
            uint32_t need = rr - (ent & 0xffffu);                          // >= 1, and the window holds that many ones
            if (kd == BMB200_BLK_BIT) {
                const uint4* w4 = reinterpret_cast<const uint4*>(rs.set.bit_pool + (rs.set.bit_base[nb] + rel) * (size_t)kBlockWords + 16u * k);
                uint32_t wsel = 0, widx = 0; bool done = false;
#pragma unroll
                for (uint32_t i = 0; i < 4; ++i) {
                    if (done) break;
                    const uint4 v = ld_nc_v4(w4 + i);
                    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                    for (uint32_t jj = 0; jj < 4; ++jj) {
                        const uint32_t pc = __popc(w[jj]);
                        if (!done) { if (need <= pc) { wsel = w[jj]; widx = 4u * i + jj; done = true; } else need -= pc; }
                    }
                }
                bit = (16u * k + widx) * 32u + __fns(wsel, 0, (int)need);
            } else {
                const uint16_t* g = gap_block_ptr(rs.set.gap_pool + rs.set.gap_base[nb] * (size_t)kGapUnit, d);
                const uint32_t firstv = g[0] & 1u;
                uint32_t kr = ent >> 16, s = k << 9;
                for (;; ++kr) {
                    const uint32_t e = g[kr];
                    if (firstv ^ ((kr - 1u) & 1u)) {
                        const uint32_t rl = e - s + 1u;
                        if (need <= rl) { bit = s + need - 1u; break; }
                        need -= rl;
                    }
                    s = e + 1u;
                }
            }
        }
        found[q] = 1; pos[q] = ((uint64_t)nb << 16) | bit;
    }
}

// ---------------------------------------------------------------------------------------------
// synthetic set generator.  Bit (v, p) of vector v is set iff u16(hash(seed_v, p)) < thr_v with
// thr_v = round(density_v * 65536): a counter-based generator, so the classify pass and the write pass
// regenerate identical blocks.  One 64-bit hash yields four bits.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t mix64(uint64_t x)
{   // splitmix64 finalizer
    x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27; x *= 0x94d049bb133111ebull;
    x ^= x >> 31;
    return x;
}
__device__ __forceinline__ uint32_t synth_word(uint64_t seed, uint32_t nb, uint32_t wi, uint32_t thr)
{
    if (thr == 0) return 0u;
    if (thr >= 65536u) return 0xffffffffu;
    uint32_t w = 0;
    const uint64_t ctr = (((uint64_t)nb << 11) | wi) << 3;      // 8 hashes per word
#pragma unroll
    for (int h = 0; h < 8; ++h) {
        const uint64_t r = mix64(seed + 0x9e3779b97f4a7c15ull * (ctr + h + 1));
        w |= (uint32_t)((uint32_t)(r & 0xffffu) < thr) << (4 * h);
        w |= (uint32_t)((uint32_t)((r >> 16) & 0xffffu) < thr) << (4 * h + 1);
        w |= (uint32_t)((uint32_t)((r >> 32) & 0xffffu) < thr) << (4 * h + 2);
        w |= (uint32_t)((uint32_t)(r >> 48) < thr) << (4 * h + 3);
    }
    return w;
}

// pass 1: CTA per (nb, v): popcount + run count -> kind and stored size
__global__ void __launch_bounds__(kPostThreads) synth_classify_kernel(uint32_t n_vec, uint32_t n_blocks,
                                                                      const uint64_t* __restrict__ seed,
                                                                      const uint32_t* __restrict__ thr, int optimize,
                                                                      uint8_t* __restrict__ kind8,
                                                                      uint16_t* __restrict__ glen)
{
    __shared__ uint32_t s_pc[8], s_tr[8], s_last[kPostThreads];
    const uint64_t item = blockIdx.x;
    const uint32_t nb = (uint32_t)(item / n_vec), v = (uint32_t)(item % n_vec);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint64_t sd = seed[v]; const uint32_t th = thr[v];
    uint32_t w[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) w[i] = synth_word(sd, nb, 8u * tid + i, th);
    s_last[tid] = w[7] >> 31;
    __syncthreads();
    uint32_t prev = tid ? s_last[tid - 1] : (w[0] & 1u);
    uint32_t pc = 0, tr = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { pc += __popc(w[i]); tr += __popc(w[i] ^ ((w[i] << 1) | prev)); prev = w[i] >> 31; }
    pc = warp_sum(pc); tr = warp_sum(tr);
    if (lane == 0) { s_pc[warp] = pc; s_tr[warp] = tr; }
    __syncthreads();
    if (tid == 0) {
        uint32_t tpc = 0, ttr = 0;
        for (int i = 0; i < 8; ++i) { tpc += s_pc[i]; ttr += s_tr[i]; }
        const uint32_t runs = ttr + 1u;
        uint32_t kd;
        if (tpc == 0) kd = BMB200_BLK_NULL;
        else if (!optimize) kd = BMB200_BLK_BIT;
        else if (tpc == 65536u) kd = BMB200_BLK_FULL;
        else if (runs < BMB200_GAP_THRESHOLD) kd = BMB200_BLK_GAP;   // optimize_bit_block src/bmblocks.h:1414-1437
        else kd = BMB200_BLK_BIT;
        kind8[item] = (uint8_t)kd;
        glen[item] = (uint16_t)((runs & 0x7fffu) | ((w[0] & 1u) << 15));   // bit 15 = first bit (tid 0 owns word 0)
    }
}

// per column: exclusive scans over the vectors -> descriptors + column totals
__global__ void __launch_bounds__(256) synth_layout_kernel(uint32_t n_vec, uint32_t flat_form, const uint8_t* __restrict__ kind8,
                                                           const uint16_t* __restrict__ glen,
                                                           uint32_t* __restrict__ desc,
                                                           uint64_t* __restrict__ col_bits, uint64_t* __restrict__ col_gaps)
{
    __shared__ uint32_t s_wb[8], s_wg[8];
    __shared__ uint32_t s_cb, s_cg;
    const uint32_t nb = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { s_cb = 0; s_cg = 0; }
    __syncthreads();
    for (uint32_t base = 0; base < n_vec; base += 256u) {
        const uint32_t v = base + tid;
        uint32_t kd = 0, nbit = 0, ngap = 0, pad = 0;
        if (v < n_vec) {
            kd = kind8[(size_t)nb * n_vec + v];
            nbit = (kd == BMB200_BLK_BIT);
            if (kd == BMB200_BLK_GAP) {
                const uint32_t gl = glen[(size_t)nb * n_vec + v];
                pad = ((gl >> 15) || !flat_form) ? 0u : 1u;     // BMB200_DESC_GAP_FLAT: lead pad iff the first run is 0
                ngap = ((gl & 0x7fffu) + 1u + pad + kGapUnit - 1u) / kGapUnit;
            }
        }
        uint32_t ib = nbit, ig = ngap;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t yb = __shfl_up_sync(0xffffffffu, ib, o), yg = __shfl_up_sync(0xffffffffu, ig, o);
            if (lane >= o) { ib += yb; ig += yg; }
        }
        if (lane == 31) { s_wb[warp] = ib; s_wg[warp] = ig; }
        __syncthreads();
        uint32_t ob = s_cb, og = s_cg, tb = 0, tg = 0;
        for (int w = 0; w < 8; ++w) { if (w < warp) { ob += s_wb[w]; og += s_wg[w]; } tb += s_wb[w]; tg += s_wg[w]; }
        if (v < n_vec) {
            const uint32_t rel = (kd == BMB200_BLK_BIT) ? ob + ib - nbit : (kd == BMB200_BLK_GAP) ? og + ig - ngap : 0u;
            desc[(size_t)nb * n_vec + v] = kd | (rel << 2) | (pad << 31) | ((kd == BMB200_BLK_GAP && flat_form) ? BMB200_DESC_GAP_FLAT : 0u);
        }
        __syncthreads();
        if (tid == 0) { s_cb += tb; s_cg += tg; }
        __syncthreads();
    }
    if (tid == 0) { col_bits[nb] = s_cb; col_gaps[nb] = s_cg; }
}

// exclusive scan of per-column totals into bit_base / gap_base ([n+1]); one CTA
__global__ void __launch_bounds__(1024) scan_u64_kernel(const uint64_t* __restrict__ in, uint32_t n, uint64_t* __restrict__ out)
{
    __shared__ uint64_t s_w[32];
    __shared__ uint64_t s_carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) { s_carry = 0; out[0] = 0; }
    __syncthreads();
    for (uint32_t base = 0; base < n; base += 1024u) {
        const uint32_t i = base + threadIdx.x;
        const uint64_t c = (i < n) ? in[i] : 0ull;
        uint64_t inc = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint64_t y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
        if (lane == 31) s_w[warp] = inc;
        __syncthreads();
        uint64_t woff = 0, total = 0;
        for (int w = 0; w < 32; ++w) { const uint64_t v = s_w[w]; if (w < warp) woff += v; total += v; }
        const uint64_t carry = s_carry;
        if (i < n) out[i + 1] = carry + woff + inc;
        __syncthreads();
        if (threadIdx.x == 0) s_carry = carry + total;
        __syncthreads();
    }
}

// pass 2: regenerate and store every BIT / GAP block in its arena slot
__global__ void __launch_bounds__(kPostThreads) synth_write_kernel(uint32_t n_vec, uint32_t n_blocks,
                                                                   const uint64_t* __restrict__ seed,
                                                                   const uint32_t* __restrict__ thr,
                                                                   const uint32_t* __restrict__ desc,
                                                                   const uint64_t* __restrict__ bit_base,
                                                                   const uint64_t* __restrict__ gap_base,
                                                                   uint32_t* __restrict__ bit_pool,
                                                                   uint16_t* __restrict__ gap_pool)
{
    __shared__ __align__(16) uint32_t s_blk[kBlockWords];
    __shared__ uint32_t s_scan[8];
    const uint64_t item = blockIdx.x;
    const uint32_t nb = (uint32_t)(item / n_vec), v = (uint32_t)(item % n_vec);
    const uint32_t d = desc[item], kd = d & 3u, rel = (d >> 2) & BMB200_DESC_REL_MASK, pad = d >> 31;
    if (kd != BMB200_BLK_BIT && kd != BMB200_BLK_GAP) return;
    const int tid = threadIdx.x;
    const uint64_t sd = seed[v]; const uint32_t th = thr[v];
    uint32_t w[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) w[i] = synth_word(sd, nb, 8u * tid + i, th);
    if (kd == BMB200_BLK_BIT) {
        uint4* dst = reinterpret_cast<uint4*>(bit_pool + (bit_base[nb] + rel) * (size_t)kBlockWords) + 2 * tid;
        dst[0] = make_uint4(w[0], w[1], w[2], w[3]);
        dst[1] = make_uint4(w[4], w[5], w[6], w[7]);
    } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) s_blk[8 * tid + i] = w[i];
        __syncthreads();
        uint16_t* unit = gap_pool + (gap_base[nb] + rel) * (size_t)kGapUnit;
        uint16_t* out = unit + pad;
        const uint32_t len = block_to_gap_256(s_blk, s_scan, out, kGapMax - 1u);
        // lead pad = 0xFFFF, zeros from buf[len] to the end of the 16-byte unit (BMB200_DESC_GAP_FLAT contract)
        const uint32_t n = len + 1u + pad, npad = (n + kGapUnit - 1u) / kGapUnit * kGapUnit;
        if (tid < (int)(npad - n)) unit[n + tid] = 0;
        if (tid == 0 && pad) unit[0] = 0xffffu;
    }
}

}  // namespace bmb200
