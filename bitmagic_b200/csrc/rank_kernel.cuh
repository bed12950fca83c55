// rank_kernel.cuh -- rank compression and decompression against a NOT-NULL vector NN (sm_90a).
//
// Replaces bm::rank_compressor<BV> (src/bmalgo.h:498-644), the step that maps the search results of a rank-select compressed
// sparse vector (bm::rsc_sparse_vector<>, src/bmsparsevec_compr.h) between its compressed index space [0, count(NN)) and the
// logical one (sparse_vector_scanner::decompress, src/bmsparsevec_algo.h:4525-4537).
//
//   decompress: bit p of the target is set  iff  NN[p] is set and compressed bit rank_NN(p) - 1 is set
//   compress:   bit r of the target is set  iff  src is set at the position of the (r+1)-th set bit of NN
//
// For block nb of NN, cnt(nb) = its popcount (the rs-index bcount) and base(nb) = the exclusive prefix
// sb_cum[nb >> 8] + (nb & 255 ? row_cum[nb - 1] : 0), the expression rs_rank_kernel uses.  Bits [base, base + cnt) of the
// compressed space belong to block nb of the logical space, in order, and lie in at most two compressed block columns.
// Neither direction carries state from one block of NN to the next, so both are one CTA per block, like every other kernel here.
//
// Each thread owns 4 words of a block.  The exclusive prefix popcount of its words inside the block (a block scan) gives the
// compressed offset of its first bit.  Bits then move between a word of NN's space and a 32-bit window of the compressed space
// with a software PDEP / PEXT (the GPU has neither instruction).  The log-step form (Hacker's Delight, 7-4 / 7-5) is used rather
// than a loop over the set bits of the mask: it costs the same ~5 rounds whatever the density, while a loop would run every lane
// of a warp as long as its densest lane (up to 32 iterations per word, 128 per thread).
#pragma once
#include "gap_expand.cuh"
#include "aux_kernels.cuh"

namespace bmb200 {

// PEXT: the bits of x selected by m, packed to the low end
__host__ __device__ __forceinline__ uint32_t pext32(uint32_t x, uint32_t m)
{
    x &= m;
    uint32_t mk = ~m << 1;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
        uint32_t mp = mk ^ (mk << 1);
        mp ^= mp << 2; mp ^= mp << 4; mp ^= mp << 8; mp ^= mp << 16;
        const uint32_t mv = mp & m;
        m = (m ^ mv) | (mv >> (1 << i));
        const uint32_t t = x & mv;
        x = (x ^ t) | (t >> (1 << i));
        mk &= ~mp;
    }
    return x;
}

// PDEP: the low popc(m) bits of x deposited, in order, at the set bits of m
__host__ __device__ __forceinline__ uint32_t pdep32(uint32_t x, uint32_t m)
{
    const uint32_t m0 = m;
    uint32_t mk = ~m << 1, a[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) {
        uint32_t mp = mk ^ (mk << 1);
        mp ^= mp << 2; mp ^= mp << 4; mp ^= mp << 8; mp ^= mp << 16;
        const uint32_t mv = mp & m;
        a[i] = mv;
        m = (m ^ mv) | (mv >> (1 << i));
        mk &= ~mp;
    }
#pragma unroll
    for (int i = 4; i >= 0; --i) {
        const uint32_t t = x << (1 << i);
        x = (x & ~a[i]) | (t & a[i]);
    }
    return x & m0;
}

// Columns of an existing result read as a source: group g's compressed column c is result column g * cols_per_group + c
struct RankSrc {
    const uint8_t*  kind;      // [n_cols] BMB200_BLK_*
    const uint32_t* blocks;    // [n_cols][2048], valid for BIT columns
    const uint16_t* gaps;      // [n_cols][1280], valid for GAP columns
    uint32_t        cols_per_group;
};

__device__ __forceinline__ uint64_t rank_base(const RsView& nn, uint32_t nb)
{
    return nn.sb_cum[nb >> 8] + ((nb & 255u) ? nn.row_cum[nb - 1] : 0u);
}

// exclusive prefix of v over the 512 threads (warp scan + warp totals, as finish_block scans its run ends); one block barrier
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* s_w)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) s_w[warp] = inc;
    __syncthreads();
    uint32_t woff = 0;
#pragma unroll
    for (int w = 0; w < kAggWarps; ++w) if (w < warp) woff += s_w[w];
    return woff + inc - v;
}

// block `d` (a descriptor of set column nb) as this thread's 4 words; a GAP block must already be expanded into Kx
__device__ __forceinline__ uint4 rank_block_words(const SetView& s, uint32_t nb, uint32_t d, const uint32_t* Kx)
{
    const uint32_t kind = d & 3u;
    if (kind == BMB200_BLK_BIT)
        return ld_stream_v4(reinterpret_cast<const uint4*>(s.bit_pool) + (s.bit_base[nb] + (d >> 2)) * (size_t)(kBlockWords / 4) + threadIdx.x);
    if (kind == BMB200_BLK_GAP) return reinterpret_cast<const uint4*>(Kx)[threadIdx.x];
    return kind == BMB200_BLK_FULL ? make_uint4(~0u, ~0u, ~0u, ~0u) : make_uint4(0u, 0u, 0u, 0u);
}
__device__ __forceinline__ const uint16_t* rank_gap_ptr(const SetView& s, uint32_t nb, uint32_t d)
{
    const uint32_t rel = d >> 2;
    return s.gap_pool + s.gap_base[nb] * (size_t)kGapUnit + (size_t)(rel & kRelMask) * kGapUnit + (rel >> 29);
}

// decompress: one CTA per (group, output column nb), grid-stride over p.n_cols = n_groups * n_blocks(NN), group-major.
// The <= 2 source columns holding bits [base, base + cnt) are staged in shared memory; the epilogue is finish_block.
__global__ void __launch_bounds__(kAggThreads, kCtasPerSm) rank_decompress_kernel(const AggParams p, const RsView nn, const RankSrc src)
{
    __shared__ __align__(16) uint32_t S[2 * kBlockWords];    // source columns c0, c0 + 1
    __shared__ __align__(16) uint32_t K[kBlockWords];        // NN GAP expansion, then the epilogue scratch
    __shared__ uint32_t s_pc[kAggWarps], s_tr[kAggWarps], s_dg[kAggWarps], s_w[kAggWarps];
    const int tid = threadIdx.x;
    const uint32_t nnb = nn.set.n_blocks, cpg = src.cols_per_group;
    const uint32_t Ss = smem_u32(S), Ks = smem_u32(K);

    for (uint32_t item = blockIdx.x; item < p.n_cols; item += gridDim.x) {
        const uint32_t g = item / nnb, nb = item - g * nnb;
        const uint32_t d = nn.set.desc[(size_t)nb * nn.set.n_vec + nn.vec];
        const uint32_t cnt = nn.bcount[nb];
        uint4 R = make_uint4(0u, 0u, 0u, 0u);
        if ((d & 3u) != BMB200_BLK_NULL && cnt) {           // uniform; a NULL block of NN never reads the source
            const uint64_t base = rank_base(nn, nb);
            const uint32_t c0 = (uint32_t)(base >> 16), o = (uint32_t)(base & 0xffffu);
            const uint32_t ncol = (((base + cnt - 1u) >> 16) != c0) ? 2u : 1u;
            uint32_t sk[2];
            bool any_gap = (d & 3u) == BMB200_BLK_GAP;
#pragma unroll
            for (uint32_t i = 0; i < 2u; ++i) {              // stage: NULL / FULL / BIT now, GAP zeroed for the expansion
                const uint32_t c = c0 + i;
                sk[i] = (i < ncol && c < cpg) ? src.kind[(size_t)g * cpg + c] : BMB200_BLK_NULL;   // past the source's columns: zeros
                if (i >= ncol) break;
                uint4 v = make_uint4(0u, 0u, 0u, 0u);
                if (sk[i] == BMB200_BLK_FULL) v = make_uint4(~0u, ~0u, ~0u, ~0u);
                else if (sk[i] == BMB200_BLK_BIT)
                    v = ld_stream_v4(reinterpret_cast<const uint4*>(src.blocks) + ((size_t)g * cpg + c) * (kBlockWords / 4) + tid);
                else if (sk[i] == BMB200_BLK_GAP) any_gap = true;
                reinterpret_cast<uint4*>(S + i * kBlockWords)[tid] = v;
            }
            if ((d & 3u) == BMB200_BLK_GAP) reinterpret_cast<uint4*>(K)[tid] = make_uint4(0u, 0u, 0u, 0u);
            if (any_gap) {
                __syncthreads();
#pragma unroll
                for (uint32_t i = 0; i < 2u; ++i)
                    if (sk[i] == BMB200_BLK_GAP) gap_expand_block(Ss + i * kBlockWords * 4u, src.gaps + ((size_t)g * cpg + c0 + i) * kGapMax, tid);
                if ((d & 3u) == BMB200_BLK_GAP) gap_expand_block(Ks, rank_gap_ptr(nn.set, nb, d), tid);
            }
            __syncthreads();
            const uint4 M = rank_block_words(nn.set, nb, d, K);
            const uint32_t m[4] = {M.x, M.y, M.z, M.w};
            uint32_t off = o + block_exclusive_scan(__popc(M.x) + __popc(M.y) + __popc(M.z) + __popc(M.w), s_w);
            uint32_t r[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t wi = off >> 5, sh = off & 31u;
                const uint32_t x = __funnelshift_r(S[wi], S[min(wi + 1u, 2u * kBlockWords - 1u)], sh);   // compressed bits [off, off + 32)
                r[k] = m[k] == ~0u ? x : m[k] ? pdep32(x, m[k]) : 0u;
                off += __popc(m[k]);
            }
            R = make_uint4(r[0], r[1], r[2], r[3]);
            __syncthreads();                                 // K is rewritten by the epilogue
        }
        finish_block<true>(p, item, nb, g, R, 2, K, s_pc, s_tr, s_dg);
        __syncthreads();
    }
}

// compress, scatter half: one CTA per block nb of NN.  src & NN of the block is extracted (PEXT per word) into the bits
// [base, base + cnt) of a zeroed dense buffer.  The block assembles its range in shared memory first; words inside the range
// belong to this block alone (plain stores), only the first and the last can be shared with a neighbouring block (atomicOr).
// finalize_blocks_kernel then classifies the buffer's columns.  Scattering by NN block keeps the load even whatever NN's
// density: a gather per output column would put all of a very sparse NN on a few CTAs.
__global__ void __launch_bounds__(kAggThreads, kCtasPerSm) rank_compress_scatter_kernel(const RsView nn, uint32_t src_vec,
                                                                                        uint32_t* __restrict__ dense)
{
    __shared__ __align__(16) uint32_t G[2][kBlockWords];     // GAP expansions: [0] NN, [1] source
    __shared__ __align__(16) uint32_t O[kBlockWords + 4];    // the block's compressed range, word-aligned at base >> 5
    __shared__ uint32_t s_w[kAggWarps];
    const int tid = threadIdx.x;
    const SetView& s = nn.set;

    for (uint32_t nb = blockIdx.x; nb < s.n_blocks; nb += gridDim.x) {
        __syncthreads();                                     // the previous block's readers of G / O / s_w are done
        const uint32_t dn = s.desc[(size_t)nb * s.n_vec + nn.vec], ds = s.desc[(size_t)nb * s.n_vec + src_vec];
        const uint32_t cnt = nn.bcount[nb];
        if ((dn & 3u) == BMB200_BLK_NULL || (ds & 3u) == BMB200_BLK_NULL || !cnt) continue;   // uniform: nothing to write
        const uint64_t base = rank_base(nn, nb);
        const uint32_t lead = (uint32_t)(base & 31u), nw = (lead + cnt + 31u) >> 5;
        for (uint32_t j = tid; j < kBlockWords + 4u; j += kAggThreads) O[j] = 0u;
        const bool gn = (dn & 3u) == BMB200_BLK_GAP, gs = (ds & 3u) == BMB200_BLK_GAP;
        if (gn) reinterpret_cast<uint4*>(G[0])[tid] = make_uint4(0u, 0u, 0u, 0u);
        if (gs) reinterpret_cast<uint4*>(G[1])[tid] = make_uint4(0u, 0u, 0u, 0u);
        if (gn || gs) {
            __syncthreads();
            if (gn) gap_expand_block(smem_u32(G[0]), rank_gap_ptr(s, nb, dn), tid);
            if (gs) gap_expand_block(smem_u32(G[1]), rank_gap_ptr(s, nb, ds), tid);
        }
        __syncthreads();
        const uint4 M = rank_block_words(s, nb, dn, G[0]), V = rank_block_words(s, nb, ds, G[1]);
        const uint32_t m[4] = {M.x, M.y, M.z, M.w}, v[4] = {V.x, V.y, V.z, V.w};
        uint32_t off = lead + block_exclusive_scan(__popc(M.x) + __popc(M.y) + __popc(M.z) + __popc(M.w), s_w);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t e = m[k] == ~0u ? v[k] : pext32(v[k], m[k]);
            if (e) {
                const uint32_t wi = off >> 5, sh = off & 31u;
                red_or_shared(&O[wi], e << sh);
                if (sh && (e >> (32u - sh))) red_or_shared(&O[wi + 1u], e >> (32u - sh));
            }
            off += __popc(m[k]);
        }
        __syncthreads();
        uint32_t* dst = dense + (base >> 5);
        for (uint32_t j = tid; j < nw; j += kAggThreads) {
            const uint32_t w = O[j];
            if (!w) continue;                                // the buffer is zeroed
            if (j == 0u || j == nw - 1u) atomicOr(dst + j, w); else dst[j] = w;
        }
    }
}

}  // namespace bmb200
