// remap_kernel.cuh -- the image of a set of ids through a sparse vector (sm_90a).
//
// Replaces bm::set2set_11_transform<SV>::remap(bv_in, sv, bv_out) (src/bmsparsevec_algo.h:2097-2205): bit v of the output is
// set iff some id i of the input (inside the vector's NOT-NULL vector when it is nullable) holds the value v = sv[i].  The
// reference enumerates the input id by id, gathers the values in 8 K batches and sets them into the output.  Here:
//   * one work item per column of the source result; the mask is the source block (NULL, FULL, bit or GAP), ANDed with the
//     NOT-NULL block of a nullable vector.  A column whose mask is empty reads no plane, and a chunk of the column without a
//     masked element is not staged, so the work follows the input's populated columns;
//   * a column whose plane blocks are all NULL (every column past the set's) maps every masked element to 0;
//   * otherwise the planes are staged chunk by chunk (stage_chunk, shared with scan_in_kernel) and each warp rebuilds the codes
//     of one 32-element word at a time with warp_transpose32;
//   * every masked code below id_max sets its bit in a zeroed dense image of max(1, 2^(n_planes - 16)) columns.  Many ids onto
//     few values is the normal case, so a warp first groups its lanes by target word (one OR per distinct word), and the
//     group's leader skips the atomic when its bits are already set: bits only ever get set, so a stale read can cost an
//     atomic but never lose a bit.
// finalize_blocks_kernel then classifies the image's columns, as for rank compression.
#pragma once
#include "scan_in_kernel.cuh"
#include "rank_kernel.cuh"

namespace bmb200 {

struct RemapParams {
    SetView   set;             // the set holding the translation vector
    RankSrc   src;             // the source result, one group: source column c = element block c
    uint32_t  n_cols;          // the source's columns = work items
    uint32_t  plane0;          // plane j (bit j of the value) = set vector plane0 + j
    uint32_t  n_planes;        // 1..32
    uint32_t  not_null;        // the NOT-NULL vector; 0xffffffff = not nullable
    uint64_t  id_max;          // values >= id_max are left out
    uint32_t* dense;           // the zeroed image, bit v = value v
    uint32_t* work_counter;
};

// dynamic shared memory of remap_kernel: the mask, the NOT-NULL GAP expansion, n_planes rows of one chunk
__host__ inline size_t remap_smem(uint32_t n_planes)
{
    return 2u * (size_t)kBlockWords * 4u + (size_t)n_planes * kInRowStride * 4u;
}

__global__ void __launch_bounds__(kAggThreads, kCtasPerSm) remap_kernel(const RemapParams rp)
{
    extern __shared__ __align__(16) uint32_t s_rm[];
    uint32_t* Mk = s_rm;                                                 // the column's mask
    uint32_t* G = Mk + kBlockWords;                                      // GAP expansion of the NOT-NULL block
    uint32_t* rows = G + kBlockWords;                                    // planes 0..n-1: one chunk each
    __shared__ uint32_t s_desc[32];
    __shared__ uint32_t s_col;
    __shared__ uint32_t s_wany[kAggWarps];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t np = rp.n_planes;
    const bool nullable = rp.not_null != 0xffffffffu;

    WorkClaim claim(rp.work_counter);
    for (;;) {
        const uint32_t c = claim.next(rp.work_counter, s_col, rp.n_cols);
        if (c >= rp.n_cols) break;
        const bool in_set = c < rp.set.n_blocks;                         // past the set's columns every plane reads 0
        const uint32_t* drow = rp.set.desc + (size_t)c * rp.set.n_vec;
        if (tid < (int)np) s_desc[tid] = in_set ? drow[rp.plane0 + tid] : (uint32_t)BMB200_BLK_NULL;
        const uint32_t sk = rp.src.kind[c];
        const uint32_t dn = !nullable ? (uint32_t)BMB200_BLK_FULL : in_set ? drow[rp.not_null] : (uint32_t)BMB200_BLK_NULL;
        if (sk == BMB200_BLK_NULL || (dn & 3u) == BMB200_BLK_NULL) continue;   // uniform: nothing to map
        const uint4* bseg = in_set ? reinterpret_cast<const uint4*>(rp.set.bit_pool) + rp.set.bit_base[c] * (size_t)(kBlockWords / 4) : nullptr;
        const uint16_t* gseg = in_set ? rp.set.gap_pool + rp.set.gap_base[c] * (size_t)kGapUnit : nullptr;

        // the mask: source block & NOT-NULL block, both GAP expansions behind one pair of barriers
        const bool gs = sk == BMB200_BLK_GAP, gn = (dn & 3u) == BMB200_BLK_GAP;
        if (gs) reinterpret_cast<uint4*>(Mk)[tid] = make_uint4(0u, 0u, 0u, 0u);
        if (gn) reinterpret_cast<uint4*>(G)[tid] = make_uint4(0u, 0u, 0u, 0u);
        if (gs || gn) {
            __syncthreads();
            if (gs) gap_expand_block(smem_u32(Mk), rp.src.gaps + (size_t)c * kGapMax, tid);
            if (gn) gap_expand_block(smem_u32(G), gap_block_ptr(gseg, dn), tid);
            __syncthreads();
        }
        uint4 m = sk == BMB200_BLK_FULL ? make_uint4(~0u, ~0u, ~0u, ~0u)
                : sk == BMB200_BLK_BIT  ? ld_stream_v4(reinterpret_cast<const uint4*>(rp.src.blocks) + (size_t)c * (kBlockWords / 4) + tid)
                                        : reinterpret_cast<const uint4*>(Mk)[tid];
        if (nullable) {
            const uint4 n = gn ? reinterpret_cast<const uint4*>(G)[tid] : block_now(bseg + tid, dn);
            m.x &= n.x; m.y &= n.y; m.z &= n.z; m.w &= n.w;
        }
        reinterpret_cast<uint4*>(Mk)[tid] = m;                           // this thread's words only
        // where the masked elements sit: thread t holds words [4t, 4t + 4), so warp w covers half of chunk w / 2
        const bool any = __any_sync(0xffffffffu, (m.x | m.y | m.z | m.w) != 0u);
        if (lane == 0) s_wany[warp] = any ? 1u : 0u;
        __syncthreads();                                                 // Mk, s_wany and s_desc are complete
        constexpr uint32_t kWarpsPerChunk = kInChunkWords / 128u;
        uint32_t chunks = 0u;
#pragma unroll
        for (int w = 0; w < kAggWarps; ++w) chunks |= s_wany[w] << (w / kWarpsPerChunk);
        if (!chunks) continue;                                           // uniform
        bool any_gap = false, all_null = true;
        for (uint32_t r = 0; r < np; ++r) {
            any_gap |= (s_desc[r] & 3u) == BMB200_BLK_GAP;
            all_null &= (s_desc[r] & 3u) == BMB200_BLK_NULL;
        }
        if (all_null) {                                                  // every masked element holds 0
            if (tid == 0 && rp.id_max > 0u && !(*rp.dense & 1u)) atomicOr(rp.dense, 1u);
            continue;
        }
        const auto desc = [&](uint32_t r) { return s_desc[r]; };
        for (uint32_t k = 0; k < kBlockWords / kInChunkWords; ++k) {
            if (!((chunks >> k) & 1u)) continue;                         // uniform
            const uint32_t c0 = k * kInChunkWords;
            stage_chunk(rows, np, desc, any_gap, bseg, gseg, c0, tid);
            for (uint32_t w = (uint32_t)warp; w < kInChunkWords; w += kAggWarps) {
                const uint32_t mw = Mk[c0 + w];
                if (!mw) continue;                                       // warp-uniform
                const uint32_t code = warp_transpose32((uint32_t)lane < np ? rows[lane * kInRowStride + w] : 0u, lane);
                const bool on = ((mw >> lane) & 1u) && code < rp.id_max;
                const uint32_t act = __ballot_sync(0xffffffffu, on);
                if (on) {
                    const uint32_t word = code >> 5;
                    const uint32_t grp = __match_any_sync(act, word);    // the lanes that hit this word
                    const uint32_t bits = __reduce_or_sync(grp, 1u << (code & 31u));
                    if ((uint32_t)lane == (uint32_t)(__ffs(grp) - 1)) {
                        uint32_t* dst = rp.dense + word;
                        if ((*dst & bits) != bits) atomicOr(dst, bits);
                    }
                }
            }
            __syncthreads();                                             // the rows are restaged by the next chunk
        }
    }
}

}  // namespace bmb200
