// shift_kernel.cuh -- SHIFT-RIGHT-AND aggregation (sm_90a).
//
// Replaces aggregator<BV>::combine_shift_right_and (src/bmaggregator.h:2494-2669): with sources v_0 .. v_{n-1}
//     T_0 = v_0,   T_k = (T_{k-1} >> 1) & v_k,   result = T_{n-1}
// where ">> 1" moves every bit to the next higher index across the whole vector (bit_block_shift_r1: w = (w << 1) | carry,
// src/bmfunc.h:6391-6410).  The reference walks the blocks in order and hands one carry bit per source from block
// to block (carry_overs[], :2485-2489).  Unrolled, the recurrence is a pure gather with no carried state:
//     result[p] = AND_k  v_k[p - s_k],   s_k = n - 1 - k,   bits before position 0 read as 0
// so every block column is independent again (the block-range sharding of the other ops applies unchanged): block nb of the
// result needs block nb of every source shifted up by s_k bits plus the top s_k bits of its block nb - 1.
//
// One CTA per column, thread t owns words [4t, 4t+4) of the result in registers.  For each source the thread needs source
// words [4t - q - 1, 4t - q + 3] (q = s_k / 32): bit-blocks come straight from HBM as two aligned 128-bit loads (the
// second one is the neighbour's first: an L1 hit), GAP blocks are expanded once into an 8 KB shared mask, NULL / FULL are
// constants; indexes below 0 fall into block nb - 1 of the same source.  Epilogue = the aggregation kernel's (popcount,
// digest, run count, kind, bit->GAP); like every AND-type result an empty digest stores nothing (:2617-2632).
#pragma once
#include "column_walk.cuh"

namespace bmb200 {

__global__ void __launch_bounds__(kAggThreads, kCtasPerSm) shift_and_kernel(const AggParams p)
{
    __shared__ __align__(16) uint32_t K[kBlockWords];        // current block of a GAP source, expanded
    __shared__ __align__(16) uint32_t K2[kBlockWords];       // previous block of a GAP source, expanded
    __shared__ uint32_t s_col;
    __shared__ uint32_t s_pc[kAggWarps], s_tr[kAggWarps], s_dg[kAggWarps];

    const int tid = threadIdx.x;
    const uint32_t M = p.set.n_vec;
    uint4* K4 = reinterpret_cast<uint4*>(K);
    uint4* K24 = reinterpret_cast<uint4*>(K2);
    const uint32_t Ks = smem_u32(K), K2s = smem_u32(K2);

    WorkClaim claim(p.work_counter);
    for (;;) {
        const uint32_t item = claim.next(p.work_counter, s_col, p.n_cols * p.n_groups);
        if (item >= p.n_cols * p.n_groups) break;
        const uint32_t colx = item / p.n_groups, grp = item - colx * p.n_groups;
        const uint32_t col = grp * p.n_cols + colx;
        const uint32_t nb = p.nb_from + colx;
        const uint32_t gb0 = p.goff[2u * grp], gb1 = p.goff[2u * grp + 1u];
        const uint32_t n = gb1 - gb0;
        const uint32_t* gmem = p.group + gb0;
        const uint32_t* drow = p.set.desc + (size_t)nb * M;
        const uint32_t* drow_prev = nb ? drow - M : nullptr;
        const uint32_t* bcur = p.set.bit_pool + p.set.bit_base[nb] * (size_t)kBlockWords;
        const uint32_t* bprev = nb ? p.set.bit_pool + p.set.bit_base[nb - 1] * (size_t)kBlockWords : nullptr;
        const uint16_t* gcur = p.set.gap_pool + p.set.gap_base[nb] * (size_t)kGapUnit;
        const uint16_t* gprev = nb ? p.set.gap_pool + p.set.gap_base[nb - 1] * (size_t)kGapUnit : nullptr;

        uint4 R = make_uint4(~0u, ~0u, ~0u, ~0u);
        for (uint32_t k = 0; k < n; ++k) {
            const uint32_t v = gmem[k];
            const uint32_t s = n - 1u - k;                       // this source is shifted up by s bits (s < 65536 checked by the host)
            const uint32_t q = s >> 5, r = s & 31u;
            const uint32_t d = drow[v];
            const uint32_t dp = (drow_prev && s) ? drow_prev[v] : BMB200_BLK_NULL;
            const uint32_t kd = d & 3u, kp = dp & 3u;
            // stage GAP blocks as bits (uniform branches: d, dp are the same for every thread)
            if (kd == BMB200_BLK_GAP || kp == BMB200_BLK_GAP) {
                __syncthreads();                                 // previous source's readers are done with K / K2
                if (kd == BMB200_BLK_GAP) K4[tid] = make_uint4(0u, 0u, 0u, 0u);
                if (kp == BMB200_BLK_GAP) K24[tid] = make_uint4(0u, 0u, 0u, 0u);
                __syncthreads();
                if (kd == BMB200_BLK_GAP) gap_expand_block(Ks, gap_block_ptr(gcur, d), tid);
                if (kp == BMB200_BLK_GAP) gap_expand_block(K2s, gap_block_ptr(gprev, dp), tid);
                __syncthreads();
            }
            const uint32_t* bc = bcur + (size_t)(d >> 2) * kBlockWords;       // valid when kd == BIT
            const uint32_t* bp = bprev ? bprev + (size_t)(dp >> 2) * kBlockWords : nullptr;   // valid when kp == BIT
            auto word = [&](int idx) -> uint32_t {               // source word idx of block nb; idx < 0: block nb - 1
                if (idx >= 0) {
                    if (kd == BMB200_BLK_BIT) return ld_nc_u32(bc + idx);
                    if (kd == BMB200_BLK_GAP) return K[idx];
                    return kd == BMB200_BLK_FULL ? 0xffffffffu : 0u;
                }
                const int j = (int)kBlockWords + idx;
                if (kp == BMB200_BLK_BIT) return ld_nc_u32(bp + j);
                if (kp == BMB200_BLK_GAP) return K2[j];
                return kp == BMB200_BLK_FULL ? 0xffffffffu : 0u;
            };
            const int base = 4 * tid - (int)q;
            uint32_t w[5];
            if (kd == BMB200_BLK_BIT && base >= 4 && (q & 3u) == 0u) {
                // interior, word-quad aligned shift: two aligned 128-bit loads cover words base-4 .. base+3 (the first one is
                // the left neighbour's second: an L1 hit)
                const uint4 a = reinterpret_cast<const uint4*>(bc)[(base >> 2) - 1];
                const uint4 b = reinterpret_cast<const uint4*>(bc)[base >> 2];
                w[0] = a.w; w[1] = b.x; w[2] = b.y; w[3] = b.z; w[4] = b.w;
            } else {
#pragma unroll
                for (int i = 0; i < 5; ++i) w[i] = word(base - 1 + i);
            }
            uint4 P;
            if (r) {
                P.x = (w[1] << r) | (w[0] >> (32u - r)); P.y = (w[2] << r) | (w[1] >> (32u - r));
                P.z = (w[3] << r) | (w[2] >> (32u - r)); P.w = (w[4] << r) | (w[3] >> (32u - r));
            } else { P.x = w[1]; P.y = w[2]; P.z = w[3]; P.w = w[4]; }
            R.x &= P.x; R.y &= P.y; R.z &= P.z; R.w &= P.w;
        }
        __syncthreads();                                         // K is reused as scratch by the epilogue
        int state = n ? 2 : 0;
        if (!n) R = make_uint4(0u, 0u, 0u, 0u);
        finish_block<true>(p, col, colx, grp, R, state, K, s_pc, s_tr, s_dg);
    }
}

}  // namespace bmb200
