// mismatch_kernel.cuh -- where two sparse vectors differ, in one pass over both vectors' planes (sm_90a).
//
// Replaces the reference's
//   sparse_vector_find_mismatch(bv, sv1, sv2, null_proc)          src/bmsparsevec_algo.h:657
//   sparse_vector_find_first_mismatch(sv1, sv2, midx, null_proc)   src/bmsparsevec_algo.h:479
// which run one bit_xor into a temporary bvector per plane, one OR pass and a NULL pass (or one find_first_mismatch per plane).
// Both are plane-parallel: per block column
//     D = OR_j (A_j ^ B_j)        (j over the union of both vectors' planes, an absent plane empty)
// plus a size range and a NULL term computed from the column index (include/bmb200.h states the two closed forms).
//   * one work item per block column; thread t owns words [4t, 4t + 4) of the column as one uint4;
//   * plane pairs are taken kMmBatch at a time: the bit-plane loads of a batch (two per pair) are issued together through
//     128-bit streaming loads; the GAP blocks of a pair are XOR-ed into one zeroed 8 KB shared buffer (run scatter with
//     red.shared.xor, so A ^ B of two GAP blocks needs no second buffer);
//   * pairs that cannot differ load nothing: both NULL, both FULL, or the same descriptor (the same stored block); a NULL /
//     FULL pair differs everywhere and saturates D, after which the column's remaining planes are not read;
//   * vector mode ends in finish_block (popcount, digest, run count, kind, bit->GAP) like every other result;
//   * FIRST mode stores no block: the CTA's lowest set bit of F is atomicMin-ed into one device u64.  Columns are claimed in
//     ascending order, so a CTA whose claimed column starts at or after the best position found so far stops: every column
//     it could still claim starts later.
#pragma once
#include "column_walk.cuh"

namespace bmb200 {

struct MismatchParams {
    AggParams out;                // set view + result buffers + work counter (one group of n_cols columns; unused by FIRST)
    uint32_t  plane0_a, n_planes_a, plane0_b, n_planes_b;
    uint32_t  not_null_a, not_null_b;   // 0xffffffff = not nullable
    uint64_t  size_a, size_b;
    uint32_t  use_null;           // BMB200_MM_USE_NULL
    unsigned long long* first;    // FIRST: lowest mismatch position found so far, ~0 = none
};

constexpr int kMmBatch = 4;       // plane pairs whose loads are issued together (one shared expansion buffer each)

// this thread's 128 bits [b0, b0 + 128) of the bit range [lo, hi)
__device__ __forceinline__ uint4 range4(uint64_t b0, uint64_t lo, uint64_t hi)
{
    uint32_t w[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const uint64_t ws = b0 + 32u * q, s = max(lo, ws), e = min(hi, ws + 32u);
        w[q] = s < e ? bit_range_mask((uint32_t)(s - ws), (uint32_t)(e - 1u - ws)) : 0u;
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

__device__ __forceinline__ uint4 xor4(const uint4& a, const uint4& b) { return make_uint4(a.x ^ b.x, a.y ^ b.y, a.z ^ b.z, a.w ^ b.w); }
__device__ __forceinline__ uint4 or4(const uint4& a, const uint4& b)  { return make_uint4(a.x | b.x, a.y | b.y, a.z | b.z, a.w | b.w); }
__device__ __forceinline__ uint4 and4(const uint4& a, const uint4& b) { return make_uint4(a.x & b.x, a.y & b.y, a.z & b.z, a.w & b.w); }
__device__ __forceinline__ uint4 andn4(const uint4& a, const uint4& b) { return make_uint4(a.x & ~b.x, a.y & ~b.y, a.z & ~b.z, a.w & ~b.w); }

template <bool FIRST>
__global__ void __launch_bounds__(kAggThreads, kCtasPerSm) mismatch_kernel(const MismatchParams mp)
{
    __shared__ __align__(16) uint32_t K[kMmBatch][kBlockWords];    // expansion buffers: the GAP blocks of pair u go to K[u]
    __shared__ uint32_t s_da[64], s_db[64], s_nn[2];                // descriptors of this column: planes of A, of B, NOT-NULL
    __shared__ uint32_t s_col, s_min;
    __shared__ uint32_t s_pc[kAggWarps], s_tr[kAggWarps], s_dg[kAggWarps];

    const AggParams& p = mp.out;
    const int tid = threadIdx.x;
    const uint32_t M = p.set.n_vec, np = max(mp.n_planes_a, mp.n_planes_b);
    const uint32_t Ks = smem_u32(K[0]);
    const bool ha = mp.not_null_a != 0xffffffffu, hb = mp.not_null_b != 0xffffffffu;
    const bool use_nn = FIRST ? mp.use_null != 0u : (ha || hb);    // FIRST with no_null compares the planes only
    const uint4 kZero = make_uint4(0u, 0u, 0u, 0u), kOnes = make_uint4(~0u, ~0u, ~0u, ~0u);

    // FIRST: a column that starts at or after the best position found so far ends the claims
    auto past_first = [&](uint32_t c) {
        return FIRST && c < p.n_cols && ((uint64_t)(p.nb_from + c) << 16) >= *(volatile unsigned long long*)mp.first;
    };
    WorkClaim claim(p.work_counter);
    for (;;) {
        const uint32_t colx = claim.next(p.work_counter, s_col, p.n_cols, past_first);
        if (colx >= p.n_cols) break;
        if (FIRST && tid == 0) s_min = 0xffffffffu;          // read after the barrier below
        const uint32_t nb = p.nb_from + colx;
        const uint32_t* drow = p.set.desc + (size_t)nb * M;
        if (tid < 64) s_da[tid] = (uint32_t)tid < mp.n_planes_a ? drow[mp.plane0_a + tid] : BMB200_BLK_NULL;
        else if (tid < 128) s_db[tid - 64] = (uint32_t)(tid - 64) < mp.n_planes_b ? drow[mp.plane0_b + tid - 64] : BMB200_BLK_NULL;
        else if (tid == 128) s_nn[0] = (use_nn && ha) ? drow[mp.not_null_a] : BMB200_BLK_NULL;
        else if (tid == 129) s_nn[1] = (use_nn && hb) ? drow[mp.not_null_b] : BMB200_BLK_NULL;
        const uint4* bseg = reinterpret_cast<const uint4*>(p.set.bit_pool) + p.set.bit_base[nb] * (size_t)(kBlockWords / 4) + tid;
        const uint16_t* gseg = p.set.gap_pool + p.set.gap_base[nb] * (size_t)kGapUnit;
        __syncthreads();

        // XOR the 1-runs of GAP block d into buffer buf, all threads
        auto expand = [&](uint32_t buf, uint32_t d) { if ((d & 3u) == BMB200_BLK_GAP) gap_expand_block(Ks + buf * kBlockWords * 4u, gap_block_ptr(gseg, d), tid); };

        uint4 D = kZero;
        bool sat = false;                                    // uniform: a NULL / FULL pair filled D
        for (uint32_t j0 = 0; j0 < np && !sat; j0 += kMmBatch) {
            uint4 X[kMmBatch];
            uint32_t gmask = 0;                              // pairs with a GAP block (uniform)
#pragma unroll
            for (int u = 0; u < kMmBatch; ++u) {
                const uint32_t j = j0 + u;
                const uint32_t da = j < np ? s_da[j] : BMB200_BLK_NULL, db = j < np ? s_db[j] : BMB200_BLK_NULL;
                const uint32_t ka = da & 3u, kb = db & 3u;
                X[u] = kZero;
                if (da == db || (ka == kb && ka <= BMB200_BLK_FULL)) continue;           // cannot differ
                if (ka <= BMB200_BLK_FULL && kb <= BMB200_BLK_FULL) { sat = true; continue; }   // NULL vs FULL
                X[u] = xor4(block_now(bseg, da), block_now(bseg, db));
                if (ka == BMB200_BLK_GAP || kb == BMB200_BLK_GAP) gmask |= 1u << u;
            }
            if (sat) break;
            if (gmask) {
#pragma unroll
                for (int u = 0; u < kMmBatch; ++u)
                    if ((gmask >> u) & 1u) reinterpret_cast<uint4*>(K[u])[tid] = kZero;
                __syncthreads();
#pragma unroll
                for (int u = 0; u < kMmBatch; ++u)
                    if ((gmask >> u) & 1u) { expand((uint32_t)u, s_da[j0 + u]); expand((uint32_t)u, s_db[j0 + u]); }
                __syncthreads();
#pragma unroll
                for (int u = 0; u < kMmBatch; ++u)
                    if ((gmask >> u) & 1u) X[u] = xor4(X[u], reinterpret_cast<const uint4*>(K[u])[tid]);
                __syncthreads();                             // the buffers are rewritten by the next batch
            }
#pragma unroll
            for (int u = 0; u < kMmBatch; ++u) D = or4(D, X[u]);
        }
        if (sat) D = kOnes;

        // NOT-NULL vectors; NULL descriptors when absent or unused
        uint4 NN[2];
        load_blocks({s_nn[0], s_nn[1]}, NN, bseg, gseg, K);
        const uint4 NA = NN[0], NB = NN[1];
        const uint64_t b0 = ((uint64_t)nb << 16) + 128u * (uint32_t)tid;
        const uint64_t sa = mp.size_a, sb = mp.size_b;
        if constexpr (!FIRST) {
            D = or4(D, range4(b0, min(sa, sb), max(sa, sb)));
            if (mp.use_null) {
                if (ha && hb) D = or4(D, xor4(NA, NB));
                else if (ha)  D = or4(D, andn4(range4(b0, 0u, sa), NA));
                else if (hb)  D = or4(D, andn4(range4(b0, 0u, sb), NB));
            } else {
                if (ha && hb) D = and4(D, or4(NA, NB));
                else if (ha)  D = and4(D, NA);
                else if (hb)  D = and4(D, NB);
            }
            finish_block<true>(p, colx, colx, 0u, D, 2, K[0], s_pc, s_tr, s_dg);
        } else {
            if (mp.use_null) {
                if (ha && hb) D = or4(D, xor4(NA, NB));
                else if (ha)  D = or4(D, xor4(NA, range4(b0, 0u, sb)));
                else if (hb)  D = or4(D, xor4(NB, range4(b0, 0u, sa)));
            }
            // lowest set bit of the column: per thread, then per warp, then one shared atomic per warp
            const uint32_t q = D.x ? 0u : D.y ? 1u : D.z ? 2u : D.w ? 3u : 4u;
            const uint32_t v = q == 0u ? D.x : q == 1u ? D.y : q == 2u ? D.z : D.w;
            const uint32_t off = q < 4u ? 128u * (uint32_t)tid + 32u * q + (uint32_t)(__ffs(v) - 1) : 0xffffffffu;
            const uint32_t wmin = __reduce_min_sync(0xffffffffu, off);
            if ((tid & 31) == 0 && wmin != 0xffffffffu) atomicMin(&s_min, wmin);
            __syncthreads();
            if (tid == 0 && s_min != 0xffffffffu) atomicMin(mp.first, ((unsigned long long)nb << 16) + s_min);
        }
    }
}

}  // namespace bmb200
