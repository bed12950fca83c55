// scan_kernel.cuh -- bit-sliced comparison scan over the planes of a sparse vector (sm_90a).
//
// Replaces the reference's sparse_vector_scanner<SV> searches for unsigned sparse vectors
//   find_eq   src/bmsparsevec_algo.h:4360-4395 (prepare_and_sub_aggregator :2593-2632 + aggregator::combine_and_sub)
//   find_gt / find_ge / find_lt / find_le / find_range   src/bmsparsevec_algo.h:1135-1182 (find_gt_horizontal & co.)
// which the reference builds out of many aggregator / bvector passes over the planes.  Here ONE pass over the
// planes of a block column answers any of them: walking the planes from the most significant bit down, every thread
// keeps, for its 128 bits of the column,
//     EQ = elements equal to the search value on all planes seen so far      (starts as the index universe U)
//     GT = elements already known to be greater
//   plane bit of the value == 1 :  EQ &= P                      (elements with a 0 here are smaller: they leave EQ)
//   plane bit of the value == 0 :  GT |= EQ & P ;  EQ &= ~P
// and the predicates fall out at the end:  eq = EQ, gt = GT, ge = GT | EQ, lt = U & ~(GT | EQ), le = U & ~GT,
// range [a, b] = ge(a) & le(b) (two state pairs in the same pass).  Every plane block is read exactly once per
// (column, value) work item; the values of one column are adjacent work items so the planes come from L2 after the
// first one (the same batching as aggregator::pipeline, agg_kernel.cuh).
//
// Up to 4 search values of a column share one pass (their states sit side by side in registers), so the plane loads and the
// GAP expansions are paid once per group of values.
// Plane blocks may be NULL / FULL / bit / GAP like any other block of the set; GAP planes are expanded through the
// 8 KB shared mask (block-wide run scatter), bit planes stream through 128-bit loads, four planes in flight.
// The result goes through the same epilogue as the aggregation kernel (popcount, digest, run count, kind, bit->GAP).
#pragma once
#include "gap_expand.cuh"

namespace bmb200 {

struct ScanParams {
    AggParams out;             // set view + result buffers + work counter (group / goff unused; n_groups = n_values)
    uint32_t  plane0;          // plane j (bit j of the value) = set vector plane0 + j
    uint32_t  n_planes;        // <= 64
    uint32_t  universe;        // set vector holding the searchable index range (size mask / NOT-NULL plane); 0xffffffff = everything
    uint32_t  pred;            // BMB200_SCAN_*
    const uint64_t* values;    // device: n_values entries (RANGE: 2 * n_values, lo then hi of each range)
};

constexpr int kScanBatch = 4;  // planes whose loads are issued together

__device__ __forceinline__ void scan_step(uint4& eq, uint4& gt, const uint4& P, bool vbit)
{
    if (vbit) { eq.x &= P.x; eq.y &= P.y; eq.z &= P.z; eq.w &= P.w; }
    else {
        gt.x |= eq.x & P.x; gt.y |= eq.y & P.y; gt.z |= eq.z & P.z; gt.w |= eq.w & P.w;
        eq.x &= ~P.x; eq.y &= ~P.y; eq.z &= ~P.z; eq.w &= ~P.w;
    }
}

// VG search values share one pass over the planes of a column (their states live side by side in registers), so plane loads
// and GAP expansions are paid once per VG searches; RANGE keeps two state pairs per value and therefore groups fewer values.
// MODE 0: find_eq only (no GT state), 1: one (EQ, GT) pair per value, 2: RANGE (two pairs per value)
template <int VG, int MODE>
__global__ void __launch_bounds__(kAggThreads, kCtasPerSm) scan_kernel(const ScanParams sp)
{
    constexpr bool RANGE = (MODE == 2), EQ_ONLY = (MODE == 0);
    constexpr int kStateRegs = VG * (EQ_ONLY ? 4 : RANGE ? 16 : 8);
    constexpr int kBatch = kStateRegs > 16 ? 2 : kScanBatch;                // planes in flight: bounded by the register budget
    __shared__ __align__(16) uint32_t K[kScanBatch][kBlockWords];   // expansion buffers: the GAP planes of one batch are expanded together
    __shared__ uint32_t s_desc[65];                          // descriptors of the planes (+ universe) of this column
    __shared__ uint32_t s_col;
    __shared__ uint64_t s_va[VG], s_vb[VG];                  // the group's search values (kept out of the register file)
    __shared__ uint32_t s_pc[kAggWarps], s_tr[kAggWarps], s_dg[kAggWarps];

    const AggParams& p = sp.out;
    const int tid = threadIdx.x;
    const uint32_t M = p.set.n_vec;
    uint4* K4 = reinterpret_cast<uint4*>(K[0]);
    const uint32_t Ks = smem_u32(K[0]);
    const uint32_t n_vg = (p.n_groups + VG - 1) / VG;        // value groups per column

    uint32_t next_item = 0;
    if (tid == 0) next_item = atomicAdd(p.work_counter, 1u);
    for (;;) {
        __syncthreads();
        if (tid == 0) s_col = next_item;
        __syncthreads();
        const uint32_t item = s_col;
        if (item >= p.n_cols * n_vg) break;
        if (tid == 0) next_item = atomicAdd(p.work_counter, 1u);
        const uint32_t colx = item / n_vg, v0 = (item - colx * n_vg) * VG;
        const uint32_t nb = p.nb_from + colx;
        const uint32_t* drow = p.set.desc + (size_t)nb * M;
        if (tid < (int)sp.n_planes) s_desc[tid] = drow[sp.plane0 + tid];
        if (tid == 64) s_desc[64] = (sp.universe == 0xffffffffu) ? BMB200_BLK_FULL : drow[sp.universe];
        const uint4* bseg = reinterpret_cast<const uint4*>(p.set.bit_pool) + p.set.bit_base[nb] * (size_t)(kBlockWords / 4) + tid;
        const uint16_t* gseg = p.set.gap_pool + p.set.gap_base[nb] * (size_t)kGapUnit;
        if (tid < VG) {
            const uint32_t vi = min(v0 + (uint32_t)tid, p.n_groups - 1u);         // a short last group repeats its last value
            uint64_t a = sp.values[RANGE ? 2u * vi : vi], b = RANGE ? sp.values[2u * vi + 1u] : 0ull;
            if (RANGE && b < a) { const uint64_t t = a; a = b; b = t; }           // find_range swaps reversed bounds, :2871-2872
            s_va[tid] = a; s_vb[tid] = b;
        }
        __syncthreads();

        // one block of the column as this thread's 4 words: GAP blocks go through the shared mask (2 block barriers)
        auto load_gap = [&](uint32_t d) -> uint4 {
            K4[tid] = make_uint4(0u, 0u, 0u, 0u);
            __syncthreads();
            const uint32_t rel = d >> 2;
            gap_expand_block(Ks, gseg + (size_t)(rel & kRelMask) * kGapUnit + (rel >> 29), tid);
            __syncthreads();
            const uint4 r = K4[tid];
            __syncthreads();
            return r;
        };
        auto load_now = [&](uint32_t d) -> uint4 {           // NULL / FULL / bit (GAP handled by the caller)
            const uint32_t kind = d & 3u;
            if (kind == BMB200_BLK_BIT) return ld_stream_v4(bseg + (size_t)(d >> 2) * (kBlockWords / 4));
            return kind == BMB200_BLK_FULL ? make_uint4(~0u, ~0u, ~0u, ~0u) : make_uint4(0u, 0u, 0u, 0u);
        };

        const uint32_t du = s_desc[64];
        const uint4 U = ((du & 3u) == BMB200_BLK_GAP) ? load_gap(du) : load_now(du);
        uint4 eqA[VG], gtA[EQ_ONLY ? 1 : VG], eqB[RANGE ? VG : 1], gtB[RANGE ? VG : 1];
#pragma unroll
        for (int g = 0; g < VG; ++g) {
            eqA[g] = U; if (!EQ_ONLY) gtA[g] = make_uint4(0u, 0u, 0u, 0u);
            // a value with bits above the top plane is greater than every element: it starts with an empty EQ state (and its low
            // bits then only feed GT |= EQ & P = 0, so they need no masking)
            if (sp.n_planes < 64u && (s_va[g] >> sp.n_planes)) eqA[g] = make_uint4(0u, 0u, 0u, 0u);
            if (RANGE) {
                eqB[g] = U; gtB[g] = make_uint4(0u, 0u, 0u, 0u);
                if (sp.n_planes < 64u && (s_vb[g] >> sp.n_planes)) eqB[g] = make_uint4(0u, 0u, 0u, 0u);
            }
        }

        for (int jt = (int)sp.n_planes - 1; jt >= 0; jt -= kBatch) {
            uint4 P[kBatch];
            uint32_t d[kBatch];
            bool any_gap = false;
#pragma unroll
            for (int u = 0; u < kBatch; ++u) {               // issue the bit-plane loads of the batch together
                const int j = jt - u;
                d[u] = (j >= 0) ? s_desc[j] : BMB200_BLK_NULL;
                if ((d[u] & 3u) != BMB200_BLK_GAP) P[u] = load_now(d[u]); else any_gap = true;
            }
            if (any_gap) {                                   // uniform: the GAP planes of the batch share one pair of barriers
#pragma unroll
                for (int u = 0; u < kBatch; ++u)
                    if ((d[u] & 3u) == BMB200_BLK_GAP) reinterpret_cast<uint4*>(K[u])[tid] = make_uint4(0u, 0u, 0u, 0u);
                __syncthreads();
#pragma unroll
                for (int u = 0; u < kBatch; ++u)
                    if ((d[u] & 3u) == BMB200_BLK_GAP) {
                        const uint32_t rel = d[u] >> 2;
                        gap_expand_block(Ks + (uint32_t)u * kBlockWords * 4u, gseg + (size_t)(rel & kRelMask) * kGapUnit + (rel >> 29), tid);
                    }
                __syncthreads();
#pragma unroll
                for (int u = 0; u < kBatch; ++u)
                    if ((d[u] & 3u) == BMB200_BLK_GAP) P[u] = reinterpret_cast<const uint4*>(K[u])[tid];
                __syncthreads();                             // the buffers are rewritten by the next batch
            }
#pragma unroll
            for (int u = 0; u < kBatch; ++u) {
                const int j = jt - u;
                if (j < 0) break;
#pragma unroll
                for (int g = 0; g < VG; ++g) {
                    if (EQ_ONLY) {
                        const uint32_t f = ((s_va[g] >> j) & 1ull) ? 0u : 0xffffffffu;       // EQ &= value bit ? P : ~P
                        eqA[g].x &= P[u].x ^ f; eqA[g].y &= P[u].y ^ f; eqA[g].z &= P[u].z ^ f; eqA[g].w &= P[u].w ^ f;
                    } else scan_step(eqA[g], gtA[g], P[u], (s_va[g] >> j) & 1ull);
                    if (RANGE) scan_step(eqB[g], gtB[g], P[u], (s_vb[g] >> j) & 1ull);
                }
            }
        }

#pragma unroll
        for (int g = 0; g < VG; ++g) {
            const uint32_t vi = v0 + (uint32_t)g;
            if (vi >= p.n_groups) break;                     // uniform
            const uint4 e = eqA[g], t = gtA[EQ_ONLY ? 0 : g];
            uint4 R;
            switch (sp.pred) {
            case BMB200_SCAN_EQ: R = e; break;
            case BMB200_SCAN_GT: R = t; break;
            case BMB200_SCAN_GE: R = make_uint4(t.x | e.x, t.y | e.y, t.z | e.z, t.w | e.w); break;
            case BMB200_SCAN_LT: R = make_uint4(U.x & ~(t.x | e.x), U.y & ~(t.y | e.y), U.z & ~(t.z | e.z), U.w & ~(t.w | e.w)); break;
            case BMB200_SCAN_LE: R = make_uint4(U.x & ~t.x, U.y & ~t.y, U.z & ~t.z, U.w & ~t.w); break;
            default: {           // RANGE: ge(a) & le(b)
                const uint4 tb = gtB[RANGE ? g : 0];
                R = make_uint4((t.x | e.x) & U.x & ~tb.x, (t.y | e.y) & U.y & ~tb.y, (t.z | e.z) & U.z & ~tb.z, (t.w | e.w) & U.w & ~tb.w);
                break; }
            }
            if (g) __syncthreads();                          // the epilogue scratch (K[0]) of the previous value is still being read
            finish_block<true>(p, vi * p.n_cols + colx, colx, vi, R, 2, K[0], s_pc, s_tr, s_dg);
        }
    }
}

}  // namespace bmb200
