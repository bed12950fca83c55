// scan_kernel.cuh -- bit-sliced comparison scan over the planes of a sparse vector (sm_90a).
//
// Replaces the reference's sparse_vector_scanner<SV> searches for unsigned, signed and float sparse vectors
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
//
// Signed vectors (ENC = kEncS2u; bm::sparse_vector<int32_t / int64_t>, src/bmbmatrix.h:2536-2569) store u = s2u(x):
// x >= 0 -> x << 1, x < 0 -> (-(x+1)) << 1 | 1, so plane 0 is the sign plane S and planes 1..n-1 hold the magnitude m
// (a negative element is -(m+1)).  The reference answers a signed inequality with several whole-vector passes
// (find_gt_horizontal_s, src/bmsparsevec_algo.h:3032-3219); here it is the same single pass:
//   * the search value is staged as s2u(v): bits 1.. are the magnitude vm (v >= 0 ? v : ~v), bit 0 its sign;
//   * the walk runs over planes n-1..1 only, giving EQm / GTm, the magnitude comparison against vm (a value with
//     magnitude bits above the top plane starts with an empty EQ state, exactly as in the unsigned walk);
//   * plane 0 is loaded once after the walk and combined per value:
//         v >= 0:  EQ = EQm & ~S    GT = GTm & ~S
//         v <  0:  EQ = EQm &  S    GT = U & ~(S & (EQm | GTm))     (non-negatives, and negatives of smaller magnitude)
//     after which ge / lt / le / range follow from (EQ, GT) as for unsigned vectors.
// find_eq (MODE 0) needs no sign combination: it walks all n planes against s2u(v), which is the exact equality of the
// stored codes and keeps the EQ-only kernel's register footprint (no S, no per-value sign).  RANGE swaps reversed bounds by
// signed order when the values are staged.
//
// Float vectors (ENC = kEncFloat; bm::sparse_vector_float<sparse_vector<unsigned>>, src/bmsparsevec_float.h) keep a float's
// sign bit in signs_, its 8 exponent bits in exponents_ and its 23 mantissa bits in mantissas_.  Every float search of the
// reference (find_gt_float & co., src/bmsparsevec_algo.h:3692-4009, 4-6 whole-vector passes each) is a comparison in the
// IEEE sign-magnitude total order of the raw bits b: key(b) = sign ? ~b : b | 0x80000000 (-0 < +0, a positive NaN above +inf,
// a negative NaN below -inf, payloads ordered by their bits).  That is the signed walk above, unchanged:
//   * the planes are [signs_, mantissa 0..22, exponent 0..7], so plane 1 + k is bit k of the magnitude b & 0x7fffffff;
//   * the search value is staged as ((b & 0x7fffffff) << 1) | (b >> 31): magnitude in bits 1.., sign in bit 0 -- the same
//     shape as s2u, and signed_combine gives exactly the key() order (negatives by falling magnitude, -0 below +0);
//   * RANGE and RANGE_OPEN swap their bounds when a > b as IEEE floats (find_range_float :3819, :3846: a NaN bound never
//     swaps, +0 / -0 compare equal), decided with integer logic on the bits so no flush-to-zero mode can change it;
//   * RANGE_OPEN (find_range_float_unbounded) is gt(a) & lt(b) = GT_a & U & ~(GT_b | EQ_b), two state pairs like RANGE.
// The float path has no find_eq (the reference has none) and so only the MODE 1 / 2 instantiations.
#pragma once
#include "column_walk.cuh"

namespace bmb200 {

struct ScanParams {
    AggParams out;             // set view + result buffers + work counter (group / goff unused; n_groups = n_values)
    uint32_t  plane0;          // plane j (bit j of the value) = set vector plane0 + j
    uint32_t  n_planes;        // <= 64 (float: <= 32)
    uint32_t  universe;        // set vector holding the searchable index range (size mask / NOT-NULL plane); 0xffffffff = everything
    uint32_t  pred;            // BMB200_SCAN_*
    const uint64_t* values;    // device: n_values entries (RANGE / RANGE_OPEN: 2 * n_values, lo then hi of each range)
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

// s2u (src/bmbmatrix.h:2536-2569) of a two's-complement int64 search value
__device__ __forceinline__ uint64_t s2u(uint64_t v)
{
    return (int64_t)v >= 0 ? v << 1 : ((~v) << 1) | 1ull;
}

// a float's 32 bits staged for the signed walk: magnitude (b & 0x7fffffff) in bits 1..31, sign in bit 0
__device__ __forceinline__ uint64_t f2u(uint64_t b)
{
    return ((b & 0x7fffffffull) << 1) | ((b >> 31) & 1ull);
}

// a > b for the IEEE floats with bits a, b (the C++ comparison find_range_float swaps on), in integer logic: false when either
// is a NaN or both are zeros, else the key() order of the bits
__device__ __forceinline__ bool float_gt(uint32_t a, uint32_t b)
{
    if ((a & 0x7fffffffu) > 0x7f800000u || (b & 0x7fffffffu) > 0x7f800000u || !((a | b) & 0x7fffffffu)) return false;
    const uint32_t ka = (a >> 31) ? ~a : a | 0x80000000u, kb = (b >> 31) ? ~b : b | 0x80000000u;
    return ka > kb;
}

// (EQm, GTm) of the magnitude walk -> (EQ, GT) of the signed comparison, S = sign plane, neg = the value is negative
__device__ __forceinline__ void signed_combine(uint4& e, uint4& t, const uint4& U, const uint4& S, bool neg)
{
    if (neg) {
        t = make_uint4(U.x & ~(S.x & (e.x | t.x)), U.y & ~(S.y & (e.y | t.y)), U.z & ~(S.z & (e.z | t.z)), U.w & ~(S.w & (e.w | t.w)));
        e = make_uint4(e.x & S.x, e.y & S.y, e.z & S.z, e.w & S.w);
    } else {
        t = make_uint4(t.x & ~S.x, t.y & ~S.y, t.z & ~S.z, t.w & ~S.w);
        e = make_uint4(e.x & ~S.x, e.y & ~S.y, e.z & ~S.z, e.w & ~S.w);
    }
}

// VG search values share one pass over the planes of a column (their states live side by side in registers), so plane loads
// and GAP expansions are paid once per VG searches; RANGE keeps two state pairs per value and therefore groups fewer values.
// MODE 0: find_eq only (no GT state), 1: one (EQ, GT) pair per value, 2: RANGE (two pairs per value)
// ENC: how elements and search values are encoded (see the file comment)
enum ScanEnc { kEncUnsigned = 0, kEncS2u = 1, kEncFloat = 2 };
template <int VG, int MODE, int ENC = kEncUnsigned>
__global__ void __launch_bounds__(kAggThreads, kCtasPerSm) scan_kernel(const ScanParams sp)
{
    constexpr bool RANGE = (MODE == 2), EQ_ONLY = (MODE == 0);
    constexpr bool SIGNED = (ENC != kEncUnsigned);                          // s2u and float elements take the signed walk
    constexpr int kLowPlane = (SIGNED && !EQ_ONLY) ? 1 : 0;                  // the signed inequalities leave the sign plane out of the walk
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
            if constexpr (ENC == kEncFloat) {
                if (RANGE && float_gt((uint32_t)a, (uint32_t)b)) { const uint64_t t = a; a = b; b = t; }   // IEEE order, :3819,3846
                a = f2u(a); b = f2u(b);
            } else if constexpr (SIGNED) {
                if (RANGE && (int64_t)b < (int64_t)a) { const uint64_t t = a; a = b; b = t; }   // signed order, :2871-2872
                a = s2u(a); b = s2u(b);
            } else if (RANGE && b < a) { const uint64_t t = a; a = b; b = t; }    // find_range swaps reversed bounds, :2871-2872
            s_va[tid] = a; s_vb[tid] = b;
        }
        __syncthreads();

        // one block of the column as this thread's 4 words: GAP blocks go through the shared mask (2 block barriers)
        auto load_gap = [&](uint32_t d) -> uint4 {
            K4[tid] = make_uint4(0u, 0u, 0u, 0u);
            __syncthreads();
            gap_expand_block(Ks, gap_block_ptr(gseg, d), tid);
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

        for (int jt = (int)sp.n_planes - 1; jt >= kLowPlane; jt -= kBatch) {
            uint4 P[kBatch];
            uint32_t d[kBatch];
            bool any_gap = false;
#pragma unroll
            for (int u = 0; u < kBatch; ++u) {               // issue the bit-plane loads of the batch together
                const int j = jt - u;
                d[u] = (j >= kLowPlane) ? s_desc[j] : BMB200_BLK_NULL;
                if ((d[u] & 3u) != BMB200_BLK_GAP) P[u] = load_now(d[u]); else any_gap = true;
            }
            if (any_gap) {                                   // uniform: the GAP planes of the batch share one pair of barriers
#pragma unroll
                for (int u = 0; u < kBatch; ++u)
                    if ((d[u] & 3u) == BMB200_BLK_GAP) reinterpret_cast<uint4*>(K[u])[tid] = make_uint4(0u, 0u, 0u, 0u);
                __syncthreads();
#pragma unroll
                for (int u = 0; u < kBatch; ++u)
                    if ((d[u] & 3u) == BMB200_BLK_GAP) gap_expand_block(Ks + (uint32_t)u * kBlockWords * 4u, gap_block_ptr(gseg, d[u]), tid);
                __syncthreads();
#pragma unroll
                for (int u = 0; u < kBatch; ++u)
                    if ((d[u] & 3u) == BMB200_BLK_GAP) P[u] = reinterpret_cast<const uint4*>(K[u])[tid];
                __syncthreads();                             // the buffers are rewritten by the next batch
            }
#pragma unroll
            for (int u = 0; u < kBatch; ++u) {
                const int j = jt - u;
                if (j < kLowPlane) break;
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

        if constexpr (kLowPlane == 1) {                      // the sign plane, folded into the states before the epilogue
            const uint32_t ds = s_desc[0];
            const uint4 S = ((ds & 3u) == BMB200_BLK_GAP) ? load_gap(ds) : load_now(ds);
#pragma unroll
            for (int g = 0; g < VG; ++g) {
                signed_combine(eqA[g], gtA[g], U, S, s_va[g] & 1ull);
                if (RANGE) signed_combine(eqB[RANGE ? g : 0], gtB[RANGE ? g : 0], U, S, s_vb[g] & 1ull);
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
            default: {           // RANGE: ge(a) & le(b); RANGE_OPEN (float only): gt(a) & lt(b)
                const uint4 tb = gtB[RANGE ? g : 0];
                if (ENC == kEncFloat && sp.pred == BMB200_SCAN_RANGE_OPEN) {
                    const uint4 eb = eqB[RANGE ? g : 0];
                    R = make_uint4(t.x & U.x & ~(tb.x | eb.x), t.y & U.y & ~(tb.y | eb.y), t.z & U.z & ~(tb.z | eb.z), t.w & U.w & ~(tb.w | eb.w));
                } else
                    R = make_uint4((t.x | e.x) & U.x & ~tb.x, (t.y | e.y) & U.y & ~tb.y, (t.z | e.z) & U.z & ~tb.z, (t.w | e.w) & U.w & ~tb.w);
                break; }
            }
            if (g) __syncthreads();                          // the epilogue scratch (K[0]) of the previous value is still being read
            finish_block<true>(p, vi * p.n_cols + colx, colx, vi, R, 2, K[0], s_pc, s_tr, s_dg);
        }
    }
}

}  // namespace bmb200
