// str_scan_kernel.cuh -- bit-sliced string equality over the planes of a string sparse vector (sm_90a).
//
// Replaces the reference's sparse_vector_scanner<str_sparse_vector<char, ...>> string searches
//   find_eq_str / find_eq_str_prefix   src/bmsparsevec_algo.h:3263-3268,3372-3419 (prepare_and_sub_aggregator :2546-2588,
//                                      add_agg_char :1817-1850 + aggregator::combine_and_sub)
//   find_eq_str(TPipe&)                :3424-3436,4579-4651 (one AND-SUB group per string)
// which the reference answers with one aggregator AND-SUB pass per query over 8 planes per character plus every tail plane.
// Plane 8k+b holds bit b of byte k of every element (basic_bmatrix::set_octet, src/bmbmatrix.h:1571-1605); NULL elements and
// positions >= size() have all planes zero.  Every thread keeps, for its 128 bits of the column, one state per query
//     EQ = elements whose planes match the query on every plane walked so far     (starts as the universe U)
//     EQ &= P ^ (query bit ? 0 : ~0)
// walking the planes from the highest one the group needs down to 0, the reference's reverse-octet order (:2557-2559), so a
// column's tail planes come first.  An exact search walks every plane (the zero-padded query must match the tail planes too,
// the SUB group of :2577-2586); a prefix search only the planes of its own bytes, j < 8 * strlen (planes above are "don't
// care" for that query).  A query with a 1-bit at a plane >= n_planes matches nothing (the get_slice_mask pre-screen,
// :2569-2570): the host stages it as dead and its state starts empty.
//
// Early exit: before the walk and at every octet boundary the CTA takes __syncthreads_or over "any state word of the group is
// non-zero"; when nothing is left the whole CTA leaves the walk (the decision is the barrier's result, so it is uniform and
// the block barriers of the GAP expansion stay matched) and writes the empty column.  A column whose universe block is NULL
// reads no plane at all.
//
// Up to 4 queries of a column share one pass (VG), plane loads are batched four at a time, GAP planes are expanded through the
// shared buffers (one pair of barriers per batch), and the result goes through finish_block like every other result.
#pragma once
#include "column_walk.cuh"

namespace bmb200 {

constexpr uint32_t kStrMaxPlanes = 2048;        // strings of up to 256 bytes
constexpr uint32_t kStrDead = 0x80000000u;      // limit word of a query that cannot match (a 1-bit above the top plane)
constexpr int kStrBatch = 4;                    // planes whose loads are issued together (a batch never straddles an octet)

struct StrScanParams {
    AggParams out;             // set view + result buffers + work counter (n_groups = n_values)
    uint32_t  plane0;          // plane 8k+b (bit b of byte k) = set vector plane0 + 8k + b
    uint32_t  n_planes;        // <= kStrMaxPlanes
    uint32_t  universe;        // set vector with the searchable indexes; 0xffffffff = everything
    uint32_t  vwords;          // staged words per query: its limit word, then ceil(n_planes / 32) words of plane bits
    const uint32_t* strs;      // device: n_values * vwords; limit = planes compared (j < limit) | kStrDead
};

template <int VG>
__global__ void __launch_bounds__(kAggThreads, kCtasPerSm) str_scan_kernel(const StrScanParams sp)
{
    __shared__ __align__(16) uint32_t K[kStrBatch][kBlockWords];   // expansion buffers of one batch's GAP planes
    __shared__ uint32_t s_str[VG][kStrMaxPlanes / 32];             // the group's queries as plane bits (NUL-padded bytes)
    __shared__ uint32_t s_lim[VG];
    __shared__ uint32_t s_col;
    __shared__ uint64_t s_seg[2];                                  // bit_base / gap_base of the column
    __shared__ uint32_t s_pc[kAggWarps], s_tr[kAggWarps], s_dg[kAggWarps];

    const AggParams& p = sp.out;
    const int tid = threadIdx.x;
    const uint32_t M = p.set.n_vec;
    const uint32_t Ks = smem_u32(K[0]);
    const uint32_t n_vg = (p.n_groups + VG - 1) / VG;

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
        for (uint32_t k = tid; k < VG * sp.vwords; k += kAggThreads) {
            const uint32_t g = k / sp.vwords, w = k - g * sp.vwords;
            const uint32_t vi = min(v0 + g, p.n_groups - 1u);            // a short last group repeats its last query
            const uint32_t x = sp.strs[(size_t)vi * sp.vwords + w];
            if (w == 0) s_lim[g] = x; else s_str[g][w - 1] = x;
        }
        if (tid == 0) { s_seg[0] = p.set.bit_base[nb]; s_seg[1] = p.set.gap_base[nb]; }
        __syncthreads();
        // the column's segments are re-read from shared memory where they are used: the walk's registers go to the states
        auto bseg = [&]() { return reinterpret_cast<const uint4*>(p.set.bit_pool) + s_seg[0] * (size_t)(kBlockWords / 4) + tid; };
        auto gseg = [&]() { return p.set.gap_pool + s_seg[1] * (size_t)kGapUnit; };
        auto desc = [&](uint32_t v) { return p.set.desc[(size_t)nb * M + v]; };

        auto load_now = [&](uint32_t d) -> uint4 {           // NULL / FULL / bit (GAP handled by the caller)
            const uint32_t kind = d & 3u;
            if (kind == BMB200_BLK_BIT) return ld_stream_v4(bseg() + (size_t)(d >> 2) * (kBlockWords / 4));
            return kind == BMB200_BLK_FULL ? make_uint4(~0u, ~0u, ~0u, ~0u) : make_uint4(0u, 0u, 0u, 0u);
        };
        // the plane batch [jb, jb + kStrBatch) of the column, planes >= top read as NULL; GAP planes share one pair of barriers
        auto load_batch = [&](int jb, int top, uint4 (&P)[kStrBatch]) {
            uint32_t d[kStrBatch];
            bool any_gap = false;
#pragma unroll
            for (int u = 0; u < kStrBatch; ++u) {
                d[u] = (jb + u < top) ? desc(sp.plane0 + jb + u) : BMB200_BLK_NULL;
                if ((d[u] & 3u) != BMB200_BLK_GAP) P[u] = load_now(d[u]); else any_gap = true;
            }
            if (any_gap) {                                   // uniform
#pragma unroll
                for (int u = 0; u < kStrBatch; ++u)
                    if ((d[u] & 3u) == BMB200_BLK_GAP) reinterpret_cast<uint4*>(K[u])[tid] = make_uint4(0u, 0u, 0u, 0u);
                __syncthreads();
#pragma unroll
                for (int u = 0; u < kStrBatch; ++u)
                    if ((d[u] & 3u) == BMB200_BLK_GAP) gap_expand_block(Ks + (uint32_t)u * kBlockWords * 4u, gap_block_ptr(gseg(), d[u]), tid);
                __syncthreads();
#pragma unroll
                for (int u = 0; u < kStrBatch; ++u)
                    if ((d[u] & 3u) == BMB200_BLK_GAP) P[u] = reinterpret_cast<const uint4*>(K[u])[tid];
                __syncthreads();                             // the buffers are rewritten by the next batch
            }
        };

        uint4 U;
        {
            const uint32_t du = (sp.universe == 0xffffffffu) ? BMB200_BLK_FULL : desc(sp.universe);
            if ((du & 3u) == BMB200_BLK_GAP) {
                reinterpret_cast<uint4*>(K[0])[tid] = make_uint4(0u, 0u, 0u, 0u);
                __syncthreads();
                gap_expand_block(Ks, gap_block_ptr(gseg(), du), tid);
                __syncthreads();
                U = reinterpret_cast<const uint4*>(K[0])[tid];
                __syncthreads();
            } else U = load_now(du);
        }
        uint4 eq[VG];
        int top = 0;
        bool live = false;
#pragma unroll
        for (int g = 0; g < VG; ++g) {
            const uint32_t lim = s_lim[g];
            eq[g] = (lim & kStrDead) ? make_uint4(0u, 0u, 0u, 0u) : U;
            if (!(lim & kStrDead)) top = max(top, (int)lim);
            live |= (eq[g].x | eq[g].y | eq[g].z | eq[g].w) != 0u;
        }

        if (__syncthreads_or(live)) {
            for (int jb = (top - 1) & ~(kStrBatch - 1); jb >= 0; jb -= kStrBatch) {
                uint4 P[kStrBatch];
                load_batch(jb, top, P);
                live = false;
#pragma unroll
                for (int g = 0; g < VG; ++g) {
                    const uint32_t bits = s_str[g][jb >> 5] >> (jb & 31);   // a batch lies inside one word of plane bits
                    const uint32_t lim = s_lim[g];
#pragma unroll
                    for (int u = 0; u < kStrBatch; ++u) {
                        if ((uint32_t)(jb + u) >= lim) continue;               // don't care (prefix) / above the group's top
                        const uint32_t f = ((bits >> u) & 1u) ? 0u : 0xffffffffu;   // EQ &= query bit ? P : ~P
                        eq[g].x &= P[u].x ^ f; eq[g].y &= P[u].y ^ f; eq[g].z &= P[u].z ^ f; eq[g].w &= P[u].w ^ f;
                    }
                    live |= (eq[g].x | eq[g].y | eq[g].z | eq[g].w) != 0u;
                }
                // octet boundary: leave the walk when no element of the column still matches any query of the group
                if ((jb & 7) == 0 && jb > 0 && !__syncthreads_or(live)) break;
            }
        }

        // the other queries' states wait in the expansion buffers K[1..VG-1] (the epilogue's scratch is K[0]), so the epilogue
        // runs with one state in registers
        constexpr int kSlot0 = VG < kStrBatch ? VG : 0;   // where query 0 waits (0: it stays in registers)
#pragma unroll
        for (int g = 0; g < VG; ++g) if (g || kSlot0) reinterpret_cast<uint4*>(K[g ? g : kSlot0])[tid] = eq[g];
#pragma unroll 1
        for (int g = 0; g < VG; ++g) {
            const uint32_t vi = v0 + (uint32_t)g;
            if (vi >= p.n_groups) break;                     // uniform
            if (g) __syncthreads();                          // the epilogue scratch (K[0]) of the previous query is still being read
            const uint4 R = (g || kSlot0) ? reinterpret_cast<const uint4*>(K[g ? g : kSlot0])[tid] : eq[0];
            finish_block<true>(p, vi * p.n_cols + colx, colx, vi, R, 2, K[0], s_pc, s_tr, s_dg);
        }
    }
}

}  // namespace bmb200
