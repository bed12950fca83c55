// scan_in_kernel.cuh -- set-membership search over the planes of a sparse vector (sm_90a).
//
// Replaces the reference's iterator form of sparse_vector_scanner<SV>::find_eq (src/bmsparsevec_algo.h:1398-1423): elements
// equal to ANY value of a list (SQL `col IN (...)`).  The reference runs one full AND-SUB aggregation over the planes per listed
// value; a bit-sliced EQ walk (scan_kernel.cuh) likewise tests one value per state.  Here the work does not grow with the list:
//   * one work item per block column; every plane block (and the universe U) of the column is read from HBM once, a chunk of
//     kInChunkWords words at a time, into shared memory rows (NULL / FULL / bit planes copied, GAP planes expanded clipped to the
//     chunk, FLAT or raw);
//   * each warp rebuilds the element codes of one 32-element word at a time: lane j reads plane j's word, a 5-step shuffle
//     butterfly transposes the 32 x 32 bit matrix, and lane i then holds the code of element i (a second transpose for planes
//     32..63 gives the high half);
//   * every code inside U is looked up in the sorted, unique code list: a branch-free binary search over the list staged in
//     shared memory (up to kInStage codes); a longer list keeps every bucket-th code there as splitters, and the search finishes
//     inside one bucket of the list in global memory (L2-resident), so a lookup costs log2(K) steps for any K;
//   * words with U = 0 are skipped whole; the result word is the ballot of the hits.
// The result block goes through finish_block (popcount, digest, run count, kind, bit->GAP) like every other scan result.
// Codes are the stored ones (s2u(x) for signed vectors): the host applies s2u, sorts, de-duplicates and drops codes with bits at
// or above n_planes, which no element can hold.
#pragma once
#include "column_walk.cuh"

namespace bmb200 {

constexpr uint32_t kInChunkWords = 256;                  // words of every plane staged per pass (8 passes per column)
constexpr uint32_t kInRowStride  = kInChunkWords + 1;    // odd row stride: lane j reading word w of row j hits bank (j + w) % 32
constexpr uint32_t kInStage      = 4096;                 // codes of the list (or its splitters) held in shared memory: 32 KB
constexpr int      kInLoads      = 4;                    // 16-byte plane loads in flight per thread while a chunk is staged

struct ScanInParams {
    AggParams out;             // set view + result buffers + work counter (one group of n_cols columns)
    uint32_t  plane0;          // plane j (bit j of the code) = set vector plane0 + j
    uint32_t  n_planes;        // 1..64
    uint32_t  universe;        // set vector holding the searchable indexes; 0xffffffff = everything
    uint32_t  n_codes;         // sorted, unique codes; 0 = nothing can match
    uint32_t  bucket;          // n_codes > kInStage: codes per bucket (splitter t = codes[t * bucket]); 0 = the list is staged whole
    uint32_t  n_stage;         // entries staged in shared memory (the list, or one splitter per bucket)
    const uint64_t* codes;     // device: n_codes codes, ascending
};

// dynamic shared memory of scan_in_kernel: the staged list, the result block, (n_planes + 1) rows of one chunk
__host__ inline size_t scan_in_smem(uint32_t n_planes)
{
    return (size_t)kInStage * 8u + (size_t)kBlockWords * 4u + (size_t)(n_planes + 1u) * kInRowStride * 4u;
}

// lane j holds row j of a 32 x 32 bit matrix (bit i = column i); returns column `lane` (bit j = bit lane of row j)
__device__ __forceinline__ uint32_t warp_transpose32(uint32_t x, int lane)
{
    constexpr uint32_t kLo[5] = {0x0000FFFFu, 0x00FF00FFu, 0x0F0F0F0Fu, 0x33333333u, 0x55555555u};   // bits i with i & s == 0
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        const int s = 16 >> k;
        const uint32_t m = kLo[k];
        const uint32_t y = __shfl_xor_sync(0xffffffffu, x, s);
        x = (lane & s) ? (x & ~m) | ((y >> s) & m) : (x & m) | ((y << s) & ~m);
    }
    return x;
}

// is c one of the codes?  L = the staged list, or the splitters of its buckets
__device__ __forceinline__ bool in_codes(uint64_t c, const uint64_t* L, const ScanInParams& sp)
{
    uint32_t base = 0, len = sp.n_stage;                     // last staged entry <= c (c >= L[0] is checked by the caller)
    while (len > 1) { const uint32_t half = len >> 1; if (L[base + half] <= c) base += half; len -= half; }
    if (!sp.bucket) return L[base] == c;
    const uint64_t* g = sp.codes + (size_t)base * sp.bucket;
    uint32_t b = 0;
    len = min(sp.bucket, sp.n_codes - base * sp.bucket);
    while (len > 1) { const uint32_t half = len >> 1; if (__ldg(g + b + half) <= c) b += half; len -= half; }
    return __ldg(g + b) == c;
}

// OR the 1-runs of one GAP block that fall inside bits [bit0, bit0 + 32 * kInChunkWords) into a zeroed chunk row, all threads
__device__ __forceinline__ void gap_expand_chunk(uint32_t* row, const uint16_t* __restrict__ g, uint32_t bit0, int tid)
{
    const uint32_t hdr = g[0];
    const uint32_t len = hdr >> 3;
    const bool odd = (hdr & 1u) != 0u;                       // first run is a 1-run
    const uint32_t nsel = odd ? (len + 1u) >> 1 : len >> 1;
    const uint16_t* a0 = g + (odd ? 0 : 1);
    const uint32_t bit1 = bit0 + 32u * kInChunkWords - 1u;
    for (uint32_t j = tid; j < nsel; j += kAggThreads) {
        uint32_t s = (odd && j == 0u) ? 0u : a0[2u * j] + 1u, e = a0[2u * j + 1u];
        if (e < bit0 || s > bit1) continue;
        s = max(s, bit0) - bit0; e = min(e, bit1) - bit0;
        const uint32_t ws = s >> 5, we = e >> 5;
        if (ws == we) { red_or_shared(row + ws, bit_range_mask(s & 31u, e & 31u)); continue; }
        red_or_shared(row + ws, 0xffffffffu << (s & 31u));   // edge words may be shared with a neighbouring run
        for (uint32_t w = ws + 1u; w < we; ++w) row[w] = 0xffffffffu;   // inner words belong to this run alone
        red_or_shared(row + we, 0xffffffffu >> (31u - (e & 31u)));
    }
}

// Stage words [c0, c0 + kInChunkWords) of the blocks desc(0..n_rows) of one column into the odd-stride rows: 16-byte loads of
// the bit blocks (kInLoads in flight per thread), scalar stores; GAP rows start zeroed and get their runs ORed in (any_gap: some
// desc(r) is GAP, the same for every thread).  Ends with a barrier, so the rows can be read.  scan_in_kernel and remap_kernel.
template <class Desc>
__device__ __forceinline__ void stage_chunk(uint32_t* rows, uint32_t n_rows, const Desc& desc, bool any_gap, const uint4* bseg,
                                            const uint16_t* gseg, uint32_t c0, int tid)
{
    const uint32_t nq = n_rows * (kInChunkWords / 4u);
    for (uint32_t q0 = tid; q0 < nq; q0 += kInLoads * kAggThreads) {
        uint4 v[kInLoads];
#pragma unroll
        for (int u = 0; u < kInLoads; ++u) {
            const uint32_t q = q0 + u * kAggThreads, r = q / (kInChunkWords / 4u);
            const uint32_t d = q < nq ? desc(r) : BMB200_BLK_NULL, kind = d & 3u;
            v[u] = make_uint4(0u, 0u, 0u, 0u);
            if (kind == BMB200_BLK_BIT) v[u] = ld_stream_v4(bseg + (size_t)(d >> 2) * (kBlockWords / 4) + c0 / 4u + q % (kInChunkWords / 4u));
            else if (kind == BMB200_BLK_FULL) v[u] = make_uint4(~0u, ~0u, ~0u, ~0u);
        }
#pragma unroll
        for (int u = 0; u < kInLoads; ++u) {
            const uint32_t q = q0 + u * kAggThreads;
            if (q >= nq) break;
            uint32_t* dst = rows + (q / (kInChunkWords / 4u)) * kInRowStride + 4u * (q % (kInChunkWords / 4u));
            dst[0] = v[u].x; dst[1] = v[u].y; dst[2] = v[u].z; dst[3] = v[u].w;
        }
    }
    if (any_gap) {
        __syncthreads();
        for (uint32_t r = 0; r < n_rows; ++r) {
            const uint32_t d = desc(r);
            if ((d & 3u) != BMB200_BLK_GAP) continue;
            gap_expand_chunk(rows + r * kInRowStride, gap_block_ptr(gseg, d), 32u * c0, tid);
        }
    }
    __syncthreads();
}

// WIDE: more than 32 planes (codes in two transposed halves)
template <bool WIDE>
__global__ void __launch_bounds__(kAggThreads, kCtasPerSm) scan_in_kernel(const ScanInParams sp)
{
    extern __shared__ __align__(16) uint64_t s_in[];
    uint64_t* L = s_in;                                                   // staged list / splitters
    uint32_t* Rw = reinterpret_cast<uint32_t*>(L + kInStage);             // the column's result block
    uint32_t* rows = Rw + kBlockWords;                                    // planes 0..n-1, universe last: one chunk each
    __shared__ uint32_t s_desc[65];                                       // plane descriptors of this column, universe in [64]
    __shared__ uint32_t s_col;
    __shared__ uint32_t s_pc[kAggWarps], s_tr[kAggWarps], s_dg[kAggWarps];

    const AggParams& p = sp.out;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t M = p.set.n_vec, np = sp.n_planes;
    for (uint32_t i = tid; i < sp.n_stage; i += kAggThreads) L[i] = sp.codes[(size_t)i * (sp.bucket ? sp.bucket : 1u)];
    const uint64_t cmin = sp.n_codes ? sp.codes[0] : 0ull, cmax = sp.n_codes ? sp.codes[sp.n_codes - 1] : 0ull;

    WorkClaim claim(p.work_counter);
    for (;;) {
        const uint32_t colx = claim.next(p.work_counter, s_col, p.n_cols);
        if (colx >= p.n_cols) break;
        const uint32_t nb = p.nb_from + colx;
        const uint32_t* drow = p.set.desc + (size_t)nb * M;
        if (tid < (int)np) s_desc[tid] = drow[sp.plane0 + tid];
        if (tid == 64) s_desc[64] = (sp.universe == 0xffffffffu) ? BMB200_BLK_FULL : drow[sp.universe];
        const uint4* bseg = reinterpret_cast<const uint4*>(p.set.bit_pool) + p.set.bit_base[nb] * (size_t)(kBlockWords / 4);
        const uint16_t* gseg = p.set.gap_pool + p.set.gap_base[nb] * (size_t)kGapUnit;
        __syncthreads();
        const uint32_t du = s_desc[64];

        if ((du & 3u) == BMB200_BLK_NULL || !sp.n_codes) {                // nothing searchable in this column
            reinterpret_cast<uint4*>(Rw)[tid] = make_uint4(0u, 0u, 0u, 0u);
        } else {
            bool any_gap = false;
            for (uint32_t r = 0; r <= np; ++r) any_gap |= ((r < np ? s_desc[r] : du) & 3u) == BMB200_BLK_GAP;
            const auto desc = [&](uint32_t r) { return r < np ? s_desc[r] : du; };   // planes, then the universe
            for (uint32_t c0 = 0; c0 < kBlockWords; c0 += kInChunkWords) {
                stage_chunk(rows, np + 1u, desc, any_gap, bseg, gseg, c0, tid);
                // one 32-element word per warp and step: transpose the planes into codes, look the codes inside U up
                for (uint32_t w = (uint32_t)warp; w < kInChunkWords; w += kAggWarps) {
                    const uint32_t uw = rows[np * kInRowStride + w];
                    uint32_t hits = 0u;
                    if (uw) {                                                 // warp-uniform
                        uint64_t c = warp_transpose32((uint32_t)lane < np ? rows[lane * kInRowStride + w] : 0u, lane);
                        if (WIDE) {
                            const uint32_t hi = (uint32_t)lane + 32u < np ? rows[(lane + 32) * kInRowStride + w] : 0u;
                            c |= (uint64_t)warp_transpose32(hi, lane) << 32;
                        }
                        const bool hit = ((uw >> lane) & 1u) && c >= cmin && c <= cmax && in_codes(c, L, sp);
                        hits = __ballot_sync(0xffffffffu, hit);
                    }
                    if (lane == 0) Rw[c0 + w] = hits;
                }
                __syncthreads();                                              // the rows are restaged by the next chunk
            }
        }
        __syncthreads();
        const uint4 R = reinterpret_cast<const uint4*>(Rw)[tid];
        finish_block<true>(p, colx, colx, 0u, R, 2, Rw, s_pc, s_tr, s_dg);
    }
}

}  // namespace bmb200
