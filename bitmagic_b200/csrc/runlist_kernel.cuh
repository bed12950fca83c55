// runlist_kernel.cuh -- the run-list companion of a set's GAP blocks (built once per set, streamed by agg_pipe_kernel).
//
// For a whole-set AND-SUB whose AND group holds no GAP block, every GAP block of the set is a SUB-group block: the GAP phase only
// clears the union of all GAP 1-runs of the column from the live mask, so block identity and order do not matter.  The companion
// re-encodes those 1-runs per column nb in two parts:
//   singles   sgl_pool word units [sgl_base[nb], sgl_base[nb+1]): the 1-runs of length 1, grouped by the 32-bit word of L they
//             fall in.  A 16-byte unit holds one word index w (0..2047) and up to 23 five-bit bit offsets inside it: u32 i = 0..2
//             holds fields 6i..6i+5 in bits [0, 30) and w's bits [2i, 2i+2) in bits [30, 32); u32 3 holds fields 18..22 in bits
//             [0, 25) and w's bits [6, 11) in bits [25, 30).  A word's n singles fill ceil(n / 23) units of its own; unused fields
//             of its last unit repeat one of its offsets (clearing a bit twice is harmless), so no count is stored;
//   long runs lr_pool units  [lr_base[nb],  lr_base[nb+1]):  one FLAT pair (s - 1 | e << 16) per 1-run [s, e] with e > s, padded
//             to 16 bytes with (0, 0) = no run.  A long run from bit 0 is stored as the single 0 plus the pair (0, e).
// At C3's densities (<= 1 %) almost every 1-run is a single bit, and a word of L collects ~70 of them per column: ~5.6 bits each
// instead of the 16 of a position.
// The build decodes every GAP block from its header, so FLAT and raw-form sets both have a companion.
// Those runs are part A of each column.  Part B lists, in the same encoding, the 1-runs of every sparse bit-block (a *listed*
// block: its list form -- 2 bytes per single, 4 per long run -- takes at most kListBitMax bytes).  A SUB-group bit-block only
// clears its 1-bits from the live mask, exactly as a GAP block's runs do, so a call whose AND group holds no listed block streams
// A + B and skips the listed 8 KB blocks.  Per column, A's and B's units are adjacent in sgl_pool ([sgl_base, sgl_mid) then
// [sgl_mid, sgl_base[nb+1])), and so are their long runs in lr_pool; each part is packed on its own.  listed: bit i = bit-block i
// of bit_pool is in part B.
// Union masks: a column whose part streams at least one full stage (kPipeStage = 8192 bytes of word units and long runs) also
// keeps that part as one 8 KB bitmap, the union of the runs its sweep clears -- U_A for part A, U_AB for A + B -- and the kernel
// streams the bitmap in their place (rl_union_kernel below).
// Order of a part's units: agg_pipe_kernel's sweep gives 16-byte unit u of a column's streamed range (from sgl_base[nb]) to lane
// u % 32 and issues one atomic per unit on its word, and a warp request is conflict-free when its 32 lanes touch 32 different
// shared-memory banks of L; word w lies in bank w & 31.  So each part is dealt out by bank: for rounds = min over banks of the
// bank's units, the unit that lane l eats holds a word of bank l (unit u of part A is lane u % 32's; part B is only ever streamed
// behind part A, so its unit u is lane (u + A's units) % 32's).  The leftover units follow, bank by bank.
#pragma once
#include "common.cuh"

namespace bmb200 {

constexpr int kRlThreads = 512;
constexpr int kRlWarps   = kRlThreads / 32;
constexpr int kRlCnt     = 2 * kRlWarps;       // u32 per column from the count pass: per-warp long-run counts of A, of B
// A bit-block is listed when 2 x singles + 4 x long runs <= kListBitMax bytes.  Every listed run is one more position for the
// consumers to sweep, so a larger threshold streams fewer bytes but sweeps more.  With one CTA per SM (H100 80GB HBM3, 400 W,
// DESIGN §6) C3 took 3.26 / 3.07 / 3.20 / 3.56 / 3.80 ms at 2048 / 3072 / 4096 / 6144 / 8192; with two CTAs per SM, whose sweeps
// overlap the other CTA's stream, 4096 is the faster of 3072 / 4096 (2.20 against 2.29 ms at 700 W).  With the singles dealt out
// by bank (above), swept with one atomic per position and a 12-stage ring, a listed position is cheaper still and the time follows
// the bytes: on another H100 80GB HBM3 at 700 W, 3 runs each alternated, C3 took 2.185-2.188 / 2.172-2.173 / 2.162-2.164 ms at
// 5120 / 5632 / 6144 and, in a second call, 2.162-2.163 / 2.154-2.156 / 2.164-2.165 ms at 6144 / 7168 / 8192, against 2.258-2.262
// for vector order at 4096.  From 6144 on the curve is flat (8192 streams only 0.7 % less), so the threshold stays at its low end,
// where the sweep has the least to do.  With the singles packed by word (above) a listed block streams fewer bytes than its list
// form, so denser blocks pay: on an H100 80GB HBM3 at 700 W (1980 MHz), 2 runs each alternated in one call, C3 took 1.329-1.332 /
// 1.320-1.322 / 1.278-1.280 / 1.326-1.327 ms at 6144 / 8192 / 12288 / 16384 (3.67 / 3.50 / 3.32 / 3.21 GB streamed per launch;
// past 12288 the extra long runs and listed positions cost more sweep than the bytes save).
constexpr uint32_t kListBitMax = 12288u;

// Where the singles of one column part go (word units, header above).  Count: put(p) counts p in rank[p >> 5] (out null).  Place:
// the r-th single taken by word w (rank[w] hands out r) goes to field r % 23 of the word's bank-local unit k = ust[w] + r / 23;
// bank b's unit k is the one lane b eats in round k while k < rounds, else leftover unit lb[b] + k - rounds.  The single of
// field 0 also writes the unit's word index and repeats its offset in the fields the word's cnt[w] singles leave empty.
// Fields and header bits are OR-ed into a zeroed pool, so ranks may come in any order; clearing bits commutes.
constexpr uint32_t kSglFields = 23u;
struct SglOut {
    uint32_t* out;             // the part's first unit, as 4 u32 each; null = count only
    uint32_t* rank;            // shared [2048]
    const uint32_t* cnt;       // shared [2048]: the part's singles per word
    const uint32_t* ust;       // shared [2048]: the word's first bank-local unit
    const uint32_t* lb;        // shared [32]: bank b's first leftover unit
    uint32_t rounds, rot;
    __device__ __forceinline__ void put(uint32_t pos) const
    {
        const uint32_t w = pos >> 5, o = pos & 31u, r = atomicAdd(&rank[w], 1u);
        if (!out) return;
        const uint32_t k = ust[w] + r / kSglFields, f = r % kSglFields, b = w & 31u;
        uint32_t* q = out + 4u * (k < rounds ? k * 32u + ((b - rot) & 31u) : lb[b] + k - rounds);
        if (f) { atomicOr(q + f / 6u, o << (5u * (f % 6u))); return; }
        uint32_t h[4] = {o | (w << 30), ((w >> 2) & 3u) << 30, ((w >> 4) & 3u) << 30, (w >> 6) << 25};
        for (uint32_t g = min(cnt[w] - r, kSglFields); g < kSglFields; ++g) h[g / 6u] |= o << (5u * (g % 6u));
#pragma unroll
        for (int i = 0; i < 4; ++i) atomicOr(q + i, h[i]);
    }
};

// The GAP block at g (= &buf[0], lead pad already skipped) with header hdr = g[0] holds gap_ones(hdr) 1-runs; gap_one_run gives
// 1-run j as bits [s, e] (run k = 2j+1 when the first run is 1, else 2j+2).
__device__ __forceinline__ uint32_t gap_ones(uint32_t hdr)
{
    const uint32_t len = hdr >> 3;
    return (hdr & 1u) ? (len + 1u) >> 1 : len >> 1;
}
__device__ __forceinline__ void gap_one_run(const uint16_t* __restrict__ g, uint32_t hdr, uint32_t j, uint32_t& s, uint32_t& e)
{
    const uint32_t k = 2u * j + ((hdr & 1u) ? 1u : 2u);
    s = (k == 1u) ? 0u : g[k - 1u] + 1u;
    e = g[k];
}

// One warp decodes the GAP block at g: singles through so, long-run pairs in order to lout[nl..) unless lout is null.  ns / nl
// are warp-uniform running counts.
__device__ __forceinline__ void rl_block(const uint16_t* __restrict__ g, uint32_t lane, uint32_t& ns, uint32_t& nl,
                                         const SglOut& so, uint32_t* lout)
{
    const uint32_t hdr = g[0], nsel = gap_ones(hdr);
    const uint32_t lt = (1u << lane) - 1u;
    for (uint32_t j0 = 0; j0 < nsel; j0 += 32u) {
        const uint32_t j = j0 + lane;
        uint32_t s = 0, e = 0;
        const bool ok = j < nsel;
        if (ok) gap_one_run(g, hdr, j, s, e);
        const bool sg = ok && (s == e || s == 0u), lg = ok && e > s;
        const uint32_t bs = __ballot_sync(0xffffffffu, sg), bl = __ballot_sync(0xffffffffu, lg);
        if (sg) so.put(s);
        if (lout && lg) lout[nl + __popc(bl & lt)] = (s ? s - 1u : 0u) | (e << 16);
        ns += __popc(bs); nl += __popc(bl);
    }
}

// Warp w of a column takes vectors [w * per, (w + 1) * per) and hands each GAP block, in vector order, to blk(g) (g = &buf[0],
// lead pad skipped) with the whole warp.  nfull (unless null) grows by the warp's FULL blocks.
template <typename F>
__device__ __forceinline__ void rl_gap_blocks(const SetView v, uint32_t nb, uint32_t warp, uint32_t lane, uint32_t* nfull, F&& blk)
{
    const uint32_t M = v.n_vec, per = (M + kRlWarps - 1u) / kRlWarps;
    const uint32_t* drow = v.desc + (size_t)nb * M;
    const uint16_t* gseg = v.gap_pool + v.gap_base[nb] * (size_t)kGapUnit;
    for (uint32_t v0 = warp * per; v0 < min(M, (warp + 1u) * per); v0 += 32u) {
        const uint32_t x = v0 + lane;
        const uint32_t d = (x < min(M, (warp + 1u) * per)) ? drow[x] : BMB200_BLK_NULL;
        uint32_t m = __ballot_sync(0xffffffffu, (d & 3u) == BMB200_BLK_GAP);
        if (nfull) *nfull += __popc(__ballot_sync(0xffffffffu, (d & 3u) == BMB200_BLK_FULL));
        while (m) {
            const int l = __ffs(m) - 1; m &= m - 1u;
            const uint32_t dl = __shfl_sync(0xffffffffu, d, l);
            blk(gseg + (size_t)((dl >> 2) & BMB200_DESC_REL_MASK) * kGapUnit + (dl >> 31));
        }
    }
}

// The column's GAP blocks through rl_block: warp w's long runs land in vector order behind those of warps < w.
__device__ __forceinline__ void rl_column(const SetView v, uint32_t nb, uint32_t warp, uint32_t lane, uint32_t& ns, uint32_t& nl,
                                          const SglOut& so, uint32_t* lout, uint32_t* nfull = nullptr)
{
    rl_gap_blocks(v, nb, warp, lane, nfull, [&](const uint16_t* g) { rl_block(g, lane, ns, nl, so, lout); });
}

__device__ __forceinline__ uint32_t warp_excl_scan(uint32_t v, uint32_t lane, uint32_t& total)
{
    uint32_t x = v;
#pragma unroll
    for (uint32_t o = 1; o < 32u; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    total = __shfl_sync(0xffffffffu, x, 31);
    return x - v;
}

// One warp lists the 1-runs of the bit-block at w, 32 consecutive words per step, in part A's encoding.  MEASURE: ns / nl grow by
// this lane's counts of singles and long runs.  Else singles go through so and, unless lout16 is null, long-run pairs in bit order
// to lout16[2 nl..), nl a warp-uniform running count.  A pair is written as its two u16 halves: the lane holding the k-th long-run
// start writes s - 1 (0 for a run from bit 0), the lane holding the k-th long-run end writes e, so a run that crosses words or
// steps needs no pairing.
template <bool MEASURE>
__device__ __forceinline__ void rl_bit_block(const uint32_t* __restrict__ w, uint32_t lane, uint32_t& ns, uint32_t& nl,
                                             const SglOut& so, uint16_t* lout16)
{
    uint32_t ne = nl;
#pragma unroll 4
    for (uint32_t i = lane; i < kBlockWords; i += 32u) {
        const uint32_t x = w[i];
        uint32_t pv = __shfl_up_sync(0xffffffffu, x, 1), nx = __shfl_down_sync(0xffffffffu, x, 1);
        if (lane == 0u)  pv = i ? w[i - 1u] : 0u;                           // the bits around the block are 0
        if (lane == 31u) nx = i + 1u < kBlockWords ? w[i + 1u] : 0u;
        const uint32_t S = x & ~((x << 1) | (pv >> 31)), E = x & ~((x >> 1) | (nx << 31));   // first / last bits of the 1-runs
        const uint32_t ls = S & ~E, le = E & ~S;                                              // ... of the long runs
        const uint32_t sm = (S & E) | (i == 0u ? ls & 1u : 0u);            // singles; a long run from bit 0 adds the single 0
        if (MEASURE) {
            ns += __popc(sm); nl += __popc(ls);
        } else {
            for (uint32_t m = sm; m; m &= m - 1u) so.put(32u * i + (uint32_t)__ffs(m) - 1u);
        }
        if (!MEASURE && lout16) {
            uint32_t tl, te;
            uint32_t ol = nl + warp_excl_scan(__popc(ls), lane, tl), oe = ne + warp_excl_scan(__popc(le), lane, te);
            for (uint32_t m = ls; m; m &= m - 1u) {
                const uint32_t s = 32u * i + (uint32_t)__ffs(m) - 1u;
                lout16[2u * ol++] = (uint16_t)(s ? s - 1u : 0u);
            }
            for (uint32_t m = le; m; m &= m - 1u) lout16[2u * oe++ + 1u] = (uint16_t)(32u * i + (uint32_t)__ffs(m) - 1u);
            nl += tl; ne += te;
        }
    }
}

// Part B of column nb: warp w takes the column's bit-blocks [w * per, (w + 1) * per), so their long runs land in bit_pool order
// behind those of warps < w.  MEASURE (count pass): measures every block, lists those within kListBitMax bytes (sets their flag,
// counts them in nlst, adds their runs to ns / nl) and counts their singles through so.  Else it lists the flagged blocks again.
template <bool MEASURE>
__device__ __forceinline__ void rl_bits(const SetView v, uint32_t nb, uint32_t warp, uint32_t lane, uint32_t& ns, uint32_t& nl,
                                        uint32_t& nlst, uint32_t* listed, const SglOut& so, uint16_t* lout16)
{
    const uint64_t b0 = v.bit_base[nb];
    const uint32_t n = (uint32_t)(v.bit_base[nb + 1] - b0), per = (n + kRlWarps - 1u) / kRlWarps;
    for (uint32_t j = warp * per; j < min(n, (warp + 1u) * per); ++j) {
        const uint64_t i = b0 + j;
        const uint32_t* blk = v.bit_pool + i * kBlockWords;
        if (MEASURE) {
            uint32_t ms = 0, ml = 0;
            rl_bit_block<true>(blk, lane, ms, ml, so, nullptr);
            const uint32_t s = warp_sum(ms), l = warp_sum(ml);
            if (2u * s + 4u * l <= kListBitMax) {
                ns += s; nl += l; ++nlst;
                if (lane == 0u) atomicOr(&listed[i >> 5], 1u << (i & 31u));
                rl_bit_block<false>(blk, lane, ms, ml, so, nullptr);
            }
        } else if ((listed[i >> 5] >> (i & 31u)) & 1u) {
            rl_bit_block<false>(blk, lane, ns, nl, so, lout16);
        }
    }
}

// Deals one column part out by bank, CTA-wide between barriers, from cnt[w] = the part's singles in word w of L (a word's singles
// fill ceil(cnt[w] / 23) units): ust[w] = the word's first unit among its bank's, lb[b] = bank b's first leftover unit, du = (full
// rounds = min over banks of the bank's units, the part's units).  ub: shared scratch [32].
__device__ __forceinline__ void rl_deal(const uint32_t* cnt, uint32_t* ust, uint32_t* ub, uint32_t* lb, uint32_t* du, uint32_t warp,
                                        uint32_t lane)
{
    for (uint32_t b = warp; b < 32u; b += kRlWarps) {        // bank b holds the words b + 32 j; lane takes j = 2 lane, 2 lane + 1
        const uint32_t w0 = b + 64u * lane, w1 = w0 + 32u;
        const uint32_t u0 = (cnt[w0] + kSglFields - 1u) / kSglFields, u1 = (cnt[w1] + kSglFields - 1u) / kSglFields;
        uint32_t t;
        const uint32_t x = warp_excl_scan(u0 + u1, lane, t);
        ust[w0] = x; ust[w1] = x + u0;
        if (lane == 0u) ub[b] = t;
    }
    __syncthreads();
    if (warp == 0u) {
        const uint32_t u = ub[lane], r = __reduce_min_sync(0xffffffffu, u);
        uint32_t t;
        lb[lane] = 32u * r + warp_excl_scan(u - r, lane, t);
        if (lane == 0u) { du[0] = r; du[1] = 32u * r + t; }
    }
    __syncthreads();
}

// pass 1, one CTA per column: per-warp long-run counts wlr[nb][w] of part A and wlr[nb][kRlWarps + w] of part B, the column's
// FULL blocks full_cnt[nb] (agg_pipe_kernel's plan: a SUB-group block is FULL when the AND group holds fewer), the listed flags
// (zeroed before the launch), the column's word units (A + B) and long-run units, and the set's totals tot = (A singles units,
// A long-run units, B singles units, B long-run units in the list form, listed blocks, A word units, B word units), zeroed before
// the launch.  The list form keeps 8 singles and 4 long runs per 16-byte unit, each column part padded on its own.
__global__ void __launch_bounds__(kRlThreads) rl_count_kernel(const SetView v, uint32_t* __restrict__ wlr, uint64_t* __restrict__ sgl_units,
                                                              uint64_t* __restrict__ lr_units, uint32_t* __restrict__ listed,
                                                              uint16_t* __restrict__ full_cnt, unsigned long long* __restrict__ tot)
{
    __shared__ uint32_t s_cnt[2][kBlockWords], s_ust[kBlockWords], s_c[5][kRlWarps], s_n[kRlWarps], s_ub[32], s_lb[32], s_du[2][2];
    const uint32_t nb = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    for (uint32_t i = threadIdx.x; i < 2u * kBlockWords; i += kRlThreads) (&s_cnt[0][0])[i] = 0u;
    __syncthreads();
    uint32_t ns = 0, nl = 0, bs = 0, bl = 0, nlst = 0, nfull = 0;
    rl_column(v, nb, warp, lane, ns, nl, SglOut{nullptr, s_cnt[0]}, nullptr, &nfull);
    rl_bits<true>(v, nb, warp, lane, bs, bl, nlst, listed, SglOut{nullptr, s_cnt[1]}, nullptr);
    if (lane == 0) {
        s_c[0][warp] = ns; s_c[1][warp] = nl; s_c[2][warp] = bs; s_c[3][warp] = bl; s_c[4][warp] = nfull; s_n[warp] = nlst;
        wlr[(size_t)nb * kRlCnt + warp] = nl; wlr[(size_t)nb * kRlCnt + kRlWarps + warp] = bl;
    }
    __syncthreads();
    rl_deal(s_cnt[0], s_ust, s_ub, s_lb, s_du[0], warp, lane);
    rl_deal(s_cnt[1], s_ust, s_ub, s_lb, s_du[1], warp, lane);
    if (threadIdx.x == 0) {
        uint32_t t[5] = {0, 0, 0, 0, 0}, f = 0;
        for (int w = 0; w < kRlWarps; ++w) {
            for (int k = 0; k < 4; ++k) t[k] += s_c[k][w];
            t[4] += s_n[w]; f += s_c[4][w];
        }
        full_cnt[nb] = (uint16_t)f;
        const uint32_t u[7] = {(t[0] + 7u) / 8u, (t[1] + 3u) / 4u, (t[2] + 7u) / 8u, (t[3] + 3u) / 4u, t[4], s_du[0][1], s_du[1][1]};
        sgl_units[nb] = u[5] + u[6];
        lr_units[nb] = u[1] + u[3];
#pragma unroll
        for (int k = 0; k < 7; ++k) if (u[k]) atomicAdd(&tot[k], (unsigned long long)u[k]);
    }
}

// pass 2, one CTA per column, into a zeroed sgl pool: per part, every warp decodes its GAP blocks (A) or lists its flagged
// bit-blocks again (B) once to count the part's singles per word, and once more to place them into the part's word units (A at
// the column's base, B behind it) and its long runs into the warp's slots, then the long-run pads
__global__ void __launch_bounds__(kRlThreads) rl_write_kernel(const SetView v, const uint32_t* __restrict__ wlr,
                                                              const uint64_t* __restrict__ sgl_base, const uint64_t* __restrict__ lr_base,
                                                              const uint32_t* __restrict__ listed, uint32_t* __restrict__ sgl,
                                                              uint32_t* __restrict__ lr, uint64_t* __restrict__ sgl_mid,
                                                              uint64_t* __restrict__ lr_mid)
{
    __shared__ uint32_t s_cnt[kBlockWords], s_rank[kBlockWords], s_ust[kBlockWords], s_ub[32], s_lb[32], s_du[2];
    const uint32_t nb = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    uint32_t nl = 0, tl = 0, bl = 0, tbl = 0, ns = 0, nx = 0, nlst = 0;
    for (uint32_t w = 0; w < (uint32_t)kRlWarps; ++w) {
        const uint32_t c = wlr[(size_t)nb * kRlCnt + w], cb = wlr[(size_t)nb * kRlCnt + kRlWarps + w];
        if (w < warp) { nl += c; bl += cb; }
        tl += c; tbl += cb;
    }
    const uint32_t lcap = (tl + 3u) / 4u * 4u, blcap = (tbl + 3u) / 4u * 4u;
    uint32_t* sout = sgl + sgl_base[nb] * 4u;
    uint32_t* lout = lr + lr_base[nb] * 4u;
    uint32_t* blout = lout + lcap;
    uint32_t ua = 0;
    for (int part = 0; part < 2; ++part) {
        for (uint32_t i = threadIdx.x; i < kBlockWords; i += kRlThreads) { s_cnt[i] = 0u; s_rank[i] = 0u; }
        __syncthreads();
        if (part == 0) rl_column(v, nb, warp, lane, ns, nx, SglOut{nullptr, s_cnt}, nullptr);
        else rl_bits<false>(v, nb, warp, lane, ns, nx, nlst, const_cast<uint32_t*>(listed), SglOut{nullptr, s_cnt}, nullptr);
        __syncthreads();
        rl_deal(s_cnt, s_ust, s_ub, s_lb, s_du, warp, lane);
        if (part == 0) {
            ua = s_du[1];
            rl_column(v, nb, warp, lane, ns, nl, SglOut{sout, s_rank, s_cnt, s_ust, s_lb, s_du[0], 0u}, lout);
        } else {
            rl_bits<false>(v, nb, warp, lane, ns, bl, nlst, const_cast<uint32_t*>(listed),
                           SglOut{sout + 4u * ua, s_rank, s_cnt, s_ust, s_lb, s_du[0], ua & 31u}, reinterpret_cast<uint16_t*>(blout));
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) { sgl_mid[nb] = sgl_base[nb] + ua; lr_mid[nb] = lr_base[nb] + lcap / 4u; }
    for (uint32_t i = tl + threadIdx.x; i < lcap; i += kRlThreads) lout[i] = 0u;
    for (uint32_t i = tbl + threadIdx.x; i < blcap; i += kRlThreads) blout[i] = 0u;
}

// Union masks, one CTA per column: un_slot[2 nb] / [2 nb + 1] = the un_pool slot of the column's U_A / U_AB (~0 = none; a column
// whose part B is empty may name one slot twice).  U_A is every bit the sweep of part A clears, U_AB every bit the sweep of A + B
// clears: both are decoded from the pools in the sweep's own layout (sgl_unit and flat_quad in agg_kernel.cuh), so a union stage
// clears exactly what the column's packed stages would.
__device__ __forceinline__ void rl_union_part(uint32_t* U, const uint4* __restrict__ sgl, uint64_t s0, uint64_t s1,
                                              const uint32_t* __restrict__ lr, uint64_t l0, uint64_t l1)
{
    for (uint64_t i = s0 + threadIdx.x; i < s1; i += kRlThreads) {       // word unit: 23 five-bit offsets inside one word
        const uint4 q = sgl[i];
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
        uint32_t m = 0;
#pragma unroll
        for (int f = 0; f < (int)kSglFields; ++f) m |= 1u << ((w[f / 6] >> (5 * (f % 6))) & 31u);
        atomicOr(&U[(q.x >> 30) | ((q.y >> 30) << 2) | ((q.z >> 30) << 4) | ((q.w >> 25) << 6)], m);
    }
    for (uint64_t i = 4u * l0 + threadIdx.x; i < 4u * l1; i += kRlThreads) {   // FLAT pair (s - 1 | e << 16): bits [s, e]; (0, 0) = none
        const uint32_t lo = lr[i] & 0xffffu, e = lr[i] >> 16;
        if (e <= lo) continue;
        for (uint32_t s = lo + 1u; s <= e; s = (s | 31u) + 1u) {
            const uint32_t n = min(e - s + 1u, 32u - (s & 31u));
            atomicOr(&U[s >> 5], (n == 32u ? ~0u : (1u << n) - 1u) << (s & 31u));
        }
    }
}

__global__ void __launch_bounds__(kRlThreads) rl_union_kernel(const uint64_t* __restrict__ sgl_base, const uint64_t* __restrict__ sgl_mid,
                                                              const uint64_t* __restrict__ lr_base, const uint64_t* __restrict__ lr_mid,
                                                              const uint4* __restrict__ sgl, const uint32_t* __restrict__ lr,
                                                              const uint32_t* __restrict__ un_slot, uint32_t* __restrict__ un_pool)
{
    __shared__ uint32_t U[kBlockWords];
    const uint32_t nb = blockIdx.x, sa = un_slot[2u * nb], sab = un_slot[2u * nb + 1u];
    if (sab == ~0u) return;                                   // U_A implies U_AB: A + B streams no less than A
    for (uint32_t i = threadIdx.x; i < kBlockWords; i += kRlThreads) U[i] = 0u;
    __syncthreads();
    rl_union_part(U, sgl, sgl_base[nb], sgl_mid[nb], lr, lr_base[nb], lr_mid[nb]);
    __syncthreads();
    if (sa != ~0u)
        for (uint32_t i = threadIdx.x; i < kBlockWords; i += kRlThreads) un_pool[(size_t)sa * kBlockWords + i] = U[i];
    __syncthreads();
    rl_union_part(U, sgl, sgl_mid[nb], sgl_base[nb + 1], lr, lr_mid[nb], lr_base[nb + 1]);
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < kBlockWords; i += kRlThreads) un_pool[(size_t)sab * kBlockWords + i] = U[i];
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
