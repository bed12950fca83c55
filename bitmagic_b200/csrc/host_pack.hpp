// host_pack.hpp -- host side of bmb200_set_upload_vectors: the block trees of n_vec vectors (kind + pointer per block slot, what
// blocks_manager::get_block_ptr(i,j) yields, src/bmblocks.h:556) are gathered into the column-major arena layout
// (include/bmb200.h, bmb200_packed_set) by a team of host threads and streamed to the GPU through a ring of pinned staging
// slots, so that packing chunk c+1 overlaps the DMA of chunk c.  Host code only: no block is interpreted here beyond the GAP
// header (length, first-run value); all set algebra stays on the device.
//
// The reference keeps every block behind two dependent pointer loads per (i,j) (src/bmaggregator.h:2278-2366 gathers them per
// block column on every call); here the gather happens ONCE per upload and the result stays resident (bm::b200::device_set).
#pragma once
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <sched.h>
#include <thread>
#include <vector>

#include "../../include/bmb200.h"

namespace bmb200 {

constexpr uint32_t kStageSlots = 4;

struct PackLayout {
    std::vector<uint32_t> desc;          // [n_blocks][n_vec]
    std::vector<uint64_t> bb, gb;        // [n_blocks + 1] prefix sums (blocks / 16-byte units)
    int rc = BMB200_OK;
};

// default team size: half of the CPUs this thread may run on (~ the physical cores of the NUMA node it is bound to), at most 32.
// The issuing thread must keep a CPU for itself: with one packer per logical CPU it was scheduled late on every chunk,
// which stretched the upload well past what the DMA needs; PCIe needs ~55 GB/s of memcpy, which 16-32 cores deliver.
inline unsigned pack_threads(unsigned want, uint64_t items)
{
    unsigned t = want;
    if (!t) {
        cpu_set_t cs; CPU_ZERO(&cs);
        unsigned allowed = (sched_getaffinity(0, sizeof cs, &cs) == 0) ? (unsigned)CPU_COUNT(&cs) : std::thread::hardware_concurrency();
        t = allowed / 2;
        if (t > 32) t = 32;
    }
    if (t == 0) t = 1;
    if (t > 64) t = 64;
    if ((uint64_t)t > items) t = (unsigned)(items ? items : 1);
    return t;
}

// pass 1: descriptors + per-column sizes.  Threads own contiguous column ranges; the prefix sums are serial (n_blocks adds).
inline void pack_layout(uint32_t n_vec, uint32_t n_blocks, const bmb200_vec_blocks* vecs, unsigned threads, PackLayout& L)
{
    L.desc.assign((size_t)n_vec * n_blocks, 0u);
    L.bb.assign((size_t)n_blocks + 1, 0); L.gb.assign((size_t)n_blocks + 1, 0);
    const unsigned T = pack_threads(threads, n_blocks);
    std::vector<int> rcs(T, BMB200_OK);
    auto work = [&](unsigned t) {
        const uint32_t lo = (uint32_t)((uint64_t)n_blocks * t / T), hi = (uint32_t)((uint64_t)n_blocks * (t + 1) / T);
        for (uint32_t nb = lo; nb < hi; ++nb) {
            uint64_t nbit = 0, ngap = 0;
            uint32_t* drow = L.desc.data() + (size_t)nb * n_vec;
            for (uint32_t v = 0; v < n_vec; ++v) {
                const uint32_t kd = (nb < vecs[v].n_blocks) ? vecs[v].kind[nb] : BMB200_BLK_NULL;
                uint32_t d = kd;
                if (kd == BMB200_BLK_BIT) {
                    if (!vecs[v].ptr[nb]) { rcs[t] = BMB200_ERR_BADARG; return; }
                    d |= (uint32_t)nbit++ << 2;
                } else if (kd == BMB200_BLK_GAP) {
                    const uint16_t* g = (const uint16_t*)vecs[v].ptr[nb];
                    if (!g) { rcs[t] = BMB200_ERR_BADARG; return; }
                    const uint32_t words = (uint32_t)(g[0] >> 3) + 1u;
                    if (words > BMB200_GAP_MAX_WORDS) { rcs[t] = BMB200_ERR_BADARG; return; }
                    // flat-streamable form (BMB200_DESC_GAP_FLAT): lead pad iff the first run is 0
                    const uint32_t pad = (g[0] & 1u) ? 0u : 1u;
                    const uint64_t units = (words + pad + BMB200_GAP_UNIT_WORDS - 1) / BMB200_GAP_UNIT_WORDS;
                    if (ngap + units > (uint64_t)BMB200_DESC_REL_MASK) { rcs[t] = BMB200_ERR_RANGE; return; }
                    d |= ((uint32_t)ngap << 2) | (pad ? BMB200_DESC_GAP_PAD : 0u) | BMB200_DESC_GAP_FLAT;
                    ngap += units;
                } else if (kd > 3u) { rcs[t] = BMB200_ERR_BADARG; return; }
                drow[v] = d;
            }
            L.bb[nb + 1] = nbit; L.gb[nb + 1] = ngap;      // per-column sizes; scanned below
        }
    };
    if (T == 1) work(0);
    else {
        std::vector<std::thread> th;
        for (unsigned t = 0; t < T; ++t) th.emplace_back(work, t);
        for (auto& x : th) x.join();
    }
    for (int r : rcs) if (r) { L.rc = r; return; }
    for (uint32_t nb = 0; nb < n_blocks; ++nb) { L.bb[nb + 1] += L.bb[nb]; L.gb[nb + 1] += L.gb[nb]; }
}

// Slab-backed sources (bmb200_set_upload_slabs): where every real block sits inside the device mirror of the host slabs, in 32-byte
// units (u32: mirrors up to 128 GB).  Threads own column ranges.  false = a block lies outside the slabs or is not 32-byte aligned.
struct SlabMap { std::vector<uint64_t> base, end, dev_off; };          // sorted by base; dev_off = byte offset of the slab inside the mirror

inline bool pack_sources(uint32_t n_vec, uint32_t n_blocks, const bmb200_vec_blocks* vecs, const PackLayout& L, const SlabMap& M,
                         unsigned threads, uint32_t* src)
{
    const unsigned T = pack_threads(threads, n_blocks);
    const size_t ns = M.base.size();
    std::vector<uint8_t> ok(T, 1);
    auto work = [&](unsigned t) {
        const uint32_t lo = (uint32_t)((uint64_t)n_blocks * t / T), hi = (uint32_t)((uint64_t)n_blocks * (t + 1) / T);
        size_t last = 0;
        for (uint32_t nb = lo; nb < hi; ++nb) {
            const uint32_t* drow = L.desc.data() + (size_t)nb * n_vec;
            uint32_t* srow = src + (size_t)nb * n_vec;
            for (uint32_t v = 0; v < n_vec; ++v) {
                const uint32_t kd = drow[v] & 3u;
                if (kd != BMB200_BLK_BIT && kd != BMB200_BLK_GAP) { srow[v] = 0; continue; }
                const uint64_t p = (uint64_t)(uintptr_t)vecs[v].ptr[nb];
                const uint64_t len = kd == BMB200_BLK_BIT ? (uint64_t)BMB200_BLOCK_BYTES
                                                          : ((uint64_t)(*(const uint16_t*)vecs[v].ptr[nb] >> 3) + 1u) * 2u;
                if (!(p >= M.base[last] && p + len <= M.end[last])) {
                    size_t a = 0, b = ns;                                   // last slab with base <= p
                    while (b - a > 1) { const size_t m = (a + b) / 2; if (M.base[m] <= p) a = m; else b = m; }
                    if (!(p >= M.base[a] && p + len <= M.end[a])) { ok[t] = 0; return; }
                    last = a;
                }
                const uint64_t off = M.dev_off[last] + (p - M.base[last]);
                if (off & 31u) { ok[t] = 0; return; }
                srow[v] = (uint32_t)(off >> 5);
            }
        }
    };
    if (T == 1) work(0);
    else {
        std::vector<std::thread> th;
        for (unsigned t = 0; t < T; ++t) th.emplace_back(work, t);
        for (auto& x : th) x.join();
    }
    for (uint8_t o : ok) if (!o) return false;
    return true;
}

// one column into its place inside a staging slot: bit-blocks at bit_dst (in descriptor order), GAP units at gap_dst
inline void pack_column(uint32_t n_vec, uint32_t nb, const bmb200_vec_blocks* vecs, const uint32_t* drow, uint8_t* bit_dst, uint8_t* gap_dst)
{
    for (uint32_t v = 0; v < n_vec; ++v) {
        const uint32_t d = drow[v], kd = d & 3u;
        if (kd == BMB200_BLK_BIT) {
            memcpy(bit_dst + (size_t)((d >> 2) & BMB200_DESC_REL_MASK) * BMB200_BLOCK_BYTES, vecs[v].ptr[nb], BMB200_BLOCK_BYTES);
        } else if (kd == BMB200_BLK_GAP) {
            const uint16_t* g = (const uint16_t*)vecs[v].ptr[nb];
            const uint32_t words = (uint32_t)(g[0] >> 3) + 1u, pad = d >> 31;
            uint16_t* dst = reinterpret_cast<uint16_t*>(gap_dst + (size_t)((d >> 2) & BMB200_DESC_REL_MASK) * 16u);
            if (pad) dst[0] = 0xffffu;
            memcpy(dst + pad, g, (size_t)words * 2u);
            const uint32_t n = words + pad, npad = (n + BMB200_GAP_UNIT_WORDS - 1) / BMB200_GAP_UNIT_WORDS * BMB200_GAP_UNIT_WORDS;
            for (uint32_t i = n; i < npad; ++i) dst[i] = 0;             // FLAT contract: zeros up to the next unit (slots are recycled)
        }
    }
}

// column chunks sized for one staging slot
struct PackChunk { uint32_t c0, c1; uint64_t bit_bytes, gap_bytes; };

inline void pack_chunks(const PackLayout& L, uint32_t n_blocks, uint64_t slot_bytes, std::vector<PackChunk>& out)
{
    uint32_t c0 = 0;
    while (c0 < n_blocks) {
        uint32_t c1 = c0; uint64_t bytes = 0;
        while (c1 < n_blocks) {
            const uint64_t col = (L.bb[c1 + 1] - L.bb[c1]) * (uint64_t)BMB200_BLOCK_BYTES + (L.gb[c1 + 1] - L.gb[c1]) * 16ull;
            if (c1 > c0 && bytes + col > slot_bytes) break;
            bytes += col; ++c1;
        }
        out.push_back({c0, c1, (L.bb[c1] - L.bb[c0]) * (uint64_t)BMB200_BLOCK_BYTES, (L.gb[c1] - L.gb[c0]) * 16ull});
        c0 = c1;
    }
}

inline uint64_t pack_max_column_bytes(const PackLayout& L, uint32_t n_blocks)
{
    uint64_t m = 0;
    for (uint32_t nb = 0; nb < n_blocks; ++nb) {
        const uint64_t col = (L.bb[nb + 1] - L.bb[nb]) * (uint64_t)BMB200_BLOCK_BYTES + (L.gb[nb + 1] - L.gb[nb]) * 16ull;
        if (col > m) m = col;
    }
    return m;
}

// The pipeline: worker threads claim columns in order and pack them into the slot of their chunk; the caller's thread (`issue`)
// is told when a chunk is complete, starts its H2D copies and later releases the slot (`released` = chunks whose slot is free again).
// Both waits block on condition variables: idle packers sleep instead of spinning next to the ones that copy.
struct PackPipeline {
    uint32_t n_vec = 0, n_blocks = 0;
    const bmb200_vec_blocks* vecs = nullptr;
    const PackLayout* L = nullptr;
    const std::vector<PackChunk>* chunks = nullptr;
    uint8_t* const* slot = nullptr;                    // kStageSlots pinned buffers
    std::vector<uint32_t> chunk_of_col;
    std::vector<std::atomic<uint32_t>> remaining;      // columns left per chunk
    std::atomic<uint32_t> next_col{0};
    std::mutex mu;
    std::condition_variable cv_free[kStageSlots], cv_done;   // packers wait per SLOT: a freed slot wakes the packers of its next chunk, not the whole team
    uint32_t released = 0;                             // guarded by mu
    std::vector<std::thread> th;

    PackPipeline(uint32_t nv, uint32_t nb, const bmb200_vec_blocks* v, const PackLayout* l, const std::vector<PackChunk>* ch, uint8_t* const* s)
        : n_vec(nv), n_blocks(nb), vecs(v), L(l), chunks(ch), slot(s), chunk_of_col(nb), remaining(ch->size())
    {
        for (size_t c = 0; c < ch->size(); ++c) {
            remaining[c].store((*ch)[c].c1 - (*ch)[c].c0, std::memory_order_relaxed);
            for (uint32_t nbk = (*ch)[c].c0; nbk < (*ch)[c].c1; ++nbk) chunk_of_col[nbk] = (uint32_t)c;
        }
    }
    void start(unsigned threads)
    {
        const unsigned T = pack_threads(threads, n_blocks);
        for (unsigned t = 0; t < T; ++t) th.emplace_back([this]() { run(); });
    }
    void run()
    {
        uint32_t seen_released = 0;
        for (;;) {
            const uint32_t nb = next_col.fetch_add(1, std::memory_order_relaxed);
            if (nb >= n_blocks) return;
            const uint32_t c = chunk_of_col[nb];
            if (c >= seen_released + kStageSlots) {                       // the slot of chunk c is still owned by chunk c - kStageSlots
                std::unique_lock<std::mutex> lk(mu);
                cv_free[c % kStageSlots].wait(lk, [&]() { return c < released + kStageSlots; });
                seen_released = released;
            }
            const PackChunk& ch = (*chunks)[c];
            uint8_t* base = slot[c % kStageSlots];
            uint8_t* bit_dst = base + (L->bb[nb] - L->bb[ch.c0]) * (uint64_t)BMB200_BLOCK_BYTES;
            uint8_t* gap_dst = base + ch.bit_bytes + (L->gb[nb] - L->gb[ch.c0]) * 16ull;
            pack_column(n_vec, nb, vecs, L->desc.data() + (size_t)nb * n_vec, bit_dst, gap_dst);
            if (remaining[c].fetch_sub(1, std::memory_order_acq_rel) == 1) {   // last column of the chunk: wake the issuing thread
                std::lock_guard<std::mutex> lk(mu);
                cv_done.notify_all();
            }
        }
    }
    void wait_chunk(uint32_t c)
    {
        if (remaining[c].load(std::memory_order_acquire) == 0) return;
        std::unique_lock<std::mutex> lk(mu);
        cv_done.wait(lk, [&]() { return remaining[c].load(std::memory_order_acquire) == 0; });
    }
    void release_through(uint32_t c)                                        // chunks [0, c) are free
    {
        uint32_t before;
        { std::lock_guard<std::mutex> lk(mu); before = released; released = c; }
        // chunks [before + kStageSlots, c + kStageSlots) became admissible: wake the slots they live in (at most all of them)
        const uint32_t span = c - before >= kStageSlots ? kStageSlots : c - before;
        for (uint32_t k = 0; k < span; ++k) cv_free[(before + k) % kStageSlots].notify_all();
    }
    void join()
    {
        next_col.store(n_blocks, std::memory_order_relaxed);
        release_through(0xffffffffu - kStageSlots);
        for (auto& x : th) x.join();
        th.clear();
    }
    ~PackPipeline() { if (!th.empty()) join(); }
};

}  // namespace bmb200
