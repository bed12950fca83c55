// bmb200_aggregator.hpp -- reference-side binding: bm::b200::aggregator<BV> and friends.
//
// This is the header a BitMagic maintainer adds next to src/bmaggregator.h to route the block algebra of
// bm::aggregator<> / bvector::bit_* / build_rs_index to libbmb200.so (include/bmb200.h).  It needs the
// reference headers on the include path (bm.h, bmaggregator.h) and only uses their PUBLIC block-manager API,
// exactly as aggregator itself does (src/bmaggregator.h:1196-1216):
//     get_blocks_manager(), get_block_ptr(i,j), BM_IS_GAP / BMGAP_PTR / FULL_BLOCK_FAKE_ADDR,
//     reserve_top_blocks, check_alloc_top_subblock, set_block_ptr, copy_bit_block, allocate_gap_block.
//
// Same member names, argument meaning and return values as bm::aggregator<BV>
// (src/bmaggregator.h:359-388 setters, :503-540 C-style entry points); errors from the C ABI surface as
// std::runtime_error because the reference's own methods have no error channel.
#ifndef BMB200_AGGREGATOR_HPP_INCLUDED
#define BMB200_AGGREGATOR_HPP_INCLUDED

#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <memory>
#include <stdexcept>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "bm.h"
#include "bmaggregator.h"

#include "bmb200.h"
#include "bmb200_alloc.hpp"

namespace bm { namespace b200 {

inline void check(int rc, const char* what)
{
    if (rc != BMB200_OK) throw std::runtime_error(std::string(what) + ": " + bmb200_error_msg(rc));
}

/// process-wide context for one device (the C ABI handle is thread-compatible, not thread-safe)
class context
{
public:
    explicit context(int device = 0) { check(bmb200_init(device, &ctx_), "bmb200_init"); }
    ~context() { if (ctx_) bmb200_destroy(ctx_); }
    context(const context&) = delete; context& operator=(const context&) = delete;
    bmb200_ctx* get() const { return ctx_; }
private:
    bmb200_ctx* ctx_ = nullptr;
};

namespace detail {

/// walk a bvector's block tree into the kind/pointer arrays bmb200_set_upload_vectors consumes
template<class BV>
struct tree_view
{
    std::vector<uint8_t> kind;
    std::vector<const void*> ptr;
    void build(const BV& bv, uint32_t n_blocks)
    {
        kind.assign(n_blocks, BMB200_BLK_NULL); ptr.assign(n_blocks, nullptr);
        const typename BV::blocks_manager_type& bman = bv.get_blocks_manager();
        if (!bman.is_init()) return;
        unsigned top = bman.top_block_size();
        for (uint32_t nb = 0; nb < n_blocks; ++nb)
        {
            unsigned i = nb >> bm::set_array_shift, j = nb & bm::set_array_mask;
            if (i >= top) break;
            const bm::word_t* blk = bman.get_block_ptr(i, j);
            if (!blk) continue;
            if (blk == FULL_BLOCK_FAKE_ADDR || blk == FULL_BLOCK_REAL_ADDR) { kind[nb] = BMB200_BLK_FULL; continue; }
            if (BM_IS_GAP(blk)) { kind[nb] = BMB200_BLK_GAP; ptr[nb] = BMGAP_PTR(blk); }
            else                { kind[nb] = BMB200_BLK_BIT; ptr[nb] = blk; }
        }
    }
};

template<class BV>
uint32_t blocks_of(const BV& bv)
{
    typename BV::size_type sz = bv.size();
    return (uint32_t)((uint64_t(sz) + 65535ull) >> 16);
}

/// store a fetched result (per-column flat form) into the target through the public block manager.  The target is REPLACED
/// (resize_target(init_clear = true), src/bmaggregator.h:2215-2219), but its existing blocks are recycled where the new block
/// has the same shape (a bit-block for a bit-block, a GAP block of the same capacity level for a GAP block): a repeated query into
/// the same target then costs one memcpy per block instead of a free + malloc pair.
/// Large results are stored by a few host threads, each owning whole top-level sub-trees (disjoint i): the block manager's
/// per-(i,j) calls touch nothing shared once the top array is reserved and no allocator pool is attached.
/// `landed` != 0: the blocks are still arriving (bmb200_result_fetch_view_async); every thread waits for the last column of a
/// top-level sub-tree before it reads that sub-tree's blocks, so the store of the first columns overlaps the D2H of the rest.
template<class BV>
void store_result(BV& target, typename BV::size_type new_size, uint32_t n_cols,
                  const uint8_t* kind, const uint64_t* off, const uint32_t* bits, const uint16_t* gaps, uint32_t nb_off = 0,
                  bmb200_result* landed = nullptr)
{
    typedef typename BV::blocks_manager_type bman_type;
    if (target.is_ro() || !target.get_blocks_manager().is_init() || target.size() != new_size)
    {   // nothing to recycle (or a frozen target, whose arena cannot be patched): start from an empty vector
        target.clear(true);
        target.resize(new_size);
        target.init();
    }
    bman_type& bman = target.get_blocks_manager();
    const unsigned i_lo = n_cols ? (nb_off >> bm::set_array_shift) : 1u, i_hi = n_cols ? ((nb_off + n_cols - 1u) >> bm::set_array_shift) : 0u;
    if (n_cols) bman.reserve_top_blocks(i_hi + 1);
    const unsigned top_size = bman.top_block_size();
    auto free_real = [&](bm::word_t* blk)
    {
        if (!IS_VALID_ADDR(blk)) return;
        if (BM_IS_GAP(blk)) bman.get_allocator().free_gap_block(BMGAP_PTR(blk), bman.glen());
        else bman.get_allocator().free_bit_block(blk);
    };
    auto drop_top = [&](unsigned i)              // top-level entry i holds nothing of the new result
    {
        bm::word_t** sub = bman.top_blocks_root()[i];
        if (!sub) return;
        if ((bm::word_t*)sub != FULL_BLOCK_FAKE_ADDR) for (unsigned j = 0; j < bm::set_sub_array_size; ++j) free_real(sub[j]);
        bman.free_top_subblock(i);
    };
    auto store_top = [&](unsigned i, bm::word_t* tb)
    {
        const uint32_t nb0 = std::max<uint32_t>(i << bm::set_array_shift, nb_off), nb1 = std::min<uint32_t>((i + 1u) << bm::set_array_shift, nb_off + n_cols);
        bool any = false;
        for (uint32_t nb = nb0; nb < nb1; ++nb) if (kind[nb - nb_off] != BMB200_BLK_NULL) { any = true; break; }
        if (!any) { drop_top(i); return; }
        if (landed && bmb200_result_fetch_wait(landed, nb1 - 1u - nb_off) != BMB200_OK) throw std::runtime_error("bmb200_result_fetch_wait");
        bm::word_t** sub = bman.check_alloc_top_subblock(i);        // (expands a FULL top-level entry into 256 FULL pointers)
        for (unsigned j = 0; j < bm::set_sub_array_size; ++j)
        {
            const uint32_t nb = (i << bm::set_array_shift) + j;
            const unsigned k = (nb >= nb0 && nb < nb1) ? kind[nb - nb_off] : BMB200_BLK_NULL;
            const uint32_t c = nb - nb_off;
            bm::word_t* oldp = sub[j];
            if (k == BMB200_BLK_NULL) { free_real(oldp); sub[j] = 0; }
            else if (k == BMB200_BLK_FULL) { free_real(oldp); sub[j] = FULL_BLOCK_FAKE_ADDR; }
            else if (k == BMB200_BLK_BIT)
            {
                const bm::word_t* src = bits + off[c] * (size_t)BMB200_BLOCK_WORDS;
                if (IS_VALID_ADDR(oldp) && !BM_IS_GAP(oldp)) std::memcpy(oldp, src, BMB200_BLOCK_BYTES);    // recycle the bit-block
                else
                {
                    free_real(oldp); sub[j] = 0;
                    std::memcpy(tb, src, BMB200_BLOCK_BYTES);                                              // SIMD-aligned staging for bit_block_stream
                    bman.copy_bit_block(i, j, tb);
                }
            }
            else
            {
                const bm::gap_word_t* g = gaps + off[c];
                const unsigned len = bm::gap_length(g) - 1;
                const int level = bm::gap_calc_level(len, bman.glen());
                if (IS_VALID_ADDR(oldp) && BM_IS_GAP(oldp) && int(bm::gap_level(BMGAP_PTR(oldp))) == level)
                {   // recycle the GAP block: same capacity level, so allocate_gap_block would hand out the same shape
                    bm::gap_word_t* gb = BMGAP_PTR(oldp);
                    std::memcpy(gb, g, (size_t)(len + 1) * sizeof(bm::gap_word_t));
                    *gb = (bm::gap_word_t)((len << 3) | (unsigned(level) << 1) | (*g & 1));
                }
                else
                {
                    free_real(oldp);
                    bm::gap_word_t* gb = bman.allocate_gap_block(unsigned(level), g);
                    sub[j] = (bm::word_t*)BMPTR_SETBIT0(gb);
                }
            }
        }
        if (sub[bm::set_sub_array_size - 1] == FULL_BLOCK_FAKE_ADDR) bman.validate_top_full(i);
    };
    unsigned T = 1;
    if (n_cols >= 2048u && !bman.get_allocator().get_pool())
    {
        static const unsigned want = []() { const char* e = getenv("BMB200_STORE_THREADS"); return e ? (unsigned)atoi(e) : 0u; }();
        T = want ? want : std::thread::hardware_concurrency(); if (!T) T = 1; if (T > 8 && !want) T = 8; if (T > i_hi - i_lo + 1u) T = i_hi - i_lo + 1u;
    }
    auto work = [&](unsigned t)
    {
        BM_DECLARE_TEMP_BLOCK(tb)
        for (unsigned i = t; i < top_size; i += T)
            if (n_cols && i >= i_lo && i <= i_hi) store_top(i, tb.begin()); else drop_top(i);
    };
    if (T <= 1) { work(0); return; }
    std::vector<std::thread> th;
    for (unsigned t = 1; t < T; ++t) th.emplace_back(work, t);
    work(0);
    for (auto& x : th) x.join();
}

/// walk the block trees of n vectors with a team of host threads (one vector at a time per thread); blocks [nb_from, nb_from + n_blocks)
template<class BV>
void build_views(const BV* const* vecs, size_t n, uint32_t nb_from, uint32_t n_blocks,
                 std::vector<tree_view<BV>>& views, std::vector<bmb200_vec_blocks>& vb)
{
    views.resize(n); vb.resize(n);
    unsigned T = std::thread::hardware_concurrency(); if (!T) T = 1; if (T > 32) T = 32; if (T > n) T = (unsigned)n;
    auto work = [&](unsigned t) {
        for (size_t k = t; k < n; k += T) {
            views[k].build(*vecs[k], nb_from + n_blocks);
            vb[k].n_blocks = n_blocks; vb[k].kind = views[k].kind.data() + nb_from; vb[k].ptr = views[k].ptr.data() + nb_from;
        }
    };
    if (T <= 1 || (uint64_t)n * n_blocks < (1u << 16)) { for (unsigned t = 0; t < T; ++t) work(t); return; }
    std::vector<std::thread> th;
    for (unsigned t = 0; t < T; ++t) th.emplace_back(work, t);
    for (auto& x : th) x.join();
}

} // namespace detail

namespace detail {
/// Slab-backed vectors (bmb200_alloc.hpp) reach the device by DMA of their slabs + a device gather, any other bm::bvector<>
/// through the host packing pipeline.  The DMA moves the WHOLE heap, so it is the road for sets of many vectors (the aggregator's
/// case: >= 64 here); begin() queues the copies before the block trees are walked, finish() lays the set out under them.
template<class BV>
struct set_uploader
{
    std::vector<bmb200_host_slab> slabs;
    bool use_slabs = false;
    void begin(bmb200_ctx* ctx, size_t n_vec)
    {
        use_slabs = false;
        if (!slab_backed<BV>::value || n_vec < 64) return;
        slab_heap::instance().snapshot(slabs);
        use_slabs = !slabs.empty() && bmb200_host_slabs_prefetch(ctx, slabs.data(), (uint32_t)slabs.size()) == BMB200_OK;
    }
    int finish(bmb200_ctx* ctx, uint32_t n_vec, uint32_t n_blocks, const bmb200_vec_blocks* vb, bmb200_set** set)
    {
        if (use_slabs) return bmb200_set_upload_slabs(ctx, n_vec, n_blocks, vb, slabs.data(), (uint32_t)slabs.size(), set);
        return bmb200_set_upload_vectors(ctx, n_vec, n_blocks, vb, set);
    }
};

/// Lowest set bit in [b0, b1] of result column `col` (one column read back: bmb200_result_fetch_column); 65536 when there is
/// none.  What aggregator::find_first_and_sub reads once the popcounts have located a non-empty column (src/bmaggregator.h:1538-1546).
inline unsigned result_column_first(bmb200_result* res, uint32_t col, unsigned b0 = 0u, unsigned b1 = 65535u)
{
    uint8_t kd = 0; std::vector<uint32_t> bits(BMB200_BLOCK_WORDS); std::vector<uint16_t> gaps(BMB200_GAP_MAX_WORDS);
    check(bmb200_result_fetch_column(res, col, &kd, bits.data(), gaps.data()), "bmb200_result_fetch_column");
    unsigned first = 65536u;
    if (kd == BMB200_BLK_FULL) first = b0;
    else if (kd == BMB200_BLK_BIT)
    {
        for (unsigned w = b0 >> 5; w <= (b1 >> 5) && first == 65536u; ++w)
        {
            uint32_t x = bits[w];
            if (w == (b0 >> 5)) x &= ~0u << (b0 & 31u);
            if (w == (b1 >> 5) && (b1 & 31u) != 31u) x &= (1u << ((b1 & 31u) + 1u)) - 1u;
            if (x) first = (w << 5) + (unsigned)__builtin_ctz(x);
        }
    }
    else if (kd == BMB200_BLK_GAP)
    {
        const unsigned len = gaps[0] >> 3; unsigned val = gaps[0] & 1u, start = 0;
        for (unsigned k = 1; k <= len && first == 65536u; ++k, val ^= 1u)
        {
            const unsigned end = gaps[k];
            if (val && end >= b0 && start <= b1) first = std::max(start, b0);
            start = end + 1u;
        }
    }
    return first;
}
}  // namespace detail

/// Residency: a set of bvectors uploaded ONCE (block trees walked and blocks packed by host threads, H2D pipelined -- all inside
/// bmb200_set_upload_vectors) and then addressed by bvector ADDRESS in every aggregator call that is given this set
/// (aggregator::set_device_set).  This is the upload / cache API SURVEY section 7 asks for: on an H100 the aggregation of a
/// 12 GiB set takes ~5 ms, its H2D over PCIe Gen5 ~240 ms, so repeated queries over long-lived vectors must not re-upload.
/// Validity: the copy is a snapshot.  Frozen vectors (bvector::freeze(), src/bm.h:1057) cannot change; for mutable vectors the
/// owner calls assign() again after a change.  stale() is a cheap O(1)-per-vector check (size, root pointer, top size) that
/// catches resizes and re-allocations of the tree but not in-place bit flips.
template<class BV>
class device_set
{
public:
    typedef typename BV::size_type size_type;
    explicit device_set(context& c) : ctx_(c) {}
    ~device_set() { release(); }
    device_set(const device_set&) = delete; device_set& operator=(const device_set&) = delete;

    /// (re)build the device copy from n vectors; nb_to != 0 uploads only the block columns [nb_from, nb_to) (one rank's shard)
    void assign(const BV* const* vecs, size_t n, uint32_t nb_from = 0, uint32_t nb_to = 0)
    {
        release();
        if (!n) return;
        uint32_t nblk = 0;
        for (size_t k = 0; k < n; ++k) nblk = std::max(nblk, detail::blocks_of(*vecs[k]));
        if (nb_to && nb_to < nblk) nblk = nb_to;
        if (nb_from >= nblk) throw std::range_error("device_set: empty block range");
        nb_from_ = nb_from; n_blocks_ = nblk - nb_from;
        std::vector<detail::tree_view<BV>> views; std::vector<bmb200_vec_blocks> vb;
        detail::set_uploader<BV> up;
        up.begin(ctx_.get(), n);
        detail::build_views(vecs, n, nb_from, n_blocks_, views, vb);
        check(up.finish(ctx_.get(), (uint32_t)n, n_blocks_, vb.data(), &set_), "bmb200_set_upload_vectors");
        index_.clear(); stamps_.resize(n); vecs_.assign(vecs, vecs + n);
        for (size_t k = 0; k < n; ++k) { index_.emplace(vecs[k], (uint32_t)k); stamps_[k] = stamp_of(*vecs[k]); }
    }
    void release() { if (set_) { bmb200_set_free(set_); set_ = nullptr; } index_.clear(); vecs_.clear(); stamps_.clear(); ++epoch_; }
    bool resident() const { return set_ != nullptr; }
    /// changes whenever the device copy is rebuilt or dropped (the aggregator caches its source -> member lookups against it)
    uint64_t epoch() const { return epoch_; }
    /// index of bv inside the set, or -1
    long index_of(const BV* bv) const { auto it = index_.find(bv); return it == index_.end() ? -1 : (long)it->second; }
    bool stale() const { for (size_t k = 0; k < vecs_.size(); ++k) if (!(stamps_[k] == stamp_of(*vecs_[k]))) return true; return false; }
    bmb200_set* handle() const { return set_; }
    uint32_t n_blocks() const { return n_blocks_; }
    uint32_t nb_from() const { return nb_from_; }
    size_t size() const { return vecs_.size(); }
    context& ctx() const { return ctx_; }
private:
    struct stamp { size_type size; const void* root; unsigned top; bool operator==(const stamp& o) const { return size == o.size && root == o.root && top == o.top; } };
    static stamp stamp_of(const BV& bv)
    {
        const typename BV::blocks_manager_type& bman = bv.get_blocks_manager();
        return stamp{bv.size(), bman.is_init() ? (const void*)bman.top_blocks_root() : nullptr, bman.is_init() ? bman.top_block_size() : 0u};
    }
    context& ctx_;
    bmb200_set* set_ = nullptr;
    uint32_t n_blocks_ = 0, nb_from_ = 0;
    uint64_t epoch_ = 0;
    std::unordered_map<const BV*, uint32_t> index_;
    std::vector<const BV*> vecs_;
    std::vector<stamp> stamps_;
};

/// Drop-in for bm::aggregator<BV>: combine_or / combine_and / combine_and_sub on the GPU.
template<class BV>
class aggregator
{
public:
    typedef BV bvector_type;
    typedef const bvector_type* bvector_type_const_ptr;
    typedef typename BV::size_type size_type;

    explicit aggregator(context& ctx) : ctx_(ctx) {}
    ~aggregator() { if (res_) bmb200_result_free(res_); }
    aggregator(const aggregator&) = delete; aggregator& operator=(const aggregator&) = delete;   // like the reference (src/bmaggregator.h:820)

    /// attach a resident set: calls whose sources are ALL members of it run on the device copy (no tree walk, no upload);
    /// any other call uploads its sources as before.  nullptr detaches.
    void set_device_set(const device_set<BV>* ds) { ds_ = ds; bound_ds_ = nullptr; }

    // ---- setters, same meaning as src/bmaggregator.h:359-388 ----
    void set_optimization(typename BV::optmode opt = BV::opt_compress) { opt_mode_ = opt; }
    size_t add(const bvector_type* bv, unsigned agr_group = 0)
    {
        if (agr_group > 1) throw std::range_error("agr_group");
        grp_[agr_group].push_back(bv);
        return grp_[agr_group].size();
    }
    void reset() { grp_[0].clear(); grp_[1].clear(); }

    /// aggregator::set_range_hint / reset_range_hint, src/bmaggregator.h:961-994: narrows find_first_and_sub to the blocks of
    /// [from, to]; a range inside ONE block additionally masks that block (the reference ANDs a range GAP block into it).
    /// Returns true for such a one-block range, like the reference.  (The combine_* calls of this binding ignore the hint.)
    bool set_range_hint(size_type from, size_type to)
    {
        range_set_ = true; range_from_ = from; range_to_ = to;
        return (from >> bm::set_block_shift) == (to >> bm::set_block_shift);
    }
    void reset_range_hint() { range_set_ = false; }

    /// aggregator::find_first_and_sub, src/bmaggregator.h:1078-1084, 1457-1549: index of the first bit of AND(group 0) - OR(group 1).
    /// The block columns the reference would visit (its per-top-block limits, :1513-1531, hint included) are aggregated in one
    /// launch, the first non-empty one is located from the per-column popcounts and only that column's block comes back.
    /// One deliberate difference: for a block where every AND source is FULL and there is no SUB group the reference returns the
    /// digest ~0 without writing its temp block (:1752-1759) and then reports the first bit of whatever that block held before;
    /// this binding reports the block's true first bit.
    bool find_first_and_sub(size_type& idx) { return find_first_and_sub(idx, grp_[0].data(), grp_[0].size(), grp_[1].data(), grp_[1].size()); }
    bool find_first_and_sub(size_type& idx, const bvector_type_const_ptr* src_and, size_t n_and,
                            const bvector_type_const_ptr* src_sub, size_t n_sub)
    {
        // -- which block columns does the reference look at? --
        unsigned top_blocks = std::max(max_top_blocks(src_and, n_and), max_top_blocks(src_sub, n_sub));
        const uint64_t nb_f = range_set_ ? (uint64_t)(range_from_ >> bm::set_block_shift) : 0u,
                       nb_t = range_set_ ? (uint64_t)(range_to_ >> bm::set_block_shift) : 0u;
        const bool one_block = range_set_ && nb_f == nb_t;
        std::vector<std::pair<uint32_t, uint32_t>> spans;          // [first, last) block columns, ascending
        if (one_block) spans.emplace_back((uint32_t)nb_f, (uint32_t)nb_f + 1u);
        else
        {
            unsigned top_from = 0;
            const unsigned top_to = (unsigned)(nb_t >> bm::set_array_shift);
            if (range_set_) { top_from = (unsigned)(nb_f >> bm::set_array_shift); if (top_to < top_blocks) top_blocks = top_to + 1u; }
            for (unsigned i = top_from; i < top_blocks; ++i)
            {
                unsigned j = 0, jmax = bm::set_sub_array_size;
                if (range_set_)
                {
                    if (i == top_from) j = (unsigned)(nb_f & bm::set_array_mask);
                    if (i == top_to) jmax = 1u + (unsigned)(nb_t & bm::set_array_mask);
                }
                else
                {
                    jmax = effective_sub_size(i, src_and, n_and, true);
                    if (!jmax) continue;
                    if (n_sub)
                    {   // (the reference narrows the scan to the SUB group's extent here and questions it itself, :1524-1530)
                        unsigned j2 = effective_sub_size(i, src_sub, n_sub, false);
                        if (j2 < jmax) jmax = j2;
                    }
                }
                if (j < jmax) spans.emplace_back((i << bm::set_array_shift) + j, (i << bm::set_array_shift) + jmax);
            }
        }
        if (!n_and || spans.empty()) return false;
        // -- one aggregation over the hull of those columns, bit-blocks kept (no re-compression: only one block is read) --
        bool own = false;
        bmb200_set* set = bind(src_and, n_and, src_sub, n_sub, own);
        struct release { bmb200_set* s; ~release() { if (s) bmb200_set_free(s); } } guard{own ? set : nullptr};
        uint32_t lo = spans.front().first, hi = spans.back().second;
        const uint32_t have_lo = nb_off_, have_hi = nb_off_ + n_blocks_;
        if (hi > have_hi) hi = have_hi;
        if (lo < have_lo) lo = have_lo;
        if (lo >= hi) return false;
        bmb200_agg_args a{BMB200_OP_AND_SUB, BMB200_F_OPT_NONE, g0_.data(), (uint32_t)n_and, n_sub ? g1_.data() : nullptr, (uint32_t)n_sub,
                          lo - nb_off_, hi - nb_off_};
        bmb200_result* res = nullptr;
        check(bmb200_aggregate(ctx_.get(), set, &a, &res), "bmb200_aggregate(find_first)");
        struct drop { bmb200_result* r; ~drop() { if (r) bmb200_result_free(r); } } rguard{res};
        std::vector<uint32_t> pop(hi - lo);
        bmb200_result_meta m{}; m.popcnt = pop.data();
        check(bmb200_result_fetch_meta(res, &m), "bmb200_result_fetch_meta");
        for (const auto& sp : spans)
            for (uint32_t nb = std::max(sp.first, lo); nb < std::min(sp.second, hi); ++nb)
            {
                if (!pop[nb - lo]) continue;
                unsigned b0 = one_block ? (unsigned)(range_from_ & bm::set_block_mask) : 0u,
                         b1 = one_block ? (unsigned)(range_to_ & bm::set_block_mask) : 65535u;
                const unsigned first = detail::result_column_first(res, nb - lo, b0, b1);
                if (first != 65536u) { idx = (size_type)((uint64_t)nb * 65536u + first); return true; }
                if (one_block) return false;
            }
        return false;
    }

    // ---- member forms ----
    void combine_or(bvector_type& target)  { combine_or(target, grp_[0].data(), grp_[0].size()); }
    void combine_and(bvector_type& target)
    {   // member combine_and routes through combine_and_sub with an empty SUB group, src/bmaggregator.h:1030-1039
        combine_and_sub(target, grp_[0].data(), grp_[0].size(), 0, 0, false);
    }
    bool combine_and_sub(bvector_type& target)
    {
        return combine_and_sub(target, grp_[0].data(), grp_[0].size(), grp_[1].data(), grp_[1].size(), false);
    }

    // ---- C-style forms, src/bmaggregator.h:503-540 ----
    void combine_or(bvector_type& target, const bvector_type_const_ptr* src, size_t n)
    {
        if (!n) { target.clear(); return; }                       // :1105-1109
        std::vector<const BV*> local(src, src + n);
        reset();                                                  // the reference drops the attached groups here (ag_.reset(), :1111)
        run(target, BMB200_OP_OR, local.data(), n, 0, 0, opt_mode_ != BV::opt_none);
    }
    void combine_and(bvector_type& target, const bvector_type_const_ptr* src, size_t n)
    {
        if (n == 1) { target = *src[0]; return; }                 // :1132-1137
        if (!n) { target.clear(); return; }
        std::vector<const BV*> local(src, src + n);
        reset();                                                  // ag_.reset(), :1143
        run(target, BMB200_OP_AND, local.data(), n, 0, 0, opt_mode_ != BV::opt_none);
    }
    /// N-way XOR (bvector::bit_xor chained, src/bm.h:6072); not a member of the reference aggregator
    void combine_xor(bvector_type& target, const bvector_type_const_ptr* src, size_t n)
    {
        if (!n) { target.clear(); return; }
        run(target, BMB200_OP_XOR, src, n, 0, 0, opt_mode_ != BV::opt_none);
    }
    /// template<class TPipe> void combine_and_sub(TPipe&), src/bmaggregator.h:427
    template<class TPipe> void combine_and_sub(TPipe& pipe) { pipe.run(); }
    bool combine_and_sub(bvector_type& target,
                         const bvector_type_const_ptr* src_and, size_t n_and,
                         const bvector_type_const_ptr* src_sub, size_t n_sub, bool any)
    {
        (void)any;   // any=true only promises the boolean (:1202-1213); the full result is computed here
        if (!src_and || !n_and) { target.clear(); return false; } // :1170-1174
        return run(target, BMB200_OP_AND_SUB, src_and, n_and, src_sub, n_sub, true /* always opt_compress, :1209 */);
    }

    /// aggregator::combine_shift_right_and, src/bmaggregator.h:473,552,2494-2530: T_0 = v_0, T_k = (T_{k-1} >> 1) & v_k
    void combine_shift_right_and(bvector_type& target)
    { combine_shift_right_and(target, grp_[0].data(), grp_[0].size(), false); }
    bool combine_shift_right_and(bvector_type& target, const bvector_type_const_ptr* src_and, size_t n_and, bool any)
    {
        (void)any;
        if (!n_and) { target.clear(); return false; }             // :2499-2503
        spare_blocks_ = 1;    // bits carried out of the last source block land in the next one (:2506-2511 keeps walking)
        bool found = run(target, BMB200_OP_SHIFT_R_AND, src_and, n_and, 0, 0, opt_mode_ != BV::opt_none);
        spare_blocks_ = 0;
        return found;
    }

    /// device-side result of the last combine_* call (valid until the next one); used by sharded_aggregator for the exchange
    bmb200_result* last_result() const { return res_; }
    /// bytes the last combine_* call read back from the device (column kinds + lengths + the result blocks themselves)
    uint64_t last_d2h_bytes() const { return last_d2h_; }

    /// popcount of AND-SUB without materialising the result (pipeline counts mode, :1397-1398)
    size_type count_and_sub(const bvector_type_const_ptr* src_and, size_t n_and,
                            const bvector_type_const_ptr* src_sub, size_t n_sub)
    {
        if (!n_and) return 0;
        bool own = false;
        bmb200_set* set = bind(src_and, n_and, src_sub, n_sub, own);
        bmb200_agg_args a{BMB200_OP_AND_SUB, BMB200_F_COUNT_ONLY, g0_.data(), (uint32_t)n_and, g1_.data(), (uint32_t)n_sub, 0, 0};
        bmb200_result* res = nullptr;
        int rc = bmb200_aggregate(ctx_.get(), set, &a, &res);
        uint64_t total = 0; int any = 0;
        if (!rc) rc = bmb200_result_total(res, &total, &any);
        if (res) bmb200_result_free(res);
        if (own) bmb200_set_free(set);
        check(rc, "bmb200_aggregate(count)");
        return (size_type)total;
    }

private:
    /// aggregator::max_top_blocks, src/bmaggregator.h:2256-2273
    static unsigned max_top_blocks(const bvector_type_const_ptr* src, size_t n)
    {
        unsigned top = 1;
        for (size_t k = 0; k < n; ++k) if (src[k]) top = std::max(top, (unsigned)src[k]->get_blocks_manager().top_block_size());
        return top;
    }
    /// aggregator::find_effective_sub_block_size, src/bmaggregator.h:1556-1599 (approximate there too: 256 for more than 32 sources)
    static unsigned effective_sub_size(unsigned i, const bvector_type_const_ptr* src, size_t n, bool top_null_as_zero)
    {
        if (n > 32) return bm::set_sub_array_size;
        unsigned max_size = 1;
        for (size_t k = 0; k < n; ++k)
        {
            const typename BV::blocks_manager_type& bman = src[k]->get_blocks_manager();
            const bm::word_t* const* sub = bman.get_topblock(i);
            if (!sub) { if (top_null_as_zero) return 0; continue; }
            if ((bm::word_t*)sub == FULL_BLOCK_FAKE_ADDR) return bm::set_sub_array_size;
            for (unsigned j = bm::set_sub_array_size - 1; j > max_size; --j) if (sub[j]) { max_size = j; break; }
            if (max_size == bm::set_sub_array_size - 1) break;
        }
        return max_size + 1;
    }

    /// sources -> (set, member indices): the attached resident set when every source lives in it, else a fresh upload
    bmb200_set* bind(const bvector_type_const_ptr* s0, size_t n0, const bvector_type_const_ptr* s1, size_t n1, bool& own)
    {
        // the same source lists against the same resident copy as the previous call (a query loop over long-lived vectors): the
        // member ids, block count and target size of that call still hold -- 16384 hash lookups and size() reads are ~1 ms
        if (ds_ && ds_->resident() && !spare_blocks_ && bound_ds_ == ds_ && bound_epoch_ == ds_->epoch() && bound_n0_ == n0 &&
            bound_.size() == n0 + n1 && (!n0 || !memcmp(bound_.data(), s0, n0 * sizeof(*s0))) &&
            (!n1 || !memcmp(bound_.data() + n0, s1, n1 * sizeof(*s1))))
        { own = false; return ds_->handle(); }
        bound_ds_ = nullptr;
        g0_.resize(n0); g1_.resize(n1);
        max_size_ = 0;
        for (size_t k = 0; k < n0 + n1; ++k)
        {
            const BV* bv = k < n0 ? s0[k] : s1[k - n0];
            if (bv->size() > max_size_) max_size_ = bv->size();   // resize_target: max over sources, :2238-2248
        }
        if (ds_ && ds_->resident() && !spare_blocks_)
        {
            bool all = true;
            for (size_t k = 0; k < n0 + n1 && all; ++k)
            {
                long ix = ds_->index_of(k < n0 ? s0[k] : s1[k - n0]);
                if (ix < 0) all = false; else (k < n0 ? g0_[k] : g1_[k - n0]) = (uint32_t)ix;
            }
            if (all)
            {
                own = false; n_blocks_ = ds_->n_blocks(); nb_off_ = ds_->nb_from();
                bound_.assign(s0, s0 + n0); bound_.insert(bound_.end(), s1, s1 + n1);
                bound_ds_ = ds_; bound_epoch_ = ds_->epoch(); bound_n0_ = n0;
                return ds_->handle();
            }
        }
        for (size_t k = 0; k < n0; ++k) g0_[k] = (uint32_t)k;
        for (size_t k = 0; k < n1; ++k) g1_[k] = (uint32_t)(n0 + k);
        own = true; nb_off_ = 0;
        return upload(s0, n0, s1, n1);
    }

    bmb200_set* upload(const bvector_type_const_ptr* s0, size_t n0, const bvector_type_const_ptr* s1, size_t n1)
    {
        n_blocks_ = 0;
        std::vector<const BV*> all(n0 + n1);
        for (size_t k = 0; k < n0 + n1; ++k)
        {
            all[k] = k < n0 ? s0[k] : s1[k - n0];
            uint32_t nb = detail::blocks_of(*all[k]);
            if (nb > n_blocks_) n_blocks_ = nb;
        }
        if (spare_blocks_ && n_blocks_ < 65536u) n_blocks_ += spare_blocks_;
        detail::set_uploader<BV> up;
        up.begin(ctx_.get(), n0 + n1);
        detail::build_views(all.data(), all.size(), 0u, n_blocks_, views_, vb_);
        bmb200_set* set = nullptr;
        check(up.finish(ctx_.get(), (uint32_t)(n0 + n1), n_blocks_, vb_.data(), &set), "bmb200_set_upload_vectors");
        return set;
    }

    bool run(bvector_type& target, int op, const bvector_type_const_ptr* s0, size_t n0,
             const bvector_type_const_ptr* s1, size_t n1, bool compress)
    {
        static const bool trace = getenv("BMB200_TRACE") != nullptr;
        auto now = []() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
        const double t0 = trace ? now() : 0;
        bool own = false;
        bmb200_set* set = bind(s0, n0, s1, n1, own);
        const double t1 = trace ? now() : 0;
        bmb200_agg_args a{op, compress ? BMB200_F_OPT_COMPRESS : BMB200_F_OPT_NONE,
                          g0_.data(), (uint32_t)n0, n1 ? g1_.data() : nullptr, (uint32_t)n1, 0, 0};
        // the result object (device buffers for every column) is recycled from call to call; the fetched blocks arrive in pinned
        // memory owned by the context (bmb200_result_fetch_view): a warm call allocates nothing on either side
        // The blocks come back in column chunks (bmb200_result_fetch_view_async): the store of the first columns runs under the
        // D2H of the rest.  Whatever happens, nothing stays in flight and a per-call set is freed when this scope ends.
        struct drain { bmb200_result*& r; uint32_t last; bmb200_set* set;
                       ~drain() { if (r) bmb200_result_fetch_wait(r, last); if (set) bmb200_set_free(set); } }
            guard{res_, n_blocks_ ? n_blocks_ - 1u : 0u, own ? set : nullptr};
        int rc = bmb200_aggregate(ctx_.get(), set, &a, &res_);
        uint64_t total = 0, nb = 0, ng = 0;
        const uint8_t* kind = nullptr; const uint64_t* off = nullptr; const uint32_t* bits = nullptr; const uint16_t* gaps = nullptr;
        if (!rc) rc = bmb200_result_fetch_view_async(res_, &kind, &off, &bits, &gaps, &nb, &ng, &total);
        check(rc, "bmb200_aggregate");
        last_d2h_ = (uint64_t)n_blocks_ * 5u + 8u + nb * (uint64_t)BMB200_BLOCK_BYTES + ng * 2u;
        const double t2 = trace ? now() : 0;
        detail::store_result(target, max_size_, n_blocks_, kind, off, bits, gaps, nb_off_, res_);
        if (trace) fprintf(stderr, "[bmb200] aggregator::run: bind %.3f ms, aggregate + fetch (%llu bit-blocks, %llu GAP words) %.3f ms, store into the target %.3f ms\n",
                           t1 - t0, (unsigned long long)nb, (unsigned long long)ng, t2 - t1, now() - t2);
        return total != 0;
    }

    context& ctx_;
    typename BV::optmode opt_mode_ = BV::opt_none;
    std::vector<const BV*> grp_[2];
    std::vector<detail::tree_view<BV>> views_;
    std::vector<bmb200_vec_blocks> vb_;
    std::vector<uint32_t> g0_, g1_;
    const device_set<BV>* ds_ = nullptr;
    const device_set<BV>* bound_ds_ = nullptr;       // bind() cache: source list of the last call that ran on ds_
    std::vector<const BV*> bound_;
    uint64_t bound_epoch_ = 0;
    size_t bound_n0_ = 0;
    uint64_t last_d2h_ = 0;
    bool range_set_ = false;
    size_type range_from_ = 0, range_to_ = 0;
    bmb200_result* res_ = nullptr;
    uint32_t n_blocks_ = 0, nb_off_ = 0;
    uint32_t spare_blocks_ = 0;
    size_type max_size_ = 0;
};

/// One rank of a block-range sharded aggregation (one process per GPU; SURVEY 8e, BASELINE config 5): this rank keeps the block
/// columns [from, to) of EVERY vector resident on its GPU, aggregates them locally with the same kernels, and the ranks exchange
/// per-column popcounts + cardinalities with one ncclAllGather (bmb200_exchange_popcounts).  Result blocks never move: the target
/// of a combine_* call holds this rank's block range only.  The 128-byte communicator id comes from rank 0
/// (sharded_aggregator::unique_id) and travels to the other ranks by whatever the application uses (MPI, sockets, files).
template<class BV>
class sharded_aggregator
{
public:
    typedef typename BV::size_type size_type;
    static void unique_id(void* id128) { check(bmb200_comm_unique_id(id128), "bmb200_comm_unique_id"); }
    sharded_aggregator(context& c, int nranks, int rank, const void* id128) : ctx_(c), agg_(c), ds_(c), nranks_(nranks), rank_(rank)
    { check(bmb200_comm_init(c.get(), nranks, rank, id128), "bmb200_comm_init"); }
    ~sharded_aggregator() { ds_.release(); bmb200_comm_destroy(ctx_.get()); }
    void set_optimization(typename BV::optmode opt = BV::opt_compress) { agg_.set_optimization(opt); }

    /// upload this rank's shard of the vectors (they stay resident until the next assign)
    void assign(const BV* const* vecs, size_t n)
    {
        uint32_t nblk = 0;
        for (size_t k = 0; k < n; ++k) nblk = std::max(nblk, detail::blocks_of(*vecs[k]));
        n_blocks_ = nblk; widest_ = 0;
        for (int r = 0; r < nranks_; ++r) { uint32_t a, b; check(bmb200_shard_range(nblk, nranks_, r, &a, &b), "bmb200_shard_range"); widest_ = std::max(widest_, b - a); }
        check(bmb200_shard_range(nblk, nranks_, rank_, &from_, &to_), "bmb200_shard_range");
        if (to_ > from_) ds_.assign(vecs, n, from_, to_); else ds_.release();
        agg_.set_device_set(&ds_);
    }
    /// transport of the exchange: 1 = ncclAllGather, 0 = nothing exchanged yet
    int exchange_mode() const { int m = 0; bmb200_exchange_mode(ctx_.get(), &m); return m; }
    uint32_t shard_from() const { return from_; }
    uint32_t shard_to() const { return to_; }

    /// same contracts as aggregator<BV>; sources must be members of the assigned set
    void combine_or(BV& target, const BV* const* src, size_t n) { agg_.combine_or(target, src, n); exchange(); }
    void combine_and(BV& target, const BV* const* src, size_t n) { agg_.combine_and(target, src, n); exchange(); }
    bool combine_and_sub(BV& target, const BV* const* src_and, size_t n_and, const BV* const* src_sub, size_t n_sub)
    { agg_.combine_and_sub(target, src_and, n_and, src_sub, n_sub, false); exchange(); return count() != 0; }

    /// global cardinality of the last result (sum over all ranks)
    uint64_t count() { fetch(); return total_; }
    /// per-column popcounts of the whole result, all shards concatenated in block order: [n_blocks]
    const std::vector<uint32_t>& block_popcounts() { fetch(); return pop_; }
private:
    void exchange()
    {
        fetched_ = false;
        if (!agg_.last_result()) throw std::logic_error("sharded_aggregator: no device result (empty source list?)");
        check(bmb200_exchange_popcounts(agg_.last_result(), widest_), "bmb200_exchange_popcounts");
    }
    void fetch()
    {
        if (fetched_) return;
        std::vector<uint32_t> all((size_t)nranks_ * widest_);
        check(bmb200_exchange_fetch(ctx_.get(), &total_, nullptr, all.data(), nullptr, nullptr), "bmb200_exchange_fetch");
        pop_.assign(n_blocks_, 0u);
        for (int r = 0; r < nranks_; ++r) { uint32_t a, b; bmb200_shard_range(n_blocks_, nranks_, r, &a, &b);
                                            std::copy(all.begin() + (size_t)r * widest_, all.begin() + (size_t)r * widest_ + (b - a), pop_.begin() + a); }
        fetched_ = true;
    }
    context& ctx_;
    aggregator<BV> agg_;
    device_set<BV> ds_;
    int nranks_, rank_;
    uint32_t n_blocks_ = 0, from_ = 0, to_ = 0, widest_ = 0;
    uint64_t total_ = 0; std::vector<uint32_t> pop_; bool fetched_ = true;
};

/// Drop-in for aggregator::pipeline<agg_opt_bvect_and_counts> + aggregator::combine_and_sub(TPipe&)
/// (src/bmaggregator.h:222-341, 1291-1453): every argument group of the pipeline runs in ONE batched launch
/// (bmb200_aggregate_batch); unique input vectors are uploaded once (the reference's pipeline_bcache).
template<class BV>
class pipeline
{
public:
    typedef typename BV::size_type size_type;
    struct arg_groups
    {
        std::vector<const BV*> arg_bv0, arg_bv1;
        size_t add(const BV* bv, unsigned agr_group) { (agr_group ? arg_bv1 : arg_bv0).push_back(bv); return (agr_group ? arg_bv1 : arg_bv0).size(); }
    };
    explicit pipeline(context& c) : ctx_(c) {}
    ~pipeline() { for (BV* p : bv_res_) delete p; }
    pipeline(const pipeline&) = delete; pipeline& operator=(const pipeline&) = delete;

    arg_groups* add() { args_.emplace_back(new arg_groups()); return args_.back().get(); }
    void set_or_target(BV* bv_or) { bv_or_ = bv_or; }
    void complete() { complete_ = true; }
    bool is_complete() const { return complete_; }
    size_type size() const { return (size_type)args_.size(); }
    std::vector<BV*>& get_bv_res_vector() { return bv_res_; }                 ///< null for an empty result, like the reference
    std::vector<size_type>& get_bv_count_vector() { return count_res_; }

    /// aggregator::combine_and_sub(TPipe&)
    void run()
    {
        if (!complete_) throw std::logic_error("pipeline::complete() not called");
        for (BV* p : bv_res_) delete p;
        const size_t ng = args_.size();
        bv_res_.assign(ng, nullptr); count_res_.assign(ng, 0);
        std::vector<const BV*> uniq; std::vector<uint32_t> members, offsets(1, 0u);
        auto index_of = [&](const BV* bv) -> uint32_t {
            for (size_t k = 0; k < uniq.size(); ++k) if (uniq[k] == bv) return (uint32_t)k;
            uniq.push_back(bv); return (uint32_t)(uniq.size() - 1);
        };
        for (auto& a : args_) {
            for (const BV* bv : a->arg_bv0) members.push_back(index_of(bv));
            offsets.push_back((uint32_t)members.size());
            for (const BV* bv : a->arg_bv1) members.push_back(index_of(bv));
            offsets.push_back((uint32_t)members.size());
        }
        if (!ng || uniq.empty()) return;
        uint32_t n_blocks = 0; size_type max_size = 0;
        for (const BV* bv : uniq) { n_blocks = std::max(n_blocks, detail::blocks_of(*bv)); if (bv->size() > max_size) max_size = bv->size(); }
        std::vector<detail::tree_view<BV>> views(uniq.size()); std::vector<bmb200_vec_blocks> vb(uniq.size());
        for (size_t k = 0; k < uniq.size(); ++k) {
            views[k].build(*uniq[k], n_blocks);
            vb[k].n_blocks = n_blocks; vb[k].kind = views[k].kind.data(); vb[k].ptr = views[k].ptr.data();
        }
        bmb200_set* set = nullptr;
        check(bmb200_set_upload_vectors(ctx_.get(), (uint32_t)uniq.size(), n_blocks, vb.data(), &set), "bmb200_set_upload_vectors");
        bmb200_batch_args a{BMB200_OP_AND_SUB, BMB200_F_OPT_COMPRESS | (bv_or_ ? BMB200_F_OR_TARGET : 0u), (uint32_t)ng,
                            members.data(), offsets.data(), 0, 0};
        bmb200_result* res = nullptr; bmb200_result* ores = nullptr;
        int rc = bmb200_aggregate_batch(ctx_.get(), set, &a, &res);
        std::vector<uint64_t> totals(ng);
        const size_t ncols = (size_t)ng * n_blocks;
        std::vector<uint8_t> kind(ncols); std::vector<uint64_t> off(ncols); std::vector<uint32_t> bits; std::vector<uint16_t> gaps;
        if (!rc) rc = bmb200_result_group_totals(res, totals.data(), (uint32_t)ng);
        if (!rc) { uint64_t nb = 0, ngw = 0; rc = bmb200_result_sizes(res, &nb, &ngw);
                   if (!rc) { bits.resize(nb * BMB200_BLOCK_WORDS); gaps.resize(ngw);
                              rc = bmb200_result_fetch(res, kind.data(), off.data(), bits.data(), gaps.data()); } }
        std::vector<uint8_t> okind(n_blocks); std::vector<uint64_t> ooff(n_blocks); std::vector<uint32_t> obits; std::vector<uint16_t> ogaps;
        if (!rc && bv_or_) {
            rc = bmb200_result_or_target(res, &ores);
            if (!rc) { uint64_t nb = 0, ngw = 0; rc = bmb200_result_sizes(ores, &nb, &ngw);
                       if (!rc) { obits.resize(nb * BMB200_BLOCK_WORDS); ogaps.resize(ngw);
                                  rc = bmb200_result_fetch(ores, okind.data(), ooff.data(), obits.data(), ogaps.data()); } }
        }
        if (ores) bmb200_result_free(ores);
        if (res) bmb200_result_free(res);
        bmb200_set_free(set);
        check(rc, "bmb200_aggregate_batch");
        for (size_t g = 0; g < ng; ++g) {
            count_res_[g] = (size_type)totals[g];
            if (!totals[g]) continue;
            bv_res_[g] = new BV();
            detail::store_result(*bv_res_[g], max_size, n_blocks, kind.data() + g * n_blocks, off.data() + g * n_blocks, bits.data(), gaps.data());
        }
        if (bv_or_) {     // the reference ORs into the caller's vector (combine_operation_block_or); same here
            BV tmp; detail::store_result(tmp, max_size, n_blocks, okind.data(), ooff.data(), obits.data(), ogaps.data());
            bv_or_->bit_or(tmp);
        }
    }
private:
    context& ctx_;
    std::vector<std::unique_ptr<arg_groups>> args_;
    std::vector<BV*> bv_res_;
    std::vector<size_type> count_res_;
    BV* bv_or_ = nullptr;
    bool complete_ = false;
};

/// 3-operand bvector ops (src/bm.h:1745-1850): target = a OP b through bmb200_binop.  Every result block gets the KIND the
/// reference's combine_operation_block_* gives it (src/bm.h:6945-7380): a NULL / FULL argument clones the other block in its own
/// kind, GAP x GAP is merged as run lists on the device (no 8 KB expansion), GAP x bit / bit x bit yield a bit-block that only
/// opt_compress re-classifies -- so calc_stat() of the target equals the reference's, not just compare() == 0.
/// `ds` (optional): a resident device_set holding both operands; otherwise they are uploaded for this call.
template<class BV>
void binop(context& c, int op, BV& t, const BV& a, const BV& b, typename BV::optmode opt = BV::opt_none, const device_set<BV>* ds = nullptr)
{
    if (&a == &b) { if (op == BMB200_OP_AND || op == BMB200_OP_OR) t = a; else t.clear(true); return; }   // src/bm.h:6190, 5978
    const BV* both[2] = {&a, &b};
    uint32_t ia = 0, ib = 1, n_blocks = 0, nb_off = 0; bmb200_set* set = nullptr; bool own = true;
    if (ds && ds->resident() && ds->index_of(&a) >= 0 && ds->index_of(&b) >= 0)
    { set = ds->handle(); ia = (uint32_t)ds->index_of(&a); ib = (uint32_t)ds->index_of(&b); n_blocks = ds->n_blocks(); nb_off = ds->nb_from(); own = false; }
    else
    {
        n_blocks = std::max(detail::blocks_of(a), detail::blocks_of(b));
        if (!n_blocks) { t.clear(true); return; }
        std::vector<detail::tree_view<BV>> views; std::vector<bmb200_vec_blocks> vb;
        detail::build_views(both, 2, 0u, n_blocks, views, vb);
        check(bmb200_set_upload_vectors(c.get(), 2, n_blocks, vb.data(), &set), "bmb200_set_upload_vectors");
    }
    bmb200_result* res = nullptr;
    int rc = bmb200_binop(c.get(), set, op, ia, ib, opt == BV::opt_compress ? BMB200_F_OPT_COMPRESS : BMB200_F_OPT_NONE, 0, 0, &res);
    uint64_t total = 0, nb = 0, ng = 0;
    const uint8_t* kind = nullptr; const uint64_t* off = nullptr; const uint32_t* bits = nullptr; const uint16_t* gaps = nullptr;
    if (!rc) rc = bmb200_result_fetch_view(res, &kind, &off, &bits, &gaps, &nb, &ng, &total);
    typename BV::size_type sz = std::max(a.size(), b.size());
    if (!rc) detail::store_result(t, sz, n_blocks, kind, off, bits, gaps, nb_off);
    if (res) bmb200_result_free(res);
    if (own) bmb200_set_free(set);
    check(rc, "bmb200_binop");
}
template<class BV> void bit_or (context& c, BV& t, const BV& a, const BV& b, typename BV::optmode opt = BV::opt_none) { binop(c, BMB200_OP_OR, t, a, b, opt); }
template<class BV> void bit_and(context& c, BV& t, const BV& a, const BV& b, typename BV::optmode opt = BV::opt_none) { binop(c, BMB200_OP_AND, t, a, b, opt); }
template<class BV> void bit_sub(context& c, BV& t, const BV& a, const BV& b, typename BV::optmode opt = BV::opt_none) { binop(c, BMB200_OP_SUB, t, a, b, opt); }
template<class BV> void bit_xor(context& c, BV& t, const BV& a, const BV& b, typename BV::optmode opt = BV::opt_none) { binop(c, BMB200_OP_XOR, t, a, b, opt); }

/// Operands that arrive as serialization BLOBs (bm::serializer<BV> output, any compression level incl. the default 6): the BLOBs
/// are decoded ON THE GPU (bmb200_set_upload_blobs) and aggregated there -- the bvectors are never materialised on the host.
/// Reference equivalent: bm::deserialize(bv_k, buf_k) for every operand (src/bmserial.h:4152) followed by
/// aggregator::combine_or / combine_and_sub (src/bmaggregator.h:1101,1162); bm::operation_deserializer<BV> (src/bmserial.h:1070)
/// is the reference's own one-BLOB-at-a-time form of "operate on a BLOB without keeping the vector".
/// `size` = size() of the serialized vectors (the result is resized to it, like resize_target does with max(source sizes)).
template<class BV>
class blob_aggregator
{
public:
    typedef typename BV::size_type size_type;
    blob_aggregator(context& c, size_type size) : ctx_(c), size_(size), n_blocks_((uint32_t)((uint64_t(size) + 65535ull) >> 16)) {}
    void set_optimization(typename BV::optmode opt = BV::opt_compress) { opt_mode_ = opt; }
    /// attach a BLOB (not owned) to group 0 (OR / AND sources) or group 1 (SUB sources), like aggregator::add(bv, group)
    size_t add(const unsigned char* buf, size_t buf_size, unsigned group = 0) { bmb200_blob b{buf, (uint64_t)buf_size}; grp_[group ? 1 : 0].push_back(b); return grp_[group ? 1 : 0].size(); }
    void reset() { grp_[0].clear(); grp_[1].clear(); }
    void combine_or(BV& target) { run(target, BMB200_OP_OR, false); }
    void combine_and(BV& target) { run(target, BMB200_OP_AND_SUB, true); }
    bool combine_and_sub(BV& target) { return run(target, BMB200_OP_AND_SUB, true); }
private:
    bool run(BV& target, int op, bool use_sub)
    {
        const size_t n0 = grp_[0].size(), n1 = use_sub ? grp_[1].size() : 0;
        if (!n0) { target.clear(true); return false; }
        std::vector<bmb200_blob> all(grp_[0]); if (n1) all.insert(all.end(), grp_[1].begin(), grp_[1].end());
        bmb200_set* set = nullptr;
        check(bmb200_set_upload_blobs(ctx_.get(), (uint32_t)all.size(), n_blocks_, all.data(), &set), "bmb200_set_upload_blobs");
        std::vector<uint32_t> g0(n0), g1(n1);
        for (size_t k = 0; k < n0; ++k) g0[k] = (uint32_t)k;
        for (size_t k = 0; k < n1; ++k) g1[k] = (uint32_t)(n0 + k);
        const bool compress = (op == BMB200_OP_AND_SUB) || opt_mode_ != BV::opt_none;      // combine_and_sub always stores through opt_compress (:1209)
        bmb200_agg_args a{op, compress ? BMB200_F_OPT_COMPRESS : BMB200_F_OPT_NONE, g0.data(), (uint32_t)n0, n1 ? g1.data() : nullptr, (uint32_t)n1, 0, 0};
        bmb200_result* res = nullptr;
        int rc = bmb200_aggregate(ctx_.get(), set, &a, &res);
        uint64_t total = 0; int any = 0, rc2 = 0;
        std::vector<uint8_t> kind(n_blocks_); std::vector<uint64_t> off(n_blocks_);
        std::vector<uint32_t> bits; std::vector<uint16_t> gaps;
        if (!rc) rc = bmb200_result_total(res, &total, &any);
        if (!rc) { uint64_t nb = 0, ng = 0; rc = bmb200_result_sizes(res, &nb, &ng);
                   if (!rc) { bits.resize(nb * BMB200_BLOCK_WORDS); gaps.resize(ng);
                              rc = bmb200_result_fetch(res, kind.data(), off.data(), bits.data(), gaps.data()); } }
        if (res) rc2 = bmb200_result_free(res);
        bmb200_set_free(set);
        check(rc, "bmb200_aggregate"); check(rc2, "bmb200_result_free");
        detail::store_result(target, size_, n_blocks_, kind.data(), off.data(), bits.data(), gaps.data());
        return any != 0;
    }
    context& ctx_;
    size_type size_;
    uint32_t n_blocks_;
    typename BV::optmode opt_mode_ = BV::opt_none;
    std::vector<bmb200_blob> grp_[2];
};

/// bvector::bit_or_and (src/bm.h:1787,6283): target |= a & b -- two launches (AND, then OR with the target)
template<class BV> void bit_or_and(context& c, BV& t, const BV& a, const BV& b, typename BV::optmode opt = BV::opt_none)
{
    BV tmp; bit_and(c, tmp, a, b, opt);
    BV res; aggregator<BV> g(c); g.set_optimization(opt); const BV* s[2] = {&t, &tmp}; g.combine_or(res, s, 2);
    t.swap(res);
}
/// bvector::merge (src/bm.h:1000,5883): t |= src; the reference may steal src's blocks, so src is left cleared here too
template<class BV> void merge(context& c, BV& t, BV& src)
{
    BV res; aggregator<BV> g(c); const BV* s[2] = {&t, &src}; g.combine_or(res, s, 2);
    t.swap(res); src.clear(true);
}

/// build_rs_index on the GPU, delivered through rs_index's own public mutators
/// (resize / set_total / set_null_super_block / set_full_super_block / register_super_block,
///  src/bmrs.h:70-113) so the unmodified reference query code (count_to / select) can use it.
template<class BV>
void build_rs_index(context& c, const BV& bv, typename BV::rs_index_type* rs)
{
    rs->init();
    if (!bv.get_blocks_manager().is_init()) return;
    typename BV::size_type last;
    if (!bv.find_reverse(last)) return;
    const typename BV::blocks_manager_type& bman = bv.get_blocks_manager();
    unsigned real_top = bman.find_real_top_blocks(), max_top = bman.find_max_top_blocks();
    uint64_t nb = uint64_t(last) >> 16;
    if (nb < uint64_t(max_top) * 256u) nb = uint64_t(max_top) * 256u;          // src/bm.h:2556-2559
    rs->set_total((typename BV::block_idx_type)(nb + 1));
    rs->resize((typename BV::block_idx_type)(nb + 1));
    rs->resize_effective_super_blocks(real_top);
    uint32_t n_blocks = max_top * 256u;
    detail::tree_view<BV> view; view.build(bv, n_blocks);
    bmb200_vec_blocks vb{n_blocks, view.kind.data(), view.ptr.data()};
    bmb200_set* set = nullptr; bmb200_rs* drs = nullptr;
    check(bmb200_set_upload_vectors(c.get(), 1, n_blocks, &vb, &set), "bmb200_set_upload_vectors");
    int rc = bmb200_rs_build(c.get(), set, 0, &drs);
    std::vector<unsigned> bcount(n_blocks); std::vector<bm::id64_t> sub(n_blocks); std::vector<uint64_t> sb(max_top + 1);
    static_assert(sizeof(bm::id64_t) == 8 && sizeof(unsigned) == 4, "index field widths");
    if (!rc) rc = bmb200_rs_export(drs, bcount.data(), (uint64_t*)sub.data(), sb.data());
    if (drs) bmb200_rs_free(drs);
    bmb200_set_free(set);
    check(rc, "bmb200_rs_build");
    bm::word_t*** root = const_cast<typename BV::blocks_manager_type&>(bman).top_blocks_root();
    for (unsigned i = 0; i < max_top; ++i)
    {
        if (!root[i]) { rs->set_null_super_block(i); continue; }
        if ((bm::word_t*)root[i] == FULL_BLOCK_FAKE_ADDR) { rs->set_full_super_block(i); continue; }
        rs->register_super_block(i, &bcount[i * 256u], &sub[i * 256u]);
    }
}

}} // namespace bm::b200

#endif
