// bmb200_scanner.hpp -- reference-side binding: bm::b200::scanner<SV>, the GPU counterpart of
// bm::sparse_vector_scanner<SV> (src/bmsparsevec_algo.h:1040-1182) for unsigned and signed bm::sparse_vector<> and
// bm::rsc_sparse_vector<>.
//
// The scanner binds to one sparse vector (like sparse_vector_scanner::bind, :1060): its bit-planes
// (sparse_vector::get_slice(j), j < effective_slices()) and its searchable universe (the NOT-NULL plane of a nullable
// vector, else [0, size())) are uploaded ONCE as vectors of a bmb200 set; every search is then one bmb200_scan launch
// (csrc/scan_kernel.cuh: one pass over the planes per block column and search value).  Same method names and
// argument meaning as the reference: find_eq / find_gt / find_ge / find_lt / find_le / find_range / find_zero /
// find_nonzero, result written into the caller's bvector (replaced, like bv_out.clear() + search).
// Batched forms take arrays of values and return one vector / count per value (the scanner's pipeline mode, :1399-1431).
//
// A rank-select compressed vector (bm::rsc_sparse_vector<unsigned>, src/bmsparsevec_compr.h) binds the same way: its planes
// hold only the NOT-NULL elements, packed to [0, effective_size()).  The set then holds the compressed planes, the universe
// [0, effective_size()) and the NOT-NULL vector NN, as wide as the logical space; the device rs index of NN is built once.
// A search scans the compressed columns and bmb200_rank_decompress maps the result to logical positions, as the reference
// scanner does for RSC vectors (src/bmsparsevec_algo.h:2300-2306,4525-4537); results are in the logical index space.
// A signed vector (value_type int32_t / int64_t) stores s2u(x) in its planes (src/bmbmatrix.h:2536-2569, plane 0 = sign);
// its searches run with BMB200_F_SIGNED and the value as a two's-complement int64_t.  find_zero / find_nonzero stay unsigned
// EQ 0 / GT 0 over the same planes, which is what the reference computes for them (an OR of all planes).
// A string vector (bm::str_sparse_vector<char, ...>, SV::is_str()) binds its planes j < rows_not_null() (plane 8k+b = bit b of
// byte k) and its universe; find_eq_str / find_eq_str_prefix / the batched string searches are bmb200_scan_str launches
// (csrc/str_scan_kernel.cuh).  A remapped vector's queries are translated on the host (remap_tosv) and only their codes go to
// the device.  The numeric searches do not compile for a string vector.
// bm::b200::rank_compressor<BV> is the device counterpart of bm::rank_compressor<BV> (src/bmalgo.h:451-644).
#ifndef BMB200_SCANNER_HPP_INCLUDED
#define BMB200_SCANNER_HPP_INCLUDED

#include "bmsparsevec.h"
#include "bmsparsevec_algo.h"
#include "bmb200_aggregator.hpp"

#include <string>

namespace bm { namespace b200 {

template<class SV>
class scanner
{
public:
    typedef typename SV::bvector_type bvector_type;
    typedef typename SV::value_type value_type;
    typedef typename bvector_type::size_type size_type;
    static constexpr bool is_signed = std::is_signed<value_type>::value;

    scanner(context& c, const SV& sv) : ctx_(c) { bind(sv); }
    ~scanner() { if (rs_) bmb200_rs_free(rs_); if (set_) bmb200_set_free(set_); }
    scanner(const scanner&) = delete; scanner& operator=(const scanner&) = delete;

    /// upload the planes + universe of `sv` (sparse_vector_scanner::bind, :1060); for an RSC vector also NN and its rs index
    void bind(const SV& sv)
    {
        if (rs_) { bmb200_rs_free(rs_); rs_ = nullptr; }
        if (set_) { bmb200_set_free(set_); set_ = nullptr; }
        size_ = sv.size();
        if constexpr (SV::is_str()) {
            // rows_not_null() string planes, trailing absent ones trimmed (their bits are all 0)
            str_sv_ = &sv;
            n_planes_ = (unsigned)sv.get_bmatrix().rows_not_null();
            while (n_planes_ > 1 && !sv.get_slice(n_planes_ - 1)) --n_planes_;
            if (!n_planes_) n_planes_ = 1;
        } else {
            n_planes_ = sv.effective_slices();
            while (n_planes_ > 1 && !sv.get_slice(n_planes_ - 1)) --n_planes_;
        }
        n_blocks_ = detail::column_count(std::max<uint64_t>(detail::size_blocks(size_), 1u), "bm::b200::scanner");
        const bvector_type* nn = sv.get_null_bvector();
        uint32_t n_vec = n_planes_ + 1;
        if constexpr (SV::is_compressed()) {
            // compressed planes: positions [0, effective_size()); the universe is that range, NN maps it to the logical space
            const size_type eff = sv.effective_size();
            scan_to_ = detail::column_count(std::max<uint64_t>(detail::size_blocks(eff), 1u), "bm::b200::scanner");
            universe_.clear(true); if (eff) universe_.set_range(0, eff - 1); universe_.optimize();
            n_vec = n_planes_ + 2;
        } else {
            if (nn) universe_ = *nn;                                     // NOT-NULL plane: finalize_search_result(:2426)
            else { universe_.clear(true); if (size_) universe_.set_range(0, size_ - 1); universe_.optimize(); }   // invert_internal(:1686) range
        }
        std::vector<detail::tree_view<bvector_type>> views(n_vec);
        std::vector<bmb200_vec_blocks> vb(n_vec);
        bvector_type empty;
        for (unsigned j = 0; j < n_vec; ++j) {
            const bvector_type* bv = j < n_planes_ ? plane(sv, j) : j == n_planes_ ? &universe_ : nn;
            views[j].build(bv ? *bv : empty, n_blocks_);                 // planes past their columns stay NULL
            vb[j].n_blocks = n_blocks_; vb[j].kind = views[j].kind.data(); vb[j].ptr = views[j].ptr.data();
        }
        check(bmb200_set_upload_vectors(ctx_.get(), n_vec, n_blocks_, vb.data(), &set_), "bmb200_set_upload_vectors");
        if constexpr (SV::is_compressed()) check(bmb200_rs_build(ctx_.get(), set_, n_planes_ + 1, &rs_), "bmb200_rs_build");
    }

    void find_eq(value_type v, bvector_type& bv_out) { one(BMB200_SCAN_EQ, v, 0, bv_out); }
    void find_gt(value_type v, bvector_type& bv_out) { one(BMB200_SCAN_GT, v, 0, bv_out); }
    void find_ge(value_type v, bvector_type& bv_out) { one(BMB200_SCAN_GE, v, 0, bv_out); }
    void find_lt(value_type v, bvector_type& bv_out) { one(BMB200_SCAN_LT, v, 0, bv_out); }
    void find_le(value_type v, bvector_type& bv_out) { one(BMB200_SCAN_LE, v, 0, bv_out); }
    void find_range(value_type from, value_type to, bvector_type& bv_out) { one(BMB200_SCAN_RANGE, from, to, bv_out); }
    // sign-agnostic in the reference (an OR of all planes): the unsigned search for 0 also on a signed vector
    void find_zero(bvector_type& bv_out)    { const uint64_t z[2] = {0, 0}; run(BMB200_SCAN_EQ, z, 1, &bv_out, nullptr, false); }
    void find_nonzero(bvector_type& bv_out) { const uint64_t z[2] = {0, 0}; run(BMB200_SCAN_GT, z, 1, &bv_out, nullptr, false); }

    // ---- string vectors (str_sparse_vector): find_eq_str / find_eq_str_prefix, src/bmsparsevec_algo.h:3263-3436 ----
    /// elements equal to s; false when there is none (or the vector is empty)
    bool find_eq_str(const char* s, bvector_type& bv_out) { str_run(&s, 1, 0u, &bv_out, nullptr); return bv_out.any(); }
    /// elements whose first strlen(s) bytes are s (the empty s: find_eq_str(""))
    bool find_eq_str_prefix(const char* s, bvector_type& bv_out) { str_run(&s, 1, BMB200_F_STR_PREFIX, &bv_out, nullptr); return bv_out.any(); }
    /// the lowest element equal to s (find_first_eq): one launch, the first non-empty column read back
    bool find_eq_str(const char* s, size_type& pos)
    {
        static_assert(SV::is_str(), "find_eq_str needs a str_sparse_vector");
        std::vector<std::string> codes;
        if (!size_ || !to_codes(&s, 1, codes)) return false;
        bmb200_result* res = launch_str(codes, BMB200_F_OPT_NONE);
        struct drop { bmb200_result* r; ~drop() { bmb200_result_free(r); } } guard{res};
        std::vector<uint32_t> pop(n_blocks_);
        bmb200_result_meta m{}; m.popcnt = pop.data();
        check(bmb200_result_fetch_meta(res, &m), "bmb200_result_fetch_meta");
        for (uint32_t nb = 0; nb < n_blocks_; ++nb) {
            if (!pop[nb]) continue;
            const unsigned first = detail::result_column_first(res, nb);
            if (first != 65536u) { pos = (size_type)((uint64_t)nb * 65536u + first); return true; }
        }
        return false;
    }
    /// pipeline + find_eq_str(TPipe&) (src/bmsparsevec_algo.h:3424-3436,4579-4651): one launch, out[k] = exact result of q[k]
    void find_eq_str_batch(const std::vector<std::string>& q, std::vector<bvector_type>& out)
    {
        std::vector<const char*> p(q.size()); for (size_t k = 0; k < q.size(); ++k) p[k] = q[k].c_str();
        out.resize(q.size());
        str_run(p.data(), p.size(), 0u, out.data(), nullptr);
    }
    /// the same searches, cardinalities only (pipeline<agg_opt_only_counts>)
    void count_eq_str_batch(const std::vector<std::string>& q, std::vector<size_type>& counts)
    {
        std::vector<const char*> p(q.size()); for (size_t k = 0; k < q.size(); ++k) p[k] = q[k].c_str();
        counts.assign(q.size(), 0);
        str_run(p.data(), p.size(), 0u, nullptr, counts.data());
    }

    /// batched searches: one launch, out[k] replaced by the result of values[k].  For a signed vector every slot holds
    /// a two's-complement int64_t: uint64_t(int64_t(v)).
    void find_batch(int pred, const std::vector<uint64_t>& values, std::vector<bvector_type>& out)
    {
        const size_t nv = pred == BMB200_SCAN_RANGE ? values.size() / 2 : values.size();
        out.resize(nv);
        run(pred, values.data(), (uint32_t)nv, out.data(), nullptr, is_signed);
    }
    /// cardinalities only (pipeline agg_opt_only_counts); values as in find_batch
    void count_batch(int pred, const std::vector<uint64_t>& values, std::vector<size_type>& counts)
    {
        const size_t nv = pred == BMB200_SCAN_RANGE ? values.size() / 2 : values.size();
        counts.assign(nv, 0);
        run(pred, values.data(), (uint32_t)nv, nullptr, counts.data(), is_signed);
    }

private:
    static const bvector_type* plane(const SV& sv, unsigned j)
    {
        if constexpr (SV::is_str()) return j < sv.get_bmatrix().rows_not_null() ? sv.get_slice(j) : nullptr;
        else return sv.get_slice(j);
    }
    /// the device form of each query: a remapped vector's codes (remap_tosv), else the bytes as they are.  Queries that cannot
    /// match get ok = false: remap_tosv finds no code, or the reference has no defined answer for them (longer than
    /// effective_max_str(), or a byte >= 0x80, whose remap row index sign-extends: DESIGN.md §3.5c).  -> any query left
    bool to_codes(const char* const* q, size_t n, std::vector<std::string>& codes, std::vector<bool>* ok = nullptr)
    {
        codes.assign(n, std::string());
        if (ok) ok->assign(n, false);
        bool any = false;
        for (size_t k = 0; k < n; ++k) {
            const char* s = q[k];
            bool good = true;
            if (*s && str_sv_->is_remap()) {
                const size_t len = std::strlen(s), ms = str_sv_->effective_max_str();
                good = len <= ms;
                for (size_t i = 0; good && i < len; ++i) good = (unsigned char)s[i] < 0x80u;
                std::vector<char> buf(ms + 1, 0);
                good = good && str_sv_->remap_tosv(buf.data(), ms, s);
                if (good) codes[k] = buf.data();
            } else codes[k] = s;
            if (ok) (*ok)[k] = good;
            any |= good;
        }
        return any;
    }
    /// one bmb200_scan_str launch over `codes` (NUL-padded slots of the longest + 1 bytes)
    bmb200_result* launch_str(const std::vector<std::string>& codes, uint32_t flags)
    {
        size_t stride = 1;
        for (const auto& c : codes) stride = std::max(stride, c.size() + 1);
        std::vector<char> slots(codes.size() * stride, 0);
        for (size_t k = 0; k < codes.size(); ++k) std::memcpy(slots.data() + k * stride, codes[k].data(), codes[k].size());
        bmb200_scan_str_args a{0u, n_planes_, n_planes_, flags, slots.data(), (uint32_t)stride, (uint32_t)codes.size(), 0u, 0u};
        bmb200_result* res = nullptr;
        check(bmb200_scan_str(ctx_.get(), set_, &a, &res), "bmb200_scan_str");
        return res;
    }
    /// string searches: out[k] / counts[k] of q[k]; a query that cannot match stays out of the launch and gets an empty slot
    void str_run(const char* const* q, size_t n, uint32_t mode, bvector_type* out, size_type* counts)
    {
        static_assert(SV::is_str(), "string searches need a str_sparse_vector");
        for (size_t k = 0; k < n; ++k) { if (out) out[k].clear(true); if (counts) counts[k] = 0; }
        std::vector<std::string> codes; std::vector<bool> ok;
        if (!n || !size_ || !to_codes(q, n, codes, &ok)) return;
        std::vector<std::string> live; std::vector<size_t> at;
        for (size_t k = 0; k < n; ++k) if (ok[k]) { live.push_back(codes[k]); at.push_back(k); }
        bmb200_result* res = launch_str(live, mode | (out ? BMB200_F_OPT_COMPRESS : BMB200_F_COUNT_ONLY));
        const uint32_t nv = (uint32_t)live.size();
        const size_t ncols = (size_t)nv * n_blocks_;
        std::vector<uint64_t> totals(nv);
        std::vector<uint8_t> kind(ncols); std::vector<uint64_t> off(ncols); std::vector<uint32_t> bits; std::vector<uint16_t> gaps;
        int rc = bmb200_result_group_totals(res, totals.data(), nv);
        if (!rc && out) { uint64_t nb = 0, ng = 0; rc = bmb200_result_sizes(res, &nb, &ng);
                          if (!rc) { bits.resize(nb * BMB200_BLOCK_WORDS); gaps.resize(ng);
                                     rc = bmb200_result_fetch(res, kind.data(), off.data(), bits.data(), gaps.data()); } }
        bmb200_result_free(res);
        check(rc, "bmb200_scan_str");
        for (uint32_t k = 0; k < nv; ++k) {
            if (counts) counts[at[k]] = (size_type)totals[k];
            if (out) detail::store_result(out[at[k]], size_, n_blocks_, kind.data() + (size_t)k * n_blocks_, off.data() + (size_t)k * n_blocks_,
                                          bits.data(), gaps.data());
        }
    }

    static uint64_t slot(value_type v)
    {
        if constexpr (is_signed) return uint64_t(int64_t(v));
        else return uint64_t(v);
    }
    void one(int pred, value_type a, value_type b, bvector_type& bv_out)
    {
        const uint64_t v[2] = {slot(a), slot(b)};
        run(pred, v, 1, &bv_out, nullptr, is_signed);
    }
    void run(int pred, const uint64_t* values, uint32_t nv, bvector_type* out, size_type* counts, bool sgn)
    {
        static_assert(!SV::is_str(), "a str_sparse_vector is searched with find_eq_str / find_eq_str_prefix");
        if (!nv) return;
        const uint32_t flags = (out ? BMB200_F_OPT_COMPRESS : BMB200_F_COUNT_ONLY) | (sgn ? BMB200_F_SIGNED : 0u);
        bmb200_scan_args a{0u, n_planes_, n_planes_, pred, flags, values, nv, 0u, scan_to_};
        bmb200_result* res = nullptr;
        int rc = bmb200_scan(ctx_.get(), set_, &a, &res);
        if constexpr (SV::is_compressed()) {
            // compressed space -> logical positions; a count-only search keeps the scan's totals (the mapping is a bijection)
            if (!rc && out) {
                bmb200_result* logical = nullptr;
                rc = bmb200_rank_decompress(ctx_.get(), rs_, res, BMB200_F_OPT_COMPRESS, &logical);
                bmb200_result_free(res); res = logical;
            }
        }
        const size_t ncols = (size_t)nv * n_blocks_;
        std::vector<uint64_t> totals(nv);
        std::vector<uint8_t> kind(ncols); std::vector<uint64_t> off(ncols); std::vector<uint32_t> bits; std::vector<uint16_t> gaps;
        if (!rc) rc = bmb200_result_group_totals(res, totals.data(), nv);
        if (!rc && out) { uint64_t nb = 0, ng = 0; rc = bmb200_result_sizes(res, &nb, &ng);
                          if (!rc) { bits.resize(nb * BMB200_BLOCK_WORDS); gaps.resize(ng);
                                     rc = bmb200_result_fetch(res, kind.data(), off.data(), bits.data(), gaps.data()); } }
        if (res) bmb200_result_free(res);
        check(rc, "bmb200_scan");
        for (uint32_t k = 0; k < nv; ++k) {
            if (counts) counts[k] = (size_type)totals[k];
            if (out) detail::store_result(out[k], size_, n_blocks_, kind.data() + (size_t)k * n_blocks_, off.data() + (size_t)k * n_blocks_,
                                          bits.data(), gaps.data());
        }
    }

    context& ctx_;
    bmb200_set* set_ = nullptr;
    bmb200_rs* rs_ = nullptr;          // RSC: rs index of NN
    const SV* str_sv_ = nullptr;       // string vector: its remap tables stay on the host (to_codes)
    bvector_type universe_;
    size_type size_ = 0;
    unsigned n_planes_ = 0;
    uint32_t n_blocks_ = 0;
    uint32_t scan_to_ = 0;             // RSC: compressed columns scanned (0 = every column)
};

/// bm::rank_compressor<BV> (src/bmalgo.h:451-644) on the device: the index vector and the source are uploaded for the call,
/// the rs index of the index vector is built on the device, and the target is replaced by the result.
template<class BV>
class rank_compressor
{
public:
    typedef typename BV::size_type size_type;
    explicit rank_compressor(context& c) : ctx_(c) {}

    /// target bit r = src at the position of the (r+1)-th set bit of bv_idx (rank_compressor::compress, src/bmalgo.h:498);
    /// bits of src outside bv_idx are dropped
    void compress(BV& bv_target, const BV& bv_idx, const BV& bv_src)
    {
        if (&bv_idx == &bv_src) { bv_target = bv_src; return; }      // src/bmalgo.h:505
        call(bv_target, bv_idx, bv_src, true);
    }
    /// target bit p = bv_idx[p] and src bit rank_idx(p) - 1 (rank_compressor::decompress, src/bmalgo.h:571)
    void decompress(BV& bv_target, const BV& bv_idx, const BV& bv_src)
    {
        if (&bv_idx == &bv_src) { bv_target = bv_src; return; }      // src/bmalgo.h:579
        call(bv_target, bv_idx, bv_src, false);
    }

private:
    void call(BV& bv_target, const BV& bv_idx, const BV& bv_src, bool comp)
    {
        uint32_t n_blocks = std::max(detail::extent_of(bv_idx), detail::extent_of(bv_src)); if (!n_blocks) n_blocks = 1;
        const BV* both[2] = {&bv_idx, &bv_src};
        std::vector<detail::tree_view<BV>> views(2); std::vector<bmb200_vec_blocks> vb(2);
        for (int k = 0; k < 2; ++k) {
            views[k].build(*both[k], n_blocks);
            vb[k].n_blocks = n_blocks; vb[k].kind = views[k].kind.data(); vb[k].ptr = views[k].ptr.data();
        }
        bmb200_set* set = nullptr; bmb200_rs* rs = nullptr; bmb200_result *src = nullptr, *res = nullptr;
        int rc = bmb200_set_upload_vectors(ctx_.get(), 2, n_blocks, vb.data(), &set);
        if (!rc) rc = bmb200_rs_build(ctx_.get(), set, 0u, &rs);
        if (!rc && comp) rc = bmb200_rank_compress(ctx_.get(), rs, 1u, BMB200_F_OPT_COMPRESS, &res);
        if (!rc && !comp) {
            // the source enters as a result, the form bmb200_rank_decompress reads: a one-source OR copies it
            const uint32_t one = 1u;
            bmb200_agg_args a{BMB200_OP_OR, BMB200_F_OPT_NONE, &one, 1u, nullptr, 0u, 0u, 0u};
            rc = bmb200_aggregate(ctx_.get(), set, &a, &src);
            if (!rc) rc = bmb200_rank_decompress(ctx_.get(), rs, src, BMB200_F_OPT_COMPRESS, &res);
        }
        uint64_t total = 0, nb = 0, ng = 0;
        const uint8_t* kind = nullptr; const uint64_t* off = nullptr; const uint32_t* bits = nullptr; const uint16_t* gaps = nullptr;
        uint32_t n_cols = 0;
        if (!rc) rc = bmb200_result_device_ptrs(res, nullptr, nullptr, nullptr, nullptr, &n_cols);
        if (!rc) rc = bmb200_result_fetch_view(res, &kind, &off, &bits, &gaps, &nb, &ng, &total);
        if (!rc) detail::store_result(bv_target, bv_target.size(), n_cols, kind, off, bits, gaps);
        if (res) bmb200_result_free(res);
        if (src) bmb200_result_free(src);
        if (rs) bmb200_rs_free(rs);
        if (set) bmb200_set_free(set);
        check(rc, comp ? "bm::b200::rank_compressor::compress" : "bm::b200::rank_compressor::decompress");
    }
    context& ctx_;
};

}} // namespace bm::b200

#endif
