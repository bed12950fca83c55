// bmb200_scanner.hpp -- reference-side binding: bm::b200::scanner<SV>, the GPU counterpart of
// bm::sparse_vector_scanner<SV> (src/bmsparsevec_algo.h:1040-1182) for unsigned and signed bm::sparse_vector<> and
// bm::rsc_sparse_vector<>.
// The iterator find_eq(first, last, bv_out) (elements equal to any listed value, src/bmsparsevec_algo.h:1398-1423) and
// count_eq(first, last) are one BMB200_SCAN_IN launch (csrc/scan_in_kernel.cuh) for the whole list.
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
// A float vector (bm::sparse_vector_float<sparse_vector<unsigned>>, src/bmsparsevec_float.h; detected like the reference's
// scanner does, through SV::sparse_vector_u) has a specialization of its own: it uploads signs_, mantissas_.get_slice(0..22) and
// exponents_.get_slice(0..7) as the planes of one BMB200_F_FLOAT scan and offers the reference's find_gt_float / find_ge_float /
// find_lt_float / find_le_float / find_range_float / find_range_float_unbounded plus batched and count-only forms.
// bm::b200::rank_compressor<BV> is the device counterpart of bm::rank_compressor<BV> (src/bmalgo.h:451-644).
// bm::b200::sparse_vector_find_mismatch / sparse_vector_find_first_mismatch compare two plain integer sparse vectors
// (src/bmsparsevec_algo.h:479,657) in one bmb200_sv_mismatch / bmb200_sv_first_mismatch launch (csrc/mismatch_kernel.cuh).
#ifndef BMB200_SCANNER_HPP_INCLUDED
#define BMB200_SCANNER_HPP_INCLUDED

#include "bmsparsevec.h"
#include "bmsparsevec_algo.h"
#include "bmb200_aggregator.hpp"

#include <algorithm>
#include <cstring>
#include <string>
#include <type_traits>

namespace bm { namespace b200 {

template<class SV, class = void>
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
        nullable_ = nn != nullptr;
        uint32_t n_vec = n_planes_ + 1;
        if constexpr (SV::is_compressed()) {
            // compressed planes: positions [0, effective_size()); the universe is that range, NN maps it to the logical space
            const size_type eff = sv.effective_size();
            scan_to_ = detail::column_count(std::max<uint64_t>(detail::size_blocks(eff), 1u), "bm::b200::scanner");
            universe_.clear(true); if (eff) universe_.set_range(0, eff - 1); universe_.optimize();
            if (nn) not_null_ = *nn;
            n_vec = n_planes_ + 2;
        } else {
            if (nn) universe_ = not_null_ = *nn;                         // NOT-NULL plane: finalize_search_result(:2426)
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

    /// elements equal to any value of [first, last): the iterator find_eq of the reference (src/bmsparsevec_algo.h:1398-1423,
    /// SQL `IN (...)`) with its effects on bv_out: the result is OR-ed into bv_out, which is not cleared, and when a listed value
    /// is 0 bv_out is then corrected to the NOT-NULL elements (correct_nulls, :2376) -- bits it held before included.  An empty
    /// range leaves bv_out untouched.  One BMB200_SCAN_IN launch reads the planes once for the whole list (one launch per
    /// BMB200_SCAN_IN_MAX_VALUES distinct values).  An RSC vector answers in logical positions, like the OR of find_eq(v).
    template<class It>
    void find_eq(It first, It last, bvector_type& bv_out)
    {
        bool any_zero = false;
        std::vector<uint64_t> v = in_slots(first, last, any_zero);
        if (v.empty()) return;
        if (size_) {
            bvector_type r;
            in_run(v, &r, nullptr);
            bv_out.bit_or(r);
        }
        if (any_zero && nullable_) bv_out.bit_and(not_null_);
    }
    /// the number of elements equal to any value of [first, last) (count-only: an RSC vector needs no rank decompression)
    template<class It>
    size_type count_eq(It first, It last)
    {
        bool any_zero = false;
        std::vector<uint64_t> v = in_slots(first, last, any_zero);
        size_type n = 0;
        if (!v.empty() && size_) in_run(v, nullptr, &n);
        return n;
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
    template<class It>
    static std::vector<uint64_t> in_slots(It first, It last, bool& any_zero)
    {
        static_assert(!SV::is_str(), "a str_sparse_vector is searched with find_eq_str / find_eq_str_batch");
        std::vector<uint64_t> v;
        for (; first != last; ++first) { const value_type x = *first; any_zero |= (x == 0); v.push_back(slot(x)); }
        return v;
    }
    /// SCAN_IN over the distinct values of v (sorted and de-duplicated here, so the launches of a long list are disjoint):
    /// *out replaced by the union, *count = its cardinality
    void in_run(std::vector<uint64_t>& v, bvector_type* out, size_type* count)
    {
        std::sort(v.begin(), v.end());
        v.erase(std::unique(v.begin(), v.end()), v.end());
        if (count) *count = 0;
        for (size_t k0 = 0; k0 < v.size(); k0 += BMB200_SCAN_IN_MAX_VALUES) {
            const uint32_t nv = (uint32_t)std::min<size_t>(v.size() - k0, BMB200_SCAN_IN_MAX_VALUES);
            bvector_type part; size_type n = 0;
            run(BMB200_SCAN_IN, v.data() + k0, nv, out ? &part : nullptr, &n, is_signed);
            if (count) *count += n;
            if (out) { if (k0) out->bit_or(part); else out->swap(part); }
        }
    }
    void run(int pred, const uint64_t* values, uint32_t nv, bvector_type* out, size_type* counts, bool sgn)
    {
        static_assert(!SV::is_str(), "a str_sparse_vector is searched with find_eq_str / find_eq_str_prefix");
        if (!nv) return;
        const uint32_t flags = (out ? BMB200_F_OPT_COMPRESS : BMB200_F_COUNT_ONLY) | (sgn ? BMB200_F_SIGNED : 0u);
        bmb200_scan_args a{0u, n_planes_, n_planes_, pred, flags, values, nv, 0u, scan_to_};
        if (pred == BMB200_SCAN_IN) nv = 1u;                       // one list, one result group
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
    bvector_type not_null_;            // nullable vectors: the NOT-NULL vector (logical positions), for correct_nulls
    bool nullable_ = false;
    size_type size_ = 0;
    unsigned n_planes_ = 0;
    uint32_t n_blocks_ = 0;
    uint32_t scan_to_ = 0;             // RSC: compressed columns scanned (0 = every column)
};

/// bm::b200::scanner for bm::sparse_vector_float<sparse_vector<unsigned>> (src/bmsparsevec_float.h, searches
/// src/bmsparsevec_algo.h:1299-1352,3692-4009).  The set holds the planes [signs_, mantissas_.get_slice(0..22),
/// exponents_.get_slice(0..7)] -- plane 1 + k is bit k of the magnitude bits & 0x7fffffff; absent slices are empty vectors and
/// trailing absent ones are trimmed -- and the universe: the NOT-NULL vector of exponents_ (which mantissas_ shares) for a
/// nullable vector, else [0, size()).  Every search is one bmb200_scan launch with BMB200_F_FLOAT, comparing in the IEEE
/// sign-magnitude total order of the bits (-0 < +0, NaNs beyond the infinities) as the reference's float searches do.
template<class SV>
class scanner<SV, std::void_t<typename SV::sparse_vector_u>>
{
public:
    typedef typename SV::bvector_type bvector_type;
    typedef typename SV::value_type value_type;
    typedef typename bvector_type::size_type size_type;
    static_assert(!SV::sparse_vector_u::is_compressed(),
                  "bm::b200::scanner: sparse_vector_float<rsc_sparse_vector<>> is not supported (its signs_ stay in the logical space)");

    scanner(context& c, const SV& sv) : ctx_(c) { bind(sv); }
    ~scanner() { if (set_) bmb200_set_free(set_); }
    scanner(const scanner&) = delete; scanner& operator=(const scanner&) = delete;

    /// upload the planes + universe of `sv`
    void bind(const SV& sv)
    {
        if (set_) { bmb200_set_free(set_); set_ = nullptr; }
        size_ = sv.size();
        n_planes_ = 32;
        while (n_planes_ > 1 && !plane(sv, n_planes_ - 1)) --n_planes_;
        n_blocks_ = detail::column_count(std::max<uint64_t>(detail::size_blocks(size_), 1u), "bm::b200::scanner");
        if (const bvector_type* nn = sv.exponents_.get_null_bvector()) universe_ = *nn;
        else { universe_.clear(true); if (size_) universe_.set_range(0, size_ - 1); universe_.optimize(); }
        const uint32_t n_vec = n_planes_ + 1;
        std::vector<detail::tree_view<bvector_type>> views(n_vec);
        std::vector<bmb200_vec_blocks> vb(n_vec);
        bvector_type empty;
        for (unsigned j = 0; j < n_vec; ++j) {
            const bvector_type* bv = j < n_planes_ ? plane(sv, j) : &universe_;
            views[j].build(bv ? *bv : empty, n_blocks_);
            vb[j].n_blocks = n_blocks_; vb[j].kind = views[j].kind.data(); vb[j].ptr = views[j].ptr.data();
        }
        check(bmb200_set_upload_vectors(ctx_.get(), n_vec, n_blocks_, vb.data(), &set_), "bmb200_set_upload_vectors");
    }

    void find_gt_float(value_type v, bvector_type& bv_out) { one(BMB200_SCAN_GT, v, v, bv_out); }
    void find_ge_float(value_type v, bvector_type& bv_out) { one(BMB200_SCAN_GE, v, v, bv_out); }
    void find_lt_float(value_type v, bvector_type& bv_out) { one(BMB200_SCAN_LT, v, v, bv_out); }
    void find_le_float(value_type v, bvector_type& bv_out) { one(BMB200_SCAN_LE, v, v, bv_out); }
    /// from <= element <= to; reversed bounds (from > to as floats) are swapped
    void find_range_float(value_type from, value_type to, bvector_type& bv_out) { one(BMB200_SCAN_RANGE, from, to, bv_out); }
    /// from < element < to; reversed bounds are swapped
    void find_range_float_unbounded(value_type from, value_type to, bvector_type& bv_out) { one(BMB200_SCAN_RANGE_OPEN, from, to, bv_out); }

    /// batched searches: one launch, out[k] replaced by the result of search k.  pred = BMB200_SCAN_GT / GE / LT / LE (one value
    /// per search) or BMB200_SCAN_RANGE / RANGE_OPEN (from, to pairs: two values per search)
    void find_batch(int pred, const std::vector<value_type>& values, std::vector<bvector_type>& out)
    {
        std::vector<uint64_t> v = slots(values);
        const size_t nv = two(pred) ? v.size() / 2 : v.size();
        out.resize(nv);
        run(pred, v.data(), (uint32_t)nv, out.data(), nullptr);
    }
    /// cardinalities only (pipeline agg_opt_only_counts); values as in find_batch
    void count_batch(int pred, const std::vector<value_type>& values, std::vector<size_type>& counts)
    {
        std::vector<uint64_t> v = slots(values);
        const size_t nv = two(pred) ? v.size() / 2 : v.size();
        counts.assign(nv, 0);
        run(pred, v.data(), (uint32_t)nv, nullptr, counts.data());
    }

private:
    /// plane j: 0 = signs_, 1..23 = mantissa slice j - 1, 24..31 = exponent slice j - 24 (nullptr when absent)
    static const bvector_type* plane(const SV& sv, unsigned j)
    {
        if (j == 0) return &sv.signs_;
        return j <= 23 ? sv.mantissas_.get_slice(j - 1) : sv.exponents_.get_slice(j - 24);
    }
    static bool two(int pred) { return pred == BMB200_SCAN_RANGE || pred == BMB200_SCAN_RANGE_OPEN; }
    static uint64_t slot(value_type v) { uint32_t b; std::memcpy(&b, &v, sizeof b); return b; }
    static std::vector<uint64_t> slots(const std::vector<value_type>& values)
    {
        std::vector<uint64_t> v(values.size());
        for (size_t k = 0; k < values.size(); ++k) v[k] = slot(values[k]);
        return v;
    }
    void one(int pred, value_type a, value_type b, bvector_type& bv_out)
    {
        const uint64_t v[2] = {slot(a), slot(b)};
        run(pred, v, 1, &bv_out, nullptr);
    }
    void run(int pred, const uint64_t* values, uint32_t nv, bvector_type* out, size_type* counts)
    {
        if (!nv) return;
        const uint32_t flags = (out ? BMB200_F_OPT_COMPRESS : BMB200_F_COUNT_ONLY) | BMB200_F_FLOAT;
        bmb200_scan_args a{0u, n_planes_, n_planes_, pred, flags, values, nv, 0u, 0u};
        bmb200_result* res = nullptr;
        int rc = bmb200_scan(ctx_.get(), set_, &a, &res);
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
    bvector_type universe_;
    size_type size_ = 0;
    unsigned n_planes_ = 0;
    uint32_t n_blocks_ = 0;
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

// ---- sparse-vector mismatch: sparse_vector_find_mismatch / sparse_vector_find_first_mismatch, src/bmsparsevec_algo.h:479,657 ----
namespace detail {

/// plain integer sparse vectors only: rsc_sparse_vector (the reference asserts in the vector form and compares compressed
/// positions in the first form), str_sparse_vector and sparse_vector_float are out of scope
template<class SV> struct mismatch_vector : std::false_type {};
template<class T, class BV> struct mismatch_vector<bm::sparse_vector<T, BV>>
    : std::integral_constant<bool, std::is_integral<T>::value && (sizeof(T) == 4 || sizeof(T) == 8)> {};

/// both vectors of a comparison uploaded into one set: the trimmed planes of sv1, then of sv2, then the NOT-NULL vectors of
/// the nullable ones, with columns covering max(sv1.size(), sv2.size()) (uploaded per call, like rank_compressor)
template<class SV>
struct mismatch_set
{
    typedef typename SV::bvector_type bvector_type;
    bmb200_set* set = nullptr;
    bmb200_mismatch_args args{};
    uint32_t n_blocks = 0;

    mismatch_set(context& ctx, const SV& sv1, const SV& sv2, bm::null_support null_proc, const char* what)
    {
        static_assert(mismatch_vector<SV>::value,
                      "bm::b200 mismatch compares bm::sparse_vector<unsigned / unsigned long long / int32_t / int64_t> only");
        std::vector<const bvector_type*> vecs;
        const unsigned na = planes(sv1, vecs), nb = planes(sv2, vecs);
        const bvector_type* nn1 = sv1.get_null_bvector();
        const bvector_type* nn2 = sv2.get_null_bvector();
        args.plane0_a = 0u; args.n_planes_a = na; args.plane0_b = na; args.n_planes_b = nb;
        args.not_null_a = nn1 ? (uint32_t)vecs.size() : 0xffffffffu; if (nn1) vecs.push_back(nn1);
        args.not_null_b = nn2 ? (uint32_t)vecs.size() : 0xffffffffu; if (nn2) vecs.push_back(nn2);
        args.size_a = uint64_t(sv1.size()); args.size_b = uint64_t(sv2.size());
        args.null_proc = null_proc == bm::use_null ? BMB200_MM_USE_NULL : BMB200_MM_NO_NULL;
        n_blocks = column_count(std::max<uint64_t>(size_blocks(std::max(args.size_a, args.size_b)), 1u), what);
        const uint32_t n_vec = std::max<uint32_t>((uint32_t)vecs.size(), 1u);
        std::vector<tree_view<bvector_type>> views(n_vec);
        std::vector<bmb200_vec_blocks> vb(n_vec);
        bvector_type empty;
        for (uint32_t j = 0; j < n_vec; ++j) {
            views[j].build(j < vecs.size() ? *vecs[j] : empty, n_blocks);
            vb[j].n_blocks = n_blocks; vb[j].kind = views[j].kind.data(); vb[j].ptr = views[j].ptr.data();
        }
        check(bmb200_set_upload_vectors(ctx.get(), n_vec, n_blocks, vb.data(), &set), "bmb200_set_upload_vectors");
    }
    ~mismatch_set() { if (set) bmb200_set_free(set); }
    mismatch_set(const mismatch_set&) = delete; mismatch_set& operator=(const mismatch_set&) = delete;

    /// the value planes j < effective_slices() (an absent one as an empty vector), trailing absent ones trimmed -> their count
    static unsigned planes(const SV& sv, std::vector<const bvector_type*>& vecs)
    {
        static const bvector_type empty;
        unsigned n = sv.effective_slices();
        auto at = [&](unsigned j) { const bvector_type* bv = sv.get_slice(j); return bv == sv.get_null_bvector() ? nullptr : bv; };
        while (n && !at(n - 1)) --n;
        for (unsigned j = 0; j < n; ++j) { const bvector_type* bv = at(j); vecs.push_back(bv ? bv : &empty); }
        return n;
    }
};

} // namespace detail

/// bm::sparse_vector_find_mismatch (src/bmsparsevec_algo.h:657) on the device: bv = the positions where sv1 and sv2 differ
/// (values, sizes, and under bm::use_null the NULLs; bm::no_null leaves positions NULL in both vectors out).  One
/// bmb200_sv_mismatch launch over both vectors' planes.  With bm::use_null and two non-nullable vectors the reference reports
/// every position [0, bm::id_max) (it inverts an empty vector); here no NULL term is added (DESIGN.md 3.5f).
template<class SV>
void sparse_vector_find_mismatch(context& ctx, typename SV::bvector_type& bv, const SV& sv1, const SV& sv2, bm::null_support null_proc)
{
    detail::mismatch_set<SV> ms(ctx, sv1, sv2, null_proc, "bm::b200::sparse_vector_find_mismatch");
    ms.args.flags = BMB200_F_OPT_COMPRESS;
    bmb200_result* res = nullptr;
    int rc = bmb200_sv_mismatch(ctx.get(), ms.set, &ms.args, &res);
    std::vector<uint8_t> kind(ms.n_blocks); std::vector<uint64_t> off(ms.n_blocks);
    std::vector<uint32_t> bits; std::vector<uint16_t> gaps;
    uint64_t nb = 0, ng = 0;
    if (!rc) rc = bmb200_result_sizes(res, &nb, &ng);
    if (!rc) { bits.resize(nb * BMB200_BLOCK_WORDS); gaps.resize(ng); rc = bmb200_result_fetch(res, kind.data(), off.data(), bits.data(), gaps.data()); }
    if (res) bmb200_result_free(res);
    check(rc, "bmb200_sv_mismatch");
    bv.clear(true);                                                  // replaced, as the reference's bv.clear()
    detail::store_result(bv, bv.size(), ms.n_blocks, kind.data(), off.data(), bits.data(), gaps.data());
}

/// bm::sparse_vector_find_first_mismatch (src/bmsparsevec_algo.h:479) on the device: the lowest position where sv1 and sv2
/// differ -> true and midx, or false and midx = bm::id_max.  One bmb200_sv_first_mismatch launch; 8 bytes come back.  The
/// reference compares GAP x GAP blocks by run ends only and can miss or postpone a difference there; this returns the true
/// lowest position (DESIGN.md 3.5f).
template<class SV>
bool sparse_vector_find_first_mismatch(context& ctx, const SV& sv1, const SV& sv2, typename SV::size_type& midx,
                                       bm::null_support null_proc = bm::use_null)
{
    detail::mismatch_set<SV> ms(ctx, sv1, sv2, null_proc, "bm::b200::sparse_vector_find_first_mismatch");
    uint64_t pos = 0; int found = 0;
    check(bmb200_sv_first_mismatch(ctx.get(), ms.set, &ms.args, &pos, &found), "bmb200_sv_first_mismatch");
    midx = found ? (typename SV::size_type)pos : (typename SV::size_type)bm::id_max;
    return found != 0;
}

// ---- set image through a sparse vector: set2set_11_transform, src/bmsparsevec_algo.h:1902-2205 ----
namespace detail {

/// the vectors the reference's remap compiles for: a plain sparse_vector whose value_type is its bvector's size_type
template<class SV> struct remap_vector : std::false_type {};
template<class T, class BV> struct remap_vector<bm::sparse_vector<T, BV>> : std::is_same<T, typename BV::size_type> {};

} // namespace detail

/// bm::set2set_11_transform<SV> on the device: attach_sv uploads the translation vector's trimmed planes and NOT-NULL vector
/// once; every remap uploads bv_in as its own set and is one bmb200_remap launch (csrc/remap_kernel.cuh).  bv_out is replaced by
/// the set of values sv[i] of the ids i of bv_in (inside the NOT-NULL vector of a nullable sv; a non-nullable sv maps ids without
/// an element, and ids past its size(), to 0), without the value bm::id_max, as the reference computes it.  compute_stats
/// changes the reference's work, not its answer, and is accepted and ignored.  Values of 2^32 and more are not covered:
/// attach_sv throws std::length_error for a vector with more than 32 effective planes (BM64ADDR only).
template<class SV>
class set2set_11_transform
{
public:
    typedef typename SV::bvector_type bvector_type;
    typedef typename SV::value_type value_type;
    typedef typename SV::size_type size_type;
    static_assert(detail::remap_vector<SV>::value,
                  "bm::b200::set2set_11_transform maps through bm::sparse_vector<bvector_type::size_type> only, as the reference");

    explicit set2set_11_transform(context& c) : ctx_(c) {}
    ~set2set_11_transform() { if (set_) bmb200_set_free(set_); }
    set2set_11_transform(const set2set_11_transform&) = delete; set2set_11_transform& operator=(const set2set_11_transform&) = delete;

    /// attach (upload) a translation vector, nullptr to detach
    void attach_sv(const SV* sv_brel, bool compute_stats = false)
    {
        (void)compute_stats;
        if (set_) { bmb200_set_free(set_); set_ = nullptr; }
        attached_ = sv_brel != nullptr;
        if (!sv_brel || (empty_ = sv_brel->empty())) return;
        std::vector<const bvector_type*> vecs;
        unsigned n = detail::mismatch_set<SV>::planes(*sv_brel, vecs);
        if (n > 32u) throw std::length_error("bm::b200::set2set_11_transform: values of 2^32 and more are not covered");
        static const bvector_type empty;
        if (!n) { vecs.push_back(&empty); n = 1; }
        args_ = bmb200_remap_args{0u, n, 0xffffffffu, BMB200_F_OPT_COMPRESS, uint64_t(bm::id_max)};
        if (const bvector_type* nn = sv_brel->get_null_bvector()) { args_.not_null = (uint32_t)vecs.size(); vecs.push_back(nn); }
        const uint32_t n_blocks = detail::column_count(std::max<uint64_t>(detail::size_blocks(sv_brel->size()), 1u),
                                                       "bm::b200::set2set_11_transform");
        std::vector<detail::tree_view<bvector_type>> views(vecs.size());
        std::vector<bmb200_vec_blocks> vb(vecs.size());
        for (size_t j = 0; j < vecs.size(); ++j) {
            views[j].build(*vecs[j], n_blocks);
            vb[j].n_blocks = n_blocks; vb[j].kind = views[j].kind.data(); vb[j].ptr = views[j].ptr.data();
        }
        check(bmb200_set_upload_vectors(ctx_.get(), (uint32_t)vecs.size(), n_blocks, vb.data(), &set_), "bmb200_set_upload_vectors");
    }

    /// bv_out = the image of bv_in through the attached vector
    void remap(const bvector_type& bv_in, bvector_type& bv_out)
    {
        bv_out.clear(true);
        if (!attached_ || empty_) return;
        const uint32_t n_blocks = std::max<uint32_t>(detail::extent_of(bv_in), 1u);
        detail::tree_view<bvector_type> view; view.build(bv_in, n_blocks);
        bmb200_vec_blocks vb{n_blocks, view.kind.data(), view.ptr.data()};
        bmb200_set* in = nullptr; bmb200_result *src = nullptr, *res = nullptr;
        int rc = bmb200_set_upload_vectors(ctx_.get(), 1u, n_blocks, &vb, &in);
        if (!rc) {
            // bv_in enters as a result, the form bmb200_remap reads: a one-source OR copies it
            const uint32_t zero = 0u;
            bmb200_agg_args a{BMB200_OP_OR, BMB200_F_OPT_NONE, &zero, 1u, nullptr, 0u, 0u, 0u};
            rc = bmb200_aggregate(ctx_.get(), in, &a, &src);
        }
        if (!rc) rc = bmb200_remap(ctx_.get(), set_, &args_, src, &res);
        uint64_t total = 0, nb = 0, ng = 0;
        const uint8_t* kind = nullptr; const uint64_t* off = nullptr; const uint32_t* bits = nullptr; const uint16_t* gaps = nullptr;
        uint32_t n_cols = 0;
        if (!rc) rc = bmb200_result_device_ptrs(res, nullptr, nullptr, nullptr, nullptr, &n_cols);
        if (!rc) rc = bmb200_result_fetch_view(res, &kind, &off, &bits, &gaps, &nb, &ng, &total);
        if (!rc) detail::store_result(bv_out, bv_out.size(), n_cols, kind, off, bits, gaps);
        if (res) bmb200_result_free(res);
        if (src) bmb200_result_free(src);
        if (in) bmb200_set_free(in);
        check(rc, "bm::b200::set2set_11_transform::remap");
    }

    /// attach sv_brel, remap, detach (the reference's remap(bv_in, sv_brel, bv_out))
    void remap(const bvector_type& bv_in, const SV& sv_brel, bvector_type& bv_out)
    {
        attach_sv(&sv_brel);
        remap(bv_in, bv_out);
        attach_sv(nullptr);
    }
    void run(const bvector_type& bv_in, const SV& sv_brel, bvector_type& bv_out) { remap(bv_in, sv_brel, bv_out); }

private:
    context& ctx_;
    bmb200_set* set_ = nullptr;
    bmb200_remap_args args_{};
    bool attached_ = false, empty_ = true;
};

}} // namespace bm::b200

#endif
