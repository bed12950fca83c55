"""Host-side mirror of ``bm::sparse_vector<unsigned, bvector<>>`` + ``bm::sparse_vector_scanner<SV>`` for the
searches the GPU path covers (reference src/bmsparsevec.h, src/bmsparsevec_algo.h:1083-1182):

    find_eq / find_gt / find_ge / find_lt / find_le / find_range / find_zero / find_nonzero

A sparse vector is bit-transposed: plane ("slice") j is the bit-vector of the elements whose bit j is set
(``sparse_vector::get_slice(j)``).  The reference answers a search with many aggregator / bvector passes over the planes
(prepare_and_sub_aggregator :2593-2632 for find_eq, find_gt_horizontal :1451-1500 for the inequalities); the GPU path
walks the planes of a block column once per search value (csrc/scan_kernel.cuh).  No comparison happens in Python:
this module only packs planes and calls the C ABI (``bmb200_scan``).

A rank-select compressed vector (``bm::rsc_sparse_vector<unsigned>``, src/bmsparsevec_compr.h) is searched the way the
reference searches it (src/bmsparsevec_algo.h:2300-2306,4525-4537): the scan runs over its compressed planes, restricted to
``[0, effective_size())``, and ``bmb200_rank_decompress`` maps the result to logical positions through the NOT-NULL vector.

Signed vectors (``sparse_vector<int32_t / int64_t>`` and their RSC forms; ``from_values(..., signed=True)``) store every
element as ``s2u(x)`` (src/bmbmatrix.h:2536-2569: ``x >= 0 -> x << 1``, ``x < 0 -> (-(x+1)) << 1 | 1``), so plane 0 is the
sign plane.  Their searches take int64 values and run with ``F_SIGNED``; ``find_zero / find_nonzero`` stay unsigned searches
for 0 over the same planes, which is what the reference computes for them (an OR of all planes).

Float vectors (``bm::sparse_vector_float<sparse_vector<unsigned>>``, ``SparseVectorFloat``) keep a float's sign bit in
``signs_``, its exponent in ``exponents_`` and its mantissa in ``mantissas_``.  Their planes are laid out as
``[signs_, mantissa 0..22, exponent 0..7]`` -- plane 1 + k is bit k of the magnitude ``bits & 0x7fffffff`` -- and their
searches (``find_gt_float`` & co.) run with ``F_FLOAT`` and float32 values.  They compare in the IEEE sign-magnitude total
order of the bits (-0 < +0, NaNs beyond the infinities), as the reference's float searches do; there is no float ``find_eq``.

``find_eq_any(values)`` / ``count_eq_any(values)`` are the reference's iterator ``find_eq(sv, start, end, bv_out)``
(src/bmsparsevec_algo.h:1398-1423, SQL ``IN (...)``) for plain, nullable, RSC and signed vectors: one ``SCAN_IN`` launch reads
the planes once for the whole list (csrc/scan_in_kernel.cuh).  They return the set of matching elements; an RSC vector answers
in logical positions.

``find_mismatch(sv1, sv2)`` / ``find_first_mismatch(sv1, sv2)`` are the reference's ``sparse_vector_find_mismatch`` /
``sparse_vector_find_first_mismatch`` (src/bmsparsevec_algo.h:657,479) for two plain ``SparseVector``s: both vectors'
planes and NOT-NULL vectors go into one set and one launch reads every plane block once (csrc/mismatch_kernel.cuh).

String vectors (``bm::str_sparse_vector<char, ...>``, ``StrSparseVector``) keep bit b of byte k of every element in plane 8k+b;
``find_eq_str`` / ``find_eq_str_prefix`` / ``count_eq_str`` run as ``bmb200_scan_str`` (csrc/str_scan_kernel.cuh).  The numeric
searches raise on a string vector.
"""
from __future__ import annotations

import numpy as np

from . import capi
from .capi import (F_COUNT_ONLY, F_FLOAT, F_OPT_COMPRESS, F_SIGNED, F_STR_PREFIX, SCAN_EQ, SCAN_GE, SCAN_GT, SCAN_IN, SCAN_LE,
                   SCAN_LT, SCAN_RANGE, SCAN_RANGE_OPEN)
from .hostfmt import BLOCK_BITS, BVector, PackedSet, bits_to_words, result_to_bvector


def s2u(values) -> np.ndarray:
    """sparse_vector<signed>::s2u (src/bmbmatrix.h:2536-2569) of int64 values: x >= 0 -> x << 1, x < 0 -> (-(x+1)) << 1 | 1."""
    x = np.ascontiguousarray(values, dtype=np.int64)
    return np.where(x >= 0, x.view(np.uint64) << np.uint64(1), ((~x).view(np.uint64) << np.uint64(1)) | np.uint64(1))


class SparseVector:
    """``bm::sparse_vector<unsigned, bvector<>>`` as the scanner sees it: ``size()``, ``effective_slices()`` planes and,
    for a nullable vector, the NOT-NULL plane (``get_null_bvector()``)."""

    def __init__(self, planes: list[BVector], size: int, not_null: BVector | None = None, signed: bool = False):
        self.planes = planes
        self.size = int(size)
        self.not_null = not_null
        self.signed = bool(signed)

    @classmethod
    def from_values(cls, values, null_mask=None, optimize: bool = True, signed: bool = False) -> "SparseVector":
        """import(values) [+ set_null where null_mask] + optimize(): plane j = elements with bit j set.  signed: the values are
        int64 and the planes hold s2u(value) (plane 0 = sign), as in sparse_vector<int32_t / int64_t>."""
        v = s2u(values) if signed else np.ascontiguousarray(values, dtype=np.uint64)
        n = v.size
        nb = max(1, (n + BLOCK_BITS - 1) // BLOCK_BITS)
        if null_mask is not None:
            v = np.where(np.asarray(null_mask, bool), 0, v)
        top = int(v.max()).bit_length() if n else 0
        planes = []
        for j in range(max(top, 1)):
            bits = np.zeros(nb * BLOCK_BITS, np.uint8)
            bits[:n] = (v >> np.uint64(j)) & np.uint64(1)
            bv = BVector.from_words(bits_to_words(bits))
            planes.append(bv.optimize() if optimize else bv)
        nn = None
        if null_mask is not None:
            bits = np.zeros(nb * BLOCK_BITS, np.uint8)
            bits[:n] = ~np.asarray(null_mask, bool)
            nn = BVector.from_words(bits_to_words(bits))
            if optimize:
                nn.optimize()
        return cls(planes, n, nn, signed)

    def effective_slices(self) -> int:
        return len(self.planes)

    def universe(self) -> BVector:
        """Searchable indexes: the NOT-NULL plane, else [0, size) (what invert_internal / finalize_search_result apply)."""
        if self.not_null is not None:
            return self.not_null
        nb = self.planes[0].n_blocks
        bits = np.zeros(nb * BLOCK_BITS, np.uint8)
        bits[:self.size] = 1
        return BVector.from_words(bits_to_words(bits)).optimize()


def f2u(values) -> np.ndarray:
    """float32 values -> their bits as the float planes hold them: magnitude (bits & 0x7fffffff) in bits 1..31, sign in bit 0"""
    b = np.ascontiguousarray(values, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((b & np.uint64(0x7FFFFFFF)) << np.uint64(1)) | (b >> np.uint64(31))


class SparseVectorFloat(SparseVector):
    """``bm::sparse_vector_float<sparse_vector<unsigned>>`` as the scanner sees it: plane 0 = ``signs_``, planes 1..23 =
    ``mantissas_.get_slice(0..22)``, planes 24..31 = ``exponents_.get_slice(0..7)``, trailing empty planes trimmed; for a
    nullable vector the NOT-NULL plane that ``mantissas_`` shares with ``exponents_``."""

    @classmethod
    def from_values(cls, values, null_mask=None, optimize: bool = True) -> "SparseVectorFloat":
        """set(i, value) for every non-NULL i (NULL elements and unassigned positions hold no bit) + optimize()"""
        sv = SparseVector.from_values(f2u(values), null_mask, optimize)
        return cls(sv.planes, sv.size, sv.not_null)


class RscSparseVector:
    """``bm::rsc_sparse_vector<unsigned>`` as the scanner sees it: the planes hold only the NOT-NULL elements, packed to the
    positions ``[0, effective_size())`` in index order; ``not_null`` (``get_null_bvector()``) maps them back to the logical
    index space of ``size`` positions."""

    def __init__(self, planes: list[BVector], size: int, not_null: BVector, signed: bool = False):
        self.planes = planes
        self.size = int(size)
        self.not_null = not_null
        self.signed = bool(signed)
        self._eff = not_null.count()

    @classmethod
    def from_values(cls, values, null_mask, optimize: bool = True, signed: bool = False) -> "RscSparseVector":
        """The nullable sparse vector of from_values(values, null_mask), rank-compressed (rsc_sparse_vector::load_from).
        signed: int64 values, s2u planes (rsc_sparse_vector<int32_t / int64_t>)."""
        v = np.ascontiguousarray(values, dtype=np.int64 if signed else np.uint64)
        keep = ~np.asarray(null_mask, bool)
        dense = SparseVector.from_values(v[keep], None, optimize, signed)
        nb = max(1, (v.size + BLOCK_BITS - 1) // BLOCK_BITS)
        bits = np.zeros(nb * BLOCK_BITS, np.uint8)
        bits[:v.size] = keep
        nn = BVector.from_words(bits_to_words(bits))
        return cls(dense.planes, v.size, nn.optimize() if optimize else nn, signed)

    def effective_size(self) -> int:
        return self._eff

    def effective_slices(self) -> int:
        return len(self.planes)

    def universe(self) -> BVector:
        """Searchable compressed positions: [0, effective_size())."""
        nb = self.planes[0].n_blocks
        bits = np.zeros(nb * BLOCK_BITS, np.uint8)
        bits[:self.effective_size()] = 1
        return BVector.from_words(bits_to_words(bits)).optimize()


class StrSparseVector:
    """``bm::str_sparse_vector<char, bvector<>, N>`` as the scanner sees it (not remapped): plane 8k+b holds bit b of byte k
    of every element (``basic_bmatrix::set_octet``), ``rows_not_null()`` planes with the trailing empty ones trimmed, NULL
    elements and positions >= size() all zero, and for a nullable vector the NOT-NULL plane."""

    def __init__(self, planes: list[BVector], size: int, not_null: BVector | None = None):
        self.planes = planes
        self.size = int(size)
        self.not_null = not_null
        self.signed = False

    @classmethod
    def from_strings(cls, strs, null_mask=None, optimize: bool = True) -> "StrSparseVector":
        """push_back(s) for every byte string [+ NULL where null_mask] + optimize()"""
        bs = [bytes(x) for x in strs]
        if any(b"\0" in b for b in bs):
            raise ValueError("a string sparse vector holds C strings: no NUL inside a string")
        n = len(bs)
        nl = np.zeros(n, bool) if null_mask is None else np.asarray(null_mask, bool)
        nb = max(1, (n + BLOCK_BITS - 1) // BLOCK_BITS)
        width = max([len(b) for b, z in zip(bs, nl) if not z], default=0)
        mat = np.zeros((nb * BLOCK_BITS, max(width, 1)), np.uint8)
        for i, b in enumerate(bs):
            if b and not nl[i]:
                mat[i, :len(b)] = np.frombuffer(b, np.uint8)
        used = np.bitwise_or.reduce(mat, axis=0)                       # which planes hold any bit
        top = max([j + 1 for j in range(8 * width) if (used[j >> 3] >> (j & 7)) & 1], default=1)
        planes = []
        for j in range(top):
            bits = (mat[:, j >> 3] >> np.uint8(j & 7)) & np.uint8(1)
            bv = BVector.from_words(bits_to_words(bits))
            planes.append(bv.optimize() if optimize else bv)
        nn = None
        if null_mask is not None:
            bits = np.zeros(nb * BLOCK_BITS, np.uint8)
            bits[:n] = ~nl
            nn = BVector.from_words(bits_to_words(bits))
            if optimize:
                nn.optimize()
        return cls(planes, n, nn)

    def effective_slices(self) -> int:
        return len(self.planes)

    universe = SparseVector.universe


class SparseVectorScanner:
    """``bm::sparse_vector_scanner<SV>`` bound to one vector (``bind``): the planes are packed and uploaded once, every
    search is one ``bmb200_scan`` launch.  Searches take one value or a list (a list = one batched launch, the
    scanner's pipeline mode) and return ``BVector`` results; ``count_*`` return cardinalities only."""

    def __init__(self, sv: SparseVector | RscSparseVector, ctx: capi.Context | None = None):
        self.ctx = ctx or capi.default_context()
        self.sv = sv
        self._rsc = isinstance(sv, RscSparseVector)
        self._str = isinstance(sv, StrSparseVector)
        self._float = isinstance(sv, SparseVectorFloat)
        vecs = list(sv.planes) + [sv.universe()]
        if self._rsc:
            # one set as wide as the logical space: compressed planes (NULL past their columns), [0, effective_size), NN
            vecs.append(sv.not_null)
        self._n_blocks = max(v.n_blocks for v in vecs)
        self._ps = PackedSet.pack(vecs, self._n_blocks)
        self._dset = capi.DeviceSet.upload(self.ctx, self._ps)
        self._universe = len(sv.planes)
        self._rs = capi.DeviceRS(self.ctx, self._dset, len(sv.planes) + 1) if self._rsc else None
        # an RSC search scans only the compressed columns
        self._scan_to = max(1, (sv.effective_size() + BLOCK_BITS - 1) // BLOCK_BITS) if self._rsc else 0

    def close(self):
        if self._rs is not None:
            self._rs.free()
            self._rs = None
        if self._dset is not None:
            self._dset.free()
            self._dset = None

    def _run(self, pred, values, count_only=False, signed=None, fl=False):
        """signed: compare as signed values (default: the vector's signedness); find_zero / find_nonzero pass False.
        fl: a float search (the *_float methods), float32 values"""
        if self._str:
            raise TypeError("numeric searches do not apply to a string vector: use find_eq_str / find_eq_str_prefix")
        if fl != self._float:
            raise TypeError("a float vector is searched with the *_float methods" if self._float else "the *_float searches need a SparseVectorFloat")
        signed = self.sv.signed if signed is None else signed
        two = pred in (SCAN_RANGE, SCAN_RANGE_OPEN)
        single = np.ndim(values) == (1 if two else 0)
        dt = np.float32 if fl else np.int64 if signed else np.uint64
        vals = np.atleast_2d(np.asarray(values, dt)) if two else np.atleast_1d(np.asarray(values, dt))
        flags = (F_COUNT_ONLY if count_only else F_OPT_COMPRESS) | (F_SIGNED if signed else 0) | (F_FLOAT if fl else 0)
        res = capi.scan(self.ctx, self._dset, pred, vals, 0, self.sv.effective_slices(), self._universe, flags, 0, self._scan_to)
        return self._results(res, vals.shape[0], count_only, single)

    def _run_in(self, values, count_only=False):
        """elements equal to any of `values` (one SCAN_IN launch); the list is de-duplicated here, and may then hold at most
        capi.SCAN_IN_MAX_VALUES values"""
        if self._str or self._float:
            raise TypeError("find_eq_any / count_eq_any search integer vectors (the reference has no float or string list form)")
        vals = np.unique(np.atleast_1d(np.asarray(values, np.int64 if self.sv.signed else np.uint64)))
        if vals.ndim != 1:
            raise ValueError("find_eq_any takes a 1-D list of values")
        if not vals.size:
            return 0 if count_only else BVector(self._n_blocks)
        flags = (F_COUNT_ONLY if count_only else F_OPT_COMPRESS) | (F_SIGNED if self.sv.signed else 0)
        res = capi.scan(self.ctx, self._dset, SCAN_IN, vals, 0, self.sv.effective_slices(), self._universe, flags, 0, self._scan_to)
        return self._results(res, 1, count_only, True)

    def _run_str(self, strs, prefix, count_only=False):
        if not self._str:
            raise TypeError("string searches need a StrSparseVector")
        single = isinstance(strs, (bytes, bytearray, str))
        qs = [q.encode() if isinstance(q, str) else bytes(q) for q in ([strs] if single else strs)]
        if any(b"\0" in q for q in qs):
            raise ValueError("a query is a C string: no NUL inside it")
        if not qs:
            return []
        flags = (F_COUNT_ONLY if count_only else F_OPT_COMPRESS) | (F_STR_PREFIX if prefix else 0)
        res = capi.scan_str(self.ctx, self._dset, qs, 0, self.sv.effective_slices(), self._universe, flags)
        return self._results(res, len(qs), count_only, single)

    def _results(self, res, nv, count_only, single):
        """a scan's result -> BVector per search (or its count); frees res"""
        try:
            if count_only:                 # rank decompression keeps the count: the totals of the compressed scan are the answer
                t = [int(x) for x in res.group_totals(nv)]
                return t[0] if single else t
            if self._rsc:
                comp, res = res, None
                try:
                    res = capi.rank_decompress(self.ctx, self._rs, comp, F_OPT_COMPRESS)
                finally:
                    comp.free()
            kind, off, bits, gaps = res.fetch()
            nb = self._n_blocks
            out = [result_to_bvector(kind[g * nb:(g + 1) * nb], off[g * nb:(g + 1) * nb], bits, gaps) for g in range(nv)]
            return out[0] if single else out
        finally:
            if res is not None:
                res.free()

    def find_eq(self, value):    return self._run(SCAN_EQ, value)
    def find_gt(self, value):    return self._run(SCAN_GT, value)
    def find_ge(self, value):    return self._run(SCAN_GE, value)
    def find_lt(self, value):    return self._run(SCAN_LT, value)
    def find_le(self, value):    return self._run(SCAN_LE, value)
    def find_range(self, lo, hi=None):
        return self._run(SCAN_RANGE, [lo, hi] if hi is not None else lo)
    # sign-agnostic (the reference ORs every plane, sign included): unsigned EQ 0 / GT 0 also for a signed vector
    def find_zero(self):         return self._run(SCAN_EQ, 0, signed=False)
    def find_nonzero(self):      return self._run(SCAN_GT, 0, signed=False)
    def count_eq(self, value):   return self._run(SCAN_EQ, value, True)
    def count_gt(self, value):   return self._run(SCAN_GT, value, True)
    def count_range(self, lo, hi=None):
        return self._run(SCAN_RANGE, [lo, hi] if hi is not None else lo, True)
    # set membership, SQL `IN (...)`: the elements equal to any listed value, NULLs excluded (a fresh result, not OR-ed into one)
    def find_eq_any(self, values):   return self._run_in(values)
    def count_eq_any(self, values):  return self._run_in(values, True)
    # float vectors: float32 values (one, or a list = one launch); ranges as (from, to) or a list of such rows
    def find_gt_float(self, value):  return self._run(SCAN_GT, value, fl=True)
    def find_ge_float(self, value):  return self._run(SCAN_GE, value, fl=True)
    def find_lt_float(self, value):  return self._run(SCAN_LT, value, fl=True)
    def find_le_float(self, value):  return self._run(SCAN_LE, value, fl=True)
    def find_range_float(self, lo, hi=None):
        return self._run(SCAN_RANGE, [lo, hi] if hi is not None else lo, fl=True)
    def find_range_float_unbounded(self, lo, hi=None):
        return self._run(SCAN_RANGE_OPEN, [lo, hi] if hi is not None else lo, fl=True)
    def count_gt_float(self, value): return self._run(SCAN_GT, value, True, fl=True)
    def count_ge_float(self, value): return self._run(SCAN_GE, value, True, fl=True)
    def count_lt_float(self, value): return self._run(SCAN_LT, value, True, fl=True)
    def count_le_float(self, value): return self._run(SCAN_LE, value, True, fl=True)
    def count_range_float(self, lo, hi=None):
        return self._run(SCAN_RANGE, [lo, hi] if hi is not None else lo, True, fl=True)
    def count_range_float_unbounded(self, lo, hi=None):
        return self._run(SCAN_RANGE_OPEN, [lo, hi] if hi is not None else lo, True, fl=True)
    # string vectors: one query (bytes / str) or a list of them (one launch)
    def find_eq_str(self, s):         return self._run_str(s, False)
    def find_eq_str_prefix(self, s):  return self._run_str(s, True)
    def count_eq_str(self, s):        return self._run_str(s, False, True)


def _mismatch_set(sv1: SparseVector, sv2: SparseVector, use_null: bool, ctx):
    """both vectors' planes, then their NOT-NULL vectors, in one uploaded set with columns covering max(size) -> dset, args"""
    for sv in (sv1, sv2):
        if type(sv) is not SparseVector:
            raise TypeError("find_mismatch / find_first_mismatch compare two plain SparseVector (not RSC, float or string)")
    vecs = list(sv1.planes) + list(sv2.planes)
    nn = []
    for sv in (sv1, sv2):
        nn.append(len(vecs) if sv.not_null is not None else capi.NO_UNIVERSE)
        if sv.not_null is not None:
            vecs.append(sv.not_null)
    nb = max([max(1, (max(sv1.size, sv2.size) + BLOCK_BITS - 1) // BLOCK_BITS)] + [v.n_blocks for v in vecs])
    dset = capi.DeviceSet.upload(ctx, PackedSet.pack(vecs, nb))
    args = capi.mismatch_args(0, len(sv1.planes), len(sv1.planes), len(sv2.planes), nn[0], nn[1], sv1.size, sv2.size,
                              capi.MM_USE_NULL if use_null else capi.MM_NO_NULL, F_OPT_COMPRESS)
    return dset, args


def find_mismatch(sv1: SparseVector, sv2: SparseVector, use_null: bool = True, ctx: capi.Context | None = None) -> BVector:
    """sparse_vector_find_mismatch(bv, sv1, sv2, use_null ? bm::use_null : bm::no_null): the positions where the vectors'
    values or sizes differ, and with use_null where exactly one of them is NULL (without it, positions NULL in both vectors
    are left out).  With use_null and two non-nullable vectors the reference reports every position up to bm::id_max; this
    adds no NULL term there (DESIGN.md 3.5f)."""
    ctx = ctx or capi.default_context()
    dset, args = _mismatch_set(sv1, sv2, use_null, ctx)
    res = None
    try:
        res = capi.sv_mismatch(ctx, dset, args)
        return result_to_bvector(*res.fetch())
    finally:
        if res is not None:
            res.free()
        dset.free()


def find_first_mismatch(sv1: SparseVector, sv2: SparseVector, use_null: bool = True, ctx: capi.Context | None = None) -> int | None:
    """sparse_vector_find_first_mismatch(sv1, sv2, midx, ...): the lowest position where the vectors differ, None when they
    do not (the reference then returns false and bm::id_max).  The reference can miss or postpone a difference inside two GAP
    blocks; this returns the true lowest position (DESIGN.md 3.5f)."""
    ctx = ctx or capi.default_context()
    dset, args = _mismatch_set(sv1, sv2, use_null, ctx)
    try:
        return capi.sv_first_mismatch(ctx, dset, args)
    finally:
        dset.free()


class Set2SetTransform:
    """``bm::set2set_11_transform<sparse_vector<unsigned>>`` with the vector attached once (``attach_sv``): its planes and
    NOT-NULL vector are uploaded at construction, and every ``remap(src)`` is one ``bmb200_remap`` launch
    (csrc/remap_kernel.cuh).  ``src`` is a ``BVector`` (uploaded for the call) or a one-group ``DeviceResult`` (a scan or
    aggregation result, read where it lies); the image comes back as a ``BVector``: the values ``sv[i]`` of the ids i of
    ``src`` (inside the NOT-NULL vector of a nullable vector; ids without an element, or past ``size``, of a non-nullable
    vector map to 0).  The value 0xFFFFFFFF (``bm::id_max`` of the 32-bit build) is left out, as the reference leaves it out."""

    ID_MAX = 0xFFFFFFFF

    def __init__(self, sv: SparseVector, ctx: capi.Context | None = None):
        if type(sv) is not SparseVector or sv.signed:
            raise TypeError("set2set_11_transform maps through an unsigned plain SparseVector (not signed, RSC, float or string)")
        if len(sv.planes) > 32:
            raise ValueError("values of a remap translation vector must fit 32 bits")
        self.ctx = ctx or capi.default_context()
        self.sv = sv
        vecs = list(sv.planes) + ([sv.not_null] if sv.not_null is not None else [])
        self._not_null = len(sv.planes) if sv.not_null is not None else capi.NO_UNIVERSE
        self._dset = capi.DeviceSet.upload(self.ctx, PackedSet.pack(vecs, max(v.n_blocks for v in vecs)))

    def close(self):
        if self._dset is not None:
            self._dset.free()
            self._dset = None

    def remap(self, src: BVector | capi.DeviceResult) -> BVector:
        if self.sv.size == 0:                                  # an empty vector has an empty image
            return BVector(1)
        own, dset = None, None
        try:
            if isinstance(src, BVector):
                # the input enters as a result, the form bmb200_remap reads: a one-source OR copies it
                dset = capi.DeviceSet.upload(self.ctx, PackedSet.pack([src]))
                own = src = capi.aggregate(self.ctx, dset, capi.OP_OR, [0])
            res = capi.remap(self.ctx, self._dset, src, 0, len(self.sv.planes), self._not_null, self.ID_MAX, F_OPT_COMPRESS)
            try:
                return result_to_bvector(*res.fetch())
            finally:
                res.free()
        finally:
            if own is not None:
                own.free()
            if dset is not None:
                dset.free()
