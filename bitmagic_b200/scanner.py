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
"""
from __future__ import annotations

import numpy as np

from . import capi
from .capi import F_COUNT_ONLY, F_OPT_COMPRESS, SCAN_EQ, SCAN_GE, SCAN_GT, SCAN_LE, SCAN_LT, SCAN_RANGE
from .hostfmt import BLOCK_BITS, BVector, PackedSet, bits_to_words, result_to_bvector


class SparseVector:
    """``bm::sparse_vector<unsigned, bvector<>>`` as the scanner sees it: ``size()``, ``effective_slices()`` planes and,
    for a nullable vector, the NOT-NULL plane (``get_null_bvector()``)."""

    def __init__(self, planes: list[BVector], size: int, not_null: BVector | None = None):
        self.planes = planes
        self.size = int(size)
        self.not_null = not_null

    @classmethod
    def from_values(cls, values, null_mask=None, optimize: bool = True) -> "SparseVector":
        """import(values) [+ set_null where null_mask] + optimize(): plane j = elements with bit j set."""
        v = np.ascontiguousarray(values, dtype=np.uint64)
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
        return cls(planes, n, nn)

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


class RscSparseVector:
    """``bm::rsc_sparse_vector<unsigned>`` as the scanner sees it: the planes hold only the NOT-NULL elements, packed to the
    positions ``[0, effective_size())`` in index order; ``not_null`` (``get_null_bvector()``) maps them back to the logical
    index space of ``size`` positions."""

    def __init__(self, planes: list[BVector], size: int, not_null: BVector):
        self.planes = planes
        self.size = int(size)
        self.not_null = not_null
        self._eff = not_null.count()

    @classmethod
    def from_values(cls, values, null_mask, optimize: bool = True) -> "RscSparseVector":
        """The nullable sparse vector of from_values(values, null_mask), rank-compressed (rsc_sparse_vector::load_from)."""
        v = np.ascontiguousarray(values, dtype=np.uint64)
        keep = ~np.asarray(null_mask, bool)
        dense = SparseVector.from_values(v[keep], None, optimize)
        nb = max(1, (v.size + BLOCK_BITS - 1) // BLOCK_BITS)
        bits = np.zeros(nb * BLOCK_BITS, np.uint8)
        bits[:v.size] = keep
        nn = BVector.from_words(bits_to_words(bits))
        return cls(dense.planes, v.size, nn.optimize() if optimize else nn)

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


class SparseVectorScanner:
    """``bm::sparse_vector_scanner<SV>`` bound to one vector (``bind``): the planes are packed and uploaded once, every
    search is one ``bmb200_scan`` launch.  Searches take one value or a list (a list = one batched launch, the
    scanner's pipeline mode) and return ``BVector`` results; ``count_*`` return cardinalities only."""

    def __init__(self, sv: SparseVector | RscSparseVector, ctx: capi.Context | None = None):
        self.ctx = ctx or capi.default_context()
        self.sv = sv
        self._rsc = isinstance(sv, RscSparseVector)
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

    def _run(self, pred, values, count_only=False):
        single = np.ndim(values) == (1 if pred == SCAN_RANGE else 0)
        vals = np.atleast_2d(values) if pred == SCAN_RANGE else np.atleast_1d(values)
        flags = F_COUNT_ONLY if count_only else F_OPT_COMPRESS
        res = capi.scan(self.ctx, self._dset, pred, vals, 0, self.sv.effective_slices(), self._universe, flags, 0, self._scan_to)
        try:
            nv = vals.shape[0]
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
        return self._run(SCAN_RANGE, np.array([lo, hi], np.uint64) if hi is not None else lo)
    def find_zero(self):         return self._run(SCAN_EQ, 0)
    def find_nonzero(self):      return self._run(SCAN_GT, 0)
    def count_eq(self, value):   return self._run(SCAN_EQ, value, True)
    def count_gt(self, value):   return self._run(SCAN_GT, value, True)
    def count_range(self, lo, hi=None):
        return self._run(SCAN_RANGE, np.array([lo, hi], np.uint64) if hi is not None else lo, True)
