"""Scanner searches over signed sparse vectors (bm::sparse_vector<int32_t / int64_t>, rsc_sparse_vector<int32_t / int64_t>).

Elements are stored as s2u(x) (plane 0 = sign plane); bmb200_scan with F_SIGNED compares them with int64 search values.
CPU: the Python mirror's signed planes == the reference's own, and orc_scan_signed (the restated contract of a scan with
F_SIGNED, oracle/bm_oracle_signed.c) == the reference's signed scanner.
GPU: bmb200_scan with F_SIGNED == orc_scan_signed under every launch variant, and SparseVectorScanner == the reference's scanner.

The reference's int64_t searches are compared only for search values inside [INT32_MIN, INT32_MAX]: with a value outside
that range its scanner does not compute the comparison (DESIGN.md, signed scanner); there the product is held to the
restated contract (orc_scan_signed, itself checked against numpy here).
"""
from __future__ import annotations

import ctypes as C
import functools
import hashlib
import os
import subprocess

import numpy as np
import pytest

import bitmagic_b200 as bm
import orclib
import rsclib as R
from bitmagic_b200.capi import BLOCK_BITS, BLOCK_WORDS, GAP_MAX_WORDS, F_SIGNED, ScanArgsC, ptr
from bitmagic_b200.hostfmt import BVector, PackedSet, bits_to_words
from test_launch_variants import assert_oracle, collect

gpu = pytest.mark.gpu
CMP = bm.F_OPT_COMPRESS
PREDS = (bm.SCAN_EQ, bm.SCAN_GT, bm.SCAN_GE, bm.SCAN_LT, bm.SCAN_LE, bm.SCAN_RANGE)
ZERO, NONZERO = 6, 7                               # find_zero / find_nonzero in the reference shims' signed entry points
I32 = (-2**31, 2**31 - 1)
I64 = (-2**63, 2**63 - 1)


# ---------------------------------------------------------------- inputs
def signed_inputs(kind: str, is64: bool, nullable: bool):
    """-> values (int64), nulls (uint8 or None).  Three block columns: random values with the type's extremes sprinkled in
    (bit planes), long runs of two values (FULL / GAP / NULL planes), and a sparse region (GAP planes)."""
    lo, hi = I64 if is64 else I32
    rng = np.random.default_rng(11 + 2 * int(is64) + 5 * int(nullable) + 17 * len(kind))
    if kind == "empty":
        return np.zeros(0, np.int64), (np.zeros(0, np.uint8) if nullable else None)
    n = 2 * BLOCK_BITS + 40000
    a, b = {"mixed": (-1000, 1000), "pos": (1, 900), "neg": (-700, -1)}[kind]
    v = rng.integers(a, b + 1, n).astype(np.int64)
    i = np.arange(n)
    run = (i >= BLOCK_BITS) & (i < 2 * BLOCK_BITS)
    v[run] = np.where((i[run] >> 12) & 1, b, a)                          # runs of the two bounds
    sparse = i >= 2 * BLOCK_BITS
    v[sparse] = np.where(rng.random(int(sparse.sum())) < 0.01, v[sparse], 0 if kind == "mixed" else a)
    if kind == "mixed":
        v[::997] = lo; v[5::991] = hi; v[7::983] = -1; v[9::977] = -2; v[11::971] = 1
    elif kind == "pos":
        v[5::991] = hi
    else:
        v[::997] = lo
    nulls = None
    if nullable:
        nulls = (rng.random(n) < 0.3).astype(np.uint8)
        nulls[BLOCK_BITS + 5000:BLOCK_BITS + 30000] = 1                      # a NULL stretch inside the runs
    return v, nulls


def search_values(vals, nulls, is64: bool, ref_range: bool):
    """Edge values: the type's extremes, -2 / -1 / 0 / 1, below the minimum and above the maximum stored, magnitudes with bits above
    the top plane.  ref_range: only values the reference's scanner is checked at (int32 range)."""
    lo, hi = I64 if is64 else I32
    live = vals if nulls is None else vals[nulls == 0]
    s = {lo, lo + 1, hi, hi - 1, -2, -1, 0, 1, 2, -3, 999, -1000, 77}
    if live.size:
        mn, mx = int(live.min()), int(live.max())
        s |= {mn, mx, max(mn - 1, lo), min(mx + 1, hi)}
    s |= {2**20, -2**20 - 1, 2**30, -2**31}
    if is64 and not ref_range:
        s |= {2**40, -2**40, 2**62, -2**62 - 1, 2**31, -2**31 - 1}
    rlo, rhi = I32 if ref_range else (lo, hi)
    return sorted(x for x in s if rlo <= x <= rhi)


def range_pairs(sv):
    """ranges spanning zero, reversed ranges, [v, v], and the extremes"""
    out = [[-5, 5], [5, -5], [0, 0], [-1, -1], [sv[0], sv[-1]], [sv[-1], sv[0]], [-2, 1], [1, -2], [sv[0], -1], [0, sv[-1]]]
    out += [[x, x] for x in sv[::3]]
    out += [[sv[k], sv[-1 - k]] for k in range(0, len(sv) // 2, 2)]
    return out


def searches(vals, nulls, is64, ref_range=True):
    sv = search_values(vals, nulls, is64, ref_range)
    return {p: (np.array(range_pairs(sv), np.int64) if p == bm.SCAN_RANGE else np.array(sv, np.int64)) for p in PREDS}


def n_cols(n):
    return max(1, (n + BLOCK_BITS - 1) // BLOCK_BITS)


CASES = [(k, is64, nl) for k in ("mixed", "pos", "neg", "empty") for is64 in (False, True) for nl in (False, True)]
CASE_IDS = [f"{k}-{'i64' if w else 'i32'}-{'null' if nl else 'plain'}" for k, w, nl in CASES]


# ---------------------------------------------------------------- checkers (oracle/signed.mk)
ORACLE_SIGNED = orclib.ORACLE_DIR / "liboracle_signed.so"
REF_SIGNED = orclib.ORACLE_DIR / "_ref" / "libbmref_signed.so"
_libs = {}


def oracle_signed() -> C.CDLL:
    """oracle/liboracle_signed.so: the plain-C oracle + orc_scan_signed, (re)built with make when stale"""
    if "oracle" not in _libs:
        srcs = [orclib.ORACLE_DIR / f for f in ("bm_oracle.c", "bm_oracle_entropy.c", "bm_synth.c", "bm_oracle_signed.c")]
        if not ORACLE_SIGNED.exists() or ORACLE_SIGNED.stat().st_mtime < max(x.stat().st_mtime for x in srcs):
            subprocess.run(["make", "-C", str(orclib.ORACLE_DIR), "-f", "signed.mk", str(ORACLE_SIGNED)], check=True, capture_output=True)
        _libs["oracle"] = C.CDLL(str(ORACLE_SIGNED))
    return _libs["oracle"]


def ref_signed() -> C.CDLL:
    if "ref" not in _libs:
        _libs["ref"] = C.CDLL(str(REF_SIGNED))
    return _libs["ref"]


def oracle_scan_signed(ps, pred, values, plane0, n_planes, universe=0xFFFFFFFF, flags=0, nb_from=0, nb_to=0):
    """orc_scan_signed (bmb200_scan with F_SIGNED restated) -> kind, popcnt, digest, nruns, blocks, gaps (value-major);
    values are int64 (passed as their two's-complement uint64 bits)"""
    vals = np.ascontiguousarray(np.asarray(values, np.int64).view(np.uint64))
    nv = vals.shape[0] if pred == bm.SCAN_RANGE else vals.size
    n = ((nb_to if nb_to else ps.n_blocks) - nb_from) * nv
    a = ScanArgsC(int(plane0), int(n_planes), int(universe), int(pred), int(flags), ptr(vals), int(nv), int(nb_from), int(nb_to))
    kind = np.zeros(n, np.uint8); pop = np.zeros(n, np.uint32); dig = np.zeros(n, np.uint64); nr = np.zeros(n, np.uint32)
    blocks = np.zeros((n, BLOCK_WORDS), np.uint32); gaps = np.zeros((n, GAP_MAX_WORDS), np.uint16)
    c = orclib._pc(ps)
    rc = oracle_signed().orc_scan_signed(C.byref(c), C.byref(a), ptr(kind), ptr(pop), ptr(dig), ptr(nr), ptr(blocks), ptr(gaps))
    assert rc == 0, f"orc_scan_signed rc={rc}"
    return kind, pop, dig, nr, blocks, gaps


def _recorded(fn):
    """orclib._recorded, keyed on libbmref_signed.so: answers under tests/golden/ref, BMB200_RECORD_REF=1 rewrites them"""
    @functools.wraps(fn)
    def call(*args, **kw):
        h = hashlib.sha256(fn.__name__.encode())
        orclib._hash_arg(args, h); orclib._hash_arg(sorted(kw.items()), h)
        path = orclib.GOLDEN_REF / f"{fn.__name__}_{h.hexdigest()[:20]}.npz"
        if REF_SIGNED.exists():
            out = fn(*args, **kw)
            if os.environ.get("BMB200_RECORD_REF"):
                orclib._save_answer(path, out)
            elif path.exists():
                assert orclib._same_answer(out, orclib._load_answer(path)), f"{path.name} differs from the reference's answer; re-record it"
            return out
        if not path.exists():
            raise FileNotFoundError(f"reference library not built and no recorded answer {path.name} for this {fn.__name__} call")
        return orclib._load_answer(path)
    return call


# ---------------------------------------------------------------- the reference (recorded answers where it is not built)
@_recorded
def ref_svs_planes(values, nulls, is64, max_planes=64):
    """The real sparse_vector<int32_t / int64_t>: its optimize()d s2u planes + the universe, as BVectors (planes..., universe)."""
    v = np.ascontiguousarray(values, dtype=np.int64)
    nl = None if nulls is None else np.ascontiguousarray(nulls, dtype=np.uint8)
    nc = n_cols(v.size)
    kind = np.zeros((max_planes + 1) * nc, np.uint8)
    blocks = np.zeros(((max_planes + 1) * nc, BLOCK_WORDS), np.uint32)
    gaps = np.zeros(((max_planes + 1) * nc, GAP_MAX_WORDS), np.uint16)
    npl = C.c_uint32(0)
    rc = ref_signed().ref_svs_planes(int(is64), ptr(v), ptr(nl) if nl is not None else C.c_void_p(0), C.c_uint64(v.size), C.c_uint32(nc),
                                     C.c_uint32(max_planes), C.byref(npl), ptr(kind), ptr(blocks), ptr(gaps))
    assert rc == 0, f"ref_svs_planes rc={rc}"
    out = []
    for j in range(npl.value + 1):
        bv = BVector(nc)
        for c in range(nc):
            k = int(kind[j * nc + c])
            if k == bm.BLK_FULL:
                bv.set_full(c)
            elif k == bm.BLK_BIT:
                bv.set_bits(c, blocks[j * nc + c])
            elif k == bm.BLK_GAP:
                g = gaps[j * nc + c]
                bv.set_gap(c, g[:(int(g[0]) >> 3) + 1])
        out.append(bv)
    return out


@_recorded
def ref_svs_scan(values, nulls, is64, pred, search):
    """The real sparse_vector_scanner<sparse_vector<int32_t / int64_t>> -> counts[n_search], words[n_search][n_cols * 2048]"""
    v = np.ascontiguousarray(values, dtype=np.int64)
    nl = None if nulls is None else np.ascontiguousarray(nulls, dtype=np.uint8)
    s = np.ascontiguousarray(search, dtype=np.int64)
    ns = s.shape[0] if pred == bm.SCAN_RANGE else s.size
    nc = n_cols(v.size)
    counts = np.zeros(ns, np.uint64); blocks = np.zeros((ns * nc, BLOCK_WORDS), np.uint32)
    rc = ref_signed().ref_svs_scan(int(is64), ptr(v), ptr(nl) if nl is not None else C.c_void_p(0), C.c_uint64(v.size), int(pred), ptr(s),
                                   C.c_uint32(ns), C.c_uint32(nc), ptr(counts), ptr(blocks))
    assert rc == 0, f"ref_svs_scan rc={rc}"
    return counts, blocks.reshape(ns, nc * BLOCK_WORDS)


@_recorded
def ref_rscs_planes(values, nulls, is64, max_planes=64):
    """The real rsc_sparse_vector<int32_t / int64_t> -> (effective_size, planes[n_planes][words], nn[words])"""
    v = np.ascontiguousarray(values, dtype=np.int64); nl = np.ascontiguousarray(nulls, dtype=np.uint8)
    nc = n_cols(v.size)
    words = np.zeros((max_planes + 1) * nc * BLOCK_WORDS, np.uint32)
    npl, eff = C.c_uint32(0), C.c_uint64(0)
    rc = ref_signed().ref_rscs_planes(int(is64), ptr(v), ptr(nl), C.c_uint64(v.size), C.c_uint32(nc), C.c_uint32(max_planes),
                                     C.byref(npl), C.byref(eff), ptr(words))
    assert rc == 0, f"ref_rscs_planes rc={rc}"
    w = words.reshape(max_planes + 1, nc * BLOCK_WORDS)
    return int(eff.value), w[:npl.value].copy(), w[npl.value].copy()


@_recorded
def ref_rscs_scan(values, nulls, is64, pred, search):
    """The real sparse_vector_scanner<rsc_sparse_vector<int32_t / int64_t>> -> counts[n_search], words[n_search][n_cols * 2048]"""
    v = np.ascontiguousarray(values, dtype=np.int64); nl = np.ascontiguousarray(nulls, dtype=np.uint8)
    s = np.ascontiguousarray(search, dtype=np.int64)
    ns = s.shape[0] if pred == bm.SCAN_RANGE else s.size
    nc = n_cols(v.size)
    counts = np.zeros(ns, np.uint64); words = np.zeros((ns, nc * BLOCK_WORDS), np.uint32)
    rc = ref_signed().ref_rscs_scan(int(is64), ptr(v), ptr(nl), C.c_uint64(v.size), int(pred), ptr(s), C.c_uint32(ns), C.c_uint32(nc),
                                   ptr(counts), ptr(words))
    assert rc == 0, f"ref_rscs_scan rc={rc}"
    return counts, words


# ---------------------------------------------------------------- numpy model of the signed comparison
def np_signed(vals, ok, pred, a, b=0):
    x = np.asarray(vals, np.int64)
    if pred == bm.SCAN_RANGE and b < a:
        a, b = b, a
    r = {bm.SCAN_EQ: x == a, bm.SCAN_GT: x > a, bm.SCAN_GE: x >= a, bm.SCAN_LT: x < a, bm.SCAN_LE: x <= a,
         bm.SCAN_RANGE: (x >= a) & (x <= b)}[pred]
    return (r & ok).astype(np.uint8)


def vec_words(bv: BVector, nc: int):
    return np.concatenate([bv.block_words(c) if c < bv.n_blocks else np.zeros(BLOCK_WORDS, np.uint32) for c in range(nc)])


# ---------------------------------------------------------------- CPU
def test_f_signed_matches_header():
    hdr = (orclib.ROOT / "include" / "bmb200.h").read_text()
    assert "#define BMB200_F_SIGNED      8u" in hdr and F_SIGNED == 8


def test_s2u_matches_reference_encoding():
    x = np.array([0, 1, -1, 2, -2, I32[0], I32[1], I64[0], I64[1]], np.int64)
    want = [0, 2, 1, 4, 3, 2**32 - 1, 2**32 - 2, 2**64 - 1, 2**64 - 2]
    assert [int(u) for u in bm.scanner.s2u(x)] == want


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_signed_planes_match_reference(case):
    kind, is64, nullable = case
    vals, nulls = signed_inputs(kind, is64, nullable)
    ref = ref_svs_planes(vals, nulls, is64)
    sv = bm.SparseVector.from_values(vals, nulls, signed=True)
    nc = n_cols(vals.size)
    assert sv.signed and sv.effective_slices() == len(ref) - 1
    for j, p in enumerate(sv.planes):
        assert np.array_equal(vec_words(p, nc), vec_words(ref[j], nc)), j
    assert np.array_equal(vec_words(sv.universe(), nc), vec_words(ref[-1], nc))


@pytest.mark.parametrize("case", [c for c in CASES if c[2]], ids=[i for c, i in zip(CASES, CASE_IDS) if c[2]])
def test_rsc_signed_planes_match_reference(case):
    kind, is64, _ = case
    vals, nulls = signed_inputs(kind, is64, True)
    eff, planes, nn = ref_rscs_planes(vals, nulls, is64)
    sv = bm.RscSparseVector.from_values(vals, nulls, signed=True)
    nc = n_cols(vals.size)
    assert sv.signed and sv.effective_size() == eff == int((nulls == 0).sum())
    assert np.array_equal(R.bits_of(nn), R.bits_of(vec_words(sv.not_null, nc)))
    if eff:
        assert sv.effective_slices() == len(planes)
    for j in range(len(planes)):
        assert np.array_equal(R.bits_of(planes[j])[:eff], R.bits_of(vec_words(sv.planes[j], nc))[:eff]), j


def ref_packed(vals, nulls, is64, gap_flat=True):
    """the reference's own planes + universe packed as one set: planes 0..npl-1, universe npl"""
    vecs = ref_svs_planes(vals, nulls, is64)
    return PackedSet.pack(vecs, max(v.n_blocks for v in vecs), gap_flat=gap_flat), len(vecs) - 1


@pytest.mark.parametrize("case", [c for c in CASES if c[0] != "empty"], ids=[i for c, i in zip(CASES, CASE_IDS) if c[0] != "empty"])
def test_orc_scan_signed_matches_reference(case):
    """orc_scan_signed on the reference's own planes == the reference's signed scanner, every predicate and edge value"""
    kind, is64, nullable = case
    vals, nulls = signed_inputs(kind, is64, nullable)
    ps, npl = ref_packed(vals, nulls, is64)
    ok = np.ones(vals.size, bool) if nulls is None else nulls == 0
    for pred, search in searches(vals, nulls, is64).items():
        counts, rw = ref_svs_scan(vals, nulls, is64, pred, search)
        okind, opop, odig, onr, oblk, ogap = oracle_scan_signed(ps, pred, search, 0, npl, npl, CMP | F_SIGNED)
        ns = len(search)
        assert np.array_equal(oblk.reshape(ns, -1), rw), (kind, pred)
        assert np.array_equal(opop.reshape(ns, -1).sum(1, dtype=np.uint64), counts)
        for k in range(ns):                                              # the reference == the signed comparison too
            a, b = (search[k] if pred == bm.SCAN_RANGE else (search[k], 0))
            assert np.array_equal(R.bits_of(rw[k])[:vals.size], np_signed(vals, ok, pred, int(a), int(b))), (pred, a, b)


@pytest.mark.parametrize("is64", [False, True])
def test_find_zero_nonzero_are_unsigned_searches(is64):
    """the reference's find_zero / find_nonzero on a signed vector == orc_scan's unsigned EQ 0 / GT 0 over the same planes"""
    vals, nulls = signed_inputs("mixed", is64, True)
    ps, npl = ref_packed(vals, nulls, is64)
    for pred, opred in ((ZERO, bm.SCAN_EQ), (NONZERO, bm.SCAN_GT)):
        counts, rw = ref_svs_scan(vals, nulls, is64, pred, np.zeros(1, np.int64))
        o = orclib.oracle_scan(ps, opred, [0], 0, npl, npl, CMP)
        assert np.array_equal(o[4].reshape(1, -1), rw) and int(counts[0]) == int(o[1].sum())


def test_orc_scan_signed_beyond_int32():
    """int64 search values outside the int32 range, where the reference is not a comparison: orc_scan_signed == numpy"""
    vals, nulls = signed_inputs("mixed", True, True)
    sv = bm.SparseVector.from_values(vals, nulls, signed=True)
    ps = PackedSet.pack(list(sv.planes) + [sv.universe()])
    npl = sv.effective_slices()
    ok = nulls == 0
    for pred, search in searches(vals, nulls, True, ref_range=False).items():
        blk = oracle_scan_signed(ps, pred, search, 0, npl, npl, CMP | F_SIGNED)[4]
        bits = R.bits_of(blk).reshape(len(search), -1)
        for k in range(len(search)):
            a, b = (search[k] if pred == bm.SCAN_RANGE else (search[k], 0))
            assert np.array_equal(bits[k, :vals.size], np_signed(vals, ok, pred, int(a), int(b))), (pred, a, b)


def test_signed_answers_recorded():
    """every reference answer the GPU tests compare against is recorded (or computed live where the reference is built)"""
    for kind, is64, nullable in CASES:
        vals, nulls = signed_inputs(kind, is64, nullable)
        ref_svs_planes(vals, nulls, is64)
        if nullable:
            ref_rscs_planes(vals, nulls, is64)
        if kind == "empty":
            continue
        for pred, search in searches(vals, nulls, is64).items():
            ref_svs_scan(vals, nulls, is64, pred, search)
            if nullable:
                ref_rscs_scan(vals, nulls, is64, pred, search)
        for pred in (ZERO, NONZERO):
            ref_svs_scan(vals, nulls, is64, pred, np.zeros(1, np.int64))
            if nullable:
                ref_rscs_scan(vals, nulls, is64, pred, np.zeros(1, np.int64))


# ---------------------------------------------------------------- GPU: bmb200_scan with F_SIGNED against orc_scan_signed
def plane_set(npl: int, gap_flat: bool, seed=5):
    """Two dummy vectors, then npl s2u planes of 3 columns (random codes / runs / sparse), then a GAP universe and a bit universe.
    -> ps, codes (u), universes {name: (vector id, bits)}"""
    rng = np.random.default_rng(seed + npl)
    n = 3 * BLOCK_BITS
    top = np.uint64(2**npl - 1) if npl < 64 else np.uint64(2**64 - 1)
    u = rng.integers(0, 2**63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)
    u &= top
    i = np.arange(n)
    u[BLOCK_BITS:2 * BLOCK_BITS] = np.where((i[BLOCK_BITS:2 * BLOCK_BITS] >> 11) & 1, u[7], u[8])
    u[2 * BLOCK_BITS:] = np.where(rng.random(BLOCK_BITS) < 0.005, u[2 * BLOCK_BITS:], np.uint64(1) & top)
    planes = []
    for j in range(npl):
        bv = BVector.from_words(bits_to_words(((u >> np.uint64(j)) & np.uint64(1)).astype(np.uint8)))
        planes.append(bv.optimize() if j % 3 else bv)                      # some planes stay raw bit-blocks
    gap_u = ((i // 3000) % 2 == 0).astype(np.uint8)
    bit_u = (rng.random(n) < 0.7).astype(np.uint8)
    dummies = [BVector.from_words(bits_to_words((rng.random(n) < 0.5).astype(np.uint8))) for _ in range(2)]
    vecs = dummies + planes + [BVector.from_words(bits_to_words(gap_u)).optimize(), BVector.from_words(bits_to_words(bit_u))]
    ps = PackedSet.pack(vecs, 3, gap_flat=gap_flat)
    universes = {"none": (0xFFFFFFFF, np.ones(n, np.uint8)), "gap": (2 + npl, gap_u), "bit": (3 + npl, bit_u)}
    return ps, u, universes


def u2s(u):
    u = np.asarray(u, np.uint64)
    return np.where(u & np.uint64(1), -(u >> np.uint64(1)).astype(np.int64) - 1, (u >> np.uint64(1)).astype(np.int64))


def signed_launches(npl, x, pred):
    """Five launches of 1..5 values (every <VG, MODE, signed> variant) holding the edge values"""
    mag = min(2**(npl - 1), I64[1]) if npl > 1 else 1                     # the smallest magnitude above the top plane (64: none)
    if pred == bm.SCAN_RANGE:
        base = [[I64[0], I64[1]], [-1, 0], [5, -5], [int(x[70000]), int(x[5])], [int(x[65536 + 400])] * 2, [-mag - 1, mag],
                [mag, I64[1]], [I64[0], -mag - 1], [0, 0], [-2, -2]]
    else:
        base = [I64[0], I64[1], -2, -1, 0, 1, int(x[123]), int(x[65536 + 1000]), int(x[3]), mag, -mag - 1, mag - 1, -mag,
                I32[0], I32[1]]
    out, off = [], 0
    for nv in range(1, 6):
        s = [base[(off + t) % len(base)] for t in range(nv)]
        if nv >= 3:
            s[-1] = s[0]
        out.append(np.array(s, np.int64))
        off += nv
    return out


@gpu
@pytest.mark.parametrize("npl", [1, 2, 33, 64])
def test_signed_scan_launch_variants(ctx, npl):
    """bmb200_scan with F_SIGNED == orc_scan_signed (kind, popcount, digest, run count, bits, GAP words) and the numpy comparison, for
    every predicate and 1..5 values per launch, plane0 > 0, universes absent / GAP / bit, FLAT and raw GAP planes; column
    sub-ranges, F_COUNT_ONLY, F_OPT_NONE, and a result recycled from an unsigned scan"""
    for gap_flat, unis in ((True, ("none", "gap", "bit")), (False, ("gap",))):
        ps, u, universes = plane_set(npl, gap_flat)
        x = u2s(u)
        dset = bm.DeviceSet.upload(ctx, ps)
        for un in unis:
            uni, ubits = universes[un]
            for pred in PREDS:
                for k, search in enumerate(signed_launches(npl, x, pred)):
                    flags = (CMP if (k + pred) % 2 else bm.F_OPT_NONE) | F_SIGNED
                    res = bm.scan(ctx, dset, pred, search, 2, npl, uni, flags)
                    got = collect(res, len(search)); res.free()
                    assert_oracle(got, oracle_scan_signed(ps, pred, search, 2, npl, uni, flags), len(search),
                                  f"npl={npl} {un} pred={pred} {search.tolist()}")
                    bits = R.bits_of(got["blocks"]).reshape(len(search), -1)
                    for g in range(len(search)):
                        a, b = (search[g] if pred == bm.SCAN_RANGE else (search[g], 0))
                        assert np.array_equal(bits[g], np_signed(x, ubits.astype(bool), pred, int(a), int(b))), (npl, un, pred, a, b)
                search = signed_launches(npl, x, pred)[2]
                for nb_from, nb_to in ((1, 0), (0, 2), (1, 2)):
                    res = bm.scan(ctx, dset, pred, search, 2, npl, uni, CMP | F_SIGNED, nb_from=nb_from, nb_to=nb_to)
                    got = collect(res, len(search)); res.free()
                    assert_oracle(got, oracle_scan_signed(ps, pred, search, 2, npl, uni, CMP | F_SIGNED, nb_from, nb_to),
                                  len(search), f"range {nb_from}-{nb_to}")
                res = bm.scan(ctx, dset, pred, search, 2, npl, uni, bm.F_COUNT_ONLY | F_SIGNED)
                got = collect(res, len(search), stored=False); res.free()
                assert_oracle(got, oracle_scan_signed(ps, pred, search, 2, npl, uni, F_SIGNED), len(search), "count-only")
                # an unsigned scan's result recycled by a signed one of the same shape
                res = bm.scan(ctx, dset, pred, search.view(np.uint64), 2, npl, uni, CMP)   # the same bits read as unsigned values
                res = bm.scan(ctx, dset, pred, search, 2, npl, uni, CMP | F_SIGNED, result=res)
                got = collect(res, len(search)); res.free()
                assert_oracle(got, oracle_scan_signed(ps, pred, search, 2, npl, uni, CMP | F_SIGNED), len(search), "recycled")
        dset.free()


@gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_signed_scanner_against_reference(ctx, case):
    """SparseVectorScanner on signed plain / nullable vectors (and their RSC forms) == the reference's signed scanner, results and
    counts, find_zero / find_nonzero included"""
    kind, is64, nullable = case
    vals, nulls = signed_inputs(kind, is64, nullable)
    nc = n_cols(vals.size)
    ok = np.ones(vals.size, bool) if nulls is None else nulls == 0
    forms = [("plain", bm.SparseVector.from_values(vals, nulls, signed=True))]
    if nullable:
        forms.append(("rsc", bm.RscSparseVector.from_values(vals, nulls, signed=True)))
    for form, sv in forms:
        sc = bm.SparseVectorScanner(sv, ctx)
        try:
            refscan = ref_rscs_scan if form == "rsc" else ref_svs_scan
            if kind == "empty":
                for pred in PREDS:
                    assert sc._run(pred, [0, 0] if pred == bm.SCAN_RANGE else 0).count() == 0
                continue
            for pred, search in searches(vals, nulls, is64).items():
                counts, rw = refscan(vals, nulls, is64, pred, search)
                got = sc._run(pred, search)
                cnt = sc._run(pred, search, count_only=True)
                for k in range(len(got)):
                    gw = vec_words(got[k], nc)
                    assert np.array_equal(gw, rw[k][:gw.size]), (form, pred, search[k])
                    assert int(counts[k]) == cnt[k] == got[k].count(), (form, pred, k)
            # the public names
            assert np.array_equal(R.bits_of(vec_words(sc.find_range(-5, 5), nc))[:vals.size], np_signed(vals, ok, bm.SCAN_RANGE, -5, 5))
            assert np.array_equal(R.bits_of(vec_words(sc.find_gt(-3), nc))[:vals.size], np_signed(vals, ok, bm.SCAN_GT, -3))
            assert sc.count_range(5, -5) == int(np_signed(vals, ok, bm.SCAN_RANGE, -5, 5).sum())
            for pred, got in ((ZERO, sc.find_zero()), (NONZERO, sc.find_nonzero())):
                counts, rw = refscan(vals, nulls, is64, pred, np.zeros(1, np.int64))
                want = R.bits_of(rw[0])[:vals.size]
                if form == "rsc" and pred == NONZERO:
                    # the reference's find_nonzero of an RSC vector answers in compressed positions; the scanner in logical ones
                    want = R.np_rank_decompress(ok.astype(np.uint8), want)
                assert np.array_equal(R.bits_of(vec_words(got, nc))[:vals.size], want), (form, pred)
                assert int(counts[0]) == got.count()
        finally:
            sc.close()


@gpu
def test_signed_binding_harness():
    import subprocess
    exe = orclib.ORACLE_DIR / "_ref" / "test_signed_binding"
    if not exe.exists():
        pytest.skip("oracle/_ref/test_signed_binding is built only where the reference tree exists")
    p = subprocess.run([str(exe)], capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-2000:]
    assert "0 failed" in p.stdout
