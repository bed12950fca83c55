"""Scanner searches over float sparse vectors (bm::sparse_vector_float<sparse_vector<unsigned>>).

The planes are [signs_, mantissa 0..22, exponent 0..7]: plane 1 + k is bit k of the magnitude bits & 0x7fffffff.
bmb200_scan with F_FLOAT compares the elements with float32 search values in the IEEE sign-magnitude total order of the bits,
key(b) = sign ? ~b : b | 0x80000000, and swaps reversed range bounds by IEEE `from > to` (a NaN bound never swaps; +0 / -0 do
not swap).  That is what the reference's find_*_float compute; this file restates it and checks it:
CPU: the Python mirror's planes == the reference's own; orc_scan_float (the restated contract, oracle/bm_oracle_float.c) ==
the reference's float scanner on a grid of special values, every predicate and every ordered pair of bounds; orc_scan_float ==
an independent numpy key() model.
GPU: bmb200_scan with F_FLOAT == orc_scan_float under every launch variant, every argument rule, and SparseVectorScanner ==
the reference's scanner.
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
from bitmagic_b200.capi import (BLOCK_BITS, BLOCK_WORDS, GAP_MAX_WORDS, F_FLOAT, F_SIGNED, SCAN_RANGE_OPEN, ScanArgsC, lib, ptr)
from bitmagic_b200.hostfmt import BVector, PackedSet, bits_to_words
from test_launch_variants import assert_oracle, collect

gpu = pytest.mark.gpu
CMP = bm.F_OPT_COMPRESS
PREDS = (bm.SCAN_GT, bm.SCAN_GE, bm.SCAN_LT, bm.SCAN_LE, bm.SCAN_RANGE, SCAN_RANGE_OPEN)
TWO = (bm.SCAN_RANGE, SCAN_RANGE_OPEN)

# special bit patterns: +-0, +-denorm_min, +-FLT_MIN, +-FLT_MAX, +-inf, +-quiet NaN, signalling NaN payloads, +-3e-39 (denormal)
SPECIAL_BITS = [0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x00800000, 0x80800000, 0x7F7FFFFF, 0xFF7FFFFF,
                0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FA00000, 0xFF800001, 0xFFA00000]
SPECIALS = np.array(SPECIAL_BITS, np.uint32).view(np.float32)
_D = np.float32(3e-39)
# 34 search values: the specials, +-3e-39, and ordinary numbers of both signs
GRID = np.concatenate([SPECIALS, np.array([_D, -_D, 1.0, -1.0, 0.5, -0.5, 2.0, -2.0, 1.5, -1.5, 100.0, -100.0, 1e10, -1e10,
                                           3.25e-20, -3.25e-20, 7.0, -7.0], np.float32)])
assert GRID.size == 34


def fbits(x) -> np.ndarray:
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def key(b) -> np.ndarray:
    """the IEEE sign-magnitude total order of float bits, as uint32"""
    b = np.asarray(b, np.uint32)
    return np.where(b >> np.uint32(31), ~b, b | np.uint32(0x80000000))


def ieee_gt(a, b) -> bool:
    """from > to as C++ floats (numpy compares floats the same way: NaN never, +0 == -0)"""
    with np.errstate(invalid="ignore"):
        return bool(np.float32(a) > np.float32(b))


def np_float(bits, ok, pred, a, b=None):
    """the numpy key() model of a float search over element bits, restricted to ok"""
    x = key(bits)
    fa, fb = np.float32(a), np.float32(b if b is not None else 0)
    if pred in TWO and ieee_gt(fa, fb):
        fa, fb = fb, fa
    ka, kb = key(fbits(fa)).item(), key(fbits(fb)).item()
    r = {bm.SCAN_GT: x > ka, bm.SCAN_GE: x >= ka, bm.SCAN_LT: x < ka, bm.SCAN_LE: x <= ka,
         bm.SCAN_RANGE: (x >= ka) & (x <= kb), SCAN_RANGE_OPEN: (x > ka) & (x < kb)}[pred]
    return (r & ok).astype(np.uint8)


# ---------------------------------------------------------------- inputs
def float_inputs(kind: str, nullable: bool):
    """-> values (float32), nulls (uint8 or None).  Three block columns: random bit patterns with the specials sprinkled in
    (bit planes), long runs of two values (FULL / GAP / NULL planes) and a sparse region of +0.0 -- unassigned positions of a
    non-nullable vector -- (GAP planes).  kind "pos": no negatives (empty sign plane); "smallexp": exponents < 128 (7 exponent
    planes); "zeromant": all-zero mantissas; "empty": no element."""
    rng = np.random.default_rng(23 + 5 * int(nullable) + 17 * len(kind))
    if kind == "empty":
        return np.zeros(0, np.float32), (np.zeros(0, np.uint8) if nullable else None)
    n = 2 * BLOCK_BITS + 40000
    b = rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)
    i = np.arange(n)
    b[::331] = np.array(SPECIAL_BITS, np.uint32)[(i[::331] // 331) % len(SPECIAL_BITS)]
    run = (i >= BLOCK_BITS) & (i < 2 * BLOCK_BITS)
    b[run] = np.where((i[run] >> 12) & 1, fbits(np.float32(-2.5)), fbits(np.float32(1.0)))
    sparse = i >= 2 * BLOCK_BITS
    b[sparse] = np.where(rng.random(int(sparse.sum())) < 0.01, b[sparse], 0)
    if kind == "pos":
        b &= np.uint32(0x7FFFFFFF)
    elif kind == "smallexp":
        b &= np.uint32(0xBFFFFFFF)                                        # exponent bit 7 clear
    elif kind == "zeromant":
        b &= np.uint32(0xFF800000)
    nulls = None
    if nullable:
        nulls = (rng.random(n) < 0.3).astype(np.uint8)
        nulls[BLOCK_BITS + 5000:BLOCK_BITS + 30000] = 1                      # a NULL stretch inside the runs
    return b.view(np.float32), nulls


def n_cols(n):
    return max(1, (n + BLOCK_BITS - 1) // BLOCK_BITS)


KINDS = ("mixed", "pos", "smallexp", "zeromant", "empty")
CASES = [(k, nl) for k in KINDS for nl in (False, True)]
CASE_IDS = [f"{k}-{'null' if nl else 'plain'}" for k, nl in CASES]


def all_pairs(vals):
    """every ordered pair of the values: equal, reversed, NaN and (+0, -0) / (-0, +0) bounds included"""
    return np.array([[a, b] for a in vals for b in vals], np.float32)


def scanner_searches():
    """what SparseVectorScanner is checked at against the reference: the grid, and ranges of a subset of it in both orders"""
    sub = GRID[[0, 1, 2, 3, 7, 8, 9, 10, 11, 12, 16, 18, 19, 22, 23, 26, 27]]
    return {p: (all_pairs(sub) if p in TWO else GRID.copy()) for p in PREDS}


# ---------------------------------------------------------------- checkers (oracle/float.mk)
ORACLE_FLOAT = orclib.ORACLE_DIR / "liboracle_float.so"
REF_FLOAT = orclib.ORACLE_DIR / "_ref" / "libbmref_float.so"
_libs = {}


def oracle_float() -> C.CDLL:
    """oracle/liboracle_float.so: the plain-C oracle + orc_scan_float, (re)built with make when stale"""
    if "oracle" not in _libs:
        srcs = [orclib.ORACLE_DIR / f for f in ("bm_oracle.c", "bm_oracle_entropy.c", "bm_synth.c", "bm_oracle_float.c")]
        if not ORACLE_FLOAT.exists() or ORACLE_FLOAT.stat().st_mtime < max(x.stat().st_mtime for x in srcs):
            subprocess.run(["make", "-C", str(orclib.ORACLE_DIR), "-f", "float.mk", str(ORACLE_FLOAT)], check=True, capture_output=True)
        _libs["oracle"] = C.CDLL(str(ORACLE_FLOAT))
    return _libs["oracle"]


def ref_float() -> C.CDLL:
    if "ref" not in _libs:
        _libs["ref"] = C.CDLL(str(REF_FLOAT))
    return _libs["ref"]


def raw_values(pred, values) -> np.ndarray:
    """float32 search values (RANGE / RANGE_OPEN: (from, to) rows) -> their bits as the uint64 slots of bmb200_scan"""
    return np.ascontiguousarray(fbits(values).astype(np.uint64))


def orc_call(ps, pred, vals_u64, plane0, n_planes, universe=0xFFFFFFFF, flags=F_FLOAT | CMP, nb_from=0, nb_to=0, out=True):
    nv = vals_u64.shape[0] if pred in TWO else vals_u64.size
    n = ((nb_to if nb_to else ps.n_blocks) - nb_from) * nv
    a = ScanArgsC(int(plane0), int(n_planes), int(universe), int(pred), int(flags), ptr(vals_u64), int(nv), int(nb_from), int(nb_to))
    kind = np.zeros(n, np.uint8); pop = np.zeros(n, np.uint32); dig = np.zeros(n, np.uint64); nr = np.zeros(n, np.uint32)
    blocks = np.zeros((n, BLOCK_WORDS), np.uint32) if out else None
    gaps = np.zeros((n, GAP_MAX_WORDS), np.uint16) if out else None
    nul = C.c_void_p(0)
    rc = oracle_float().orc_scan_float(C.byref(orclib._pc(ps)), C.byref(a), ptr(kind), ptr(pop), ptr(dig), ptr(nr),
                                       ptr(blocks) if out else nul, ptr(gaps) if out else nul)
    return rc, (kind, pop, dig, nr, blocks, gaps)


def oracle_scan_float(ps, pred, values, plane0, n_planes, universe=0xFFFFFFFF, flags=F_FLOAT | CMP, nb_from=0, nb_to=0):
    """orc_scan_float (bmb200_scan with F_FLOAT restated) -> kind, popcnt, digest, nruns, blocks, gaps (value-major)"""
    rc, out = orc_call(ps, pred, raw_values(pred, values), plane0, n_planes, universe, flags, nb_from, nb_to)
    assert rc == 0, f"orc_scan_float rc={rc}"
    return out


def _recorded(fn):
    """orclib._recorded, keyed on libbmref_float.so: answers under tests/golden/ref, BMB200_RECORD_REF=1 rewrites them"""
    @functools.wraps(fn)
    def call(*args, **kw):
        h = hashlib.sha256(fn.__name__.encode())
        orclib._hash_arg(args, h); orclib._hash_arg(sorted(kw.items()), h)
        path = orclib.GOLDEN_REF / f"{fn.__name__}_{h.hexdigest()[:20]}.npz"
        if REF_FLOAT.exists():
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
def _nulls_arg(nulls):
    return (np.ascontiguousarray(nulls, np.uint8), ) if nulls is not None else (None, )


def dense_words(bv: BVector, nc: int):
    return np.concatenate([bv.block_words(c) if c < bv.n_blocks else np.zeros(BLOCK_WORDS, np.uint32) for c in range(nc)])


@_recorded
def ref_svf_planes_digest(values, nulls):
    """The real sparse_vector_float: sha256 of the dense words of its optimize()d planes in the device layout, then of the
    universe -> (n_planes + 1, 32) uint8"""
    v = np.ascontiguousarray(values, dtype=np.float32)
    nl, = _nulls_arg(nulls)
    nc = n_cols(v.size)
    kind = np.zeros(33 * nc, np.uint8)
    blocks = np.zeros((33 * nc, BLOCK_WORDS), np.uint32)
    gaps = np.zeros((33 * nc, GAP_MAX_WORDS), np.uint16)
    npl = C.c_uint32(0)
    rc = ref_float().ref_svf_planes(ptr(v), ptr(nl) if nl is not None else C.c_void_p(0), C.c_uint64(v.size), C.c_uint32(nc),
                                    C.byref(npl), ptr(kind), ptr(blocks), ptr(gaps))
    assert rc == 0, f"ref_svf_planes rc={rc}"
    return row_digests(blocks[:(npl.value + 1) * nc].reshape(npl.value + 1, nc * BLOCK_WORDS))


def _ref_scan_words(values, nulls, pred, search):
    v = np.ascontiguousarray(values, dtype=np.float32)
    nl, = _nulls_arg(nulls)
    s = np.ascontiguousarray(search, dtype=np.float32)
    ns = s.shape[0] if pred in TWO else s.size
    nc = n_cols(v.size)
    counts = np.zeros(ns, np.uint64); blocks = np.zeros((ns * nc, BLOCK_WORDS), np.uint32)
    rc = ref_float().ref_svf_scan(ptr(v), ptr(nl) if nl is not None else C.c_void_p(0), C.c_uint64(v.size), int(pred), ptr(s),
                                  C.c_uint32(ns), C.c_uint32(nc), ptr(counts), ptr(blocks))
    assert rc == 0, f"ref_svf_scan rc={rc}"
    return counts, blocks.reshape(ns, nc * BLOCK_WORDS)


def row_digests(words) -> np.ndarray:
    """sha256 of every row of result words -> (rows, 32) uint8: a whole-grid answer recorded in a few KB"""
    return np.array([np.frombuffer(hashlib.sha256(np.ascontiguousarray(r).tobytes()).digest(), np.uint8) for r in words])


@_recorded
def ref_svf_scan_digest(values, nulls, pred, search):
    """The same searches -> counts[n_search], sha256 of each result's words [n_search][32]"""
    counts, words = _ref_scan_words(values, nulls, pred, search)
    return counts, row_digests(words)


# ---------------------------------------------------------------- CPU
def test_float_constants_match_header():
    hdr = (orclib.ROOT / "include" / "bmb200.h").read_text()
    assert "#define BMB200_F_FLOAT      32u" in hdr and F_FLOAT == 32 and bm.F_FLOAT == F_FLOAT
    assert "#define BMB200_SCAN_RANGE_OPEN 6" in hdr and SCAN_RANGE_OPEN == 6 and bm.SCAN_RANGE_OPEN == 6


def test_f2u_layout():
    """staged bits: magnitude in bits 1..31, sign in bit 0; -0 stages to 1, +0 to 0"""
    x = np.array([0.0, -0.0, 1.0, -1.0], np.float32)
    assert [int(u) for u in bm.scanner.f2u(x)] == [0, 1, 0x3F800000 << 1, (0x3F800000 << 1) | 1]


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_float_planes_match_reference(case):
    """SparseVectorFloat.from_values builds the reference's planes [signs_, mantissa 0..22, exponent 0..7] and universe"""
    kind, nullable = case
    vals, nulls = float_inputs(kind, nullable)
    ref = ref_svf_planes_digest(vals, nulls)
    sv = bm.SparseVectorFloat.from_values(vals, nulls)
    nc = n_cols(vals.size)
    assert sv.effective_slices() == len(ref) - 1
    want_planes = {"smallexp": 31, "zeromant": 32, "empty": 1}.get(kind)
    if want_planes:
        assert sv.effective_slices() == want_planes, kind
    if kind == "pos":
        assert not R.bits_of(dense_words(sv.planes[0], nc)).any()            # no negatives: the sign plane is empty
    if kind == "zeromant":
        assert all(not R.bits_of(dense_words(sv.planes[j], nc)).any() for j in range(1, 24))
    got = row_digests(np.stack([dense_words(p, nc) for p in list(sv.planes) + [sv.universe()]]))
    for j in range(len(ref)):
        assert np.array_equal(got[j], ref[j]), j


@pytest.mark.parametrize("nullable", [False, True], ids=["plain", "null"])
def test_orc_scan_float_matches_reference_on_grid(nullable):
    """orc_scan_float on the reference's planes == the reference's float scanner and the numpy key() model: every predicate at
    the 34 grid values, and every ordered pair of them as the bounds of both ranges"""
    vals, nulls = float_inputs("mixed", nullable)
    sv = bm.SparseVectorFloat.from_values(vals, nulls)                     # the reference's planes (test_float_planes_match_reference)
    ps, npl = PackedSet.pack(list(sv.planes) + [sv.universe()]), sv.effective_slices()
    ok = np.ones(vals.size, bool) if nulls is None else nulls == 0
    bits = fbits(vals)
    for pred in PREDS:
        search = all_pairs(GRID) if pred in TWO else GRID.copy()
        counts, dig = ref_svf_scan_digest(vals, nulls, pred, search)
        okind, opop, odig, onr, oblk, ogap = oracle_scan_float(ps, pred, search, 0, npl, npl)
        ns = len(search)
        ow = oblk.reshape(ns, -1)
        assert np.array_equal(row_digests(ow), dig), pred
        assert np.array_equal(opop.reshape(ns, -1).sum(1, dtype=np.uint64), counts), pred
        ob = R.bits_of(ow).reshape(ns, -1)[:, :vals.size]
        for k in range(ns):
            a, b = (search[k] if pred in TWO else (search[k], None))
            assert np.array_equal(ob[k], np_float(bits, ok, pred, a, b)), (pred, fbits(a), b)


def test_float_bound_swap_rules():
    """find_range_float(+0, -0) is empty, (-0, +0) holds both zeros, a NaN bound never swaps, equal bounds hold the value"""
    vals = np.array([0.0, -0.0, 1.0, -1.0, np.nan, np.inf, -np.inf, 2.0], np.float32)
    vals[4] = np.array([0x7FC00000], np.uint32).view(np.float32)[0]
    sv = bm.SparseVectorFloat.from_values(vals)
    ps = PackedSet.pack(list(sv.planes) + [sv.universe()])
    npl = sv.effective_slices()
    nan = vals[4]
    cases = [((0.0, -0.0), bm.SCAN_RANGE, []), ((-0.0, 0.0), bm.SCAN_RANGE, [0, 1]), ((1.0, 1.0), bm.SCAN_RANGE, [2]),
             ((1.0, 1.0), SCAN_RANGE_OPEN, []), ((2.0, -1.0), bm.SCAN_RANGE, [0, 1, 2, 3, 7]),
             ((2.0, -1.0), SCAN_RANGE_OPEN, [0, 1, 2]), ((nan, -np.inf), bm.SCAN_RANGE, []),
             ((-np.inf, nan), bm.SCAN_RANGE, [0, 1, 2, 3, 4, 5, 6, 7]), ((-np.inf, nan), SCAN_RANGE_OPEN, [0, 1, 2, 3, 5, 7])]
    for (a, b), pred, want in cases:
        blk = oracle_scan_float(ps, pred, np.array([[a, b]], np.float32), 0, npl, npl)[4]
        got = np.flatnonzero(R.bits_of(blk)[:vals.size]).tolist()
        assert got == want, (a, b, pred, got)


@pytest.mark.parametrize("kind", ["pos", "smallexp", "zeromant"])
def test_orc_scan_float_matches_numpy(kind):
    """orc_scan_float on the mirror's planes == the numpy key() model, nullable vector, grid values and pairs"""
    vals, nulls = float_inputs(kind, True)
    sv = bm.SparseVectorFloat.from_values(vals, nulls)
    ps = PackedSet.pack(list(sv.planes) + [sv.universe()])
    npl = sv.effective_slices()
    ok = nulls == 0
    bits = fbits(vals)
    sub = GRID[::3]
    for pred in PREDS:
        search = all_pairs(sub) if pred in TWO else GRID.copy()
        ob = R.bits_of(oracle_scan_float(ps, pred, search, 0, npl, npl)[4]).reshape(len(search), -1)
        for k in range(len(search)):
            a, b = (search[k] if pred in TWO else (search[k], None))
            assert np.array_equal(ob[k, :vals.size], np_float(bits, ok, pred, a, b)), (kind, pred, k)


def test_float_answers_recorded():
    """every reference answer the tests compare against is recorded (or computed live where the reference is built)"""
    for kind, nullable in CASES:
        vals, nulls = float_inputs(kind, nullable)
        ref_svf_planes_digest(vals, nulls)
        if kind == "empty":
            continue
        for pred, search in scanner_searches().items():
            ref_svf_scan_digest(vals, nulls, pred, search)
    for nullable in (False, True):
        vals, nulls = float_inputs("mixed", nullable)
        for pred in PREDS:
            ref_svf_scan_digest(vals, nulls, pred, all_pairs(GRID) if pred in TWO else GRID.copy())


# ---------------------------------------------------------------- GPU: bmb200_scan with F_FLOAT against orc_scan_float
def plane_set(npl: int, gap_flat: bool, seed=5):
    """Two dummy vectors, then npl float planes of 3 columns (random bits / runs / sparse +0.0), then a GAP universe and a bit
    universe.  -> ps, element bits, universes {name: (vector id, bits)}"""
    rng = np.random.default_rng(seed + npl)
    n = 3 * BLOCK_BITS
    mag = np.uint32((1 << (npl - 1)) - 1)
    b = rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)
    b[::97] = np.array(SPECIAL_BITS, np.uint32)[(np.arange(n)[::97] // 97) % len(SPECIAL_BITS)]
    i = np.arange(n)
    b[BLOCK_BITS:2 * BLOCK_BITS] = np.where((i[BLOCK_BITS:2 * BLOCK_BITS] >> 11) & 1, b[7], b[8])
    b[2 * BLOCK_BITS:] = np.where(rng.random(BLOCK_BITS) < 0.005, b[2 * BLOCK_BITS:], np.uint32(0))
    b = (b & np.uint32(0x80000000)) | (b & mag)                             # magnitudes that fit the npl - 1 magnitude planes
    u = bm.scanner.f2u(b.view(np.float32))
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
    return ps, b, universes


def float_launches(npl, bits, pred):
    """launches of 1, 2, 3, 5 and 64 values (every <VG, MODE> float variant, short last groups) holding the edge values: the
    specials, the grid, stored elements and the smallest magnitude above the top plane"""
    x = bits.view(np.float32)
    above = np.array([min(1 << (npl - 1), 0x7F800000) if npl < 32 else 0x7F800000], np.uint32).view(np.float32)[0]
    base = list(GRID) + [x[123], x[65536 + 1000], x[3], x[140000], above, -above]
    if pred in TWO:
        base = [[a, b] for a, b in zip(base, base[7:] + base[:7])] + [[0.0, -0.0], [-0.0, 0.0], [x[5], x[5]], [above, -above]]
    out, off = [], 0
    for nv in (1, 2, 3, 5, 64):
        s = [base[(off + t) % len(base)] for t in range(nv)]
        if nv >= 3:
            s[-1] = s[0]
        out.append(np.array(s, np.float32))
        off += nv
    return out


@gpu
@pytest.mark.parametrize("npl", [1, 24, 28, 32])
def test_float_scan_launch_variants(ctx, npl):
    """bmb200_scan with F_FLOAT == orc_scan_float (kind, popcount, digest, run count, bits, GAP words) and the numpy key() model, for
    every predicate and 1 / 2 / 3 / 5 / 64 values per launch, plane0 > 0, universes absent / GAP / bit, FLAT and raw GAP planes;
    column sub-ranges, F_COUNT_ONLY, F_OPT_NONE, and a result recycled from an unsigned scan.  npl 24 = no exponent planes,
    28 = trimmed exponent planes"""
    for gap_flat, unis in ((True, ("none", "gap", "bit")), (False, ("gap",))):
        ps, bits, universes = plane_set(npl, gap_flat)
        dset = bm.DeviceSet.upload(ctx, ps)
        for un in unis:
            uni, ubits = universes[un]
            for pred in PREDS:
                for k, search in enumerate(float_launches(npl, bits, pred)):
                    flags = (CMP if (k + pred) % 2 else bm.F_OPT_NONE) | F_FLOAT
                    res = bm.scan(ctx, dset, pred, search, 2, npl, uni, flags)
                    got = collect(res, len(search)); res.free()
                    assert_oracle(got, oracle_scan_float(ps, pred, search, 2, npl, uni, flags), len(search),
                                  f"npl={npl} {un} pred={pred} {fbits(search).tolist()}")
                    gb = R.bits_of(got["blocks"]).reshape(len(search), -1)
                    for g in range(len(search)):
                        a, b = (search[g] if pred in TWO else (search[g], None))
                        assert np.array_equal(gb[g], np_float(bits, ubits.astype(bool), pred, a, b)), (npl, un, pred, g)
                search = float_launches(npl, bits, pred)[2]
                for nb_from, nb_to in ((1, 0), (0, 2), (1, 2)):
                    res = bm.scan(ctx, dset, pred, search, 2, npl, uni, CMP | F_FLOAT, nb_from=nb_from, nb_to=nb_to)
                    got = collect(res, len(search)); res.free()
                    assert_oracle(got, oracle_scan_float(ps, pred, search, 2, npl, uni, CMP | F_FLOAT, nb_from, nb_to),
                                  len(search), f"range {nb_from}-{nb_to}")
                res = bm.scan(ctx, dset, pred, search, 2, npl, uni, bm.F_COUNT_ONLY | F_FLOAT)
                got = collect(res, len(search), stored=False); res.free()
                assert_oracle(got, oracle_scan_float(ps, pred, search, 2, npl, uni, F_FLOAT), len(search), "count-only")
                # an unsigned scan's result recycled by a float one of the same shape
                upred = bm.SCAN_RANGE if pred in TWO else pred
                res = bm.scan(ctx, dset, upred, fbits(search).astype(np.uint64), 2, npl, uni, CMP)
                res = bm.scan(ctx, dset, pred, search, 2, npl, uni, CMP | F_FLOAT, result=res)
                got = collect(res, len(search)); res.free()
                assert_oracle(got, oracle_scan_float(ps, pred, search, 2, npl, uni, CMP | F_FLOAT), len(search), "recycled")
        dset.free()


@gpu
def test_float_scan_bad_arguments(ctx):
    """BMB200_ERR_BADARG: F_FLOAT with F_SIGNED, with SCAN_EQ, with n_planes > 32, a value slot with bits above 31, and
    RANGE_OPEN without F_FLOAT; orc_scan_float refuses the same float calls.  A valid call on the same set succeeds."""
    ps, bits, universes = plane_set(32, True)
    dset = bm.DeviceSet.upload(ctx, ps)
    ok1 = raw_values(bm.SCAN_GT, np.array([1.0, -2.0], np.float32))
    ok2 = raw_values(SCAN_RANGE_OPEN, np.array([[1.0, -2.0]], np.float32))
    big1 = ok1.copy(); big1[1] |= np.uint64(1) << np.uint64(32)
    big2 = ok2.copy(); big2[0, 1] |= np.uint64(1) << np.uint64(63)
    calls = [(bm.SCAN_GT, ok1, 32, F_FLOAT | F_SIGNED), (bm.SCAN_EQ, ok1, 32, F_FLOAT), (bm.SCAN_GT, ok1, 33, F_FLOAT),
             (bm.SCAN_GT, big1, 32, F_FLOAT), (SCAN_RANGE_OPEN, big2, 32, F_FLOAT), (bm.SCAN_RANGE, big2, 32, F_FLOAT),
             (SCAN_RANGE_OPEN, ok2, 32, 0), (SCAN_RANGE_OPEN, ok2, 32, F_SIGNED), (7, ok2, 32, F_FLOAT)]
    for pred, vals, npl, flags in calls:
        nv = vals.shape[0] if pred in TWO else vals.size
        a = ScanArgsC(0, npl, 0xFFFFFFFF, pred, flags | CMP, ptr(vals), nv, 0, 0)
        h = C.c_void_p(0)
        rc = lib().bmb200_scan(ctx._h, dset._h, C.byref(a), C.byref(h))
        assert rc == 2 and not h.value, (pred, npl, flags, rc)
        if flags & F_FLOAT:
            assert orc_call(ps, pred, vals, 0, npl, flags=flags | CMP, out=False)[0] == 2, (pred, npl, flags)
    for pred, vals in ((bm.SCAN_GT, ok1), (SCAN_RANGE_OPEN, ok2)):
        nv = vals.shape[0] if pred in TWO else vals.size
        a = ScanArgsC(2, 32, 0xFFFFFFFF, pred, F_FLOAT | CMP, ptr(vals), nv, 0, 0)
        h = C.c_void_p(0)
        assert lib().bmb200_scan(ctx._h, dset._h, C.byref(a), C.byref(h)) == 0 and h.value
        assert lib().bmb200_result_free(h) == 0
    dset.free()


@gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_float_scanner_against_reference(ctx, case):
    """SparseVectorScanner on plain / nullable float vectors == the reference's float scanner, results and counts, and the public
    names against the numpy key() model"""
    kind, nullable = case
    vals, nulls = float_inputs(kind, nullable)
    nc = n_cols(vals.size)
    ok = np.ones(vals.size, bool) if nulls is None else nulls == 0
    sc = bm.SparseVectorScanner(bm.SparseVectorFloat.from_values(vals, nulls), ctx)
    try:
        if kind == "empty":
            for pred in PREDS:
                assert sc._run(pred, [0.0, 1.0] if pred in TWO else 0.0, fl=True).count() == 0
            return
        for pred, search in scanner_searches().items():
            counts, dig = ref_svf_scan_digest(vals, nulls, pred, search)
            got = sc._run(pred, search, fl=True)
            cnt = sc._run(pred, search, count_only=True, fl=True)
            gd = row_digests(np.stack([dense_words(g, nc) for g in got]))
            for k in range(len(got)):
                assert np.array_equal(gd[k], dig[k]), (pred, fbits(search[k]))
                assert int(counts[k]) == cnt[k] == got[k].count(), (pred, k)
        bits = fbits(vals)
        words = lambda bv: R.bits_of(dense_words(bv, nc))[:vals.size]
        assert np.array_equal(words(sc.find_range_float(-1.0, 1.0)), np_float(bits, ok, bm.SCAN_RANGE, -1.0, 1.0))
        assert np.array_equal(words(sc.find_range_float_unbounded(1.0, -2.5)), np_float(bits, ok, SCAN_RANGE_OPEN, -2.5, 1.0))
        assert np.array_equal(words(sc.find_gt_float(-2.5)), np_float(bits, ok, bm.SCAN_GT, -2.5))
        assert np.array_equal(words(sc.find_ge_float(1.0)), np_float(bits, ok, bm.SCAN_GE, 1.0))
        assert np.array_equal(words(sc.find_lt_float(-0.0)), np_float(bits, ok, bm.SCAN_LT, -0.0))
        assert np.array_equal(words(sc.find_le_float(0.0)), np_float(bits, ok, bm.SCAN_LE, 0.0))
        for fn, pred, args in ((sc.count_gt_float, bm.SCAN_GT, (0.5,)), (sc.count_ge_float, bm.SCAN_GE, (-1.0,)),
                               (sc.count_lt_float, bm.SCAN_LT, (2.0,)), (sc.count_le_float, bm.SCAN_LE, (-2.5,)),
                               (sc.count_range_float, bm.SCAN_RANGE, (1.0, -1.0)),
                               (sc.count_range_float_unbounded, SCAN_RANGE_OPEN, (-3.0, 3.0))):
            assert fn(*args) == int(np_float(bits, ok, pred, *args).sum()), pred
        with pytest.raises(TypeError):
            sc.find_gt(1)
    finally:
        sc.close()


@gpu
def test_float_binding_harness():
    exe = orclib.ORACLE_DIR / "_ref" / "test_float_binding"
    if not exe.exists():
        pytest.skip("oracle/_ref/test_float_binding is built only where the reference tree exists")
    p = subprocess.run([str(exe)], capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-2000:]
    assert "0 failed" in p.stdout
