"""Set-membership search (SQL `IN (...)`): the reference's iterator sparse_vector_scanner::find_eq(sv, start, end, bv_out).

bmb200_scan with SCAN_IN answers R = U & {i : code(i) in codes(list)} in one launch for the whole list.
CPU: orc_scan_in (the restated contract, oracle/bm_oracle_in.c) on the reference's own planes == the reference's iterator
find_eq (recorded as counts + SHA-256 digests of the result words) and == np.isin & U; the reference's bv_out semantics (OR into
bv_out, correct_nulls when 0 is listed) match the model the C++ binding mirrors; RSC: the OR of the reference's single-value
find_eq == np.isin & NOT-NULL in logical positions.
GPU: bmb200_scan(SCAN_IN) == orc_scan_in under every launch variant and list length, SparseVectorScanner.find_eq_any /
count_eq_any == the reference, and the C++ binding harness.

Signed int64 lists with values outside the int32 range are held to orc_scan_in and numpy only (the reference's int64 searches
do not compute the comparison there; DESIGN.md, signed scanner).
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
from bitmagic_b200.capi import BLOCK_BITS, BLOCK_WORDS, GAP_MAX_WORDS, F_SIGNED, SCAN_IN, SCAN_IN_MAX_VALUES, ScanArgsC, ptr
from bitmagic_b200.hostfmt import BVector, PackedSet, bits_to_words
from test_launch_variants import assert_oracle, collect

gpu = pytest.mark.gpu
CMP = bm.F_OPT_COMPRESS
TYPES = {"u32": (0, False, 0, 2**32 - 1), "u64": (1, False, 0, 2**64 - 1), "i32": (2, True, -2**31, 2**31 - 1),
         "i64": (3, True, -2**63, 2**63 - 1)}
CASES = [(t, nl) for t in TYPES for nl in (False, True)]
CASE_IDS = [f"{t}-{'null' if nl else 'plain'}" for t, nl in CASES]
STAGE = 4096                                       # codes staged in shared memory by scan_in_kernel (kInStage)


# ---------------------------------------------------------------- inputs
def in_inputs(t: str, nullable: bool):
    """-> values (int64; the bits of a uint64 for u64), nulls (uint8 or None).  Three block columns: random values (bit planes),
    runs of two values (FULL / GAP / NULL planes), a sparse region of zeros (GAP planes); the type's extremes sprinkled in."""
    _, sgn, lo, hi = TYPES[t]
    rng = np.random.default_rng(31 + 3 * TYPES[t][0] + int(nullable))
    n = 2 * BLOCK_BITS + 40000
    a, b = (-1000, 1000) if sgn else (1, 2000)
    v = rng.integers(a, b + 1, n).astype(np.int64)
    i = np.arange(n)
    run = (i >= BLOCK_BITS) & (i < 2 * BLOCK_BITS)
    v[run] = np.where((i[run] >> 12) & 1, b, a)
    sparse = i >= 2 * BLOCK_BITS
    v[sparse] = np.where(rng.random(int(sparse.sum())) < 0.01, v[sparse], 0)
    v[::997] = np.array(lo).astype(np.int64) if sgn else 0
    v[5::991] = np.array(hi, dtype=np.uint64).view(np.int64) if not sgn else hi
    nulls = None
    if nullable:
        nulls = (rng.random(n) < 0.3).astype(np.uint8)
        nulls[BLOCK_BITS + 5000:BLOCK_BITS + 30000] = 1
    return v, nulls


def in_lists(t: str, ref_range: bool = True):
    """Lists: 0 alone, one present value, duplicates + absent values + codes above the top plane + the type's extremes, a list
    with 0 inside, and 10^5 values.  ref_range: signed values inside the int32 range only (where the reference is compared)."""
    _, sgn, lo, hi = TYPES[t]
    if sgn and ref_range:
        lo, hi = max(lo, -2**31), min(hi, 2**31 - 1)
    rng = np.random.default_rng(77 + TYPES[t][0])
    a, b = (-1000, 1000) if sgn else (1, 2000)
    cast = (lambda x: np.array(x, np.int64)) if sgn else (lambda x: np.array([int(y) for y in x], np.uint64).view(np.int64))
    big = np.concatenate([rng.integers(max(a - 50, 0) if not sgn else a - 50, b + 50, 60000), rng.integers(0, 1 << 20, 40000)]).astype(np.int64)
    out = [cast([0]), cast([a + 7]), cast([b, b, a, 3, 3, b + 1, 5000, 1 << 21, lo, hi, hi - 1]), cast([0, 17, 0, a, 1 << 30]), big]
    if sgn and not ref_range:
        out.append(np.array([2**40, -2**40, 2**62, -2**62 - 1, 2**31, -2**31 - 1, 0, 5, -5], np.int64))
    return out


def n_cols(n):
    return max(1, (n + BLOCK_BITS - 1) // BLOCK_BITS)


def codes_of(vals, sgn):
    """the stored codes of int64 values (s2u for a signed type, the bits for an unsigned one)"""
    return bm.scanner.s2u(vals) if sgn else np.asarray(vals, np.int64).view(np.uint64)


def np_in(vals, ok, lst, sgn):
    return (np.isin(codes_of(vals, sgn), codes_of(lst, sgn)) & ok).astype(np.uint8)


def words_digest(words) -> np.ndarray:
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(words, np.uint32).tobytes()).digest(), np.uint8).copy()


# ---------------------------------------------------------------- checkers (oracle/in.mk)
ORACLE_IN = orclib.ORACLE_DIR / "liboracle_in.so"
REF_IN = orclib.ORACLE_DIR / "_ref" / "libbmref_in.so"
_libs = {}


def oracle_in() -> C.CDLL:
    if "oracle" not in _libs:
        srcs = [orclib.ORACLE_DIR / f for f in ("bm_oracle.c", "bm_oracle_entropy.c", "bm_synth.c", "bm_oracle_in.c")]
        if not ORACLE_IN.exists() or ORACLE_IN.stat().st_mtime < max(x.stat().st_mtime for x in srcs):
            subprocess.run(["make", "-C", str(orclib.ORACLE_DIR), "-f", "in.mk", str(ORACLE_IN)], check=True, capture_output=True)
        _libs["oracle"] = C.CDLL(str(ORACLE_IN))
    return _libs["oracle"]


def ref_in() -> C.CDLL:
    if "ref" not in _libs:
        _libs["ref"] = C.CDLL(str(REF_IN))
    return _libs["ref"]


def oracle_scan_in(ps, values, plane0, n_planes, universe=0xFFFFFFFF, flags=0, nb_from=0, nb_to=0):
    """orc_scan_in -> kind, popcnt, digest, nruns, blocks, gaps (one group); values int64 or uint64"""
    vals = np.ascontiguousarray(np.asarray(values).astype(np.int64 if np.asarray(values).dtype.kind == "i" else np.uint64).view(np.uint64))
    n = (nb_to if nb_to else ps.n_blocks) - nb_from
    a = ScanArgsC(int(plane0), int(n_planes), int(universe), SCAN_IN, int(flags), ptr(vals), int(vals.size), int(nb_from), int(nb_to))
    kind = np.zeros(n, np.uint8); pop = np.zeros(n, np.uint32); dig = np.zeros(n, np.uint64); nr = np.zeros(n, np.uint32)
    blocks = np.zeros((n, BLOCK_WORDS), np.uint32); gaps = np.zeros((n, GAP_MAX_WORDS), np.uint16)
    c = orclib._pc(ps)
    rc = oracle_in().orc_scan_in(C.byref(c), C.byref(a), ptr(kind), ptr(pop), ptr(dig), ptr(nr), ptr(blocks), ptr(gaps))
    assert rc == 0, f"orc_scan_in rc={rc}"
    return kind, pop, dig, nr, blocks, gaps


def _recorded(fn):
    """orclib._recorded, keyed on libbmref_in.so: answers under tests/golden/ref, BMB200_RECORD_REF=1 rewrites them"""
    @functools.wraps(fn)
    def call(*args, **kw):
        h = hashlib.sha256(fn.__name__.encode())
        orclib._hash_arg(args, h); orclib._hash_arg(sorted(kw.items()), h)
        path = orclib.GOLDEN_REF / f"{fn.__name__}_{h.hexdigest()[:20]}.npz"
        if REF_IN.exists():
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


def _nl(nulls):
    return ptr(nulls) if nulls is not None else C.c_void_p(0)


@_recorded
def ref_in_planes(t, values, nulls, max_planes=64):
    """the real sparse_vector<T>'s optimize()d planes + its universe, as BVectors (planes..., universe)"""
    v = np.ascontiguousarray(values, np.int64)
    nl = None if nulls is None else np.ascontiguousarray(nulls, np.uint8)
    nc = n_cols(v.size)
    kind = np.zeros((max_planes + 1) * nc, np.uint8)
    blocks = np.zeros(((max_planes + 1) * nc, BLOCK_WORDS), np.uint32)
    gaps = np.zeros(((max_planes + 1) * nc, GAP_MAX_WORDS), np.uint16)
    npl = C.c_uint32(0)
    rc = ref_in().ref_in_planes(TYPES[t][0], ptr(v), _nl(nl), C.c_uint64(v.size), C.c_uint32(nc), C.c_uint32(max_planes), C.byref(npl),
                                ptr(kind), ptr(blocks), ptr(gaps))
    assert rc == 0, f"ref_in_planes rc={rc}"
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
def ref_in_find(t, values, nulls, lst, prefill=0):
    """the reference's iterator find_eq into bv_out (pre-filled with every prefill-th position of [0, n + 1000) when prefill > 0)
    -> (count, SHA-256 of the result words over n_cols + 1 columns)"""
    v = np.ascontiguousarray(values, np.int64); s = np.ascontiguousarray(lst, np.int64)
    nl = None if nulls is None else np.ascontiguousarray(nulls, np.uint8)
    nc = n_cols(v.size) + 1
    cnt = C.c_uint64(0); words = np.zeros(nc * BLOCK_WORDS, np.uint32)
    rc = ref_in().ref_in_find(TYPES[t][0], ptr(v), _nl(nl), C.c_uint64(v.size), ptr(s), C.c_uint64(s.size), C.c_uint32(prefill),
                              C.c_uint32(nc), C.byref(cnt), ptr(words))
    assert rc == 0, f"ref_in_find rc={rc}"
    return np.array([cnt.value], np.uint64), words_digest(words)


@_recorded
def ref_in_rsc(t, values, nulls, lst):
    """rsc_sparse_vector<T>: the OR over the list of the single-value find_eq (logical positions) -> (count, SHA-256 of the words)"""
    v = np.ascontiguousarray(values, np.int64); s = np.ascontiguousarray(lst, np.int64)
    nl = np.ascontiguousarray(nulls, np.uint8)
    nc = n_cols(v.size) + 1
    cnt = C.c_uint64(0); words = np.zeros(nc * BLOCK_WORDS, np.uint32)
    rc = ref_in().ref_in_rsc(TYPES[t][0], ptr(v), ptr(nl), C.c_uint64(v.size), ptr(s), C.c_uint64(s.size), 0, C.c_uint32(nc),
                             C.byref(cnt), ptr(words))
    assert rc == 0, f"ref_in_rsc rc={rc}"
    return np.array([cnt.value], np.uint64), words_digest(words)


def padded(bits, nc):
    """a 0/1 array of positions -> dense words of nc columns"""
    b = np.zeros(nc * BLOCK_BITS, np.uint8)
    b[:bits.size] = bits
    return bits_to_words(b)


def ref_packed(t, vals, nulls):
    vecs = ref_in_planes(t, vals, nulls)
    return PackedSet.pack(vecs, max(v.n_blocks for v in vecs)), len(vecs) - 1


# ---------------------------------------------------------------- CPU
def test_scan_in_matches_header():
    hdr = (orclib.ROOT / "include" / "bmb200.h").read_text()
    assert "#define BMB200_SCAN_IN     7" in hdr and SCAN_IN == 7 and bm.SCAN_IN == 7
    assert "#define BMB200_SCAN_IN_MAX_VALUES (1u << 20)" in hdr and SCAN_IN_MAX_VALUES == 1 << 20


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_orc_scan_in_matches_reference(case):
    """orc_scan_in on the reference's own planes == the reference's iterator find_eq == np.isin & U, every list; and the
    reference's effect on a pre-filled bv_out == (bv_out | R), then & NOT-NULL when 0 is listed (what the binding mirrors)"""
    t, nullable = case
    sgn = TYPES[t][1]
    vals, nulls = in_inputs(t, nullable)
    ps, npl = ref_packed(t, vals, nulls)
    ok = np.ones(vals.size, bool) if nulls is None else nulls == 0
    nc = n_cols(vals.size) + 1
    for lst in in_lists(t):
        cnt, dg = ref_in_find(t, vals, nulls, lst)
        blk = oracle_scan_in(ps, lst, 0, npl, npl, CMP | (F_SIGNED if sgn else 0))[4]
        ow = np.concatenate([blk.reshape(-1), np.zeros((nc - blk.shape[0]) * BLOCK_WORDS, np.uint32)])
        want = np_in(vals, ok, lst, sgn)
        assert np.array_equal(R.bits_of(ow)[:vals.size], want), (t, lst[:4])
        assert np.array_equal(words_digest(ow), dg) and int(cnt[0]) == int(want.sum()), (t, lst[:4])
        pre = np.zeros(vals.size + 1000, np.uint8); pre[::7] = 1
        model = pre.copy(); model[:vals.size] |= want
        if nullable and (np.asarray(lst) == 0).any():
            model[:vals.size] &= ok; model[vals.size:] = 0
        pcnt, pdg = ref_in_find(t, vals, nulls, lst, 7)
        assert np.array_equal(words_digest(padded(model, nc)), pdg) and int(pcnt[0]) == int(model.sum()), (t, "prefill", lst[:4])


@pytest.mark.parametrize("t", list(TYPES))
def test_rsc_or_of_find_eq_is_logical(t):
    """rsc_sparse_vector<T>: the OR of the reference's single-value find_eq == np.isin & NOT-NULL in logical positions"""
    sgn = TYPES[t][1]
    vals, nulls = in_inputs(t, True)
    ok = nulls == 0
    nc = n_cols(vals.size) + 1
    for lst in in_lists(t)[:4]:
        cnt, dg = ref_in_rsc(t, vals, nulls, lst)
        want = np_in(vals, ok, lst, sgn)
        assert np.array_equal(words_digest(padded(want, nc)), dg) and int(cnt[0]) == int(want.sum()), (t, lst)


def test_orc_scan_in_beyond_int32():
    """int64 lists outside the int32 range, where the reference is not a comparison: orc_scan_in == numpy"""
    vals, nulls = in_inputs("i64", True)
    sv = bm.SparseVector.from_values(vals, nulls, signed=True)
    ps = PackedSet.pack(list(sv.planes) + [sv.universe()])
    npl = sv.effective_slices()
    ok = nulls == 0
    for lst in in_lists("i64", ref_range=False):
        blk = oracle_scan_in(ps, lst, 0, npl, npl, CMP | F_SIGNED)[4]
        assert np.array_equal(R.bits_of(blk.reshape(-1))[:vals.size], np_in(vals, ok, lst, True)), lst[:4]


def test_in_answers_recorded():
    """every reference answer the GPU tests compare against is recorded (or computed live where the reference is built)"""
    for t, nullable in CASES:
        vals, nulls = in_inputs(t, nullable)
        ref_in_planes(t, vals, nulls)
        for lst in in_lists(t):
            ref_in_find(t, vals, nulls, lst)
            ref_in_find(t, vals, nulls, lst, 7)
        if nullable:
            for lst in in_lists(t)[:4]:
                ref_in_rsc(t, vals, nulls, lst)


# ---------------------------------------------------------------- GPU: bmb200_scan(SCAN_IN) against orc_scan_in
def plane_set(npl: int, gap_flat: bool, seed=9):
    """Two dummy vectors, npl planes of 3 columns (random codes / runs of two codes / sparse), a GAP and a bit universe.
    -> ps, codes, universes {name: (vector id, bits)}"""
    rng = np.random.default_rng(seed + npl)
    n = 3 * BLOCK_BITS
    top = np.uint64(2**npl - 1) if npl < 64 else np.uint64(2**64 - 1)
    u = rng.integers(0, 2**63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)
    u[:BLOCK_BITS // 2] %= np.uint64(3000)                                # repeated small codes: lists hit many elements
    u &= top
    i = np.arange(n)
    u[BLOCK_BITS:2 * BLOCK_BITS] = np.where((i[BLOCK_BITS:2 * BLOCK_BITS] >> 11) & 1, u[7], u[8])
    u[2 * BLOCK_BITS:] = np.where(rng.random(BLOCK_BITS) < 0.005, u[2 * BLOCK_BITS:], np.uint64(0))
    planes = []
    for j in range(npl):
        bv = BVector.from_words(bits_to_words(((u >> np.uint64(j)) & np.uint64(1)).astype(np.uint8)))
        planes.append(bv.optimize() if j % 3 else bv)
    gap_u = ((i // 3000) % 2 == 0).astype(np.uint8)
    bit_u = (rng.random(n) < 0.7).astype(np.uint8)
    dummies = [BVector.from_words(bits_to_words((rng.random(n) < 0.5).astype(np.uint8))) for _ in range(2)]
    vecs = dummies + planes + [BVector.from_words(bits_to_words(gap_u)).optimize(), BVector.from_words(bits_to_words(bit_u))]
    ps = PackedSet.pack(vecs, 3, gap_flat=gap_flat)
    universes = {"none": (0xFFFFFFFF, np.ones(n, np.uint8)), "gap": (2 + npl, gap_u), "bit": (3 + npl, bit_u)}
    return ps, u, universes


def code_lists(u, npl, rng):
    """K = 1, 2, 5, 500: present codes, 0, absent codes, codes above the top plane, duplicates"""
    above = [2**npl, 2**npl + 3, 2**63] if npl < 64 else []
    out = []
    for k in (1, 2, 5, 500):
        lst = list(rng.choice(u, k).astype(np.uint64))
        if k >= 5:
            lst[:5] = [np.uint64(0), u[7], u[7], np.uint64(12345), u[3]]
            lst += [np.uint64(x) for x in above]
        out.append(np.array(lst, np.uint64))
    return out


def check(ctx, dset, ps, lst, npl, uni, flags, ubits=None, x=None, nb_from=0, nb_to=0, result=None, what=""):
    stored = not flags & bm.F_COUNT_ONLY
    res = bm.scan(ctx, dset, SCAN_IN, lst, 2, npl, uni, flags, nb_from, nb_to, result=result)
    got = collect(res, 1, stored); res.free()
    o = oracle_scan_in(ps, lst, 2, npl, uni, flags, nb_from, nb_to)
    assert_oracle(got, o, 1, what)
    if ubits is not None and stored:
        sgn = bool(flags & F_SIGNED)
        want = (np.isin(x, codes_of(lst, True) if sgn else np.asarray(lst, np.uint64)) & ubits.astype(bool)).astype(np.uint8)
        assert np.array_equal(R.bits_of(got["blocks"].reshape(-1)), want), what


@gpu
@pytest.mark.parametrize("npl", [1, 2, 21, 33, 64])
def test_scan_in_launch_variants(ctx, npl):
    """bmb200_scan(SCAN_IN) == orc_scan_in (kind, popcount, digest, run count, bits, GAP words) and np.isin & U: K = 1, 2, 5,
    500 with 0, duplicates, absent codes and codes above the top plane; plane0 > 0; universes absent / GAP / bit; FLAT and raw
    GAP planes; F_OPT_NONE / F_OPT_COMPRESS / F_COUNT_ONLY; F_SIGNED; column sub-ranges; a result recycled from an EQ scan"""
    rng = np.random.default_rng(100 + npl)
    for gap_flat, unis in ((True, ("none", "gap", "bit")), (False, ("gap",))):
        ps, u, universes = plane_set(npl, gap_flat)
        dset = bm.DeviceSet.upload(ctx, ps)
        for un in unis:
            uni, ubits = universes[un]
            for k, lst in enumerate(code_lists(u, npl, rng)):
                tag = f"npl={npl} {un} flat={gap_flat} K={lst.size}"
                check(ctx, dset, ps, lst, npl, uni, CMP if k % 2 else bm.F_OPT_NONE, ubits, u, what=tag)
                check(ctx, dset, ps, lst, npl, uni, bm.F_COUNT_ONLY, what=tag + " count-only")
                # F_SIGNED: the same codes passed as the signed values whose s2u they are
                s = np.where(lst & np.uint64(1), -(lst >> np.uint64(1)).astype(np.int64) - 1, (lst >> np.uint64(1)).astype(np.int64))
                check(ctx, dset, ps, s, npl, uni, CMP | F_SIGNED, ubits, u, what=tag + " signed")
            lst = code_lists(u, npl, rng)[2]
            for nb_from, nb_to in ((1, 0), (0, 2), (1, 2)):
                check(ctx, dset, ps, lst, npl, uni, CMP, nb_from=nb_from, nb_to=nb_to, what=f"npl={npl} {un} cols {nb_from}-{nb_to}")
            # a multi-value EQ scan's result (3 groups) recycled by SCAN_IN (one group)
            res = bm.scan(ctx, dset, bm.SCAN_EQ, lst[:3], 2, npl, uni, CMP)
            check(ctx, dset, ps, lst, npl, uni, CMP, ubits, u, result=res, what=f"npl={npl} {un} recycled")
        dset.free()


@gpu
def test_scan_in_list_lengths(ctx):
    """K = 65 536 and 2^20 (splitters + buckets in global memory), and K at the shared-memory staging bound and +-1"""
    npl = 21
    ps, u, universes = plane_set(npl, True)
    dset = bm.DeviceSet.upload(ctx, ps)
    rng = np.random.default_rng(5)
    present = np.unique(u)
    for k in (STAGE - 1, STAGE, STAGE + 1, 65536, 1 << 20):
        lst = np.unique(np.concatenate([rng.choice(present, min(k // 2, present.size), replace=False),
                                        rng.integers(0, 2**npl, 3 * k, dtype=np.uint64)]))
        lst = rng.permutation(lst[:k] if lst.size >= k else lst)
        assert lst.size == k
        for un in ("none", "bit"):
            uni, ubits = universes[un]
            check(ctx, dset, ps, lst, npl, uni, CMP, ubits, u, what=f"K={k} {un}")
    dset.free()


@gpu
def test_scan_in_past_65536_columns(ctx):
    """a set of 65 540 columns searched from column 65 536 on: the columns past 2^32 bits"""
    npl, nb = 3, 65540
    rng = np.random.default_rng(3)
    codes = rng.integers(0, 8, (4, BLOCK_BITS)).astype(np.uint64)
    planes = []
    for j in range(npl):
        bv = BVector(nb)
        for c in range(4):
            bv.set_bits(65536 + c, bits_to_words(((codes[c] >> np.uint64(j)) & np.uint64(1)).astype(np.uint8)))
        planes.append(bv)
    dummies = [BVector(nb), BVector(nb)]
    ps = PackedSet.pack(dummies + planes, nb)
    dset = bm.DeviceSet.upload(ctx, ps)
    lst = np.array([0, 3, 5], np.uint64)
    res = bm.scan(ctx, dset, SCAN_IN, lst, 2, npl, bm.NO_UNIVERSE, CMP, 65536, 0)
    got = collect(res, 1); res.free()
    want = np.isin(codes, lst).astype(np.uint8)
    assert np.array_equal(R.bits_of(got["blocks"].reshape(-1)), want.reshape(-1))
    assert got["totals"][0] == int(want.sum())
    dset.free()


@gpu
def test_scan_in_errors(ctx):
    """BADARG: F_FLOAT, flags outside COUNT_ONLY / OPT_COMPRESS / SIGNED, an empty list; RANGE: more than SCAN_IN_MAX_VALUES
    values, planes or universe outside the set"""
    ps, u, universes = plane_set(4, True)
    dset = bm.DeviceSet.upload(ctx, ps)
    lst = np.array([1, 2], np.uint64)
    cases = [(dict(values=lst, flags=bm.F_FLOAT), 2), (dict(values=np.zeros(0, np.uint64)), 2), (dict(values=lst, flags=bm.F_OR_TARGET), 2),
             (dict(values=np.arange(SCAN_IN_MAX_VALUES + 1, dtype=np.uint64)), 3), (dict(values=lst, plane0=ps.n_vec - 3), 3),
             (dict(values=lst, universe=ps.n_vec), 3), (dict(values=lst, nb_from=3), 3)]
    for kw, code in cases:
        a = dict(plane0=2, n_planes=4, universe=bm.NO_UNIVERSE, flags=CMP, nb_from=0)
        a.update(kw)
        with pytest.raises(bm.BMB200Error) as e:
            bm.scan(ctx, dset, SCAN_IN, a["values"], a["plane0"], a["n_planes"], a["universe"], a["flags"], a["nb_from"])
        assert e.value.code == code, kw.keys()
    # the longest list is accepted
    res = bm.scan(ctx, dset, SCAN_IN, np.arange(SCAN_IN_MAX_VALUES, dtype=np.uint64), 2, 4, bm.NO_UNIVERSE, CMP)
    assert res.group_totals(1)[0] == 3 * BLOCK_BITS
    res.free()
    dset.free()


@gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_scanner_eq_any_against_reference(ctx, case):
    """SparseVectorScanner.find_eq_any / count_eq_any on plain, nullable, RSC and signed vectors == the reference"""
    t, nullable = case
    sgn = TYPES[t][1]
    vals, nulls = in_inputs(t, nullable)
    nc = n_cols(vals.size) + 1
    ok = np.ones(vals.size, bool) if nulls is None else nulls == 0
    pyvals = vals if sgn else vals.view(np.uint64)
    forms = [("plain", bm.SparseVector.from_values(pyvals, nulls, signed=sgn))]
    if nullable:
        forms.append(("rsc", bm.RscSparseVector.from_values(pyvals, nulls, signed=sgn)))
    for form, sv in forms:
        sc = bm.SparseVectorScanner(sv, ctx)
        try:
            for k, lst in enumerate(in_lists(t)):
                if form == "rsc" and k >= 4:
                    continue
                cnt, dg = ref_in_rsc(t, vals, nulls, lst) if form == "rsc" else ref_in_find(t, vals, nulls, lst)
                q = lst if sgn else lst.view(np.uint64)
                got = sc.find_eq_any(q)
                gw = got.to_words()
                gw = np.concatenate([gw, np.zeros(nc * BLOCK_WORDS - gw.size, np.uint32)])
                assert np.array_equal(words_digest(gw), dg), (form, t, lst[:4])
                assert got.count() == int(cnt[0]) == sc.count_eq_any(q), (form, t, lst[:4])
                assert np.array_equal(R.bits_of(gw)[:vals.size], np_in(vals, ok, lst, sgn)), (form, t)
        finally:
            sc.close()


@gpu
def test_in_binding_harness():
    exe = orclib.ORACLE_DIR / "_ref" / "test_in_binding"
    if not exe.exists():
        pytest.skip("oracle/_ref/test_in_binding is built only where the reference tree exists")
    p = subprocess.run([str(exe)], capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-2000:]
    assert "0 failed" in p.stdout
