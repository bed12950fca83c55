"""Sparse-vector mismatch: the reference's sparse_vector_find_mismatch / sparse_vector_find_first_mismatch.

bmb200_sv_mismatch answers the vector form D and bmb200_sv_first_mismatch the lowest set bit of F (include/bmb200.h) in one
launch over both vectors' planes.
CPU: orc_sv_mismatch / orc_sv_first_mismatch (the restated contract, oracle/bm_oracle_mismatch.c) == the reference (recorded as
counts + SHA-256 digests of the result words and first positions) wherever the reference is right, == the closed forms
evaluated with the reference's own bvector ops everywhere, and == numpy.  Both reference defects are pinned on their own.
The oracle runs on the package's own planes of the same values (SparseVector.from_values): the same bits the reference's
sparse_vector holds, in NULL / FULL / GAP / bit blocks.
GPU: both entry points == the oracle under every launch variant, every error case, the Python helpers against the recorded
reference answers, and the C++ binding harnesses (32- and 64-bit addressing).
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
from bitmagic_b200 import scanner
from bitmagic_b200.capi import BLOCK_BITS, BLOCK_WORDS, GAP_MAX_WORDS, MM_NO_NULL, MM_USE_NULL, NO_UNIVERSE, mismatch_args, ptr
from bitmagic_b200.hostfmt import BVector, PackedSet, bits_to_words
from test_launch_variants import assert_oracle, collect

gpu = pytest.mark.gpu
B = BLOCK_BITS
TYPES = {"u32": (0, False, 0, 2**32 - 1), "u64": (1, False, 0, 2**64 - 1), "i32": (2, True, -2**31, 2**31 - 1),
         "i64": (3, True, -2**63, 2**63 - 1)}
PAIRINGS = [(a, b) for a in (False, True) for b in (False, True)]
ID_MAX32 = 0xFFFFFFFF


# ---------------------------------------------------------------- inputs
def base_values(t: str, n: int, seed: int):
    """int64 values (the bits of a uint64 for u64): random (bit planes), runs of two values (FULL / GAP / NULL planes), a sparse
    region of zeros (GAP planes), the type's extremes sprinkled in"""
    _, sgn, lo, hi = TYPES[t]
    rng = np.random.default_rng(seed)
    a, b = (-1000, 1000) if sgn else (1, 2000)
    v = rng.integers(a, b + 1, n).astype(np.int64)
    i = np.arange(n)
    run = (i >= B) & (i < 2 * B)
    v[run] = np.where((i[run] >> 12) & 1, b, a)
    sparse = i >= 2 * B
    v[sparse] = np.where(rng.random(int(sparse.sum())) < 0.01, v[sparse], 0)
    v[::997] = lo if sgn else 0
    v[5::991] = hi if sgn else np.array(hi, np.uint64).view(np.int64)
    return v


def mm_pairs(t: str, nl1: bool, nl2: bool):
    """(name, v1, nulls1, v2, nulls2): identical vectors, single differences at element 0, at the last element and across a
    column boundary, different sizes (inside a column, on a column edge), different plane counts, unrelated vectors"""
    k = TYPES[t][0]
    n = 2 * B + 40000
    v1 = base_values(t, n, 31 + k)
    rng = np.random.default_rng(57 + k + 2 * nl1 + 4 * nl2)
    n1 = (rng.random(n) < 0.3).astype(np.uint8) if nl1 else None
    if n1 is not None:
        n1[B + 5000:B + 30000] = 1

    def nulls(m, flip=0.0):
        if not nl2:
            return None
        out = np.zeros(m, np.uint8) if n1 is None else np.resize(n1, m).copy()
        if n1 is None or flip:
            out |= (rng.random(m) < (flip or 0.3)).astype(np.uint8)
        return out

    out = [("identical", v1, n1, v1.copy(), nulls(n))]
    e = v1.copy(); e[0] ^= 1
    out.append(("first", v1, n1, e, nulls(n)))
    e = v1.copy(); e[-1] ^= 4
    out.append(("last", v1, n1, e, nulls(n)))
    e = v1.copy(); e[B - 1] ^= 2; e[B] ^= 8
    out.append(("column edge", v1, n1, e, nulls(n)))
    out.append(("shorter", v1, n1, v1[:n - 1234].copy(), nulls(n - 1234)))
    out.append(("cut at a column edge", v1, n1, v1[:2 * B].copy(), nulls(2 * B)))
    few = np.abs(v1) % 7 if TYPES[t][1] else v1.view(np.uint64).astype(np.uint64) % np.uint64(7)
    out.append(("fewer planes", v1, n1, few.astype(np.int64), nulls(n, 0.05)))
    out.append(("unrelated", v1, n1, base_values(t, n + 999, 99 + k), nulls(n + 999, 0.2)))
    return out


def make_sv(t, vals, nulls):
    sgn = TYPES[t][1]
    return bm.SparseVector.from_values(vals if sgn else vals.view(np.uint64), nulls, signed=sgn)


def codes(t, vals):
    return bm.scanner.s2u(vals) if TYPES[t][1] else np.asarray(vals, np.int64).view(np.uint64)


def n_cols(n):
    return max(1, (n + B - 1) // B)


def np_forms(t, v1, n1, v2, n2, use_null):
    """numpy restatement of D (vector form) and F (first form) over n_cols(max size) columns -> (D bits, F bits)"""
    sa, sb = v1.size, v2.size
    N = n_cols(max(sa, sb)) * B
    ca = np.zeros(N, np.uint64); cb = np.zeros(N, np.uint64)
    ca[:sa] = np.where(n1.astype(bool), 0, codes(t, v1)) if n1 is not None else codes(t, v1)
    cb[:sb] = np.where(n2.astype(bool), 0, codes(t, v2)) if n2 is not None else codes(t, v2)
    pos = np.arange(N)
    diff = ca != cb
    na = np.zeros(N, bool); nb = np.zeros(N, bool)
    if n1 is not None: na[:sa] = n1 == 0
    if n2 is not None: nb[:sb] = n2 == 0
    ha, hb = n1 is not None, n2 is not None
    D = diff | ((pos >= min(sa, sb)) & (pos < max(sa, sb)))
    F = diff.copy()
    if use_null:
        if ha and hb: D |= na ^ nb; F |= na ^ nb
        elif ha: D |= (pos < sa) & ~na; F |= na ^ (pos < sb)
        elif hb: D |= (pos < sb) & ~nb; F |= nb ^ (pos < sa)
    else:
        if ha and hb: D &= na | nb
        elif ha: D &= na
        elif hb: D &= nb
    return D.astype(np.uint8), F.astype(np.uint8)


def words_digest(words) -> np.ndarray:
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(words, np.uint32).tobytes()).digest(), np.uint8).copy()


def padded(bits, nc):
    b = np.zeros(nc * B, np.uint8)
    b[:bits.size] = bits[:nc * B]
    return bits_to_words(b)


# ---------------------------------------------------------------- checkers (oracle/mismatch.mk)
ORACLE_MM = orclib.ORACLE_DIR / "liboracle_mismatch.so"
REF_MM = orclib.ORACLE_DIR / "_ref" / "libbmref_mismatch.so"
_libs = {}


def oracle_mm() -> C.CDLL:
    if "oracle" not in _libs:
        srcs = [orclib.ORACLE_DIR / f for f in ("bm_oracle.c", "bm_oracle_entropy.c", "bm_synth.c", "bm_oracle_mismatch.c")]
        if not ORACLE_MM.exists() or ORACLE_MM.stat().st_mtime < max(x.stat().st_mtime for x in srcs):
            subprocess.run(["make", "-C", str(orclib.ORACLE_DIR), "-f", "mismatch.mk", str(ORACLE_MM)], check=True, capture_output=True)
        _libs["oracle"] = C.CDLL(str(ORACLE_MM))
    return _libs["oracle"]


def ref_mm() -> C.CDLL:
    if "ref" not in _libs:
        _libs["ref"] = C.CDLL(str(REF_MM))
    return _libs["ref"]


def oracle_mismatch(ps, a):
    """orc_sv_mismatch -> kind, popcnt, digest, nruns, blocks, gaps (one group)"""
    n = (a.nb_to if a.nb_to else ps.n_blocks) - a.nb_from
    kind = np.zeros(n, np.uint8); pop = np.zeros(n, np.uint32); dig = np.zeros(n, np.uint64); nr = np.zeros(n, np.uint32)
    blocks = np.zeros((n, BLOCK_WORDS), np.uint32); gaps = np.zeros((n, GAP_MAX_WORDS), np.uint16)
    c = orclib._pc(ps)
    rc = oracle_mm().orc_sv_mismatch(C.byref(c), C.byref(a), ptr(kind), ptr(pop), ptr(dig), ptr(nr), ptr(blocks), ptr(gaps))
    assert rc == 0, f"orc_sv_mismatch rc={rc}"
    return kind, pop, dig, nr, blocks, gaps


def oracle_first(ps, a):
    """orc_sv_first_mismatch -> position or None"""
    pos, found = C.c_uint64(0), C.c_int(0)
    c = orclib._pc(ps)
    rc = oracle_mm().orc_sv_first_mismatch(C.byref(c), C.byref(a), C.byref(pos), C.byref(found))
    assert rc == 0, f"orc_sv_first_mismatch rc={rc}"
    assert found.value or pos.value == 2**64 - 1
    return int(pos.value) if found.value else None


def _recorded(fn):
    """orclib._recorded, keyed on libbmref_mismatch.so: answers under tests/golden/ref, BMB200_RECORD_REF=1 rewrites them"""
    @functools.wraps(fn)
    def call(*args, **kw):
        h = hashlib.sha256(fn.__name__.encode())
        orclib._hash_arg(args, h); orclib._hash_arg(sorted(kw.items()), h)
        path = orclib.GOLDEN_REF / f"{fn.__name__}_{h.hexdigest()[:20]}.npz"
        if REF_MM.exists():
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


def _arr(v):
    return np.ascontiguousarray(v, np.int64)


def _nl(nulls):
    return ptr(np.ascontiguousarray(nulls, np.uint8)) if nulls is not None else C.c_void_p(0)


@_recorded
def ref_mm_answers(t, v1, n1, v2, n2):
    """the reference on one pair, both null_proc values (index 0 = no_null, 1 = use_null), over n_cols(max size) + 1 columns:
    -> find_mismatch count[2] + digest[2, 32], find_first_mismatch found[2] + midx[2], and the closed forms through its bvector
    ops: vector form count[2] + digest[2, 32], first form found[2] + midx[2]"""
    v1, v2 = _arr(v1), _arr(v2)
    n1 = None if n1 is None else np.ascontiguousarray(n1, np.uint8)
    n2 = None if n2 is None else np.ascontiguousarray(n2, np.uint8)
    nc = n_cols(max(v1.size, v2.size)) + 1
    cnt = np.zeros(2, np.uint64); dg = np.zeros((2, 32), np.uint8); ff = np.zeros(2, np.int32); fm = np.zeros(2, np.uint64)
    ccnt = np.zeros(2, np.uint64); cdg = np.zeros((2, 32), np.uint8); cf = np.zeros(2, np.int32); cm = np.zeros(2, np.uint64)
    words = np.zeros(nc * BLOCK_WORDS, np.uint32)
    pa = (TYPES[t][0], ptr(v1), _nl(n1), C.c_uint64(v1.size), ptr(v2), _nl(n2), C.c_uint64(v2.size))
    for np_ in (0, 1):
        c, f, m = C.c_uint64(0), C.c_int(0), C.c_uint64(0)
        assert ref_mm().ref_mm_find(*pa, np_, C.c_uint32(nc), C.byref(c), ptr(words)) == 0
        cnt[np_], dg[np_] = c.value, words_digest(words)
        assert ref_mm().ref_mm_first(*pa, np_, C.byref(f), C.byref(m)) == 0
        ff[np_], fm[np_] = f.value, m.value
        assert ref_mm().ref_mm_closed(*pa, np_, 0, C.c_uint32(nc), C.byref(c), ptr(words), C.byref(f), C.byref(m)) == 0
        ccnt[np_], cdg[np_] = c.value, words_digest(words)
        assert ref_mm().ref_mm_closed(*pa, np_, 1, C.c_uint32(nc), C.byref(c), ptr(words), C.byref(f), C.byref(m)) == 0
        cf[np_], cm[np_] = f.value, m.value
    return cnt, dg, ff, fm, ccnt, cdg, cf, cm


def mm_set(svs):
    """(sv1, sv2) -> PackedSet of sv1's planes, sv2's planes, their NOT-NULL vectors, and the args for it"""
    sv1, sv2 = svs
    vecs = list(sv1.planes) + list(sv2.planes)
    nn = []
    for sv in svs:
        nn.append(len(vecs) if sv.not_null is not None else NO_UNIVERSE)
        if sv.not_null is not None:
            vecs.append(sv.not_null)
    nb = max([n_cols(max(sv1.size, sv2.size))] + [v.n_blocks for v in vecs])
    return PackedSet.pack(vecs, nb), dict(plane0_a=0, n_planes_a=len(sv1.planes), plane0_b=len(sv1.planes),
                                          n_planes_b=len(sv2.planes), not_null_a=nn[0], not_null_b=nn[1],
                                          size_a=sv1.size, size_b=sv2.size)


# ---------------------------------------------------------------- CPU
def test_mismatch_header_constants():
    hdr = (orclib.ROOT / "include" / "bmb200.h").read_text()
    assert "#define BMB200_MM_NO_NULL  0" in hdr and "#define BMB200_MM_USE_NULL 1" in hdr
    assert (MM_NO_NULL, MM_USE_NULL) == (0, 1) and (bm.MM_NO_NULL, bm.MM_USE_NULL) == (0, 1)
    for f in ("plane0_a", "n_planes_a", "plane0_b", "n_planes_b", "not_null_a", "not_null_b", "size_a", "size_b", "null_proc",
              "flags", "nb_from", "nb_to"):
        assert f in hdr
    assert C.sizeof(bm.capi.MismatchArgsC) == 56


@pytest.mark.parametrize("t", list(TYPES))
@pytest.mark.parametrize("pairing", PAIRINGS, ids=["plain-plain", "plain-null", "null-plain", "null-null"])
def test_orc_mismatch_matches_reference(t, pairing):
    """orc_sv_mismatch / orc_sv_first_mismatch == numpy, == the closed forms through the reference's bvector ops, and == the
    reference's own functions wherever they are right (its two defects are checked to be the only differences)"""
    nl1, nl2 = pairing
    for name, v1, n1, v2, n2 in mm_pairs(t, nl1, nl2):
        svs = (make_sv(t, v1, n1), make_sv(t, v2, n2))
        ps, kw = mm_set(svs)
        cnt, dg, ff, fm, ccnt, cdg, cf, cm = ref_mm_answers(t, v1, n1, v2, n2)
        nc = ps.n_blocks + 1
        for use in (0, 1):
            what = (t, pairing, name, use)
            a = mismatch_args(**kw, null_proc=use, flags=bm.F_OPT_COMPRESS)
            blk = oracle_mismatch(ps, a)[4]
            ow = np.concatenate([blk.reshape(-1), np.zeros(BLOCK_WORDS, np.uint32)])
            D, F = np_forms(t, v1, n1, v2, n2, use)
            assert np.array_equal(R.bits_of(ow)[:D.size], D), what
            assert np.array_equal(words_digest(ow), cdg[use]) and int(ccnt[use]) == int(D.sum()), what
            if use and not nl1 and not nl2:          # defect 1: the reference adds all of [0, id_max)
                assert int(cnt[use]) == ID_MAX32, what
                assert np.array_equal(words_digest(padded(np.ones(nc * B, np.uint8), nc)), dg[use]), what
            else:
                assert np.array_equal(words_digest(ow), dg[use]) and int(cnt[use]) == int(D.sum()), what
            first = oracle_first(ps, a)
            nz = np.flatnonzero(F)
            assert first == (int(nz[0]) if nz.size else None), what
            assert bool(cf[use]) == (first is not None) and (first is None or int(cm[use]) == first), what
            if bool(ff[use]) != bool(cf[use]) or int(fm[use]) != int(cm[use]):      # defect 2: missed or postponed only
                assert first is not None and (not ff[use] or int(fm[use]) > first), what
            if first is None:
                assert not ff[use] and int(fm[use]) == ID_MAX32, what


def test_reference_defect_use_null_without_nulls():
    """defect 1: use_null with two non-nullable vectors -- the reference reports every position [0, id_max), the closed form
    through its bvector ops and orc_sv_mismatch add no NULL term"""
    v1 = np.arange(B, dtype=np.int64) % 5
    v2 = v1 + 1
    cnt, dg, ff, fm, ccnt, cdg, cf, cm = ref_mm_answers("u32", v1, None, v2, None)
    assert int(cnt[1]) == ID_MAX32 and int(ccnt[1]) == B == int(cnt[0])
    ps, kw = mm_set((make_sv("u32", v1, None), make_sv("u32", v2, None)))
    o = oracle_mismatch(ps, mismatch_args(**kw, null_proc=MM_USE_NULL))
    assert int(o[1].sum()) == B and np.array_equal(words_digest(np.concatenate([o[4].reshape(-1), np.zeros(BLOCK_WORDS, np.uint32)])), cdg[1])


@pytest.mark.parametrize("split", [(1000, 1000), (10, 20)])
def test_reference_defect_gap_first_runs(split):
    """defect 2: GAP x GAP planes whose first runs differ.  {[0,999]} vs {[1000,65535]}: the reference finds nothing;
    {[0,9]} vs {[20,65535]}: it answers 10.  The true first difference is 0 (closed form through its bvector ops, orc)."""
    e1, s2 = split
    i = np.arange(B)
    v1 = (i < e1).astype(np.int64)
    v2 = (i >= s2).astype(np.int64)
    cnt, dg, ff, fm, ccnt, cdg, cf, cm = ref_mm_answers("u32", v1, None, v2, None)
    for use in (0, 1):
        assert cf[use] and int(cm[use]) == 0
        if split == (1000, 1000):
            assert not ff[use] and int(fm[use]) == ID_MAX32
        else:
            assert ff[use] and int(fm[use]) == 10
    ps, kw = mm_set((make_sv("u32", v1, None), make_sv("u32", v2, None)))
    assert all((int(d) & 3) == bm.BLK_GAP for d in ps.desc)                       # the planes are GAP blocks
    assert oracle_first(ps, mismatch_args(**kw, null_proc=MM_NO_NULL)) == 0


def test_mismatch_answers_recorded():
    """every reference answer the GPU tests compare against is recorded (or computed live where the reference is built)"""
    for t in TYPES:
        for nl1, nl2 in PAIRINGS:
            for name, v1, n1, v2, n2 in mm_pairs(t, nl1, nl2):
                ref_mm_answers(t, v1, n1, v2, n2)


# ---------------------------------------------------------------- GPU: the C ABI against the oracle
def plane_set(npa: int, npb: int, nn_kind: str, gap_flat: bool, seed=9, ncols=3):
    """Two dummy vectors, then npa planes of A and npb planes of B over ncols columns (B = A with a few differences per
    column and random extra planes), then NA and NB as GAP or bit vectors (nn_kind 'none' / 'gap' / 'bit').
    -> ps, kw of the mismatch args"""
    rng = np.random.default_rng(seed + 7 * npa + npb)
    n = ncols * B
    ua = rng.integers(0, 2**63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)
    i = np.arange(n)
    ua[:B // 2] %= np.uint64(3000)
    if ncols > 1:
        ua[B:2 * B] = np.where((i[B:2 * B] >> 11) & 1, ua[7], ua[8])
    if ncols > 2:
        ua[2 * B:] = np.where(rng.random(n - 2 * B) < 0.005, ua[2 * B:], np.uint64(0))
    ub = ua.copy()
    ub[rng.integers(0, n, 40)] ^= rng.integers(0, 2**63, 40, dtype=np.uint64)
    ub[-1] ^= np.uint64(1)

    def planes(u, k):
        out = []
        for j in range(k):
            bv = BVector.from_words(bits_to_words(((u >> np.uint64(j)) & np.uint64(1)).astype(np.uint8)))
            out.append(bv.optimize() if j % 3 else bv)
        return out
    vecs = [BVector.from_words(bits_to_words((rng.random(n) < 0.5).astype(np.uint8))) for _ in range(2)]
    vecs += planes(ua, npa) + planes(ub, npb)
    kw = dict(plane0_a=2, n_planes_a=npa, plane0_b=2 + npa, n_planes_b=npb, not_null_a=NO_UNIVERSE, not_null_b=NO_UNIVERSE,
              size_a=n - 3000, size_b=n - 1000)
    if nn_kind != "none":
        for k in range(2):
            bits = ((i // (2000 + 300 * k)) % 2 == 0).astype(np.uint8) if nn_kind == "gap" else (rng.random(n) < 0.7).astype(np.uint8)
            bv = BVector.from_words(bits_to_words(bits))
            kw["not_null_a" if k == 0 else "not_null_b"] = len(vecs)
            vecs.append(bv.optimize() if nn_kind == "gap" else bv)
    return PackedSet.pack(vecs, ncols, gap_flat=gap_flat), kw


def check(ctx, dset, ps, a, result=None, what=""):
    stored = not a.flags & bm.F_COUNT_ONLY
    res = bm.sv_mismatch(ctx, dset, a, result=result)
    got = collect(res, 1, stored); res.free()
    assert_oracle(got, oracle_mismatch(ps, a), 1, what)
    assert bm.sv_first_mismatch(ctx, dset, a) == oracle_first(ps, a), what + " first"


@gpu
@pytest.mark.parametrize("np_", [(1, 1), (2, 1), (21, 21), (33, 21), (64, 64), (21, 64)], ids=lambda x: f"{x[0]}-{x[1]}")
def test_sv_mismatch_launch_variants(ctx, np_):
    """bmb200_sv_mismatch == orc_sv_mismatch (kind, popcount, digest, run count, bits, GAP words) and bmb200_sv_first_mismatch
    == orc_sv_first_mismatch: plane0 > 0, n_planes_a != n_planes_b, NOT-NULL vectors absent / GAP / bit (and one-sided), FLAT
    and raw GAP planes, both null_proc values, every flag, column sub-ranges, a result recycled from a scan"""
    npa, npb = np_
    for gap_flat, kinds in ((True, ("none", "gap", "bit")), (False, ("gap",))):
        for nn_kind in kinds:
            ps, kw = plane_set(npa, npb, nn_kind, gap_flat)
            dset = bm.DeviceSet.upload(ctx, ps)
            variants = [kw]
            if nn_kind != "none":
                variants += [dict(kw, not_null_b=NO_UNIVERSE), dict(kw, not_null_a=NO_UNIVERSE)]
            for v in variants:
                for use in (MM_NO_NULL, MM_USE_NULL):
                    for flags in (bm.F_OPT_NONE, bm.F_OPT_COMPRESS, bm.F_COUNT_ONLY):
                        a = mismatch_args(**v, null_proc=use, flags=flags)
                        check(ctx, dset, ps, a, what=f"{np_} {nn_kind} flat={gap_flat} use={use} flags={flags} {v['not_null_a']},{v['not_null_b']}")
            for nb_from, nb_to in ((1, 0), (0, 2), (1, 2)):
                a = mismatch_args(**kw, null_proc=MM_USE_NULL, flags=bm.F_OPT_COMPRESS, nb_from=nb_from, nb_to=nb_to)
                check(ctx, dset, ps, a, what=f"{np_} {nn_kind} cols {nb_from}-{nb_to}")
            # equal sizes, the same planes on both sides: nothing differs (the descriptor short cut), found == 0
            same = dict(kw, plane0_b=kw["plane0_a"], n_planes_b=kw["n_planes_a"], not_null_b=kw["not_null_a"], size_b=kw["size_a"])
            a = mismatch_args(**same, null_proc=MM_USE_NULL, flags=bm.F_OPT_COMPRESS)
            check(ctx, dset, ps, a, what=f"{np_} {nn_kind} self")
            assert bm.sv_first_mismatch(ctx, dset, a) is None
            # a multi-value EQ scan's result (3 groups) recycled by the mismatch (one group)
            res = bm.scan(ctx, dset, bm.SCAN_EQ, [0, 1, 2], 2, npa, NO_UNIVERSE, bm.F_OPT_COMPRESS)
            check(ctx, dset, ps, mismatch_args(**kw, null_proc=MM_USE_NULL, flags=bm.F_OPT_COMPRESS), result=res, what=f"{np_} recycled")
            dset.free()


def single_plane_set(ncols, cols_a, cols_b, nn=None):
    """one plane per vector over ncols columns: column c of A / B is a FULL block when c is in cols_a / cols_b, else NULL;
    nn = (NA, NB) as BVectors or None"""
    a, b = BVector(ncols), BVector(ncols)
    for c in cols_a:
        a.set_full(c)
    for c in cols_b:
        b.set_full(c)
    vecs = [a, b] + (list(nn) if nn else [])
    kw = dict(plane0_a=0, n_planes_a=1, plane0_b=1, n_planes_b=1, not_null_a=2 if nn else NO_UNIVERSE,
              not_null_b=3 if nn else NO_UNIVERSE, size_a=ncols * B, size_b=ncols * B)
    return PackedSet.pack(vecs, ncols), kw


@gpu
def test_first_mismatch_positions(ctx):
    """the first form: a difference only at the last bit of the last column; only in the NULL term; many differing columns
    (the earliest wins whatever order the CTAs finish in); equal vectors; a set of 65 540 columns (positions past 2^32)"""
    n = 300
    rng = np.random.default_rng(4)
    # the last bit of the last column
    u = rng.integers(0, 2**21, n * 1024, dtype=np.uint64)
    va = np.zeros(n * B, np.uint64); va[::64] = u
    vb = va.copy(); vb[-1] ^= np.uint64(1 << 20)
    for use in (MM_NO_NULL, MM_USE_NULL):
        sva, svb = bm.SparseVector.from_values(va), bm.SparseVector.from_values(vb)
        ps, kw = mm_set((sva, svb))
        dset = bm.DeviceSet.upload(ctx, ps)
        a = mismatch_args(**kw, null_proc=use)
        assert bm.sv_first_mismatch(ctx, dset, a) == n * B - 1 == oracle_first(ps, a)
        dset.free()
    # only in the NULL term: equal values, NA and NB differ at one bit of column 200
    nulls_a = np.zeros(n * B, np.uint8); nulls_b = nulls_a.copy(); nulls_b[200 * B + 77] = 1
    va2 = va.copy(); va2[200 * B + 77] = 0
    ps, kw = mm_set((bm.SparseVector.from_values(va2, nulls_a), bm.SparseVector.from_values(va2, nulls_b)))
    dset = bm.DeviceSet.upload(ctx, ps)
    assert bm.sv_first_mismatch(ctx, dset, mismatch_args(**kw, null_proc=MM_USE_NULL)) == 200 * B + 77
    assert bm.sv_first_mismatch(ctx, dset, mismatch_args(**kw, null_proc=MM_NO_NULL)) is None
    dset.free()
    # many differing columns, repeated launches: always the earliest
    ps, kw = single_plane_set(2000, range(0, 2000, 2), range(1, 2000, 2))
    dset = bm.DeviceSet.upload(ctx, ps)
    for lo in (0, 1, 777, 1999):
        a = mismatch_args(**kw, null_proc=MM_USE_NULL, nb_from=lo)
        for _ in range(5):
            assert bm.sv_first_mismatch(ctx, dset, a) == lo * B
    dset.free()
    # equal vectors
    ps, kw = single_plane_set(500, range(0, 500, 3), range(0, 500, 3))
    dset = bm.DeviceSet.upload(ctx, ps)
    for use in (MM_NO_NULL, MM_USE_NULL):
        assert bm.sv_first_mismatch(ctx, dset, mismatch_args(**kw, null_proc=use)) is None
        res = bm.sv_mismatch(ctx, dset, mismatch_args(**kw, null_proc=use, flags=bm.F_COUNT_ONLY))
        assert res.group_totals(1)[0] == 0
        res.free()
    dset.free()


@gpu
def test_mismatch_past_65536_columns(ctx):
    """a set of 65 540 columns: differences, sizes and NULL terms past 2^32 bits, both forms"""
    nb = 65540
    rng = np.random.default_rng(3)
    a, b = BVector(nb), BVector(nb)
    wa = bits_to_words((rng.random(B) < 0.4).astype(np.uint8))
    a.set_bits(65537, wa)
    wb = wa.copy(); wb[100] ^= np.uint32(1 << 5)
    b.set_bits(65537, wb)
    na = BVector(nb); na.set_full(65538)
    ps = PackedSet.pack([a, b, na], nb)
    dset = bm.DeviceSet.upload(ctx, ps)
    G = 65537 * B
    kw = dict(plane0_a=0, n_planes_a=1, plane0_b=1, n_planes_b=1, not_null_a=NO_UNIVERSE, not_null_b=NO_UNIVERSE,
              size_a=nb * B, size_b=nb * B - 5)
    a1 = mismatch_args(**kw, null_proc=MM_USE_NULL, flags=bm.F_OPT_COMPRESS, nb_from=65536)
    assert bm.sv_first_mismatch(ctx, dset, a1) == G + 100 * 32 + 5
    check(ctx, dset, ps, a1, what="past 2^32")
    res = bm.sv_mismatch(ctx, dset, a1)
    assert res.group_totals(1)[0] == 1 + 5
    res.free()
    a2 = mismatch_args(**dict(kw, not_null_a=2), null_proc=MM_USE_NULL, flags=bm.F_OPT_COMPRESS, nb_from=65536)
    check(ctx, dset, ps, a2, what="past 2^32, NULL term")
    dset.free()


@gpu
def test_mismatch_errors(ctx):
    """BADARG: other null_proc or flags, more than 64 planes, planes or NOT-NULL ids outside the set; RANGE: column ranges"""
    ps, kw = plane_set(4, 4, "gap", True)
    dset = bm.DeviceSet.upload(ctx, ps)
    M = ps.n_vec
    cases = [(dict(null_proc=2), 2), (dict(flags=bm.F_SIGNED), 2), (dict(flags=bm.F_OR_TARGET), 2),
             (dict(n_planes_a=65, plane0_a=0), 2), (dict(n_planes_b=65, plane0_b=0), 2),
             (dict(plane0_a=M - 3), 2), (dict(plane0_b=M - 1), 2), (dict(not_null_a=M), 2), (dict(not_null_b=M + 5), 2),
             (dict(nb_from=3), 3), (dict(nb_to=4), 3), (dict(nb_from=2, nb_to=1), 3)]
    for kwx, code in cases:
        args = dict(kw, null_proc=MM_USE_NULL, flags=bm.F_OPT_COMPRESS)
        args.update(kwx)
        for fn in (bm.sv_mismatch, bm.sv_first_mismatch):
            with pytest.raises(bm.BMB200Error) as e:
                fn(ctx, dset, mismatch_args(**args))
            assert e.value.code == code, (kwx, fn.__name__)
    # the limits themselves are accepted: 0 planes, 64 planes inside the set
    for kwx in (dict(n_planes_a=0), dict(n_planes_b=0, plane0_b=M)):
        check(ctx, dset, ps, mismatch_args(**dict(kw, **kwx), null_proc=MM_USE_NULL), what=str(kwx))
    dset.free()


@gpu
@pytest.mark.parametrize("t", list(TYPES))
def test_python_helpers_against_reference(ctx, t):
    """scanner.find_mismatch / find_first_mismatch on every pairing == the recorded reference answers (its closed form where
    the reference is defective)"""
    for nl1, nl2 in PAIRINGS:
        for name, v1, n1, v2, n2 in mm_pairs(t, nl1, nl2):
            cnt, dg, ff, fm, ccnt, cdg, cf, cm = ref_mm_answers(t, v1, n1, v2, n2)
            sv1, sv2 = make_sv(t, v1, n1), make_sv(t, v2, n2)
            nc = n_cols(max(v1.size, v2.size)) + 1
            for use in (0, 1):
                what = (t, nl1, nl2, name, use)
                got = scanner.find_mismatch(sv1, sv2, bool(use), ctx)
                gw = got.to_words()
                gw = np.concatenate([gw, np.zeros(nc * BLOCK_WORDS - gw.size, np.uint32)])
                assert np.array_equal(words_digest(gw), cdg[use]) and got.count() == int(ccnt[use]), what
                if not (use and not nl1 and not nl2):
                    assert np.array_equal(words_digest(gw), dg[use]), what
                first = scanner.find_first_mismatch(sv1, sv2, bool(use), ctx)
                assert (first is not None) == bool(cf[use]) and (first is None or first == int(cm[use])), what


@gpu
@pytest.mark.parametrize("exe", ["test_mismatch_binding", "test_mismatch_binding64"])
def test_mismatch_binding_harness(exe):
    path = orclib.ORACLE_DIR / "_ref" / exe
    if not path.exists():
        pytest.skip(f"oracle/_ref/{exe} is built only where the reference tree exists")
    p = subprocess.run([str(path)], capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-2000:]
    assert " 0 failed" in p.stdout
