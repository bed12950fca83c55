"""Scanner string searches over string sparse vectors (bm::str_sparse_vector<char, bvector<>, N>).

Plane 8k+b holds bit b of byte k of every element; bmb200_scan_str answers find_eq_str (exact), find_eq_str_prefix
(F_STR_PREFIX) and batches of them in one launch.
CPU: the Python mirror's planes == the reference's own, and orc_scan_str (the restated contract, oracle/bm_oracle_str.c) == the
reference's find_eq_str / find_eq_str_prefix / first match / pipeline on plain, nullable and remapped vectors.
GPU: bmb200_scan_str == orc_scan_str under every launch variant, and SparseVectorScanner == the reference's scanner.

Queries of a remapped vector are compared with the reference only where it defines an answer: not longer than
effective_max_str() - 1 and no byte >= 0x80 (DESIGN.md §3.5c); the product answers the others "no match".
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
from bitmagic_b200.capi import BLOCK_BITS, BLOCK_WORDS, GAP_MAX_WORDS, F_STR_PREFIX, ScanStrArgsC, ptr, str_slots
from bitmagic_b200.hostfmt import BVector, PackedSet
from test_launch_variants import assert_oracle, collect

gpu = pytest.mark.gpu
CMP = bm.F_OPT_COMPRESS
EXACT, PREFIX, FIRST, PIPE, PIPE_COUNTS = 0, 1, 2, 3, 4      # ref_str_find modes


# ---------------------------------------------------------------- inputs
def dictionary(rng, n=200, alpha=b"abcmxyz"):
    out = set()
    while len(out) < n:
        out.add(bytes(rng.choice(list(alpha), int(rng.integers(1, 13))).astype(np.uint8)))
    return sorted(out)


def str_inputs(kind: str, nullable: bool):
    """-> strings (list of bytes), nulls (uint8 or None).  Three block columns: dictionary words (bit planes), runs of two words
    that share their first letter (FULL and GAP planes), a sparse region of empty strings (GAP planes).  "high" adds words with
    bytes >= 0x80."""
    rng = np.random.default_rng(31 + 7 * int(nullable) + 13 * len(kind))
    if kind == "empty":
        return [], (np.zeros(0, np.uint8) if nullable else None)
    words = dictionary(rng)
    if kind == "high":
        words += [b"caf\xc3\xa9", b"\xff\xfe", b"a\x80"]
    n = 2 * BLOCK_BITS + 40000
    pick = rng.integers(0, len(words), n)
    s = [words[k] for k in pick]
    for i in range(BLOCK_BITS, 2 * BLOCK_BITS):
        s[i] = b"mango" if (i >> 12) & 1 else b"melon"
    sparse = rng.random(n - 2 * BLOCK_BITS) < 0.01
    for i in range(2 * BLOCK_BITS, n):
        if not sparse[i - 2 * BLOCK_BITS]:
            s[i] = b""
    s[n - 1] = b"zyxwvutsrqponmlkjihg"                                    # the longest stored string
    nulls = None
    if nullable:
        nulls = (rng.random(n) < 0.3).astype(np.uint8)
        nulls[BLOCK_BITS + 5000:BLOCK_BITS + 30000] = 1
        nulls[n - 1] = 0
    return s, nulls


def queries(strs, kind):
    """the empty string, single letters, the run words and their common prefix, the longest stored string and a longer one,
    strict prefixes of stored words, absent words and letters"""
    q = [b"", b"a", b"m", b"me", b"mango", b"melon", b"man", b"zyxwvutsrqponmlkjihg", b"zyxwvutsrqponmlkjihgf", b"q", b"mq",
         b"abcabcabcabcabcabcabcabc"]
    live = sorted({x for x in strs if x})
    q += [w for w in live[::max(1, len(live) // 12)]][:12]
    q += [w[:2] for w in live[:40] if len(w) > 2][:4]
    if kind == "high":
        q += [b"caf\xc3\xa9", b"caf", b"\xff", b"\xff\xfe", b"a\x80"]
    return list(dict.fromkeys(q))


def n_cols(n):
    return max(1, (n + BLOCK_BITS - 1) // BLOCK_BITS)


CASES = [(k, nl) for k in ("words", "high", "empty") for nl in (False, True)]
CASE_IDS = [f"{k}-{'null' if nl else 'plain'}" for k, nl in CASES]


# ---------------------------------------------------------------- checkers (oracle/str.mk)
ORACLE_STR = orclib.ORACLE_DIR / "liboracle_str.so"
REF_STR = orclib.ORACLE_DIR / "_ref" / "libbmref_str.so"
_libs = {}


def oracle_str() -> C.CDLL:
    """oracle/liboracle_str.so: the plain-C oracle + orc_scan_str, (re)built with make when stale"""
    if "oracle" not in _libs:
        srcs = [orclib.ORACLE_DIR / f for f in ("bm_oracle.c", "bm_oracle_entropy.c", "bm_synth.c", "bm_oracle_str.c")]
        if not ORACLE_STR.exists() or ORACLE_STR.stat().st_mtime < max(x.stat().st_mtime for x in srcs):
            subprocess.run(["make", "-C", str(orclib.ORACLE_DIR), "-f", "str.mk", str(ORACLE_STR)], check=True, capture_output=True)
        _libs["oracle"] = C.CDLL(str(ORACLE_STR))
    return _libs["oracle"]


def ref_str() -> C.CDLL:
    if "ref" not in _libs:
        _libs["ref"] = C.CDLL(str(REF_STR))
    return _libs["ref"]


def as_slots(strs):
    if isinstance(strs, np.ndarray):
        return np.ascontiguousarray(strs, np.uint8), strs.shape[1]
    return str_slots(strs)


def str_args(slots, stride, plane0, n_planes, universe, flags, nb_from=0, nb_to=0, nv=None):
    return ScanStrArgsC(int(plane0), int(n_planes), int(universe), int(flags), ptr(slots) if slots.size else C.c_void_p(0), int(stride),
                        int(slots.shape[0] if nv is None else nv), int(nb_from), int(nb_to))


def oracle_scan_str(ps, strs, plane0, n_planes, universe=0xFFFFFFFF, flags=0, nb_from=0, nb_to=0):
    """orc_scan_str (bmb200_scan_str restated) -> kind, popcnt, digest, nruns, blocks, gaps (value-major)"""
    slots, stride = as_slots(strs)
    nv = slots.shape[0]
    n = ((nb_to if nb_to else ps.n_blocks) - nb_from) * nv
    a = str_args(slots, stride, plane0, n_planes, universe, flags, nb_from, nb_to)
    kind = np.zeros(n, np.uint8); pop = np.zeros(n, np.uint32); dig = np.zeros(n, np.uint64); nr = np.zeros(n, np.uint32)
    blocks = np.zeros((n, BLOCK_WORDS), np.uint32); gaps = np.zeros((n, GAP_MAX_WORDS), np.uint16)
    c = orclib._pc(ps)
    rc = oracle_str().orc_scan_str(C.byref(c), C.byref(a), ptr(kind), ptr(pop), ptr(dig), ptr(nr), ptr(blocks), ptr(gaps))
    assert rc == 0, f"orc_scan_str rc={rc}"
    return kind, pop, dig, nr, blocks, gaps


def _recorded(fn):
    """orclib._recorded, keyed on libbmref_str.so: answers under tests/golden/ref, BMB200_RECORD_REF=1 rewrites them"""
    @functools.wraps(fn)
    def call(*args, **kw):
        h = hashlib.sha256(fn.__name__.encode())
        orclib._hash_arg(args, h); orclib._hash_arg(sorted(kw.items()), h)
        path = orclib.GOLDEN_REF / f"{fn.__name__}_{h.hexdigest()[:20]}.npz"
        if REF_STR.exists():
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


def _vec(strs, nulls):
    slots, stride = str_slots(strs) if len(strs) else (np.zeros((0, 1), np.uint8), 1)
    nl = None if nulls is None else np.ascontiguousarray(nulls, np.uint8)
    return slots, stride, nl


# ---------------------------------------------------------------- the reference (recorded answers where it is not built)
@_recorded
def ref_str_planes(slots, nulls, remap, max_planes=256):
    """The real str_sparse_vector<char, bvector<>, 32>, optimize()d (remap()ed first if asked): planes..., universe as BVectors,
    and effective_max_str()"""
    n, stride = slots.shape
    nc = n_cols(n)
    kind = np.zeros((max_planes + 1) * nc, np.uint8)
    blocks = np.zeros(((max_planes + 1) * nc, BLOCK_WORDS), np.uint32)
    gaps = np.zeros(((max_planes + 1) * nc, GAP_MAX_WORDS), np.uint16)
    npl, ms = C.c_uint32(0), C.c_uint32(0)
    rc = ref_str().ref_str_planes(ptr(slots), C.c_uint32(stride), C.c_uint64(n), ptr(nulls) if nulls is not None else C.c_void_p(0),
                                  int(remap), C.c_uint32(nc), C.c_uint32(max_planes), C.byref(npl), C.byref(ms), ptr(kind), ptr(blocks), ptr(gaps))
    assert rc == 0, f"ref_str_planes rc={rc}"
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
    return out, int(ms.value)


@_recorded
def ref_str_remap(slots, nulls, q):
    """remap_tosv of every query against the remap()ed vector -> (codes as NUL-padded slots, ok[])"""
    n, stride = slots.shape
    qs = np.ascontiguousarray(q, np.uint8)
    out = np.zeros_like(qs); ok = np.zeros(qs.shape[0], np.uint8)
    rc = ref_str().ref_str_remap(ptr(slots), C.c_uint32(stride), C.c_uint64(n), ptr(nulls) if nulls is not None else C.c_void_p(0),
                                 ptr(qs), C.c_uint32(qs.shape[1]), C.c_uint32(qs.shape[0]), ptr(out), ptr(ok))
    assert rc == 0, f"ref_str_remap rc={rc}"
    return out, ok


@_recorded
def ref_str_find(slots, nulls, remap, mode, q):
    """The real sparse_vector_scanner on that vector: mode EXACT / PREFIX / FIRST / PIPE / PIPE_COUNTS ->
    found[nq], pos[nq], counts[nq], words[nq][n_cols * 2048]"""
    n, stride = slots.shape
    qs = np.ascontiguousarray(q, np.uint8)
    nq, nc = qs.shape[0], n_cols(n)
    found = np.zeros(nq, np.uint8); pos = np.zeros(nq, np.uint64); counts = np.zeros(nq, np.uint64)
    words = np.zeros((nq, nc * BLOCK_WORDS), np.uint32)
    rc = ref_str().ref_str_find(ptr(slots), C.c_uint32(stride), C.c_uint64(n), ptr(nulls) if nulls is not None else C.c_void_p(0),
                                int(remap), int(mode), ptr(qs), C.c_uint32(qs.shape[1]), C.c_uint32(nq), C.c_uint32(nc),
                                ptr(found), ptr(pos), ptr(counts), ptr(words))
    assert rc == 0, f"ref_str_find rc={rc}"
    if mode in (FIRST, PIPE_COUNTS):
        words = np.zeros((nq, 0), np.uint32)
    return found, pos, counts, words


# ---------------------------------------------------------------- helpers
def vec_words(bv: BVector, nc: int):
    return np.concatenate([bv.block_words(c) if c < bv.n_blocks else np.zeros(BLOCK_WORDS, np.uint32) for c in range(nc)])


def np_match(strs, nulls, q, prefix):
    """the contract on the host strings: element == q (prefix: starts with q; the empty q: the empty string), NOT-NULL"""
    ok = np.ones(len(strs), bool) if nulls is None else nulls == 0
    if prefix and q:
        hit = np.array([x.startswith(q) for x in strs], bool)
    else:
        hit = np.array([x == q for x in strs], bool)
    return (hit & ok).astype(np.uint8)


def ref_packed(slots, nulls, remap=0):
    vecs, ms = ref_str_planes(slots, nulls, remap)
    return PackedSet.pack(vecs, max(v.n_blocks for v in vecs)), len(vecs) - 1, ms


def defined_for_remap(q, max_str):
    return len(q) < max_str and all(b < 0x80 for b in q)


# ---------------------------------------------------------------- CPU
def test_f_str_prefix_matches_header():
    hdr = (orclib.ROOT / "include" / "bmb200.h").read_text()
    assert "#define BMB200_F_STR_PREFIX 16u" in hdr and F_STR_PREFIX == 16


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_str_planes_match_reference(case):
    kind, nullable = case
    strs, nulls = str_inputs(kind, nullable)
    slots, stride, nl = _vec(strs, nulls)
    ref, _ = ref_str_planes(slots, nl, 0)
    sv = bm.StrSparseVector.from_strings(strs, nulls)
    nc = n_cols(len(strs))
    assert sv.effective_slices() == len(ref) - 1
    for j, p in enumerate(sv.planes):
        assert np.array_equal(vec_words(p, nc), vec_words(ref[j], nc)), j
    assert np.array_equal(vec_words(sv.universe(), nc), vec_words(ref[-1], nc))


@pytest.mark.parametrize("remap", [0, 1], ids=["plain-codes", "remapped"])
@pytest.mark.parametrize("case", [c for c in CASES if c[0] != "empty"], ids=[i for c, i in zip(CASES, CASE_IDS) if c[0] != "empty"])
def test_orc_scan_str_matches_reference(case, remap):
    """orc_scan_str on the reference's own planes == the reference's find_eq_str, find_eq_str_prefix, first match and pipeline"""
    kind, nullable = case
    strs, nulls = str_inputs(kind, nullable)
    slots, stride, nl = _vec(strs, nulls)
    ps, npl, ms = ref_packed(slots, nl, remap)
    q = queries(strs, kind)
    if remap:
        q = [x for x in q if defined_for_remap(x, ms)]
    qslots, _ = str_slots(q)
    codes = qslots
    if remap:
        codes, ok = ref_str_remap(slots, nl, qslots)
    nq = len(q)
    for mode, flags in ((EXACT, CMP), (PREFIX, CMP | F_STR_PREFIX)):
        found, _, counts, rw = ref_str_find(slots, nl, remap, mode, qslots)
        o = oracle_scan_str(ps, codes, 0, npl, npl, flags)
        ob = o[4].reshape(nq, -1)
        for k in range(nq):
            if remap and not ok[k]:                                      # no code for a character: no launch, no match
                assert counts[k] == 0 and not found[k], q[k]
                continue
            if not q[k]:
                # the reference's find_zero ORs effective_slices() planes, which a string vector leaves at 1: its answer for the
                # empty string is "plane 0 is clear", not "every plane is clear" (DESIGN.md §3.5c).  The product follows the contract.
                if not remap:
                    ok0 = np.ones(len(strs), bool) if nulls is None else nulls == 0
                    even = np.array([not x or not (x[0] & 1) for x in strs], bool)
                    assert np.array_equal(R.bits_of(rw[k])[:len(strs)], (even & ok0).astype(np.uint8))
                assert np.array_equal(R.bits_of(ob[k])[:len(strs)], np_match(strs, nulls, b"", False))
                continue
            assert np.array_equal(ob[k], rw[k]), (mode, q[k])
            assert int(o[1].reshape(nq, -1)[k].sum()) == int(counts[k]) and bool(found[k]) == bool(counts[k]), (mode, q[k])
            assert np.array_equal(R.bits_of(rw[k])[:len(strs)], np_match(strs, nulls, q[k], mode == PREFIX)), (mode, q[k])
    exact = R.bits_of(oracle_scan_str(ps, codes, 0, npl, npl, CMP)[4]).reshape(nq, -1)
    found, pos, _, _ = ref_str_find(slots, nl, remap, FIRST, qslots)
    for k in range(nq):
        if not q[k]:
            continue                                                     # find_zero: see above
        hits = np.flatnonzero(exact[k]) if (not remap or ok[k]) else []
        assert bool(found[k]) == (len(hits) > 0) and (not found[k] or int(pos[k]) == int(hits[0])), q[k]
    ne = [k for k in range(nq) if q[k]]                                  # the pipeline takes non-empty strings
    pq, _ = str_slots([q[k] for k in ne])
    _, _, pcounts, pw = ref_str_find(slots, nl, remap, PIPE, pq)
    _, _, ccounts, _ = ref_str_find(slots, nl, remap, PIPE_COUNTS, pq)
    for i, k in enumerate(ne):
        want = exact[k] if (not remap or ok[k]) else np.zeros_like(exact[k])
        assert np.array_equal(R.bits_of(pw[i]), want) and int(pcounts[i]) == int(ccounts[i]) == int(want.sum()), q[k]


def test_orc_scan_str_rejects_bad_args():
    ps = PackedSet.pack([bm.BVector.from_words(np.zeros(BLOCK_WORDS, np.uint32))] * 3)
    slots, stride = str_slots([b"ab"])
    c = orclib._pc(ps)
    out = [np.zeros(1, np.uint8), np.zeros(1, np.uint32), np.zeros(1, np.uint64), np.zeros(1, np.uint32)]
    call = lambda a: oracle_str().orc_scan_str(C.byref(c), C.byref(a), *(ptr(x) for x in out), None, None)
    assert call(str_args(slots, stride, 0, 2049, 0xFFFFFFFF, 0)) == bm.capi.ERR_BADARG
    full = np.full((1, 4), ord("a"), np.uint8)                          # no NUL inside the slot
    assert call(str_args(full, 4, 0, 2, 0xFFFFFFFF, 0)) == bm.capi.ERR_BADARG
    assert call(str_args(np.zeros((0, 1), np.uint8), 1, 0, 2, 0xFFFFFFFF, 0, nv=1)) == bm.capi.ERR_BADARG
    assert call(str_args(slots, stride, 0, 2, 0xFFFFFFFF, 0)) == 0


def test_scan_str_rejects_null_pointers():
    """the product's entry point refuses null handles and arguments before it needs a device"""
    slots, stride = str_slots([b"ab"])
    a = str_args(slots, stride, 0, 2, 0xFFFFFFFF, 0)
    r = C.c_void_p(0)
    lib = bm.capi.lib()
    assert lib.bmb200_scan_str(None, None, C.byref(a), C.byref(r)) == bm.capi.ERR_BADARG
    assert lib.bmb200_scan_str(None, None, None, C.byref(r)) == bm.capi.ERR_BADARG
    assert lib.bmb200_scan_str(None, None, C.byref(a), None) == bm.capi.ERR_BADARG


def test_str_answers_recorded():
    """every reference answer the tests compare against is recorded (or computed live where the reference is built)"""
    for kind, nullable in CASES:
        strs, nulls = str_inputs(kind, nullable)
        slots, stride, nl = _vec(strs, nulls)
        ref_str_planes(slots, nl, 0)
        if kind == "empty":
            continue
        for remap in (0, 1):
            _, _, ms = ref_packed(slots, nl, remap)
            q = queries(strs, kind)
            if remap:
                q = [x for x in q if defined_for_remap(x, ms)]
            qslots, _ = str_slots(q)
            if remap:
                ref_str_remap(slots, nl, qslots)
            for mode in (EXACT, PREFIX, FIRST):
                ref_str_find(slots, nl, remap, mode, qslots)
            pq, _ = str_slots([x for x in q if x])
            ref_str_find(slots, nl, remap, PIPE, pq)
            ref_str_find(slots, nl, remap, PIPE_COUNTS, pq)


# ---------------------------------------------------------------- GPU: bmb200_scan_str against orc_scan_str
def plane_set(strs, nulls, gap_flat=True):
    """Two dummy vectors, then the mirror's planes, then its universe and a bit-block universe.
    -> ps, n_planes, universes {name: (vector id, bits)}"""
    rng = np.random.default_rng(3)
    sv = bm.StrSparseVector.from_strings(strs, nulls)
    nb = sv.planes[0].n_blocks
    npl = sv.effective_slices()
    bit_u = (rng.random(nb * BLOCK_BITS) < 0.7).astype(np.uint8)
    dummies = [BVector.from_words(R.words_of((rng.random(nb * BLOCK_BITS) < 0.5).astype(np.uint8), nb)) for _ in range(2)]
    vecs = dummies + list(sv.planes) + [sv.universe(), BVector.from_words(R.words_of(bit_u, nb))]
    ps = PackedSet.pack(vecs, nb, gap_flat=gap_flat)
    uni = np.zeros(nb * BLOCK_BITS, np.uint8)
    uni[:len(strs)] = 1 if nulls is None else (nulls == 0)
    return ps, npl, {"none": (0xFFFFFFFF, np.ones(nb * BLOCK_BITS, np.uint8)), "sv": (2 + npl, uni), "bit": (3 + npl, bit_u)}


def launches(q):
    """launches of 1, 2, 3, 4, 5 and 64 queries (every VG, short last groups) out of the query list"""
    out, off = [], 0
    for nv in (1, 2, 3, 4, 5, 64):
        out.append([q[(off + t) % len(q)] for t in range(nv)])
        off += nv
    return out


@gpu
@pytest.mark.parametrize("kind", ["words", "high"])
def test_scan_str_launch_variants(ctx, kind):
    """bmb200_scan_str == orc_scan_str (kind, popcount, digest, run count, bits, GAP words, group totals) and the host string
    comparison, exact and prefix, 1..5 and 64 queries per launch, plane0 > 0, universes absent / NOT-NULL / bit, FLAT and raw GAP
    planes; column sub-ranges, F_COUNT_ONLY, F_OPT_NONE, and recycled results of the right and the wrong shape"""
    strs, nulls = str_inputs(kind, True)
    stored = [b"" if z else x for x, z in zip(strs, nulls)]              # a NULL element's planes are all 0: the empty string
    q = queries(strs, kind)
    for gap_flat, unis in ((True, ("none", "sv", "bit")), (False, ("sv",))):
        ps, npl, universes = plane_set(strs, nulls, gap_flat)
        dset = bm.DeviceSet.upload(ctx, ps)
        for un in unis:
            uni, ubits = universes[un]
            for pflag in (0, F_STR_PREFIX):
                for k, search in enumerate(launches(q)):
                    flags = (CMP if k % 2 else bm.F_OPT_NONE) | pflag
                    res = bm.scan_str(ctx, dset, search, 2, npl, uni, flags)
                    got = collect(res, len(search)); res.free()
                    assert_oracle(got, oracle_scan_str(ps, search, 2, npl, uni, flags), len(search), f"{un} flags={flags} nv={len(search)}")
                    bits = R.bits_of(got["blocks"]).reshape(len(search), -1)
                    for g, s in enumerate(search):
                        want = np_match(stored, None, s, bool(pflag)) & ubits[:len(strs)]
                        assert np.array_equal(bits[g, :len(strs)], want), (un, pflag, s)
                search = launches(q)[4]
                for nb_from, nb_to in ((1, 0), (0, 2), (1, 2)):
                    res = bm.scan_str(ctx, dset, search, 2, npl, uni, CMP | pflag, nb_from=nb_from, nb_to=nb_to)
                    got = collect(res, len(search)); res.free()
                    assert_oracle(got, oracle_scan_str(ps, search, 2, npl, uni, CMP | pflag, nb_from, nb_to), len(search),
                                  f"range {nb_from}-{nb_to}")
                res = bm.scan_str(ctx, dset, search, 2, npl, uni, bm.F_COUNT_ONLY | pflag)
                got = collect(res, len(search), stored=False); res.free()
                assert_oracle(got, oracle_scan_str(ps, search, 2, npl, uni, pflag), len(search), "count-only")
                # recycled: a result of the same shape (from a numeric scan), then one of another shape
                res = bm.scan(ctx, dset, bm.SCAN_EQ, np.arange(len(search), dtype=np.uint64), 2, 8, uni, CMP)
                res = bm.scan_str(ctx, dset, search, 2, npl, uni, CMP | pflag, result=res)
                got = collect(res, len(search))
                assert_oracle(got, oracle_scan_str(ps, search, 2, npl, uni, CMP | pflag), len(search), "recycled")
                res = bm.scan_str(ctx, dset, search[:2], 2, npl, uni, CMP | pflag, result=res)
                got = collect(res, 2); res.free()
                assert_oracle(got, oracle_scan_str(ps, search[:2], 2, npl, uni, CMP | pflag), 2, "recycled, other shape")
        dset.free()


@gpu
def test_scan_str_edges(ctx):
    """n_planes 2048 (256-byte strings), a column every query leaves at its first octet, a lone survivor at bit 65535 that walks
    down to plane 0, a NULL universe column, and a vector of size 0"""
    rng = np.random.default_rng(9)
    n = 3 * BLOCK_BITS
    long_a = bytes(rng.integers(1, 256, 255).astype(np.uint8)) + b"\xc1"     # plane 2047 is set
    long_b = long_a[:255] + b"\x81"                                      # differs from long_a in the top octet only
    strs = [b"k%d" % (i % 50) for i in range(n)]
    for i in range(0, BLOCK_BITS, 4099):
        strs[i] = long_a
    strs[BLOCK_BITS - 1] = long_b                                        # bit 65535 of column 0
    strs[BLOCK_BITS + 17] = long_b
    nulls = np.zeros(n, np.uint8)
    nulls[2 * BLOCK_BITS:] = 1                                           # column 2: NULL universe block
    ps, npl, universes = plane_set(strs, nulls)
    assert npl == 2048
    dset = bm.DeviceSet.upload(ctx, ps)
    uni = universes["sv"][0]
    q = [long_a, long_b, long_a[:200], long_b[:255], b"k1", b"k", b"\xfe" * 3, b"", long_a + b"x"]
    for flags in (CMP, CMP | F_STR_PREFIX, bm.F_OPT_NONE):
        for search in (q, [long_b], q[:3]):
            res = bm.scan_str(ctx, dset, search, 2, npl, uni, flags)
            got = collect(res, len(search)); res.free()
            assert_oracle(got, oracle_scan_str(ps, search, 2, npl, uni, flags), len(search), f"edges flags={flags}")
            bits = R.bits_of(got["blocks"]).reshape(len(search), -1)
            for g, s in enumerate(search):
                assert np.array_equal(bits[g, :n], np_match(strs, nulls, s, bool(flags & F_STR_PREFIX))), s[:8]
    res = bm.scan_str(ctx, dset, [long_b], 2, npl, uni, CMP)
    assert R.bits_of(collect(res)["blocks"])[:BLOCK_BITS].nonzero()[0].tolist() == [BLOCK_BITS - 1]
    res.free()
    dset.free()
    # size 0: one empty column, nothing matches
    ps, npl, universes = plane_set([], None)
    dset = bm.DeviceSet.upload(ctx, ps)
    for flags in (CMP, CMP | F_STR_PREFIX):
        res = bm.scan_str(ctx, dset, [b"", b"a"], 2, npl, universes["sv"][0], flags)
        got = collect(res, 2); res.free()
        assert got["total"] == 0
        assert_oracle(got, oracle_scan_str(ps, [b"", b"a"], 2, npl, universes["sv"][0], flags), 2, "size 0")
    dset.free()


@gpu
def test_scan_str_rejects_bad_args(ctx):
    ps, npl, _ = plane_set([b"ab", b"cd"], None)
    dset = bm.DeviceSet.upload(ctx, ps)
    lib = bm.capi.lib()
    slots, stride = str_slots([b"ab"])
    r = C.c_void_p(0)
    for a, code in ((str_args(slots, stride, 0, 2049, 0xFFFFFFFF, 0), bm.capi.ERR_BADARG),
                    (str_args(np.full((1, 4), 97, np.uint8), 4, 0, 2, 0xFFFFFFFF, 0), bm.capi.ERR_BADARG),
                    (str_args(slots, stride, 0, 2, 0xFFFFFFFF, 0, nv=0), bm.capi.ERR_BADARG),
                    (str_args(slots, stride, 0, 2, 0xFFFFFFFF, bm.F_SIGNED), bm.capi.ERR_BADARG),
                    (str_args(slots, stride, 1, ps.n_vec, 0xFFFFFFFF, 0), bm.capi.ERR_RANGE),
                    (str_args(slots, stride, 0, 2, ps.n_vec, 0), bm.capi.ERR_RANGE)):
        assert lib.bmb200_scan_str(ctx._h, dset._h, C.byref(a), C.byref(r)) == code
        assert not r.value
    dset.free()


@gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_str_scanner_against_reference(ctx, case):
    """SparseVectorScanner on the mirror == the reference's find_eq_str / find_eq_str_prefix / pipeline counts; and on the
    reference's remapped planes, with the reference's query codes, == its remapped searches"""
    kind, nullable = case
    strs, nulls = str_inputs(kind, nullable)
    slots, stride, nl = _vec(strs, nulls)
    nc = n_cols(len(strs))
    sc = bm.SparseVectorScanner(bm.StrSparseVector.from_strings(strs, nulls), ctx)
    try:
        if kind == "empty":
            assert sc.count_eq_str([b"", b"a"]) == [0, 0] and sc.find_eq_str_prefix(b"a").count() == 0
            return
        with pytest.raises(TypeError):
            sc.find_eq(3)
        q = queries(strs, kind)
        qslots, _ = str_slots(q)
        for mode, fn in ((EXACT, sc.find_eq_str), (PREFIX, sc.find_eq_str_prefix)):
            found, _, counts, rw = ref_str_find(slots, nl, 0, mode, qslots)
            got = fn(q)
            for k in range(len(q)):
                if not q[k]:                                             # the reference's find_zero: see test_orc_scan_str_matches_reference
                    assert np.array_equal(R.bits_of(vec_words(got[k], nc))[:len(strs)], np_match(strs, nulls, b"", False))
                    continue
                assert np.array_equal(vec_words(got[k], nc), rw[k]), (mode, q[k])
                assert got[k].count() == int(counts[k])
        _, _, ccounts, _ = ref_str_find(slots, nl, 0, PIPE_COUNTS, str_slots([x for x in q if x])[0])
        assert sc.count_eq_str([x for x in q if x]) == [int(c) for c in ccounts]
    finally:
        sc.close()
    # remapped: the reference's own planes + its codes for the queries it defines
    vecs, ms = ref_str_planes(slots, nl, 1)
    rsv = bm.StrSparseVector(vecs[:-1], len(strs), vecs[-1] if nullable else None)
    q = [x for x in queries(strs, kind) if defined_for_remap(x, ms)]
    qslots, _ = str_slots(q)
    codes, ok = ref_str_remap(slots, nl, qslots)
    sc = bm.SparseVectorScanner(rsv, ctx)
    try:
        live = [k for k in range(len(q)) if ok[k]]
        cq = [bytes(codes[k]).split(b"\0")[0] for k in live]
        for mode, fn in ((EXACT, sc.find_eq_str), (PREFIX, sc.find_eq_str_prefix)):
            found, _, counts, rw = ref_str_find(slots, nl, 1, mode, qslots)
            got = fn(cq)
            for i, k in enumerate(live):
                if not q[k]:
                    continue
                assert np.array_equal(vec_words(got[i], nc), rw[k]) and got[i].count() == int(counts[k]), (mode, q[k])
            assert all(counts[k] == 0 for k in range(len(q)) if not ok[k])
    finally:
        sc.close()


@gpu
def test_str_binding_harness():
    exe = orclib.ORACLE_DIR / "_ref" / "test_str_binding"
    if not exe.exists():
        pytest.skip("oracle/_ref/test_str_binding is built only where the reference tree exists")
    p = subprocess.run([str(exe)], capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-2000:]
    assert "0 failed" in p.stdout
