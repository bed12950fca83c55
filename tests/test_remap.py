"""Set image through a sparse vector: the reference's set2set_11_transform<SV>::remap(bv_in, sv, bv_out).

bmb200_remap maps the set bits i of a device result through the planes of a sparse vector to the set of values sv[i]
(include/bmb200.h), in one pass over the source's populated columns (csrc/remap_kernel.cuh).
CPU: the unmodified reference (oracle/remap.mk, 32- and 64-bit addressing; recorded as counts + SHA-256 digests of the image)
== the numpy restatement on every case of the contract: ids past size(), unassigned elements, explicit zeros, NULLs, the empty
vector, a pre-filled bv_out, attach_sv(sv, true), the value 0xffffffff in both builds and an all-ids-to-one-value case.
GPU: the C ABI == numpy, with kinds, popcounts, digests, run counts and GAP words == the C oracle's classification of the image,
under both flags, for 1 to 32 planes, FLAT and raw sets, every block kind, nullable and plain vectors, sources longer and
shorter than the set, sources chained from bm.aggregate and bm.scan, recycled results, an image over all 65536 columns and
every error case; the Python class against the recorded reference answers, and the C++ binding harnesses.
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
from bitmagic_b200.capi import BLOCK_BITS, NO_UNIVERSE, ptr
from bitmagic_b200.hostfmt import BVector, PackedSet, bits_to_words, words_to_bits

gpu = pytest.mark.gpu
B = BLOCK_BITS
ID_MAX32, ID_MAX64 = 0xFFFFFFFF, (1 << 48) - 1
REF_LIBS = {False: orclib.ORACLE_DIR / "_ref" / "libbmref_remap.so", True: orclib.ORACLE_DIR / "_ref" / "libbmref_remap64.so"}
_libs = {}


# ---------------------------------------------------------------- the contract in numpy
def np_image(values, nulls, ids, id_max=ID_MAX32) -> np.ndarray:
    """the sorted values sv[i] of the ids i (inside NOT-NULL when nullable; a plain vector maps ids past size() to 0), < id_max"""
    values = np.asarray(values, np.uint64)
    n = values.size
    if n == 0:
        return np.zeros(0, np.uint64)
    ids = np.unique(np.asarray(ids, np.uint64))
    inside = ids[ids < n].astype(np.int64)
    if nulls is not None:
        v = values[inside[np.asarray(nulls, bool)[inside] == 0]]
    else:
        v = values[inside]
        if (ids >= n).any():
            v = np.append(v, np.uint64(0))
    v = np.unique(v)
    return v[v < np.uint64(id_max)]


def digest(positions) -> np.ndarray:
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(positions, np.uint64).tobytes()).digest(), np.uint8).copy()


# ---------------------------------------------------------------- the reference (oracle/remap.mk)
def ref_lib(addr64: bool) -> C.CDLL:
    if addr64 not in _libs:
        _libs[addr64] = C.CDLL(str(REF_LIBS[addr64]))
    return _libs[addr64]


def _recorded(fn):
    """orclib._recorded, keyed on the reference shim: answers under tests/golden/ref, BMB200_RECORD_REF=1 rewrites them"""
    @functools.wraps(fn)
    def call(*args, **kw):
        h = hashlib.sha256(fn.__name__.encode())
        orclib._hash_arg(args, h); orclib._hash_arg(sorted(kw.items()), h)
        path = orclib.GOLDEN_REF / f"{fn.__name__}_{h.hexdigest()[:20]}.npz"
        if all(p.exists() for p in REF_LIBS.values()):
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


@_recorded
def ref_remap(values, nulls, ids, addr64, mode):
    """set2set_11_transform::remap of the unmodified reference -> (count, SHA-256 of the image's values as u64).
    mode 1: attach_sv(&sv, true) + remap(bv_in, bv_out); mode 2: bv_out pre-filled"""
    dt = np.uint64 if addr64 else np.uint32
    lib = ref_lib(addr64)
    assert lib.ref_remap_word_bytes() == np.dtype(dt).itemsize
    v = np.ascontiguousarray(values, dt)
    i = np.ascontiguousarray(ids, dt)
    nl = ptr(np.ascontiguousarray(nulls, np.uint8)) if nulls is not None else C.c_void_p(0)
    cap = int(v.size) + 2
    out = np.zeros(cap, dt)
    cnt = C.c_uint64(0)
    assert lib.ref_remap(ptr(v), nl, C.c_uint64(v.size), ptr(i), C.c_uint64(i.size), int(mode), C.byref(cnt), ptr(out), C.c_uint64(cap)) == 0
    return int(cnt.value), digest(out[:min(cnt.value, cap)].astype(np.uint64))


# ---------------------------------------------------------------- cases
def example(nullable):
    """the contract's example: {2:25, 3:35, 7:75, 256:2001, 1000:2000}; the nullable one with an explicit 9:0"""
    v = np.zeros(1001, np.uint64)
    for k, x in ((2, 25), (3, 35), (7, 75), (256, 2001), (1000, 2000)):
        v[k] = x
    if not nullable:
        return v, None, np.array([1, 2, 7, 300, 5000000])
    nulls = np.ones(1001, np.uint8)
    nulls[[2, 3, 7, 9, 256, 1000]] = 0
    return v, nulls, np.array([1, 2, 7, 9, 5000000])


def random_case(seed, n, top, nullable, density):
    rng = np.random.default_rng(seed)
    v = rng.integers(0, top, n, dtype=np.uint64)
    v[rng.random(n) < 0.2] = 0                                               # unassigned / explicit zeros
    nulls = (rng.random(n) < 0.25).astype(np.uint8) if nullable else None
    ids = np.flatnonzero(rng.random(n + 3 * B) < density)                    # also past size()
    return v, nulls, ids


def cpu_cases():
    out = [("example", *example(False), False), ("example nullable", *example(True), False)]
    for nullable in (False, True):
        out.append((f"random nullable={nullable}", *random_case(3 + nullable, 3 * B + 321, 5000, nullable, 0.3), False))
        out.append((f"random 64 nullable={nullable}", *random_case(5 + nullable, 2 * B + 11, 1 << 30, nullable, 0.05), True))
    out.append(("empty vector", np.zeros(0, np.uint64), None, np.array([0, 4, 70000]), False))
    out.append(("empty nullable", np.zeros(0, np.uint64), np.zeros(0, np.uint8), np.array([0, 4]), True))
    top = np.zeros(5000, np.uint64); top[::7] = ID_MAX32; top[3] = 12
    out.append(("0xffffffff in 32 bits", top, None, np.arange(0, 6000, 3), False))
    out.append(("0xffffffff in 64 bits", top, None, np.arange(0, 6000, 3), True))
    t48 = top.copy(); t48[::11] = ID_MAX64; t48[5] = ID_MAX64 - 1
    out.append(("2^48-1 in 64 bits", t48, None, np.arange(6000), True))
    out.append(("all to one value", np.full(3 * B + 5, 777, np.uint64), None, np.arange(3 * B + 5), False))
    return out


CPU_CASES = cpu_cases()


# ---------------------------------------------------------------- CPU
def test_remap_header_and_struct():
    hdr = (orclib.ROOT / "include" / "bmb200.h").read_text()
    assert "bmb200_remap                  <- set2set_11_transform::remap" in hdr
    assert "src/bmsparsevec_algo.h:2097-2205" in hdr
    for f in ("plane0, n_planes;", "not_null;", "flags;", "id_max;", "} bmb200_remap_args;"):
        assert f in hdr
    assert C.sizeof(bm.capi.RemapArgsC) == 24 and bm.capi.RemapArgsC.id_max.offset == 16
    assert "bmb200_remap" in bm.capi.SYMBOLS


@pytest.mark.parametrize("case", CPU_CASES, ids=[c[0] for c in CPU_CASES])
@pytest.mark.parametrize("mode", [0, 1, 2], ids=["remap", "attach_sv-stats", "prefilled"])
def test_reference_matches_contract(case, mode):
    name, values, nulls, ids, addr64 = case
    want = np_image(values, nulls, ids, ID_MAX64 if addr64 else ID_MAX32)
    cnt, dg = ref_remap(values, nulls, ids, addr64, mode)
    assert cnt == want.size and np.array_equal(dg, digest(want)), (name, cnt, want[:10])


def test_contract_examples():
    assert np_image(*example(False)).tolist() == [0, 25, 75]
    assert np_image(*example(True)).tolist() == [0, 25, 75]
    _, v, nl, ids, _ = CPU_CASES[-4]
    assert ID_MAX32 not in np_image(v, nl, ids, ID_MAX32) and ID_MAX32 in np_image(v, nl, ids, ID_MAX64)


@pytest.mark.parametrize("order", [0, 1, 2])
def test_reference_defect_id_max_as_65535(order):
    """the reference passes the gathered values to bvector::set(ids, n, BM_SORTED) unsorted; a value bm::id_max that is neither
    first nor last of its batch comes back as the value 65535, which no id maps to (DESIGN.md 3.5g).  The contract, and the
    device, leave bm::id_max out wherever it sits."""
    vals = [[5, ID_MAX32, 7], [ID_MAX32, 5, 7], [5, 7, ID_MAX32]][order]
    ids = np.arange(3)
    want = np_image(np.array(vals, np.uint64), None, ids)
    assert want.tolist() == [5, 7]
    cnt, dg = ref_remap(np.array(vals, np.uint64), None, ids, False, 0)
    if order == 0:
        assert cnt == 3 and np.array_equal(dg, digest(np.array([5, 7, 65535], np.uint64)))
    else:
        assert cnt == 2 and np.array_equal(dg, digest(want))


# ---------------------------------------------------------------- GPU helpers
def gpu_vector(n_planes, nullable, seed=11):
    """values < 2^n_planes over 4 columns + 500 elements: iid (bit planes), one constant with its top bit set (FULL / NULL
    planes), runs of two values (GAP planes), sparse (GAP planes); NOT-NULL: iid (bit), all (FULL), runs (GAP), none (NULL)"""
    rng = np.random.default_rng(seed + n_planes)
    n = 4 * B + 500
    top = np.uint64((1 << n_planes) - 1)
    v = rng.integers(0, 1 << n_planes, n, dtype=np.uint64)
    i = np.arange(n)
    v[B:2 * B] = top ^ np.uint64(rng.integers(0, 1 << n_planes) & ((1 << max(n_planes - 1, 0)) - 1))
    v[2 * B:3 * B] = np.where((i[2 * B:3 * B] >> 9) & 1, top, np.uint64(1 << (n_planes - 1)))
    sparse = np.zeros(B, np.uint64); hit = rng.random(B) < 0.01
    sparse[hit] = rng.integers(0, 1 << n_planes, int(hit.sum()), dtype=np.uint64)
    v[3 * B:4 * B] = sparse
    if n_planes == 32:
        v[[5, 70, 3 * B + 17]] = ID_MAX32
    nulls = None
    if nullable:
        nulls = (rng.random(n) < 0.2).astype(np.uint8)
        nulls[B:2 * B] = 0
        nulls[2 * B:3 * B] = (i[2 * B:3 * B] >> 11) & 1
        nulls[3 * B:4 * B] = 1
    v = np.where(nulls.astype(bool), np.uint64(0), v) if nulls is not None else v
    return v, nulls


def source_bits(n_cols, seed):
    """source ids over n_cols columns: NULL, FULL, GAP (runs) and bit (random) columns in turn"""
    rng = np.random.default_rng(seed)
    bits = np.zeros(n_cols * B, np.uint8)
    for c in range(n_cols):
        s = slice(c * B, (c + 1) * B)
        k = c % 4
        if k == 1:
            bits[s] = 1
        elif k == 2:
            bits[s] = (np.arange(B) >> 8) & 1
        elif k == 3:
            bits[s] = rng.random(B) < 0.3
    return bits


def check_image(res, want, n_planes, flags, what):
    """res == the image `want`: its bits, and kinds, popcounts, digests, run counts and GAP words == the C oracle's
    classification (finalize_blocks_kernel runs the aggregation epilogue) of the populated columns plus one empty column;
    every other column must match that empty one"""
    cols = max(1, 1 << max(n_planes - 16, 0))
    assert res.n_cols == cols, what
    kind, pop, dig, nr = res.meta()
    assert res.total() == (want.size, want.size > 0) and int(res.group_totals(1)[0]) == want.size, what
    bv = bm.result_to_bvector(*res.fetch())
    assert np.array_equal(bv.positions(), want), what
    used = np.unique((want >> np.uint64(16)).astype(np.int64))
    empty = np.setdiff1d(np.arange(min(cols, used.size + 1)), used)[:1]
    sel = np.concatenate([used, empty]).astype(np.int64)
    bits = np.zeros(sel.size * B, np.uint8)
    for k, c in enumerate(used):
        w = want[(want >> np.uint64(16)) == np.uint64(c)] & np.uint64(0xFFFF)
        bits[k * B + w.astype(np.int64)] = 1
    ok, opop, odig, onr, oblk, ogap = orclib.oracle_aggregate(PackedSet.pack([BVector.from_words(bits_to_words(bits))], sel.size),
                                                              bm.OP_OR, [0], None, flags)
    for k, c in enumerate(sel):
        assert (kind[c], pop[c], dig[c], nr[c]) == (ok[k], opop[k], odig[k], onr[k]), (what, int(c))
        assert np.array_equal(bv.block_words(int(c)), oblk[k]), (what, int(c))
        if ok[k] == bm.BLK_GAP:
            assert np.array_equal(bv.blocks[int(c)], ogap[k, :(int(ogap[k, 0]) >> 3) + 1]), (what, int(c))
    rest = np.ones(cols, bool); rest[sel] = False
    if empty.size:
        for a, o in ((kind, ok), (pop, opop), (dig, odig), (nr, onr)):
            assert (a[rest] == o[-1]).all(), what


def upload_vector(ctx, v, nulls, n_planes, flat, extra=()):
    """planes 0..n_planes-1 (absent high planes empty), then the NOT-NULL vector, then `extra` vectors"""
    sv = bm.SparseVector.from_values(v, nulls)
    planes = list(sv.planes) + [BVector(sv.planes[0].n_blocks) for _ in range(n_planes - len(sv.planes))]
    vecs = planes + ([sv.not_null] if nulls is not None else []) + list(extra)
    ps = PackedSet.pack(vecs, max(x.n_blocks for x in vecs), gap_flat=flat)
    return bm.DeviceSet.upload(ctx, ps), (n_planes if nulls is not None else NO_UNIVERSE), ps


# ---------------------------------------------------------------- GPU
@gpu
@pytest.mark.parametrize("n_planes", [1, 2, 16, 17, 21, 31, 32])
@pytest.mark.parametrize("flat", [True, False], ids=["flat", "raw"])
@pytest.mark.parametrize("nullable", [False, True], ids=["plain", "nullable"])
def test_remap_against_numpy(ctx, n_planes, flat, nullable):
    v, nulls = gpu_vector(n_planes, nullable)
    dset, nn, _ = upload_vector(ctx, v, nulls, n_planes, flat)
    out = None
    for n_src in (3, 7):                                                    # shorter and longer than the set's 5 columns
        bits = source_bits(n_src, n_planes + n_src)
        sset = bm.DeviceSet.upload(ctx, PackedSet.pack([BVector.from_words(bits_to_words(bits)).optimize()], n_src, gap_flat=flat))
        for sflags in (bm.F_OPT_COMPRESS, bm.F_OPT_NONE):                   # GAP source columns under compress
            src = bm.aggregate(ctx, sset, bm.OP_OR, [0], None, sflags)
            for flags, id_max in ((bm.F_OPT_COMPRESS, ID_MAX32), (bm.F_OPT_NONE, ID_MAX32),
                                  (bm.F_OPT_COMPRESS, ID_MAX64 if n_planes == 32 else 1000)):
                want = np_image(v, nulls, np.flatnonzero(bits), id_max)
                out = bm.remap(ctx, dset, src, 0, n_planes, nn, id_max, flags, out)   # recycled across calls
                check_image(out, want, n_planes, flags, (n_planes, flat, nullable, n_src, sflags, flags, id_max))
            src.free()
        sset.free()
    out.free(); dset.free()


@gpu
def test_remap_chained_sources(ctx):
    """a source from bm.scan and one from bm.aggregate, remapped where they lie; the translation vector sits at plane0 > 0"""
    v, nulls = gpu_vector(21, True, seed=3)
    rng = np.random.default_rng(5)
    a = BVector.from_words(bits_to_words(rng.random(6 * B) < 0.05)).optimize()
    b = BVector.from_words(bits_to_words(np.repeat(rng.random(6 * B // 256) < 0.5, 256))).optimize()
    sv = bm.SparseVector.from_values(v, nulls)
    vecs = [a, b] + list(sv.planes) + [sv.not_null]
    ps = PackedSet.pack(vecs, 6)
    dset = bm.DeviceSet.upload(ctx, ps)
    nn = 2 + len(sv.planes)
    agg = bm.aggregate(ctx, dset, bm.OP_OR, [0, 1], None, bm.F_OPT_COMPRESS)
    ids = np.flatnonzero(words_to_bits(a.to_words() | b.to_words()))
    for flags in (bm.F_OPT_COMPRESS, bm.F_OPT_NONE):
        res = bm.remap(ctx, dset, agg, 2, len(sv.planes), nn, ID_MAX32, flags)
        check_image(res, np_image(v, nulls, ids), len(sv.planes), flags, ("aggregate", flags))
        res.free()
    # elements >= 300000 inside NOT-NULL, as a scan finds them, then their distinct values
    scan = bm.scan(ctx, dset, bm.SCAN_GE, [300000], 2, len(sv.planes), nn, bm.F_OPT_COMPRESS)
    hit = np.flatnonzero((v >= 300000) & (nulls == 0))
    res = bm.remap(ctx, dset, scan, 2, len(sv.planes), nn, ID_MAX32, bm.F_OPT_COMPRESS)
    check_image(res, np_image(v, nulls, hit), len(sv.planes), bm.F_OPT_COMPRESS, "scan")
    res.free(); scan.free(); agg.free(); dset.free()


@gpu
def test_remap_all_65536_columns(ctx):
    """32 planes: one value in every image column (the last one 0xffffffff, left out), plus iid 32-bit values"""
    rng = np.random.default_rng(9)
    i = np.arange(B, dtype=np.uint64)
    v = np.concatenate([(i << np.uint64(16)) | ((i * np.uint64(7)) & np.uint64(0xFFFF)), i | np.uint64(0xFFFF0000),
                        rng.integers(0, 1 << 32, B, dtype=np.uint64)])
    v[B - 1] = ID_MAX32
    dset, nn, _ = upload_vector(ctx, v, None, 32, True)
    src_bits = np.ones(3 * B, np.uint8)
    sset = bm.DeviceSet.upload(ctx, PackedSet.pack([BVector.from_words(bits_to_words(src_bits))], 3))
    src = bm.aggregate(ctx, sset, bm.OP_OR, [0], None, bm.F_OPT_COMPRESS)
    want = np_image(v, None, np.arange(3 * B))
    for flags in (bm.F_OPT_COMPRESS, bm.F_OPT_NONE):
        res = bm.remap(ctx, dset, src, 0, 32, nn, ID_MAX32, flags)
        assert res.n_cols == 65536
        kind, pop, _, _ = res.meta()
        assert np.array_equal(pop, np.bincount((want >> np.uint64(16)).astype(np.int64), minlength=65536))
        assert (pop > 0).all() and res.total() == (want.size, True)
        if flags == bm.F_OPT_COMPRESS:
            assert (kind == bm.BLK_GAP).all()
        else:
            assert (kind == bm.BLK_BIT).all()
        got = bm.result_to_bvector(*res.fetch())
        assert np.array_equal(got.positions().astype(np.uint64), want)
        res.free()
    src.free(); sset.free(); dset.free()


@gpu
def test_remap_all_to_one_value(ctx):
    """M:1 at its extreme: every element of a 6-column vector holds 12345, every id in the source"""
    v = np.full(6 * B - 9, 12345, np.uint64)
    for nullable in (False, True):
        nulls = np.zeros(v.size, np.uint8) if nullable else None
        dset, nn, _ = upload_vector(ctx, v, nulls, 14, True)
        sset = bm.DeviceSet.upload(ctx, PackedSet.pack([BVector.from_words(bits_to_words(np.ones(6 * B, np.uint8)))], 6))
        src = bm.aggregate(ctx, sset, bm.OP_OR, [0], None, bm.F_OPT_COMPRESS)
        res = bm.remap(ctx, dset, src, 0, 14, nn, ID_MAX32, bm.F_OPT_COMPRESS)
        # the 9 ids past size(): 0 for the plain vector, nothing for the nullable one
        want = np.array([12345], np.uint64) if nullable else np.array([0, 12345], np.uint64)
        check_image(res, want, 14, bm.F_OPT_COMPRESS, nullable)
        res.free(); src.free(); sset.free(); dset.free()


@gpu
def test_remap_errors(ctx):
    v, nulls = gpu_vector(8, True)
    dset, nn, ps = upload_vector(ctx, v, nulls, 8, True)
    M = ps.n_vec
    sset = bm.DeviceSet.upload(ctx, PackedSet.pack([BVector.from_words(bits_to_words(source_bits(5, 1)))] * 2, 5))
    src = bm.aggregate(ctx, sset, bm.OP_OR, [0], None, bm.F_OPT_COMPRESS)
    lib = bm.capi.lib()

    def code(fn):
        with pytest.raises(bm.BMB200Error) as e:
            fn()
        return e.value.code

    rm = functools.partial(bm.remap, ctx, dset)
    assert code(lambda: rm(src, 0, 0, nn)) == 2                              # n_planes == 0
    assert code(lambda: rm(src, 0, 33, nn)) == 3                             # n_planes > 32
    assert code(lambda: rm(src, 2, 8, nn)) == 2                              # planes past the set
    assert code(lambda: rm(src, M - 1, 2)) == 2
    assert code(lambda: rm(src, 0, 8, M)) == 2                               # NOT-NULL id outside the set
    for f in (bm.F_COUNT_ONLY, bm.F_SIGNED, bm.F_OR_TARGET, 64):
        assert code(lambda: rm(src, 0, 8, nn, flags=f)) == 2
    assert code(lambda: rm(src, 0, 8, nn, result=src)) == 2                  # src == *inout
    cnt = bm.aggregate(ctx, sset, bm.OP_OR, [0], None, bm.F_COUNT_ONLY)      # no stored blocks
    assert code(lambda: rm(cnt, 0, 8, nn)) == 2
    two = bm.aggregate_batch(ctx, sset, bm.OP_OR, [([0], []), ([1], [])], bm.F_OPT_COMPRESS)   # two groups
    assert code(lambda: rm(two, 0, 8, nn)) == 2
    ctx2 = bm.Context(0)                                                     # a foreign context
    s2 = bm.DeviceSet.upload(ctx2, PackedSet.pack([BVector.from_words(bits_to_words(source_bits(5, 1)))], 5))
    src2 = bm.aggregate(ctx2, s2, bm.OP_OR, [0], None, bm.F_OPT_COMPRESS)
    assert code(lambda: rm(src2, 0, 8, nn)) == 2
    assert code(lambda: bm.remap(ctx2, dset, src2, 0, 8, nn)) == 2
    args = bm.capi.RemapArgsC(0, 8, nn, 0, ID_MAX32)
    out = C.c_void_p(0)
    assert lib.bmb200_remap(None, dset._h, C.byref(args), src._h, C.byref(out)) == 2
    assert lib.bmb200_remap(ctx._h, None, C.byref(args), src._h, C.byref(out)) == 2
    assert lib.bmb200_remap(ctx._h, dset._h, None, src._h, C.byref(out)) == 2
    assert lib.bmb200_remap(ctx._h, dset._h, C.byref(args), None, C.byref(out)) == 2
    assert lib.bmb200_remap(ctx._h, dset._h, C.byref(args), src._h, None) == 2
    assert not out.value                                                     # no result left behind by a refused call
    # the last plane and the last vector as NOT-NULL are inside the set
    ok = rm(src, 0, 8, nn)
    assert ok.n_cols == 1
    src2.free(); s2.free(); ctx2.close()
    for r in (ok, two, cnt, src):
        r.free()
    sset.free(); dset.free()


@gpu
@pytest.mark.parametrize("case", [c for c in CPU_CASES if not c[4]], ids=[c[0] for c in CPU_CASES if not c[4]])
def test_python_class_against_reference(ctx, case):
    """Set2SetTransform(sv).remap(BVector) and .remap(DeviceResult) == the recorded answers of the 32-bit reference"""
    name, values, nulls, ids, _ = case
    cnt, dg = ref_remap(values, nulls, ids, False, 0)
    sv = bm.SparseVector.from_values(values, nulls) if values.size else bm.SparseVector([BVector(1)], 0, None)
    tr = bm.Set2SetTransform(sv, ctx)
    n_cols = int(ids.max()) // B + 1 if ids.size else 1
    bits = np.zeros(n_cols * B, np.uint8); bits[ids] = 1
    bv_in = BVector.from_words(bits_to_words(bits)).optimize()
    got = tr.remap(bv_in)
    assert got.count() == cnt and np.array_equal(digest(got.positions()), dg), name
    dset = bm.DeviceSet.upload(ctx, PackedSet.pack([bv_in]))
    src = bm.aggregate(ctx, dset, bm.OP_OR, [0], None, bm.F_OPT_COMPRESS)
    got = tr.remap(src)
    assert got.count() == cnt and np.array_equal(digest(got.positions()), dg), name
    src.free(); dset.free(); tr.close()


@gpu
@pytest.mark.parametrize("exe", ["test_remap_binding", "test_remap_binding64"])
def test_remap_binding_harness(exe):
    path = orclib.ORACLE_DIR / "_ref" / exe
    if not path.exists():
        pytest.skip(f"oracle/_ref/{exe} is built only where the reference tree exists")
    p = subprocess.run([str(path)], capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-2000:]
    assert " 0 failed" in p.stdout
