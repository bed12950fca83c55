"""ctypes access to the CHECKERS (test infrastructure): oracle/liboracle.so (plain-C restatement) and, when
present, oracle/_ref/libbmref*.so (the unmodified reference compiled from /root/reference/src).
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference may import this."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

from bitmagic_b200.capi import (AggArgsC, BLOCK_WORDS, GAP_MAX_WORDS, PackedSetC, ScanArgsC, SCAN_RANGE, packed_c, ptr)  # noqa: F401

ROOT = Path(__file__).resolve().parent.parent
ORACLE_DIR = ROOT / "oracle"

_oracle = None
_ref = {}


def oracle() -> C.CDLL:
    global _oracle
    if _oracle is None:
        so = ORACLE_DIR / "liboracle.so"
        srcs = [ORACLE_DIR / "bm_oracle.c", ORACLE_DIR / "bm_oracle_entropy.c", ORACLE_DIR / "bm_synth.c"]
        if not so.exists() or so.stat().st_mtime < max(x.stat().st_mtime for x in srcs):
            subprocess.run(["make", "-C", str(ORACLE_DIR), str(so)], check=True, capture_output=True)
        _oracle = C.CDLL(str(so))
        _oracle.orc_synth_free.restype = None
        _oracle.orc_synth_packed.restype = None
        _oracle.orc_bit_block_count.restype = C.c_uint32
        _oracle.orc_block_digest.restype = C.c_uint64
        _oracle.orc_bit_block_calc_change.restype = C.c_uint32
        _oracle.orc_bit_to_gap.restype = C.c_uint32
        _oracle.orc_gap_bit_count.restype = C.c_uint32
        _oracle.orc_gap_bfind.restype = C.c_uint32
        _oracle.orc_gap_bit_count_range.restype = C.c_uint32
        _oracle.orc_bit_block_count_range.restype = C.c_uint32
    return _oracle


def _ref_name(addr64=False) -> str:
    """addr64: False = 32-bit addressing / AVX2 (the reference's own build flags), True = -DBM64ADDR, "avx512" = -DBMAVX512OPT"""
    return {False: "libbmref.so", True: "libbmref64.so", "avx512": "libbmref_avx512.so"}[addr64]


def have_ref(addr64=False) -> bool:
    return (ORACLE_DIR / "_ref" / _ref_name(addr64)).exists()


# Answers of the reference for the calls the tests make, one file per call, named by a hash of the function and its arguments.
# Where the reference library is built, the calls go to it, and BMB200_RECORD_REF=1 (re)writes these files; elsewhere the
# recorded answers stand in for it, so a checkout without the reference still compares against what the reference computed.
GOLDEN_REF = ROOT / "tests" / "golden" / "ref"


def have_ref_answers() -> bool:
    return have_ref() or GOLDEN_REF.is_dir()


def _hash_arg(x, h):
    if isinstance(x, np.ndarray):
        h.update(f"a{x.dtype.str}{x.shape}".encode()); h.update(np.ascontiguousarray(x).tobytes())
    elif hasattr(x, "gap_pool"):                                             # PackedSet
        h.update(f"ps{x.n_vec},{x.n_blocks}".encode())
        for a in (x.desc, x.bit_base, x.gap_base, x.bit_pool, x.gap_pool):
            _hash_arg(a, h)
    elif isinstance(x, (list, tuple, range)):
        h.update(b"[")
        for e in x:
            _hash_arg(e, h)
        h.update(b"]")
    elif isinstance(x, (bool, np.bool_)):
        h.update(b"T" if x else b"F")
    elif isinstance(x, (int, np.integer)):
        h.update(f"i{int(x)}".encode())
    else:
        h.update(repr(x).encode())


def _save_answer(path: Path, out) -> None:
    from bitmagic_b200.hostfmt import PackedSet
    items = list(out) if isinstance(out, tuple) else [out]
    arrays, tags = {}, []
    for i, x in enumerate(items):
        if isinstance(x, list):                                              # list of BVector (ref_sv_planes)
            ps = PackedSet.pack(x, gap_flat=False)
            tags.append("P")
            for a in ("desc", "bit_base", "gap_base", "bit_pool", "gap_pool"):
                arrays[f"o{i}_{a}"] = getattr(ps, a)
            arrays[f"o{i}_shape"] = np.array([ps.n_vec, ps.n_blocks])
        else:
            tags.append("b" if isinstance(x, bool) else "i" if isinstance(x, int) else "t" if isinstance(x, tuple) else "a")
            arrays[f"o{i}"] = np.asarray(x)
    path.parent.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(path, tags=np.array("".join(tags) + ("" if isinstance(out, tuple) else "!")), **arrays)


def _load_answer(path: Path):
    from bitmagic_b200.hostfmt import PackedSet
    with np.load(path) as z:
        tags = str(z["tags"])
        items = []
        for i, t in enumerate(tags.rstrip("!")):
            if t == "P":
                nv, nb = (int(x) for x in z[f"o{i}_shape"])
                ps = PackedSet(nv, nb, *(z[f"o{i}_{a}"] for a in ("desc", "bit_base", "gap_base", "bit_pool", "gap_pool")))
                items.append([ps.vector(v) for v in range(nv)])
            else:
                a = z[f"o{i}"]
                items.append(bool(a) if t == "b" else int(a) if t == "i" else tuple(a.tolist()) if t == "t" else a)
    return items[0] if tags.endswith("!") else tuple(items)


def _same_answer(live, rec) -> bool:
    """live == recorded, item by item; timings (plain tuples of floats) are not part of an answer."""
    from bitmagic_b200.hostfmt import PackedSet
    if isinstance(live, tuple) and not all(isinstance(x, float) for x in live):
        return len(live) == len(rec) and all(_same_answer(a, b) for a, b in zip(live, rec))
    if isinstance(live, tuple):
        return True
    if isinstance(live, list):
        pa, pb = PackedSet.pack(live, gap_flat=False), PackedSet.pack(rec, gap_flat=False)
        return all(np.array_equal(getattr(pa, a), getattr(pb, a)) for a in ("desc", "bit_base", "gap_base", "bit_pool", "gap_pool"))
    return bool(np.array_equal(np.asarray(live), np.asarray(rec)))


def _recorded(fn=None, *, entry=None):
    """entry: the shim function the call needs.  A reference library built from an older shim that lacks it is treated as absent
    for this call, so the recorded answer stands in for it as it does where no library was built."""
    import functools
    import hashlib
    import os

    if fn is None:
        return functools.partial(_recorded, entry=entry)

    def live(addr64):
        return have_ref(addr64) and (entry is None or hasattr(ref(addr64), entry))

    @functools.wraps(fn)
    def call(*args, **kw):
        h = hashlib.sha256(fn.__name__.encode())
        _hash_arg(args, h); _hash_arg(sorted(kw.items()), h)
        path = GOLDEN_REF / f"{fn.__name__}_{h.hexdigest()[:20]}.npz"
        if live(kw.get("addr64", False)):
            out = fn(*args, **kw)
            if os.environ.get("BMB200_RECORD_REF"):
                _save_answer(path, out)
            elif path.exists():             # a recorded answer that no longer matches the reference is stale: say so here
                assert _same_answer(out, _load_answer(path)), f"{path.name} differs from the reference's answer; re-record it"
            return out
        if not path.exists():
            raise FileNotFoundError(f"reference library not built (or without this entry) and no recorded answer {path.name} for this {fn.__name__} call")
        return _load_answer(path)
    return call


def cpu_has_avx512() -> bool:
    try:
        flags = next(ln for ln in open("/proc/cpuinfo") if ln.startswith("flags")).split()
    except Exception:
        return False
    return all(f in flags for f in ("avx512f", "avx512bw", "avx512vl", "avx512dq"))


def ref(addr64=False) -> C.CDLL:
    key = addr64
    if key not in _ref:
        lib = C.CDLL(str(ORACLE_DIR / "_ref" / _ref_name(addr64)))
        lib.ref_simd.restype = C.c_char_p
        lib.ref_job_create.restype = C.c_void_p
        lib.ref_job_free.restype = None
        _ref[key] = lib
    return _ref[key]


class HostSynth:
    """orc_synth_create (oracle/bm_synth.c): the benchmark's generator restated on the host -> a PackedSet whose arrays are
    views into the C object (kept alive by this wrapper)."""

    def __init__(self, n_vec, n_blocks, density, seed, optimize, threads=0):
        import os
        from bitmagic_b200.hostfmt import PackedSet
        dens = np.ascontiguousarray(density, dtype=np.float64); sd = np.ascontiguousarray(seed, dtype=np.uint64)
        assert dens.size == n_vec and sd.size == n_vec
        self.h = C.c_void_p(0)
        rc = oracle().orc_synth_create(C.c_uint32(n_vec), C.c_uint32(n_blocks), ptr(dens), ptr(sd), int(bool(optimize)),
                                       int(threads or os.cpu_count() or 1), C.byref(self.h))
        assert rc == 0, f"orc_synth_create rc={rc}"
        c = PackedSetC()
        oracle().orc_synth_packed(self.h, C.byref(c))
        self.c = c

        def view(p, n, ct, dt):
            if not n:
                return np.zeros(0, dt)
            return np.ctypeslib.as_array(C.cast(p, C.POINTER(ct)), shape=(n,))
        bb = view(c.bit_base, n_blocks + 1, C.c_uint64, np.uint64); gb = view(c.gap_base, n_blocks + 1, C.c_uint64, np.uint64)
        self.ps = PackedSet(n_vec, n_blocks, view(c.desc, n_vec * n_blocks, C.c_uint32, np.uint32), bb, gb,
                            view(c.bit_pool, int(bb[-1]) * BLOCK_WORDS, C.c_uint32, np.uint32),
                            view(c.gap_pool, int(gb[-1]) * 8, C.c_uint16, np.uint16))

    def free(self):
        if self.h:
            self.ps = None
            oracle().orc_synth_free(self.h)
            self.h = C.c_void_p(0)

    def __del__(self):  # pragma: no cover
        try:
            self.free()
        except Exception:
            pass


class RefJob:
    """Persistent reference job (oracle/ref_shim.cpp ref_job_*): bvectors built once, T worker threads, timed passes,
    per-column kind / popcount / digest / GAP length of the result."""

    def __init__(self, ps, op, g0, g1=None, flags=0, threads=1, nb_from=0, nb_to=0, variant=False):
        self.lib = ref(variant)
        a, self._keep = _args(op, g0, g1, flags, nb_from, nb_to)
        c = _pc(ps)
        self.n_cols = (nb_to if nb_to else ps.n_blocks) - nb_from
        self.h = C.c_void_p(self.lib.ref_job_create(C.byref(c), C.byref(a), int(threads)))
        assert self.h, "ref_job_create failed"
        self.threads = self.lib.ref_job_threads(self.h)

    def run(self, repeats=1):
        sec = np.zeros(repeats, np.float64); tot = C.c_uint64(0)
        rc = self.lib.ref_job_run(self.h, int(repeats), ptr(sec), C.byref(tot))
        assert rc == 0, f"ref_job_run rc={rc}"
        return sec, tot.value

    def export(self):
        n = self.n_cols
        kind = np.zeros(n, np.uint8); pop = np.zeros(n, np.uint32); dig = np.zeros(n, np.uint64); gl = np.zeros(n, np.uint32)
        rc = self.lib.ref_job_export(self.h, ptr(kind), ptr(pop), ptr(dig), ptr(gl))
        assert rc == 0, f"ref_job_export rc={rc}"
        return kind, pop, dig, gl

    def free(self):
        if self.h:
            self.lib.ref_job_free(self.h)
            self.h = C.c_void_p(0)

    def __del__(self):  # pragma: no cover
        try:
            self.free()
        except Exception:
            pass


def _args(op, g0, g1, flags, nb_from=0, nb_to=0):
    g0 = np.ascontiguousarray(g0, dtype=np.uint32)
    g1 = np.ascontiguousarray(g1 if g1 is not None else [], dtype=np.uint32)
    a = AggArgsC(int(op), int(flags), ptr(g0) if g0.size else C.c_void_p(0), g0.size,
                 ptr(g1) if g1.size else C.c_void_p(0), g1.size, int(nb_from), int(nb_to))
    return a, (g0, g1)


def _pc(ps) -> PackedSetC:
    return packed_c(ps.n_vec, ps.n_blocks, ps.desc, ps.bit_base, ps.gap_base, ps.bit_pool, ps.gap_pool)


def oracle_aggregate(ps, op, g0, g1=None, flags=0, nb_from=0, nb_to=0):
    """-> kind, popcnt, digest, nruns, blocks[n_cols][2048], gaps[n_cols][1280]"""
    n = (nb_to if nb_to else ps.n_blocks) - nb_from
    a, keep = _args(op, g0, g1, flags, nb_from, nb_to)
    kind = np.zeros(n, np.uint8); pop = np.zeros(n, np.uint32); dig = np.zeros(n, np.uint64); nr = np.zeros(n, np.uint32)
    blocks = np.zeros((n, BLOCK_WORDS), np.uint32); gaps = np.zeros((n, GAP_MAX_WORDS), np.uint16)
    c = _pc(ps)
    rc = oracle().orc_aggregate(C.byref(c), C.byref(a), ptr(kind), ptr(pop), ptr(dig), ptr(nr), ptr(blocks), ptr(gaps))
    assert rc == 0, f"orc_aggregate rc={rc}"
    return kind, pop, dig, nr, blocks, gaps


@_recorded
def ref_synth_columns(n_vec, n_blocks, density, seed, optimize, op, g0, g1=None, flags=0):
    """The reference aggregator (a RefJob on every host core) over the benchmark generator's set for these parameters ->
    total, kind, popcnt, digest, GAP length of every column, and the stored bytes of the generated set.  Keyed by the
    generator's parameters, so that full-size sets are neither hashed nor, where the answers are recorded, generated."""
    import os
    threads = os.cpu_count() or 1
    hs = HostSynth(n_vec, n_blocks, density, seed, optimize, threads=threads)
    job = RefJob(hs.ps, op, g0, g1, flags, threads=threads)
    sec, tot = job.run(1)
    k, p, d, gl = job.export()
    stored = hs.ps.stored_bytes()
    job.free(); hs.free()
    return int(tot), k, p, d, gl, int(stored)


@_recorded
def ref_aggregate(ps, op, g0, g1=None, flags=0, horizontal=False, addr64=False):
    """The real reference -> kind, popcnt, blocks, gaps, any"""
    n = ps.n_blocks
    a, keep = _args(op, g0, g1, flags)
    kind = np.zeros(n, np.uint8); pop = np.zeros(n, np.uint32)
    blocks = np.zeros((n, BLOCK_WORDS), np.uint32); gaps = np.zeros((n, GAP_MAX_WORDS), np.uint16)
    any_ = C.c_int(0)
    c = _pc(ps)
    if horizontal:
        rc = ref(addr64).ref_aggregate_horizontal(C.byref(c), C.byref(a), ptr(kind), ptr(pop), ptr(blocks))
    else:
        rc = ref(addr64).ref_aggregate(C.byref(c), C.byref(a), ptr(kind), ptr(pop), ptr(blocks), ptr(gaps), C.byref(any_))
    assert rc == 0, f"ref_aggregate rc={rc}"
    return kind, pop, blocks, gaps, bool(any_.value)


@_recorded
def ref_binop(ps, op, va, vb, compress=False):
    """op: 0 OR 1 AND 2 SUB 3 XOR (bvector::bit_* 3-operand) -> kind, popcnt, blocks, count"""
    n = ps.n_blocks
    kind = np.zeros(n, np.uint8); pop = np.zeros(n, np.uint32); blocks = np.zeros((n, BLOCK_WORDS), np.uint32)
    cnt = C.c_uint64(0)
    c = _pc(ps)
    rc = ref().ref_binop(C.byref(c), int(op), int(va), int(vb), int(compress), ptr(kind), ptr(pop), ptr(blocks), C.byref(cnt))
    assert rc == 0
    return kind, pop, blocks, cnt.value


@_recorded(entry="ref_binop_gaps")
def ref_binop_gaps(ps, op, va, vb, compress=False):
    """ref_binop with the result's GAP words: op 0 OR 1 AND 2 SUB 3 XOR -> kind, popcnt, blocks, gaps[n_cols][1280]"""
    n = ps.n_blocks
    kind = np.zeros(n, np.uint8); pop = np.zeros(n, np.uint32)
    blocks = np.zeros((n, BLOCK_WORDS), np.uint32); gaps = np.zeros((n, GAP_MAX_WORDS), np.uint16)
    c = _pc(ps)
    rc = ref().ref_binop_gaps(C.byref(c), int(op), int(va), int(vb), int(compress), ptr(kind), ptr(pop), ptr(blocks), ptr(gaps))
    assert rc == 0, f"ref_binop_gaps rc={rc}"
    return kind, pop, blocks, gaps


@_recorded
def ref_count_op(ps, op, va, vb) -> int:
    out = C.c_uint64(0)
    c = _pc(ps)
    rc = ref().ref_count_op(C.byref(c), int(op), int(va), int(vb), C.byref(out))
    assert rc == 0
    return out.value


@_recorded
def ref_optimize(ps, v):
    n = ps.n_blocks
    kind = np.zeros(n, np.uint8); pop = np.zeros(n, np.uint32)
    blocks = np.zeros((n, BLOCK_WORDS), np.uint32); gaps = np.zeros((n, GAP_MAX_WORDS), np.uint16)
    c = _pc(ps)
    rc = ref().ref_optimize(C.byref(c), int(v), ptr(kind), ptr(pop), ptr(blocks), ptr(gaps))
    assert rc == 0
    return kind, pop, blocks, gaps


def oracle_rs_build(ps, v):
    nb = ps.n_blocks; nsb = (nb + 255) // 256
    bc = np.zeros(nb, np.uint32); sc = np.zeros(nb, np.uint64); sb = np.zeros(nsb + 1, np.uint64)
    c = _pc(ps)
    rc = oracle().orc_rs_build(C.byref(c), int(v), ptr(bc), ptr(sc), ptr(sb))
    assert rc == 0
    return bc, sc, sb


@_recorded
def ref_rs_build(ps, v, addr64=False):
    nb = ps.n_blocks; nsb = (nb + 255) // 256
    bc = np.zeros(nb, np.uint32); sc = np.zeros(nb, np.uint64); sb = np.zeros(nsb + 1, np.uint64)
    tot = C.c_uint64(0)
    c = _pc(ps)
    rc = ref(addr64).ref_rs_build(C.byref(c), int(v), ptr(bc), ptr(sc), ptr(sb), C.byref(tot))
    assert rc == 0
    return bc, sc, sb, tot.value


def oracle_rank(ps, v, pos):
    p = np.ascontiguousarray(pos, dtype=np.uint64); out = np.zeros(p.size, np.uint64)
    c = _pc(ps)
    rc = oracle().orc_rank_batch(C.byref(c), int(v), ptr(p), C.c_uint64(p.size), ptr(out))
    assert rc == 0
    return out


def oracle_select(ps, v, rank):
    r = np.ascontiguousarray(rank, dtype=np.uint64)
    pos = np.zeros(r.size, np.uint64); found = np.zeros(r.size, np.uint8)
    c = _pc(ps)
    rc = oracle().orc_select_batch(C.byref(c), int(v), ptr(r), C.c_uint64(r.size), ptr(pos), ptr(found))
    assert rc == 0
    return pos, found.astype(bool)


@_recorded
def ref_rank_select(ps, v, pos, rank, addr64=False):
    """-> rank_out, pos_out, found, (sec_build, sec_rank, sec_select)"""
    p = np.ascontiguousarray(pos, dtype=np.uint64); r = np.ascontiguousarray(rank, dtype=np.uint64)
    ro = np.zeros(p.size, np.uint64); po = np.zeros(r.size, np.uint64); fo = np.zeros(r.size, np.uint8)
    tb, tr, ts = C.c_double(0), C.c_double(0), C.c_double(0)
    c = _pc(ps)
    rc = ref(addr64).ref_rank_select(C.byref(c), int(v), ptr(p), C.c_uint64(p.size), ptr(ro),
                                     ptr(r), C.c_uint64(r.size), ptr(po), ptr(fo),
                                     C.byref(tb), C.byref(tr), C.byref(ts))
    assert rc == 0
    return ro, po, fo.astype(bool), (tb.value, tr.value, ts.value)


def ref_time_aggregate(ps, op, g0, g1=None, flags=0, threads=1, repeats=3, nb_from=0, nb_to=0, addr64=False):
    a, keep = _args(op, g0, g1, flags, nb_from, nb_to)
    best = C.c_double(0); tot = C.c_uint64(0)
    c = _pc(ps)
    rc = ref(addr64).ref_time_aggregate(C.byref(c), C.byref(a), int(threads), int(repeats), C.byref(best), C.byref(tot))
    assert rc == 0
    return best.value, tot.value


@_recorded
def ref_pipeline(ps, groups, want_or=False):
    """The real aggregator::pipeline -> counts[n_groups], kind/pop/blocks [n_groups][n_blocks], (or_kind, or_blocks)"""
    mem, off = [], [0]
    for g0, g1 in groups:
        mem.extend(int(x) for x in g0); off.append(len(mem))
        mem.extend(int(x) for x in (g1 if g1 is not None else [])); off.append(len(mem))
    members = np.ascontiguousarray(mem, dtype=np.uint32); offsets = np.ascontiguousarray(off, dtype=np.uint32)
    ng, nb = len(groups), ps.n_blocks
    counts = np.zeros(ng, np.uint64); kind = np.zeros((ng, nb), np.uint8); pop = np.zeros((ng, nb), np.uint32)
    blocks = np.zeros((ng, nb, BLOCK_WORDS), np.uint32)
    or_kind = np.zeros(nb, np.uint8); or_blocks = np.zeros((nb, BLOCK_WORDS), np.uint32)
    c = _pc(ps)
    rc = ref().ref_pipeline(C.byref(c), ng, ptr(members), ptr(offsets), int(want_or), ptr(counts), ptr(kind), ptr(pop), ptr(blocks),
                            ptr(or_kind), ptr(or_blocks))
    assert rc == 0
    return counts, kind, pop, blocks, or_kind, or_blocks


def oracle_scan(ps, pred, values, plane0, n_planes, universe=0xFFFFFFFF, flags=0, nb_from=0, nb_to=0):
    """orc_scan -> kind, popcnt, digest, nruns, blocks[n_values*n_cols][2048], gaps[...][1280] (value-major)"""
    vals = np.ascontiguousarray(values, dtype=np.uint64)
    nv = vals.shape[0] if pred == SCAN_RANGE else vals.size
    n = ((nb_to if nb_to else ps.n_blocks) - nb_from) * nv
    a = ScanArgsC(int(plane0), int(n_planes), int(universe), int(pred), int(flags), ptr(vals), int(nv), int(nb_from), int(nb_to))
    kind = np.zeros(n, np.uint8); pop = np.zeros(n, np.uint32); dig = np.zeros(n, np.uint64); nr = np.zeros(n, np.uint32)
    blocks = np.zeros((n, BLOCK_WORDS), np.uint32); gaps = np.zeros((n, GAP_MAX_WORDS), np.uint16)
    c = _pc(ps)
    rc = oracle().orc_scan(C.byref(c), C.byref(a), ptr(kind), ptr(pop), ptr(dig), ptr(nr), ptr(blocks), ptr(gaps))
    assert rc == 0, f"orc_scan rc={rc}"
    return kind, pop, dig, nr, blocks, gaps


@_recorded
def ref_sv_planes(values, nulls=None, max_planes=64):
    """The real bm::sparse_vector<unsigned>: its optimize()d planes + the universe as a list of BVector (planes..., universe)."""
    import bitmagic_b200 as bm
    v = np.ascontiguousarray(values, dtype=np.uint32)
    nl = None if nulls is None else np.ascontiguousarray(nulls, dtype=np.uint8)
    n_cols = max(1, (v.size + 65535) // 65536)
    kind = np.zeros((max_planes + 1) * n_cols, np.uint8)
    blocks = np.zeros(((max_planes + 1) * n_cols, BLOCK_WORDS), np.uint32)
    gaps = np.zeros(((max_planes + 1) * n_cols, GAP_MAX_WORDS), np.uint16)
    npl = C.c_uint32(0)
    rc = ref().ref_sv_planes(ptr(v), ptr(nl) if nl is not None else C.c_void_p(0), C.c_uint64(v.size), C.c_uint32(n_cols), C.c_uint32(max_planes),
                             C.byref(npl), ptr(kind), ptr(blocks), ptr(gaps))
    assert rc == 0, f"ref_sv_planes rc={rc}"
    out = []
    for j in range(npl.value + 1):
        bv = bm.BVector(n_cols)
        for c in range(n_cols):
            k = int(kind[j * n_cols + c])
            if k == bm.BLK_FULL:
                bv.set_full(c)
            elif k == bm.BLK_BIT:
                bv.set_bits(c, blocks[j * n_cols + c])
            elif k == bm.BLK_GAP:
                g = gaps[j * n_cols + c]
                bv.set_gap(c, g[:(int(g[0]) >> 3) + 1])
        out.append(bv)
    return out


@_recorded
def ref_sv_scan(values, nulls, pred, search):
    """The real sparse_vector_scanner -> counts[n_search], kind, popcnt, blocks[n_search*n_cols][2048] (value-major)"""
    v = np.ascontiguousarray(values, dtype=np.uint32)
    nl = None if nulls is None else np.ascontiguousarray(nulls, dtype=np.uint8)
    sv = np.ascontiguousarray(search, dtype=np.uint32)
    ns = sv.shape[0] if pred == SCAN_RANGE else sv.size
    n_cols = max(1, (v.size + 65535) // 65536)
    counts = np.zeros(ns, np.uint64); kind = np.zeros(ns * n_cols, np.uint8); pop = np.zeros(ns * n_cols, np.uint32)
    blocks = np.zeros((ns * n_cols, BLOCK_WORDS), np.uint32)
    rc = ref().ref_sv_scan(ptr(v), ptr(nl) if nl is not None else C.c_void_p(0), C.c_uint64(v.size), int(pred), ptr(sv), C.c_uint32(ns),
                           C.c_uint32(n_cols), ptr(counts), ptr(kind), ptr(pop), ptr(blocks))
    assert rc == 0, f"ref_sv_scan rc={rc}"
    return counts, kind, pop, blocks


def ref_sv_time_scan(values, nulls, pred, search, repeats=2):
    """seconds (best of repeats) for the reference scanner to answer all `search` values + the summed cardinality"""
    v = np.ascontiguousarray(values, dtype=np.uint32)
    nl = None if nulls is None else np.ascontiguousarray(nulls, dtype=np.uint8)
    sv = np.ascontiguousarray(search, dtype=np.uint32)
    ns = sv.shape[0] if pred == SCAN_RANGE else sv.size
    sec, tot = C.c_double(0), C.c_uint64(0)
    rc = ref().ref_sv_time_scan(ptr(v), ptr(nl) if nl is not None else C.c_void_p(0), C.c_uint64(v.size), int(pred), ptr(sv), C.c_uint32(ns),
                                int(repeats), C.byref(sec), C.byref(tot))
    assert rc == 0, f"ref_sv_time_scan rc={rc}"
    return sec.value, tot.value


def ref_serialize(ps, v, level, addr64=False):
    """bm::serializer<> at `level` on vector v of the packed set -> bytes (addr64: the BM64ADDR build of the reference)"""
    cap = int(ps.n_blocks) * 8300 + 4096
    out = np.zeros(cap, np.uint8); size = C.c_uint64(0)
    c = _pc(ps)
    rc = ref(addr64).ref_serialize(C.byref(c), C.c_uint32(v), int(level), ptr(out), C.c_uint64(cap), C.byref(size))
    assert rc == 0, f"ref_serialize rc={rc}"
    return out[:size.value].copy()


def ref_serialize_bookmarks(ps, v, level, interval):
    """bm::serializer<> with set_bookmarks(true, interval): BLOB of vector v at the given compression level"""
    cap = 64 + ps.n_blocks * (BLOCK_WORDS * 4 + 64)
    out = np.zeros(cap, np.uint8); size = C.c_uint64(0)
    c = _pc(ps)
    rc = ref().ref_serialize_bookmarks(C.byref(c), C.c_uint32(v), C.c_int(level), C.c_uint32(interval), ptr(out), C.c_uint64(cap), C.byref(size))
    assert rc == 0, f"ref_serialize_bookmarks rc={rc}"
    return out[:size.value].copy()


def ref_deserialize(blob, n_cols, addr64=False):
    """bm::deserialize -> kind, popcnt, blocks[n_cols][2048], gaps[n_cols][1280]"""
    b = np.ascontiguousarray(blob, dtype=np.uint8)
    kind = np.zeros(n_cols, np.uint8); pop = np.zeros(n_cols, np.uint32)
    blocks = np.zeros((n_cols, BLOCK_WORDS), np.uint32); gaps = np.zeros((n_cols, GAP_MAX_WORDS), np.uint16)
    rc = ref(addr64).ref_deserialize(ptr(b), C.c_uint32(n_cols), ptr(kind), ptr(pop), ptr(blocks), ptr(gaps))
    assert rc == 0, f"ref_deserialize rc={rc}"
    return kind, pop, blocks, gaps


def oracle_deserialize(blob, n_cols):
    """orc_deserialize -> rc, kind, blocks[n_cols][2048], gaps[n_cols][1280]"""
    b = np.ascontiguousarray(blob, dtype=np.uint8)
    kind = np.zeros(n_cols, np.uint8)
    blocks = np.zeros((n_cols, BLOCK_WORDS), np.uint32); gaps = np.zeros((n_cols, GAP_MAX_WORDS), np.uint16)
    rc = oracle().orc_deserialize(ptr(b), C.c_uint64(b.size), C.c_uint32(n_cols), ptr(kind), ptr(blocks), ptr(gaps))
    return rc, kind, blocks, gaps


_blobhost = None


def blobhost() -> C.CDLL:
    """Host build of the product's BLOB walker / entropy decoder header (oracle/blob_host_check.cpp): a checker, not a product path."""
    global _blobhost
    if _blobhost is None:
        so = ORACLE_DIR / "libblobhost.so"
        srcs = [ORACLE_DIR / "blob_host_check.cpp", ROOT / "bitmagic_b200" / "csrc" / "blob_entropy.cuh"]
        if not so.exists() or so.stat().st_mtime < max(x.stat().st_mtime for x in srcs):
            subprocess.run(["make", "-C", str(ORACLE_DIR), str(so)], check=True, capture_output=True)
        _blobhost = C.CDLL(str(so))
    return _blobhost


def blob_host_check(blob, n_cols):
    """-> rc, kind, decoded (1 = block came from an entropy-coded token), gap_words, blocks, gaps, n_entropy_tokens"""
    b = np.ascontiguousarray(blob, dtype=np.uint8)
    kind = np.zeros(n_cols, np.uint8); dec = np.zeros(n_cols, np.uint8); gw = np.zeros(n_cols, np.uint32)
    blocks = np.zeros((n_cols, BLOCK_WORDS), np.uint32); gaps = np.zeros((n_cols, GAP_MAX_WORDS), np.uint16)
    n_ent = C.c_uint32(0); n_seg = C.c_uint32(0)
    rc = blobhost().blob_host_check(ptr(b), C.c_uint64(b.size), C.c_uint32(n_cols), ptr(kind), ptr(dec), ptr(gw), ptr(blocks), ptr(gaps),
                                    C.byref(n_ent), C.byref(n_seg))
    blob_host_check.last_segments = n_seg.value
    return rc, kind, dec, gw, blocks, gaps, n_ent.value


def oracle_token_hist(enable=True):
    """256 counters filled by orc_deserialize (one per serializer token type met); call with False to switch off"""
    h = np.zeros(256, np.uint32)
    oracle().orc_set_token_hist(ptr(h) if enable else C.c_void_p(0))
    return h
