"""ctypes binding of libbmb200.so (the C ABI declared in include/bmb200.h).

The shared library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).  There is no
fallback: if the library is missing, or no H100 is present, every entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ.get("BMB200_LIB", str(_HERE / "libbmb200.so")))   # load another build, e.g. to compare two builds on the same inputs

# ---- constants (mirror include/bmb200.h) ----
OK = 0
ERR_BADALLOC, ERR_BADARG, ERR_RANGE, ERR_RS_IDX_MISSING = 1, 2, 3, 7
ERR_CUDA, ERR_NODEVICE, ERR_UNSUPPORTED = 200, 201, 202
BLOCK_WORDS, BLOCK_BYTES, BLOCK_BITS = 2048, 8192, 65536
GAP_MAX_WORDS, GAP_THRESHOLD, GAP_UNIT_WORDS, SUPERBLOCK = 1280, 1276, 8, 256
BLK_NULL, BLK_FULL, BLK_BIT, BLK_GAP = 0, 1, 2, 3
OP_OR, OP_AND, OP_AND_SUB, OP_XOR, OP_SHIFT_R_AND = 0, 1, 2, 3, 4
F_COUNT_ONLY, F_OPT_NONE, F_OPT_COMPRESS, F_OR_TARGET = 1, 0, 2, 4

# every symbol include/bmb200.h declares (checked by tests/test_cabi_symbols.py)
SYMBOLS = [
    "bmb200_init", "bmb200_destroy", "bmb200_error_msg", "bmb200_last_error", "bmb200_ctx_set_stream",
    "bmb200_ctx_get_stream", "bmb200_ctx_sync", "bmb200_ctx_launch_count", "bmb200_device_info", "bmb200_ctx_set_tuning",
    "bmb200_set_upload", "bmb200_set_upload_vectors", "bmb200_set_adopt_device", "bmb200_set_info",
    "bmb200_set_column_sizes", "bmb200_set_download", "bmb200_set_device_ptrs", "bmb200_set_free",
    "bmb200_synth_set", "bmb200_aggregate", "bmb200_result_optimize", "bmb200_result_total",
    "bmb200_result_fetch_meta", "bmb200_result_sizes", "bmb200_result_fetch", "bmb200_result_device_ptrs",
    "bmb200_result_free", "bmb200_aggregate_host", "bmb200_rs_build", "bmb200_rs_export", "bmb200_rs_total",
    "bmb200_rank_batch", "bmb200_select_batch", "bmb200_rank_batch_dev", "bmb200_select_batch_dev",
    "bmb200_rs_free", "bmb200_rs_rebuild", "bmb200_aggregate_batch", "bmb200_result_group_totals", "bmb200_result_or_target",
    "bmb200_scan", "bmb200_set_upload_blobs", "bmb200_result_fetch_view", "bmb200_ctx_bind_host_numa",
    "bmb200_shard_range", "bmb200_comm_unique_id", "bmb200_comm_init", "bmb200_comm_info", "bmb200_comm_destroy",
    "bmb200_exchange_popcounts", "bmb200_exchange_fence", "bmb200_exchange_fetch", "bmb200_ctx_trim", "bmb200_binop",
    "bmb200_set_upload_slabs", "bmb200_host_slabs_prefetch", "bmb200_host_slab_alloc", "bmb200_host_slab_free",
    "bmb200_result_fetch_view_async", "bmb200_result_fetch_wait", "bmb200_exchange_mode",
    "bmb200_result_fetch_column", "bmb200_set_run_lists", "bmb200_set_bit_run_lists",
    "bmb200_rank_decompress", "bmb200_rank_compress",
]
OP_SUB = 5
COMM_ID_BYTES = 128
TUNE_GAP_MODE, TUNE_CTAS_PER_SM, TUNE_HOST_THREADS, TUNE_AGG_PIPELINE, TUNE_RUN_LISTS = 0, 1, 2, 3, 4


class PackedSetC(C.Structure):
    _fields_ = [
        ("n_vec", C.c_uint32), ("n_blocks", C.c_uint32),
        ("desc", C.c_void_p), ("bit_base", C.c_void_p), ("gap_base", C.c_void_p),
        ("bit_pool", C.c_void_p), ("gap_pool", C.c_void_p),
    ]


class VecBlocksC(C.Structure):
    _fields_ = [("n_blocks", C.c_uint32), ("kind", C.c_void_p), ("ptr", C.c_void_p)]


class HostSlabC(C.Structure):
    _fields_ = [("base", C.c_void_p), ("bytes", C.c_uint64)]


class AggArgsC(C.Structure):
    _fields_ = [
        ("op", C.c_int32), ("flags", C.c_uint32),
        ("group0", C.c_void_p), ("n0", C.c_uint32),
        ("group1", C.c_void_p), ("n1", C.c_uint32),
        ("nb_from", C.c_uint32), ("nb_to", C.c_uint32),
    ]


class BatchArgsC(C.Structure):
    _fields_ = [
        ("op", C.c_int32), ("flags", C.c_uint32), ("n_groups", C.c_uint32),
        ("members", C.c_void_p), ("offsets", C.c_void_p),
        ("nb_from", C.c_uint32), ("nb_to", C.c_uint32),
    ]


class BlobC(C.Structure):
    _fields_ = [("data", C.c_void_p), ("size", C.c_uint64)]


class ScanArgsC(C.Structure):
    _fields_ = [
        ("plane0", C.c_uint32), ("n_planes", C.c_uint32), ("universe", C.c_uint32),
        ("pred", C.c_int32), ("flags", C.c_uint32),
        ("values", C.c_void_p), ("n_values", C.c_uint32),
        ("nb_from", C.c_uint32), ("nb_to", C.c_uint32),
    ]


SCAN_EQ, SCAN_GT, SCAN_GE, SCAN_LT, SCAN_LE, SCAN_RANGE = range(6)
NO_UNIVERSE = 0xFFFFFFFF


class ResultMetaC(C.Structure):
    _fields_ = [("kind", C.c_void_p), ("popcnt", C.c_void_p), ("digest", C.c_void_p), ("nruns", C.c_void_p)]


class BMB200Error(RuntimeError):
    def __init__(self, code: int, what: str, detail: str = ""):
        self.code = code
        super().__init__(f"{what}: error {code} ({_msg(code)})" + (f" [{detail}]" if detail else ""))


_lib = None


def lib() -> C.CDLL:
    """Load libbmb200.so; fail loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise ImportError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
                "bitmagic_b200 has no CPU fallback.")
        _lib = C.CDLL(str(LIB_PATH))
        _lib.bmb200_error_msg.restype = C.c_char_p
        _lib.bmb200_error_msg.argtypes = [C.c_int]
        for name in SYMBOLS:
            if name != "bmb200_error_msg":
                getattr(_lib, name).restype = C.c_int
    return _lib


def _msg(code: int) -> str:
    try:
        return lib().bmb200_error_msg(code).decode()
    except Exception:  # pragma: no cover
        return "?"


def ptr(a) -> C.c_void_p:
    if a is None:
        return C.c_void_p(0)
    return C.c_void_p(a.ctypes.data)


def packed_c(n_vec, n_blocks, desc, bit_base, gap_base, bit_pool, gap_pool) -> PackedSetC:
    return PackedSetC(int(n_vec), int(n_blocks), ptr(desc), ptr(bit_base), ptr(gap_base),
                      ptr(bit_pool) if bit_pool is not None and bit_pool.size else C.c_void_p(0),
                      ptr(gap_pool) if gap_pool is not None and gap_pool.size else C.c_void_p(0))


class Context:
    """One per process per GPU (bmb200_ctx)."""

    def __init__(self, device: int = 0):
        self._h = C.c_void_p(0)
        rc = lib().bmb200_init(int(device), C.byref(self._h))
        if rc != OK:
            raise BMB200Error(rc, "bmb200_init")
        self.device = device

    def check(self, rc: int, what: str):
        if rc != OK:
            buf = C.create_string_buffer(512)
            lib().bmb200_last_error(self._h, buf, C.c_size_t(512))
            raise BMB200Error(rc, what, buf.value.decode(errors="replace"))

    def close(self):
        if self._h:
            lib().bmb200_destroy(self._h)
            self._h = C.c_void_p(0)

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        self.check(lib().bmb200_ctx_sync(self._h), "ctx_sync")

    def set_stream(self, cuda_stream: int):
        self.check(lib().bmb200_ctx_set_stream(self._h, C.c_void_p(int(cuda_stream))), "ctx_set_stream")

    def get_stream(self) -> int:
        s = C.c_void_p(0)
        self.check(lib().bmb200_ctx_get_stream(self._h, C.byref(s)), "ctx_get_stream")
        return int(s.value or 0)

    def set_tuning(self, key: int, value: int):
        self.check(lib().bmb200_ctx_set_tuning(self._h, int(key), int(value)), "ctx_set_tuning")

    def launch_count(self) -> int:
        n = C.c_uint64(0)
        self.check(lib().bmb200_ctx_launch_count(self._h, C.byref(n)), "launch_count")
        return int(n.value)

    def trim(self):
        """Give the parked device arena (bmb200_set_free keeps the last freed set's arrays for the next upload) back to the driver."""
        self.check(lib().bmb200_ctx_trim(self._h), "ctx_trim")

    def bind_host_numa(self) -> int:
        """Pin the calling thread to the CPUs of this GPU's NUMA node (bmb200_ctx_bind_host_numa); -> node or -1."""
        node = C.c_int(-1)
        self.check(lib().bmb200_ctx_bind_host_numa(self._h, C.byref(node)), "ctx_bind_host_numa")
        return node.value

    # ---- multi-GPU exchange (one process per GPU): see include/bmb200.h "multi-GPU" ----
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = C.create_string_buffer(COMM_ID_BYTES)
        rc = lib().bmb200_comm_unique_id(buf)
        if rc != OK:
            raise BMB200Error(rc, "comm_unique_id")
        return buf.raw

    def comm_init(self, nranks: int, rank: int, comm_id: bytes):
        assert len(comm_id) == COMM_ID_BYTES
        self.check(lib().bmb200_comm_init(self._h, int(nranks), int(rank), C.c_char_p(comm_id)), "comm_init")

    def comm_destroy(self):
        self.check(lib().bmb200_comm_destroy(self._h), "comm_destroy")

    def exchange_popcounts(self, res: "DeviceResult", cols_per_rank: int = 0):
        self.check(lib().bmb200_exchange_popcounts(res._h, int(cols_per_rank)), "exchange_popcounts")

    def exchange_mode(self) -> int:
        """0 = no exchange yet, 1 = ncclAllGather on the side stream, 2 = peer-memory pushes (CUDA IPC over NVLink)"""
        m = C.c_int(0)
        self.check(lib().bmb200_exchange_mode(self._h, C.byref(m)), "exchange_mode")
        return m.value

    def exchange_fence(self):
        self.check(lib().bmb200_exchange_fence(self._h), "exchange_fence")

    def exchange_fetch(self, nranks: int, cols_per_rank: int, want_popcounts: bool = True):
        """-> (global cardinality, per-rank cardinalities [nranks], per-column popcounts [nranks, cols_per_rank] or None)"""
        tot = C.c_uint64(0); rt = np.zeros(nranks, np.uint64)
        pop = np.zeros((nranks, cols_per_rank), np.uint32) if want_popcounts else None
        self.check(lib().bmb200_exchange_fetch(self._h, C.byref(tot), ptr(rt), ptr(pop), None, None), "exchange_fetch")
        return tot.value, rt, pop

    def device_info(self) -> dict:
        sm, ma, mi, hbm = C.c_int(0), C.c_int(0), C.c_int(0), C.c_uint64(0)
        self.check(lib().bmb200_device_info(self._h, C.byref(sm), C.byref(ma), C.byref(mi), C.byref(hbm)), "device_info")
        return {"sm_count": sm.value, "cc": (ma.value, mi.value), "hbm_bytes": hbm.value}


_default_ctx: dict[int, Context] = {}


def default_context(device: int | None = None) -> Context:
    if device is None:
        device = int(os.environ.get("LOCAL_RANK", "0"))
    if device not in _default_ctx:
        _default_ctx[device] = Context(device)
    return _default_ctx[device]


class DeviceSet:
    """Device-resident packed column-major set (bmb200_set)."""

    def __init__(self, ctx: Context, handle: C.c_void_p):
        self.ctx, self._h = ctx, handle
        nv, nb, nbit, ngap = C.c_uint32(0), C.c_uint32(0), C.c_uint64(0), C.c_uint64(0)
        ctx.check(lib().bmb200_set_info(handle, C.byref(nv), C.byref(nb), C.byref(nbit), C.byref(ngap)), "set_info")
        self.n_vec, self.n_blocks = nv.value, nb.value
        self.n_bit_blocks, self.n_gap_units = nbit.value, ngap.value

    @classmethod
    def upload(cls, ctx: Context, ps) -> "DeviceSet":
        h = C.c_void_p(0)
        c = packed_c(ps.n_vec, ps.n_blocks, ps.desc, ps.bit_base, ps.gap_base, ps.bit_pool, ps.gap_pool)
        ctx.check(lib().bmb200_set_upload(ctx._h, C.byref(c), C.byref(h)), "set_upload")
        ctx.sync()   # the host arrays may be released by the caller right after
        return cls(ctx, h)

    @classmethod
    def upload_vectors(cls, ctx: Context, vectors, n_blocks: int | None = None) -> "DeviceSet":
        """Gather per-vector block trees (hostfmt.BVector) through bmb200_set_upload_vectors."""
        if n_blocks is None:
            n_blocks = max(v.n_blocks for v in vectors)
        arr = (VecBlocksC * len(vectors))()
        keep = []
        for i, v in enumerate(vectors):
            kind = np.ascontiguousarray(v.kind, dtype=np.uint8)
            ptrs = np.zeros(v.n_blocks, dtype=np.uint64)
            for nb in range(v.n_blocks):
                if kind[nb] == BLK_BIT or kind[nb] == BLK_GAP:
                    blk = v.blocks[nb]
                    keep.append(blk)
                    ptrs[nb] = blk.ctypes.data
            keep += [kind, ptrs]
            arr[i] = VecBlocksC(v.n_blocks, ptr(kind), ptr(ptrs))
        h = C.c_void_p(0)
        ctx.check(lib().bmb200_set_upload_vectors(ctx._h, len(vectors), int(n_blocks), arr, C.byref(h)), "set_upload_vectors")
        return cls(ctx, h)

    @classmethod
    def upload_slabs(cls, ctx: Context, vectors, n_blocks: int | None = None, slab_bytes: int = 1 << 20, pinned: bool = True,
                     prefetch: bool = False, stray: bool = False) -> "DeviceSet":
        """bmb200_set_upload_slabs: the blocks of `vectors` (hostfmt.BVector) are first laid into a few host slabs the way a
        slab-backed block allocator would hold them (64-byte aligned, in allocation order = vector by vector), then uploaded by
        DMA of the slabs + the device gather.  pinned: slabs from bmb200_host_slab_alloc (else numpy memory); prefetch: queue the
        DMA with bmb200_host_slabs_prefetch first; stray: leave one block outside every slab (the call must fall back)."""
        if n_blocks is None:
            n_blocks = max(v.n_blocks for v in vectors)
        slabs, views, keep = [], [], []
        cur = {"buf": None, "used": 0}

        def new_slab(need):
            size = max(slab_bytes, need)
            if pinned:
                p = C.c_void_p(0)
                ctx.check(lib().bmb200_host_slab_alloc(C.c_uint64(size), C.byref(p)), "host_slab_alloc")
                buf = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(size,))
                slabs.append([p.value, buf, 0, True])
            else:
                raw = np.zeros(size + 64, dtype=np.uint8)
                off = (-raw.ctypes.data) % 64
                buf = raw[off:off + size]
                keep.append(raw)
                slabs.append([buf.ctypes.data, buf, 0, False])
            cur["buf"], cur["used"] = slabs[-1], 0

        def place(blk):
            b = np.ascontiguousarray(blk).view(np.uint8)
            need = (b.size + 63) & ~63
            if cur["buf"] is None or cur["buf"][1].size - cur["buf"][2] < need:
                new_slab(need)
            sl = cur["buf"]
            sl[1][sl[2]:sl[2] + b.size] = b
            addr = sl[0] + sl[2]
            sl[2] += need
            return addr

        arr = (VecBlocksC * len(vectors))()
        strayed = not stray
        for i, v in enumerate(vectors):
            kind = np.ascontiguousarray(v.kind, dtype=np.uint8)
            ptrs = np.zeros(v.n_blocks, dtype=np.uint64)
            for nb in range(v.n_blocks):
                if kind[nb] == BLK_BIT or kind[nb] == BLK_GAP:
                    if not strayed:
                        blk = np.ascontiguousarray(v.blocks[nb]); keep.append(blk); ptrs[nb] = blk.ctypes.data; strayed = True
                    else:
                        ptrs[nb] = place(v.blocks[nb])
            keep += [kind, ptrs]
            arr[i] = VecBlocksC(v.n_blocks, ptr(kind), ptr(ptrs))
        carr = (HostSlabC * max(1, len(slabs)))()
        for k, sl in enumerate(slabs):
            carr[k].base = sl[0]; carr[k].bytes = sl[2]
        try:
            if prefetch:
                ctx.check(lib().bmb200_host_slabs_prefetch(ctx._h, carr, len(slabs)), "host_slabs_prefetch")
            h = C.c_void_p(0)
            ctx.check(lib().bmb200_set_upload_slabs(ctx._h, len(vectors), int(n_blocks), arr, carr, len(slabs), C.byref(h)), "set_upload_slabs")
        finally:
            ctx.sync()
            for sl in slabs:
                if sl[3]:
                    lib().bmb200_host_slab_free(C.c_void_p(sl[0]))
        return cls(ctx, h)

    @classmethod
    def upload_blobs(cls, ctx: Context, blobs, n_blocks: int) -> "DeviceSet":
        """bmb200_set_upload_blobs: every vector arrives as a BitMagic serialization BLOB (bytes / uint8 array) and is decoded
        on the GPU (deserialize-to-device); raises BMB200Error(ERR_UNSUPPORTED) for encodings the device decoder does not cover."""
        arrs = [np.ascontiguousarray(np.frombuffer(b, dtype=np.uint8) if isinstance(b, (bytes, bytearray)) else b, dtype=np.uint8) for b in blobs]
        carr = (BlobC * len(arrs))()
        for i, a in enumerate(arrs):
            carr[i].data = a.ctypes.data; carr[i].size = a.size
        h = C.c_void_p(0)
        ctx.check(lib().bmb200_set_upload_blobs(ctx._h, len(arrs), int(n_blocks), carr, C.byref(h)), "set_upload_blobs")
        return cls(ctx, h)

    @classmethod
    def synth(cls, ctx: Context, n_vec: int, n_blocks: int, density, seed, optimize: bool) -> "DeviceSet":
        d = np.ascontiguousarray(density, dtype=np.float64)
        s = np.ascontiguousarray(seed, dtype=np.uint64)
        assert d.size == n_vec and s.size == n_vec
        h = C.c_void_p(0)
        ctx.check(lib().bmb200_synth_set(ctx._h, int(n_vec), int(n_blocks), ptr(d), ptr(s), int(bool(optimize)), C.byref(h)), "synth_set")
        return cls(ctx, h)

    def column_sizes(self, nb_from: int, nb_to: int) -> tuple[int, int]:
        a, b = C.c_uint64(0), C.c_uint64(0)
        self.ctx.check(lib().bmb200_set_column_sizes(self._h, int(nb_from), int(nb_to), C.byref(a), C.byref(b)), "set_column_sizes")
        return a.value, b.value

    def download(self, nb_from: int = 0, nb_to: int | None = None):
        """Columns [nb_from, nb_to) as a host PackedSet."""
        from .hostfmt import PackedSet
        nb_to = self.n_blocks if nb_to is None else nb_to
        nbit, ngap = self.column_sizes(nb_from, nb_to)
        nc = nb_to - nb_from
        desc = np.empty(nc * self.n_vec, dtype=np.uint32)
        bb = np.empty(nc + 1, dtype=np.uint64)
        gb = np.empty(nc + 1, dtype=np.uint64)
        bp = np.empty(nbit * BLOCK_WORDS, dtype=np.uint32)
        gp = np.empty(ngap * GAP_UNIT_WORDS, dtype=np.uint16)
        self.ctx.check(lib().bmb200_set_download(self._h, int(nb_from), int(nb_to), ptr(desc), ptr(bb), ptr(gb),
                                                 ptr(bp) if nbit else C.c_void_p(0), ptr(gp) if ngap else C.c_void_p(0)),
                       "set_download")
        return PackedSet(self.n_vec, nc, desc, bb, gb, bp, gp)

    def device_ptrs(self) -> PackedSetC:
        c = PackedSetC()
        self.ctx.check(lib().bmb200_set_device_ptrs(self._h, C.byref(c)), "set_device_ptrs")
        return c

    def run_list_bytes(self) -> tuple[int, int]:
        """(singles, long runs) bytes of the set's run-list companion; (0, 0) while none is built (TUNE_RUN_LISTS)."""
        a, b = C.c_uint64(0), C.c_uint64(0)
        self.ctx.check(lib().bmb200_set_run_lists(self._h, C.byref(a), C.byref(b)), "set_run_lists")
        return a.value, b.value

    def bit_run_list_bytes(self) -> tuple[int, int, int]:
        """(singles, long runs) bytes of the companion's part B, the listed sparse bit-blocks, and how many blocks it lists;
        (0, 0, 0) while none is built."""
        a, b, n = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self.ctx.check(lib().bmb200_set_bit_run_lists(self._h, C.byref(a), C.byref(b), C.byref(n)), "set_bit_run_lists")
        return a.value, b.value, n.value

    def stored_bytes(self) -> int:
        """Algorithmic source bytes: 8192 per bit-block + the 16-byte units of the GAP blocks."""
        return self.n_bit_blocks * BLOCK_BYTES + self.n_gap_units * GAP_UNIT_WORDS * 2

    def free(self):
        if self._h:
            lib().bmb200_set_free(self._h)
            self._h = C.c_void_p(0)

    def __del__(self):  # pragma: no cover
        try:
            self.free()
        except Exception:
            pass


class DeviceResult:
    """Device-resident aggregation result (bmb200_result)."""

    def __init__(self, ctx: Context):
        self.ctx = ctx
        self._h = C.c_void_p(0)
        self.n_cols = 0

    def total(self) -> tuple[int, bool]:
        t, a = C.c_uint64(0), C.c_int(0)
        self.ctx.check(lib().bmb200_result_total(self._h, C.byref(t), C.byref(a)), "result_total")
        return t.value, bool(a.value)

    def meta(self):
        n = self.n_cols
        kind = np.empty(n, np.uint8); pop = np.empty(n, np.uint32)
        dig = np.empty(n, np.uint64); nr = np.empty(n, np.uint32)
        m = ResultMetaC(ptr(kind), ptr(pop), ptr(dig), ptr(nr))
        self.ctx.check(lib().bmb200_result_fetch_meta(self._h, C.byref(m)), "result_fetch_meta")
        return kind, pop, dig, nr

    def fetch(self):
        """(kind[n], off[n], bits[n_bit*2048], gaps[n_gap_words]) -- per-vector flat form."""
        nb, ng = C.c_uint64(0), C.c_uint64(0)
        self.ctx.check(lib().bmb200_result_sizes(self._h, C.byref(nb), C.byref(ng)), "result_sizes")
        kind = np.empty(self.n_cols, np.uint8); off = np.empty(self.n_cols, np.uint64)
        bits = np.empty(nb.value * BLOCK_WORDS, np.uint32); gaps = np.empty(ng.value, np.uint16)
        self.ctx.check(lib().bmb200_result_fetch(self._h, ptr(kind), ptr(off),
                                                 ptr(bits) if nb.value else C.c_void_p(0),
                                                 ptr(gaps) if ng.value else C.c_void_p(0)), "result_fetch")
        return kind, off, bits, gaps

    def fetch_column(self, col: int):
        """bmb200_result_fetch_column -> (kind, bits[2048] | None, gap words | None) of ONE result column."""
        kind = C.c_uint8(0)
        bits = np.empty(BLOCK_WORDS, np.uint32); gaps = np.empty(1280, np.uint16)
        self.ctx.check(lib().bmb200_result_fetch_column(self._h, int(col), C.byref(kind), ptr(bits), ptr(gaps)), "result_fetch_column")
        k = kind.value
        return k, (bits if k == BLK_BIT else None), (gaps[:(int(gaps[0]) >> 3) + 1] if k == BLK_GAP else None)

    def group_totals(self, n_groups: int) -> np.ndarray:
        t = np.zeros(n_groups, np.uint64)
        self.ctx.check(lib().bmb200_result_group_totals(self._h, ptr(t), int(n_groups)), "result_group_totals")
        return t

    def or_target(self, n_cols: int) -> "DeviceResult":
        o = DeviceResult(self.ctx)
        self.ctx.check(lib().bmb200_result_or_target(self._h, C.byref(o._h)), "result_or_target")
        o.n_cols = n_cols
        return o

    def device_ptrs(self) -> dict:
        b, p, d, f, n = C.c_void_p(0), C.c_void_p(0), C.c_void_p(0), C.c_void_p(0), C.c_uint32(0)
        self.ctx.check(lib().bmb200_result_device_ptrs(self._h, C.byref(b), C.byref(p), C.byref(d), C.byref(f), C.byref(n)), "result_device_ptrs")
        return {"blocks": b.value or 0, "popcnt": p.value or 0, "digest": d.value or 0, "kind": f.value or 0, "n_cols": n.value}

    def free(self):
        if self._h:
            lib().bmb200_result_free(self._h)
            self._h = C.c_void_p(0)

    def __del__(self):  # pragma: no cover
        try:
            self.free()
        except Exception:
            pass


def aggregate(ctx: Context, dset: DeviceSet, op: int, group0, group1=None, flags: int = 0,
              nb_from: int = 0, nb_to: int = 0, result: DeviceResult | None = None) -> DeviceResult:
    """bmb200_aggregate: asynchronous launch; the result stays in HBM."""
    g0 = np.ascontiguousarray(group0, dtype=np.uint32)
    g1 = np.ascontiguousarray(group1 if group1 is not None else [], dtype=np.uint32)
    args = AggArgsC(int(op), int(flags), ptr(g0) if g0.size else C.c_void_p(0), g0.size,
                    ptr(g1) if g1.size else C.c_void_p(0), g1.size, int(nb_from), int(nb_to))
    res = result if result is not None else DeviceResult(ctx)
    ctx.check(lib().bmb200_aggregate(ctx._h, dset._h, C.byref(args), C.byref(res._h)), "aggregate")
    res.n_cols = (nb_to if nb_to else dset.n_blocks) - nb_from
    return res


def binop(ctx: Context, dset: DeviceSet, op: int, va: int, vb: int, flags: int = 0, nb_from: int = 0, nb_to: int = 0,
          result: DeviceResult | None = None) -> DeviceResult:
    """bmb200_binop: two-operand bvector op (OP_OR / OP_AND / OP_XOR / OP_SUB) with the reference's per-block result kinds
    (GAP x GAP merged as run lists on the device)."""
    res = result if result is not None else DeviceResult(ctx)
    ctx.check(lib().bmb200_binop(ctx._h, dset._h, int(op), int(va), int(vb), int(flags), int(nb_from), int(nb_to), C.byref(res._h)), "binop")
    res.n_cols = (nb_to if nb_to else dset.n_blocks) - nb_from
    return res


def aggregate_batch(ctx: Context, dset: DeviceSet, op: int, groups, flags: int = 0, nb_from: int = 0, nb_to: int = 0,
                    result: DeviceResult | None = None) -> DeviceResult:
    """bmb200_aggregate_batch: `groups` = [(group0, group1), ...]; the result has len(groups) * n_cols columns, group-major."""
    mem, off = [], [0]
    for g0, g1 in groups:
        mem.extend(int(x) for x in g0); off.append(len(mem))
        mem.extend(int(x) for x in (g1 if g1 is not None else [])); off.append(len(mem))
    members = np.ascontiguousarray(mem, dtype=np.uint32); offsets = np.ascontiguousarray(off, dtype=np.uint32)
    args = BatchArgsC(int(op), int(flags), len(groups), ptr(members) if members.size else C.c_void_p(0), ptr(offsets), int(nb_from), int(nb_to))
    res = result if result is not None else DeviceResult(ctx)
    ctx.check(lib().bmb200_aggregate_batch(ctx._h, dset._h, C.byref(args), C.byref(res._h)), "aggregate_batch")
    res.n_cols = ((nb_to if nb_to else dset.n_blocks) - nb_from) * len(groups)
    return res


def scan(ctx: Context, dset: DeviceSet, pred: int, values, plane0: int, n_planes: int, universe: int = NO_UNIVERSE,
         flags: int = 0, nb_from: int = 0, nb_to: int = 0, result: DeviceResult | None = None) -> DeviceResult:
    """bmb200_scan: bit-sliced comparison of the sparse vector whose plane j is set vector plane0 + j against every search
    value (SCAN_RANGE: rows of (lo, hi)); the result has n_values * n_cols columns, value-major."""
    vals = np.ascontiguousarray(values, dtype=np.uint64)
    nv = vals.shape[0] if pred == SCAN_RANGE else vals.size
    if pred == SCAN_RANGE and (vals.ndim != 2 or vals.shape[1] != 2):
        raise ValueError("SCAN_RANGE takes an array of (lo, hi) rows")
    args = ScanArgsC(int(plane0), int(n_planes), int(universe), int(pred), int(flags), ptr(vals), int(nv), int(nb_from), int(nb_to))
    res = result if result is not None else DeviceResult(ctx)
    ctx.check(lib().bmb200_scan(ctx._h, dset._h, C.byref(args), C.byref(res._h)), "scan")
    res.n_cols = ((nb_to if nb_to else dset.n_blocks) - nb_from) * int(nv)
    return res


def _sized(res: DeviceResult) -> DeviceResult:
    res.n_cols = res.device_ptrs()["n_cols"]
    return res


def rank_decompress(ctx: Context, rs: "DeviceRS", res: DeviceResult, flags: int = 0, result: DeviceResult | None = None) -> DeviceResult:
    """bmb200_rank_decompress (rank_compressor::decompress): every group of `res`, read as bits of the compressed index space
    of the NOT-NULL vector `rs` was built on, mapped to its logical positions.  The result has n_groups * rs.dset.n_blocks
    columns, group-major."""
    out = result if result is not None else DeviceResult(ctx)
    ctx.check(lib().bmb200_rank_decompress(ctx._h, rs._h, res._h, int(flags), C.byref(out._h)), "rank_decompress")
    return _sized(out)


def rank_compress(ctx: Context, rs: "DeviceRS", src_vec: int, flags: int = 0, result: DeviceResult | None = None) -> DeviceResult:
    """bmb200_rank_compress (rank_compressor::compress): vector src_vec of the set `rs` was built on, restricted to the
    NOT-NULL vector and packed to its ranks; one group of max(1, ceil(count / 65536)) columns."""
    out = result if result is not None else DeviceResult(ctx)
    ctx.check(lib().bmb200_rank_compress(ctx._h, rs._h, int(src_vec), int(flags), C.byref(out._h)), "rank_compress")
    return _sized(out)


def aggregate_host(ctx: Context, ps, op: int, group0, group1=None, flags: int = 0):
    """bmb200_aggregate_host: host packed set in, host metadata out (H2D + kernel + D2H in one call)."""
    g0 = np.ascontiguousarray(group0, dtype=np.uint32)
    g1 = np.ascontiguousarray(group1 if group1 is not None else [], dtype=np.uint32)
    args = AggArgsC(int(op), int(flags), ptr(g0) if g0.size else C.c_void_p(0), g0.size,
                    ptr(g1) if g1.size else C.c_void_p(0), g1.size, 0, 0)
    n = ps.n_blocks
    kind = np.empty(n, np.uint8); pop = np.empty(n, np.uint32); dig = np.empty(n, np.uint64); nr = np.empty(n, np.uint32)
    m = ResultMetaC(ptr(kind), ptr(pop), ptr(dig), ptr(nr))
    tot = C.c_uint64(0)
    c = packed_c(ps.n_vec, ps.n_blocks, ps.desc, ps.bit_base, ps.gap_base, ps.bit_pool, ps.gap_pool)
    ctx.check(lib().bmb200_aggregate_host(ctx._h, C.byref(c), C.byref(args), C.byref(m), C.byref(tot)), "aggregate_host")
    return kind, pop, dig, nr, tot.value


class DeviceRS:
    """Device-resident rank-select index (bmb200_rs) over one vector of a DeviceSet."""

    def __init__(self, ctx: Context, dset: DeviceSet, vec: int):
        self.ctx, self.dset, self.vec = ctx, dset, vec
        self._h = C.c_void_p(0)
        ctx.check(lib().bmb200_rs_build(ctx._h, dset._h, int(vec), C.byref(self._h)), "rs_build")

    def rebuild(self):
        self.ctx.check(lib().bmb200_rs_rebuild(self._h), "rs_rebuild")

    def export(self):
        nb = self.dset.n_blocks
        nsb = (nb + 255) // 256
        bc = np.empty(nb, np.uint32); sc = np.empty(nb, np.uint64); sb = np.empty(nsb + 1, np.uint64)
        self.ctx.check(lib().bmb200_rs_export(self._h, ptr(bc), ptr(sc), ptr(sb)), "rs_export")
        return bc, sc, sb

    def total(self) -> int:
        t = C.c_uint64(0)
        self.ctx.check(lib().bmb200_rs_total(self._h, C.byref(t)), "rs_total")
        return t.value

    def rank(self, pos) -> np.ndarray:
        p = np.ascontiguousarray(pos, dtype=np.uint64)
        out = np.empty(p.size, np.uint64)
        self.ctx.check(lib().bmb200_rank_batch(self._h, ptr(p), C.c_uint64(p.size), ptr(out)), "rank_batch")
        return out

    def select(self, rank) -> tuple[np.ndarray, np.ndarray]:
        r = np.ascontiguousarray(rank, dtype=np.uint64)
        pos = np.empty(r.size, np.uint64); found = np.empty(r.size, np.uint8)
        self.ctx.check(lib().bmb200_select_batch(self._h, ptr(r), C.c_uint64(r.size), ptr(pos), ptr(found)), "select_batch")
        return pos, found.astype(bool)

    def rank_dev(self, d_pos: int, n: int, d_out: int):
        self.ctx.check(lib().bmb200_rank_batch_dev(self._h, C.c_void_p(d_pos), C.c_uint64(n), C.c_void_p(d_out)), "rank_batch_dev")

    def select_dev(self, d_rank: int, n: int, d_pos: int, d_found: int):
        self.ctx.check(lib().bmb200_select_batch_dev(self._h, C.c_void_p(d_rank), C.c_uint64(n), C.c_void_p(d_pos), C.c_void_p(d_found)), "select_batch_dev")

    def free(self):
        if self._h:
            lib().bmb200_rs_free(self._h)
            self._h = C.c_void_p(0)

    def __del__(self):  # pragma: no cover
        try:
            self.free()
        except Exception:
            pass
