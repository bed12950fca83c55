#!/usr/bin/env python
"""Set image through a sparse vector (bmb200_remap, set2set_11_transform::remap) on nullable sparse_vector<unsigned> of 250 M
elements (3 815 block columns of bit-blocks), a 5-element NULL plate after every 64th element (svsample06's pattern).
  python scripts/bench_remap.py [n_elements]   -> one JSON line
Workloads:
  (a) uniform 24-bit values, sources at 1 % and 100 % density: one-block-per-word scatter into a 2 MiB image;
  (b) Zipf(1) values over 1 000 categories, source at 100 %: many ids onto few image words, the contention case;
  (c) uniform 32-bit values, source at 10 %: a 512 MiB image of 65 536 columns, so its zeroing and classification show.
The source is a device result (a one-source OR of the uploaded id set), as a scan or aggregation result would be.  Per
workload: the call time from CUDA events over warmed calls, the remap-kernel and finalize-kernel times from torch.profiler's
CUDA activity, and the stored bytes the kernel must read (plane, NOT-NULL and source blocks of the columns with ids) over the
remap-kernel time.  The reference's remap on one host core comes from oracle/_ref/libbmref_remap.so (oracle/remap.mk), with
its count checked against the device's, and the contract's count (numpy) is checked too: the reference's image departs from
the contract on some inputs (DESIGN.md 3.5g)."""
import ctypes as C
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))
import torch                 # noqa: E402
import bitmagic_b200 as bm   # noqa: E402
from bitmagic_b200.capi import BLOCK_BITS, BLOCK_WORDS, BLK_BIT  # noqa: E402
from bench_scan_in import card, timed  # noqa: E402
from bench_sv_mismatch import kernel_ms, stored_bytes  # noqa: E402

REF = ROOT / "oracle" / "_ref" / "libbmref_remap.so"
HBM_TBPS = 3.35             # H100 SXM data sheet


def vec(bits, nb):
    w = np.zeros(nb * BLOCK_WORDS, np.uint32)
    p = np.packbits(bits, bitorder="little")
    w.view(np.uint8)[:p.size] = p
    return bm.BVector.from_words(w)


def planes_of(vals, nulls, n_planes, nb):
    return [vec(((vals >> np.uint32(j)) & np.uint32(1)).astype(np.uint8), nb) for j in range(n_planes)] + [vec(1 - nulls, nb)]


def ref_time(vals, nulls, ids):
    v = np.ascontiguousarray(vals, np.uint32); i = np.ascontiguousarray(ids, np.uint32); nl = np.ascontiguousarray(nulls, np.uint8)
    p = bm.capi.ptr
    cnt, sec = C.c_uint64(0), C.c_double(0)
    rc = C.CDLL(str(REF)).ref_remap_time(p(v), p(nl), C.c_uint64(v.size), p(i), C.c_uint64(i.size), 1, C.byref(cnt), C.byref(sec))
    assert rc == 0, f"ref_remap_time rc={rc}"
    return sec.value, cnt.value


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    n = int(args[0]) if args else 250_000_000
    if not torch.cuda.is_available():
        raise SystemExit("bench_remap: no CUDA device")
    t0 = time.time()
    rng = np.random.default_rng(5)
    nb = (n + BLOCK_BITS - 1) // BLOCK_BITS
    nulls = ((np.arange(n, dtype=np.uint64) % 64) - 1 < 5).astype(np.uint8)
    ranks = np.arange(1, 1001, dtype=np.float64)
    vectors = {
        "uniform24": (rng.integers(0, 1 << 24, n, dtype=np.uint32), 24),
        "zipf1000": (rng.choice(1000, n, p=(1 / ranks) / (1 / ranks).sum()).astype(np.uint32), 10),
        "uniform32": (rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32), 32),
    }
    workloads = [("a_uniform24_src1pct", "uniform24", 0.01), ("a_uniform24_src100pct", "uniform24", 1.0),
                 ("b_zipf1000_src100pct", "zipf1000", 1.0), ("c_uniform32_src10pct", "uniform32", 0.10)]
    ctx = bm.Context(0)
    ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    out = {"bench": "remap", "elements": n, "block_columns": nb, **card(), "hbm_datasheet_TBps": HBM_TBPS, "results": {}}
    for name, vname, density in workloads:
        vals, npl = vectors[vname]
        vals = np.where(nulls == 1, np.uint32(0), vals)
        vecs = planes_of(vals, nulls, npl, nb)
        ids_bits = np.ones(n, np.uint8) if density >= 1.0 else (rng.random(n) < density).astype(np.uint8)
        if density >= 1.0:                                   # every id: FULL source blocks
            srcv = bm.BVector(nb)
            for c in range(nb):
                srcv.set_full(c)
        else:
            srcv = vec(ids_bits, nb)
        dset = bm.DeviceSet.upload(ctx, bm.PackedSet.pack(vecs))
        sset = bm.DeviceSet.upload(ctx, bm.PackedSet.pack([srcv]))
        src = bm.aggregate(ctx, sset, bm.OP_OR, [0], None, bm.F_OPT_COMPRESS)
        call = lambda r=None: bm.remap(ctx, dset, src, 0, npl, npl, 0xFFFFFFFF, bm.F_OPT_COMPRESS, r)   # noqa: E731
        res = call()
        ms = timed(lambda: call(res), 10)
        total = res.total()[0]
        k_remap = kernel_ms(lambda: call(res), "remap_kernel")
        k_fin = kernel_ms(lambda: call(res), "finalize_blocks_kernel")
        res.free()
        nbytes = stored_bytes(vecs) + 8192 * int((srcv.kind == BLK_BIT).sum())     # every column holds ids here
        gbps = nbytes / (k_remap * 1e-3) / 1e9 if k_remap else None
        r = {"planes": npl, "source_density": density, "image_columns": max(1, 1 << max(npl - 16, 0)), "count": int(total),
             "call_ms": ms, "remap_kernel_ms": k_remap if k_remap else "not measured",
             "finalize_kernel_ms": k_fin if k_fin else "not measured", "stored_MiB_read": nbytes / 2**20,
             "GBps": gbps if gbps else "not measured", "of_datasheet": gbps / (HBM_TBPS * 1e3) if gbps else "not measured"}
        sel = vals[(ids_bits == 1) & (nulls == 0)]
        want = np.unique(sel[sel != np.uint32(0xFFFFFFFF)]).size         # the contract's count, without bm::id_max
        r["numpy_count"] = int(want)
        r["numpy_counts_equal"] = int(want) == int(total)
        if REF.exists():
            sec, rcnt = ref_time(vals, nulls, np.flatnonzero(ids_bits))
            r["reference_1core"] = {"remap_s": sec, "count": rcnt, "counts_equal": rcnt == total, "speedup": sec / (ms * 1e-3)}
        else:
            r["reference_1core"] = "not measured (reference library not built)"
        out["results"][name] = r
        src.free(); sset.free(); dset.free()
        print(json.dumps({name: r}), file=sys.stderr, flush=True)
    out["wall_s"] = round(time.time() - t0, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
