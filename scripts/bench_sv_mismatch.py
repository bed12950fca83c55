#!/usr/bin/env python
"""Sparse-vector mismatch (bmb200_sv_mismatch / bmb200_sv_first_mismatch) on the workload of scripts/bench_scan_in.py: two
nullable sparse_vector<unsigned> of 250 M elements, values uniform in [1, 1 250 000] (21 planes, 3 815 block columns of
bit-blocks), a 5-element NULL plate after every 64th element.
  python scripts/bench_sv_mismatch.py [n_elements]   -> one JSON line
Versions of the second vector: identical (a separately stored copy, so every block is read), 0.1 % of the elements changed,
and one change at the last element (the first form's worst case: no column can be skipped).  Per version and entry point
(use_null): the call time from CUDA events over warmed calls, the kernel time per launch from torch.profiler's CUDA activity,
and the stored bytes of both vectors (planes + NOT-NULL) over the kernel time, against the data sheet's 3.35 TB/s and against
the read ceiling that scripts/microbench_read.cu measures in the same run.  The reference's sparse_vector_find_mismatch and
sparse_vector_find_first_mismatch on one host core come from oracle/_ref/libbmref_mismatch.so (oracle/mismatch.mk)."""
import ctypes as C
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))
import torch                 # noqa: E402
import bitmagic_b200 as bm   # noqa: E402
from bitmagic_b200.capi import BLK_BIT, BLK_GAP  # noqa: E402
from bench_scan_in import card, plane_vectors, svsample06, timed  # noqa: E402

REF_MM = ROOT / "oracle" / "_ref" / "libbmref_mismatch.so"
HBM_TBPS = 3.35             # H100 SXM data sheet


def stored_bytes(vecs):
    """bytes a launch must read once: 8 KB per bit-block, 2 bytes per GAP word"""
    total = 0
    for v in vecs:
        total += 8192 * int((v.kind == BLK_BIT).sum())
        total += sum(2 * v.blocks[c].size for c in np.flatnonzero(v.kind == BLK_GAP))
    return total


def kernel_ms(fn, name, reps=5):
    """device time per launch of the kernels whose name holds `name`, from torch.profiler's CUDA activity: the total over the
    launches the profiler recorded, divided by their number (it may drop some), or None when no launch was recorded"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if name in e.key]
    n = sum(e.count for e in ev)
    us = sum(getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0) for e in ev)
    return us / 1e3 / n if n else None


def read_ceiling():
    """GB/s of scripts/microbench_read.cu, compiled into a temporary directory (None when nvcc or the run fails)"""
    with tempfile.TemporaryDirectory() as tmp:
        exe = Path(tmp) / "microbench_read"
        try:
            subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-o", str(exe),
                            str(ROOT / "scripts" / "microbench_read.cu")], check=True, capture_output=True, timeout=600)
            p = subprocess.run([str(exe)], check=True, capture_output=True, text=True, timeout=600)
            return json.loads(p.stdout.strip().splitlines()[-1])["read_ceiling_GBps"]
        except (OSError, subprocess.SubprocessError, ValueError, KeyError):
            return None


def ref_time(v1, n1, v2, n2):
    """the reference's two functions on one core (use_null) -> (find s, count, first s, found, midx)"""
    a, b = np.ascontiguousarray(v1, np.int64), np.ascontiguousarray(v2, np.int64)
    p = bm.capi.ptr
    sf, cnt, s1, found, midx = C.c_double(0), C.c_uint64(0), C.c_double(0), C.c_int(0), C.c_uint64(0)
    rc = C.CDLL(str(REF_MM)).ref_mm_time(0, p(a), p(n1), C.c_uint64(a.size), p(b), p(n2), C.c_uint64(b.size), 1, 1,
                                         C.byref(sf), C.byref(cnt), C.byref(s1), C.byref(found), C.byref(midx))
    assert rc == 0, f"ref_mm_time rc={rc}"
    return sf.value, cnt.value, s1.value, bool(found.value), midx.value


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    n = int(args[0]) if args else 250_000_000
    if not torch.cuda.is_available():
        raise SystemExit("bench_sv_mismatch: no CUDA device")
    t0 = time.time()
    rng = np.random.default_rng(6)
    vals, nulls = svsample06(n, rng)
    changed = vals.copy()
    idx = rng.choice(n, n // 1000, replace=False)
    changed[idx] = np.where(nulls[idx] == 1, 0, (changed[idx] % 1_250_000) + 1)
    last = vals.copy()
    last[-1] = 1 if last[-1] != 1 else 2
    nulls[-1] = 0
    versions = {"identical": vals, "changed_0.1pct": changed, "last_element": last}
    base = plane_vectors(vals, nulls)
    vecs = list(base)
    offs = {}
    for name, v in versions.items():
        offs[name] = len(vecs)
        vecs += list(base) if name == "identical" else plane_vectors(v, nulls)     # packed again: a copy of its own
        assert len(vecs) - offs[name] == len(base), "every version has the planes of the first vector"
    npl = len(base) - 1
    ps = bm.PackedSet.pack(vecs)
    ctx = bm.Context(0)
    ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    dset = bm.DeviceSet.upload(ctx, ps)
    ceiling = read_ceiling()
    out = {"bench": "sv_mismatch", "workload": "svsample06 pairs", "elements": n, "planes": npl, "block_columns": ps.n_blocks,
           **card(), "hbm_datasheet_TBps": HBM_TBPS, "read_ceiling_GBps": ceiling if ceiling else "not measured", "results": {}}
    for name, v in versions.items():
        o = offs[name]
        nbytes = stored_bytes(base) + stored_bytes(vecs[o:o + npl + 1])
        a = bm.capi.mismatch_args(0, npl, o, npl, npl, o + npl, n, n, bm.MM_USE_NULL, bm.F_COUNT_ONLY)
        a_st = bm.capi.mismatch_args(0, npl, o, npl, npl, o + npl, n, n, bm.MM_USE_NULL, bm.F_OPT_COMPRESS)
        r = {"stored_MiB_read": nbytes / 2**20}
        res = bm.sv_mismatch(ctx, dset, a)
        ms = timed(lambda: bm.sv_mismatch(ctx, dset, a, result=res), 10)
        cnt = int(res.group_totals(1)[0])
        kms = kernel_ms(lambda: bm.sv_mismatch(ctx, dset, a, result=res), "mismatch_kernel<false>")
        res.free()
        res = bm.sv_mismatch(ctx, dset, a_st)
        ms_st = timed(lambda: bm.sv_mismatch(ctx, dset, a_st, result=res), 10)
        res.free()
        first = bm.sv_first_mismatch(ctx, dset, a)
        ms_f = timed(lambda: bm.sv_first_mismatch(ctx, dset, a), 10)
        kms_f = kernel_ms(lambda: bm.sv_first_mismatch(ctx, dset, a), "mismatch_kernel<true>")
        for key, call_ms, k_ms in (("find_mismatch", ms, kms), ("find_first_mismatch", ms_f, kms_f)):
            t = k_ms or call_ms
            gbps = nbytes / (t * 1e-3) / 1e9
            r[key] = {"call_ms": call_ms, "kernel_ms": k_ms if k_ms else "not measured", "GBps": gbps,
                      "of_datasheet": gbps / (HBM_TBPS * 1e3), "of_read_ceiling": gbps / ceiling if ceiling else "not measured"}
        r["find_mismatch"]["stored_call_ms"] = ms_st
        r["count"] = cnt
        r["first"] = first
        if REF_MM.exists():
            sf, rcnt, s1, rfound, rmidx = ref_time(vals, nulls, v, nulls)
            r["reference_1core"] = {"find_mismatch_s": sf, "count": rcnt, "counts_equal": rcnt == cnt,
                                    "find_first_mismatch_s": s1, "first": rmidx if rfound else None,
                                    "first_equal": (rmidx if rfound else None) == first,
                                    "speedup_find_mismatch": sf / (ms * 1e-3), "speedup_find_first_mismatch": s1 / (ms_f * 1e-3)}
        else:
            r["reference_1core"] = "not measured (reference library not built)"
        out["results"][name] = r
    dset.free()
    out["wall_s"] = round(time.time() - t0, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
