#!/usr/bin/env python
"""Scanner row (SURVEY 8 f2): bmb200_scan vs bm::sparse_vector_scanner<> on the same sparse vector.
  python scripts/bench_scan.py [n_elements]            -> one JSON line
  python scripts/bench_scan.py --signed [n_elements]   -> one JSON line for a signed vector (sparse_vector<int32_t>, F_SIGNED)
  python scripts/bench_scan.py --float [n_elements]    -> one JSON line for a float vector (sparse_vector_float, F_FLOAT)
Workloads: "dense" = uniform 20-bit values (bit-block planes), "sparse" = 99.6 % zeros (GAP planes).
The GPU answers all search values in ONE launch (values of a column adjacent -> planes from L2); the reference answers
them one by one on one host core.  Algorithmic bytes of a scan = stored bytes of the planes + universe, once per value."""
import ctypes as C
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import torch                 # noqa: E402
import bitmagic_b200 as bm   # noqa: E402
import orclib                # noqa: E402


def run(name, vals, ctx, preds, n_search=64):
    planes = orclib.ref_sv_planes(vals, None)
    ps = bm.PackedSet.pack(planes)
    npl = len(planes) - 1
    dset = bm.DeviceSet.upload(ctx, ps)
    rng = np.random.default_rng(3)
    out = {"elements": int(vals.size), "planes": npl, "block_columns": ps.n_blocks, "stored_MiB": ps.stored_bytes() / 2**20,
           "kinds": {k: int((ps.kinds() == v).sum()) for k, v in (("null", 0), ("full", 1), ("bit", 2), ("gap", 3))}}
    for pname, pred in preds:
        search = rng.choice(vals, n_search).astype(np.uint64)
        if pred == bm.SCAN_RANGE:
            search = np.stack([search, search + 1000], 1)
        res = bm.scan(ctx, dset, pred, search, 0, npl, npl, bm.F_OPT_COMPRESS)
        ctx.sync()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 10
        ev0.record(torch.cuda.current_stream())
        for _ in range(reps):
            bm.scan(ctx, dset, pred, search, 0, npl, npl, bm.F_OPT_COMPRESS, result=res)
        ev1.record(torch.cuda.current_stream())
        torch.cuda.synchronize()
        ms = ev0.elapsed_time(ev1) / reps
        tot_gpu = int(res.group_totals(n_search).sum())
        res.free()
        ref_s = search.astype(np.uint32)[:16]
        sec, tot_ref = orclib.ref_sv_time_scan(vals, None, pred, ref_s, repeats=1)
        r16 = bm.scan(ctx, dset, pred, search[:16], 0, npl, npl, bm.F_COUNT_ONLY)
        same = int(r16.group_totals(16).sum()) == tot_ref
        r16.free()
        out[pname] = {"gpu_ms_per_launch": ms, "searches_per_launch": n_search, "gpu_searches_per_s": n_search / (ms * 1e-3),
                      "gpu_plane_GBps": ps.stored_bytes() * n_search / (ms * 1e-3) / 1e9, "result_bits": tot_gpu,
                      "ref_ms_per_search_1core": sec * 1e3 / 16, "ref_searches_per_s_1core": 16 / sec, "counts_equal_first16": bool(same),
                      "speedup_vs_1core": (n_search / (ms * 1e-3)) / (16 / sec)}
    dset.free()
    return out


REF_SIGNED = ROOT / "oracle" / "_ref" / "libbmref_signed.so"     # oracle/signed.mk


def ref_svs_time_scan(vals, pred, search, repeats=1):
    """signed twin of orclib.ref_sv_time_scan: sparse_vector<int32_t> + sparse_vector_scanner on one core -> (seconds, total)"""
    v = np.ascontiguousarray(vals, np.int64); s = np.ascontiguousarray(search, np.int64)
    ns = s.shape[0] if pred == bm.SCAN_RANGE else s.size
    sec, tot = C.c_double(0), C.c_uint64(0)
    rc = C.CDLL(str(REF_SIGNED)).ref_svs_time_scan(0, bm.capi.ptr(v), C.c_void_p(0), C.c_uint64(v.size), int(pred), bm.capi.ptr(s), C.c_uint32(ns),
                                        int(repeats), C.byref(sec), C.byref(tot))
    assert rc == 0, f"ref_svs_time_scan rc={rc}"
    return sec.value, tot.value


def run_signed(vals, ctx, preds, n_search=64):
    """the signed pass: s2u planes, values spanning zero, every search with F_SIGNED in one launch"""
    sv = bm.SparseVector.from_values(vals, signed=True)
    ps = bm.PackedSet.pack(list(sv.planes) + [sv.universe()])
    npl = sv.effective_slices()
    dset = bm.DeviceSet.upload(ctx, ps)
    rng = np.random.default_rng(3)
    flags = bm.F_OPT_COMPRESS | bm.F_SIGNED
    out = {"elements": int(vals.size), "planes": npl, "block_columns": ps.n_blocks, "stored_MiB": ps.stored_bytes() / 2**20}
    for pname, pred in preds:
        search = rng.choice(vals, n_search).astype(np.int64)
        if pred == bm.SCAN_RANGE:
            search = np.stack([search, search + 1000], 1)
        res = bm.scan(ctx, dset, pred, search, 0, npl, npl, flags)
        ctx.sync()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 10
        ev0.record(torch.cuda.current_stream())
        for _ in range(reps):
            bm.scan(ctx, dset, pred, search, 0, npl, npl, flags, result=res)
        ev1.record(torch.cuda.current_stream())
        torch.cuda.synchronize()
        ms = ev0.elapsed_time(ev1) / reps
        res.free()
        entry = {"gpu_ms_per_launch": ms, "searches_per_launch": n_search, "gpu_us_per_search": ms * 1e3 / n_search,
                 "stored_bytes_per_search": ps.stored_bytes(), "gpu_plane_GBps": ps.stored_bytes() * n_search / (ms * 1e-3) / 1e9}
        if REF_SIGNED.exists():
            sec, tot_ref = ref_svs_time_scan(vals, pred, search[:16])
            r16 = bm.scan(ctx, dset, pred, search[:16], 0, npl, npl, bm.F_COUNT_ONLY | bm.F_SIGNED)
            entry.update({"ref_ms_per_search_1core": sec * 1e3 / 16, "counts_equal_first16": int(r16.group_totals(16).sum()) == tot_ref,
                          "speedup_vs_1core": (n_search / (ms * 1e-3)) / (16 / sec)})
            r16.free()
        else:
            entry["ref_ms_per_search_1core"] = "not measured (reference library not built)"
        out[pname] = entry
    dset.free()
    return out


REF_FLOAT = ROOT / "oracle" / "_ref" / "libbmref_float.so"       # oracle/float.mk


def ref_svf_time_scan(vals, pred, search, repeats=1):
    """float twin of orclib.ref_sv_time_scan: sparse_vector_float + sparse_vector_scanner on one core -> (seconds, total)"""
    v = np.ascontiguousarray(vals, np.float32); s = np.ascontiguousarray(search, np.float32)
    ns = s.shape[0] if pred in (bm.SCAN_RANGE, bm.SCAN_RANGE_OPEN) else s.size
    sec, tot = C.c_double(0), C.c_uint64(0)
    rc = C.CDLL(str(REF_FLOAT)).ref_svf_time_scan(bm.capi.ptr(v), C.c_void_p(0), C.c_uint64(v.size), int(pred), bm.capi.ptr(s), C.c_uint32(ns),
                                                  int(repeats), C.byref(sec), C.byref(tot))
    assert rc == 0, f"ref_svf_time_scan rc={rc}"
    return sec.value, tot.value


def run_float(vals, ctx, preds, n_search=64):
    """the float pass: sign + 31 magnitude planes, values of both signs, every search with F_FLOAT in one launch"""
    sv = bm.SparseVectorFloat.from_values(vals)
    ps = bm.PackedSet.pack(list(sv.planes) + [sv.universe()])
    npl = sv.effective_slices()
    dset = bm.DeviceSet.upload(ctx, ps)
    rng = np.random.default_rng(3)
    flags = bm.F_OPT_COMPRESS | bm.F_FLOAT
    out = {"elements": int(vals.size), "planes": npl, "block_columns": ps.n_blocks, "stored_MiB": ps.stored_bytes() / 2**20}
    for pname, pred in preds:
        search = rng.choice(vals, n_search).astype(np.float32)
        if pred in (bm.SCAN_RANGE, bm.SCAN_RANGE_OPEN):
            search = np.stack([search, search + np.abs(search) * np.float32(0.1) + np.float32(1)], 1)
        res = bm.scan(ctx, dset, pred, search, 0, npl, npl, flags)
        ctx.sync()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 10
        ev0.record(torch.cuda.current_stream())
        for _ in range(reps):
            bm.scan(ctx, dset, pred, search, 0, npl, npl, flags, result=res)
        ev1.record(torch.cuda.current_stream())
        torch.cuda.synchronize()
        ms = ev0.elapsed_time(ev1) / reps
        res.free()
        entry = {"gpu_ms_per_launch": ms, "searches_per_launch": n_search, "gpu_us_per_search": ms * 1e3 / n_search,
                 "stored_bytes_per_search": ps.stored_bytes(), "gpu_plane_GBps": ps.stored_bytes() * n_search / (ms * 1e-3) / 1e9}
        if REF_FLOAT.exists():
            sec, tot_ref = ref_svf_time_scan(vals, pred, search[:16])
            r16 = bm.scan(ctx, dset, pred, search[:16], 0, npl, npl, bm.F_COUNT_ONLY | bm.F_FLOAT)
            entry.update({"ref_ms_per_search_1core": sec * 1e3 / 16, "counts_equal_first16": int(r16.group_totals(16).sum()) == tot_ref,
                          "speedup_vs_1core": (n_search / (ms * 1e-3)) / (16 / sec)})
            r16.free()
        else:
            entry["ref_ms_per_search_1core"] = "not measured (reference library not built)"
        out[pname] = entry
    dset.free()
    return out


def power_limit():
    """the card's enforced power limit (read-only query), part of any number this prints"""
    import subprocess
    try:
        p = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return p.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    n = int(args[0]) if args else 1 << 24
    ctx = bm.Context(0)
    ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    rng = np.random.default_rng(11)
    if "--signed" in sys.argv[1:]:
        preds = [("find_eq", bm.SCAN_EQ), ("find_gt", bm.SCAN_GT), ("find_lt", bm.SCAN_LT), ("find_range", bm.SCAN_RANGE)]
        vals = rng.integers(-(1 << 19), 1 << 19, n).astype(np.int64)          # 20-bit codes: sign plane + 19 magnitude planes
        props = torch.cuda.get_device_properties(0)
        t0 = time.time()
        res = {"signed20": run_signed(vals, ctx, preds)}
        print(json.dumps({"bench": "scan_signed", "n": n, "device": props.name, "power_limit": power_limit(), "wall_s": round(time.time() - t0, 1),
                          "results": res}))
        return
    if "--float" in sys.argv[1:]:
        preds = [("find_gt_float", bm.SCAN_GT), ("find_lt_float", bm.SCAN_LT), ("find_range_float", bm.SCAN_RANGE),
                 ("find_range_float_unbounded", bm.SCAN_RANGE_OPEN)]
        vals = (rng.standard_normal(n) * 1000).astype(np.float32)           # both signs, full mantissas: all 32 planes are bit planes
        props = torch.cuda.get_device_properties(0)
        t0 = time.time()
        res = {"normal1000": run_float(vals, ctx, preds)}
        print(json.dumps({"bench": "scan_float", "n": n, "device": props.name, "power_limit": power_limit(), "wall_s": round(time.time() - t0, 1),
                          "results": res}))
        return
    preds = [("find_eq", bm.SCAN_EQ), ("find_gt", bm.SCAN_GT), ("find_range", bm.SCAN_RANGE)]
    dense = rng.integers(0, 1 << 20, n).astype(np.uint32)
    sparse = np.where(rng.random(n) < 0.004, rng.integers(1, 1 << 16, n), 0).astype(np.uint32)
    t0 = time.time()
    res = {"dense20": run("dense20", dense, ctx, preds), "sparse16": run("sparse16", sparse, ctx, preds)}
    print(json.dumps({"bench": "scan", "n": n, "wall_s": round(time.time() - t0, 1), "results": res}))


if __name__ == "__main__":
    main()
