#!/usr/bin/env python
"""Set-membership search (SCAN_IN, the iterator find_eq of sparse_vector_scanner) on the workload of the reference's sample
svsample06: a nullable sparse_vector<unsigned> of 250 M elements, values uniform in [1, 1 250 000] (21 planes, 3 815 block
columns), a 5-element NULL plate after every 64th element.
  python scripts/bench_scan_in.py [n_elements]   -> one JSON line
Per list length K (1, 16, 500, 65 536, 2^20 distinct values from the value range): the SCAN_IN launch, count-only and stored;
for K <= 500 the device's own alternative, one count-only SCAN_EQ launch over the same K values (K separate searches); and the
reference's iterator find_eq on one host core over the first 16 values (oracle/_ref/libbmref_in.so).  Times are CUDA events over
warmed calls (the host's sort of the list included); the kernel time alone comes from torch.profiler's CUDA activity, and
effective GB/s = stored bytes of the planes + universe / kernel time (the bytes a launch must read once)."""
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch                 # noqa: E402
import bitmagic_b200 as bm   # noqa: E402
from bitmagic_b200.capi import BLOCK_BITS, BLOCK_WORDS  # noqa: E402

REF_IN = ROOT / "oracle" / "_ref" / "libbmref_in.so"     # oracle/in.mk
VALUE_MAX = 1_250_000
KS = (1, 16, 500, 65536, 1 << 20)


def svsample06(n, rng):
    """values uniform in [1, VALUE_MAX]; element i is NULL when i % 64 is 1..5 (the sample's back-inserter plate)"""
    vals = rng.integers(1, VALUE_MAX + 1, n, dtype=np.uint32)
    nulls = ((np.arange(n, dtype=np.uint64) % 64) - 1 < 5).astype(np.uint8)
    vals[nulls == 1] = 0
    return vals, nulls


def plane_vectors(vals, nulls):
    """the 21 planes + the NOT-NULL vector as bit-block BVectors (every block of this workload is a bit-block)"""
    nb = (vals.size + BLOCK_BITS - 1) // BLOCK_BITS
    def vec(bits):
        w = np.zeros(nb * BLOCK_WORDS, np.uint32)
        p = np.packbits(bits, bitorder="little")
        w.view(np.uint8)[:p.size] = p
        return bm.BVector.from_words(w)
    top = int(vals.max()).bit_length()
    return [vec(((vals >> np.uint32(j)) & np.uint32(1)).astype(np.uint8)) for j in range(top)] + [vec(1 - nulls)]


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(torch.cuda.current_stream())
    for _ in range(reps):
        fn()
    ev1.record(torch.cuda.current_stream())
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / reps


def kernel_ms(fn, name, reps=5):
    """device time of the kernels whose name holds `name`, per call, from torch.profiler's CUDA activity (None if not available)"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
        us = [getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0) for e in prof.key_averages() if name in e.key]
        return sum(us) / 1e3 / reps if us else None
    except Exception:                                   # a profiler without CUDA activity: the event times stand alone
        return None


def card():
    """name, power limit and SM clocks, read in the same run as the numbers (read-only query)"""
    try:
        p = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, pl, sm, smax = [x.strip() for x in p.stdout.strip().split(",")]
        return {"device": name, "power_limit": pl, "sm_clock": sm, "sm_clock_max": smax}
    except (OSError, subprocess.SubprocessError, ValueError):
        return {"device": torch.cuda.get_device_properties(0).name, "power_limit": "unknown", "sm_clock": "unknown"}


def ref_time(vals, nulls, lst):
    """the reference's iterator find_eq on one core -> (seconds, count)"""
    v = np.ascontiguousarray(vals, np.int64); s = np.ascontiguousarray(lst, np.int64); nl = np.ascontiguousarray(nulls, np.uint8)
    sec, tot = C.c_double(0), C.c_uint64(0)
    rc = C.CDLL(str(REF_IN)).ref_in_time(0, bm.capi.ptr(v), bm.capi.ptr(nl), C.c_uint64(v.size), bm.capi.ptr(s), C.c_uint64(s.size), 1,
                                         C.byref(sec), C.byref(tot))
    assert rc == 0, f"ref_in_time rc={rc}"
    return sec.value, tot.value


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    n = int(args[0]) if args else 250_000_000
    if not torch.cuda.is_available():
        raise SystemExit("bench_scan_in: no CUDA device")
    t0 = time.time()
    rng = np.random.default_rng(6)
    vals, nulls = svsample06(n, rng)
    vecs = plane_vectors(vals, nulls)
    ps = bm.PackedSet.pack(vecs)
    npl = len(vecs) - 1
    ctx = bm.Context(0)
    ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    dset = bm.DeviceSet.upload(ctx, ps)
    stored = ps.stored_bytes()
    out = {"bench": "scan_in", "workload": "svsample06", "elements": n, "planes": npl, "block_columns": ps.n_blocks,
           "stored_MiB": stored / 2**20, **card(), "results": {}}
    pool = rng.permutation(np.arange(1, VALUE_MAX + 1, dtype=np.uint64))[:max(KS)]      # distinct values of the range
    for k in KS:
        lst = pool[:k]
        r = {}
        res = bm.scan(ctx, dset, bm.SCAN_IN, lst, 0, npl, npl, bm.F_COUNT_ONLY)
        ms = timed(lambda: bm.scan(ctx, dset, bm.SCAN_IN, lst, 0, npl, npl, bm.F_COUNT_ONLY, result=res), 10)
        cnt = int(res.group_totals(1)[0]); res.free()
        res = bm.scan(ctx, dset, bm.SCAN_IN, lst, 0, npl, npl, bm.F_OPT_COMPRESS)
        ms_st = timed(lambda: bm.scan(ctx, dset, bm.SCAN_IN, lst, 0, npl, npl, bm.F_OPT_COMPRESS, result=res), 10)
        assert int(res.group_totals(1)[0]) == cnt
        res.free()
        res = bm.scan(ctx, dset, bm.SCAN_IN, lst, 0, npl, npl, bm.F_COUNT_ONLY)
        kms = kernel_ms(lambda: bm.scan(ctx, dset, bm.SCAN_IN, lst, 0, npl, npl, bm.F_COUNT_ONLY, result=res), "scan_in_kernel")
        res.free()
        r.update({"in_count_only_ms": ms, "in_stored_ms": ms_st, "in_kernel_ms": kms if kms else "not measured",
                  "in_effective_GBps": stored / ((kms or ms) * 1e-3) / 1e9, "count": cnt})
        if k <= 500:
            res = bm.scan(ctx, dset, bm.SCAN_EQ, lst, 0, npl, npl, bm.F_COUNT_ONLY)
            ms_eq = timed(lambda: bm.scan(ctx, dset, bm.SCAN_EQ, lst, 0, npl, npl, bm.F_COUNT_ONLY, result=res), 3 if k > 16 else 10)
            eq_cnt = int(res.group_totals(k).sum()); res.free()
            r.update({"eq_count_only_ms": ms_eq, "in_speedup_vs_eq": ms_eq / ms, "counts_equal_eq": eq_cnt == cnt})
        out["results"][str(k)] = r
    if REF_IN.exists():
        lst16 = pool[:16]
        sec, tot = ref_time(vals, nulls, lst16)
        ms16 = out["results"]["16"]["in_count_only_ms"]
        out["reference_1core_k16"] = {"ref_s": sec, "ref_count": tot, "counts_equal": tot == out["results"]["16"]["count"],
                                      "speedup_vs_1core": sec / (ms16 * 1e-3)}
    else:
        out["reference_1core_k16"] = "not measured (reference library not built)"
    dset.free()
    out["wall_s"] = round(time.time() - t0, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
