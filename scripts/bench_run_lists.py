"""C3's data through the whole-set AND-SUB kernel with the run-list companion (TUNE_RUN_LISTS 1) and without it (0), alternated,
CUDA events over 20 calls, for an AND group of bit-block vectors ({1, 2}: parts A and B are used) and one with a GAP vector
({1, 601}: the companion is not), both with the coverage planes off (TUNE_COVERAGE 0); then, for the AND group of bit-block
vectors, the same calls through the coverage plane of its size (ms_coverage, streamed_bytes_coverage: 8 KB per AND-group
bit-block in the columns whose plane is not full and 8 KB per stored plane column) and its one-time build (the first call with
TUNE_COVERAGE 2 minus a steady call); streamed_bytes is what the library's default path streams.  Prints ms per call, the bytes each launch streams (unlisted bit-blocks, the companion parts it
reads, with the singles as streamed: packed word units, or the list form in builds before them) next to bench.py's algorithmic
bytes (which count every stored block), part B's size and listed blocks, how many columns stream a union mask (8 KB each, in
place of their parts), the one-time build, popcount / digest equality, and the card it ran on.
python scripts/bench_run_lists.py   (from the repository root, on an H100)"""
import json
import subprocess
import sys
import time
from pathlib import Path
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import numpy as np, torch, bitmagic_b200 as bm
import bench

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
ctx = bm.Context(0)
stream = torch.cuda.current_stream(); ctx.set_stream(stream.cuda_stream)
dens, seed, opt = bench.workload_inputs("c3", 0)
n_vec, n_cols = 1024, 16384
dset = bm.DeviceSet.synth(ctx, n_vec, n_cols, dens, seed, opt); ctx.sync()
counts, gap_words = bench.device_set_stats(ctx, dset, torch)
print(json.dumps({"card": card, "source_blocks": counts}))
has_coverage = hasattr(bm.capi.lib(), "bmb200_set_coverage")
if has_coverage:
    ctx.set_tuning(bm.capi.TUNE_COVERAGE, 0)


def call(g0, g1, res=None):
    return bm.aggregate(ctx, dset, bm.OP_AND_SUB, g0, g1, bm.F_OPT_COMPRESS, result=res)


def timed(g0, g1):
    """ms per call over 20 calls after 3 warm-up calls, and the last result's popcount sum, digest XOR and result bytes"""
    res = None
    for w in range(3):
        res = call(g0, g1, res)
    ctx.sync()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(20):
        res = call(g0, g1, res)
    b.record(); ctx.sync()
    k, p, d, n = res.meta()
    res_bytes = int((k == bm.BLK_BIT).sum()) * 8192 + int(2 * (n[k == bm.BLK_GAP].astype(np.int64) + 1).sum())
    res.free()
    return round(a.elapsed_time(b) / 20, 4), int(p.astype(np.int64).sum()), int(np.bitwise_xor.reduce(d)), res_bytes


def and_bit_blocks(g0):
    """AND-group bit-blocks in the columns where no AND member is NULL (the coverage path streams no other column's members)"""
    ptrs = dset.device_ptrs()

    class Wrap:
        def __init__(self, addr, shape):
            self.__cuda_array_interface__ = {"shape": shape, "typestr": "<i4", "data": (addr, False), "version": 2}
    desc = torch.as_tensor(Wrap(ptrs.desc, (n_cols, n_vec)), device="cuda:%d" % ctx.device)[:, g0] & 3
    live = (desc != bm.BLK_NULL).all(dim=1, keepdim=True)
    return int(((desc == bm.BLK_BIT) & live).sum())


for g0 in ([0, 1], [0, 600]):
    g1 = np.array([v for v in range(n_vec) if v not in g0], np.uint32)
    out = {"and_group": [v + 1 for v in g0]}
    if dset.run_list_bytes() == (0, 0):       # the default rule builds on the second qualifying call: time both
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)
        res = call(g0, g1); ctx.sync(); res.free()
        t0 = time.perf_counter(); res = call(g0, g1); ctx.sync(); out["second_call_ms"] = round((time.perf_counter() - t0) * 1e3, 2); res.free()
        out["built"] = dset.run_list_bytes() != (0, 0)
    for rep in range(2):
        for mode in (0, 1):
            ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, mode)
            ms, pop, dig, res_bytes = timed(g0, g1)
            out.setdefault("ms_mode%d" % mode, []).append(ms)
            out.setdefault("pop%d" % mode, pop)
            out.setdefault("dig%d" % mode, dig)
    sgl, lr = dset.run_list_bytes()
    bsgl, blr, listed = dset.bit_run_list_bytes()
    if hasattr(bm.capi.lib(), "bmb200_set_packed_singles"):     # singles as streamed; older builds stream the list form
        out["list_form_singles"] = {"a": sgl, "b": bsgl}
        sgl, bsgl = dset.packed_singles_bytes()
    alg = counts["bit"] * 8192 + gap_words * 2 + res_bytes + n_cols * 12
    un_a, un_ab = dset.run_list_unions() if hasattr(bm.capi.lib(), "bmb200_set_run_list_unions") else (0, 0)
    out["union_columns"] = {"a": un_a, "ab": un_ab}
    if g0 == [0, 1]:          # A + B in place of the GAP segments and the listed bit-blocks
        # a union column streams one 8 KB mask in place of its parts; the parts' sizes are only known summed over the set
        if un_ab not in (0, n_cols):
            sys.exit("only some columns stream a union mask: the streamed bytes need per-column part sizes")
        src = (counts["bit"] - listed) * 8192 + (n_cols * 8192 if un_ab else sgl + lr + bsgl + blr)
    else:
        src = counts["bit"] * 8192 + dset.n_gap_units * 16
    streamed = src + res_bytes + n_cols * 12
    pop_ref, dig_ref = out["pop0"], out["dig0"]
    out["same"] = out.pop("pop0") == out.pop("pop1") and out.pop("dig0") == out.pop("dig1")
    out["companion_bytes"] = {"singles": sgl, "long_runs": lr}
    out["part_b"] = {"singles": bsgl, "long_runs": blr, "listed_blocks": listed, "listed_per_column": round(listed / n_cols, 2)}
    out["bench_algorithmic_bytes"] = alg
    out["streamed_bytes_mode1"] = streamed
    out["streamed_gbs_mode1"] = round(streamed / (min(out["ms_mode1"]) * 1e-3) / 1e9, 1)
    if "second_call_ms" in out:
        out["build_ms"] = round(out["second_call_ms"] - min(out["ms_mode1"]), 2)     # the building call minus a steady call
    out["streamed_bytes"] = streamed
    if has_coverage and g0 == [0, 1]:       # the coverage plane of n0 = 2, built on its first call and nothing else with it
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 0); ctx.set_tuning(bm.capi.TUNE_COVERAGE, 2)
        t0 = time.perf_counter(); call(g0, g1).free(); ctx.sync(); first_ms = (time.perf_counter() - t0) * 1e3
        stored, one = dset.coverage(len(g0))
        timings = [timed(g0, g1) for _ in range(2)]
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1); ctx.set_tuning(bm.capi.TUNE_COVERAGE, 0)
        if one:
            sys.exit("some columns have a full plane: the streamed bytes need to know which")
        cov = (and_bit_blocks(g0) + stored) * 8192 + timings[0][3] + n_cols * 12
        out["coverage_columns"] = {"stored": stored, "one": one}
        out["ms_coverage"] = [t[0] for t in timings]
        out["coverage_same"] = all(t[1:3] == (pop_ref, dig_ref) for t in timings)
        out["coverage_build_ms"] = round(first_ms - min(out["ms_coverage"]), 2)
        out["streamed_bytes_coverage"] = out["streamed_bytes"] = cov
        out["streamed_gbs_coverage"] = round(cov / (min(out["ms_coverage"]) * 1e-3) / 1e9, 1)
    print(json.dumps(out))
dset.free()
