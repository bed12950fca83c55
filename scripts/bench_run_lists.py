"""C3's data through the whole-set AND-SUB kernel with the run-list companion (TUNE_RUN_LISTS 1) and without it (0), alternated,
CUDA events over 20 calls, for an AND group of bit-block vectors ({1, 2}: parts A and B are used) and one with a GAP vector
({1, 601}: the companion is not).  Prints ms per call, the bytes each launch streams (unlisted bit-blocks, the companion parts it
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


def call(g0, g1, res=None):
    return bm.aggregate(ctx, dset, bm.OP_AND_SUB, g0, g1, bm.F_OPT_COMPRESS, result=res)


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
            res = None
            for w in range(3):
                res = call(g0, g1, res)
            ctx.sync()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(20):
                res = call(g0, g1, res)
            b.record(); ctx.sync()
            out.setdefault("ms_mode%d" % mode, []).append(round(a.elapsed_time(b) / 20, 4))
            k, p, d, n = res.meta()
            out.setdefault("pop%d" % mode, int(p.astype(np.int64).sum()))
            out.setdefault("dig%d" % mode, int(np.bitwise_xor.reduce(d)))
            res_bytes = int((k == bm.BLK_BIT).sum()) * 8192 + int(2 * (n[k == bm.BLK_GAP].astype(np.int64) + 1).sum())
            res.free()
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
    out["same"] = out.pop("pop0") == out.pop("pop1") and out.pop("dig0") == out.pop("dig1")
    out["companion_bytes"] = {"singles": sgl, "long_runs": lr}
    out["part_b"] = {"singles": bsgl, "long_runs": blr, "listed_blocks": listed, "listed_per_column": round(listed / n_cols, 2)}
    out["bench_algorithmic_bytes"] = alg
    out["streamed_bytes_mode1"] = streamed
    out["streamed_gbs_mode1"] = round(streamed / (min(out["ms_mode1"]) * 1e-3) / 1e9, 1)
    if "second_call_ms" in out:
        out["build_ms"] = round(out["second_call_ms"] - min(out["ms_mode1"]), 2)     # the building call minus a steady call
    print(json.dumps(out))
dset.free()
