"""C3's data with different AND groups (bit-block vectors only, or with GAP-block vectors in them): agg_pipe_kernel
(TUNE_AGG_PIPELINE 1) against agg_kernel (0), alternated, CUDA events over 20 calls, popcounts and digests compared.
python scripts/bench_agg_pipeline.py   (from the repository root, on an H100)"""
import sys, json
from pathlib import Path
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import numpy as np, torch, bitmagic_b200 as bm
import bench
ctx = bm.Context(0)
stream = torch.cuda.current_stream(); ctx.set_stream(stream.cuda_stream)
dens, seed, opt = bench.workload_inputs("c3", 0)
dset = bm.DeviceSet.synth(ctx, 1024, 16384, dens, seed, opt); ctx.sync()
for g0 in ([0, 1], [0, 600], [1, 300, 700]):
    g1 = np.array([v for v in range(1024) if v not in g0], np.uint32)
    out = {}
    for rep in range(2):
        for mode in (0, 1):
            ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, mode)
            res = None
            for w in range(3):
                res = bm.aggregate(ctx, dset, bm.OP_AND_SUB, g0, g1, bm.F_OPT_COMPRESS, result=res)
            ctx.sync()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(20):
                res = bm.aggregate(ctx, dset, bm.OP_AND_SUB, g0, g1, bm.F_OPT_COMPRESS, result=res)
            b.record(); ctx.sync()
            out.setdefault(mode, []).append(round(a.elapsed_time(b) / 20, 4))
            k, p, d, n = res.meta()
            out.setdefault("pop%d" % mode, int(p.astype(np.int64).sum()))
            out.setdefault("dig%d" % mode, int(np.bitwise_xor.reduce(d)))
            res.free()
    print(json.dumps({"and_group": g0, "ms_agg_kernel": out[0], "ms_pipe": out[1], "same": out["pop0"] == out["pop1"] and out["dig0"] == out["dig1"]}))
