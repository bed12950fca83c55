"""Scanner searches over a rank-select compressed sparse vector (bm::rsc_sparse_vector<unsigned>) on one GPU: the bit-sliced
scan over the compressed planes (bmb200_scan), the rank decompression to logical positions (bmb200_rank_decompress), and the
whole search, against the same searches over the equivalent plain nullable sparse vector (bmb200_scan in the logical space),
alternated in one process.  Prints one JSON line.

The vector: 2^log2_size logical positions; its NOT-NULL vector NN cycles through NULL, FULL, GAP (1-runs of 1024 bits) and BIT
(iid 1/2) blocks, four of each per 16 blocks; every NOT-NULL element holds a random 16-bit value (16 planes).
Parity: every result column (kind, popcount, digest, run count) of the RSC search equals the plain search's, and every
cardinality equals a numpy count over the values."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import bitmagic_b200 as bm                                                   # noqa: E402
from bitmagic_b200 import capi                                               # noqa: E402
from bitmagic_b200.hostfmt import BLOCK_BITS, BVector, PackedSet, bits_to_words   # noqa: E402

N_PLANES = 16


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return out[0].strip(), float(out[1])
    except Exception:
        return "unknown", None


def build(log2_size, seed):
    rng = np.random.default_rng(seed)
    n = 1 << log2_size
    nb = n // BLOCK_BITS
    i = np.arange(BLOCK_BITS)
    nn = np.zeros(n, np.uint8)
    for b in range(nb):
        k = (b % 16) // 4
        blk = nn[b * BLOCK_BITS:(b + 1) * BLOCK_BITS]
        if k == 1: blk[:] = 1
        elif k == 2: blk[:] = ((i >> 10) & 1) == 0
        elif k == 3: blk[:] = rng.random(BLOCK_BITS) < 0.5
    pos = np.flatnonzero(nn)
    vals_c = rng.integers(0, 1 << N_PLANES, pos.size).astype(np.uint32)     # values of the NOT-NULL elements, in order
    eff = pos.size
    ncomp = max(1, (eff + BLOCK_BITS - 1) // BLOCK_BITS)
    nn_v = BVector.from_words(bits_to_words(nn)).optimize()
    comp, logical = [], []
    for j in range(N_PLANES):
        bj = ((vals_c >> j) & 1).astype(np.uint8)
        cb = np.zeros(ncomp * BLOCK_BITS, np.uint8); cb[:eff] = bj
        comp.append(BVector.from_words(bits_to_words(cb)))
        lb = np.zeros(n, np.uint8); lb[pos] = bj
        logical.append(BVector.from_words(bits_to_words(lb)).optimize())
    ub = np.zeros(ncomp * BLOCK_BITS, np.uint8); ub[:eff] = 1
    uni = BVector.from_words(bits_to_words(ub)).optimize()
    rsc_ps = PackedSet.pack(comp + [uni, nn_v], nb)
    plain_ps = PackedSet.pack(logical + [nn_v], nb)
    return vals_c, eff, ncomp, nb, rsc_ps, plain_ps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2-size", type=int, default=31)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    import torch
    name, power = card()
    vals_c, eff, ncomp, nb, rsc_ps, plain_ps = build(a.log2_size, a.seed)
    ctx = bm.default_context(0)
    ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    rset, pset = capi.DeviceSet.upload(ctx, rsc_ps), capi.DeviceSet.upload(ctx, plain_ps)
    del rsc_ps, plain_ps
    rs = capi.DeviceRS(ctx, rset, N_PLANES + 1)
    rng = np.random.default_rng(a.seed + 1)
    batches = {"find_eq": (bm.SCAN_EQ, rng.integers(0, 1 << N_PLANES, 8).astype(np.uint64)),
               "find_range": (bm.SCAN_RANGE, np.sort(rng.integers(0, 1 << N_PLANES, (4, 2)), axis=1).astype(np.uint64))}
    F = bm.F_OPT_COMPRESS
    ev = lambda: torch.cuda.Event(enable_timing=True)                       # noqa: E731
    out = {"metric": "rsc scan ms per batch", "card": name, "power_limit_w": power, "logical_bits": 1 << a.log2_size,
           "effective_size": int(eff), "planes": N_PLANES, "reps": a.reps, "batches": {}}
    parity = True
    for label, (pred, vals) in batches.items():
        nv = vals.shape[0]
        sres = dres = pres = None
        t = {"scan": [], "decompress": [], "rsc_total": [], "plain": []}
        for r in range(a.warmup + a.reps):
            e0, e1, e2, e3, e4 = ev(), ev(), ev(), ev(), ev()
            e0.record()
            sres = capi.scan(ctx, rset, pred, vals, 0, N_PLANES, N_PLANES, F, 0, ncomp, result=sres)
            e1.record()
            dres = capi.rank_decompress(ctx, rs, sres, F, result=dres)
            e2.record()
            e3.record()
            pres = capi.scan(ctx, pset, pred, vals, 0, N_PLANES, N_PLANES, F, result=pres)     # universe = NN
            e4.record()
            torch.cuda.synchronize()
            if r >= a.warmup:
                t["scan"].append(e0.elapsed_time(e1)); t["decompress"].append(e1.elapsed_time(e2))
                t["rsc_total"].append(e0.elapsed_time(e2)); t["plain"].append(e3.elapsed_time(e4))
        ma, mb = dres.meta(), pres.meta()
        same_cols = all(np.array_equal(x, y) for x, y in zip(ma, mb))
        tot = dres.group_totals(nv)
        if pred == bm.SCAN_EQ:
            want = [int((vals_c == v).sum()) for v in vals]
        else:
            want = [int(((vals_c >= lo) & (vals_c <= hi)).sum()) for lo, hi in vals]
        same_counts = [int(x) for x in tot] == want and [int(x) for x in sres.group_totals(nv)] == want
        parity = parity and same_cols and same_counts
        kind, off, bits, gaps = dres.fetch()
        res_bytes = bits.nbytes + gaps.nbytes
        read = rset.stored_bytes() + res_bytes
        med = {k: float(np.median(v)) for k, v in t.items()}
        out["batches"][label] = {"values": int(nv), "ms": med, "ms_min": {k: float(np.min(v)) for k, v in t.items()},
                                 "stored_bytes_read": int(read), "result_bytes": int(res_bytes),
                                 "tb_per_s": read / (med["rsc_total"] * 1e-3) / 1e12,
                                 "frac_of_3_35_tbs": read / (med["rsc_total"] * 1e-3) / 3.35e12,
                                 "plain_stored_bytes": int(pset.stored_bytes()),
                                 "parity": {"columns_equal_plain": bool(same_cols), "counts_equal_numpy": bool(same_counts)}}
        for h in (sres, dres, pres):
            h.free()
    out["parity"] = bool(parity)
    rs.free(); rset.free(); pset.free()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
