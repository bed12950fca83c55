"""String searches over a string sparse vector (bm::str_sparse_vector<char, ...>) on one GPU: batches of find_eq_str and
find_eq_str_prefix queries as one bmb200_scan_str launch each.  Prints one JSON line per workload.

Workloads (2^log2_size strings each, drawn from one seeded synthetic dictionary: Zipf(1.1) word frequencies, lengths 3-20 over
a 26-letter alphabet):
  unsorted   the strings in draw order;
  sorted     the same strings sorted, the order in which the reference's reverse-octet walk is said to pay off;
  remapped   the unsorted vector remap()ed by the reference (planes and query codes from the reference library).
Queries: 64 exact (dictionary words by frequency, some absent) and 64 prefix (2-4 leading bytes of dictionary words).
Reported: GPU ms per launch (CUDA events, median of --reps after --warmup), searches/s, stored bytes of planes + universe, the
reference's ms per search on one core (through oracle/_ref/libbmref_str.so, first 16 queries of each kind), whether the first 16
counts of each kind equal the reference's, and the card name and power limit read in the same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bitmagic_b200 as bm                                                   # noqa: E402
from bitmagic_b200 import capi                                               # noqa: E402
from bitmagic_b200.hostfmt import BLOCK_BITS, BVector, PackedSet, bits_to_words   # noqa: E402

REF_STR = ROOT / "oracle" / "_ref" / "libbmref_str.so"
MAX_LEN = 20


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return out[0].strip(), float(out[1])
    except Exception:
        return "unknown", None


def dictionary(rng, n_words):
    """-> sorted unique words as an (n, MAX_LEN + 1) NUL-padded uint8 matrix"""
    lens = rng.integers(3, MAX_LEN + 1, 2 * n_words)
    letters = rng.integers(ord("a"), ord("z") + 1, (2 * n_words, MAX_LEN)).astype(np.uint8)
    letters[np.arange(MAX_LEN)[None, :] >= lens[:, None]] = 0
    mat = np.zeros((2 * n_words, MAX_LEN + 1), np.uint8)
    mat[:, :MAX_LEN] = letters
    mat = np.unique(mat, axis=0)[:n_words]                                  # unique rows, in byte (= string) order
    return mat


def planes_of(mat_rows, nb):
    """plane 8k+b of the strings (rows of NUL-padded bytes), trailing empty planes trimmed"""
    n = mat_rows.shape[0]
    planes = []
    used = np.bitwise_or.reduce(mat_rows, axis=0)
    top = max([j + 1 for j in range(8 * MAX_LEN) if (used[j >> 3] >> (j & 7)) & 1], default=1)
    for j in range(top):
        bits = np.zeros(nb * BLOCK_BITS, np.uint8)
        bits[:n] = (mat_rows[:, j >> 3] >> (j & 7)) & 1
        planes.append(BVector.from_words(bits_to_words(bits)).optimize())
    return planes


def universe(n, nb):
    bits = np.zeros(nb * BLOCK_BITS, np.uint8)
    bits[:n] = 1
    return BVector.from_words(bits_to_words(bits)).optimize()


def ref_lib():
    if not REF_STR.exists():
        return None
    return C.CDLL(str(REF_STR))


def ref_planes_remapped(ref, slots, nb):
    n, stride = slots.shape
    max_planes = 8 * MAX_LEN
    kind = np.zeros((max_planes + 1) * nb, np.uint8)
    blocks = np.zeros(((max_planes + 1) * nb, 2048), np.uint32)
    gaps = np.zeros(((max_planes + 1) * nb, 1280), np.uint16)
    npl, ms = C.c_uint32(0), C.c_uint32(0)
    rc = ref.ref_str_planes(capi.ptr(slots), C.c_uint32(stride), C.c_uint64(n), None, 1, C.c_uint32(nb), C.c_uint32(max_planes),
                            C.byref(npl), C.byref(ms), capi.ptr(kind), capi.ptr(blocks), capi.ptr(gaps))
    assert rc == 0, rc
    vecs = []
    for j in range(npl.value + 1):
        bv = BVector(nb)
        for c in range(nb):
            k = int(kind[j * nb + c])
            if k == bm.BLK_FULL: bv.set_full(c)
            elif k == bm.BLK_BIT: bv.set_bits(c, blocks[j * nb + c])
            elif k == bm.BLK_GAP:
                g = gaps[j * nb + c]
                bv.set_gap(c, g[:(int(g[0]) >> 3) + 1])
        vecs.append(bv)
    return vecs, int(ms.value)


def ref_remap(ref, slots, q):
    out = np.zeros_like(q); ok = np.zeros(q.shape[0], np.uint8)
    rc = ref.ref_str_remap(capi.ptr(slots), C.c_uint32(slots.shape[1]), C.c_uint64(slots.shape[0]), None, capi.ptr(q),
                           C.c_uint32(q.shape[1]), C.c_uint32(q.shape[0]), capi.ptr(out), capi.ptr(ok))
    assert rc == 0, rc
    return out, ok


def ref_counts(ref, slots, remap, mode, q):
    nq = q.shape[0]
    found = np.zeros(nq, np.uint8); pos = np.zeros(nq, np.uint64); counts = np.zeros(nq, np.uint64)
    nc = max(1, (slots.shape[0] + BLOCK_BITS - 1) // BLOCK_BITS)
    words = np.zeros((nq, nc * 2048), np.uint32)
    rc = ref.ref_str_find(capi.ptr(slots), C.c_uint32(slots.shape[1]), C.c_uint64(slots.shape[0]), None, int(remap), int(mode),
                          capi.ptr(q), C.c_uint32(q.shape[1]), C.c_uint32(nq), C.c_uint32(nc), capi.ptr(found), capi.ptr(pos),
                          capi.ptr(counts), capi.ptr(words))
    assert rc == 0, rc
    return counts


def ref_ms_per_search(ref, slots, remap, mode, q):
    sec, tot = C.c_double(0), C.c_uint64(0)
    rc = ref.ref_str_time(capi.ptr(slots), C.c_uint32(slots.shape[1]), C.c_uint64(slots.shape[0]), None, int(remap), int(mode),
                          capi.ptr(q), C.c_uint32(q.shape[1]), C.c_uint32(q.shape[0]), 1, C.byref(sec), C.byref(tot))
    assert rc == 0, rc
    return 1e3 * sec.value / q.shape[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2-size", type=int, default=24)
    ap.add_argument("--words", type=int, default=200000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--no-ref", action="store_true", help="skip the reference's timing and counts")
    ap.add_argument("--workloads", default="unsorted,sorted,remapped")
    a = ap.parse_args()
    import torch
    name, power = card()
    rng = np.random.default_rng(a.seed)
    n = 1 << a.log2_size
    nb = max(1, n // BLOCK_BITS)
    dmat = dictionary(rng, a.words)
    zipf = 1.0 / np.arange(1, dmat.shape[0] + 1) ** 1.1
    rank = rng.permutation(dmat.shape[0])                                  # word frequencies do not follow their sort order
    p = zipf[rank]; p /= p.sum()
    idx = rng.choice(dmat.shape[0], n, p=p)
    by_freq = np.argsort(-p)
    exact_idx = np.concatenate([by_freq[:48], rng.integers(0, dmat.shape[0], 12)])
    q_exact = np.concatenate([dmat[exact_idx], np.zeros((4, MAX_LEN + 1), np.uint8)])
    q_exact[-4:, :5] = np.frombuffer(b"qqqqq", np.uint8)                   # absent words
    q_exact[-3:, 4] = 0; q_exact[-2:, 3] = 0; q_exact[-1:, 2] = 0
    q_prefix = dmat[by_freq[rng.integers(0, 2000, 64)]].copy()
    for k, L in enumerate(rng.integers(2, 5, 64)):
        q_prefix[k, L:] = 0
    ctx = bm.default_context(0)
    ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    ref = None if a.no_ref else ref_lib()

    for wl in a.workloads.split(","):
        order = np.sort(idx) if wl == "sorted" else idx                    # dmat rows are in string order
        slots = dmat[order]
        qe, qp = q_exact, q_prefix
        if wl == "remapped":
            if ref is None:
                print(json.dumps({"workload": wl, "skipped": "reference library not built"}), flush=True)
                continue
            vecs, max_str = ref_planes_remapped(ref, slots, nb)
            planes, uni = vecs[:-1], vecs[-1]
            qe, oke = ref_remap(ref, slots, q_exact)
            qp, okp = ref_remap(ref, slots, q_prefix)
            qe, qp = qe[oke.astype(bool)], qp[okp.astype(bool)]            # queries without codes match nothing: no launch slot
        else:
            planes, uni = planes_of(slots, nb), universe(n, nb)
        ps = PackedSet.pack(planes + [uni], nb)
        dset = capi.DeviceSet.upload(ctx, ps)
        npl = len(planes)
        line = {"workload": wl, "n": n, "n_planes": npl, "stored_bytes": int(dset.stored_bytes()), "gpu": name, "power_limit_w": power}
        for kind, q, flags in (("exact", qe, bm.F_OPT_COMPRESS), ("prefix", qp, bm.F_OPT_COMPRESS | bm.F_STR_PREFIX)):
            res = None
            for _ in range(a.warmup):
                res = capi.scan_str(ctx, dset, q, 0, npl, npl, flags, result=res)
            times = []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                res = capi.scan_str(ctx, dset, q, 0, npl, npl, flags, result=res)
                e1.record()
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
            counts = res.group_totals(q.shape[0])
            res.free()
            ms = float(np.median(times))
            line[f"{kind}_queries"] = int(q.shape[0])
            line[f"{kind}_gpu_ms_per_launch"] = round(ms, 4)
            line[f"{kind}_searches_per_s"] = round(q.shape[0] / (ms * 1e-3), 1)
            line[f"{kind}_matches"] = int(counts.sum())
            if ref is not None:
                src = q_exact if kind == "exact" else q_prefix
                remap = 1 if wl == "remapped" else 0
                if remap:
                    # per query its count, 0 where it has no code; the reference is asked only where it defines an answer (a query
                    # shorter than effective_max_str())
                    ok = (oke if kind == "exact" else okp).astype(bool)
                    ours_all = np.zeros(src.shape[0], np.uint64)
                    ours_all[ok] = counts
                    keep = np.flatnonzero((src != 0).sum(1) < max_str)[:16]
                    rq, ours = src[keep], ours_all[keep]
                else:
                    rq, ours = src[:16], counts[:16]
                rc = ref_counts(ref, slots, remap, 0 if kind == "exact" else 1, rq)
                line[f"{kind}_counts_match_reference_16"] = bool(np.array_equal(ours, rc))
                line[f"{kind}_ref_ms_per_search_1core"] = round(ref_ms_per_search(ref, slots, remap, 0 if kind == "exact" else 1, rq), 3)
        dset.free()
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
