"""Result retrieval parity: every fetch route of every result producer, at the column counts where the compaction and the
chunked view change shape.

A result reaches its caller through bmb200_result_fetch, bmb200_result_fetch_column, bmb200_result_fetch_view or
bmb200_result_fetch_view_async + bmb200_result_fetch_wait.  The compacted forms take each column's slot from the host (BIT
columns: the running count of BIT columns; GAP columns: the running sum of ceil((nruns + 1) / 8) * 8 words) while the device
copies as many words as the GAP header says and zero-pads the rest of the slot, and the asynchronous view brings the blocks back
in up to 8 column chunks, one event each.  Every check here compares the fetched arrays word for word with the layout
include/bmb200.h documents, built from the oracle's columns: offsets, BIT blocks, GAP headers with their level bits, run ends
and pad words.  Results of 1, 7, 2047, 2048, 2049 and 2051 (8 x 256 + 3: a short last chunk) columns, batch results that pass
2048 columns only through their groups, all-NULL / all-FULL / all-BIT / all-GAP results, chunks of NULL / FULL columns between
populated ones, and GAP columns at the capacity levels (124 / 125, 252 / 253, 508 / 509 runs) and at the GAP limit."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

import bitmagic_b200 as bm
import gen
import orclib
import rsclib as R
from bitmagic_b200.capi import (BLK_BIT, BLK_FULL, BLK_GAP, BLK_NULL, BLOCK_BITS, BLOCK_WORDS, ERR_BADARG, GAP_THRESHOLD,
                                GAP_UNIT_WORDS, MM_USE_NULL, NO_UNIVERSE, SCAN_IN, TUNE_COVERAGE, mismatch_args)
from bitmagic_b200.hostfmt import BVector, PackedSet, bits_to_gap, bits_to_words, gap_to_bits
from test_launch_variants import REF_OP, raises_code
from test_plane_search_grid import MERGE_RUNS, NPL, P0, MainSet, mm_kw, model_oracle, rank_set, singles_gap, str_queries
from test_scan_in import oracle_scan_in
from test_scan_str import oracle_scan_str
from test_sv_mismatch import oracle_mismatch

pytestmark = pytest.mark.gpu
CMP = bm.F_OPT_COMPRESS
FLAGS = (CMP, 0)

# ------------------------------------------------------------------ the set

NB = 8 * 256 + 3                 # columns of the set: the widest result has a last async chunk shorter than the others
NV = 12                          # vectors 0 .. 11
Z = (770, 1290)                  # only NULL / FULL blocks: chunks 3 and 4 of every 2047 .. 2051-column result lie inside
Z_FULL = (1290, 1300)            # vectors 1 and 2 FULL, the rest NULL
Z_BIT = (1300, 1310)             # every vector but 10, 11 a dense iid bit-block
Z_GAP = (1310, 1320)             # vector 1 a GAP block of a few dozen runs, the rest NULL
RUNS_E = [2, 7, 15, 124, 125, 127, 252, 253, 255, 508, 509, 1271, 1275, 1276, 1277]   # run counts of vector 0's blocks in E, E2
E = (40, 40 + len(RUNS_E))       # vector 0 alone: OR / XOR results with exactly these run counts
E2 = (80, 80 + len(RUNS_E))      # vector 0, vectors 1..9 FULL: AND results with exactly these run counts
M = (120, 120 + 3 * len(MERGE_RUNS))   # vectors 10, 11: GAP singles whose OR / XOR has a run count of MERGE_RUNS
# (lo, hi) column ranges of the result shapes: 1 and 7 columns in E, 2047, 2048, 2049 and 2051 columns
SHAPES = [(45, 46), (40, 47), (0, 2047), (1, 2049), (2, 2051), (0, NB)]
GROUPS = {bm.OP_OR: (list(range(NV)), None), bm.OP_AND: (list(range(10)), None),
          bm.OP_AND_SUB: ([0, 1, 2, 3], [10, 11, 7]), bm.OP_XOR: ([0, 3, 5, 7, 10, 11], None)}


def in_(c, r):
    return r[0] <= c < r[1]


def build_set(seed=8100):
    rng = np.random.default_rng(seed)
    pool = gen.mixed_vectors(rng, 6, 60)
    vecs = [BVector(NB) for _ in range(NV)]
    exact = []
    for r in RUNS_E:
        w = gen.block_with_exact_runs(r)
        exact.append((w, bits_to_gap(w) if r < GAP_THRESHOLD else None))
    for c in range(NB):
        if in_(c, M):                     # the singles of column c, split between vectors 10 and 11 at one cut
            k = c - M[0]
            r = MERGE_RUNS[k % len(MERGE_RUNS)]
            at0 = r % 2 == 0
            pos = 10 + 3 * np.arange((r - 1 - at0) // 2)
            if at0:
                pos = np.concatenate([[0], pos])
            cut = pos.size // 2 if k < len(MERGE_RUNS) else int(rng.integers(max(0, pos.size - 630), min(pos.size, 630) + 1))
        for v, vec in enumerate(vecs):
            if in_(c, Z):
                if (v == 1 and c % 3 == 0) or (v == 2 and c % 5 == 0):
                    vec.set_full(c)
            elif in_(c, Z_FULL):
                if v in (1, 2):
                    vec.set_full(c)
            elif in_(c, Z_BIT):
                if v < 10:
                    vec.set_bits(c, bits_to_words(rng.random(BLOCK_BITS) < 0.5))
            elif in_(c, Z_GAP):
                if v == 1:
                    vec.set_gap(c, bits_to_gap(gen.block_with_runs(rng, int(rng.integers(20, 60)))))
            elif in_(c, E) or in_(c, E2):
                w, g = exact[c - (E[0] if in_(c, E) else E2[0])]
                if v == 0:
                    vec.set_bits(c, w) if g is None else vec.set_gap(c, g)
                elif in_(c, E2) and v < 10:
                    vec.set_full(c)
            elif in_(c, M):
                if v >= 10:
                    vec.set_gap(c, singles_gap(pos[:cut] if v == 10 else pos[cut:]))
            elif v < 10:                  # vectors 10, 11 hold nothing outside M
                src = pool[int(rng.integers(0, len(pool)))]
                nb = int(rng.integers(0, src.n_blocks))
                k = src.kind[nb]
                if k == BLK_FULL:
                    vec.set_full(c)
                elif k == BLK_GAP:
                    vec.set_gap(c, src.blocks[nb])
                elif k == BLK_BIT:
                    vec.set_bits(c, src.blocks[nb])
    return PackedSet.pack(vecs, NB)


@pytest.fixture(scope="module")
def fs(ctx):
    ps = build_set()
    dset = bm.DeviceSet.upload(ctx, ps)
    yield ps, dset
    dset.free()


def agg_oracle(ps, op, flags, lo=0, hi=NB, groups=None):
    g0, g1 = groups if groups is not None else GROUPS[op]
    return orclib.oracle_aggregate(ps, op, g0, g1, flags, lo, hi)


def cat(parts):
    return tuple(np.concatenate([p[i] for p in parts]) for i in range(6))


def sl(o, lo, hi):
    return tuple(x[lo:hi] for x in o)


# ------------------------------------------------------------------ the checks

def chunks(n):
    """Column ranges of the asynchronous view's D2H chunks: 8 of ceil(n / 8) columns from 2048 columns on, else one."""
    nch = 8 if n >= 2048 else 1
    cc = -(-n // nch)
    return [(k * cc, min(n, (k + 1) * cc)) for k in range(nch)]


def layout(kind, nr):
    """The documented compacted layout: off[] of BIT / GAP columns, GAP slot words per column."""
    n = kind.size
    isbit, isgap = kind == BLK_BIT, kind == BLK_GAP
    slot = np.where(isgap, (nr.astype(np.uint64) + 1 + GAP_UNIT_WORDS - 1) // GAP_UNIT_WORDS * GAP_UNIT_WORDS, 0).astype(np.uint64)
    off = np.zeros(n, np.uint64)
    off[isbit] = np.arange(int(isbit.sum()), dtype=np.uint64)
    off[isgap] = (np.cumsum(slot) - slot)[isgap]
    return off, slot


def check_routes(res, o, n_groups=1, what="", nr_oracle=True):
    """Every route of `res` == the oracle columns o = (kind, pop, digest, nruns, blocks[n][2048], gaps[n][1280]) in the
    documented layout.  nr_oracle=False: the oracle's run counts are not compared (its GAP words still fix them)."""
    okind, opop, odig, onr, oblk, ogap = o
    n = res.n_cols
    assert okind.size == n, what
    kind, pop, dig, nr = res.meta()
    assert np.array_equal(kind, okind), f"{what}: kinds"
    assert np.array_equal(pop, opop), f"{what}: popcounts"
    assert np.array_equal(dig, odig), f"{what}: digests"
    if nr_oracle:
        assert np.array_equal(nr, onr), f"{what}: run counts"
    off, slot = layout(kind, nr)
    isbit, isgap, stored = kind == BLK_BIT, kind == BLK_GAP, (kind == BLK_BIT) | (kind == BLK_GAP)
    exp_bits = np.ascontiguousarray(oblk[isbit]).reshape(-1)
    exp_gaps = np.zeros(int(slot.sum()), np.uint16)
    for c in np.flatnonzero(isgap):
        ln = int(ogap[c, 0]) >> 3
        assert ln == nr[c] and ln + 1 <= slot[c], f"{what}: column {c}: GAP length {ln}, nruns {nr[c]}, slot {slot[c]}"
        exp_gaps[int(off[c]):int(off[c]) + ln + 1] = ogap[c, :ln + 1]
    total = int(opop.sum())
    assert int(res.group_totals(n_groups).sum()) == total, f"{what}: group totals"
    nb, ng = res.sizes()
    assert (nb, ng) == (int(isbit.sum()), exp_gaps.size), f"{what}: sizes"

    def same(k, of, bits, gaps, route):
        assert np.array_equal(k, okind), f"{what} [{route}]: kinds"
        assert np.array_equal(of[stored], off[stored]), f"{what} [{route}]: offsets"
        assert bits.size == exp_bits.size and np.array_equal(bits, exp_bits), f"{what} [{route}]: bit-blocks"
        assert gaps.size == exp_gaps.size and np.array_equal(gaps, exp_gaps), f"{what} [{route}]: GAP words"

    # 1) asynchronous view: as soon as the wait for a chunk's last column returns, sample that chunk's blocks (4 words of every
    #    bit-block, every GAP word; last ones first, they land last), then check every chunk against the layout.  What is
    #    sampled is worked out before the view, so that the first wait follows it at once.
    spans = []
    for lo, hi in chunks(n):
        b = lo + np.flatnonzero(isbit[lo:hi]); g = lo + np.flatnonzero(isgap[lo:hi])
        bi = np.arange((int(off[b[-1]]) + 1) * BLOCK_WORDS - 1, int(off[b[0]]) * BLOCK_WORDS - 1, -BLOCK_WORDS // 4) if b.size else None
        gi = np.arange(int(off[g[-1]] + slot[g[-1]]) - 1, int(off[g[0]]) - 1, -1) if g.size else None
        spans.append((hi - 1, bi, gi))
    snaps = []
    k, of, bits, gaps, vnb, vng, vtot = res.fetch_view(wait=False)
    for last, bi, gi in spans:
        res.fetch_wait(last)
        snaps.append((bits[bi] if bi is not None else None, gaps[gi] if gi is not None else None))
    assert np.array_equal(k, okind) and np.array_equal(of[stored], off[stored]), f"{what} [async]: kinds / offsets"
    assert (vnb, vng, vtot) == (nb, ng, total), f"{what} [async]: sizes / total"
    res.fetch_wait(n - 1)
    res.fetch_wait(n + 100)
    for ci, ((lo, hi), (_, bi, gi), (sb, sg)) in enumerate(zip(chunks(n), spans, snaps)):
        if bi is not None:
            assert np.array_equal(sb, exp_bits[bi]), f"{what} [async]: chunk {ci}: bit-blocks at its wait"
        if gi is not None:
            assert np.array_equal(sg, exp_gaps[gi]), f"{what} [async]: chunk {ci}: GAP words at its wait"
        for c in range(lo, hi):
            if isbit[c]:
                s = int(off[c]) * BLOCK_WORDS
                assert np.array_equal(bits[s:s + BLOCK_WORDS], oblk[c]), f"{what} [async]: chunk {ci}: bits of column {c}"
            elif isgap[c]:
                s = int(off[c])
                assert np.array_equal(gaps[s:s + int(slot[c])], exp_gaps[s:s + int(slot[c])]), f"{what} [async]: chunk {ci}: GAP slot of column {c}"
    same(k, of, bits.copy(), gaps.copy(), "async")
    # 2) synchronous view
    k, of, bits, gaps, vnb, vng, vtot = res.fetch_view()
    assert (vnb, vng, vtot) == (nb, ng, total), f"{what} [view]: sizes / total"
    same(k, of, bits, gaps, "view")
    # 3) caller-owned buffers
    same(*res.fetch(), "fetch")
    # 4) one column at a time
    for c in range(n):
        kd, b, g = res.fetch_column(c)
        assert kd == okind[c], f"{what} [column]: kind of column {c}"
        if kd == BLK_BIT:
            assert np.array_equal(b, oblk[c]), f"{what} [column]: bits of column {c}"
        elif kd == BLK_GAP:
            ln = int(ogap[c, 0]) >> 3
            assert np.array_equal(g, ogap[c, :ln + 1]), f"{what} [column]: GAP words of column {c}"
    return kind


def gaps_from_bits(o, kinds):
    """o with the GAP words of the GAP columns of `kinds` rebuilt from the bits (bit_block_to_gap, level from the length)."""
    okind, opop, odig, onr, oblk, ogap = o
    ogap = ogap.copy()
    for c in np.flatnonzero(kinds == BLK_GAP):
        g = bits_to_gap(oblk[c])
        ogap[c, :] = 0
        ogap[c, :g.size] = g
    return kinds, opop, odig, onr, oblk, ogap


def run_counts(o):
    """Run counts of the GAP and BIT columns of an oracle result."""
    okind, _, _, onr, _, _ = o
    return {int(r) for r in onr[okind == BLK_GAP]}, {int(r) for r in onr[okind == BLK_BIT]}


# ------------------------------------------------------------------ producers: aggregate

@pytest.mark.parametrize("op", [bm.OP_OR, bm.OP_AND, bm.OP_AND_SUB, bm.OP_XOR], ids=["or", "and", "and_sub", "xor"])
def test_aggregate_every_shape(ctx, fs, op):
    """bmb200_aggregate (OR / AND / AND-SUB / XOR), F_OPT_COMPRESS and F_OPT_NONE, over 1, 7, 2047, 2048, 2049 and 2051 columns:
    every route == orc_aggregate in the documented layout; the compressed results hold GAP columns at every capacity level."""
    ps, dset = fs
    # the widest shape makes result_compact_kernel's CTAs (sm_count x 8 at most) loop over the columns
    assert max(hi - lo for lo, hi in SHAPES) > ctx.device_info()["sm_count"] * 8
    for flags in FLAGS:
        full = agg_oracle(ps, op, flags)
        if flags == CMP and op in (bm.OP_OR, bm.OP_AND):
            gap_runs, bit_runs = run_counts(full)
            assert {124, 125, 252, 253, 508, 509, 127, 255, 1271, 1275} <= gap_runs and {1276, 1277} <= bit_runs, op
        for lo, hi in SHAPES:
            res = bm.aggregate(ctx, dset, op, *GROUPS[op], flags, lo, hi)
            check_routes(res, sl(full, lo, hi), what=f"op={op} flags={flags} [{lo},{hi})")
            res.free()


def test_aggregate_uniform_results(ctx, fs):
    """All-NULL (nothing stored, nothing in flight), all-FULL, all-BIT and all-GAP results, and a 520-column result of NULL /
    FULL columns only: every route, fetch_wait past the end included."""
    ps, dset = fs
    cases = [(bm.OP_AND, [10, 11], None, CMP, 0, NB, BLK_NULL), (bm.OP_AND, [0, 1], None, 0, 800, 807, BLK_NULL),
             (bm.OP_OR, [1, 2], None, CMP, *Z_FULL, BLK_FULL), (bm.OP_AND, [1], None, CMP, *Z_BIT, BLK_BIT),
             (bm.OP_OR, [1, 3], None, 0, *Z_BIT, BLK_BIT), (bm.OP_OR, [1], None, CMP, *Z_GAP, BLK_GAP),
             (bm.OP_OR, [1, 2], None, CMP, *Z, None)]
    for op, g0, g1, flags, lo, hi, want in cases:
        o = agg_oracle(ps, op, flags, lo, hi, (g0, g1))
        if want is not None:
            assert (o[0] == want).all(), (op, g0, lo, hi)
        else:
            assert set(o[0].tolist()) == {BLK_NULL, BLK_FULL}
        res = bm.aggregate(ctx, dset, op, g0, g1, flags, lo, hi)
        check_routes(res, o, what=f"uniform op={op} {g0} [{lo},{hi})")
        if want == BLK_NULL:
            assert res.sizes() == (0, 0)
            _, _, bits, gaps, nb, ng, tot = res.fetch_view(wait=False)
            assert (bits.size, gaps.size, nb, ng, tot) == (0, 0, 0, 0, 0)
            for c in (0, res.n_cols - 1, res.n_cols + 100):
                res.fetch_wait(c)
        res.free()


def test_async_wait_covers_the_last_chunk(ctx):
    """A 32768-column result whose blocks all sit in its last chunk (4096 bit-blocks, 32 MB; the seven chunks before it hold
    NULL columns only): when fetch_wait(last column) returns, every block has landed.  A wait on the chunk before returns as
    the 32 MB start to cross PCIe, so the host's read right after it would almost always find blocks that have not landed yet
    (a race, not a certainty, but one the host wins by a wide margin)."""
    n, nbit = 8 * 4096, 4096
    rng = np.random.default_rng(8500)
    blocks = rng.integers(0, 2**32, (nbit, BLOCK_WORDS), dtype=np.uint64).astype(np.uint32)
    v = BVector(n)
    for k in range(nbit):
        v.set_bits(n - nbit + k, blocks[k])
    want = blocks.reshape(-1)
    idx = np.arange(want.size - 1, -1, -BLOCK_WORDS // 4)
    dset = bm.DeviceSet.upload(ctx, PackedSet.pack([v], n))
    res = None
    try:
        res = bm.aggregate(ctx, dset, bm.OP_OR, [0], None, CMP)
        kind, of, bits, gaps, nb, ng, tot = res.fetch_view(wait=False)
        res.fetch_wait(n - 1)
        got = bits[idx]
        assert (nb, ng, tot) == (nbit, 0, int(np.bitwise_count(blocks).sum()))
        assert np.array_equal(got, want[idx]), "blocks of the last chunk were read before they landed"
        assert (kind[:n - nbit] == BLK_NULL).all() and (kind[n - nbit:] == BLK_BIT).all()
        assert np.array_equal(of[n - nbit:], np.arange(nbit)) and np.array_equal(bits, want)
    finally:
        if res is not None:
            res.free()
        dset.free()


def test_whole_set_and_sub_coverage_on_and_off(ctx, fs):
    """Whole-set AND-SUB (agg_pipe_kernel) without the coverage plane (TUNE_COVERAGE 0) and on it (2), 2049 and 2051 columns,
    both opt modes: every route == orc_aggregate.  The plane serves AND groups whose members hold no GAP block, so this runs on
    a copy of the set whose AND-group vectors keep their GAP blocks as bit-blocks of the same bits; the plane of |AND group| is
    absent after the first leg and built after the second."""
    ps0, _ = fs
    g0, g1 = [1, 2], [0] + list(range(3, NV))
    vecs = [ps0.vector(v) for v in range(NV)]
    for v in g0:
        for c in np.flatnonzero(vecs[v].kind == BLK_GAP):
            vecs[v].set_bits(int(c), gap_to_bits(vecs[v].blocks[c]))
    ps = PackedSet.pack(vecs, NB)
    assert not (ps.kinds()[:, g0] == BLK_GAP).any() and (ps.kinds()[:, g1] == BLK_GAP).any()
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        for cov in (0, 2):
            ctx.set_tuning(TUNE_COVERAGE, cov)
            for flags in FLAGS:
                full = agg_oracle(ps, bm.OP_AND_SUB, flags, groups=(g0, g1))
                for lo, hi in ((2, NB), (0, NB)):
                    res = bm.aggregate(ctx, dset, bm.OP_AND_SUB, g0, g1, flags, lo, hi)
                    if flags == CMP:
                        assert {BLK_FULL, BLK_BIT, BLK_GAP} <= set(full[0][lo:hi].tolist())
                    check_routes(res, sl(full, lo, hi), what=f"whole-set AND-SUB coverage={cov} flags={flags} [{lo},{hi})")
                    res.free()
            stored, one = dset.coverage(len(g0))
            if cov == 0:
                assert (stored, one) == (0, 0), "a plane was built with TUNE_COVERAGE 0"
            else:
                assert stored > 0, "the AND-SUB calls ran without the coverage plane"
    finally:
        ctx.set_tuning(TUNE_COVERAGE, 1)
        dset.free()


def test_shift_right_and(ctx, fs):
    """OP_SHIFT_R_AND over 2051 and 2048 columns, both opt modes: every route == orc_aggregate."""
    ps, dset = fs
    g = [1, 2, 3]
    for flags in FLAGS:
        full = agg_oracle(ps, bm.OP_SHIFT_R_AND, flags, groups=(g, None))
        for lo, hi in ((0, NB), (1, 2049)):
            res = bm.aggregate(ctx, dset, bm.OP_SHIFT_R_AND, g, None, flags, lo, hi)
            check_routes(res, sl(full, lo, hi), what=f"shift flags={flags} [{lo},{hi})")
            res.free()


def test_batch_and_or_target(ctx, fs):
    """bmb200_aggregate_batch of 3 groups whose flat column count (3 x 700, 3 x 683 = 2049) passes 2048 only through the groups,
    and its OR target: every route == orc_aggregate per group, and == the union through the result rules."""
    ps, dset = fs
    groups = [([0, 1], None), ([2, 3, 4], None), ([10, 11], None)]
    for flags, (lo, hi) in ((CMP, (60, 760)), (0, (1300, 1983)), (CMP, (1300, 1983))):
        per = [agg_oracle(ps, bm.OP_OR, flags, lo, hi, g) for g in groups]
        res = bm.aggregate_batch(ctx, dset, bm.OP_OR, groups, flags | bm.F_OR_TARGET, lo, hi)
        assert res.n_cols == 3 * (hi - lo) > 2048
        check_routes(res, cat(per), 3, what=f"batch flags={flags} [{lo},{hi})")
        union = np.bitwise_or.reduce(np.stack([p[4] for p in per]), axis=0)
        o = res.or_target(hi - lo)
        check_routes(o, model_oracle(list(union), flags), what=f"OR target flags={flags} [{lo},{hi})")
        o.free(); res.free()


# ------------------------------------------------------------------ producers: binop

BINOP_PAIRS = ((0, 1), (10, 11))
BINOP_KINDS = Path(__file__).resolve().parent / "golden" / "result_fetch_binop_kinds.npz"


def binop_key(op, va, vb, compress):
    return f"op{REF_OP[op]}_{va}_{vb}_{int(compress)}"


def ref_binop_kinds(ps):
    """Result kinds of bvector::bit_or / bit_and / bit_sub / bit_xor over the set's operand pairs, both opt modes, from the
    reference library (orclib.ref_binop_gaps)."""
    return {binop_key(op, va, vb, cmp): orclib.ref_binop_gaps(ps, REF_OP[op], va, vb, cmp)[0]
            for op in REF_OP for va, vb in BINOP_PAIRS for cmp in (False, True)}


def record_binop_kinds():
    """(Re)write the recorded kinds from the reference library (the set is rebuilt from its seed), from the repository root:
    PYTHONPATH=.:tests python -c 'import test_result_fetch as t; t.record_binop_kinds()'"""
    np.savez_compressed(BINOP_KINDS, **ref_binop_kinds(build_set()))


@pytest.fixture(scope="module")
def binop_kinds(fs):
    """The reference's kinds: live where its library is built (and then equal to the recorded ones), else the recorded ones."""
    with np.load(BINOP_KINDS) as f:
        rec = {k: f[k] for k in f.files}
    if not orclib.have_ref():
        return rec
    live = ref_binop_kinds(fs[0])
    assert live.keys() == rec.keys() and all(np.array_equal(live[k], rec[k]) for k in live), \
        f"{BINOP_KINDS.name} differs from the reference's kinds; re-record it with record_binop_kinds()"
    return live


@pytest.mark.parametrize("op", list(REF_OP), ids=["or", "and", "sub", "xor"])
def test_binop_every_shape(ctx, fs, binop_kinds, op):
    """bmb200_binop of every op over mixed columns (vectors 0, 1) and over GAP x GAP merges (vectors 10, 11, 1276 runs a GAP
    column, 1277 a bit-block), both opt modes, 1 .. 2051 columns: every route == orc_aggregate's bits in the documented layout,
    kinds == the reference's (binop_kinds)."""
    ps, dset = fs
    aop = bm.OP_AND_SUB if op == bm.capi.OP_SUB else op
    for va, vb in BINOP_PAIRS:
        g = ([va], [vb]) if op == bm.capi.OP_SUB else ([va, vb], None)
        for flags in FLAGS:
            full = agg_oracle(ps, aop, CMP, groups=g)
            ref_kind = binop_kinds[binop_key(op, va, vb, flags == CMP)]
            for lo, hi in (SHAPES if va == 0 else [(M[0], M[1]), (0, NB)]):
                res = bm.capi.binop(ctx, dset, op, va, vb, flags, lo, hi)
                kind = res.meta()[0]
                assert np.array_equal(kind, ref_kind[lo:hi]), f"binop op={op} ({va},{vb}) flags={flags}: kinds vs reference"
                o = sl(full, lo, hi)
                assert ((kind != BLK_NULL) | (o[1] == 0)).all() and ((kind != BLK_FULL) | (o[1] == BLOCK_BITS)).all()
                if va == 10 and op == bm.OP_OR and hi - lo == NB:
                    nr = res.meta()[3]
                    assert {124, 125, 252, 253, 508, 509, 1276} <= set(nr[kind == BLK_GAP].tolist()) and 1277 in nr[kind == BLK_BIT]
                check_routes(res, gaps_from_bits(o, kind), what=f"binop op={op} ({va},{vb}) flags={flags} [{lo},{hi})", nr_oracle=False)
                res.free()


# ------------------------------------------------------------------ producers: scans

def test_scan_every_shape(ctx, fs):
    """bmb200_scan EQ and RANGE over planes 1 .. 9 of the set, both opt modes, 1 .. 2051 columns: every route == orc_scan."""
    ps, dset = fs
    for pred, vals in ((bm.SCAN_EQ, np.array([0], np.uint64)), (bm.SCAN_EQ, np.array([6], np.uint64)),
                       (bm.SCAN_RANGE, np.array([[3, 200]], np.uint64))):
        for flags in FLAGS:
            full = orclib.oracle_scan(ps, pred, vals, 1, 9, NO_UNIVERSE, flags)
            for lo, hi in SHAPES:
                res = bm.scan(ctx, dset, pred, vals, 1, 9, NO_UNIVERSE, flags, lo, hi)
                check_routes(res, sl(full, lo, hi), what=f"scan pred={pred} {vals.tolist()} flags={flags} [{lo},{hi})")
                res.free()


@pytest.fixture(scope="module")
def planes(ctx):
    ms = MainSet(300, seed=8200, sample=4)
    dset = bm.DeviceSet.upload(ctx, ms.ps[True])
    yield ms, dset
    dset.free()


def test_plane_searches(ctx, planes):
    """SCAN_IN, scan_str (7 queries x 293 columns = 2051 columns) and sv_mismatch over the plane-search set, both opt modes:
    every route == orc_scan_in / orc_scan_str / orc_sv_mismatch."""
    ms, dset = planes
    ps = ms.ps[True]
    rng = np.random.default_rng(8300)
    lst = np.unique(np.concatenate([ms.eq_values(rng, 5), ms.pool[rng.integers(0, ms.pool.size, 40)]]))
    q = str_queries(ms, rng, 7, False)
    for flags in FLAGS:
        res = bm.scan(ctx, dset, SCAN_IN, lst, P0, NPL, 0, flags, 1, 300)
        check_routes(res, oracle_scan_in(ps, lst, P0, NPL, 0, flags, 1, 300), what=f"SCAN_IN flags={flags}")
        res.free()
        res = bm.scan_str(ctx, dset, q, P0, NPL, NO_UNIVERSE, flags, nb_from=3, nb_to=296)
        assert res.n_cols == 2051
        check_routes(res, oracle_scan_str(ps, q, P0, NPL, NO_UNIVERSE, flags, 3, 296), 7, what=f"scan_str flags={flags}")
        res.free()
        a = mismatch_args(**mm_kw(ms), null_proc=MM_USE_NULL, flags=flags, nb_from=0, nb_to=300)
        res = bm.sv_mismatch(ctx, dset, a)
        check_routes(res, oracle_mismatch(ps, a), what=f"sv_mismatch flags={flags}")
        res.free()


# ------------------------------------------------------------------ producers: rank compression

def test_rank_decompress_and_compress(ctx):
    """bmb200_rank_decompress of a 2-group source (2 x 1025 columns) and bmb200_rank_compress, both opt modes: every route ==
    the numpy rank compressor through orc_aggregate's result rules."""
    n = 1025
    vecs, nn_bits, src_bits = rank_set(n, seed=8400)
    dset = bm.DeviceSet.upload(ctx, PackedSet.pack(vecs, n))
    rs = bm.DeviceRS(ctx, dset, 0)
    src = bm.aggregate_batch(ctx, dset, bm.OP_OR, [([1], []), ([2], [])], CMP)
    want = []
    for s in (np.concatenate(src_bits[0]), np.concatenate(src_bits[1])):
        r = 0
        for c in range(n):
            cnt = int(nn_bits[c].sum())
            want.append(R.words_of(R.np_rank_decompress(nn_bits[c], s[r:r + cnt]), 1))
            r += cnt
    total = sum(int(b.sum()) for b in nn_bits)
    ncomp = -(-total // BLOCK_BITS)
    comp = R.words_of(np.concatenate([R.np_rank_compress(nn_bits[c], src_bits[2][c]) for c in range(n)]), ncomp).reshape(ncomp, -1)
    for flags in FLAGS:
        out = bm.rank_decompress(ctx, rs, src, flags)
        assert out.n_cols == 2 * n
        check_routes(out, model_oracle(want, flags), 2, what=f"rank_decompress flags={flags}")
        out.free()
        out = bm.rank_compress(ctx, rs, 3, flags)
        check_routes(out, model_oracle(list(comp), flags), what=f"rank_compress flags={flags}")
        out.free()
    src.free(); rs.free(); dset.free()


# ------------------------------------------------------------------ state across calls

def test_recycled_result_every_route(ctx, fs):
    """One result handle recycled through producers of other shapes: 2051 columns then 7, compress on then off, a 3-group batch
    then a single aggregate, a scan then a binop of the same shape, each after an asynchronous view of the previous answer:
    every route returns the fresh answer."""
    ps, dset = fs
    g = GROUPS[bm.OP_OR]
    steps = [
        (lambda r: bm.aggregate(ctx, dset, bm.OP_OR, *g, CMP, 0, NB, result=r), lambda: agg_oracle(ps, bm.OP_OR, CMP), 1),
        (lambda r: bm.aggregate(ctx, dset, bm.OP_XOR, *GROUPS[bm.OP_XOR], CMP, 0, NB, result=r), lambda: agg_oracle(ps, bm.OP_XOR, CMP), 1),
        (lambda r: bm.aggregate(ctx, dset, bm.OP_OR, *g, 0, 0, NB, result=r), lambda: agg_oracle(ps, bm.OP_OR, 0), 1),
        (lambda r: bm.aggregate(ctx, dset, bm.OP_AND, *GROUPS[bm.OP_AND], CMP, 80, 87, result=r),
         lambda: agg_oracle(ps, bm.OP_AND, CMP, 80, 87), 1),
        (lambda r: bm.aggregate_batch(ctx, dset, bm.OP_OR, [([0], None), ([1], None), ([2], None)], CMP, 1, 684, result=r),
         lambda: cat([agg_oracle(ps, bm.OP_OR, CMP, 1, 684, ([v], None)) for v in (0, 1, 2)]), 3),
        (lambda r: bm.aggregate(ctx, dset, bm.OP_OR, *g, CMP, 0, 2049, result=r), lambda: agg_oracle(ps, bm.OP_OR, CMP, 0, 2049), 1),
        (lambda r: bm.scan(ctx, dset, bm.SCAN_EQ, [0], 1, 9, NO_UNIVERSE, CMP, 0, 2049, result=r),
         lambda: orclib.oracle_scan(ps, bm.SCAN_EQ, [0], 1, 9, NO_UNIVERSE, CMP, 0, 2049), 1),
        (lambda r: bm.aggregate(ctx, dset, bm.OP_AND, [10, 11], None, CMP, 0, 2049, result=r),
         lambda: agg_oracle(ps, bm.OP_AND, CMP, 0, 2049, ([10, 11], None)), 1),
    ]
    r = None
    for i, (call, oracle, ng) in enumerate(steps):
        if r is not None:
            r.fetch_view(wait=False)          # the previous answer's view, waited for before the next call as the contract asks
            r.fetch_wait(r.n_cols - 1)
        r = call(r)
        check_routes(r, oracle(), ng, what=f"recycle step {i}")
    r.free()


def test_two_views_alternate_pinned_buffers(ctx, fs):
    """An asynchronous view of one result, waited for, then a view of another: the second view lands in the other pinned block
    buffer, so the first view's blocks still read as its own result."""
    ps, dset = fs
    a = bm.aggregate(ctx, dset, bm.OP_OR, *GROUPS[bm.OP_OR], CMP, 0, NB)
    b = bm.aggregate(ctx, dset, bm.OP_OR, *GROUPS[bm.OP_OR], CMP, *E)
    oa, ob = agg_oracle(ps, bm.OP_OR, CMP), agg_oracle(ps, bm.OP_OR, CMP, *E)
    na, nb_ = a.sizes(), b.sizes()
    assert na[0] >= nb_[0] > 0 and na[1] >= nb_[1] > 0   # b fits in a's buffers, so neither view needs new ones
    for first_async in (True, False):
        b.fetch_view()                        # both pinned buffers at least this large before the views that are compared
        a.fetch_view()
        ka, offa, bitsa, gapsa, _, _, _ = a.fetch_view(wait=not first_async)
        a.fetch_wait(a.n_cols - 1)
        ka, offa = ka.copy(), offa.copy()     # kind / off live in the one meta buffer every view shares
        want_bits = np.ascontiguousarray(oa[4][ka == BLK_BIT]).reshape(-1)
        assert np.array_equal(bitsa, want_bits)
        kb, offb, bitsb, gapsb, _, _, _ = b.fetch_view(wait=False)
        b.fetch_wait(b.n_cols - 1)
        assert np.array_equal(bitsb, np.ascontiguousarray(ob[4][kb == BLK_BIT]).reshape(-1)), "second view"
        if first_async:
            assert np.array_equal(bitsa, want_bits), "the second view overwrote the first view's blocks"
            gs = np.flatnonzero(ka == BLK_GAP)
            for c in gs:
                s = int(offa[c]); ln = int(oa[5][c, 0]) >> 3
                assert np.array_equal(gapsa[s:s + ln + 1], oa[5][c, :ln + 1]), f"the second view overwrote GAP column {c}"
    a.free(); b.free()


def test_optimize_is_idempotent(ctx, fs):
    """optimize() twice before any fetch changes nothing (compress results, a GAP-merging binop, an OR target); it refuses an
    F_OPT_NONE result and a COUNT_ONLY one with BADARG."""
    ps, dset = fs
    res = bm.aggregate(ctx, dset, bm.OP_OR, *GROUPS[bm.OP_OR], CMP, 0, NB)
    res.optimize(); res.optimize()
    check_routes(res, agg_oracle(ps, bm.OP_OR, CMP), what="optimized OR")
    res.free()
    res = bm.aggregate_batch(ctx, dset, bm.OP_OR, [([0], None), ([1], None), ([2], None)], CMP | bm.F_OR_TARGET, 1, 684)
    res.optimize()
    o = res.or_target(683)
    o.optimize(); o.optimize()
    union = np.bitwise_or.reduce(np.stack([agg_oracle(ps, bm.OP_OR, CMP, 1, 684, ([v], None))[4] for v in (0, 1, 2)]), axis=0)
    check_routes(o, model_oracle(list(union), CMP), what="optimized OR target")
    o.free(); res.free()
    res = bm.capi.binop(ctx, dset, bm.OP_XOR, 10, 11, CMP)
    res.optimize(); res.optimize()
    full = agg_oracle(ps, bm.OP_XOR, CMP, groups=([10, 11], None))
    check_routes(res, gaps_from_bits(full, res.meta()[0]), what="optimized binop", nr_oracle=False)
    res.free()
    for flags in (0, bm.F_COUNT_ONLY, bm.F_COUNT_ONLY | CMP):
        res = bm.aggregate(ctx, dset, bm.OP_OR, *GROUPS[bm.OP_OR], flags)
        raises_code(ERR_BADARG, res.optimize)
        res.free()


def test_count_only_and_null_out_pointers(ctx, fs):
    """Every fetch route of a COUNT_ONLY result (also one recycled from a stored result with a view in flight), and a view with
    any of its four out pointers NULL, return BADARG."""
    ps, dset = fs
    stored = bm.aggregate(ctx, dset, bm.OP_OR, *GROUPS[bm.OP_OR], CMP, 0, NB)
    stored.fetch_view(wait=False)
    stored.fetch_wait(NB - 1)
    for op, flags, into in ((bm.OP_OR, CMP, stored), (bm.OP_AND, 0, None)):
        res = bm.aggregate(ctx, dset, op, *GROUPS[op], bm.F_COUNT_ONLY | flags, result=into)
        assert res.total()[0] == int(agg_oracle(ps, op, flags)[1].sum())
        raises_code(ERR_BADARG, res.fetch)
        raises_code(ERR_BADARG, res.sizes)
        raises_code(ERR_BADARG, res.fetch_column, 0)
        raises_code(ERR_BADARG, res.fetch_view)
        raises_code(ERR_BADARG, res.fetch_view, False)
        res.free()
    res = bm.aggregate(ctx, dset, bm.OP_OR, *GROUPS[bm.OP_OR], CMP, 0, 7)
    lib = bm.capi.lib()
    for fn in (lib.bmb200_result_fetch_view, lib.bmb200_result_fetch_view_async):
        for k in range(4):
            outs = [C.c_void_p(0) for _ in range(4)]
            args = [None if j == k else C.byref(outs[j]) for j in range(4)]
            assert fn(res._h, *args, None, None, None) == ERR_BADARG, (fn, k)
    check_routes(res, agg_oracle(ps, bm.OP_OR, CMP, 0, 7), what="after the refused views")
    res.free()
