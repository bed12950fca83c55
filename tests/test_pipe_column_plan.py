"""The whole-set AND-SUB kernel's column plan: with the run-list companion, the producer warp decides from the AND-group members alone
(and the companion's per-column FULL count) which streamed stages are AND-group bit-blocks, how many there are and the result
state, and the consumers never read the column's descriptor row.  Columns whose AND members are NULL, FULL or bit-blocks, whose SUB
group holds a FULL block, whose AND members' bit-blocks sit behind listed (unstreamed) blocks, AND groups of 1 and 64 members given
out of vector order, the last stream index of a 4096-vector column, sub-ranges, count-only calls and C3's generator must agree bit
for bit with the companion switched off, with the general kernel and with the oracle."""
import numpy as np
import pytest

import bitmagic_b200 as bm
from bitmagic_b200.hostfmt import bits_to_gap, bits_to_words, BLOCK_BITS
from test_run_list_union import WORDS, check

pytestmark = pytest.mark.gpu

C = bm.F_OPT_COMPRESS
N_COLS = 10


def sparse_words(rng, n):
    """n isolated bits at even positions: a bit-block the companion lists in part B."""
    return bits_to_words(np.isin(np.arange(BLOCK_BITS), 2 * rng.choice(BLOCK_BITS // 2, n, replace=False)).astype(np.uint8))


def gap_block(rng, n):
    bits = np.zeros(BLOCK_BITS, np.uint8)
    bits[2 * rng.choice(BLOCK_BITS // 2, n, replace=False)] = 1
    return bits_to_gap(bits_to_words(bits))


def drop(v, c):
    v.kind[c] = bm.BLK_NULL
    v.blocks.pop(c)


def plan_set(rng, n_and, and_density):
    """Listed sparse vectors and GAP vectors interleaved with n_and dense AND-group candidates (so every AND member's bit-block has
    listed blocks below it in the column's bit pool), one dense SUB vector and one SUB vector NULL except where a column makes it
    FULL.  Returns (vectors, AND member ids in descending order).
      column 1: AND member a NULL            column 2: AND member a FULL
      column 3: the SUB vector FULL          column 4: every AND member FULL (no AND-group bit-block)
      column 5: every AND member FULL and the SUB vector FULL
      column 6: AND member a NULL and the SUB vector FULL
      column 7: AND member b FULL            columns 0, 8, 9: plain"""
    vecs, and_ids = [], []
    for k in range(n_and):
        for _ in range(2):
            sv = bm.BVector(N_COLS)
            for c in range(N_COLS):
                if rng.random() < 0.8:
                    sv.set_bits(c, sparse_words(rng, int(rng.integers(50, 400))))
            vecs.append(sv)
        gv = bm.BVector(N_COLS)
        for c in range(N_COLS):
            gv.set_gap(c, gap_block(rng, int(rng.integers(20, 300))))
        vecs.append(gv)
        and_ids.append(len(vecs))
        vecs.append(bm.BVector.random(N_COLS, and_density, rng))
    vecs.append(bm.BVector.random(N_COLS, 0.05, rng))
    sub_full = bm.BVector(N_COLS)
    for c in (3, 5, 6):
        sub_full.set_full(c)
    vecs.append(sub_full)
    a, b = vecs[and_ids[0]], vecs[and_ids[-1]]
    drop(a, 1); a.set_full(2)
    for i in and_ids:
        vecs[i].set_full(4); vecs[i].set_full(5)
    drop(a, 6)
    if b is not a:
        b.set_full(7)
    return vecs, and_ids[::-1]


@pytest.mark.parametrize("n_and", [1, 2, 64])
def test_plan_member_kinds(ctx, n_and):
    rng = np.random.default_rng(4100 + n_and)
    vecs, g0 = plan_set(rng, n_and, 0.5 if n_and <= 2 else 0.9)
    ps = bm.PackedSet.pack(vecs)
    g1 = [int(v) for v in rng.permutation([v for v in range(len(vecs)) if v not in g0])]
    check(ctx, ps, g0, g1, C)
    check(ctx, ps, g0, g1, 0, 2, 8)
    check(ctx, ps, g0, g1, bm.F_COUNT_ONLY, 1, 0)


def test_plan_last_stream_index(ctx):
    """4096 vectors in one column: 4095 unlisted bit-blocks and a GAP block, so the union mask is stage 4095 and the AND group
    holds the column's first and last streamed bit-block (indices 0 and 4094)."""
    rng = np.random.default_rng(4199)
    vecs = []
    for v in range(4095):
        w = rng.integers(0, 1 << 32, WORDS, dtype=np.uint32)
        if v not in (0, 4094):
            w[:WORDS // 2] = 0
        bv = bm.BVector(1); bv.set_bits(0, w); vecs.append(bv)
    bits = np.zeros(BLOCK_BITS, np.uint8)
    bits[32 * rng.choice(WORDS // 2, 600, replace=False) + rng.integers(1, 31, 600)] = 1
    g = bm.BVector(1); g.set_gap(0, bits_to_gap(bits_to_words(bits))); vecs.append(g)
    ps = bm.PackedSet.pack(vecs)
    assert check(ctx, ps, [4094, 0], [v for v in range(4096) if v not in (0, 4094)], C) == (1, 1)


def test_plan_c3_recipe(ctx):
    """C3's generator over 64 columns with its AND group (vectors 0 and 1; bench.py counts from 1): the companion path equals the
    streamed kernel without it and the general kernel, whole and uncompressed over a sub-range."""
    import bench
    from test_run_lists import run
    dens, seed, opt = bench.workload_inputs("c3", 0)
    n_vec, n_cols = 1024, 64
    dset = bm.DeviceSet.synth(ctx, n_vec, n_cols, dens, seed, opt)
    g0, g1 = [0, 1], np.arange(2, n_vec, dtype=np.uint32)
    got = []
    try:
        for pipe, rl in ((1, 2), (1, 0), (0, 0)):
            ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, pipe)
            ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, rl)
            got.append(run(ctx, dset, g0, g1, C, 0, 0))
            got.append(run(ctx, dset, g0, g1, 0, 5, 40))
        assert dset.run_list_unions() == (n_cols, n_cols)
    finally:
        ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, 1)
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)
        dset.free()
    for i in (2, 4):
        for j in (0, 1):
            for k in got[j]:
                assert np.array_equal(np.asarray(got[i + j][k]), np.asarray(got[j][k])), (i, j, k)
