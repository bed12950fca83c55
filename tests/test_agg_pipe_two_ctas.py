"""The whole-set AND-SUB kernel runs two CTAs per SM, each with 8 consumer warps, an 8-stage ring cut among 4 warp groups, and 8
words of the live mask per thread.  Around that shape: grids of 1, SMs - 1, 2 SMs - 1, 2 SMs, 2 SMs + 1 and more columns than
CTAs with nb_from > 0; 4096 vectors (16 descriptors per consumer thread); an AND group with GAP blocks (the FLAT GAP-segment path
with AND-group blanking); count-only calls and a one-group batch with an OR target; columns of 0, 1, 3, 4, 5 and 9 companion
stages around the 4 warp groups.  Every case must agree bit for bit with the general kernel (TUNE_AGG_PIPELINE 0) and the oracle."""
import numpy as np
import pytest

import bitmagic_b200 as bm
import gen
import orclib
from test_agg_pipeline import run
from test_agg_pipe_stages import STAGE, singles_for, singles_set

pytestmark = pytest.mark.gpu

C = bm.F_OPT_COMPRESS
OP = bm.OP_AND_SUB


def both_paths(ctx, ps, g0, g1, flags, nb_from=0, nb_to=0, run_lists=(0, 2)):
    """Streamed kernel under each TUNE_RUN_LISTS value and the general kernel: every output equal, and equal to the oracle."""
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        new = []
        for rl in run_lists:
            ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, rl)
            new.append(run(ctx, dset, OP, g0, g1, flags, nb_from, nb_to))
        ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, 0)
        old = run(ctx, dset, OP, g0, g1, flags, nb_from, nb_to)
    finally:
        ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, 1)
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)
        dset.free()
    for rl, got in zip(run_lists, new):
        for k in got:
            assert np.array_equal(np.asarray(got[k]), np.asarray(old[k])), (rl, k)
    okind, opop, odig, onr, oblk, ogap = orclib.oracle_aggregate(ps, OP, g0, g1, flags, nb_from, nb_to or ps.n_blocks)
    assert np.array_equal(old["blocks"], oblk)
    assert np.array_equal(old["kind"], okind) and np.array_equal(old["pop"], opop)
    assert np.array_equal(old["dig"], odig) and np.array_equal(old["nr"], onr)
    return old


def sparse_set(rng, n_blocks, n_sub=6):
    """Two dense bit-block vectors (the AND group) and SUB-group vectors of GAP and bit-blocks."""
    vecs = [bm.BVector.random(n_blocks, 0.5, rng), bm.BVector.random(n_blocks, 0.6, rng)]
    vecs += [bm.BVector.random(n_blocks, (0.002, 0.01, 0.05, 0.2)[k % 4], rng).optimize() for k in range(n_sub)]
    return vecs


def test_grid_edges(ctx):
    """Grids of 1 column, SMs - 1, 2 SMs - 1, 2 SMs, 2 SMs + 1 and 3 SMs + 7 columns (more than the resident CTAs), starting at
    column 3."""
    sms = ctx.device_info()["sm_count"]
    nb_from = 3
    rng = np.random.default_rng(901)
    ps = bm.PackedSet.pack(sparse_set(rng, nb_from + 3 * sms + 7))
    n = ps.n_vec
    for cols in (1, sms - 1, 2 * sms - 1, 2 * sms, 2 * sms + 1, 3 * sms + 7):
        res = both_paths(ctx, ps, [0, 1], list(range(2, n)), C, nb_from, nb_from + cols)
        assert res["kind"].size == cols and res["pop"].sum() > 0


def test_4096_vectors(ctx):
    """16 descriptors per consumer thread: AND groups of bit-blocks only (companion or FLAT segment) and with a GAP vector in the
    last classification trip."""
    rng = np.random.default_rng(902)
    vecs = gen.mixed_vectors(rng, 4096, 2, p_null=0.05, p_full=0.01, p_gap=0.6)
    vecs[0] = bm.BVector.random(2, 0.7, rng)
    vecs[4095] = bm.BVector.random(2, 0.8, rng)
    ps = bm.PackedSet.pack(vecs)
    gap_vec = next(v for v in range(4095, 3839, -1) if (ps.desc[v::ps.n_vec] & 3 == bm.BLK_GAP).all())
    for g0 in ([0, 4095], [0, gap_vec]):
        g1 = [v for v in range(4096) if v not in g0]
        both_paths(ctx, ps, g0, g1, C)


def test_and_group_gap_blocks(ctx):
    """An AND group holding GAP blocks (as AND = {1, 601} on the bench's data): GAP segments streamed in FLAT form with the
    AND-group blocks applied in place and blanked in the stages, over more columns than CTAs."""
    sms = ctx.device_info()["sm_count"]
    rng = np.random.default_rng(903)
    vecs = sparse_set(rng, 2 * sms + 40, n_sub=10)
    ps = bm.PackedSet.pack(vecs)
    assert (ps.desc[7::ps.n_vec] & 3 == bm.BLK_GAP).any()
    n = ps.n_vec
    both_paths(ctx, ps, [0, 7], [v for v in range(n) if v not in (0, 7)], C, 5, 0)


def test_count_only_and_or_target_batch(ctx):
    """F_COUNT_ONLY, and a one-group batch with C | OR_TARGET: popcounts, digests, kinds, totals and the OR target agree between
    the two kernels and with the oracle."""
    sms = ctx.device_info()["sm_count"]
    rng = np.random.default_rng(904)
    ps = bm.PackedSet.pack(sparse_set(rng, 2 * sms + 3))
    n = ps.n_vec
    g0, g1 = [0, 1], list(range(2, n))
    okind, opop, odig, onr, oblk, ogap = orclib.oracle_aggregate(ps, OP, g0, g1, C, 0, ps.n_blocks)
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        for pipe in (1, 0):
            ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, pipe)
            res = bm.aggregate(ctx, dset, OP, g0, g1, bm.F_COUNT_ONLY)
            kind, pop, dig, nr = res.meta()
            assert np.array_equal(pop, opop) and res.total()[0] == int(opop.sum()), pipe
            res.free()
            res = bm.aggregate_batch(ctx, dset, OP, [(g0, g1)], C | bm.F_OR_TARGET)
            kind, pop, dig, nr = res.meta()
            assert np.array_equal(kind, okind) and np.array_equal(pop, opop) and np.array_equal(dig, odig), pipe
            o = res.or_target(ps.n_blocks)
            bv = bm.result_to_bvector(*o.fetch())
            assert np.array_equal(np.stack([bv.block_words(c) for c in range(ps.n_blocks)]), oblk), pipe
            o.free(); res.free()
    finally:
        ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, 1)
        dset.free()


def test_companion_stages_around_the_groups(ctx):
    """Columns of 0, 1, 3, 4, 5 and 9 companion stages (fewer, as many as, and more than the 4 warp groups; more than the
    8-stage ring), partial and full last stages, repeated over more columns than CTAs so the ring wraps at every offset."""
    sms = ctx.device_info()["sm_count"]
    rng = np.random.default_rng(905)
    shape = [(0, 0), (1, 16), (3, 528), (4, STAGE), (5, 4096), (9, 8176), (4, 4112), (5, 16)]
    per_col = [singles_for(*shape[c % len(shape)]) for c in range(2 * sms + 11)]
    ps = bm.PackedSet.pack(singles_set(rng, per_col))
    n = ps.n_vec
    both_paths(ctx, ps, [0, 1], list(range(2, n)), C, run_lists=(2,))
