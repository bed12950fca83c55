"""Whole-set AND-SUB aggregations (group0 + group1 name every vector once) take the streamed-column kernel; tuning key
TUNE_AGG_PIPELINE = 0 keeps them on the general kernel.  Both paths must agree bit for bit with each other and with the oracle:
blocks, GAP words, kinds, popcounts, digests, run counts and totals."""
import numpy as np
import pytest

import bitmagic_b200 as bm
import gen
import orclib

pytestmark = pytest.mark.gpu

C = bm.F_OPT_COMPRESS


def run(ctx, dset, op, g0, g1, flags, nb_from, nb_to):
    res = bm.aggregate(ctx, dset, op, g0, g1, flags, nb_from, nb_to)
    kind, pop, dig, nr = res.meta()
    total, any_ = res.total()
    fk, off, bits, gaps = res.fetch()
    bv = bm.result_to_bvector(fk, off, bits, gaps)
    blocks = np.stack([bv.block_words(c) for c in range(kind.size)])
    gflat = np.concatenate([bv.blocks[c] for c in range(kind.size) if kind[c] == bm.BLK_GAP]) \
        if (kind == bm.BLK_GAP).any() else np.zeros(0, np.uint16)
    res.free()
    return dict(kind=kind, pop=pop, dig=dig, nr=nr, total=total, any=any_, blocks=blocks, gflat=gflat)


def check_paths(ctx, ps, op, g0, g1, flags, nb_from=0, nb_to=0):
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, 1)
        new = run(ctx, dset, op, g0, g1, flags, nb_from, nb_to)
        ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, 0)
        old = run(ctx, dset, op, g0, g1, flags, nb_from, nb_to)
    finally:
        ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, 1)
        dset.free()
    for k in new:
        assert np.array_equal(np.asarray(new[k]), np.asarray(old[k])), k
    hi = nb_to or ps.n_blocks
    okind, opop, odig, onr, oblk, ogap = orclib.oracle_aggregate(ps, op, g0, g1, flags, nb_from, hi)
    assert np.array_equal(new["blocks"], oblk)
    assert np.array_equal(new["kind"], okind)
    assert np.array_equal(new["pop"], opop)
    assert np.array_equal(new["dig"], odig)
    assert np.array_equal(new["nr"], onr)
    assert new["total"] == int(opop.sum()) and new["any"] == bool(opop.sum())
    glen = np.where(okind == bm.BLK_GAP, (ogap[:, 0] >> 3) + 1, 0)
    oflat = np.concatenate([ogap[c, :glen[c]] for c in range(len(okind))]) if glen.sum() else np.zeros(0, np.uint16)
    assert np.array_equal(new["gflat"], oflat)


def whole_set_groups(rng, op, n):
    perm = rng.permutation(n)
    na = int(rng.integers(1, min(n, 4) + 1))
    return perm[:na], perm[na:]


@pytest.mark.parametrize("n_vec", [3, 17, 1024, 1500, 4096])
def test_whole_set_paths_agree(ctx, n_vec):
    """Mixed block kinds; the AND group (1-4 random vectors) usually holds GAP blocks, whose 0-runs the streamed path applies in
    place while it blanks them in the staged segment.  Raw-form sets keep agg_kernel in both arms (the selection rule)."""
    op = bm.OP_AND_SUB
    rng = np.random.default_rng(1000 * op + n_vec)
    n_blocks = 5 if n_vec < 1024 else 2
    vecs = gen.mixed_vectors(rng, n_vec, n_blocks, p_null=0.04, p_full=0.03)
    g0, g1 = whole_set_groups(rng, op, n_vec)
    for gap_flat in (True, False):
        ps = bm.PackedSet.pack(vecs, gap_flat=gap_flat)
        for flags in (0, C):
            check_paths(ctx, ps, op, g0, g1, flags)


def test_whole_set_many_columns(ctx):
    """More columns than SMs (every CTA streams several columns back to back) and columns of more stages than the ring holds
    (~24 bit-blocks and more than 16 stages of GAP blocks per column)."""
    op = bm.OP_AND_SUB
    rng = np.random.default_rng(5 + op)
    vecs = [bm.BVector.random(300, 0.5 / (k + 1) if k < 24 else 0.003 * (k % 3 + 1), rng).optimize() for k in range(112)]
    ps = bm.PackedSet.pack(vecs)
    assert ps.bit_base[1] - ps.bit_base[0] > 16 and (ps.gap_base[1] - ps.gap_base[0]) * 16 > 16 * 8192
    n = len(vecs)
    for g0 in ([0, 1], [0, 60]):             # AND group of bit-blocks only (pure FLAT window); one with a GAP vector in it
        g1 = [v for v in rng.permutation(n) if v not in g0]
        check_paths(ctx, ps, op, g0, g1, C)
        check_paths(ctx, ps, op, g0, g1, 0, 37, 0)


def test_whole_set_shapes(ctx):
    """Edge blocks (all-zero / all-one GAP, first-run-1 blocks, FULL, NULL), columns with no bit-blocks or no GAP blocks,
    an AND group of GAP blocks, sub-ranges starting past column 0, sets whose row length is not a multiple of 4."""
    op = bm.OP_AND_SUB
    rng = np.random.default_rng(77 + op)
    n_blocks = 6
    vecs = gen.edge_vectors(n_blocks) + gen.mixed_vectors(rng, 9, n_blocks, p_null=0.1, p_full=0.05, p_gap=0.5)
    for v in gen.mixed_vectors(rng, 6, n_blocks, p_null=0.0, p_full=0.0, p_gap=1.0):     # GAP-only vectors
        vecs.append(v)
    vecs += gen.mixed_vectors(rng, 2, n_blocks, p_null=0.0, p_full=0.0, p_gap=0.0)       # bit-only vectors (the FLAT-window AND group)
    for v in vecs:                                                                       # column 2: no GAP blocks, column 3: no bit-blocks
        if v.kind[2] == bm.BLK_GAP:
            v.set_bits(2, v.block_words(2))
        if v.kind[3] == bm.BLK_BIT:
            v.kind[3] = bm.BLK_NULL
            v.blocks.pop(3, None)
    n = len(vecs)
    ps = bm.PackedSet.pack(vecs)
    for g0 in ([n - 2, n - 1], [n - 8, n - 7]):               # AND group of bit-only vectors, then of GAP-only vectors
        g1 = [v for v in rng.permutation(n) if v not in g0]
        for nb_from, nb_to in ((0, 0), (1, 0), (2, 5), (5, 6)):
            check_paths(ctx, ps, op, g0, g1, C, nb_from, nb_to)
