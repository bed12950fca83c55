"""Coverage planes of the whole-set AND-SUB kernel: for an AND group of n0 members holding no GAP block, the kernel streams the AND
members' bit-blocks and the set's plane GT_n0 = {x : more than n0 vectors hold x}, folded as a SUB-group bit-block, in place of the
SUB group.  Each case runs four ways -- the plane (TUNE_COVERAGE 2), no plane with the run-list companion and without it, the
general kernel -- and against the oracle, bit for bit on kinds, popcounts, digests, GAP lengths, blocks and totals; the plane's
stored and everywhere-covered columns must equal a host count of cnt > n0."""
import numpy as np
import pytest

import bitmagic_b200 as bm
import orclib
from bitmagic_b200.hostfmt import bits_to_gap, bits_to_words, gap_to_bits, words_to_bits, BLOCK_BITS
from test_pipe_column_plan import plan_set, sparse_words
from test_run_list_union import outputs

pytestmark = pytest.mark.gpu

C = bm.F_OPT_COMPRESS
OP = bm.OP_AND_SUB
WAYS = (("coverage", 1, 0, 2), ("companion", 1, 2, 0), ("segments", 1, 0, 0), ("agg_kernel", 0, 0, 0))


def tune(ctx, pipe=1, rl=1, cov=1):
    ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, pipe)
    ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, rl)
    ctx.set_tuning(bm.capi.TUNE_COVERAGE, cov)


def host_coverage(ps, n0):
    """(stored columns, everywhere-covered columns) of GT_n0, counted on the host."""
    stored = one = 0
    for nb in range(ps.n_blocks):
        cnt = np.zeros(BLOCK_BITS, np.int64)
        for v in range(ps.n_vec):
            k, data = ps.block(v, nb)
            if k == bm.BLK_FULL:
                cnt += 1
            elif k == bm.BLK_BIT:
                cnt += words_to_bits(data)
            elif k == bm.BLK_GAP:
                cnt += words_to_bits(gap_to_bits(data))
        gt = cnt > n0
        one += int(gt.all()); stored += int(gt.any() and not gt.all())
    return stored, one


def want(ps, g0, g1, flags, nb_from, nb_to):
    hi = nb_to or ps.n_blocks
    okind, opop, odig, onr, oblk, ogap = orclib.oracle_aggregate(ps, OP, g0, g1, flags & ~bm.F_COUNT_ONLY, nb_from, hi)
    glen = np.where(okind == bm.BLK_GAP, (ogap[:, 0] >> 3) + 1, 0)
    oflat = np.concatenate([ogap[c, :glen[c]] for c in range(len(okind))]) if glen.sum() else np.zeros(0, np.uint16)
    return dict(pop=opop, total=int(opop.sum()), any=bool(opop.sum()), kind=okind, dig=odig, nr=onr, gflat=oflat, blocks=oblk)


def four_ways(ctx, dset, g0, g1, flags, nb_from=0, nb_to=0):
    got = {}
    try:
        for name, pipe, rl, cov in WAYS:
            tune(ctx, pipe, rl, cov)
            got[name] = outputs(ctx, dset, g0, g1, flags, nb_from, nb_to)
    finally:
        tune(ctx)
    return got


def check(ctx, ps, g0, g1, flags, nb_from=0, nb_to=0, dset=None, used=True):
    """The four ways and the oracle agree; the plane of |g0| is built (used) or not, with the host's column counts."""
    own = dset is None
    if own:
        dset = bm.DeviceSet.upload(ctx, ps)
    try:
        got = four_ways(ctx, dset, g0, g1, flags, nb_from, nb_to)
        built = dset.coverage(len(g0))
    finally:
        if own:
            dset.free()
    w = want(ps, g0, g1, flags, nb_from, nb_to)
    for path, g in got.items():
        for k in g:
            assert np.array_equal(np.asarray(g[k]), np.asarray(w[k])), (path, k)
    if used:
        assert built == host_coverage(ps, len(g0)), built
    else:
        assert built == (0, 0)
    return built


@pytest.mark.parametrize("gap_flat", [True, False])
@pytest.mark.parametrize("n_and", [1, 2, 3, 64])
def test_coverage_member_kinds(ctx, n_and, gap_flat):
    """AND members NULL, FULL or bit-blocks behind listed blocks, a FULL SUB-group block, members named in descending order;
    FLAT and raw-form GAP blocks; whole, sub-range and count-only calls."""
    rng = np.random.default_rng(5100 + n_and)
    vecs, g0 = plan_set(rng, n_and, 0.5 if n_and <= 3 else 0.97)
    ps = bm.PackedSet.pack(vecs, gap_flat=gap_flat)
    g1 = [int(v) for v in rng.permutation([v for v in range(len(vecs)) if v not in g0])]
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        check(ctx, ps, g0, g1, C, dset=dset)
        check(ctx, ps, g0, g1, 0, 2, 8, dset=dset)
        check(ctx, ps, g0, g1, bm.F_COUNT_ONLY, 1, 0, dset=dset)
    finally:
        dset.free()


def test_coverage_listed_and_member(ctx):
    """A sparse bit-block vector (listed by the companion in every column) in the AND group is streamed like any bit-block."""
    rng = np.random.default_rng(5200)
    vecs, g0 = plan_set(rng, 2, 0.5)
    assert all(k in (bm.BLK_BIT, bm.BLK_NULL) for k in vecs[0].kind)
    g0 = [g0[0], 0]
    ps = bm.PackedSet.pack(vecs)
    check(ctx, ps, g0, [v for v in range(len(vecs)) if v not in g0], C)


def test_coverage_zero_one_stored(ctx):
    """Column 0: no SUB bit, the plane is empty (kCovZero); column 1: both AND members and a SUB vector FULL (three FULL blocks,
    the plane is full: kCovOne, a NULL result); column 2: AND member a and a SUB vector FULL, member b and a SUB bit-block that is
    its complement, so every bit counts 3 (full again, from the counts); columns 3, 4: stored planes."""
    rng = np.random.default_rng(5300)
    n = 5
    a, b = bm.BVector.random(n, 0.5, rng), bm.BVector.random(n, 0.7, rng)
    a.set_full(1); b.set_full(1); a.set_full(2)
    s_full, s_bits = bm.BVector(n), bm.BVector(n)
    s_full.set_full(1); s_full.set_full(2)
    s_bits.set_bits(2, ~b.block_words(2))
    for c in (3, 4):
        s_bits.set_bits(c, sparse_words(rng, 3000))
    g = bm.BVector(n)
    g.set_gap(4, bits_to_gap(bits_to_words(np.isin(np.arange(BLOCK_BITS), rng.choice(BLOCK_BITS, 500, replace=False)))))
    ps = bm.PackedSet.pack([s_bits, a, g, b, s_full])
    assert check(ctx, ps, [3, 1], [0, 2, 4], C) == (2, 2)


def test_coverage_groups_share_one_plane(ctx):
    """Three AND groups of 2 on one set use the plane built by the first; the default rule builds it on the third call."""
    rng = np.random.default_rng(5400)
    vecs = [bm.BVector.random(6, 0.3 + 0.1 * k, rng) for k in range(5)]
    vecs += [bm.BVector.random(6, 0.003 * (k + 1), rng).optimize() for k in range(20)]
    ps = bm.PackedSet.pack(vecs)
    everyone = range(len(vecs))
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        tune(ctx)
        seen = []
        for _ in range(3):
            bm.aggregate(ctx, dset, OP, [4, 0], [v for v in everyone if v not in (4, 0)], C).free()
            seen.append(dset.coverage(2))
        assert seen[:2] == [(0, 0), (0, 0)] and seen[2] == host_coverage(ps, 2) and seen[2][0] > 0
        for g0 in ([1, 2], [3, 0], [2, 4]):
            assert check(ctx, ps, g0, [v for v in everyone if v not in g0], C, dset=dset) == seen[2]
    finally:
        tune(ctx)
        dset.free()


def test_coverage_4096_vectors(ctx):
    """4096 vectors in one column: 4095 bit-blocks and a GAP block; AND = the first and the last bit-block."""
    rng = np.random.default_rng(5500)
    vecs = []
    for v in range(4095):
        w = rng.integers(0, 1 << 32, 2048, dtype=np.uint32)
        if v not in (0, 4094):
            w[:] = 0
            w[rng.integers(0, 2048, 3)] = np.uint32(1) << rng.integers(0, 32, 3, dtype=np.uint32)
        bv = bm.BVector(1); bv.set_bits(0, w); vecs.append(bv)
    bits = np.zeros(BLOCK_BITS, np.uint8)
    bits[rng.choice(BLOCK_BITS, 600, replace=False)] = 1
    g = bm.BVector(1); g.set_gap(0, bits_to_gap(bits_to_words(bits))); vecs.append(g)
    ps = bm.PackedSet.pack(vecs)
    assert check(ctx, ps, [4094, 0], [v for v in range(4096) if v not in (0, 4094)], C) == (1, 0)


def test_coverage_fallbacks(ctx):
    """An AND group holding a GAP block builds no plane; a fifth AND-group size on a set with four planes builds none either."""
    rng = np.random.default_rng(5600)
    vecs = [bm.BVector.random(4, 0.6, rng) for _ in range(6)]
    vecs += [bm.BVector.random(4, 0.0004 * (k + 1), rng).optimize() for k in range(10)]
    ps = bm.PackedSet.pack(vecs)
    assert (ps.kinds()[:, 8] == bm.BLK_GAP).any()
    everyone = range(len(vecs))
    check(ctx, ps, [0, 8], [v for v in everyone if v not in (0, 8)], C, used=False)
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        for n0 in (1, 2, 3, 4):
            assert check(ctx, ps, list(range(n0)), list(range(n0, len(vecs))), C, dset=dset)[0] > 0
        check(ctx, ps, list(range(5)), list(range(5, len(vecs))), C, dset=dset, used=False)
        check(ctx, ps, list(range(5)), list(range(5, len(vecs))), 0, 1, 3, dset=dset, used=False)
    finally:
        dset.free()


def test_coverage_c3_recipe(ctx):
    """C3's generator over 40 columns with its AND group (vectors 0 and 1): whole and over a sub-range, uncompressed and count-only."""
    import bench
    dens, seed, opt = bench.workload_inputs("c3", 0)
    n_vec, n_cols = 1024, 40
    dset = bm.DeviceSet.synth(ctx, n_vec, n_cols, dens, seed, opt)
    g0, g1 = [0, 1], np.arange(2, n_vec, dtype=np.uint32)
    try:
        runs = [four_ways(ctx, dset, g0, g1, *a) for a in ((C, 0, 0), (0, 5, 33), (bm.F_COUNT_ONLY, 3, 0))]
        stored, one = dset.coverage(2)
    finally:
        dset.free()
    assert stored + one == n_cols and stored > 0
    for got in runs:
        for path, g in got.items():
            for k in g:
                assert np.array_equal(np.asarray(g[k]), np.asarray(got["agg_kernel"][k])), (path, k)
