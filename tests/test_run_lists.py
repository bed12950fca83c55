"""The run-list companion of a set's GAP blocks (singles as u16 positions, long runs as FLAT pairs, per column), streamed by the
whole-set AND-SUB kernel in place of the GAP segments when the AND group holds no GAP block.  TUNE_RUN_LISTS 2 (build on the first
call) and 0 (never) must agree bit for bit with each other and with the oracle, the companion's size must match a host count of the
set's runs, and an AND group with a GAP vector must run without it."""
import numpy as np
import pytest

import bitmagic_b200 as bm
import gen
import orclib
from bitmagic_b200.hostfmt import bits_to_gap, bits_to_words, BLOCK_BITS

pytestmark = pytest.mark.gpu

C = bm.F_OPT_COMPRESS
OP = bm.OP_AND_SUB


def run(ctx, dset, g0, g1, flags, nb_from, nb_to):
    res = bm.aggregate(ctx, dset, OP, g0, g1, flags, nb_from, nb_to)
    kind, pop, dig, nr = res.meta()
    total, any_ = res.total()
    fk, off, bits, gaps = res.fetch()
    bv = bm.result_to_bvector(fk, off, bits, gaps)
    blocks = np.stack([bv.block_words(c) for c in range(kind.size)])
    gflat = np.concatenate([bv.blocks[c] for c in range(kind.size) if kind[c] == bm.BLK_GAP]) \
        if (kind == bm.BLK_GAP).any() else np.zeros(0, np.uint16)
    res.free()
    return dict(kind=kind, pop=pop, dig=dig, nr=nr, total=total, any=any_, blocks=blocks, gflat=gflat)


def host_run_list_bytes(ps):
    """(singles, long runs) bytes of the companion, counted on the host: per column, a u16 per 1-run of length 1 or starting at
    bit 0 and a u32 per 1-run longer than one bit, each part padded to 16 bytes."""
    sgl = lr = 0
    for nb in range(ps.n_blocks):
        ns = nl = 0
        for v in range(ps.n_vec):
            k, g = ps.block(v, nb)
            if k != bm.BLK_GAP:
                continue
            n, first = int(g[0]) >> 3, int(g[0]) & 1
            ends = g[1:n + 1].astype(np.int64)
            starts = np.concatenate([[0], ends[:-1] + 1])
            one = ((np.arange(n) & 1) ^ first) == 1
            s, e = starts[one], ends[one]
            ns += int(((s == e) | (s == 0)).sum()); nl += int((e > s).sum())
        sgl += (ns + 7) // 8 * 16; lr += (nl + 3) // 4 * 16
    return sgl, lr


def check_run_lists(ctx, ps, g0, g1, flags, nb_from=0, nb_to=0, expect_used=True):
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 2)
        new = run(ctx, dset, g0, g1, flags, nb_from, nb_to)
        built = dset.run_list_bytes()
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 0)
        old = run(ctx, dset, g0, g1, flags, nb_from, nb_to)
    finally:
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)
        dset.free()
    assert built == (host_run_list_bytes(ps) if expect_used else (0, 0))
    for k in new:
        assert np.array_equal(np.asarray(new[k]), np.asarray(old[k])), k
    hi = nb_to or ps.n_blocks
    okind, opop, odig, onr, oblk, ogap = orclib.oracle_aggregate(ps, OP, g0, g1, flags, nb_from, hi)
    assert np.array_equal(new["blocks"], oblk)
    assert np.array_equal(new["kind"], okind)
    assert np.array_equal(new["pop"], opop)
    assert np.array_equal(new["dig"], odig)
    assert np.array_equal(new["nr"], onr)
    assert new["total"] == int(opop.sum()) and new["any"] == bool(opop.sum())
    glen = np.where(okind == bm.BLK_GAP, (ogap[:, 0] >> 3) + 1, 0)
    oflat = np.concatenate([ogap[c, :glen[c]] for c in range(len(okind))]) if glen.sum() else np.zeros(0, np.uint16)
    assert np.array_equal(new["gflat"], oflat)


def run_block(rng, n_runs, max_len):
    """GAP block of n_runs disjoint 1-runs of length 1 .. max_len at random places."""
    bits = np.zeros(BLOCK_BITS, np.uint8)
    for s in rng.choice(BLOCK_BITS, size=n_runs, replace=False):
        bits[s:s + int(rng.integers(1, max_len + 1))] = 1
    return bits_to_gap(bits_to_words(bits))


def shaped_vectors(rng, n_blocks):
    """Edge blocks, blocks of singles only, of long runs only, of neither (all-zero), of runs at bit 0 and at bit 65535,
    and two bit-only vectors for the AND group; column 2 has no GAP blocks, column 3 no bit-blocks."""
    vecs = gen.edge_vectors(n_blocks) + gen.mixed_vectors(rng, 6, n_blocks, p_null=0.1, p_full=0.05, p_gap=0.6)
    for style in range(4):
        v = bm.BVector(n_blocks)
        for nb in range(n_blocks):
            if style == 0:
                v.set_gap(nb, run_block(rng, int(rng.integers(1, 400)), 1))                   # singles only
            elif style == 1:
                w = np.zeros(BLOCK_BITS, np.uint8)                                            # long runs only
                for s in rng.choice(BLOCK_BITS // 8, size=int(rng.integers(1, 60)), replace=False):
                    w[8 * s:8 * s + int(rng.integers(2, 8))] = 1
                v.set_gap(nb, bits_to_gap(bits_to_words(w)))
            elif style == 2:
                v.set_gap(nb, gen.gap_from_runs([0, 7, 9, 65534, 65535], 1))                  # singles at 0 and 65535, a long run
            else:
                v.set_gap(nb, gen.gap_from_runs([41, 65535], 1))                              # a long run from bit 0
        vecs.append(v)
    vecs += gen.mixed_vectors(rng, 2, n_blocks, p_null=0.0, p_full=0.0, p_gap=0.0)
    for v in vecs:
        if v.kind[2] == bm.BLK_GAP:
            v.set_bits(2, v.block_words(2))
        if v.kind[3] == bm.BLK_BIT:
            v.kind[3] = bm.BLK_NULL
            v.blocks.pop(3, None)
    return vecs


def test_run_lists_shapes(ctx):
    """FLAT and raw-form sets, sub-ranges, with and without compression; the AND group is the two bit-only vectors."""
    rng = np.random.default_rng(41)
    n_blocks = 6
    vecs = shaped_vectors(rng, n_blocks)
    n = len(vecs)
    g0 = [n - 2, n - 1]
    g1 = [v for v in rng.permutation(n) if v not in g0]
    for gap_flat in (True, False):
        ps = bm.PackedSet.pack(vecs, gap_flat=gap_flat)
        for nb_from, nb_to in ((0, 0), (1, 0), (2, 5), (5, 6)):
            check_run_lists(ctx, ps, g0, g1, C, nb_from, nb_to)
        check_run_lists(ctx, ps, g0, g1, 0)


def test_run_lists_long_parts_many_columns(ctx):
    """Columns whose singles part alone is longer than the 16-stage ring (> 128 KB), and more columns than SMs."""
    rng = np.random.default_rng(42)
    n_blocks, n_gap = 3, 160
    vecs = [bm.BVector.random(n_blocks, 0.3, rng), bm.BVector.random(n_blocks, 0.5, rng)]
    for k in range(n_gap):
        v = bm.BVector(n_blocks)
        for nb in range(n_blocks):
            v.set_gap(nb, run_block(rng, 600 if k % 8 else 300, 1 if k % 8 else 4))
        vecs.append(v)
    ps = bm.PackedSet.pack(vecs)
    assert host_run_list_bytes(ps)[0] > 16 * 8192 * n_blocks
    check_run_lists(ctx, ps, [0, 1], list(range(2, len(vecs))), C)

    vecs = [bm.BVector.random(200, 0.4, rng)] + [bm.BVector.random(200, 0.5 / (k + 1) if k < 6 else 0.002 * (k % 3 + 1), rng).optimize()
                                                  for k in range(15)]
    ps = bm.PackedSet.pack(vecs)
    g1 = list(rng.permutation(np.arange(1, len(vecs))))
    check_run_lists(ctx, ps, [0], g1, C)
    check_run_lists(ctx, ps, [0], g1, 0, 37, 0)


def test_run_lists_fall_back_and_build_rule(ctx):
    """An AND group holding a GAP vector runs without the companion and builds none; under the default rule the first qualifying
    call builds nothing and the second builds it."""
    rng = np.random.default_rng(43)
    n_blocks = 4
    vecs = [bm.BVector.random(n_blocks, 0.5, rng)] + [bm.BVector.random(n_blocks, 0.004 * (k + 1), rng).optimize() for k in range(12)]
    ps = bm.PackedSet.pack(vecs)
    assert (ps.kinds()[:, 1] == bm.BLK_GAP).any()
    check_run_lists(ctx, ps, [0, 1], list(range(2, 13)), C, expect_used=False)

    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)
        out = []
        for _ in range(2):
            res = bm.aggregate(ctx, dset, OP, [0, 1], list(range(2, 13)), C)
            res.free()
            out.append(dset.run_list_bytes())
        for _ in range(2):
            res = bm.aggregate(ctx, dset, OP, [0], list(range(1, 13)), C)
            out.append(dset.run_list_bytes())
            kind, pop, dig, nr = res.meta()
            res.free()
    finally:
        dset.free()
    assert out[:3] == [(0, 0), (0, 0), (0, 0)]
    assert out[3] == host_run_list_bytes(ps) and out[3][0] > 0
    okind, opop, odig, onr, _, _ = orclib.oracle_aggregate(ps, OP, [0], list(range(1, 13)), C, 0, n_blocks)
    assert np.array_equal(kind, okind) and np.array_equal(pop, opop) and np.array_equal(dig, odig) and np.array_equal(nr, onr)
