"""Stage boundaries of the whole-set AND-SUB kernel's GAP phase: every GAP or companion stage is split into slices between the
consumer warps of one group, so columns of 0, 1, 15, 16, 17 and 33 companion stages, last stages of 16 to 8176 bytes (some
slices empty or partial), a ring that wraps across columns whose stage counts are not multiples of the ring, more columns than
SMs, and AND-group GAP blocks that straddle slice and stage boundaries must all agree bit for bit with the general kernel
(TUNE_AGG_PIPELINE 0) and with the oracle."""
import numpy as np
import pytest

import bitmagic_b200 as bm
import orclib
from bitmagic_b200.hostfmt import bits_to_gap, bits_to_words, BLOCK_BITS
from test_agg_pipeline import run

pytestmark = pytest.mark.gpu

C = bm.F_OPT_COMPRESS
OP = bm.OP_AND_SUB
STAGE = 8192
EVEN = np.arange(2, BLOCK_BITS, 2)


def singles_gap(rng, k):
    """GAP block of k isolated 1-bits (each a companion single)."""
    bits = np.zeros(BLOCK_BITS, np.uint8)
    bits[rng.choice(EVEN, size=k, replace=False)] = 1
    return bits_to_gap(bits_to_words(bits))


def singles_for(stages, last):
    """Singles per column for `stages` companion stages whose last one holds `last` bytes (u16 positions, 16-byte units)."""
    return 0 if stages == 0 else ((stages - 1) * STAGE + last) // 2


def singles_set(rng, per_col, per_block=500):
    """Two dense bit-block vectors (the AND group) and GAP-only vectors whose blocks hold per_col[c] singles in column c."""
    n_blocks = len(per_col)
    vecs = [bm.BVector.random(n_blocks, 0.5, rng), bm.BVector.random(n_blocks, 0.5, rng)]
    n_gap = max(1, -(-max(per_col) // per_block))
    gap_vecs = [bm.BVector(n_blocks) for _ in range(n_gap)]
    for c, total in enumerate(per_col):
        left = total
        for v in gap_vecs:
            k = min(per_block, left)
            if k:
                v.set_gap(c, singles_gap(rng, k))
            left -= k
    return vecs + gap_vecs


def check(ctx, ps, g0, g1, run_lists):
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 2 if run_lists else 0)
        new = run(ctx, dset, OP, g0, g1, C, 0, 0)
        built = dset.run_list_bytes()
        ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, 0)
        old = run(ctx, dset, OP, g0, g1, C, 0, 0)
    finally:
        ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, 1)
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)
        dset.free()
    for k in new:
        assert np.array_equal(np.asarray(new[k]), np.asarray(old[k])), k
    okind, opop, odig, onr, oblk, ogap = orclib.oracle_aggregate(ps, OP, g0, g1, C, 0, ps.n_blocks)
    assert np.array_equal(new["blocks"], oblk)
    assert np.array_equal(new["kind"], okind) and np.array_equal(new["pop"], opop)
    assert np.array_equal(new["dig"], odig) and np.array_equal(new["nr"], onr)
    return built


def test_companion_stage_counts_and_last_stage_sizes(ctx):
    """Columns of 0, 1, 15, 16, 17 and 33 singles stages whose last stage holds 16, 496, 512, 528 or 8176 bytes, and one of two
    full stages; consecutive columns wrap the ring at different offsets."""
    rng = np.random.default_rng(71)
    shape = [(0, 0), (1, 16), (15, 496), (16, 512), (17, 528), (33, 8176), (2, STAGE), (1, 8176)]
    per_col = [singles_for(n, last) for n, last in shape]
    ps = bm.PackedSet.pack(singles_set(rng, per_col))
    n = ps.n_vec
    sgl, lr = check(ctx, ps, [0, 1], list(range(2, n)), True)
    assert (sgl, lr) == (2 * sum(per_col), 0)


def test_companion_many_columns(ctx):
    """More columns than SMs, each of 0 to 3 companion stages with a partial last stage."""
    rng = np.random.default_rng(72)
    per_col = [singles_for(c % 4, (16, 528, 4096, 8176)[c % 4]) for c in range(150)]
    ps = bm.PackedSet.pack(singles_set(rng, per_col, per_block=450))
    n = ps.n_vec
    sgl, lr = check(ctx, ps, [0, 1], list(range(2, n)), True)
    assert (sgl, lr) == (2 * sum(per_col), 0)


def test_and_group_gap_blocks_straddle_slices_and_stages(ctx):
    """FLAT GAP segments with AND-group GAP blocks (blanked per slice) that cross slice and stage boundaries."""
    rng = np.random.default_rng(73)
    n_blocks, n_sub = 6, 40
    vecs = [bm.BVector.random(n_blocks, 0.5, rng), bm.BVector(n_blocks), bm.BVector(n_blocks)]
    for c in range(n_blocks):
        vecs[1].set_gap(c, singles_gap(rng, 600))
        vecs[2].set_gap(c, singles_gap(rng, 300))
    subs = [bm.BVector(n_blocks) for _ in range(n_sub)]
    for c in range(n_blocks):
        for v in subs:
            v.set_gap(c, singles_gap(rng, int(rng.integers(1, 600))))
    # AND-group GAP vectors in the middle of the segment, behind SUB-group blocks of varying length
    vecs = vecs[:1] + subs[:7] + [vecs[1]] + subs[7:19] + [vecs[2]] + subs[19:]
    ps = bm.PackedSet.pack(vecs)
    g0 = [0, 8, 21]
    crossed = set()
    for c in range(n_blocks):
        for v in g0[1:]:
            d = int(ps.desc[c * ps.n_vec + v])
            lo = ((d >> 2) & 0x0FFFFFFF) * 16
            hi = lo + 2 * (d >> 31) + 2 * ((int(ps.block(v, c)[1][0]) >> 3) + 1)
            for b in range(STAGE // 2, hi, STAGE // 2):      # slice boundaries of two warps per stage, then stage boundaries
                if lo < b < hi:
                    crossed.add("stage" if b % STAGE == 0 else "slice")
    assert crossed == {"slice", "stage"}
    g1 = [v for v in range(len(vecs)) if v not in g0]
    assert check(ctx, ps, g0, g1, True) == (0, 0)        # an AND group with GAP blocks streams the GAP segments
