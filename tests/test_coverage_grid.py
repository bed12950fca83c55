"""The coverage path's column hand-out: the whole-set AND-SUB kernel's coverage instantiation runs three CTAs per SM with a
6-stage ring, and each CTA streams columns until the range is used up.  Column counts around that grid (one column, a partial
wave, a full one, one column past it, two waves and a tail), all starting past column 0, with NULL-result columns (a NULL AND
member, an everywhere-covered plane) and empty-plane columns interleaved with stored planes, and AND groups of 1, 2 and 64
members must agree bit for bit with the companion, the segment path, the general kernel and the oracle."""
import numpy as np
import pytest

import bitmagic_b200 as bm
from test_coverage_plane import check
from test_pipe_column_plan import drop

pytestmark = pytest.mark.gpu

C = bm.F_OPT_COMPRESS
NB_FROM = 3


def grid(ctx):
    """CTAs of the whole-set AND-SUB kernel on the coverage path: three per SM."""
    return 3 * ctx.device_info()["sm_count"]


def mixed_set(rng, n_cols):
    """AND members a, b and SUB vectors s (bit-blocks) and g (GAP blocks).  Column c % 6 == 1: a NULL (a NULL result);
    c % 6 == 3: no SUB block (the plane of 2 is empty, kCovZero); c % 6 == 5: a, b and s FULL (the plane of 2 is full, kCovOne);
    every other column: a stored plane."""
    a, b, s = bm.BVector.random(n_cols, 0.5, rng), bm.BVector.random(n_cols, 0.25, rng), bm.BVector.random(n_cols, 0.3, rng)
    g = bm.BVector.random(n_cols, 0.002, rng).optimize()
    for c in range(n_cols):
        if c % 6 == 1:
            drop(a, c)
        elif c % 6 == 3:
            drop(s, c)
            drop(g, c)
        elif c % 6 == 5:
            a.set_full(c); b.set_full(c); s.set_full(c)
    return [s, a, g, b]


@pytest.fixture(scope="module")
def two_waves(ctx):
    rng = np.random.default_rng(5700)
    ps = bm.PackedSet.pack(mixed_set(rng, NB_FROM + 2 * grid(ctx) + 7 + 2))
    dset = bm.DeviceSet.upload(ctx, ps)
    yield ps, dset
    dset.free()


@pytest.mark.parametrize("cols", ["1", "grid-1", "grid", "grid+1", "2grid+7"])
def test_grid_column_counts(ctx, two_waves, cols):
    ps, dset = two_waves
    n = {"1": 1, "grid-1": grid(ctx) - 1, "grid": grid(ctx), "grid+1": grid(ctx) + 1, "2grid+7": 2 * grid(ctx) + 7}[cols]
    check(ctx, ps, [1, 3], [0, 2], C, NB_FROM, NB_FROM + n, dset=dset)


def test_grid_one_and_member(ctx, two_waves):
    ps, dset = two_waves
    check(ctx, ps, [1], [0, 2, 3], C, NB_FROM, NB_FROM + 2 * grid(ctx) + 7, dset=dset)


def test_grid_64_and_members(ctx):
    """64 AND members, FULL except a bit-block in every 16th column of each (a few per column) and member 7 NULL in columns
    c % 9 == 4; column c % 9 == 2 holds no SUB block, c % 9 == 6 only FULL SUB blocks (every bit counts more than 64)."""
    rng = np.random.default_rng(5800)
    n_cols = NB_FROM + grid(ctx) + 1 + 2
    members = []
    for m in range(64):
        v = bm.BVector(n_cols)
        for c in range(n_cols):
            if c % 9 == 4 and m == 7:
                continue
            if (c + m) % 16 == 0:
                v.set_bits(c, rng.integers(0, 1 << 32, 2048, dtype=np.uint32))
            else:
                v.set_full(c)
        members.append(v)
    s, g = bm.BVector.random(n_cols, 0.3, rng), bm.BVector.random(n_cols, 0.002, rng).optimize()
    for c in range(n_cols):
        if c % 9 == 2:
            drop(s, c)
            drop(g, c)
        elif c % 9 == 6:
            s.set_full(c); g.set_full(c)
    ps = bm.PackedSet.pack([s] + members + [g])
    g0 = list(range(64, 0, -1))
    check(ctx, ps, g0, [0, 65], C, NB_FROM, NB_FROM + grid(ctx) + 1)
