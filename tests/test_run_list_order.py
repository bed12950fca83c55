"""Order of the run-list companion's singles: each column part is dealt out by shared-memory bank of the live mask (position p lies
in bank (p >> 5) & 31), so that in every full round of 32 sixteen-byte units the unit a lane of the sweep eats holds 8 positions of
that lane's bank; what is left over follows, then the pad (runlist_kernel.cuh).  A numpy restatement of the rule is checked on
random and adversarial bank histograms without a GPU; on the GPU, columns built to hit the order's edges must agree bit for bit
between the companion path, the streamed kernel without it, the general kernel and the oracle, at unchanged companion sizes."""
import numpy as np
import pytest

import bitmagic_b200 as bm
import orclib
from bitmagic_b200.hostfmt import bits_to_gap, bits_to_words, BLOCK_BITS

C = bm.F_OPT_COMPRESS
OP = bm.OP_AND_SUB


def bank(p):
    return (np.asarray(p, np.int64) >> 5) & 31


def deal(positions, rot=0):
    """One column part as rl_write_kernel stores it, ranks in input order: (u16 slots padded to whole units, full rounds).
    rot = 16-byte units streamed ahead of the part (0 for part A, A's units for part B)."""
    pos = np.asarray(positions, np.int64)
    n = pos.size
    cnt = np.bincount(bank(pos), minlength=32)
    rounds = int(cnt.min()) // 8
    out = np.full((n + 7) // 8 * 8, -1, np.int64)
    taken = np.zeros(32, np.int64)
    left = rounds * 256
    for p in pos:
        b = int(bank(p)); j = int(taken[b]); taken[b] += 1
        if j // 8 < rounds:
            out[((j // 8) * 32 + (b - rot) % 32) * 8 + j % 8] = p
        else:
            out[left] = p; left += 1
    if n:
        out[n:] = out[n - 1]
    return out, rounds


def positions_for(rng, counts):
    """counts[b] positions of bank b (any of the bank's 64 words, any bit), shuffled."""
    pos = [32 * (32 * int(rng.integers(0, 64)) + b) + int(rng.integers(0, 32)) for b in range(32) for _ in range(int(counts[b]))]
    return rng.permutation(np.asarray(pos, np.int64))


HISTOGRAMS = {
    "random": lambda rng: rng.integers(0, 200, 32),
    "balanced": lambda rng: rng.poisson(300, 32),
    "one bank empty": lambda rng: np.where(np.arange(32) == 7, 0, rng.integers(50, 100, 32)),
    "all in one bank": lambda rng: np.where(np.arange(32) == 19, 1000, 0),
    "counts of 0 to 7": lambda rng: rng.integers(0, 8, 32),
    "exactly 8 * 32 * 3": lambda rng: np.full(32, 24),
    "exactly 8 * 32": lambda rng: np.full(32, 8),
    "one entry": lambda rng: np.where(np.arange(32) == 0, 1, 0),
    "none": lambda rng: np.zeros(32, np.int64),
}


@pytest.mark.parametrize("name", list(HISTOGRAMS))
def test_dealing_rule(name):
    """The dealt part is a permutation of its entries plus the pad (repeats of its last entry), and unit u of the first
    rounds * 32 units holds 8 positions of the bank of the lane that eats it, (u + rot) % 32."""
    rng = np.random.default_rng(1100 + list(HISTOGRAMS).index(name))
    counts = HISTOGRAMS[name](rng)
    pos = positions_for(rng, counts)
    for rot in (0, 1, 13, 31):
        out, rounds = deal(pos, rot)
        n = pos.size
        assert rounds == int(np.min(counts)) // 8
        assert out.size == (n + 7) // 8 * 8 and np.array_equal(np.sort(out[:n]), np.sort(pos))
        assert n == 0 or (out[n:] == out[n - 1]).all()
        units = bank(out[:rounds * 256]).reshape(-1, 8)
        assert (units == ((np.arange(rounds * 32) + rot) % 32)[:, None]).all()
        if name.startswith("exactly"):
            assert rounds * 256 == n                                    # no leftovers, no pad


# ---- GPU: columns at the order's edges ----

def spread(rng, counts, n_blocks, cap):
    """Blocks of isolated single bits (even bit offsets, so no two are adjacent): counts[b] singles of bank b in all, dealt
    round-robin over n_blocks blocks of at most cap singles each.  Returns one 65536-bit array per non-empty block."""
    per = [[] for _ in range(n_blocks)]
    k = 0
    for b in range(32):
        slots = rng.permutation(64 * 16)[:int(np.ceil(counts[b] / n_blocks))]      # (word of the bank, even bit) per block
        for i in range(int(counts[b])):
            s = int(slots[i // n_blocks])
            per[k % n_blocks].append(32 * (32 * (s // 16) + b) + 2 * (s % 16)); k += 1
    out = []
    for p in per:
        assert len(set(p)) == len(p) <= cap
        if p:
            bits = np.zeros(BLOCK_BITS, np.uint8); bits[p] = 1
            out.append(bits)
    return out


N_GAP, N_SPARSE = 8, 4          # GAP vectors (part A, at most 500 singles a block) and sparse bit-block vectors (part B)


def column_shapes(rng):
    """(part A per-bank counts, part B per-bank counts) per column."""
    z = np.zeros(32, np.int64)
    one = lambda b, n: np.where(np.arange(32) == b, n, 0)
    hole = lambda b, n: np.where(np.arange(32) == b, 0, n)
    return [
        (one(5, 900), one(31, 300)),                                    # every single in one bank
        (hole(7, 40), hole(0, 20)),                                     # an empty bank: many singles, no full round
        (rng.multinomial(100, [1 / 32] * 32), rng.multinomial(37, [1 / 32] * 32)),   # fewer than 256 singles
        (np.full(32, 24), np.full(32, 16)),                             # exactly rounds * 256, B behind a multiple of 32 units
        (np.full(32, 16) + one(3, 8), np.full(32, 16)),                 # A's 65 units rotate B's exact rounds by one lane
        (rng.poisson(100, 32), rng.poisson(50, 32)),                    # full rounds and leftovers, as on dense data
        (z, rng.integers(0, 8, 32)),                                    # no part A
        (rng.integers(0, 8, 32), z),                                    # no part B
        (z, z),                                                         # neither
        (np.full(32, 8) + one(0, 3), np.full(32, 8) + one(31, 5)),      # one round, leftovers and a pad in both parts
    ]


def edge_set(rng, reps=2):
    """Two dense bit-block vectors (the AND group), N_GAP GAP vectors and N_SPARSE sparse bit-block vectors whose singles follow
    column_shapes, `reps` times over."""
    shapes = column_shapes(rng) * reps
    n_blocks = len(shapes)
    vecs = [bm.BVector.random(n_blocks, 0.5, rng), bm.BVector.random(n_blocks, 0.6, rng)]
    gaps = [bm.BVector(n_blocks) for _ in range(N_GAP)]
    sparse = [bm.BVector(n_blocks) for _ in range(N_SPARSE)]
    for c, (ca, cb) in enumerate(shapes):
        for v, bits in zip(gaps, spread(rng, ca, N_GAP, 500)):
            v.set_gap(c, bits_to_gap(bits_to_words(bits)))
        for v, bits in zip(sparse, spread(rng, cb, N_SPARSE, 2048)):
            v.set_bits(c, bits_to_words(bits))
    return vecs + gaps + sparse, shapes


def outputs(ctx, dset, g0, g1, flags, nb_from, nb_to):
    res = bm.aggregate(ctx, dset, OP, g0, g1, flags, nb_from, nb_to)
    kind, pop, dig, nr = res.meta()
    total, any_ = res.total()
    out = dict(pop=pop, total=total, any=any_)
    if not flags & bm.F_COUNT_ONLY:
        bv = bm.result_to_bvector(*res.fetch())
        out.update(kind=kind, dig=dig, nr=nr, blocks=np.stack([bv.block_words(c) for c in range(kind.size)]))
    res.free()
    return out


def check(ctx, ps, shapes, g0, g1, flags, nb_from=0, nb_to=0):
    """Companion built on the first call, streamed kernel without it, general kernel: all equal and equal to the oracle; the
    companion's sizes are one u16 per single, each column part padded to 16 bytes and nothing more."""
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        got = []
        for pipe, rl in ((1, 2), (1, 0), (0, 0)):
            ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, pipe)
            ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, rl)
            got.append(outputs(ctx, dset, g0, g1, flags, nb_from, nb_to))
            if rl:
                sizes = dset.run_list_bytes() + dset.bit_run_list_bytes()
    finally:
        ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, 1)
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)
        dset.free()
    pad = lambda n: (int(n) + 7) // 8 * 16
    n_listed = sum(min(int(cb.sum()), N_SPARSE) for _, cb in shapes)
    assert sizes == (sum(pad(ca.sum()) for ca, _ in shapes), 0, sum(pad(cb.sum()) for _, cb in shapes), 0, n_listed)
    okind, opop, odig, onr, oblk, ogap = orclib.oracle_aggregate(ps, OP, g0, g1, flags & ~bm.F_COUNT_ONLY, nb_from, nb_to or ps.n_blocks)
    want = dict(pop=opop, total=int(opop.sum()), any=bool(opop.sum()), kind=okind, dig=odig, nr=onr, blocks=oblk)
    for g in got:
        for k in g:
            assert np.array_equal(np.asarray(g[k]), np.asarray(want[k])), k


@pytest.mark.gpu
def test_order_edges_parts_a_and_b(ctx):
    """AND group of the two dense vectors: parts A and B are streamed.  Whole set, a sub-range from column 3, without
    compression, and count-only."""
    rng = np.random.default_rng(1201)
    vecs, shapes = edge_set(rng)
    ps = bm.PackedSet.pack(vecs)
    g0, g1 = [0, 1], [int(v) for v in rng.permutation(np.arange(2, len(vecs)))]
    check(ctx, ps, shapes, g0, g1, C)
    check(ctx, ps, shapes, g0, g1, C, 3, 0)
    check(ctx, ps, shapes, g0, g1, 0, 5, 17)
    check(ctx, ps, shapes, g0, g1, bm.F_COUNT_ONLY)
    check(ctx, ps, shapes, g0, g1, bm.F_COUNT_ONLY, 3, 0)


@pytest.mark.gpu
def test_order_edges_part_a_only(ctx):
    """An AND group holding a listed vector streams part A alone (from unit 0 of each column, without part B behind it) and every
    bit-block as a block."""
    rng = np.random.default_rng(1202)
    vecs, shapes = edge_set(rng)
    ps = bm.PackedSet.pack(vecs)
    listed = 2 + N_GAP                                                 # the first sparse bit-block vector
    assert (ps.kinds()[:, listed] == bm.BLK_BIT).any()
    g0 = [0, listed]
    g1 = [v for v in range(len(vecs)) if v not in g0]
    check(ctx, ps, shapes, g0, g1, C)
    check(ctx, ps, shapes, g0, g1, C, 3, 0)


@pytest.mark.gpu
def test_order_raw_form_set(ctx):
    """A set packed in the raw GAP form has the same companion: the build decodes GAP blocks from their headers."""
    rng = np.random.default_rng(1203)
    vecs, shapes = edge_set(rng, reps=1)
    ps = bm.PackedSet.pack(vecs, gap_flat=False)
    check(ctx, ps, shapes, [0, 1], list(range(2, len(vecs))), C)
