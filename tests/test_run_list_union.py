"""Union masks of the run-list companion: a column whose part A (or parts A + B) takes 8192 bytes or more as streamed keeps that
part as one 8 KB bitmap, the union of the runs its sweep clears, and the whole-set AND-SUB kernel streams the bitmap as one more
SUB-group bit stage in place of the packed part.  Columns built on each side of that choice must agree bit for bit between the
companion path, the streamed kernel without it, the general kernel and the oracle, and the number of union columns must match a
host count of the rule."""
import numpy as np
import pytest

import bitmagic_b200 as bm
import orclib
from bitmagic_b200.hostfmt import bits_to_gap, bits_to_words, words_to_bits, BLOCK_BITS
from test_bit_run_lists import LIST_MAX

pytestmark = pytest.mark.gpu

C = bm.F_OPT_COMPRESS
OP = bm.OP_AND_SUB
WORDS = 2048
FIELDS = 23
STAGE = 8192                   # bytes of one pipeline stage = one union mask


def runs_of_bits(bits):
    d = np.diff(np.concatenate([[0], bits.astype(np.int8), [0]]))
    return np.flatnonzero(d == 1), np.flatnonzero(d == -1) - 1


def runs_of_gap(g):
    n, first = int(g[0]) >> 3, int(g[0]) & 1
    ends = g[1:n + 1].astype(np.int64)
    starts = np.concatenate([[0], ends[:-1] + 1])
    one = ((np.arange(n) & 1) ^ first) == 1
    return starts[one], ends[one]


def part_bytes(runs):
    """Bytes a column part streams packed: a 16-byte word unit per 23 singles of one word (a run from bit 0 adds the single 0)
    and a 16-byte unit per 4 long runs."""
    if not runs:
        return 0
    s = np.concatenate([r[0] for r in runs]); e = np.concatenate([r[1] for r in runs])
    sg = s[(s == e) | (s == 0)]
    cnt = np.bincount(sg >> 5, minlength=WORDS)
    return 16 * int(((cnt + FIELDS - 1) // FIELDS).sum() + (int((e > s).sum()) + 3) // 4)


def host_part_bytes(ps):
    """(part A bytes, part B bytes) per column: A = the runs of every GAP block, B = those of every listed bit-block."""
    a, b = [], []
    for nb in range(ps.n_blocks):
        ra, rb = [], []
        for v in range(ps.n_vec):
            k, data = ps.block(v, nb)
            if k == bm.BLK_GAP:
                ra.append(runs_of_gap(data))
            elif k == bm.BLK_BIT:
                s, e = runs_of_bits(words_to_bits(data))
                if 2 * int(((s == e) | (s == 0)).sum()) + 4 * int((e > s).sum()) <= LIST_MAX:
                    rb.append((s, e))
        a.append(part_bytes(ra)); b.append(part_bytes(rb))
    return np.array(a), np.array(b)


def host_unions(ps):
    a, b = host_part_bytes(ps)
    return int((a >= STAGE).sum()), int((a + b >= STAGE).sum())


def outputs(ctx, dset, g0, g1, flags, nb_from, nb_to):
    res = bm.aggregate(ctx, dset, OP, g0, g1, flags, nb_from, nb_to)
    kind, pop, dig, nr = res.meta()
    total, any_ = res.total()
    out = dict(pop=pop, total=total, any=any_)
    if not flags & bm.F_COUNT_ONLY:
        fk, off, bits, gaps = res.fetch()
        bv = bm.result_to_bvector(fk, off, bits, gaps)
        gflat = np.concatenate([bv.blocks[c] for c in range(kind.size) if kind[c] == bm.BLK_GAP]) \
            if (kind == bm.BLK_GAP).any() else np.zeros(0, np.uint16)
        out.update(kind=kind, dig=dig, nr=nr, gflat=gflat, blocks=np.stack([bv.block_words(c) for c in range(kind.size)]))
    res.free()
    return out


def check(ctx, ps, g0, g1, flags, nb_from=0, nb_to=0):
    """Companion built on the first call, streamed kernel without it, general kernel and oracle: all equal; union columns as the
    host counts them.  Returns the device's (U_A columns, U_AB columns)."""
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        assert dset.run_list_unions() == (0, 0)
        got = []
        for pipe, rl in ((1, 2), (1, 0), (0, 0)):
            ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, pipe)
            ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, rl)
            got.append(outputs(ctx, dset, g0, g1, flags, nb_from, nb_to))
            if rl:
                unions = dset.run_list_unions()
                built = dset.run_list_bytes()
    finally:
        ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, 1)
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)
        dset.free()
    assert built != (0, 0)
    assert unions == host_unions(ps)
    hi = nb_to or ps.n_blocks
    okind, opop, odig, onr, oblk, ogap = orclib.oracle_aggregate(ps, OP, g0, g1, flags & ~bm.F_COUNT_ONLY, nb_from, hi)
    glen = np.where(okind == bm.BLK_GAP, (ogap[:, 0] >> 3) + 1, 0)
    oflat = np.concatenate([ogap[c, :glen[c]] for c in range(len(okind))]) if glen.sum() else np.zeros(0, np.uint16)
    want = dict(pop=opop, total=int(opop.sum()), any=bool(opop.sum()), kind=okind, dig=odig, nr=onr, gflat=oflat, blocks=oblk)
    for path, g in zip(("companion", "no companion", "agg_kernel"), got):
        for k in g:
            assert np.array_equal(np.asarray(g[k]), np.asarray(want[k])), (path, k)
    return unions


# ---- columns on each side of the 8 KB choice ----

N_GAP, N_LGAP, N_SPARSE = 64, 8, 4     # GAP vectors of singles and of long runs (part A), listed bit-block vectors (part B)


def words_hist(rng, n, big=None):
    """n distinct words holding one single each (+ word big[0] holding big[1] singles): n (+ ceil(big[1] / 23)) word units."""
    cnt = np.zeros(WORDS, np.int64)
    cnt[rng.permutation(WORDS)[:n]] = 1
    if big:
        cnt[big[0]] = big[1]
    return cnt


# (part A singles per word, part A long runs, part B singles per word, part B long runs) per column; units of 16 bytes
def column_shapes(rng):
    h, z = lambda n, big=None: words_hist(rng, n, big), np.zeros(WORDS, np.int64)
    return [
        (h(511), 0, z, 0),            # 0: A = 8176 bytes, no B: packed
        (h(512), 0, z, 0),            # 1: A = 8192, B empty: U_A, and U_AB is the same mask
        (h(513), 0, h(40), 0),        # 2: A = 8208: U_A and U_AB
        (h(300), 0, h(300), 0),       # 3: A below 8 KB, A + B above: U_AB only
        (z, 0, z, 0),                 # 4: no parts
        (z, 2100, z, 0),              # 5: long runs only (525 units)
        (h(500), 44, h(1), 0),        # 6: A = 500 + 11 units = 8176, A + B = 8192: U_AB only
        (h(480, (5, 1000)), 0, h(100), 50),   # 7: a word of 1000 singles (44 units), B long runs
        (h(20), 3, h(10), 2),         # 8: small: packed
        (h(600), 0, h(30), 0),        # 9: FULL in AND vector 0
        (h(600), 0, h(30), 0),        # 10: NULL in AND vector 1
        (h(600), 0, h(30), 0),        # 11: FULL in a SUB-group vector
    ]


DESIGN_A = {0: 8176, 1: 8192, 2: 8208, 3: 4800, 4: 0, 5: 8400, 6: 8176}
DESIGN_B = {0: 0, 1: 0, 2: 640, 3: 4800, 4: 0, 5: 0, 6: 16}


def spread(rng, cnt, n_vec):
    """cnt[w] isolated singles of word w (even offsets) over n_vec blocks, at most 16 per (block, word)."""
    bits = np.zeros((n_vec, BLOCK_BITS), np.uint8)
    for w in np.flatnonzero(cnt):
        start = int(rng.integers(n_vec))
        for k in range(int(cnt[w])):
            bits[(start + k // 16) % n_vec, 32 * w + 2 * (k % 16)] = 1
    return bits


def long_runs(rng, n, n_vec):
    """n runs of 2 .. 7 bits at 8 p + 1 over n_vec blocks (none from bit 0, none adjacent), one crossing many words and one to
    bit 65535 in the first block."""
    bits = np.zeros((n_vec, BLOCK_BITS), np.uint8)
    if n >= 2:
        bits[0, 100:3101] = 1; bits[0, 65000:] = 1; n -= 2
    for v in range(n_vec):
        k = n // n_vec + (v < n % n_vec)
        for p in rng.choice(np.arange(400, 8100), size=k, replace=False):
            bits[v, 8 * p + 1:8 * p + 1 + int(rng.integers(2, 8))] = 1
    return bits


def edge_set(rng, listed_and=False):
    """Two dense bit vectors (the AND group), the part A and part B vectors of column_shapes, one SUB vector FULL in column 11 and
    NULL elsewhere, and with listed_and a vector listed in every column (for an AND group that streams part A only)."""
    shapes = column_shapes(rng)
    n = len(shapes)
    vecs = [bm.BVector.random(n, 0.5, rng), bm.BVector.random(n, 0.6, rng)]
    vecs[0].set_full(9)
    vecs[1].kind[10] = bm.BLK_NULL; vecs[1].blocks.pop(10)
    gaps = [bm.BVector(n) for _ in range(N_GAP + N_LGAP)]
    sparse = [bm.BVector(n) for _ in range(N_SPARSE + 1)]
    for c, (ca, la, cb, lb) in enumerate(shapes):
        for v, bits in zip(gaps, np.concatenate([spread(rng, ca, N_GAP), long_runs(rng, la, N_LGAP)])):
            if bits.any():
                v.set_gap(c, bits_to_gap(bits_to_words(bits)))
        for v, bits in zip(sparse, np.concatenate([spread(rng, cb, N_SPARSE), long_runs(rng, lb, 1)])):
            if bits.any():
                v.set_bits(c, bits_to_words(bits))
    full = bm.BVector(n); full.set_full(11)
    vecs += gaps + sparse + [full]
    if listed_and:
        lv = bm.BVector(n)
        for c in range(n):
            lv.set_bits(c, bits_to_words(np.isin(np.arange(BLOCK_BITS), 2 * rng.choice(BLOCK_BITS // 2, 5000, replace=False))))
        vecs.append(lv)
    return vecs


def test_union_edges_parts_a_and_b(ctx):
    """AND group of the two dense vectors: columns stream U_AB where A + B reaches 8 KB.  Whole set, sub-ranges, without
    compression, and count-only."""
    rng = np.random.default_rng(2101)
    vecs = edge_set(rng)
    ps = bm.PackedSet.pack(vecs)
    a, b = host_part_bytes(ps)
    assert {c: int(a[c]) for c in DESIGN_A} == DESIGN_A and {c: int(b[c]) for c in DESIGN_B} == DESIGN_B
    assert host_unions(ps) == (7, 9)                   # U_A: 1 2 5 7 9 10 11; U_AB also 3 6; neither 0 4 8
    g0, g1 = [0, 1], [int(v) for v in rng.permutation(np.arange(2, len(vecs)))]
    check(ctx, ps, g0, g1, C)
    check(ctx, ps, g0, g1, C, 3, 0)
    check(ctx, ps, g0, g1, 0, 5, 10)
    check(ctx, ps, g0, g1, bm.F_COUNT_ONLY)


def test_union_edges_part_a_only(ctx):
    """An AND group holding a listed vector streams part A alone (U_A where A reaches 8 KB) and every bit-block as a block."""
    rng = np.random.default_rng(2102)
    vecs = edge_set(rng, listed_and=True)
    ps = bm.PackedSet.pack(vecs)
    a, _ = host_part_bytes(ps)
    assert {c: int(a[c]) for c in DESIGN_A} == DESIGN_A
    g0 = [0, len(vecs) - 1]
    g1 = [v for v in range(len(vecs)) if v not in g0]
    check(ctx, ps, g0, g1, C)
    check(ctx, ps, g0, g1, 0, 2, 8)


def test_union_raw_form_set(ctx):
    """A set packed in the raw GAP form has the same companion and union masks."""
    rng = np.random.default_rng(2103)
    ps = bm.PackedSet.pack(edge_set(rng), gap_flat=False)
    check(ctx, ps, [0, 1], list(range(2, ps.n_vec)), C)


def test_union_role_table_edge(ctx):
    """4096 vectors in one column: 4095 unlisted bit-blocks and one GAP block of 600 singles, so the union stage is bit stage
    4095, the last entry of the kernel's role table.  The SUB-group bit-blocks only cover the upper half of the block, so the
    lower half of the result is the AND group minus the union."""
    rng = np.random.default_rng(2104)
    vecs = []
    for v in range(4095):
        w = rng.integers(0, 1 << 32, WORDS, dtype=np.uint32)
        if v >= 2:
            w[:WORDS // 2] = 0
        bv = bm.BVector(1); bv.set_bits(0, w); vecs.append(bv)
    bits = np.zeros(BLOCK_BITS, np.uint8)
    bits[32 * rng.choice(WORDS // 2, 600, replace=False) + rng.integers(1, 31, 600)] = 1
    g = bm.BVector(1); g.set_gap(0, bits_to_gap(bits_to_words(bits))); vecs.append(g)
    ps = bm.PackedSet.pack(vecs)
    assert ps.n_vec == 4096 and int(ps.bit_base[1]) == 4095
    assert check(ctx, ps, [0, 1], list(range(2, 4096)), C) == (1, 1)


def test_union_c3_recipe(ctx):
    """C3's generator (vector k at density 0.5 / k, optimized) over 48 columns: every column streams U_AB, and the default rule's
    second call, which builds the companion, equals never building it."""
    import bench
    from test_run_lists import run
    dens, seed, opt = bench.workload_inputs("c3", 0)
    n_vec, n_cols = 1024, 48
    dset = bm.DeviceSet.synth(ctx, n_vec, n_cols, dens, seed, opt)
    g0, g1 = [0, 1], np.arange(2, n_vec, dtype=np.uint32)
    try:
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)
        out = [run(ctx, dset, g0, g1, C, 0, 0) for _ in range(2)]
        unions = dset.run_list_unions()
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 0)
        ref = run(ctx, dset, g0, g1, C, 0, 0)
    finally:
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)
        dset.free()
    assert unions == (n_cols, n_cols)
    for got in out:
        for k in ref:
            assert np.array_equal(np.asarray(got[k]), np.asarray(ref[k])), k
