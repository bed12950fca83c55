"""Packed singles of the run-list companion: a column part is a run of 16-byte word units, each holding the index of one 32-bit word
of the live mask and up to 23 five-bit bit offsets inside it; a word's n singles fill ceil(n / 23) units of its own, unused fields
repeat a used one, and the units are dealt out by bank (runlist_kernel.cuh).  A numpy restatement of packing and dealing is checked
on random and adversarial word histograms without a GPU; on the GPU, columns built at the units' and banks' edges must agree bit
for bit between the companion path, the streamed kernel without it, the general kernel and the oracle, with packed sizes equal to
a host count and the list-form sizes unchanged."""
from collections import Counter

import numpy as np
import pytest

import bitmagic_b200 as bm
import orclib
from bitmagic_b200.hostfmt import bits_to_gap, bits_to_words, BLOCK_BITS

C = bm.F_OPT_COMPRESS
OP = bm.OP_AND_SUB
FIELDS = 23
WORDS = 2048


def units_of(n):
    return (np.asarray(n, np.int64) + FIELDS - 1) // FIELDS


def pack(positions, rot=0):
    """One column part as rl_write_kernel stores it, ranks in input order: ((units, 4) uint32, full rounds).
    rot = 16-byte units streamed ahead of the part (0 for part A, A's units for part B)."""
    pos = np.asarray(positions, np.int64)
    cnt = np.bincount(pos >> 5, minlength=WORDS)
    nu = units_of(cnt)
    ust = np.zeros(WORDS, np.int64)
    ub = np.zeros(32, np.int64)
    for b in range(32):                       # a word's first unit among its bank's: words b, b + 32, ... in order
        w = b + 32 * np.arange(64)
        ust[w] = np.cumsum(nu[w]) - nu[w]
        ub[b] = nu[w].sum()
    rounds = int(ub.min())
    lb = (32 * rounds + np.cumsum(ub - rounds) - (ub - rounds)).tolist()
    out = [[0, 0, 0, 0] for _ in range(int(ub.sum()))]
    rank = [0] * WORDS
    cnt, ust = cnt.tolist(), ust.tolist()
    for p in pos.tolist():
        w, o = p >> 5, p & 31
        r = rank[w]; rank[w] += 1
        k, f, b = ust[w] + r // FIELDS, r % FIELDS, w & 31
        q = out[k * 32 + (b - rot) % 32 if k < rounds else lb[b] + k - rounds]
        q[f // 6] |= o << (5 * (f % 6))
        if f == 0:
            for i, h in enumerate(((w & 3) << 30, ((w >> 2) & 3) << 30, ((w >> 4) & 3) << 30, (w >> 6) << 25)):
                q[i] |= h
            for g in range(min(cnt[w] - r, FIELDS), FIELDS):
                q[g // 6] |= o << (5 * (g % 6))
    return np.asarray(out, np.uint32).reshape(-1, 4), rounds


def unpack(units):
    """(word, [23 offsets]) per unit, as agg_pipe_kernel's sweep reads it."""
    u = units.astype(np.int64)
    word = (u[:, 0] >> 30) | ((u[:, 1] >> 30) << 2) | ((u[:, 2] >> 30) << 4) | ((u[:, 3] >> 25) << 6)
    offs = np.stack([(u[:, f // 6] >> (5 * (f % 6))) & 31 for f in range(FIELDS)], axis=1)
    return word, offs


def positions_for(rng, cnt):
    """cnt[w] singles of word w at distinct random offsets (repeats past 32 per word), shuffled."""
    pos = [32 * w + int(o) for w in np.flatnonzero(cnt) for o in np.resize(rng.permutation(32), int(cnt[w]))]
    return rng.permutation(np.asarray(pos, np.int64))


def hist(pairs):
    h = np.zeros(WORDS, np.int64)
    for w, n in pairs:
        h[w] = n
    return h


def bank_words(b, n):
    return b + 32 * np.arange(n)


HISTOGRAMS = {
    "unit edges": lambda rng: hist(zip(rng.permutation(WORDS)[:6], (1, 22, 23, 24, 46, 47))),
    "one word of thousands": lambda rng: hist([(int(rng.integers(WORDS)), 4000), (5, 3)]),
    "all in one bank": lambda rng: hist((int(w), int(rng.integers(1, 80))) for w in bank_words(19, 64)),
    "one bank empty": lambda rng: np.where((np.arange(WORDS) & 31) == 7, 0, rng.integers(0, 60, WORDS)),
    "exact rounds": lambda rng: hist((b, 46) for b in range(32)),
    "random": lambda rng: rng.poisson(72, WORDS),
    "one single": lambda rng: hist([(1234, 1)]),
    "none": lambda rng: np.zeros(WORDS, np.int64),
}


@pytest.mark.parametrize("name", list(HISTOGRAMS))
def test_packing_rule(name):
    """A word's singles fill ceil(n / 23) units of that word alone, every (word, offset) survives with the pads repeating the
    word's own offsets, and unit u of the first rounds * 32 holds a word of the bank of the lane that eats it, (u + rot) % 32."""
    rng = np.random.default_rng(1300 + list(HISTOGRAMS).index(name))
    cnt = HISTOGRAMS[name](rng)
    pos = positions_for(rng, cnt)
    nu = units_of(cnt)
    for rot in (0, 1, 13, 31):
        out, rounds = pack(pos, rot)
        assert out.shape[0] == nu.sum()
        assert rounds == min(int(nu[b::32].sum()) for b in range(32))
        word, offs = unpack(out)
        assert np.array_equal(np.bincount(word, minlength=WORDS), nu)
        for w in np.flatnonzero(cnt):
            want = Counter((pos[pos >> 5 == w] & 31).tolist())
            got = Counter(offs[word == w].ravel().tolist())
            extra = got - want
            assert not want - got and set(extra) <= set(want) and sum(extra.values()) == nu[w] * FIELDS - cnt[w]
        full = np.arange(rounds * 32)
        assert ((word[full] & 31) == (full + rot) % 32).all()
        if name == "exact rounds":
            assert rounds == 2 and out.shape[0] == 64                        # no leftovers


# ---- GPU: columns at the units' and banks' edges ----

N_GAP, N_SPARSE = 64, 4       # GAP vectors (part A) and sparse bit-block vectors (part B); each holds at most 16 singles a word


def column_shapes(rng):
    """(part A singles per word, part B singles per word) per column; A's words hold at most 16 * N_GAP singles, B's 16 * N_SPARSE."""
    z = np.zeros(WORDS, np.int64)
    edges = lambda: hist(zip(rng.permutation(WORDS)[:6], (1, 22, 23, 24, 46, 47)))
    exact = hist((b, 46) for b in range(32))
    return [
        (edges(), edges()),                                                             # ceil(n / 23) at its edges
        (hist([(int(rng.integers(WORDS)), 1000)]), hist([(77, 64)])),                   # one word holding thousands of singles
        (hist((int(w), 30) for w in bank_words(5, 40)), hist((int(w), 23) for w in bank_words(31, 9))),   # all in one bank
        (np.where((np.arange(WORDS) & 31) == 7, 0, rng.integers(0, 3, WORDS)),          # an empty bank: no full round
         np.where((np.arange(WORDS) & 31) == 0, 0, rng.integers(0, 2, WORDS))),
        (exact, exact),                                                                 # exact rounds, B behind 64 units
        (exact + hist([(3, 5)]), exact),                                                # A's 65 units rotate B's rounds by one lane
        (np.minimum(rng.poisson(3, WORDS), 60), np.minimum(rng.poisson(1, WORDS), 30)),  # full rounds and leftovers
        (z, edges()),                                                                   # no part A
        (edges(), z),                                                                   # no part B
        (z, z),                                                                         # neither
    ]


def spread(rng, cnt, n_vec):
    """cnt[w] isolated singles of word w (even offsets, so no two are adjacent) spread over n_vec blocks, at most one per
    (block, word, offset).  Returns one 65536-bit array per block (None when empty)."""
    bits = np.zeros((n_vec, BLOCK_BITS), np.uint8)
    for w in np.flatnonzero(cnt):
        start = int(rng.integers(n_vec))
        assert cnt[w] <= 16 * n_vec
        for k in range(int(cnt[w])):
            bits[(start + k // 16) % n_vec, 32 * w + 2 * (k % 16)] = 1
    return [b if b.any() else None for b in bits]


def edge_set(rng, reps=2):
    """Two dense bit-block vectors (the AND group), N_GAP GAP vectors and N_SPARSE sparse bit-block vectors whose singles follow
    column_shapes, `reps` times over."""
    shapes = column_shapes(rng) * reps
    n_blocks = len(shapes)
    vecs = [bm.BVector.random(n_blocks, 0.5, rng), bm.BVector.random(n_blocks, 0.6, rng)]
    gaps = [bm.BVector(n_blocks) for _ in range(N_GAP)]
    sparse = [bm.BVector(n_blocks) for _ in range(N_SPARSE)]
    for c, (ca, cb) in enumerate(shapes):
        for v, bits in zip(gaps, spread(rng, ca, N_GAP)):
            if bits is not None:
                v.set_gap(c, bits_to_gap(bits_to_words(bits)))
        for v, bits in zip(sparse, spread(rng, cb, N_SPARSE)):
            if bits is not None:
                v.set_bits(c, bits_to_words(bits))
    n_listed = sum(int((v.kind == bm.BLK_BIT).sum()) for v in sparse)
    return vecs + gaps + sparse, shapes, n_listed


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


def check(ctx, ps, shapes, n_listed, g0, g1, flags, nb_from=0, nb_to=0):
    """Companion built on the first call, streamed kernel without it, general kernel: all equal and equal to the oracle; packed
    singles are ceil(n / 23) units per word and part, the list-form sizes one u16 per single, each column part padded to 16 bytes."""
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        got = []
        for pipe, rl in ((1, 2), (1, 0), (0, 0)):
            ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, pipe)
            ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, rl)
            got.append(outputs(ctx, dset, g0, g1, flags, nb_from, nb_to))
            if rl:
                packed = dset.packed_singles_bytes()
                sizes = dset.run_list_bytes() + dset.bit_run_list_bytes()
    finally:
        ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, 1)
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)
        dset.free()
    assert packed == (16 * sum(int(units_of(ca).sum()) for ca, _ in shapes), 16 * sum(int(units_of(cb).sum()) for _, cb in shapes))
    pad = lambda n: (int(n) + 7) // 8 * 16
    assert sizes == (sum(pad(ca.sum()) for ca, _ in shapes), 0, sum(pad(cb.sum()) for _, cb in shapes), 0, n_listed)
    okind, opop, odig, onr, oblk, ogap = orclib.oracle_aggregate(ps, OP, g0, g1, flags & ~bm.F_COUNT_ONLY, nb_from, nb_to or ps.n_blocks)
    want = dict(pop=opop, total=int(opop.sum()), any=bool(opop.sum()), kind=okind, dig=odig, nr=onr, blocks=oblk)
    for g in got:
        for k in g:
            assert np.array_equal(np.asarray(g[k]), np.asarray(want[k])), k


@pytest.mark.gpu
def test_packed_edges_parts_a_and_b(ctx):
    """AND group of the two dense vectors: parts A and B are streamed.  Whole set, a sub-range from column 3, without
    compression, and count-only."""
    rng = np.random.default_rng(1301)
    vecs, shapes, n_listed = edge_set(rng)
    ps = bm.PackedSet.pack(vecs)
    g0, g1 = [0, 1], [int(v) for v in rng.permutation(np.arange(2, len(vecs)))]
    check(ctx, ps, shapes, n_listed, g0, g1, C)
    check(ctx, ps, shapes, n_listed, g0, g1, C, 3, 0)
    check(ctx, ps, shapes, n_listed, g0, g1, 0, 5, 17)
    check(ctx, ps, shapes, n_listed, g0, g1, bm.F_COUNT_ONLY)


@pytest.mark.gpu
def test_packed_edges_part_a_only(ctx):
    """An AND group holding a listed vector streams part A alone and every bit-block as a block."""
    rng = np.random.default_rng(1302)
    vecs, shapes, n_listed = edge_set(rng)
    ps = bm.PackedSet.pack(vecs)
    listed = 2 + N_GAP                                                 # the first sparse bit-block vector
    assert (ps.kinds()[:, listed] == bm.BLK_BIT).any()
    g0 = [0, listed]
    g1 = [v for v in range(len(vecs)) if v not in g0]
    check(ctx, ps, shapes, n_listed, g0, g1, C)
    check(ctx, ps, shapes, n_listed, g0, g1, C, 3, 0)


@pytest.mark.gpu
def test_packed_raw_form_set(ctx):
    """A set packed in the raw GAP form has the same companion."""
    rng = np.random.default_rng(1303)
    vecs, shapes, n_listed = edge_set(rng, reps=1)
    ps = bm.PackedSet.pack(vecs, gap_flat=False)
    check(ctx, ps, shapes, n_listed, [0, 1], list(range(2, len(vecs))), C)
