"""Plane-search kernels at grid scale: every CTA (every warp, for the GAP merge) works through several populated columns.

The scan, set-membership, string, mismatch, shift and rank kernels claim work items (columns, or columns x value groups) until
the range is used up, with sm_count x ctas_per_sm CTAs.  What one column leaves behind -- GAP expansion buffers, descriptors,
staged rows, the prefetched claim -- must not leak into the next one.  The sets here are built column by column from per-column
element codes, each column one of SHAPES at random, so the columns one CTA takes in turn switch between bit, GAP, FULL / NULL
and unread planes.  Launches of grid - 1, grid + 1 and 3 * grid + 7 work items (and the same again with one CTA per SM) must
agree with the oracles bit for bit, GAP words and their headers included, and with the numpy model on a sample of columns.

The CPU tests at the end check that the generators produce what the GPU tests rely on."""
import numpy as np
import pytest

import bitmagic_b200 as bm
import orclib
import rsclib as R
from bitmagic_b200.capi import (BLK_BIT, BLK_FULL, BLK_GAP, BLK_NULL, BLOCK_BITS, F_FLOAT, F_SIGNED, F_STR_PREFIX, GAP_THRESHOLD,
                                MM_NO_NULL, MM_USE_NULL, NO_UNIVERSE, SCAN_IN, SCAN_RANGE_OPEN, TUNE_CTAS_PER_SM, mismatch_args)
from bitmagic_b200.hostfmt import BVector, PackedSet, bits_to_gap, gap_level
from test_launch_variants import REF_OP, assert_oracle, assert_same, collect
from test_scan_float import orc_call
from test_scan_in import oracle_scan_in
from test_scan_signed import oracle_scan_signed
from test_scan_str import oracle_scan_str
from test_sv_mismatch import oracle_first, oracle_mismatch

gpu = pytest.mark.gpu
B = BLOCK_BITS
CMP = bm.F_OPT_COMPRESS
CTAS_PER_SM = 2                      # agg_kernel's resident CTAs per SM (kCtasPerSm): the default of TUNE_CTAS_PER_SM
MERGE_WARPS = 4 * 8                  # gap_merge_kernel: 4 warps per CTA, 8 CTAs per SM

SHAPES = ("iid", "runs", "const", "sparse_exc", "near_limit", "all_gap", "null_uni", "no_match")
SH = {s: k for k, s in enumerate(SHAPES)}
NPL = 64                             # planes of the element codes: vectors 1 .. 64
P0 = 1
NPB = 21                             # planes of the edited copy the mismatch tests compare against: vectors 65 .. 85
PB0 = P0 + NPL
U2 = PB0 + NPB                       # the universe with a few bits flipped (the mismatch NULL term): vector 86
HOT = 4                              # codes every searched column holds at least once


# ------------------------------------------------------------------ sizes

def grid(ctx, ctas=CTAS_PER_SM):
    """CTAs of a work_grid launch with enough items: sm_count x ctas per SM."""
    return ctx.device_info()["sm_count"] * ctas


def targets(g):
    """Work items per launch: just under one CTA each, just over, and three items per CTA and a tail."""
    return [g - 1, g + 1, 3 * g + 7]


def n_cols_for(g):
    """Columns of a set that holds [nb_from, nb_from + 3g + 7) for nb_from up to 3, with a column past nb_to."""
    return 3 * g + 12


def col_range(k, t, passes=1):
    """Launch k of a sequence: t columns (even k) or t work items of `passes` value groups each (odd k), from column 1 + k % 3."""
    cols = t if k % 2 == 0 else -(-t // passes)
    lo = 1 + k % 3
    return lo, lo + cols


def target(g, k, ctas):
    """Work items of launch k: the three sizes in turn; with one CTA per SM, the largest."""
    return targets(g)[k % 3 if ctas == CTAS_PER_SM else 2]


def assert_deep(items, g):
    """The largest launch gives every CTA (warp) at least three items."""
    assert max(items) >= 3 * g, (max(items), g)


# ------------------------------------------------------------------ the element codes

def str_code(b: bytes) -> int:
    return int.from_bytes(b.ljust(8, b"\0")[:8], "little")


def code_str(c: int) -> bytes:
    return int(c).to_bytes(8, "little").rstrip(b"\0")


def code_pools(rng):
    """(pool, hot, absent): present codes are strings of 0..8 bytes 'a'..'z' (code 0 = the empty string) and their bitwise
    complements; absent codes start with a byte in '!'..'/', which no present string has, so no search matches them."""
    alpha = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", np.uint8)
    def strings(n, first=None):
        out = []
        for _ in range(n):
            ln = int(rng.integers(1, 9))
            s = bytes(alpha[rng.integers(0, alpha.size, ln)])
            if first is not None:
                s = bytes([int(rng.integers(first[0], first[1]))]) + s[1:]
            out.append(str_code(s))
        return out
    pool = np.unique(np.array([0] + strings(3000), np.uint64))
    hot = np.array(strings(HOT), np.uint64)
    absent = np.unique(np.array(strings(400, (0x21, 0x30)), np.uint64))
    return pool, hot, absent


def full_string(rng):
    """An 8-byte string whose complement is a string too (every byte of both non-zero)."""
    return np.uint64(str_code(bytes(rng.integers(0x61, 0x7B, 8).astype(np.uint8))))


def column_codes(rng, shape, pool, hot, absent):
    """65536 element codes of one column of the given shape."""
    pick = lambda n: pool[rng.integers(0, pool.size, n)]  # noqa: E731
    if shape in ("iid", "null_uni"):
        u = pick(B)
    elif shape == "no_match":
        return absent[rng.integers(0, absent.size, B)]
    elif shape == "const":
        return np.full(B, hot[rng.integers(0, HOT)], np.uint64)
    elif shape == "runs":                         # ~170 runs of long and short lengths, single-element runs among them
        singles = rng.integers(1, B - 2, 10)
        cuts = np.unique(np.concatenate([rng.choice(np.arange(1, B - 1), 150, replace=False), singles, singles + 1]))
        vals = np.concatenate([hot, pool])[rng.integers(0, HOT + pool.size, cuts.size + 1)]
        u = np.repeat(vals, np.diff(np.concatenate([[0], cuts, [B]])))
    elif shape == "sparse_exc":                   # one code with a few dozen exceptions: GAP planes with few runs
        u = np.full(B, hot[rng.integers(0, HOT)], np.uint64)
        u[rng.choice(B, 30, replace=False)] = pick(30)
    else:                                         # x / ~x runs: every plane flips at every cut
        x = full_string(rng)
        n = int(rng.integers(1270, 1282)) if shape == "near_limit" else int(rng.integers(20, 300))
        cuts = np.sort(rng.choice(np.arange(1, B), n - 1, replace=False))
        first = int(rng.integers(0, 2))
        alt = (np.arange(n) + first) & 1
        u = np.repeat(np.where(alt == 1, ~x, x).astype(np.uint64), np.diff(np.concatenate([[0], cuts, [B]])))
    return u


def plane_bits(u, n):
    """(n, 65536) uint8: bit j of every code."""
    b = np.unpackbits(np.ascontiguousarray(u, np.uint64).view(np.uint8).reshape(-1, 8), axis=1, bitorder="little")
    return np.ascontiguousarray(b[:, :n].T)


def words_rows(bits):
    return np.packbits(bits, axis=-1, bitorder="little").view("<u4").astype(np.uint32)


def store_column(vecs, c, bits, keep_bits):
    """Block c of vecs[j] from bits[j]: NULL / FULL when constant, GAP when it fits unless keep_bits(j) (a GAP-able block kept as
    a bit-block), else a bit-block."""
    runs = np.count_nonzero(bits[:, 1:] != bits[:, :-1], axis=1) + 1
    words = words_rows(bits)
    for j, v in enumerate(vecs):
        if runs[j] == 1:
            if bits[j, 0]:
                v.set_full(c)
        elif runs[j] < GAP_THRESHOLD and not keep_bits(j):
            ends = np.concatenate([np.flatnonzero(bits[j, 1:] != bits[j, :-1]), [B - 1]]).astype(np.uint16)
            g = np.empty(ends.size + 1, np.uint16)
            g[1:] = ends
            g[0] = int(bits[j, 0]) | (gap_level(int(ends.size)) << 1) | (int(ends.size) << 3)
            v.set_gap(c, g)
        else:
            v.set_bits(c, words[j])


def universe_column(rng, u_vec, c, kind):
    """Universe block c: 'gap' (a few hundred runs), 'bit' (iid 0.7), 'full', or nothing (NULL)."""
    if kind == "full":
        u_vec.set_full(c)
    elif kind == "gap":
        cuts = np.sort(rng.choice(np.arange(1, B), int(rng.integers(2, 400)), replace=False))
        bits = (np.searchsorted(cuts, np.arange(B), side="right") + int(rng.integers(0, 2))) & 1
        u_vec.set_gap(c, bits_to_gap(words_rows(bits.astype(np.uint8))))
    elif kind == "bit":
        u_vec.set_bits(c, words_rows((rng.random(B) < 0.7).astype(np.uint8)))


class MainSet:
    """Vector 0: universe U; 1..64: the planes of the element codes; 65..85: planes of an edited copy of their low 21 bits;
    86: U with bits flipped in a few columns.  Planes (j + c) % 3 == 0 of GAP-able blocks stay bit-blocks (except in all_gap
    columns), and every plane of the copy stays a bit-block in column c_mid.

    Edits of the copy: one element of column c_mid in a plane whose block of the original is GAP; elements of every fifth column
    past c_mid in planes 1..20 (so the 1-plane comparison never sees them); one element of column `last` in plane 0.  U2 differs
    from U in column c_null and in a few columns past it."""

    def __init__(self, n_cols, seed=7100, sample=12):
        rng = np.random.default_rng(seed)
        self.n_cols = N = n_cols
        self.last = N - 2
        shapes = rng.integers(0, len(SHAPES), N)
        shapes[rng.choice(np.arange(1, N - 1), len(SHAPES), replace=False)] = np.arange(len(SHAPES))
        if shapes[self.last] == SH["null_uni"]:
            shapes[self.last] = SH["iid"]
        self.shapes = shapes
        self.pool, self.hot, self.absent = code_pools(rng)
        ukind = np.array(["gap", "bit", "full"])[rng.integers(0, 3, N)]
        ukind[shapes == SH["null_uni"]] = "null"
        self.ukind = ukind
        # c_mid: a runs / sparse_exc column about a third in; c_null about half way
        cand = [c for c in range(N // 3, N - 2) if shapes[c] in (SH["runs"], SH["sparse_exc"]) and ukind[c] != "null"]
        self.c_mid = cand[0]
        self.c_null = next(c for c in range(N // 2, N - 2) if ukind[c] in ("gap", "bit", "full"))
        self.sample = sorted(set(rng.choice(np.arange(1, N - 1), min(sample, N - 2), replace=False).tolist())
                             | {int(np.flatnonzero(shapes == s)[0]) for s in range(len(SHAPES))} | {self.c_mid, self.last})
        self.codes = {}                           # sample column -> codes
        self.ubits = {}                           # sample column -> universe bits
        self.edits = {}                           # column -> [(position in the column, xor delta)]
        U, U2v = BVector(N), BVector(N)
        planes = [BVector(N) for _ in range(NPL)]
        copy = [BVector(N) for _ in range(NPB)]
        mask_b = np.uint64(2**NPB - 1)
        for c in range(N):
            shape = SHAPES[shapes[c]]
            u = column_codes(rng, shape, self.pool, self.hot, self.absent)
            universe_column(rng, U, c, ukind[c])
            ub = R.bits_of(U.block_words(c))
            if shape not in ("const", "no_match"):      # a hot code inside the universe: the hot codes lead the EQ lists
                u[int(rng.choice(np.flatnonzero(ub))) if ub.any() else 0] = self.hot[rng.integers(0, HOT)]
            bits = plane_bits(u, NPL)
            store_column(planes, c, bits, lambda j: shape != "all_gap" and (j + c) % 3 == 0)
            ed = []
            if c == self.c_mid:
                j = next(j for j in range(1, NPB) if planes[j].kind[c] == BLK_GAP)
                ed.append((int(rng.choice(np.flatnonzero(ub))), np.uint64(1 << j)))
            elif c == self.last:
                ed.append((int(rng.choice(np.flatnonzero(ub))) if ub.any() else 5, np.uint64(1)))
            elif c > self.c_mid and c % 5 == 0:
                for p in rng.choice(B, 3, replace=False):
                    ed.append((int(p), np.uint64(int(rng.integers(1, 2**(NPB - 1))) << 1)))
            ub2 = (u & mask_b).copy()
            for p, d in ed:
                ub2[p] ^= d
            if ed:
                self.edits[c] = ed
            store_column(copy, c, plane_bits(ub2, NPB), lambda j: c == self.c_mid or (j + c) % 3 == 0)
            if c == self.c_null or (c > self.c_null and c % 11 == 0):
                flip = ub.copy()
                flip[int(rng.integers(0, B))] ^= 1
                if c == self.c_null:
                    self.null_pos = c * B + int(np.flatnonzero(flip != ub)[0])
                U2v.set_bits(c, words_rows(flip))
            elif U.kind[c] != BLK_NULL:
                if U.kind[c] == BLK_FULL:
                    U2v.set_full(c)
                elif U.kind[c] == BLK_GAP:
                    U2v.set_gap(c, U.blocks[c])
                else:
                    U2v.set_bits(c, U.blocks[c])
            if c in self.sample:
                self.codes[c] = u
                self.ubits[c] = ub
        self.vecs = [U] + planes + copy + [U2v]
        self.ps = {flat: PackedSet.pack(self.vecs, N, gap_flat=flat) for flat in (True, False)}

    def searched(self):
        """Columns every EQ / IN / string search launch can hit: not no_match, universe not NULL."""
        return [c for c in range(self.n_cols) if self.shapes[c] != SH["no_match"] and self.ukind[c] != "null"]

    def eq_values(self, rng, nv):
        """nv codes present in the set, the hot codes first."""
        v = list(self.hot[:min(nv, HOT)]) + list(self.pool[rng.integers(0, self.pool.size, max(0, nv - HOT))])
        return np.array(v[:nv], np.uint64)

    def first_positions(self):
        """(first mismatch of plane 0 only, of the 21 planes, of the NULL term only): the intended first differences."""
        (pl, _), = self.edits[self.last]
        (pm, _), = self.edits[self.c_mid]
        return self.last * B + pl, self.c_mid * B + pm, self.null_pos


def mm_kw(ms, **kw):
    base = dict(plane0_a=P0, n_planes_a=NPB, plane0_b=PB0, n_planes_b=NPB, not_null_a=0, not_null_b=U2,
                size_a=ms.n_cols * B - 3000, size_b=ms.n_cols * B - 1000)
    base.update(kw)
    return base


# ------------------------------------------------------------------ numpy models on sample columns

def sample_block(got, g, nb_from, nb_to, c):
    """Bits of column c of group g of a result over [nb_from, nb_to)."""
    return R.bits_of(got["blocks"][g * (nb_to - nb_from) + c - nb_from])


def check_model(ms, got, nb_from, nb_to, models, uni):
    """models[g](codes) -> bool per element, before the universe; every sample column inside the range, every group."""
    for c in ms.sample:
        if not nb_from <= c < nb_to:
            continue
        ok = ms.ubits[c].astype(bool) if uni != NO_UNIVERSE else np.ones(B, bool)
        for g, m in enumerate(models):
            want = (m(ms.codes[c]) & ok).astype(np.uint8)
            assert np.array_equal(sample_block(got, g, nb_from, nb_to, c), want), (c, SHAPES[ms.shapes[c]], g)


def unsigned_model(pred, s, mask):
    if pred == bm.SCAN_RANGE:
        lo, hi = sorted(int(x) for x in s)
        return lambda u: ((u & mask) >= np.uint64(lo)) & ((u & mask) <= np.uint64(hi))
    x = np.uint64(int(s))
    return {bm.SCAN_EQ: lambda u: (u & mask) == x, bm.SCAN_GT: lambda u: (u & mask) > x, bm.SCAN_GE: lambda u: (u & mask) >= x,
            bm.SCAN_LT: lambda u: (u & mask) < x, bm.SCAN_LE: lambda u: (u & mask) <= x}[pred]


def str_model(q, prefix):
    qc = np.uint64(str_code(q))
    if prefix and q:
        m = np.uint64(2**(8 * len(q)) - 1)
        return lambda u: (u & m) == qc
    return lambda u: u == qc


def no_match_columns_empty(ms, got, nb_from, nb_to, n_groups):
    """Every result word of a no_match column is zero."""
    w = nb_to - nb_from
    for c in range(nb_from, nb_to):
        if ms.shapes[c] == SH["no_match"]:
            assert all(got["pop"][g * w + c - nb_from] == 0 for g in range(n_groups)), c


# ------------------------------------------------------------------ fixtures

@pytest.fixture(scope="module")
def main(ctx):
    ms = MainSet(n_cols_for(grid(ctx)))
    dsets = {flat: bm.DeviceSet.upload(ctx, ms.ps[flat]) for flat in (True, False)}
    yield ms, dsets
    for d in dsets.values():
        d.free()


@pytest.fixture(params=[CTAS_PER_SM, 1], ids=["ctas2", "ctas1"])
def ctas(request, ctx):
    """TUNE_CTAS_PER_SM for the work_grid kernels that follow it; restored afterwards (ctx is session-wide)."""
    ctx.set_tuning(TUNE_CTAS_PER_SM, request.param)
    yield request.param
    ctx.set_tuning(TUNE_CTAS_PER_SM, CTAS_PER_SM)


def run_scan(ctx, ms, dset, ps, pred, vals, npl, uni, flags, lo, hi, oracle):
    res = bm.scan(ctx, dset, pred, vals, P0, npl, uni, flags, nb_from=lo, nb_to=hi)
    nv = len(vals)
    got = collect(res, nv); res.free()
    assert_oracle(got, oracle(ps, pred, vals, P0, npl, uni, flags, lo, hi), nv, f"pred={pred} npl={npl} nv={nv} [{lo},{hi}) flags={flags}")
    return got


def passes(pred, nv):
    vg = 1 if nv == 1 else (4 if pred == bm.SCAN_EQ and nv >= 4 else 2)
    return -(-nv // vg)


# ------------------------------------------------------------------ GPU: unsigned, signed and float scans

def unsigned_searches(ms, rng, pred, nv, npl):
    mask = 2**npl - 1 if npl < 64 else 2**64 - 1
    v = ms.eq_values(rng, nv) if pred == bm.SCAN_EQ else ms.pool[rng.integers(0, ms.pool.size, nv)]
    v = [int(x) & mask for x in v]
    if pred == bm.SCAN_RANGE:
        w = [int(x) & mask for x in ms.pool[rng.integers(0, ms.pool.size, nv)]]
        return np.array([[a, b] for a, b in zip(v, w)], np.uint64)
    return np.array(v, np.uint64)


@gpu
@pytest.mark.parametrize("npl", [1, 33, 64])
def test_scan_unsigned(ctx, main, ctas, npl):
    """bmb200_scan, every <VG, MODE> kernel (1..5 values of EQ / GT / GE / LT / LE / RANGE) over 1, 33 and 64 planes from plane 1,
    grid - 1 / grid + 1 / 3 grid + 7 items or columns, universes absent / mixed GAP, bit, FULL and NULL, FLAT and raw GAP planes:
    == orc_scan and the value model on the sample columns."""
    ms, dsets = main
    g = grid(ctx)
    rng = np.random.default_rng(200 + npl)
    if ctas == 1:
        launches = [(bm.SCAN_EQ, 1), (bm.SCAN_EQ, 4), (bm.SCAN_GT, 5)]
    elif npl == 64:         # EQ: VG 1, 2, 4 with short last groups; the inequalities and RANGE: VG 1, 2
        nvs = {bm.SCAN_EQ: (1, 2, 3, 4, 5), bm.SCAN_GT: (1, 2, 5), bm.SCAN_GE: (3,), bm.SCAN_LT: (4,), bm.SCAN_LE: (1, 5),
               bm.SCAN_RANGE: (1, 2, 5)}
        launches = [(p, nv) for p, v in nvs.items() for nv in v]
    else:
        launches = [(p, nv) for p in (bm.SCAN_EQ, bm.SCAN_LE, bm.SCAN_RANGE) for nv in (1, 3, 5)]
    mask = np.uint64(2**npl - 1) if npl < 64 else np.uint64(2**64 - 1)
    items, k = [], 0
    for pred, nv in launches:
        flat = k % 4 != 3
        uni = 0 if k % 2 == 0 else NO_UNIVERSE
        lo, hi = col_range(k, target(g, k, ctas), passes(pred, nv))
        vals = unsigned_searches(ms, rng, pred, nv, npl)
        got = run_scan(ctx, ms, dsets[flat], ms.ps[flat], pred, vals, npl, uni, CMP if k % 2 else 0, lo, hi, orclib.oracle_scan)
        check_model(ms, got, lo, hi, [unsigned_model(pred, s, mask) for s in vals], uni)
        if pred == bm.SCAN_EQ and npl == 64:
            no_match_columns_empty(ms, got, lo, hi, nv)
        items.append((hi - lo) * passes(pred, nv))
        k += 1
    assert_deep(items, g)


@gpu
def test_scan_signed_and_float(ctx, main, ctas):
    """F_SIGNED (64 s2u planes; EQ / GT / RANGE) and F_FLOAT (32 sign + magnitude planes; GT / LE / RANGE / RANGE_OPEN) with 1 and
    5 values at the three launch sizes: == orc_scan_signed / orc_scan_float."""
    ms, dsets = main
    g = grid(ctx)
    rng = np.random.default_rng(300)
    u2s = lambda c: (c >> np.uint64(1)).astype(np.int64) ^ -(c & np.uint64(1)).astype(np.int64)  # noqa: E731
    items, k = [], 0
    for pred in (bm.SCAN_EQ, bm.SCAN_GT, bm.SCAN_RANGE):
        for nv in ((1, 5) if ctas == CTAS_PER_SM else (5,)):
            lo, hi = col_range(k, target(g, k, ctas), passes(pred, nv))
            c = ms.eq_values(rng, nv) if pred == bm.SCAN_EQ else ms.pool[rng.integers(0, ms.pool.size, nv)]
            vals = u2s(c)
            if pred == bm.SCAN_RANGE:
                vals = np.stack([vals, u2s(ms.pool[rng.integers(0, ms.pool.size, nv)])], 1)
            flat = k % 3 != 2
            run_scan(ctx, ms, dsets[flat], ms.ps[flat], pred, vals, NPL, 0, F_SIGNED | (CMP if k % 2 else 0), lo, hi, oracle_scan_signed)
            items.append((hi - lo) * passes(pred, nv))
            k += 1

    def orc_float(ps, pred, vals, plane0, npl, uni, flags, lo, hi):
        rc, out = orc_call(ps, pred, np.ascontiguousarray(vals.view(np.uint32).astype(np.uint64)), plane0, npl, uni, flags, lo, hi)
        assert rc == 0
        return out
    for pred in (bm.SCAN_GT, bm.SCAN_LE, bm.SCAN_RANGE, SCAN_RANGE_OPEN):
        for nv in ((1, 5) if ctas == CTAS_PER_SM else (5,)):
            lo, hi = col_range(k, target(g, k, ctas), passes(pred, nv))
            shape = (nv, 2) if pred in (bm.SCAN_RANGE, SCAN_RANGE_OPEN) else (nv,)
            key = (ms.pool[rng.integers(0, ms.pool.size, int(np.prod(shape)))] & np.uint64(0xFFFFFFFF)).astype(np.uint32)
            fb = (key >> np.uint32(1)) | ((key & np.uint32(1)) << np.uint32(31))          # f2u inverted: the float of a stored key
            vals = fb.reshape(shape).view(np.float32)
            flat = k % 3 != 2
            run_scan(ctx, ms, dsets[flat], ms.ps[flat], pred, vals, 32, 0, F_FLOAT | (CMP if k % 2 else 0), lo, hi, orc_float)
            items.append((hi - lo) * passes(pred, nv))
            k += 1
    assert_deep(items, g)


# ------------------------------------------------------------------ GPU: set membership and strings

@gpu
@pytest.mark.parametrize("npl", [21, 33])
def test_scan_in(ctx, main, ctas, npl):
    """SCAN_IN with K = 5 (the list staged whole) and K = 5000 (above the 4096-code staging bound: splitters and buckets), 21 and
    33 (WIDE) planes, at the three launch sizes: == orc_scan_in and np.isin & U on the sample columns."""
    ms, dsets = main
    g = grid(ctx)
    rng = np.random.default_rng(400 + npl)
    mask = np.uint64(2**npl - 1)
    items = []
    for k, (K, t) in enumerate([(5, 0), (5000, 1), (5000, 2), (5, 2)] if ctas == CTAS_PER_SM else [(5000, 2)]):
        lo = 1 + k % 3
        hi = lo + targets(g)[t]
        lst = ms.eq_values(rng, 5) & mask
        if K > 5:
            lst = np.concatenate([lst, ms.pool[rng.integers(0, ms.pool.size, K // 2)] & mask,
                                  rng.integers(0, 2**npl, K, dtype=np.uint64)])
            lst = np.unique(lst)[:K]
            assert lst.size == K
        flat, uni = k % 2 == 0, (0 if k != 1 else NO_UNIVERSE)
        res = bm.scan(ctx, dsets[flat], SCAN_IN, lst, P0, npl, uni, CMP if k % 2 else 0, lo, hi)
        got = collect(res, 1); res.free()
        assert_oracle(got, oracle_scan_in(ms.ps[flat], lst, P0, npl, uni, CMP if k % 2 else 0, lo, hi), 1, f"IN K={K} [{lo},{hi})")
        check_model(ms, got, lo, hi, [lambda u: np.isin(u & mask, lst)], uni)
        items.append(hi - lo)
    assert_deep(items, g)


def str_queries(ms, rng, nv, prefix):
    """nv strings present in the set (the hot ones first); prefix: their first 1..len bytes"""
    out = []
    for c in ms.eq_values(rng, nv):
        s = code_str(c)
        if prefix and s:
            s = s[:int(rng.integers(1, len(s) + 1))]
        out.append(s)
    return out


@gpu
def test_scan_str(ctx, main, ctas):
    """bmb200_scan_str over the 64 planes (strings of up to 8 bytes), exact and prefix, 1..5 queries per launch, at the three
    launch sizes: == orc_scan_str and the string comparison on the sample columns; no_match columns stay empty."""
    ms, dsets = main
    g = grid(ctx)
    rng = np.random.default_rng(500)
    items, k = [], 0
    for pflag in (0, F_STR_PREFIX):
        for nv in ((1, 2, 3, 4, 5) if ctas == CTAS_PER_SM else (4,)):
            q = str_queries(ms, rng, nv, bool(pflag))
            lo, hi = col_range(k, target(g, k, ctas), passes(bm.SCAN_EQ, nv))
            flat, uni = k % 3 != 1, (0 if k % 2 else NO_UNIVERSE)
            flags = pflag | (CMP if k % 2 else 0)
            res = bm.scan_str(ctx, dsets[flat], q, P0, NPL, uni, flags, nb_from=lo, nb_to=hi)
            got = collect(res, nv); res.free()
            assert_oracle(got, oracle_scan_str(ms.ps[flat], q, P0, NPL, uni, flags, lo, hi), nv, f"str {q} flags={flags} [{lo},{hi})")
            check_model(ms, got, lo, hi, [str_model(s, bool(pflag)) for s in q], uni)
            no_match_columns_empty(ms, got, lo, hi, nv)
            items.append((hi - lo) * passes(bm.SCAN_EQ, nv))
            k += 1
    assert_deep(items, g)


# ------------------------------------------------------------------ GPU: mismatch

@gpu
def test_sv_mismatch(ctx, main, ctas):
    """bmb200_sv_mismatch (21 planes against the edited copy, NOT-NULL U against U2, both null_proc values) at the three launch
    sizes == orc_sv_mismatch; bmb200_sv_first_mismatch == orc_sv_first_mismatch == the intended position: in the last column
    (plane 0 only), in a GAP-vs-bit pair of a middle column with later columns differing too, only in the NULL term."""
    ms, dsets = main
    g = grid(ctx)
    items = []
    for k, t in enumerate(targets(g)):
        lo, hi = col_range(k, t)
        flat = k != 1
        for use in (MM_USE_NULL, MM_NO_NULL):
            a = mismatch_args(**mm_kw(ms), null_proc=use, flags=CMP if use == MM_USE_NULL else 0, nb_from=lo, nb_to=hi)
            res = bm.sv_mismatch(ctx, dsets[flat], a)
            got = collect(res, 1); res.free()
            assert_oracle(got, oracle_mismatch(ms.ps[flat], a), 1, f"mismatch [{lo},{hi}) use={use}")
            assert bm.sv_first_mismatch(ctx, dsets[flat], a) == oracle_first(ms.ps[flat], a)
        items.append(hi - lo)
    assert_deep(items, g)
    p_last, p_mid, p_null = ms.first_positions()
    N = ms.n_cols
    full = dict(size_a=N * B, size_b=N * B)
    cases = [(mm_kw(ms, n_planes_a=1, n_planes_b=1, not_null_a=NO_UNIVERSE, not_null_b=NO_UNIVERSE, **full), MM_USE_NULL, p_last),
             (mm_kw(ms, not_null_b=0, **full), MM_USE_NULL, p_mid),
             (mm_kw(ms, not_null_a=NO_UNIVERSE, not_null_b=NO_UNIVERSE, **full), MM_NO_NULL, p_mid),
             (mm_kw(ms, plane0_b=P0, **full), MM_USE_NULL, p_null),
             (mm_kw(ms, plane0_b=P0, **full), MM_NO_NULL, None)]
    for kw, use, want in cases:
        for flat in (True, False):
            a = mismatch_args(**kw, null_proc=use, nb_from=1, nb_to=ms.last + 1)
            assert bm.sv_first_mismatch(ctx, dsets[flat], a) == want == oracle_first(ms.ps[flat], a), (kw, use, flat)


# ------------------------------------------------------------------ GPU: SHIFT-R-AND

@gpu
def test_shift_right_and(ctx, main, ctas):
    """OP_SHIFT_R_AND over plane groups through bmb200_aggregate and a batch of four groups (n_cols x n_groups items) at the three
    launch sizes: == orc_aggregate."""
    ms, dsets = main
    g = grid(ctx)
    groups = [([5, 6, 7], []), ([1, 40, 41, 9], []), ([33], []), ([60, 12], [])]
    items = []
    for k, t in enumerate(targets(g)):
        lo, hi = col_range(k, t)
        flat = k != 1
        ps = ms.ps[flat]
        res = bm.aggregate(ctx, dsets[flat], bm.OP_SHIFT_R_AND, groups[k][0], None, CMP, lo, hi)
        got = collect(res); res.free()
        assert_oracle(got, orclib.oracle_aggregate(ps, bm.OP_SHIFT_R_AND, groups[k][0], None, CMP, lo, hi), 1, f"shift [{lo},{hi})")
        lo, hi = col_range(k + 1, t, len(groups))
        res = bm.aggregate_batch(ctx, dsets[flat], bm.OP_SHIFT_R_AND, groups, 0 if k % 2 else CMP, lo, hi)
        got = collect(res, len(groups)); res.free()
        o = [orclib.oracle_aggregate(ps, bm.OP_SHIFT_R_AND, g0, None, 0 if k % 2 else CMP, lo, hi) for g0, _ in groups]
        assert_oracle(got, tuple(np.concatenate([p[i] for p in o]) for i in range(6)), len(groups), f"shift batch [{lo},{hi})")
        items.append((hi - lo) * len(groups))
    assert_deep(items, g)


# ------------------------------------------------------------------ GPU: rank decompression / compression

def rank_set(n_cols, seed=7300):
    """NN populated in every column (FULL, GAP with a few hundred holes, bit-block of density 0.97); sources: iid 0.3 bit-blocks,
    GAP runs, and a mix with NULL and FULL columns.  -> vectors, NN bits per column, source bits per column"""
    rng = np.random.default_rng(seed)
    nn, vecs = BVector(n_cols), [BVector(n_cols) for _ in range(3)]
    nn_bits, src_bits = [], [[], [], []]
    for c in range(n_cols):
        k = c % 3 if rng.random() < 0.5 else int(rng.integers(0, 3))
        if k == 0:
            b = np.ones(B, np.uint8)
        elif k == 1:
            b = np.ones(B, np.uint8)
            for s in rng.choice(np.arange(0, B - 8), int(rng.integers(1, 300)), replace=False):
                b[s:s + int(rng.integers(1, 8))] = 0
        else:
            b = (rng.random(B) < 0.97).astype(np.uint8)
        store_column([nn], c, b[None], lambda j: k == 2)
        nn_bits.append(b)
        cols = [(rng.random(B) < 0.3).astype(np.uint8),
                ((np.searchsorted(np.sort(rng.choice(np.arange(1, B), int(rng.integers(2, 600)), replace=False)), np.arange(B), side="right")
                  + int(rng.integers(0, 2))) & 1).astype(np.uint8),
                [np.zeros(B, np.uint8), np.ones(B, np.uint8), (rng.random(B) < 0.01).astype(np.uint8)][int(rng.integers(0, 3))]]
        for v, (vec, b2) in enumerate(zip(vecs, cols)):
            store_column([vec], c, b2[None], lambda j: v == 0)
            src_bits[v].append(b2)
    return [nn] + vecs, nn_bits, src_bits


def model_oracle(words_cols, flags):
    """Kinds, popcounts, digests, run counts, bits and GAP words of a result holding these columns: orc_aggregate of a one-member
    AND over them stored as bit-blocks (an empty column is NULL in every opt mode, as rank results are)."""
    v = BVector(len(words_cols))
    for c, w in enumerate(words_cols):
        v.set_bits(c, w)
    return orclib.oracle_aggregate(PackedSet.pack([v]), bm.OP_AND, [0], None, flags)


@gpu
def test_rank_decompress_and_compress(ctx):
    """bmb200_rank_decompress of a 3-group source and bmb200_rank_compress of every source, NN populated in every one of
    3 * (2 sm_count) + 40 columns (rank_decompress_kernel, rank_compress_scatter_kernel, finalize_blocks_kernel at fixed two CTAs
    per SM): == the numpy rank compressor per column, through orc_aggregate's result rules."""
    sm2 = grid(ctx)
    n = 3 * sm2 + 40
    vecs, nn_bits, src_bits = rank_set(n)
    dset = bm.DeviceSet.upload(ctx, PackedSet.pack(vecs, n))
    rs = bm.DeviceRS(ctx, dset, 0)
    # decompress: the 3 sources read as compressed bits (one group each)
    src = bm.aggregate_batch(ctx, dset, bm.OP_OR, [([1], []), ([2], []), ([3], [])], CMP)
    comp_all = [np.concatenate(s) for s in src_bits]
    for flags in (CMP, 0):
        out = bm.rank_decompress(ctx, rs, src, flags)
        want = []
        for s in comp_all:
            r = 0
            for c in range(n):
                cnt = int(nn_bits[c].sum())
                want.append(R.words_of(R.np_rank_decompress(nn_bits[c], s[r:r + cnt]), 1))
                r += cnt
        assert_oracle(collect(out, 3), model_oracle(want, flags), 3, f"rank_decompress flags={flags}")
        out.free()
    src.free()
    assert 3 * n >= 3 * sm2
    # compress every source
    total = sum(int(b.sum()) for b in nn_bits)
    ncomp = -(-total // B)
    assert ncomp >= 3 * sm2
    for v in range(3):
        bits = np.concatenate([R.np_rank_compress(nn_bits[c], src_bits[v][c]) for c in range(n)])
        want = R.words_of(bits, ncomp).reshape(ncomp, -1)
        out = bm.rank_compress(ctx, rs, 1 + v, CMP)
        assert_oracle(collect(out), model_oracle(list(want), CMP), 1, f"rank_compress {v}")
        out.free()
    rs.free(); dset.free()


# ------------------------------------------------------------------ GPU: GAP x GAP merge

def singles_gap(pos):
    """GAP block of isolated single bits at sorted positions (none adjacent)."""
    pos = np.asarray(pos, np.int64)
    if not pos.size:
        return np.array([1 << 3, B - 1], np.uint16)
    ends = np.stack([pos - 1, pos], 1).ravel()
    ends = ends[ends >= 0]
    if ends[-1] != B - 1:
        ends = np.concatenate([ends, [B - 1]])
    n = ends.size
    return np.concatenate([[(1 if pos[0] == 0 else 0) | (gap_level(n) << 1) | (n << 3)], ends]).astype(np.uint16)


MERGE_RUNS = [2, 3, 123, 124, 125, 126, 251, 252, 253, 507, 508, 509, 1275, 1276, 1277, 1278]


def merge_set(n_cols, seed=7400):
    """Two GAP vectors: column c holds single bits with a merged (OR / XOR) run count from MERGE_RUNS or drawn from 1..1300, split
    between the operands at a cut; the all-zero block now and then."""
    rng = np.random.default_rng(seed)
    va, vb = BVector(n_cols), BVector(n_cols)
    for c in range(n_cols):
        r = MERGE_RUNS[c % len(MERGE_RUNS)] if c < len(MERGE_RUNS) or rng.random() < 0.6 else int(rng.integers(1, 1301))
        at0 = r % 2 == 0
        m = (r - 1 - at0) // 2
        pos = 10 + 3 * np.arange(m)
        if at0:
            pos = np.concatenate([[0], pos])
        cut = int(rng.integers(max(0, pos.size - 630), min(pos.size, 630) + 1))     # both operands below 1276 runs
        va.set_gap(c, singles_gap(pos[:cut]))
        vb.set_gap(c, singles_gap(pos[cut:]))
    return PackedSet.pack([va, vb], n_cols)


def binop_oracle(ps, op, lo, hi):
    """The GAP x GAP result model: orc_aggregate's bits, popcounts, digests and run counts; kind GAP up to 1276 runs (the all-ones
    block included), bit-block above, NULL when empty; GAP words of the merged runs at their level."""
    g0, g1 = ([0], [1]) if op == bm.capi.OP_SUB else ([0, 1], None)
    okind, opop, odig, onr, oblk, ogap = orclib.oracle_aggregate(ps, bm.OP_AND_SUB if op == bm.capi.OP_SUB else op, g0, g1, CMP, lo, hi)
    kind = np.where(opop == 0, BLK_NULL, np.where(onr > GAP_THRESHOLD, BLK_BIT, BLK_GAP)).astype(np.uint8)
    for c in np.flatnonzero((kind == BLK_GAP) & (okind != BLK_GAP)):
        g = bits_to_gap(oblk[c])
        ogap[c, :] = 0
        ogap[c, :g.size] = g
    return kind, opop, odig, onr, oblk, ogap


@gpu
@pytest.mark.parametrize("op", list(REF_OP))
def test_binop_gap_merge(ctx, op):
    """bmb200_binop over GAP x GAP columns (gap_merge_kernel: one warp per column) at sm_count x 32 warps - 1, + 1 and 3 x + 7
    columns, merged run counts straddling 124 / 252 / 508 / 1276: == the GAP x GAP model."""
    w = grid(ctx, MERGE_WARPS)
    ps = merge_set(n_cols_for(w))
    dset = bm.DeviceSet.upload(ctx, ps)
    items = []
    for k, t in enumerate(targets(w)):
        lo, hi = col_range(k, t)
        o = binop_oracle(ps, op, lo, hi)
        if op == bm.OP_OR and k == 2:
            assert {124, 125, 252, 253, 508, 509, 1276, 1277} <= set(o[3].tolist())
        for flags in ((CMP, 0) if k == 2 and op == bm.OP_OR else (CMP,)):
            res = bm.capi.binop(ctx, dset, op, 0, 1, flags, lo, hi)
            got = collect(res); res.free()
            assert np.array_equal(got["kind"], o[0]), f"op={op} [{lo},{hi}) flags={flags}: kinds"
            assert_oracle(got, o, 1, f"binop op={op} [{lo},{hi}) flags={flags}")
        items.append(hi - lo)
    assert_deep(items, w)
    dset.free()


# ------------------------------------------------------------------ GPU: recycled results

@gpu
def test_recycled_results_across_grid_sizes(ctx, main):
    """A 3 grid + 7 column scan result recycled by a grid - 1 column mismatch, that one by a 3 grid + 7 column string search, and
    a grid - 1 column SCAN_IN result by a 3 grid + 7 column SHIFT-R-AND batch: each == a fresh call."""
    ms, dsets = main
    g = grid(ctx)
    d = dsets[True]
    rng = np.random.default_rng(600)
    big, small = col_range(0, 3 * g + 7), col_range(0, g - 1)
    vals = ms.eq_values(rng, 3)
    q = str_queries(ms, rng, 2, False)
    mm = mismatch_args(**mm_kw(ms), null_proc=MM_USE_NULL, flags=CMP, nb_from=small[0], nb_to=small[1])
    steps = [
        (lambda r: bm.scan(ctx, d, bm.SCAN_EQ, vals, P0, NPL, 0, CMP, *big, result=r), 3),
        (lambda r: bm.sv_mismatch(ctx, d, mm, result=r), 1),
        (lambda r: bm.scan_str(ctx, d, q, P0, NPL, NO_UNIVERSE, 0, *big, result=r), 2),
        (lambda r: bm.scan(ctx, d, SCAN_IN, vals, P0, 33, 0, CMP, *small, result=r), 1),
        (lambda r: bm.aggregate_batch(ctx, d, bm.OP_SHIFT_R_AND, [([5, 6], []), ([7], [])], CMP, *big, result=r), 2),
    ]
    r = None
    for i, (call, ng) in enumerate(steps):
        f = call(None)
        want = collect(f, ng); f.free()
        r = call(r)
        assert_same(collect(r, ng), want, f"step {i}")
    r.free()


# ------------------------------------------------------------------ CPU: the generators

SMALL_COLS = 60


@pytest.fixture(scope="module")
def small():
    return MainSet(SMALL_COLS, seed=7101, sample=SMALL_COLS)


def test_every_shape_and_plane_kind_occurs(small):
    ms = small
    assert set(ms.shapes[1:-1].tolist()) == set(range(len(SHAPES)))
    kinds = ms.ps[True].kinds()
    assert {int(k) for k in np.unique(kinds[:, P0:P0 + NPL])} == {BLK_NULL, BLK_FULL, BLK_BIT, BLK_GAP}
    assert {int(k) for k in np.unique(kinds[:, 0])} == {BLK_NULL, BLK_FULL, BLK_BIT, BLK_GAP}
    for s in ("iid", "runs", "near_limit", "all_gap"):
        cols = np.flatnonzero(ms.shapes == SH[s])
        k = kinds[cols, P0:P0 + NPL]
        if s == "iid":
            assert (k == BLK_BIT).any()
        if s == "all_gap":
            assert ((k == BLK_GAP) | (k == BLK_NULL) | (k == BLK_FULL)).all() and (k == BLK_GAP).any()
        if s in ("runs", "near_limit"):
            assert (k == BLK_GAP).any() and (k == BLK_BIT).any()  # GAP-able planes kept as bit-blocks among them
    const = np.flatnonzero(ms.shapes == SH["const"])
    assert np.isin(kinds[const, P0:P0 + NPL], [BLK_NULL, BLK_FULL]).all()
    assert (kinds[ms.ukind == "null", 0] == BLK_NULL).all() and (ms.ukind == "null").any()
    # GAP planes at their largest: some near_limit block has more than 1200 runs
    near = [int(ms.vecs[P0 + j].blocks[c][0]) >> 3 for c in np.flatnonzero(ms.shapes == SH["near_limit"]) for j in range(NPL)
            if ms.vecs[P0 + j].kind[c] == BLK_GAP]
    assert max(near) > 1200
    # GAP blocks with first run 0 and with first run 1
    firsts = {int(v.blocks[c][0]) & 1 for v in ms.vecs[P0:P0 + NPL] for c in range(ms.n_cols) if v.kind[c] == BLK_GAP}
    assert firsts == {0, 1}


def test_both_gap_forms(small):
    flat, raw = small.ps[True], small.ps[False]
    g_flat = (flat.desc & 3) == BLK_GAP
    assert g_flat.any() and np.array_equal(g_flat, (raw.desc & 3) == BLK_GAP)
    assert (flat.desc[g_flat] & (1 << 30)).all() and not (raw.desc[g_flat] & (1 << 30)).any()
    for v in (1, 30, 0):
        assert small.ps[True].vector(v).compare(small.vecs[v]) == 0 and small.ps[False].vector(v).compare(small.vecs[v]) == 0


def test_every_searched_column_has_hits(small):
    """The EQ searches of the GPU tests (the hot codes lead every list) hit every column but the no_match and NULL-universe ones;
    no present code matches in a no_match column, whole or as a string prefix."""
    ms = small
    hot = ms.eq_values(np.random.default_rng(0), 5)
    for c in range(1, ms.n_cols - 1):
        u, ok = ms.codes[c], ms.ubits[c].astype(bool)
        hit = np.isin(u, hot) & ok
        if ms.shapes[c] == SH["no_match"]:
            assert not np.isin(u, ms.pool).any() and not np.isin(u, hot).any()
            first = u & np.uint64(0xFF)
            assert ((first >= 0x21) & (first < 0x30)).all()
        elif ms.ukind[c] != "null":
            assert hit.any(), (c, SHAPES[ms.shapes[c]])


def test_intended_first_mismatches_are_the_true_ones(small):
    ms = small
    p_last, p_mid, p_null = ms.first_positions()
    N = ms.n_cols
    full = dict(size_a=N * B, size_b=N * B)
    kinds = ms.ps[True].kinds()
    (pm, d), = ms.edits[ms.c_mid]
    j = int(d).bit_length() - 1
    assert kinds[ms.c_mid, P0 + j] == BLK_GAP and kinds[ms.c_mid, PB0 + j] == BLK_BIT
    assert ms.c_mid < ms.last and any(c > ms.c_mid for c in ms.edits if c != ms.last)
    cases = [(mm_kw(ms, n_planes_a=1, n_planes_b=1, not_null_a=NO_UNIVERSE, not_null_b=NO_UNIVERSE, **full), MM_USE_NULL, p_last),
             (mm_kw(ms, not_null_b=0, **full), MM_USE_NULL, p_mid),
             (mm_kw(ms, not_null_a=NO_UNIVERSE, not_null_b=NO_UNIVERSE, **full), MM_NO_NULL, p_mid),
             (mm_kw(ms, plane0_b=P0, **full), MM_USE_NULL, p_null),
             (mm_kw(ms, plane0_b=P0, **full), MM_NO_NULL, None)]
    for kw, use, want in cases:
        for flat in (True, False):
            assert oracle_first(ms.ps[flat], mismatch_args(**kw, null_proc=use, nb_from=1, nb_to=ms.last + 1)) == want, (kw, use)
    # the vector form differs in the edited columns and nowhere else (NULL term aside)
    a = mismatch_args(**mm_kw(ms, not_null_a=NO_UNIVERSE, not_null_b=NO_UNIVERSE, **full), null_proc=MM_NO_NULL)
    pop = oracle_mismatch(ms.ps[True], a)[1]
    assert set(np.flatnonzero(pop).tolist()) == set(ms.edits)


def test_oracles_agree_with_numpy_on_sample_columns(small):
    """orc_scan / orc_scan_in / orc_scan_str on a few columns == the models the GPU tests apply to their sample columns."""
    ms = small
    rng = np.random.default_rng(1)
    ps = ms.ps[True]
    lo, hi = 1, ms.n_cols - 1
    full = np.uint64(2**64 - 1)
    for pred in (bm.SCAN_EQ, bm.SCAN_GT, bm.SCAN_LE, bm.SCAN_RANGE):
        vals = unsigned_searches(ms, rng, pred, 3, NPL)
        got = {"blocks": orclib.oracle_scan(ps, pred, vals, P0, NPL, 0, CMP, lo, hi)[4]}
        check_model(ms, got, lo, hi, [unsigned_model(pred, s, full) for s in vals], 0)
    mask = np.uint64(2**33 - 1)
    lst = np.unique(np.concatenate([ms.eq_values(rng, 5), ms.pool[:5000]]) & mask)
    got = {"blocks": oracle_scan_in(ps, lst, P0, 33, 0, CMP, lo, hi)[4]}
    check_model(ms, got, lo, hi, [lambda u: np.isin(u & mask, lst)], 0)
    for prefix in (False, True):
        q = str_queries(ms, rng, 3, prefix)
        got = {"blocks": oracle_scan_str(ps, q, P0, NPL, NO_UNIVERSE, F_STR_PREFIX if prefix else 0, lo, hi)[4]}
        check_model(ms, got, lo, hi, [str_model(s, prefix) for s in q], NO_UNIVERSE)


def test_merge_set_run_counts():
    """The GAP x GAP operands are valid GAP blocks, and their OR has every run count of MERGE_RUNS."""
    ps = merge_set(len(MERGE_RUNS) * 3)
    o = binop_oracle(ps, bm.OP_OR, 0, 0)
    assert set(MERGE_RUNS) <= set(o[3].tolist())
    for c in range(ps.n_blocks):
        for v in (0, 1):
            k, g = ps.block(v, c)
            assert k == BLK_GAP and (int(g[0]) >> 3) < GAP_THRESHOLD
