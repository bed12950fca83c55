"""Launch paths the other parity tests do not reach, each against the oracle and a plain numpy model of the operation:
long SHIFT-R-AND chains (shifts up to 65535 bits, per-group offsets), batches of every op over every member-list shape,
whole-set AND-SUB counts and OR targets, every scan kernel variant with 1..64 planes and 64-bit values, result kinds at the
GAP capacity limits, and results recycled across calls that differ in op, flags, width and entry point.

The numpy models are pinned against the oracle or the reference by the CPU tests at the end of this file."""
import numpy as np
import pytest

import bitmagic_b200 as bm
import gen
import orclib
import test_gpu_parity as tgp
import test_run_lists as trl
from bitmagic_b200.hostfmt import BLOCK_BITS, bits_to_gap, bits_to_words, calc_change, gap_level, words_to_bits

C = bm.F_OPT_COMPRESS
gpu = pytest.mark.gpu
needs_ref_answers = pytest.mark.skipif(not orclib.have_ref_answers(), reason="neither oracle/_ref/libbmref.so nor tests/golden/ref/")


# ------------------------------------------------------------------ shared helpers

def collect(res, n_groups=1, stored=True):
    """Everything a caller can read back from a result: metadata, totals, `any`, group totals and (stored) bits + GAP words."""
    kind, pop, dig, nr = res.meta()
    total, any_ = res.total()
    got = dict(kind=kind, pop=pop, dig=dig, nr=nr, total=total, any=any_, totals=res.group_totals(n_groups))
    if stored:
        fk, off, bits, gaps = res.fetch()
        assert np.array_equal(fk, kind)
        bv = bm.result_to_bvector(fk, off, bits, gaps)
        got["blocks"] = np.stack([bv.block_words(c) for c in range(kind.size)])
        got["gaps"] = [bv.blocks[c] if kind[c] == bm.BLK_GAP else None for c in range(kind.size)]
    return got


def assert_same(a, b, what=""):
    assert a.keys() == b.keys(), what
    for k in a:
        if k == "gaps":
            assert len(a[k]) == len(b[k]) and all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(a[k], b[k])), f"{what}: {k}"
        else:
            assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), f"{what}: {k}"


def oracle(ps, op, g0, g1, flags, nb_from=0, nb_to=0):
    """orc_aggregate for the stored result of a call with these flags (count-only / OR target do not change a group's result)."""
    return orclib.oracle_aggregate(ps, op, g0, g1, flags & C, nb_from, nb_to or ps.n_blocks)


def assert_oracle(got, o, n_groups=1, what=""):
    """got (collect) == the oracle's columns o (value- or group-major, n_groups groups), GAP words with their headers included."""
    okind, opop, odig, onr, oblk, ogap = o
    assert np.array_equal(got["pop"], opop), f"{what}: popcounts"
    assert np.array_equal(got["dig"], odig), f"{what}: digests"
    assert np.array_equal(got["nr"], onr), f"{what}: run counts"
    assert np.array_equal(got["kind"], okind), f"{what}: kinds {got['kind']} vs {okind}"
    assert np.array_equal(got["totals"], opop.reshape(n_groups, -1).sum(1, dtype=np.uint64)), f"{what}: group totals"
    assert got["total"] == int(opop.sum()) and got["any"] == bool(opop.sum()), f"{what}: total / any"
    if "blocks" in got:
        assert np.array_equal(got["blocks"], oblk), f"{what}: bits"
        for c in np.flatnonzero(okind == bm.BLK_GAP):
            assert np.array_equal(got["gaps"][c], ogap[c, :(int(ogap[c, 0]) >> 3) + 1]), f"{what}: GAP words of column {c}"


def concat_oracle(parts):
    return tuple(np.concatenate([p[i] for p in parts]) for i in range(6))


def bits_of(blocks):
    return words_to_bits(np.ascontiguousarray(blocks).reshape(-1))


def digest_of(bits):
    """64-wave non-zero bitmap of one block (calc_block_digest0)."""
    return sum(1 << w for w in range(64) if bits[w * 1024:(w + 1) * 1024].any())


def raises_code(code, fn, *a, **kw):
    with pytest.raises(bm.capi.BMB200Error) as e:
        fn(*a, **kw)
    assert e.value.code == code, str(e.value)


# ------------------------------------------------------------------ A. long SHIFT-R-AND chains

SHIFT_COLS = 5                                  # four data columns + the spare NULL column the carry out of column 3 lands in
SHIFT_N = [201, 256, 257, 1024, 4097, 32768, 65535, 65536]
F, B, G, N = range(4)                           # vector ids of shift_vectors()


def shift_vectors(seed=3):
    """F all-FULL; B mostly-ones bit-blocks with sparse zero bits, bits 0 and 65535 among them; G mostly-ones GAP blocks (first run
    1) with a few hundred zero runs; N FULL / bit / NULL / GAP in columns 0..3.  Column 4 is NULL everywhere."""
    rng = np.random.default_rng(seed)
    vf, vb, vg, vn = (bm.BVector(SHIFT_COLS) for _ in range(4))
    for c in range(4):
        vf.set_full(c)
        bits = np.ones(BLOCK_BITS, np.uint8)
        bits[rng.choice(BLOCK_BITS, 60, replace=False)] = 0
        bits[[0, BLOCK_BITS - 1]] = 0
        vb.set_bits(c, bits_to_words(bits))
        bits = np.ones(BLOCK_BITS, np.uint8)
        for s in rng.choice(np.arange(1, BLOCK_BITS - 8), 200, replace=False):
            bits[s:s + int(rng.integers(1, 4))] = 0
        vg.set_gap(c, bits_to_gap(bits_to_words(bits)))
    vn.set_full(0)
    vn.set_bits(1, vb.block_words(2))
    vn.set_gap(3, vg.blocks[1])
    return [vf, vb, vg, vn]


def shift_group(n):
    """n sources, mostly F, with B / G / N at chosen shifts s = n - 1 - k: word-quad aligned (the 128-bit path) and not, whole
    words and not, shifts that reach far into block nb - 1 (a GAP source there is read from K2 far below its last words)."""
    place = {n - 1: B}
    place.update({0: B, 1: G, 31: N, 32: B, 33: G, 128: B, 129: G, 160: B, 200: G, 255: N, 2049: N, 4096: B, 4097: G, 32767: G,
                  32768: B, 65503: G, 65504: B, 65535: G})
    g = [F] * n
    for s, v in place.items():
        if s < n:
            g[n - 1 - s] = v
    return g


def shift_closed_form(vecs, g):
    """result[p] = AND_k v_k[p - s_k], bits before position 0 read as 0, bits past the last column dropped.  The copies of F are one
    interval: ones from the largest of their shifts to 4 * 65536 + the smallest."""
    n, total = len(g), SHIFT_COLS * BLOCK_BITS
    shifts = {}
    for k, v in enumerate(g):
        shifts.setdefault(v, []).append(n - 1 - k)
    out = np.ones(total, np.uint8)
    for v, ss in shifts.items():
        if v == F:
            m = np.zeros(total, np.uint8)
            m[max(ss):4 * BLOCK_BITS + min(ss)] = 1
            out &= m
            continue
        bits = words_to_bits(vecs[v].to_words())
        for s in ss:
            sh = np.zeros(total, np.uint8)
            sh[s:] = bits[:total - s]
            out &= sh
    return out


def test_shift_group_covers_the_shift_classes():
    """The placements reach every class of shift the kernel distinguishes (pure host check of the test's own inputs)."""
    seen = set()
    for n in SHIFT_N:
        g = shift_group(n)
        for k, v in enumerate(g):
            if v != F:
                s = n - 1 - k
                seen |= {("quad0" if (s >> 5) % 4 == 0 else "quad"), ("word" if s % 32 == 0 else "bit"), s}
                if v == G and s >= 2048:
                    seen.add("gap_far")
    assert {"quad0", "quad", "word", "bit", 65535, 65504, 65503, "gap_far"} <= seen


@gpu
@pytest.mark.parametrize("n", SHIFT_N)
def test_long_shift_chains(ctx, n):
    """SHIFT-R-AND chains of up to 65536 sources (shifts up to 65535 bits) == the closed form and the oracle's per-source carry walk,
    flags 0 and C, and a shard (nb_from > 0) == the same columns of the full result."""
    vecs = shift_vectors()
    g = shift_group(n)
    want = shift_closed_form(vecs, g)
    assert want.any() and not want.all()
    ps = bm.PackedSet.pack(vecs)
    expect = {flags: oracle(ps, bm.OP_SHIFT_R_AND, g, None, flags) for flags in (0, C)}
    for flat in (True, False):
        ps = bm.PackedSet.pack(vecs, gap_flat=flat)
        dset = bm.DeviceSet.upload(ctx, ps)
        for flags in (0, C):
            o = expect[flags]
            assert np.array_equal(bits_of(o[4]), want)
            res = bm.aggregate(ctx, dset, bm.OP_SHIFT_R_AND, g, None, flags)
            got = collect(res); res.free()
            assert_oracle(got, o, what=f"n={n} flags={flags} flat={flat}")
            assert np.array_equal(bits_of(got["blocks"]), want)
        if flat:
            res = bm.aggregate(ctx, dset, bm.OP_SHIFT_R_AND, g, None, C, nb_from=2, nb_to=SHIFT_COLS)
            got = collect(res); res.free()
            assert_oracle(got, oracle(ps, bm.OP_SHIFT_R_AND, g, None, C, 2, SHIFT_COLS), what=f"n={n} shard")
            assert np.array_equal(bits_of(got["blocks"]), want[2 * BLOCK_BITS:])
        dset.free()


@gpu
def test_shift_batch_and_limits(ctx):
    """A batch of shift groups of different lengths (an empty one among them): every group's columns == its own oracle result and
    its own single aggregate; 65536 sources are accepted, 65537 refused with ERR_RANGE (single call and batch)."""
    vecs = shift_vectors()
    ps = bm.PackedSet.pack(vecs)
    dset = bm.DeviceSet.upload(ctx, ps)
    groups = [(shift_group(4097), []), ([], []), ([B], []), ([G, N], []), (shift_group(257), []), (shift_group(65536), [])]
    ng, nb = len(groups), ps.n_blocks
    for flags, nb_from in ((0, 0), (C, 0), (C, 1)):
        res = bm.aggregate_batch(ctx, dset, bm.OP_SHIFT_R_AND, groups, flags, nb_from=nb_from)
        got = collect(res, ng); res.free()
        o = concat_oracle([oracle(ps, bm.OP_SHIFT_R_AND, g0, None, flags, nb_from, nb) for g0, _ in groups])
        assert_oracle(got, o, ng, what=f"shift batch flags={flags} nb_from={nb_from}")
        w = nb - nb_from
        for gi, (g0, _) in enumerate(groups):
            single = collect(bm.aggregate(ctx, dset, bm.OP_SHIFT_R_AND, g0, None, flags, nb_from=nb_from))
            for k in ("kind", "pop", "dig", "nr", "blocks"):
                assert np.array_equal(single[k], got[k][gi * w:(gi + 1) * w]), (gi, k)
    raises_code(bm.capi.ERR_RANGE, bm.aggregate, ctx, dset, bm.OP_SHIFT_R_AND, [F] * 65537)
    raises_code(bm.capi.ERR_RANGE, bm.aggregate_batch, ctx, dset, bm.OP_SHIFT_R_AND, [([B], []), ([F] * 65537, [])])
    dset.free()


# ------------------------------------------------------------------ B. batches of every op

def batch_set(seed, op):
    """>= 16 GAP blocks per column (the FLAT window of a whole-pool group) and the edge blocks.  AND / XOR / SHIFT-R-AND: mixed block
    kinds.  OR / AND-SUB: sparse GAP vectors and the edge vectors without FULL blocks (AND-SUB: after four dense bit vectors for its AND
    groups), so that unions over the whole pool and subtractions of it are not trivially full or empty."""
    rng = np.random.default_rng(seed)
    if op in (bm.OP_OR, bm.OP_AND_SUB):
        edge = gen.edge_vectors(4)
        vecs = [bm.BVector.random(4, 0.7, rng) for _ in range(4 if op == bm.OP_AND_SUB else 0)]
        vecs += [bm.BVector.random(4, 10 ** rng.uniform(-3.6, -2.4), rng).optimize() for _ in range(60)] + edge[:2] + edge[3:]
    else:
        vecs = gen.mixed_vectors(rng, 64, 4, p_null=0.05, p_full=0.03, p_gap=0.6) + gen.edge_vectors(4)
    ps = bm.PackedSet.pack(vecs)
    assert all(int((ps.kinds()[c] == bm.BLK_GAP).sum()) >= 16 for c in range(ps.n_blocks))
    return rng, vecs, ps


def batch_groups(rng, op, n):
    """Sorted whole pool (streamed, FLAT window), > 1024 members with duplicates (several classification passes), descending (gather),
    one or two members, empty.  AND-SUB: a small AND group with each of these shapes as its SUB group."""
    shapes = [list(range(n)), rng.integers(0, n, 1100).tolist(), list(range(n - 1, 1, -3)), [7, 40], [int(rng.integers(0, n))], []]
    if op == bm.OP_AND_SUB:
        return [([1], shapes[0][2:]), ([2, 3], shapes[1]), ([3, 0], shapes[2]), ([9], shapes[3]), (shapes[4], [5]), ([], [])]
    if op == bm.OP_AND:            # long AND groups are empty; the short ones carry the bits
        return [(shapes[0], []), (shapes[1], []), (shapes[2][:3], []), (shapes[3], []), (shapes[4], []), ([], [])]
    return [(s, []) for s in shapes]


@gpu
@pytest.mark.parametrize("op", [bm.OP_OR, bm.OP_AND, bm.OP_XOR, bm.OP_SHIFT_R_AND, bm.OP_AND_SUB])
def test_batches_of_every_op(ctx, op):
    """bmb200_aggregate_batch for every op over every member-list shape, flags 0 / C / C|OR_TARGET / COUNT_ONLY, nb_from 0 and 1,
    GAP mode 0 and 1: each group == its own single aggregate == the oracle, group totals, OR target == union of the groups."""
    rng, vecs, ps = batch_set(50 + op, op)
    groups = batch_groups(rng, op, ps.n_vec)
    ng = len(groups)
    dset = bm.DeviceSet.upload(ctx, ps)
    cache = {}
    try:
        for mode in (0, 1):
            ctx.set_tuning(bm.capi.TUNE_GAP_MODE, mode)
            for nb_from in (0, 1):
                w = ps.n_blocks - nb_from
                for flags in (0, C, C | bm.F_OR_TARGET, bm.F_COUNT_ONLY):
                    key = (flags & C, nb_from)
                    if key not in cache:
                        cache[key] = [oracle(ps, op, g0, g1, flags, nb_from) for g0, g1 in groups]
                    per = cache[key]
                    stored = not flags & bm.F_COUNT_ONLY
                    res = bm.aggregate_batch(ctx, dset, op, groups, flags, nb_from=nb_from)
                    what = f"op={op} mode={mode} nb_from={nb_from} flags={flags}"
                    got = collect(res, ng, stored)
                    assert_oracle(got, concat_oracle(per), ng, what)
                    if flags & bm.F_OR_TARGET:
                        o = res.or_target(w)
                        union = np.bitwise_or.reduce(np.stack([p[4] for p in per]), axis=0)
                        ob = bm.result_to_bvector(*o.fetch())
                        assert np.array_equal(np.stack([ob.block_words(c) for c in range(w)]), union), what + ": OR target"
                        o.free()
                    res.free()
                    if flags in (0, bm.F_COUNT_ONLY):
                        for gi, (g0, g1) in enumerate(groups):
                            r1 = bm.aggregate(ctx, dset, op, g0, g1, flags, nb_from=nb_from)
                            single = collect(r1, 1, stored); r1.free()
                            for k in ("kind", "pop", "dig", "nr") + (("blocks",) if stored else ()):
                                assert np.array_equal(single[k], got[k][gi * w:(gi + 1) * w]), f"{what} group {gi}: {k}"
    finally:
        ctx.set_tuning(bm.capi.TUNE_GAP_MODE, 0)
        dset.free()


# ------------------------------------------------------------------ C. whole-set AND-SUB: counts and OR target

@gpu
def test_whole_set_count_only_and_or_target(ctx):
    """Whole-set AND-SUB (agg_pipe_kernel when the pipeline is on) with F_COUNT_ONLY, and as a one-group batch with C | OR_TARGET,
    under TUNE_RUN_LISTS 0 / 2 and TUNE_AGG_PIPELINE 1 / 0: totals, per-column popcounts, digests, kinds and the OR target == the
    oracle in every arm."""
    rng = np.random.default_rng(61)
    vecs = trl.shaped_vectors(rng, 6)
    n = len(vecs)
    g0 = [n - 2, n - 1]
    g1 = [v for v in rng.permutation(n).tolist() if v not in g0]
    ps = bm.PackedSet.pack(vecs)
    o0, oc = oracle(ps, bm.OP_AND_SUB, g0, g1, 0), oracle(ps, bm.OP_AND_SUB, g0, g1, C)
    assert oc[1].sum() > 0
    try:
        for pipe in (1, 0):
            for rl in (0, 2):
                ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, pipe)
                ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, rl)
                dset = bm.DeviceSet.upload(ctx, ps)
                what = f"pipeline={pipe} run_lists={rl}"
                res = bm.aggregate(ctx, dset, bm.OP_AND_SUB, g0, g1, bm.F_COUNT_ONLY)
                assert_oracle(collect(res, 1, stored=False), o0, what=what + " count-only")
                res.free()
                res = bm.aggregate_batch(ctx, dset, bm.OP_AND_SUB, [(g0, g1)], C | bm.F_OR_TARGET)
                assert_oracle(collect(res), oc, what=what + " batch")
                o = res.or_target(ps.n_blocks)
                assert_oracle(collect(o), oc, what=what + " OR target")
                o.free(); res.free()
                dset.free()
    finally:
        ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, 1)
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)


# ------------------------------------------------------------------ D. scan launch shapes

SCAN_PLANES = [1, 32, 33, 63, 64]
SCAN_COLS = 3
SPECIAL = [0, 1, 2**32 - 1, 2**32, 2**63, 2**64 - 1]
CONST = 0xA5A5A5A5A5A5A5A5


def scan_values(npl, seed=9):
    """Element values over SCAN_COLS columns, masked to npl bits: column 0 random 64-bit values with the special values sprinkled in,
    column 1 runs of ~300 equal values (GAP planes), column 2 one constant (FULL / NULL planes)."""
    rng = np.random.default_rng(seed)
    mask = np.uint64(2**npl - 1)
    c0 = rng.integers(0, 2**64, BLOCK_BITS, dtype=np.uint64)
    c0[rng.choice(BLOCK_BITS, 600, replace=False)] = np.array(SPECIAL * 100, np.uint64)
    pool = np.array(SPECIAL + rng.integers(0, 2**64, 10, dtype=np.uint64).tolist(), np.uint64)
    c1 = np.repeat(pool[rng.integers(0, pool.size, BLOCK_BITS // 300 + 1)], 300)[:BLOCK_BITS]
    c2 = np.full(BLOCK_BITS, CONST, np.uint64)
    return np.concatenate([c0, c1, c2]) & mask


def scan_universes(seed=10):
    """(GAP universe, bit-block universe) over SCAN_COLS columns."""
    rng = np.random.default_rng(seed)
    ug, ub = bm.BVector(SCAN_COLS), bm.BVector(SCAN_COLS)
    for c in range(SCAN_COLS):
        ug.set_gap(c, gen.gap_from_runs([99, 39999 - 1000 * c, 49999, 64999, 65535], 0))
        ub.set_bits(c, bits_to_words(rng.random(BLOCK_BITS) < 0.7))
    return ug, ub


def scan_set(npl, gap_flat=True):
    """[dummy] + the npl planes of scan_values + [GAP universe, bit universe]: plane0 = 1."""
    vals = scan_values(npl)
    planes = [bm.BVector.from_words(bits_to_words(((vals >> np.uint64(j)) & np.uint64(1)).astype(np.uint8))).optimize() for j in range(npl)]
    ug, ub = scan_universes()
    dummy = bm.BVector.random(SCAN_COLS, 0.5, np.random.default_rng(11))
    ps = bm.PackedSet.pack([dummy] + planes + [ug, ub], gap_flat=gap_flat)
    return vals, ps, {"none": (bm.NO_UNIVERSE, None), "gap": (npl + 1, ug), "bit": (npl + 2, ub)}


def scan_model(vals, pred, search, uni=None):
    """Value-major bits of every search: rebuild each element's value from the planes (vals) and apply the predicate."""
    out = []
    for s in search:
        if pred == bm.SCAN_RANGE:
            lo, hi = sorted(int(x) for x in s)
            m = (vals >= np.uint64(lo)) & (vals <= np.uint64(hi))
        else:
            x = np.uint64(int(s))
            m = {bm.SCAN_EQ: vals == x, bm.SCAN_GT: vals > x, bm.SCAN_GE: vals >= x, bm.SCAN_LT: vals < x, bm.SCAN_LE: vals <= x}[pred]
        if uni is not None:
            m &= words_to_bits(uni.to_words()).astype(bool)
        out.append(m.astype(np.uint8))
    return np.concatenate(out)


def scan_searches(npl, vals, pred):
    """Five launches of 1, 2, 3, 4, 5 values (every <VG, MODE> variant, every short last group) that together hold every special value,
    values above the top plane, duplicates in one launch; RANGE: [0, 2^64-1], [2^63, 2^64-1], a reversed range, lo == hi."""
    if pred == bm.SCAN_RANGE:
        base = [[0, 2**64 - 1], [2**63, 2**64 - 1], [int(vals[70000]), int(vals[5])], [int(vals[65536 + 400])] * 2, [2**32 - 1, 2**32],
                [1, CONST], [0, 0], [2**npl if npl < 64 else 2**64 - 2, 2**64 - 1]]
    else:
        base = SPECIAL + [CONST & (2**npl - 1), int(vals[123]), int(vals[65536 + 1000])] + ([2**npl, 2**npl + 5] if npl < 64 else [])
    out, off = [], 0
    for nv in range(1, 6):
        s = [base[(off + t) % len(base)] for t in range(nv)]
        if nv >= 3:
            s[-1] = s[0]                                   # a duplicate value in one launch
        out.append(s)
        off += nv
    return out


@gpu
@pytest.mark.parametrize("npl", SCAN_PLANES)
def test_scan_launch_shapes(ctx, npl):
    """Every scan kernel variant (1..5 values per launch for every predicate), 1 / 32 / 33 / 63 / 64 planes over 64-bit element values,
    universe absent / GAP / bit-block, FLAT and raw planes: == the oracle and the numpy model; nb_from > 0, nb_to < n_blocks and the
    count-only totals against both too."""
    for gap_flat, unis in ((True, ("none", "gap", "bit")), (False, ("gap",))):
        vals, ps, universes = scan_set(npl, gap_flat)
        dset = bm.DeviceSet.upload(ctx, ps)
        for un in unis:
            uni, ubv = universes[un]
            for pred in (bm.SCAN_EQ, bm.SCAN_GT, bm.SCAN_GE, bm.SCAN_LT, bm.SCAN_LE, bm.SCAN_RANGE):
                for search in scan_searches(npl, vals, pred):
                    blocks = tgp.check_scan(ctx, ps, dset, pred, search, 1, npl, uni, C if (len(search) + pred) % 2 else 0)
                    assert np.array_equal(bits_of(blocks), scan_model(vals, pred, search, ubv)), (npl, un, pred, search)
                # column sub-ranges and count-only totals, 3 values
                search = scan_searches(npl, vals, pred)[2]
                model = scan_model(vals, pred, search, ubv).reshape(len(search), SCAN_COLS, BLOCK_BITS)
                for nb_from, nb_to in ((1, 0), (0, 2), (1, 2)):
                    hi = nb_to or SCAN_COLS
                    res = bm.scan(ctx, dset, pred, search, 1, npl, uni, C, nb_from=nb_from, nb_to=nb_to)
                    got = collect(res, len(search)); res.free()
                    assert_oracle(got, orclib.oracle_scan(ps, pred, search, 1, npl, uni, C, nb_from, nb_to), len(search), f"scan range {nb_from}-{nb_to}")
                    assert np.array_equal(bits_of(got["blocks"]), model[:, nb_from:hi].reshape(-1))
                res = bm.scan(ctx, dset, pred, search, 1, npl, uni, bm.F_COUNT_ONLY)
                got = collect(res, len(search), stored=False); res.free()
                assert np.array_equal(got["totals"], model.reshape(len(search), -1).sum(1, dtype=np.uint64))
                assert np.array_equal(got["pop"], model.sum(2, dtype=np.uint32).reshape(-1))
                assert_oracle(got, orclib.oracle_scan(ps, pred, search, 1, npl, uni, 0), len(search), "scan count-only")
        dset.free()


# ------------------------------------------------------------------ E. result kinds at the GAP limits

BINOP_RUNS = [2, 124, 125, 252, 253, 508, 509, 1275, 1276, 1277]
REF_OP = {bm.OP_OR: 0, bm.OP_AND: 1, bm.capi.OP_SUB: 2, bm.OP_XOR: 3}


def exact_run_bits(runs, at0, at_end):
    """Isolated single bits with exactly `runs` runs: optional 1 at bit 0, m bits at 10 + 3i, optional 1 at bit 65535."""
    m = (runs - 1 - at0 - at_end) // 2
    assert 2 * m + 1 + at0 + at_end == runs and m >= 0
    bits = np.zeros(BLOCK_BITS, np.uint8)
    bits[10 + 3 * np.arange(m)] = 1
    bits[0], bits[BLOCK_BITS - 1] = at0, at_end
    return bits, 10 + 3 * (m // 2) - 1


def binop_cases():
    """(result bits, cut) per column: all-zero, all-ones, then every count of BINOP_RUNS once with the runs away from bit 65535 and
    once touching it (and bit 0 where the parity allows both)."""
    cases = [(np.zeros(BLOCK_BITS, np.uint8), 1000), (np.ones(BLOCK_BITS, np.uint8), 1000)]
    for r in BINOP_RUNS:
        odd = (r - 1) % 2
        cases.append(exact_run_bits(r, odd, 0))
        cases.append(exact_run_bits(r, 0, 1) if odd else exact_run_bits(r, 1, 1))
    return cases


def binop_operands(op, res, cut):
    """GAP operands a, b with a OP b == res: res is split at `cut` (a zero bit) between the two operands."""
    first = np.arange(BLOCK_BITS) < cut
    ones, zeros = np.ones(BLOCK_BITS, np.uint8), np.zeros(BLOCK_BITS, np.uint8)
    if op in (bm.OP_OR, bm.OP_XOR):
        a, b = np.where(first, res, zeros), np.where(first, zeros, res)
    elif op == bm.OP_AND:
        a, b = np.where(first, res, ones), np.where(first, ones, res)
    else:                                                       # SUB: a & ~b
        a, b = np.where(first, res, ones), np.where(first, zeros, 1 - res)
    return a.astype(np.uint8), b.astype(np.uint8)


def binop_set(op):
    """Two GAP-only vectors (0 = a, 1 = b): column c holds the operands of binop_cases()[c]."""
    cases = binop_cases()
    va, vb = bm.BVector(len(cases)), bm.BVector(len(cases))
    for c, (res, cut) in enumerate(cases):
        a, b = binop_operands(op, res, cut)
        for v, x in ((va, a), (vb, b)):
            g = bits_to_gap(bits_to_words(x))
            assert (int(g[0]) >> 3) < bm.capi.GAP_THRESHOLD
            v.set_gap(c, g)
    return bm.PackedSet.pack([va, vb])


def binop_model(ps, op, va, vb):
    """The reference's result of a GAP x GAP column (gap_buff_op + clone_gap_block): the merged run list as a GAP block at level
    gap_calc_level(runs); all-zero -> nothing stored; more than 1276 runs -> bit-block.  -> dict like collect()."""
    f = {bm.OP_OR: np.bitwise_or, bm.OP_AND: np.bitwise_and, bm.OP_XOR: np.bitwise_xor, bm.capi.OP_SUB: lambda x, y: x & (1 - y)}[op]
    kind, pop, dig, nr, blocks, gaps = [], [], [], [], [], []
    for c in range(ps.n_blocks):
        a = words_to_bits(ps.vector(va).block_words(c))
        b = words_to_bits(ps.vector(vb).block_words(c))
        r = f(a, b).astype(np.uint8)
        w = bits_to_words(r)
        runs = calc_change(w)
        if runs > bm.capi.GAP_THRESHOLD:
            k = bm.BLK_BIT
        elif runs == 1 and not r[0]:
            k = bm.BLK_NULL
        else:
            k = bm.BLK_GAP
        g = bits_to_gap(w) if k == bm.BLK_GAP else None
        if g is not None:
            assert (int(g[0]) >> 1) & 3 == gap_level(runs)
        kind.append(k); pop.append(int(r.sum())); dig.append(digest_of(r)); nr.append(runs); blocks.append(w); gaps.append(g)
    pop = np.array(pop, np.uint32)
    return dict(kind=np.array(kind, np.uint8), pop=pop, dig=np.array(dig, np.uint64), nr=np.array(nr, np.uint32),
                total=int(pop.sum()), any=bool(pop.sum()), totals=np.array([pop.sum()], np.uint64), blocks=np.stack(blocks), gaps=gaps)


def model_slice(m, lo, hi):
    out = {k: (v[lo:hi] if k in ("kind", "pop", "dig", "nr", "blocks", "gaps") else v) for k, v in m.items()}
    out["total"] = int(out["pop"].sum()); out["any"] = bool(out["total"]); out["totals"] = np.array([out["total"]], np.uint64)
    return out


@gpu
@pytest.mark.parametrize("op", list(REF_OP))
def test_binop_result_kinds_at_the_gap_limits(ctx, op):
    """bmb200_binop over GAP x GAP columns whose merged result has exactly 1 (all-zero and all-ones), 2, 124 / 125, 252 / 253, 508 / 509
    and 1275 / 1276 / 1277 runs, runs touching bits 0 and 65535, and a == b: kinds, GAP words with their level, bits, popcounts, run
    counts, digests == the model, flags 0 and C, sub-ranges == the columns of the full-range result."""
    ps = binop_set(op)
    dset = bm.DeviceSet.upload(ctx, ps)
    for va, vb in ((0, 1), (0, 0), (1, 1)):
        want = binop_model(ps, op, va, vb)
        if (va, vb) == (0, 1):
            assert sorted(set(want["nr"].tolist())) == [1] + BINOP_RUNS
        for flags in (0, C):
            res = bm.capi.binop(ctx, dset, op, va, vb, flags)
            assert_same(collect(res), want, f"op={op} ({va},{vb}) flags={flags}")
            res.free()
            for lo, hi in ((3, 9), (1, 0), (ps.n_blocks - 1, 0)):
                res = bm.capi.binop(ctx, dset, op, va, vb, flags, lo, hi)
                assert_same(collect(res), model_slice(want, lo, hi or ps.n_blocks), f"op={op} ({va},{vb}) flags={flags} [{lo},{hi})")
                res.free()
    dset.free()


EPILOGUE_RUNS = [2, 123, 124, 125, 126, 252, 253, 508, 509, 1275, 1276, 1277]


def epilogue_set(seed=12):
    """Vector 0: bit-blocks with exactly EPILOGUE_RUNS[c] runs; 1: dense random bit-blocks X; 2: vector 0 XOR X (bit-blocks)."""
    rng = np.random.default_rng(seed)
    e, x, y = (bm.BVector(len(EPILOGUE_RUNS)) for _ in range(3))
    for c, r in enumerate(EPILOGUE_RUNS):
        w = gen.block_with_exact_runs(r)
        assert calc_change(w) == r
        xw = rng.integers(0, 2**32, 2048, dtype=np.uint64).astype(np.uint32)
        e.set_bits(c, w); x.set_bits(c, xw); y.set_bits(c, w ^ xw)
    return bm.PackedSet.pack([e, x, y])


@gpu
def test_aggregation_epilogue_at_the_gap_limits(ctx):
    """The aggregation epilogue with C stores GAP only below 1276 runs, at the level of the run count: a one-member OR and a two-member
    XOR whose results have exactly 123 .. 1277 runs == the oracle, kinds and GAP levels as the rule says."""
    ps = epilogue_set()
    dset = bm.DeviceSet.upload(ctx, ps)
    runs = np.array(EPILOGUE_RUNS)
    for op, g0 in ((bm.OP_OR, [0]), (bm.OP_XOR, [1, 2]), (bm.OP_OR, [0, 0])):
        got = tgp.check_vs_oracle(ctx, ps, op, g0, None, C, dset)
        assert np.array_equal(got["nr"], runs)
        assert np.array_equal(got["kind"], np.where(runs < bm.capi.GAP_THRESHOLD, bm.BLK_GAP, bm.BLK_BIT))
        res = bm.aggregate(ctx, dset, op, g0, None, C)
        gaps = collect(res)["gaps"]; res.free()
        for c in np.flatnonzero(runs < bm.capi.GAP_THRESHOLD):
            assert (int(gaps[c][0]) >> 1) & 3 == gap_level(int(runs[c])) and int(gaps[c][0]) >> 3 == runs[c]
    dset.free()


# ------------------------------------------------------------------ F. recycled results

def recycle_set(seed=14):
    rng = np.random.default_rng(seed)
    vecs = gen.mixed_vectors(rng, 14, 4, p_null=0.05, p_full=0.05, p_gap=0.5) + gen.edge_vectors(4)[:2]
    return bm.PackedSet.pack(vecs)


def fresh(fn, *a, n_groups=1, stored=True, **kw):
    res = fn(*a, **kw)
    got = collect(res, n_groups, stored)
    res.free()
    return got


@gpu
def test_recycled_results_equal_fresh_calls(ctx):
    """result= a handle of an earlier call, for aggregate / aggregate_batch / scan / binop, across a change of op, compress <-> none,
    count-only <-> stored, OR target -> none, column count, and entry point (binop -> aggregate, aggregate -> binop, scan -> batch):
    everything fetched == a fresh call, totals, `any` and GAP words included."""
    ps = recycle_set()
    dset = bm.DeviceSet.upload(ctx, ps)
    n = ps.n_vec
    AS, OR = bm.OP_AND_SUB, bm.OP_OR
    agg = lambda op, g0, g1, flags, **kw: (bm.aggregate, ctx, dset, op, g0, g1, flags)  # noqa: E731
    steps = [  # (call, kw, stored)
        (agg(OR, list(range(n)), None, bm.F_COUNT_ONLY), {}, False),
        (agg(OR, list(range(n)), None, C), {}, True),                           # count-only -> stored
        (agg(AS, [0, 1], list(range(2, n)), C), {}, True),                      # op
        (agg(AS, [0, 1], list(range(2, n)), 0), {}, True),                      # compress -> none
        (agg(bm.OP_XOR, [3, 4, 5], None, C), {}, True),                         # none -> compress, op
        (agg(bm.OP_XOR, [3, 4, 5], None, bm.F_COUNT_ONLY), {}, False),          # stored -> count-only
        (agg(bm.OP_AND, [0, 2], None, C), dict(nb_from=1), True),               # column count
        ((bm.capi.binop, ctx, dset, bm.capi.OP_SUB, 2, 3, C), dict(nb_from=1), True),    # aggregate -> binop
        ((bm.capi.binop, ctx, dset, bm.OP_XOR, 4, 5, 0), {}, True),             # binop, column count
        (agg(bm.OP_SHIFT_R_AND, [6, 7, 8], None, 0), {}, True),                 # binop -> aggregate
    ]
    r = bm.DeviceResult(ctx)
    for i, (call, kw, stored) in enumerate(steps):
        fn, *a = call
        want = fresh(fn, *a, stored=stored, **kw)
        r = fn(*a, result=r, **kw)
        assert_same(collect(r, 1, stored), want, f"step {i}")
    r.free()

    groups = [([0], list(range(5, n))), ([1, 2], [3]), ([4], [])]
    bsteps = [
        (bm.OP_OR, [(list(range(n)), []), ([3, 4], []), ([], [])], C | bm.F_OR_TARGET),
        (AS, groups, C),                                                        # OR target -> none, op
        (AS, groups, bm.F_COUNT_ONLY),
        (AS, groups, C | bm.F_OR_TARGET),                                       # count-only -> stored + OR target
        (bm.OP_XOR, [([0, 1, 2], []), ([5], []), (list(range(n)), [])], 0),     # OR target -> none, compress -> none
    ]
    r = bm.DeviceResult(ctx)
    for i, (op, gs, flags) in enumerate(bsteps):
        stored = not flags & bm.F_COUNT_ONLY
        want = fresh(bm.aggregate_batch, ctx, dset, op, gs, flags, n_groups=3, stored=stored)
        r = bm.aggregate_batch(ctx, dset, op, gs, flags, result=r)
        assert_same(collect(r, 3, stored), want, f"batch step {i}")
        if flags & bm.F_OR_TARGET:
            f = bm.aggregate_batch(ctx, dset, op, gs, flags)
            fo, o = f.or_target(ps.n_blocks), r.or_target(ps.n_blocks)
            assert_same(collect(o), collect(fo), f"batch step {i}: OR target")
            fo.free(); o.free(); f.free()
    # scan -> scan (another predicate, count-only) -> batch of as many groups
    sargs = (ctx, dset)
    r = bm.scan(*sargs, bm.SCAN_EQ, [0, 1, 5], 0, 6, bm.NO_UNIVERSE, C, result=r)
    assert_same(collect(r, 3), fresh(bm.scan, *sargs, bm.SCAN_EQ, [0, 1, 5], 0, 6, bm.NO_UNIVERSE, C, n_groups=3), "scan")
    r = bm.scan(*sargs, bm.SCAN_RANGE, [[1, 9], [7, 2], [0, 63]], 0, 6, 9, bm.F_COUNT_ONLY, result=r)
    assert_same(collect(r, 3, False), fresh(bm.scan, *sargs, bm.SCAN_RANGE, [[1, 9], [7, 2], [0, 63]], 0, 6, 9, bm.F_COUNT_ONLY,
                                             n_groups=3, stored=False), "scan count-only")
    r = bm.scan(*sargs, bm.SCAN_GT, [0, 1, 5], 0, 6, 9, 0, result=r)
    assert_same(collect(r, 3), fresh(bm.scan, *sargs, bm.SCAN_GT, [0, 1, 5], 0, 6, 9, 0, n_groups=3), "scan after count-only")
    r = bm.aggregate_batch(ctx, dset, AS, groups, C, result=r)
    assert_same(collect(r, 3), fresh(bm.aggregate_batch, ctx, dset, AS, groups, C, n_groups=3), "scan -> batch")
    r.free()
    dset.free()


@gpu
def test_or_target_of_a_recycled_result_without_one_is_refused(ctx):
    """A batch launched without F_OR_TARGET into a result recycled from a batch that had one keeps the OR buffer;
    bmb200_result_or_target must refuse it (ERR_BADARG) instead of returning the earlier call's union, and work again once a batch
    with F_OR_TARGET has been launched into it."""
    ps = recycle_set()
    dset = bm.DeviceSet.upload(ctx, ps)
    n = ps.n_vec
    groups = [([0], list(range(3, n))), ([1], [2])]
    r = bm.aggregate_batch(ctx, dset, bm.OP_AND_SUB, groups, C | bm.F_OR_TARGET)
    r.or_target(ps.n_blocks).free()
    r = bm.aggregate_batch(ctx, dset, bm.OP_OR, [([4, 5], []), ([6], [])], C, result=r)
    raises_code(bm.capi.ERR_BADARG, r.or_target, ps.n_blocks)
    r = bm.aggregate(ctx, dset, bm.OP_OR, [4, 5], None, C, result=bm.aggregate_batch(ctx, dset, bm.OP_OR, [([1], [])], C | bm.F_OR_TARGET))
    raises_code(bm.capi.ERR_BADARG, r.or_target, ps.n_blocks)
    r.free()
    r = bm.aggregate_batch(ctx, dset, bm.OP_OR, [([4, 5], []), ([6], [])], C)
    raises_code(bm.capi.ERR_BADARG, r.or_target, ps.n_blocks)
    r = bm.aggregate_batch(ctx, dset, bm.OP_OR, [([4, 5], []), ([6], [])], C | bm.F_OR_TARGET, result=r)
    o = r.or_target(ps.n_blocks)
    _, _, _, _, want, _ = oracle(ps, bm.OP_OR, [4, 5, 6], None, C)
    ob = bm.result_to_bvector(*o.fetch())
    assert np.array_equal(np.stack([ob.block_words(c) for c in range(ps.n_blocks)]), want)
    o.free(); r.free(); dset.free()


# ------------------------------------------------------------------ CPU: the models against the oracle and the reference

@needs_ref_answers
def test_shift_65536_chain_oracle_matches_reference():
    """One n = 65536 chain: the oracle's per-source carry walk == aggregator::combine_shift_right_and == the closed form."""
    vecs = shift_vectors()
    ps = bm.PackedSet.pack(vecs)
    g = shift_group(65536)
    want = shift_closed_form(vecs, g)
    okind, opop, odig, onr, oblk, ogap = oracle(ps, bm.OP_SHIFT_R_AND, g, None, C)
    rkind, rpop, rblk, rgap, rany = orclib.ref_aggregate(ps, bm.OP_SHIFT_R_AND, g, None, C)
    assert np.array_equal(bits_of(oblk), want) and np.array_equal(rblk, oblk)
    assert np.array_equal(rpop, opop) and np.array_equal(rkind, okind) and np.array_equal(rgap, ogap) and rany == bool(opop.sum())


def test_shift_closed_form_matches_oracle():
    """The closed form against the oracle on chains of every length the GPU tests use but the longest."""
    vecs = shift_vectors()
    ps = bm.PackedSet.pack(vecs)
    for n in SHIFT_N[:5]:
        g = shift_group(n)
        assert np.array_equal(bits_of(oracle(ps, bm.OP_SHIFT_R_AND, g, None, 0)[4]), shift_closed_form(vecs, g)), n


@pytest.mark.parametrize("npl", [1, 33, 64])
def test_scan_model_matches_oracle(npl):
    """The scan model (values rebuilt from the planes, predicate applied) == orc_scan, every predicate, GAP and bit universes."""
    vals, ps, universes = scan_set(npl)
    for un in ("none", "gap", "bit"):
        uni, ubv = universes[un]
        for pred in (bm.SCAN_EQ, bm.SCAN_GT, bm.SCAN_GE, bm.SCAN_LT, bm.SCAN_LE, bm.SCAN_RANGE):
            search = scan_searches(npl, vals, pred)[4]
            oblk = orclib.oracle_scan(ps, pred, search, 1, npl, uni, C)[4]
            model = scan_model(vals, pred, search, ubv)
            assert model.any() and np.array_equal(bits_of(oblk), model), (npl, un, pred, search)


@needs_ref_answers
@pytest.mark.parametrize("op", list(REF_OP))
@pytest.mark.parametrize("compress", [False, True])
def test_binop_model_matches_reference(op, compress):
    """The GAP x GAP result model (kinds, GAP words and levels, bits, popcounts) == bvector::bit_or / bit_and / bit_sub / bit_xor."""
    ps = binop_set(op)
    for va, vb in ((0, 1), (1, 1)):
        want = binop_model(ps, op, va, vb)
        rkind, rpop, rblk, rgap = orclib.ref_binop_gaps(ps, REF_OP[op], va, vb, compress)
        assert np.array_equal(rkind, want["kind"]), (op, va, vb, rkind, want["kind"])
        assert np.array_equal(rpop, want["pop"]) and np.array_equal(rblk, want["blocks"])
        for c in range(ps.n_blocks):
            if want["gaps"][c] is not None:
                assert np.array_equal(rgap[c, :want["gaps"][c].size], want["gaps"][c]), c
