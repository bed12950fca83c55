"""Block columns past 65535, i.e. bit positions past 2^32: the address range a BM64ADDR build of bm::bvector<> reaches.

CPU: the plain-C oracle against the reference built with -DBM64ADDR (oracle/_ref/libbmref64.so) on sets of 66 000 block
columns whose blocks sit on both sides of column 65535 / 65536 (bit 2^32), and the host-only store_result_check64.
GPU: every device entry point on such sets against the oracle -- scans (plain, signed, string), two-operand ops with their
result kinds, SHIFT-R-AND carries across column 65535, whole-set AND-SUB under every pipeline / run-list setting and column
offset, single-column fetches and group totals, rank compression where the compressed positions pass 2^32, deserialization of
64-bit BLOB streams -- and the BM64ADDR builds of the bvector-level binding harnesses.

The expected results are compared column by column; no test expands a set to one byte per bit (that would be 4 GB here)."""
from __future__ import annotations

import subprocess

import numpy as np
import pytest

import bitmagic_b200 as bm
import orclib
import rsclib as R
from bitmagic_b200.hostfmt import BLOCK_BITS, BLOCK_WORDS, bits_to_gap, bits_to_words

gpu = pytest.mark.gpu
C = bm.F_OPT_COMPRESS
NB = 66000                                        # block columns of every set here: 66000 * 65536 bits > 2^32
EDGE = list(range(65528, 65546))                  # the columns around 2^32 (column 65536 starts at bit 2^32)
COLS = [0, 3] + EDGE + [NB - 1]                   # every populated column
G = 1 << 32
needs_ref64 = pytest.mark.skipif(not orclib.have_ref(True), reason="oracle/_ref/libbmref64.so not built")


# ---------------------------------------------------------------- fixtures
def rand_words(rng, density):
    return bits_to_words(rng.random(BLOCK_BITS) < density)


def run_gap(rng, n_runs):
    """a GAP block of n_runs 1-runs of random length"""
    b = np.zeros(BLOCK_BITS, np.uint8)
    for s in rng.choice(BLOCK_BITS - 64, n_runs, replace=False):
        b[s:s + 1 + int(rng.integers(0, 40))] = 1
    return bits_to_gap(bits_to_words(b))


def edge_vector(rng, density, p_full=0.1, p_gap=0.3, p_null=0.15, cols=COLS):
    """one vector of NB columns: bit / GAP / FULL / NULL blocks in `cols` only"""
    v = bm.BVector(NB)
    for c in cols:
        r = rng.random()
        if r < p_null and c not in (65535, 65536):          # the two columns at bit 2^32 are never empty
            continue
        if r < p_null + p_full:
            v.set_full(c)
        elif r < p_null + p_full + p_gap:
            v.set_gap(c, run_gap(rng, int(rng.integers(1, 300))))
        else:
            v.set_bits(c, rand_words(rng, density))
    return v


def edge_set(seed, nv, **kw):
    rng = np.random.default_rng(seed)
    return [edge_vector(rng, 0.6 / (k + 1), **kw) for k in range(nv)]


WINDOWS = [(0, 6), (EDGE[0], EDGE[-1] + 1), (NB - 1, NB)]     # every populated column, and the empty column 5


def oracle_windowed(fn, nv, *args):
    """fn(*args, nb_from, nb_to) -> 6 arrays, value-major over nv values, evaluated on WINDOWS only (the oracle's scans expand
    every column, minutes at 66 000 columns).  Every other column is empty in every vector, so its answer is column 5's.
    -> full-length kind / popcount / digest / run-count arrays and {result column: bits / GAP words} of the windows"""
    parts = [fn(*args, a, b) for a, b in WINDOWS]
    meta = []
    for i in range(4):
        full = np.repeat(parts[0][i].reshape(nv, 6)[:, 5:6], NB, axis=1)
        for p, (a, b) in zip(parts, WINDOWS):
            full[:, a:b] = p[i].reshape(nv, b - a)
        meta.append(full.reshape(-1))
    blk, gap = {}, {}
    for p, (a, b) in zip(parts, WINDOWS):
        for k in range(nv):
            for c in range(a, b):
                blk[k * NB + c] = p[4][k * (b - a) + c - a]
                gap[k * NB + c] = p[5][k * (b - a) + c - a]
    return (*meta, blk, gap)


def check_result(res, o, n_groups=1, stored=True, what=""):
    """a device result == the oracle's columns o: kinds, popcounts, digests, run counts, totals, and (stored) the bits of every
    bit-block and the words of every GAP block -- read in the result's compact form, never expanded.  o's bits and GAP words
    are arrays over every column or, from oracle_windowed, maps of the columns that can hold them."""
    okind, opop, odig, onr, oblk, ogap = o
    if isinstance(oblk, dict):
        cols = np.array(sorted(oblk), np.int64)
        assert not np.isin(np.flatnonzero((okind == bm.BLK_BIT) | (okind == bm.BLK_GAP)), cols, invert=True).any()
        idx = {c: i for i, c in enumerate(cols.tolist())}
        oblk = np.stack([oblk[c] for c in cols.tolist()]); ogap = np.stack([ogap[c] for c in cols.tolist()])
        row = lambda c: idx[int(c)]
    else:
        row = lambda c: int(c)
    kind, pop, dig, nr = res.meta()
    assert np.array_equal(kind, okind), f"{what}: kinds differ at columns {np.flatnonzero(kind != okind)[:10]}"
    assert np.array_equal(pop, opop), f"{what}: popcounts differ at columns {np.flatnonzero(pop != opop)[:10]}"
    assert np.array_equal(dig, odig) and np.array_equal(nr, onr), f"{what}: digests / run counts"
    assert np.array_equal(res.group_totals(n_groups), opop.reshape(n_groups, -1).sum(1, dtype=np.uint64)), f"{what}: group totals"
    total, any_ = res.total()
    assert total == int(opop.sum(dtype=np.uint64)) and any_ == bool(total), f"{what}: total"
    if not stored:
        return
    fk, off, bits, gaps = res.fetch()
    assert np.array_equal(fk, okind)
    cb = np.flatnonzero(fk == bm.BLK_BIT)
    want = oblk[[row(c) for c in cb]] if cb.size else np.zeros((0, BLOCK_WORDS), np.uint32)
    assert np.array_equal(bits.reshape(-1, BLOCK_WORDS)[off[cb].astype(np.int64)], want), f"{what}: bits"
    for c in np.flatnonzero(fk == bm.BLK_GAP):
        g = ogap[row(c)]
        n = (int(g[0]) >> 3) + 1
        assert np.array_equal(gaps[int(off[c]):int(off[c]) + n], g[:n]), f"{what}: GAP words of column {c}"


# ---------------------------------------------------------------- CPU: the oracle against the BM64ADDR reference
@needs_ref64
def test_oracle_matches_reference64_past_column_65535():
    """orc_aggregate == bm::aggregator of the BM64ADDR reference on a 66 000-column set, every op, both storage modes"""
    ps = bm.PackedSet.pack(edge_set(64, 8))
    for op, g0, g1, flags in [(bm.OP_OR, range(8), None, 0), (bm.OP_OR, range(8), None, C), (bm.OP_AND, [0, 1, 2], None, C),
                              (bm.OP_AND_SUB, [0, 1], range(2, 8), C), (bm.OP_XOR, [0, 3, 5], None, 0)]:
        g0 = list(g0); g1 = list(g1) if g1 is not None else None
        rkind, rpop, rblk, rgap, rany = orclib.ref_aggregate(ps, op, g0, g1, flags, addr64=True)
        okind, opop, odig, onr, oblk, ogap = orclib.oracle_aggregate(ps, op, g0, g1, flags)
        # (an uncompressed XOR of GAP blocks stays GAP in the reference and is a bit-block in the oracle, at any column)
        assert (op == bm.OP_XOR or np.array_equal(rkind, okind)) and np.array_equal(rpop, opop), (op, flags)
        nz = np.flatnonzero(okind != bm.BLK_NULL)
        assert np.array_equal(rblk[nz], oblk[nz]) and rany == bool(opop.sum()), (op, flags)
        if op == bm.OP_OR:
            assert opop[65535] and opop[65536], "the set must straddle bit 2^32"


@needs_ref64
def test_oracle_rank_select_matches_reference64_past_2_32():
    ps = bm.PackedSet.pack(edge_set(65, 2))
    rng = np.random.default_rng(3)
    pos = np.concatenate([rng.integers(0, NB * BLOCK_BITS, 4000), [G - 1, G, G + 1, 65535 * BLOCK_BITS, NB * BLOCK_BITS - 1]]).astype(np.uint64)
    total = int(orclib.oracle_rank(ps, 1, [NB * BLOCK_BITS - 1])[0])
    rank = np.concatenate([rng.integers(1, total + 1, 4000), [0, total, total + 1]]).astype(np.uint64)
    r_rank, r_pos, r_found, _ = orclib.ref_rank_select(ps, 1, pos, rank, addr64=True)
    o_pos, o_found = orclib.oracle_select(ps, 1, rank)
    assert np.array_equal(r_rank, orclib.oracle_rank(ps, 1, pos))
    assert np.array_equal(r_found, o_found) and np.array_equal(r_pos[r_found], o_pos[o_found])
    assert int(o_pos[o_found].max()) >= G


@needs_ref64
@pytest.mark.parametrize("level", [0, 2, 6])
def test_oracle_deserializes_reference64_streams_past_column_65535(level):
    """BM64ADDR BLOBs (64-bit header fields, block indexes past 65535): the oracle's decoder == bm::deserialize == the vector"""
    vecs = edge_set(66, 4)
    ps = bm.PackedSet.pack(vecs)
    for v in range(ps.n_vec):
        blob = orclib.ref_serialize(ps, v, level, addr64=True)
        rkind, rpop, rblk, rgap = orclib.ref_deserialize(blob, NB, addr64=True)
        rc, okind, oblk, ogap = orclib.oracle_deserialize(blob, NB)
        assert rc == 0 and np.array_equal(okind, rkind), (level, v)
        want = np.stack([vecs[v].block_words(c) for c in COLS])
        assert np.array_equal(rblk[COLS], want) and np.array_equal(oblk[COLS], want), (level, v)
        assert not rpop[np.setdiff1d(np.arange(NB), COLS)].any()


def test_store_result_check64():
    """host-only: the binding's result store at shard offsets past column 65535 and its upload extent (BM64ADDR build)"""
    exe = orclib.ORACLE_DIR / "_ref" / "store_result_check64"
    if not exe.exists():
        pytest.skip("oracle/_ref/store_result_check64 is built only where the reference tree exists")
    p = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "OK" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


# ---------------------------------------------------------------- GPU: C-ABI parity past column 65535
@gpu
@pytest.mark.parametrize("signed", [False, True])
def test_scan_past_column_65535(ctx, signed):
    """bmb200_scan (plain and F_SIGNED) over 12 planes + a universe whose populated columns sit around 2^32"""
    import test_scan_signed as tss
    vecs = edge_set(67 + signed, 13, p_null=0.05)
    ps = bm.PackedSet.pack(vecs)
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        if signed:
            cases = [(bm.SCAN_EQ, [0, -1, 5, -2048]), (bm.SCAN_LT, [0, -3, 1000]), (bm.SCAN_GE, [-(1 << 11), 7]),
                     (bm.SCAN_RANGE, [[-100, 100], [5, -5]])]
        else:
            cases = [(bm.SCAN_EQ, [0, 1, 4095, 4096]), (bm.SCAN_GT, [0, 2000]), (bm.SCAN_LE, [17, 4095]), (bm.SCAN_RANGE, [[3, 900], [50, 2]])]
        flags = C | (bm.F_SIGNED if signed else 0)
        for pred, vals in cases:
            nv = len(vals)
            res = bm.scan(ctx, dset, pred, vals, 0, 12, 12, flags)
            o = oracle_windowed(tss.oracle_scan_signed if signed else orclib.oracle_scan, nv, ps, pred, vals, 0, 12, 12, flags)
            check_result(res, o, nv, what=f"scan pred {pred} signed={signed}")
            res.free()
            res = bm.scan(ctx, dset, pred, vals, 0, 12, bm.NO_UNIVERSE, flags | bm.F_COUNT_ONLY)
            o = oracle_windowed(tss.oracle_scan_signed if signed else orclib.oracle_scan, nv, ps, pred, vals, 0, 12, bm.NO_UNIVERSE, flags)
            assert np.array_equal(res.group_totals(nv), o[1].reshape(nv, -1).sum(1, dtype=np.uint64)), f"count-only pred {pred}"
            res.free()
    finally:
        dset.free()


@gpu
@pytest.mark.parametrize("prefix", [False, True])
def test_scan_str_past_column_65535(ctx, prefix):
    """bmb200_scan_str over 16 string planes (two bytes) + a universe, populated around 2^32"""
    import test_scan_str as tst
    vecs = edge_set(69 + prefix, 17, p_null=0.05, p_full=0.25)
    ps = bm.PackedSet.pack(vecs)
    dset = bm.DeviceSet.upload(ctx, ps)
    flags = C | (bm.F_STR_PREFIX if prefix else 0)

    def stored(c, p):                             # the string the planes hold at bit p of column c
        bits = [(int(vecs[j].block_words(c)[p >> 5]) >> (p & 31)) & 1 for j in range(16)]
        s = bytes(sum(bits[8 * k + b] << b for b in range(8)) for k in range(2))
        return s.split(b"\0")[0]
    held = [stored(c, p) for c, p in ((65535, 65535), (65536, 0), (65536, 777), (65537, 12345))]
    try:
        for strs in ([b"\xff\xff", b"\x01", b"a"] + held, [b"\xff", b"\x03\x80", b"", b"\x7f\xff\x01"] + [h[:1] for h in held]):
            res = bm.scan_str(ctx, dset, strs, 0, 16, 16, flags)
            check_result(res, oracle_windowed(tst.oracle_scan_str, len(strs), ps, strs, 0, 16, 16, flags), len(strs), what=f"scan_str {strs} prefix={prefix}")
            res.free()
    finally:
        dset.free()


@gpu
def test_binop_every_op_past_column_65535(ctx):
    """bmb200_binop OR / AND / XOR / SUB over columns around 2^32: bits against the oracle; result kinds against the same op on
    the same blocks moved down to columns 0.. (the reference's binop where its library is present, else the device's)"""
    vecs = edge_set(71, 4, p_gap=0.45, p_full=0.15)
    ps = bm.PackedSet.pack(vecs)
    lo = bm.PackedSet.pack([v.slice(EDGE[0], EDGE[-1] + 1) for v in vecs])
    dset = bm.DeviceSet.upload(ctx, ps)
    dlo = bm.DeviceSet.upload(ctx, lo)
    agg_of = {bm.OP_OR: bm.OP_OR, bm.OP_AND: bm.OP_AND, bm.OP_XOR: bm.OP_XOR}
    ref_op = {bm.OP_OR: 0, bm.OP_AND: 1, bm.capi.OP_SUB: 2, bm.OP_XOR: 3}
    try:
        for op in (bm.OP_OR, bm.OP_AND, bm.OP_XOR, bm.capi.OP_SUB):
            for va, vb in ((0, 1), (2, 3), (1, 2)):
                if op == bm.capi.OP_SUB:
                    o = orclib.oracle_aggregate(ps, bm.OP_AND_SUB, [va], [vb], 0)
                else:
                    o = orclib.oracle_aggregate(ps, agg_of[op], [va, vb], None, 0)
                for flags in (0, C):
                    res = bm.capi.binop(ctx, dset, op, va, vb, flags)
                    kind, pop, _, _ = res.meta()
                    assert np.array_equal(pop, o[1]), (op, va, vb, flags)
                    fk, off, bits, gaps = res.fetch()
                    got = bm.result_to_bvector(fk, off, bits, gaps)
                    assert np.array_equal(np.stack([got.block_words(c) for c in COLS]), o[4][COLS]), (op, va, vb, flags)
                    if orclib.have_ref():
                        want_kind = orclib.ref_binop(lo, ref_op[op], va, vb, bool(flags))[0]
                    else:
                        r2 = bm.capi.binop(ctx, dlo, op, va, vb, flags); want_kind = r2.meta()[0]; r2.free()
                    assert np.array_equal(kind[EDGE[0]:EDGE[-1] + 1], want_kind), (op, va, vb, flags)
                    res.free()
    finally:
        dlo.free(); dset.free()


@gpu
def test_shift_right_and_carries_across_column_65535(ctx):
    """SHIFT-R-AND chains of 2..6 sources, dense in columns 65534..65537: at every step bit 2^32 - 1 (the last bit of column 65535)
    moves to bit 2^32"""
    rng = np.random.default_rng(72)
    vecs = []
    for k in range(6):
        v = bm.BVector(NB)
        for c in (0, 65534, 65535, 65536, 65537, NB - 1):
            w = rand_words(rng, 0.85)
            if c == 65535:
                w[-1] |= np.uint32(0xFF000000)        # the last 8 bits below 2^32 and the first 8 above it in every source:
            if c == 65536:
                w[0] |= np.uint32(0xFF)               # T_k keeps bit 2^32, carried out of column 65535 at every step
            v.set_bits(c, w)
        if k == 3:
            v.set_full(65536)
        if k >= 4:
            v.optimize()
        vecs.append(v)
    ps = bm.PackedSet.pack(vecs)
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        for n in range(2, 7):
            for flags in (0, C):
                res = bm.aggregate(ctx, dset, bm.OP_SHIFT_R_AND, list(range(n)), None, flags)
                o = orclib.oracle_aggregate(ps, bm.OP_SHIFT_R_AND, list(range(n)), None, flags)
                check_result(res, o, what=f"shift-r-and n={n} flags={flags}")
                assert o[4][65536][0] & 1, "the carry out of column 65535 must survive"
                res.free()
    finally:
        dset.free()


def and_sub_set(seed):
    """AND group: two dense vectors of bit and FULL blocks, no GAP block and no sparse (listed) bit-block, so that the whole-set
    kernel may stream the run-list companion; SUB group: GAP sources of isolated singles and runs (part A) and sparse bit-blocks
    (part B).  Populated around 2^32 and in the last column."""
    rng = np.random.default_rng(seed)
    cols = EDGE + [NB - 1]
    vecs = [edge_vector(rng, 0.7, p_full=0.2, p_gap=0.0, p_null=0.0, cols=cols), edge_vector(rng, 0.6, p_full=0.1, p_gap=0.0, p_null=0.0, cols=cols)]
    for k in range(6):
        v = bm.BVector(NB)
        for c in cols:
            r = rng.random()
            if r < 0.4:
                v.set_gap(c, run_gap(rng, int(rng.integers(1, 200))))
            elif r < 0.7:
                v.set_bits(c, rand_words(rng, 0.003))
            elif r < 0.75:
                v.set_full(c)
        vecs.append(v)
    return vecs


@gpu
@pytest.mark.parametrize("pipeline", [0, 1])
@pytest.mark.parametrize("run_lists", [0, 2])
def test_whole_set_and_sub_past_column_65535(ctx, pipeline, run_lists):
    """whole-set AND-SUB under TUNE_AGG_PIPELINE x TUNE_RUN_LISTS, columns from 0, 65530 and 65536 to the end, stored,
    count-only, and as a batch with an OR target.  With the streamed kernel and TUNE_RUN_LISTS 2 the calls take the run-list
    companion, parts A and B, whose sizes must equal a host count of the set's runs; otherwise no companion is built."""
    from test_bit_run_lists import host_bit_run_list_bytes
    from test_run_lists import host_run_list_bytes
    vecs = and_sub_set(73)
    ps = bm.PackedSet.pack(vecs)
    g0, g1 = [0, 1], list(range(2, len(vecs)))
    assert not any((v.kind == bm.BLK_GAP).any() for v in vecs[:2]), "a GAP block in the AND group disables the run lists"
    ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, pipeline)
    ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, run_lists)
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        for nb_from in (0, 65530, 65536):
            o = orclib.oracle_aggregate(ps, bm.OP_AND_SUB, g0, g1, C, nb_from, NB)
            res = bm.aggregate(ctx, dset, bm.OP_AND_SUB, g0, g1, C, nb_from, NB)
            check_result(res, o, what=f"and-sub nb_from={nb_from}")
            res.free()
            res = bm.aggregate(ctx, dset, bm.OP_AND_SUB, g0, g1, C | bm.F_COUNT_ONLY, nb_from, NB)
            check_result(res, o, stored=False, what=f"and-sub count-only nb_from={nb_from}")
            res.free()
        if pipeline and run_lists:
            a_bytes, b_bytes = dset.run_list_bytes(), dset.bit_run_list_bytes()
            assert a_bytes == host_run_list_bytes(ps) and a_bytes != (0, 0), f"part A: {a_bytes}"
            assert b_bytes == host_bit_run_list_bytes(ps) and b_bytes[2] > 0, f"part B: {b_bytes}"
        else:
            assert dset.run_list_bytes() == (0, 0) and dset.bit_run_list_bytes() == (0, 0, 0)
        groups = [(g0, g1), ([0], [2, 3]), ([1, 0], [4, 5, 6, 7])]
        o = [orclib.oracle_aggregate(ps, bm.OP_AND_SUB, a, b, C, 65530, NB) for a, b in groups]
        res = bm.aggregate_batch(ctx, dset, bm.OP_AND_SUB, groups, C | bm.F_OR_TARGET, 65530, NB)
        check_result(res, tuple(np.concatenate([x[i] for x in o]) for i in range(6)), len(groups), what="batch")
        ores = res.or_target(NB - 65530)
        fk, off, bits, gaps = ores.fetch()
        got = bm.result_to_bvector(fk, off, bits, gaps)
        want = o[0][4] | o[1][4] | o[2][4]
        assert np.array_equal(np.stack([got.block_words(c - 65530) for c in EDGE[2:] + [NB - 1]]), want[[c - 65530 for c in EDGE[2:] + [NB - 1]]])
        assert not ores.meta()[1][np.setdiff1d(np.arange(NB - 65530), [c - 65530 for c in EDGE[2:] + [NB - 1]])].any()
        ores.free(); res.free()
    finally:
        ctx.set_tuning(bm.capi.TUNE_AGG_PIPELINE, 1)
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)
        dset.free()


@gpu
def test_fetch_column_and_group_totals_past_column_65535(ctx):
    vecs = edge_set(74, 5)
    ps = bm.PackedSet.pack(vecs)
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        groups = [([0, 1], None), ([2], [3, 4])]
        res = bm.aggregate_batch(ctx, dset, bm.OP_AND_SUB, groups, C)
        o = [orclib.oracle_aggregate(ps, bm.OP_AND_SUB, a, b, C) for a, b in groups]
        assert np.array_equal(res.group_totals(2), np.array([x[1].sum(dtype=np.uint64) for x in o], np.uint64))
        for g in range(2):
            for c in COLS:
                k, bits, gap = res.fetch_column(g * NB + c)
                assert k == o[g][0][c], (g, c)
                if k == bm.BLK_BIT:
                    assert np.array_equal(bits, o[g][4][c]), (g, c)
                if k == bm.BLK_GAP:
                    assert np.array_equal(gap, o[g][5][c, :gap.size]), (g, c)
        res.free()
    finally:
        dset.free()


@gpu
def test_rank_compress_decompress_with_base_past_2_32(ctx):
    """NN = 65 537 FULL blocks (count 2^32 + 65536) then a bit-block, a GAP block and a sparse block: compressed positions of the
    tail pass 2^32.  The expected result is computed block by block: inside the FULL prefix rank compression is the identity,
    the tail is restated in numpy on its own three blocks."""
    rng = np.random.default_rng(75)
    nb = 65541
    nn = bm.BVector(nb)
    for c in range(65537):
        nn.set_full(c)
    tail = [rng.random(BLOCK_BITS) < 0.4, np.zeros(BLOCK_BITS, bool), rng.random(BLOCK_BITS) < 0.002]
    for s in range(100, BLOCK_BITS - 300, 900):
        tail[1][s:s + 250] = True
    nn.set_bits(65537, bits_to_words(tail[0])); nn.set_gap(65538, bits_to_gap(bits_to_words(tail[1]))); nn.set_bits(65539, bits_to_words(tail[2]))
    src = bm.BVector(nb)
    src_cols = {c: rng.random(BLOCK_BITS) < 0.3 for c in (0, 65535, 65536, 65537, 65538, 65539, 65540)}   # 65540: outside NN, dropped
    for c, b in src_cols.items():
        src.set_bits(c, bits_to_words(b))
    comp_in = bm.BVector(nb)                      # a vector in the compressed space, for decompression
    cin_cols = {c: rng.random(BLOCK_BITS) < 0.2 for c in (1, 65535, 65536, 65537, 65538)}
    for c, b in cin_cols.items():
        comp_in.set_bits(c, bits_to_words(b))
    nn_tail = np.concatenate([t.astype(np.uint8) for t in tail])
    src_tail = np.concatenate([src_cols[c].astype(np.uint8) for c in (65537, 65538, 65539)])
    want_tail = R.np_rank_compress(nn_tail, src_tail)          # compressed bits from position 65537 * 65536 on
    n_tail_cols = -(-int(nn_tail.sum()) // BLOCK_BITS)
    want_tail_words = R.words_of(want_tail, n_tail_cols).reshape(-1, BLOCK_WORDS)
    ps = bm.PackedSet.pack([nn, src, comp_in])
    dset = bm.DeviceSet.upload(ctx, ps)
    rs = bm.DeviceRS(ctx, dset, 0)
    try:
        assert rs.total() == 65537 * BLOCK_BITS + int(nn_tail.sum())
        comp = bm.rank_compress(ctx, rs, 1, C)
        assert comp.n_cols == 65537 + n_tail_cols
        fk, off, bits, gaps = comp.fetch()
        got = bm.result_to_bvector(fk, off, bits, gaps)
        pop = comp.meta()[1]
        for c in (0, 65535, 65536):
            assert np.array_equal(got.block_words(c), bits_to_words(src_cols[c])), c
        for k in range(n_tail_cols):
            assert np.array_equal(got.block_words(65537 + k), want_tail_words[k]), 65537 + k
        live = [0, 65535, 65536] + [65537 + k for k in range(n_tail_cols)]
        assert not pop[np.setdiff1d(np.arange(comp.n_cols), live)].any()
        assert comp.total()[0] == sum(int(src_cols[c].sum()) for c in (0, 65535, 65536)) + int(want_tail.sum())
        # decompression of comp_in (entered as a result, the form bmb200_rank_decompress reads)
        src_res = bm.aggregate(ctx, dset, bm.OP_OR, [2], None, 0)
        back = bm.rank_decompress(ctx, rs, src_res, C)
        assert back.n_cols == nb
        fk, off, bits, gaps = back.fetch()
        got = bm.result_to_bvector(fk, off, bits, gaps)
        for c in (1, 65535, 65536):
            assert np.array_equal(got.block_words(c), bits_to_words(cin_cols[c])), c
        cin_tail = np.concatenate([cin_cols[c].astype(np.uint8) for c in (65537, 65538)])
        want_back = R.np_rank_decompress(nn_tail, cin_tail)
        for k in range(3):
            assert np.array_equal(got.block_words(65537 + k), bits_to_words(want_back[k * BLOCK_BITS:(k + 1) * BLOCK_BITS].astype(bool))), 65537 + k
        bpop = back.meta()[1]
        assert not bpop[np.setdiff1d(np.arange(nb), [1, 65535, 65536, 65537, 65538, 65539])].any()
        for h in (back, src_res, comp):
            h.free()
    finally:
        rs.free(); dset.free()


@gpu
@needs_ref64
@pytest.mark.parametrize("level", [2, 6])
def test_upload_blobs_of_reference64_streams_past_column_65535(ctx, level):
    """bmb200_set_upload_blobs on BM64ADDR BLOBs of vectors whose blocks lie past column 65535 == bm::deserialize"""
    vecs = edge_set(76, 6)
    ps = bm.PackedSet.pack(vecs)
    blobs = [orclib.ref_serialize(ps, v, level, addr64=True) for v in range(ps.n_vec)]
    dset = bm.DeviceSet.upload_blobs(ctx, blobs, NB)
    try:
        got = dset.download()
        for v in range(ps.n_vec):
            rkind, _, rblk, rgap = orclib.ref_deserialize(blobs[v], NB, addr64=True)
            bv = got.vector(v)
            assert np.array_equal(bv.kind, rkind), f"level {level} vector {v}: kinds"
            assert np.array_equal(np.stack([bv.block_words(c) for c in COLS]), rblk[COLS]), f"level {level} vector {v}: bits"
        o = orclib.oracle_aggregate(ps, bm.OP_AND_SUB, [0, 1], [2, 3, 4, 5], C)
        res = bm.aggregate(ctx, dset, bm.OP_AND_SUB, [0, 1], [2, 3, 4, 5], C)
        assert np.array_equal(res.meta()[1], o[1])
        res.free()
    finally:
        dset.free()


@gpu
@pytest.mark.parametrize("name", ["test_cxx_binding64", "test_rsc_binding64", "test_signed_binding64", "test_str_binding64"])
def test_binding_harness_bm64addr(name):
    """the bvector-level binding harnesses built with -DBM64ADDR: their 32-bit checks on 2^48 - 1-bit default vectors, plus
    vectors, sparse vectors and rank compression past 2^32, against the unmodified reference"""
    exe = orclib.ORACLE_DIR / "_ref" / name
    if not exe.exists():
        pytest.skip(f"oracle/_ref/{name} is built only where the reference tree exists")
    p = subprocess.run([str(exe)], capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-2000:]
    assert ("OK:" if name == "test_cxx_binding64" else " 0 failed") in p.stdout, p.stdout[-2000:]
