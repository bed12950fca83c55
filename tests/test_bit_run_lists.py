"""Part B of the run-list companion: the 1-runs of every sparse SUB-group bit-block (a listed block: its list takes at most
kListBitMax bytes), streamed by the whole-set AND-SUB kernel in place of the listed 8 KB blocks when the AND group holds no GAP
block and no listed block.  Building on the first call (TUNE_RUN_LISTS 2) and never building (0) must agree bit for bit with each
other and with the oracle, and part B's size must match a host count of the listed blocks' runs."""
import re
from pathlib import Path

import numpy as np
import pytest

import bitmagic_b200 as bm
import gen
import orclib
from bitmagic_b200.hostfmt import bits_to_words, BLOCK_BITS
from test_run_lists import run, host_run_list_bytes, run_block

pytestmark = pytest.mark.gpu

C = bm.F_OPT_COMPRESS
OP = bm.OP_AND_SUB
LIST_MAX = int(re.search(r"kListBitMax\s*=\s*(\d+)u", (Path(bm.__file__).parent / "csrc" / "runlist_kernel.cuh").read_text()).group(1))


def block_runs(words):
    """(singles, long runs) of a bit-block in the companion's encoding: a run from bit 0 longer than one bit counts in both."""
    bits = np.unpackbits(np.asarray(words, np.uint32).view(np.uint8), bitorder="little").astype(np.int8)
    d = np.diff(np.concatenate([[0], bits, [0]]))
    s, e = np.flatnonzero(d == 1), np.flatnonzero(d == -1) - 1
    return int(((s == e) | (s == 0)).sum()), int((e > s).sum())


def host_bit_run_list_bytes(ps):
    """(singles bytes, long-run bytes, listed blocks) of part B, counted on the host, each column's parts padded to 16 bytes."""
    sgl = lr = n = 0
    for nb in range(ps.n_blocks):
        ns = nl = 0
        for v in range(ps.n_vec):
            k, w = ps.block(v, nb)
            if k != bm.BLK_BIT:
                continue
            s, l = block_runs(w)
            if 2 * s + 4 * l <= LIST_MAX:
                ns += s; nl += l; n += 1
        sgl += (ns + 7) // 8 * 16; lr += (nl + 3) // 4 * 16
    return sgl, lr, n


def check(ctx, ps, g0, g1, flags, nb_from=0, nb_to=0, part_b=True):
    dset = bm.DeviceSet.upload(ctx, ps)
    try:
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 2)
        new = run(ctx, dset, g0, g1, flags, nb_from, nb_to)
        a_bytes, b_bytes = dset.run_list_bytes(), dset.bit_run_list_bytes()
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 0)
        old = run(ctx, dset, g0, g1, flags, nb_from, nb_to)
    finally:
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)
        dset.free()
    assert a_bytes == host_run_list_bytes(ps)
    assert b_bytes == host_bit_run_list_bytes(ps)
    assert b_bytes[2] > 0
    if part_b:                        # the call really had listed blocks to skip: none in the AND group
        listed = {v for v in range(ps.n_vec) for nb in range(ps.n_blocks)
                  if ps.block(v, nb)[0] == bm.BLK_BIT and 2 * block_runs(ps.block(v, nb)[1])[0] + 4 * block_runs(ps.block(v, nb)[1])[1] <= LIST_MAX}
        assert not listed & set(g0)
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


def bits_block(positions_runs):
    """Bit-block with the given inclusive 1-runs [(s, e), ...]."""
    bits = np.zeros(BLOCK_BITS, np.uint8)
    for s, e in positions_runs:
        bits[s:e + 1] = 1
    return bits_to_words(bits)


def singles_block(rng, n):
    """Bit-block of exactly n isolated single bits (even positions, no two adjacent)."""
    return bits_block([(2 * int(p), 2 * int(p)) for p in rng.choice(BLOCK_BITS // 2, size=n, replace=False)])


def longs_block(rng, n):
    """Bit-block of exactly n runs of 2 .. 7 bits, none from bit 0."""
    return bits_block([(8 * int(p) + 1, 8 * int(p) + int(rng.integers(2, 8))) for p in rng.choice(BLOCK_BITS // 8, size=n, replace=False)])


def shaped_vectors(rng, n_blocks):
    """Two dense bit vectors for the AND group, then bit-blocks at the listing edge, at the block's edges and across words, of
    singles only and long runs only, a vector sparse in some columns and dense in others, GAP and mixed vectors.  Column 0 has
    every bit-block listed, column 1 none."""
    vecs = [bm.BVector.random(n_blocks, 0.5, rng), bm.BVector.random(n_blocks, 0.3, rng)]
    edge = [
        lambda: singles_block(rng, LIST_MAX // 2),                   # exactly kListBitMax bytes: listed
        lambda: singles_block(rng, LIST_MAX // 2 + 1),               # 2 bytes over: streamed
        lambda: longs_block(rng, LIST_MAX // 4),                     # exactly, as long runs
        lambda: longs_block(rng, LIST_MAX // 4 + 1),
        lambda: bits_block([(0, 0), (31, 32), (63, 95), (1020, 1030), (4095, 4096), (65535, 65535)]),
        lambda: bits_block([(0, 40), (100, 100), (65500, 65535)]),  # a long run from bit 0, one to bit 65535
        lambda: singles_block(rng, int(rng.integers(1, 300))),
        lambda: longs_block(rng, int(rng.integers(1, 300))),
    ]
    for mk in edge:
        v = bm.BVector(n_blocks)
        for nb in range(n_blocks):
            v.set_bits(nb, mk())
        vecs.append(v)
    v = bm.BVector(n_blocks)                                            # listed in even columns only
    for nb in range(n_blocks):
        v.set_bits(nb, singles_block(rng, 200) if nb % 2 == 0 else bits_to_words(rng.random(BLOCK_BITS) < 0.3))
    vecs.append(v)
    for k in range(3):
        v = bm.BVector(n_blocks)
        for nb in range(n_blocks):
            v.set_gap(nb, run_block(rng, int(rng.integers(1, 300)), 1 + k))
        vecs.append(v)
    vecs += gen.mixed_vectors(rng, 4, n_blocks, p_null=0.1, p_full=0.0, p_gap=0.5)
    for v in vecs[2:]:                                                  # column 0: only listed bit-blocks; column 1: none
        if v.kind[0] == bm.BLK_BIT and 2 * block_runs(v.blocks[0])[0] + 4 * block_runs(v.blocks[0])[1] > LIST_MAX:
            v.set_bits(0, singles_block(rng, 50))
        if v.kind[1] == bm.BLK_BIT and 2 * block_runs(v.blocks[1])[0] + 4 * block_runs(v.blocks[1])[1] <= LIST_MAX:
            v.set_bits(1, bits_to_words(rng.random(BLOCK_BITS) < 0.3))
    return vecs


def test_bit_run_lists_shapes(ctx):
    """FLAT and raw-form sets, sub-ranges, with and without compression; the AND group is the two dense vectors."""
    rng = np.random.default_rng(51)
    n_blocks = 6
    vecs = shaped_vectors(rng, n_blocks)
    g0 = [0, 1]
    g1 = [v for v in rng.permutation(len(vecs)) if v not in g0]
    for gap_flat in (True, False):
        ps = bm.PackedSet.pack(vecs, gap_flat=gap_flat)
        kinds = ps.kinds()
        assert (kinds[0] == bm.BLK_BIT).sum() > 2 and (kinds[1] == bm.BLK_BIT).sum() > 2
        for nb_from, nb_to in ((0, 0), (1, 0), (2, 5), (5, 6)):
            check(ctx, ps, g0, g1, C, nb_from, nb_to)
        check(ctx, ps, g0, g1, 0)


def test_bit_run_lists_and_group_listed(ctx):
    """An AND group holding a listed vector streams part A only (every bit-block) and is still equal."""
    rng = np.random.default_rng(52)
    vecs = shaped_vectors(rng, 4)
    g0 = [0, 2]                                                         # vector 2 is listed in every column
    g1 = [v for v in range(len(vecs)) if v not in g0]
    check(ctx, bm.PackedSet.pack(vecs), g0, g1, C, part_b=False)


def test_bit_run_lists_long_parts_many_columns(ctx):
    """B singles of a column longer than the 16-stage ring (> 128 KB), and more columns than SMs."""
    rng = np.random.default_rng(53)
    n_blocks = 2
    vecs = [bm.BVector.random(n_blocks, 0.5, rng)]
    for k in range(4 * BLOCK_BITS // LIST_MAX + 8):
        v = bm.BVector(n_blocks)
        for nb in range(n_blocks):
            v.set_bits(nb, singles_block(rng, LIST_MAX // 2 - int(rng.integers(0, 50))))
        vecs.append(v)
    v = bm.BVector(n_blocks)
    for nb in range(n_blocks):
        v.set_gap(nb, run_block(rng, 100, 3))
    vecs.append(v)
    ps = bm.PackedSet.pack(vecs)
    assert host_bit_run_list_bytes(ps)[0] > 16 * 8192 * n_blocks
    check(ctx, ps, [0], list(range(1, len(vecs))), C)

    n_blocks = 200
    vecs = [bm.BVector.random(n_blocks, 0.4, rng)] + [bm.BVector.random(n_blocks, d, rng) for d in (0.3, 0.05, 0.02, 0.01, 0.004)]
    vecs += [bm.BVector.random(n_blocks, 0.002 * (k + 1), rng).optimize() for k in range(4)]
    ps = bm.PackedSet.pack(vecs)
    g1 = list(rng.permutation(np.arange(1, len(vecs))))
    check(ctx, ps, [0], g1, C)
    check(ctx, ps, [0], g1, 0, 37, 0)


def test_bit_run_lists_c3_recipe(ctx):
    """C3's generator (vector k at density 0.5 / k, optimized) over 48 columns: the default rule's second call, which builds the
    companion and streams A + B, against never building; part B lists the sparser bit-block vectors and never the AND group."""
    import bench
    dens, seed, opt = bench.workload_inputs("c3", 0)
    n_vec, n_cols = 1024, 48
    dset = bm.DeviceSet.synth(ctx, n_vec, n_cols, dens, seed, opt)
    g0, g1 = [0, 1], np.arange(2, n_vec, dtype=np.uint32)
    try:
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)
        out = []
        for _ in range(2):
            out.append(run(ctx, dset, g0, g1, C, 0, 0))
        sgl, lr, n = dset.bit_run_list_bytes()
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 0)
        ref = run(ctx, dset, g0, g1, C, 0, 0)
    finally:
        ctx.set_tuning(bm.capi.TUNE_RUN_LISTS, 1)
        dset.free()
    assert sgl > 0 and 20 * n_cols <= n <= 48 * n_cols     # 50 bit-block vectors per column, 1 and 2 too dense to list
    for got in out:
        for k in ref:
            assert np.array_equal(np.asarray(got[k]), np.asarray(ref[k])), k
