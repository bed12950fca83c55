"""Rank-select compressed sparse vectors (bm::rsc_sparse_vector<unsigned>): rank decompression / compression on the device
(bmb200_rank_decompress / bmb200_rank_compress, csrc/rank_kernel.cuh) and scanner searches over the compressed planes.

CPU tests pin the numpy restatement of rank_compressor and the Python RSC model to the real reference (recorded answers where
the reference is not built); GPU tests check the device against both."""
import numpy as np
import pytest

import bitmagic_b200 as bm
import rsclib as R
from bitmagic_b200.hostfmt import BLOCK_BITS, BVector, PackedSet, bits_to_words, calc_change

gpu = pytest.mark.gpu
RNG_SEED = 20261015


# ---------------------------------------------------------------- inputs
def nn_kinds(n_blocks=520):
    """NOT-NULL bits with every block kind: NULL, FULL (also at an unaligned base), BIT (iid), GAP with a first 1-run and a
    first 0-run, single bits (unaligned bases), a NULL superblock (blocks 256..511) and blocks after it."""
    rng = np.random.default_rng(RNG_SEED)
    b = np.zeros(n_blocks * BLOCK_BITS, np.uint8)
    i = np.arange(BLOCK_BITS)
    for nb in list(range(40)) + list(range(n_blocks - 4, n_blocks)):
        k = nb % 8
        blk = b[nb * BLOCK_BITS:(nb + 1) * BLOCK_BITS]
        if k == 1: blk[:] = 1
        elif k == 2: blk[:] = rng.random(BLOCK_BITS) < 0.3
        elif k == 3: blk[:] = ((i >> 7) & 3) == 0                    # GAP, first run is a 1-run
        elif k == 4: blk[:] = ((i >> 7) & 3) == 1                    # GAP, first run is a 0-run
        elif k == 5: blk[:] = rng.random(BLOCK_BITS) < 0.001
        elif k == 6: blk[:] = rng.random(BLOCK_BITS) < 0.97
        elif k == 7: blk[12345 + nb] = 1                             # one bit: the next block's base is not word-aligned
    return b


def nn_exact():
    """count(NN) an exact multiple of 65536: three FULL blocks between NULL ones"""
    b = np.zeros(5 * BLOCK_BITS, np.uint8)
    for nb in (0, 2, 4):
        b[nb * BLOCK_BITS:(nb + 1) * BLOCK_BITS] = 1
    return b


NN_CASES = {"kinds": nn_kinds, "exact": nn_exact}


def comp_sources(nn_bits):
    """vectors of the compressed space, as wide as NN: iid with bits past count(NN), runs, all ones, empty, sparse"""
    rng = np.random.default_rng(RNG_SEED + 1)
    n = nn_bits.size
    cnt = int(nn_bits.sum())
    i = np.arange(n)
    s_iid = (rng.random(n) < 0.5).astype(np.uint8)
    s_runs = (((i >> 9) % 5) == 0).astype(np.uint8)
    s_full = np.zeros(n, np.uint8); s_full[:cnt] = 1
    s_none = np.zeros(n, np.uint8)
    s_sparse = (rng.random(n) < 0.0005).astype(np.uint8)
    return [s_iid, s_runs, s_full, s_none, s_sparse]


def logical_sources(nn_bits):
    """vectors of the logical space: subsets of NN (iid, runs) and one that is not a subset"""
    rng = np.random.default_rng(RNG_SEED + 2)
    n = nn_bits.size
    i = np.arange(n)
    sub_iid = nn_bits & (rng.random(n) < 0.4)
    sub_runs = nn_bits & (((i >> 11) & 1) == 0)
    not_sub = (rng.random(n) < 0.2).astype(np.uint8)
    return [sub_iid.astype(np.uint8), sub_runs.astype(np.uint8), not_sub]


def words(bits):
    return R.words_of(bits, (len(bits) + BLOCK_BITS - 1) // BLOCK_BITS)


def scan_inputs(kind):
    """(values, nulls) of a nullable vector: runs of NOT-NULL, iid NULLs, empty, and all NOT-NULL"""
    rng = np.random.default_rng(RNG_SEED + 3)
    if kind == "empty":
        return np.zeros(0, np.uint32), np.zeros(0, np.uint8)
    n = 3 * BLOCK_BITS + 777
    vals = rng.integers(0, 1200, n).astype(np.uint32)
    vals[:5000] = 0
    if kind == "dense":
        return vals, np.zeros(n, np.uint8)
    i = np.arange(n)
    nulls = np.where(i < BLOCK_BITS, rng.random(n) < 0.6, ((i >> 10) & 1) == 1).astype(np.uint8)
    nulls[2 * BLOCK_BITS:2 * BLOCK_BITS + 30000] = 0
    return vals, nulls


SEARCH = {
    bm.SCAN_EQ: np.array([0, 3, 77, 1199, 5000], np.uint32),
    bm.SCAN_GT: np.array([0, 600, 1199], np.uint32),
    bm.SCAN_GE: np.array([1, 600, 1200], np.uint32),
    bm.SCAN_LT: np.array([0, 600, 5000], np.uint32),
    bm.SCAN_LE: np.array([0, 600, 1199], np.uint32),
    bm.SCAN_RANGE: np.array([[2, 40], [900, 100], [0, 0], [1199, 9999]], np.uint32),
}


# ---------------------------------------------------------------- CPU: checkers against the reference
def test_numpy_rank_compressor_against_reference():
    for name, mk in NN_CASES.items():
        nn = mk()
        cnt = int(nn.sum())
        ncomp = max(1, (cnt + BLOCK_BITS - 1) // BLOCK_BITS)
        for k, s in enumerate(logical_sources(nn)[:2]):                 # the reference requires src to be a subset of idx
            rc, rw = R.ref_rank_compress(words(nn), words(s), ncomp)
            exp = R.np_rank_compress(nn, s)
            assert rc == int(exp.sum()) and np.array_equal(R.bits_of(rw)[:cnt], exp), (name, k)
        for k, s in enumerate(comp_sources(nn)):
            s = s.copy(); s[cnt:] = 0                                     # the reference reads past count(idx) out of range
            rc, rw = R.ref_rank_decompress(words(nn), words(s), nn.size // BLOCK_BITS)
            exp = R.np_rank_decompress(nn, s)
            assert rc == int(exp.sum()) and np.array_equal(R.bits_of(rw), exp), (name, k)


@pytest.mark.parametrize("kind", ["mixed", "dense", "empty"])
def test_rsc_model_against_reference(kind):
    vals, nulls = scan_inputs(kind)
    eff, planes, nn = R.ref_rsc_planes(vals, nulls)
    sv = bm.RscSparseVector.from_values(vals, nulls)
    assert sv.effective_size() == eff == int((nulls == 0).sum())
    nc = max(1, (vals.size + BLOCK_BITS - 1) // BLOCK_BITS)
    assert np.array_equal(R.bits_of(nn), R.bits_of(R.words_of(R.bits_of(sv.not_null.to_words()), nc)))
    if eff:
        assert sv.effective_slices() == len(planes)
    for j in range(len(planes)):                                          # compressed planes: bits [0, effective_size())
        assert np.array_equal(R.bits_of(planes[j])[:eff], R.bits_of(sv.planes[j].to_words())[:eff]), j
        assert not R.bits_of(planes[j])[eff:].any()


def test_rsc_scan_answers_recorded():
    """every reference search the GPU tests compare against is recorded (or computed live where the reference is built)"""
    for kind in ("mixed", "dense", "empty"):
        vals, nulls = scan_inputs(kind)
        for pred, search in SEARCH.items():
            counts, w = R.ref_rsc_scan(vals, nulls, pred, search)
            assert counts.size == (search.shape[0])
            assert all(int(c) == int(R.bits_of(w[k]).sum()) for k, c in enumerate(counts))


# ---------------------------------------------------------------- GPU helpers
def result_words(res, n_groups):
    kind, off, bits, gaps = res.fetch()
    nb = kind.size // n_groups
    return [bm.result_to_bvector(kind[g * nb:(g + 1) * nb], off[g * nb:(g + 1) * nb], bits, gaps).to_words() for g in range(n_groups)]


def expected_kind(w, compress):
    if not w.any():
        return bm.BLK_NULL
    if not compress:
        return bm.BLK_BIT
    runs = calc_change(w)
    return bm.BLK_FULL if runs == 1 else bm.BLK_GAP if runs < bm.capi.GAP_THRESHOLD else bm.BLK_BIT


def check_meta(res, exp_words, n_groups, compress):
    kind, pop, dig, nr = res.meta()
    totals = res.group_totals(n_groups)
    nb = kind.size // n_groups
    for g in range(n_groups):
        e = exp_words[g].reshape(nb, -1)
        assert int(totals[g]) == int(R.bits_of(exp_words[g]).sum()), g
        for c in range(nb):
            assert pop[g * nb + c] == int(R.bits_of(e[c]).sum()), (g, c)
            assert kind[g * nb + c] == expected_kind(e[c], compress), (g, c)


def upload(ctx, vecs, flat=True):
    ps = PackedSet.pack(vecs, max(v.n_blocks for v in vecs), gap_flat=flat)
    return bm.DeviceSet.upload(ctx, ps)


def bvec(bits):
    return BVector.from_words(words(bits)).optimize()


# ---------------------------------------------------------------- GPU: rank decompression / compression
@gpu
@pytest.mark.parametrize("case", list(NN_CASES))
@pytest.mark.parametrize("flat", [True, False])
@pytest.mark.parametrize("flags", [bm.F_OPT_COMPRESS, bm.F_OPT_NONE])
def test_rank_decompress(ctx, case, flat, flags):
    nn = NN_CASES[case]()
    cnt = int(nn.sum())
    srcs = comp_sources(nn)
    dset = upload(ctx, [bvec(nn)] + [bvec(s) for s in srcs], flat)
    rs = bm.DeviceRS(ctx, dset, 0)
    nnb = dset.n_blocks
    groups = [([1 + k], None) for k in range(len(srcs))]                 # 5 groups: several value groups of a scan batch
    ncomp = max(1, (cnt + BLOCK_BITS - 1) // BLOCK_BITS)
    out = None
    for src_flags, nb_to in ((bm.F_OPT_COMPRESS, 0), (bm.F_OPT_NONE, 0), (bm.F_OPT_COMPRESS, max(1, ncomp - 1))):
        src = bm.aggregate_batch(ctx, dset, bm.OP_OR, groups, src_flags, 0, nb_to)
        out = bm.rank_decompress(ctx, rs, src, flags, out)                # *inout reuse from the second round on
        assert out.n_cols == len(groups) * nnb
        cpg = nb_to or nnb
        exp = []
        for k, s in enumerate(srcs):
            s = s.copy(); s[cpg * BLOCK_BITS:] = 0                        # a source shorter than count(NN) reads 0 past its columns
            exp.append(words(R.np_rank_decompress(nn, s)))
            if nb_to == 0 and k in (1, 3, 4):                             # within count(NN) the reference agrees
                sc = s.copy(); sc[cnt:] = 0
                rc, rw = R.ref_rank_decompress(words(nn), words(sc), nnb)
                assert np.array_equal(rw, exp[-1]) and rc == int(R.bits_of(rw).sum())
        got = result_words(out, len(groups))
        for k in range(len(groups)):
            assert np.array_equal(got[k], exp[k]), (case, src_flags, nb_to, k)
        check_meta(out, exp, len(groups), flags == bm.F_OPT_COMPRESS)
        src.free()
    out.free(); rs.free(); dset.free()


@gpu
@pytest.mark.parametrize("case", list(NN_CASES))
@pytest.mark.parametrize("flat", [True, False])
def test_rank_compress(ctx, case, flat):
    nn = NN_CASES[case]()
    cnt = int(nn.sum())
    srcs = logical_sources(nn)
    dset = upload(ctx, [bvec(nn)] + [bvec(s) for s in srcs], flat)
    rs = bm.DeviceRS(ctx, dset, 0)
    ncomp = max(1, (cnt + BLOCK_BITS - 1) // BLOCK_BITS)
    out = None
    for k, s in enumerate(srcs):
        for flags in (bm.F_OPT_COMPRESS, bm.F_OPT_NONE):
            out = bm.rank_compress(ctx, rs, 1 + k, flags, out)
            assert out.n_cols == ncomp
            exp = words(np.pad(R.np_rank_compress(nn, s), (0, ncomp * BLOCK_BITS - cnt)))
            got = result_words(out, 1)[0]
            assert np.array_equal(got, exp), (case, k, flags)
            check_meta(out, [exp], 1, flags == bm.F_OPT_COMPRESS)
            if k < 2:                                                     # subsets of NN: the reference agrees
                rc, rw = R.ref_rank_compress(words(nn), words(s), ncomp)
                assert np.array_equal(rw, exp) and rc == int(R.bits_of(exp).sum())
            else:                                                         # not a subset: compress(src & NN)
                assert np.array_equal(got, words(np.pad(R.np_rank_compress(nn, s & nn), (0, ncomp * BLOCK_BITS - cnt))))
    out.free(); rs.free(); dset.free()


@gpu
def test_rank_round_trips(ctx):
    nn = nn_kinds()
    cnt = int(nn.sum())
    s = logical_sources(nn)[2]                                           # not a subset: the round trip gives s & NN
    x = comp_sources(nn)[0]; x[cnt:] = 0
    dset = upload(ctx, [bvec(nn), bvec(s), bvec(x)])
    rs = bm.DeviceRS(ctx, dset, 0)
    c = bm.rank_compress(ctx, rs, 1, bm.F_OPT_COMPRESS)
    d = bm.rank_decompress(ctx, rs, c, bm.F_OPT_COMPRESS)
    assert np.array_equal(result_words(d, 1)[0], words(s & nn))
    c.free(); d.free()
    src = bm.aggregate(ctx, dset, bm.OP_OR, [2], None, bm.F_OPT_COMPRESS)
    d = bm.rank_decompress(ctx, rs, src, bm.F_OPT_COMPRESS)
    y = BVector.from_words(result_words(d, 1)[0]).optimize()
    dset2 = upload(ctx, [bvec(nn), y])
    rs2 = bm.DeviceRS(ctx, dset2, 0)
    c = bm.rank_compress(ctx, rs2, 1, bm.F_OPT_COMPRESS)
    assert np.array_equal(R.bits_of(result_words(c, 1)[0])[:cnt], x[:cnt])
    for h in (c, d, src, rs2, dset2, rs, dset):
        h.free()


@gpu
def test_rank_bad_arguments(ctx):
    nn = nn_exact()
    dset = upload(ctx, [bvec(nn), bvec(nn)])
    rs = bm.DeviceRS(ctx, dset, 0)
    with pytest.raises(bm.BMB200Error) as e:
        bm.rank_compress(ctx, rs, 1, bm.F_COUNT_ONLY)
    assert e.value.code == bm.capi.ERR_BADARG
    with pytest.raises(bm.BMB200Error) as e:
        bm.rank_compress(ctx, rs, 2, bm.F_OPT_NONE)
    assert e.value.code == bm.capi.ERR_RANGE
    cnt_only = bm.aggregate(ctx, dset, bm.OP_OR, [1], None, bm.F_COUNT_ONLY)
    with pytest.raises(bm.BMB200Error) as e:
        bm.rank_decompress(ctx, rs, cnt_only, bm.F_OPT_NONE)          # a count-only result holds no blocks to read
    assert e.value.code == bm.capi.ERR_BADARG
    src = bm.aggregate(ctx, dset, bm.OP_OR, [1], None, bm.F_OPT_NONE)
    with pytest.raises(bm.BMB200Error) as e:
        bm.rank_decompress(ctx, rs, src, bm.F_OR_TARGET)
    assert e.value.code == bm.capi.ERR_BADARG
    for h in (src, cnt_only, rs, dset):
        h.free()


# ---------------------------------------------------------------- GPU: RSC scanner searches
@gpu
@pytest.mark.parametrize("kind", ["mixed", "dense", "empty"])
def test_rsc_scanner_against_reference(ctx, kind):
    vals, nulls = scan_inputs(kind)
    sv = bm.RscSparseVector.from_values(vals, nulls)
    sc = bm.SparseVectorScanner(sv, ctx)
    try:
        for pred, search in SEARCH.items():
            counts, rw = R.ref_rsc_scan(vals, nulls, pred, search)
            got = sc._run(pred, search)                                  # one batched launch (+ one decompression)
            cnt = sc._run(pred, search, count_only=True)
            for k in range(len(got)):
                gw = got[k].to_words()
                assert np.array_equal(gw, rw[k][:gw.size]), (kind, pred, k)
                assert int(counts[k]) == cnt[k] == got[k].count(), (kind, pred, k)
        # single searches through the public names
        eq77 = sc.find_eq(77)
        assert np.array_equal(eq77.to_words(), R.ref_rsc_scan(vals, nulls, bm.SCAN_EQ, SEARCH[bm.SCAN_EQ])[1][2][:eq77.to_words().size])
        assert sc.count_eq(77) == eq77.count()
        if kind == "dense":                                              # NN all set: the same answer as the plain scanner
            plain = bm.SparseVectorScanner(bm.SparseVector.from_values(vals, nulls), ctx)
            try:
                for pred, search in SEARCH.items():
                    a, b = sc._run(pred, search), plain._run(pred, search)
                    assert all(x.compare(y) == 0 for x, y in zip(a, b)), pred
            finally:
                plain.close()
    finally:
        sc.close()


@gpu
def test_rsc_binding_harness():
    import subprocess
    exe = R.orclib.ORACLE_DIR / "_ref" / "test_rsc_binding"
    if not exe.exists():
        pytest.skip("oracle/_ref/test_rsc_binding is built only where the reference tree exists")
    p = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-2000:]
    assert "0 failed" in p.stdout
