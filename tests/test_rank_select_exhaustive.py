"""Rank / select against a plain numpy model at every position and every rank of boundary-shaped blocks.

Next to the reference-format fields, the device index (csrc/aux_kernels.cuh) keeps a fine index of its own: per block 128
window entries (the ones before each 512-bit window, and for GAP blocks the run that holds the window's first bit), 8 block
pivots, and 16 row pivots per 256-block superblock.  rs_rank_kernel and rs_select_kernel answer from it.  Sampled queries
almost never land on a window start, on a rank equal to a pivot, or on a run that ends at a window edge.  So these tests ask
every position and every rank of blocks built to put their run ends and ones exactly there, in FLAT and raw GAP form.  They
also cover superblock layouts (empty, all FULL, one group only, ragged), sets of more than 1024 superblocks (where
rs_scan_sb_kernel carries its running total from one 1024-wide pass to the next), the device entry points past one grid
trip, and a rebuild after the bits change in place.

The model (RSModel) is one uint64 cumsum per block plus the running block totals.  The CPU tests at the end pin it to the
oracle and to the reference on a boundary sample of every corpus vector."""
import ctypes
import functools

import numpy as np
import pytest

import bitmagic_b200 as bm
import gen
import orclib
from bitmagic_b200.hostfmt import BLOCK_BITS as BB, bits_to_words, words_to_bits

gpu = pytest.mark.gpu
needs_ref_answers = pytest.mark.skipif(not orclib.have_ref_answers(), reason="neither oracle/_ref/libbmref.so nor tests/golden/ref/")
KIND = {bm.BLK_NULL: "NULL", bm.BLK_FULL: "FULL", bm.BLK_BIT: "BIT", bm.BLK_GAP: "GAP"}
U64 = np.uint64


# ------------------------------------------------------------------ the plain model

class RSModel:
    """rank(p) = ones in [0, p], the total at or past the end; select(r) = position of the r-th one, found only for
    1 <= r <= total.  Built from per-block counts, so a vector of 2^34 bits that is mostly NULL costs only its non-NULL blocks."""

    def __init__(self, bv: bm.BVector):
        self.bv, self.n = bv, bv.n_blocks
        cnt = np.zeros(self.n, U64)
        cnt[bv.kind == bm.BLK_FULL] = BB
        for nb in bv.blocks:
            if bv.kind[nb] in (bm.BLK_BIT, bm.BLK_GAP):
                cnt[nb] = int(self.bits(nb).sum())
        self.cnt = cnt
        self.pre = np.zeros(self.n + 1, U64)
        np.cumsum(cnt, out=self.pre[1:])
        self.total = int(self.pre[-1])

    def bits(self, nb):
        return words_to_bits(self.bv.block_words(nb))

    def block_rank(self, nb):
        """inclusive rank of every offset of block nb"""
        k = self.bv.kind[nb]
        if k == bm.BLK_NULL:
            c = np.zeros(BB, U64)
        elif k == bm.BLK_FULL:
            c = np.arange(1, BB + 1, dtype=U64)
        else:
            c = np.cumsum(self.bits(nb), dtype=U64)
        return self.pre[nb] + c

    def sb_count(self):
        """running totals at superblock starts, as rs_index keeps them: nsb + 1 entries"""
        nsb = (self.n + 255) // 256
        return self.pre[np.minimum(np.arange(nsb + 1) * 256, self.n)]

    @staticmethod
    def _by_block(nb, idx):
        """idx grouped by nb[idx] -> (block, indices) pairs"""
        idx = idx[np.argsort(nb[idx], kind="stable")]
        blocks, starts = np.unique(nb[idx], return_index=True)
        return zip(blocks.tolist(), np.split(idx, starts[1:]))

    def rank(self, pos):
        pos = np.asarray(pos, U64)
        out = np.full(pos.size, self.total, U64)
        nb = pos >> U64(16)
        off = (pos & U64(0xFFFF)).astype(np.int64)
        for b, part in self._by_block(nb, np.flatnonzero(nb < self.n)):
            k = self.bv.kind[b]
            if k == bm.BLK_NULL:
                out[part] = self.pre[b]
            elif k == bm.BLK_FULL:
                out[part] = self.pre[b] + off[part].astype(U64) + U64(1)
            else:
                out[part] = self.pre[b] + np.cumsum(self.bits(b), dtype=U64)[off[part]]
        return out

    def select(self, ranks):
        r = np.asarray(ranks, U64)
        pos = np.zeros(r.size, U64)
        found = (r >= 1) & (r <= U64(self.total))
        idx = np.flatnonzero(found)
        nb = np.zeros(r.size, np.int64)
        nb[idx] = np.searchsorted(self.pre[1:], r[idx], side="left")        # first block whose running total reaches r
        for b, part in self._by_block(nb, idx):
            rr = (r[part] - self.pre[b]).astype(np.int64)                   # 1-based rank inside the block
            inb = rr - 1 if self.bv.kind[b] == bm.BLK_FULL else np.flatnonzero(self.bits(b))[rr - 1]
            pos[part] = U64(b * BB) + inb.astype(U64)
        return pos, found


# ------------------------------------------------------------------ corpus of boundary-shaped blocks

WIN = 512
RS3 = (21824, 43648)          # rs3 borders: the reference's sub-block counts end there
AUX = (32736, 54560)          # aux borders of bit-blocks


def gap_corpus():
    """(label, GAP block) with run ends placed on the fine-index windows, the rs3 and aux borders and the capacity levels;
    every shape with the first run 0 and 1 (FLAT form: with and without the lead pad)."""
    ks = np.arange(128) * WIN
    out = []

    def add(label, ends):
        e = sorted({int(x) for x in ends if 0 <= int(x) < BB - 1}) + [BB - 1]
        for first in (0, 1):
            out.append((f"GAP {label}, first run {first}", gen.gap_from_runs(e, first)))

    add("run ends at 512k-1, 512k, 512k+1", np.concatenate([ks - 1, ks, ks + 1]))
    for d in (-1, 0, 1):
        add(f"run ends at 512k{d:+d}", ks + d)
    for name, (b0, b1) in (("rs3", RS3), ("aux", AUX)):
        add(f"run ends at the {name} borders -1/0/+1", [b0 - 1, b0, b0 + 1, b1 - 1, b1, b1 + 1])
        for d in (-1, 0, 1):
            add(f"run ends at the {name} borders{d:+d}", [b0 + d, b1 + d])
    add("first run of one bit", [0])
    add("last run of one bit", [BB - 2])
    add("1 run", [])
    add("2 runs", [BB // 2 - 1])
    for n in (124, 125, 252, 253, 508, 509, 1275):
        add(f"{n} runs", (BB // n) * np.arange(1, n) - 1)
    return out


def bit_corpus():
    """(label, bit-block words): all ones in a non-FULL block, single bits on word and window edges, one live window,
    pivot ties, alternating words."""
    out = []

    def add(label, bits):
        out.append((f"BIT {label}", bits_to_words(bits)))

    edges = [0, 31, 32, 511, 512, BB - 1]
    add("all ones", np.ones(BB, np.uint8))
    b = np.zeros(BB, np.uint8); b[edges] = 1
    add("one bit at each of 0, 31, 32, 511, 512, 65535", b)
    for e in edges:
        b = np.zeros(BB, np.uint8); b[e] = 1
        add(f"only bit {e}", b)
    for w in (0, 1, 64, 127):
        b = np.zeros(BB, np.uint8); b[w * WIN:(w + 1) * WIN] = 1
        add(f"only window {w}, all ones", b)
    b = np.zeros(BB, np.uint8); b[16 * WIN:] = 1
    add("windows 0..15 empty, then all ones (ranks tie at every pivot)", b)
    b = np.zeros(BB, np.uint8); b[::WIN] = 1; b[WIN - 1::WIN] = 1
    add("first and last bit of every window", b)
    out.append(("BIT alternating 0xAAAAAAAA", np.full(2048, 0xAAAAAAAA, np.uint32)))
    out.append(("BIT alternating 0x55555555", np.full(2048, 0x55555555, np.uint32)))
    return out


def interleave(items, n_blocks):
    """Corpus blocks at the even slots; FULL and NULL alternate at the odd slots, so each block has one of each as neighbours."""
    bv = bm.BVector(n_blocks)
    labels = ["NULL"] * n_blocks
    for i, (label, data) in enumerate(items):
        nb = 2 * i
        (bv.set_gap if data.dtype == np.uint16 else bv.set_bits)(nb, data)
        labels[nb] = label
        if i % 2 == 0:
            bv.set_full(nb + 1); labels[nb + 1] = "FULL"
    return bv, labels


@functools.lru_cache(maxsize=None)
def corpus():
    """-> (vectors, labels per block, models): vector 0 = the GAP corpus, vector 1 = the bit-block corpus"""
    g, b = gap_corpus(), bit_corpus()
    n = 2 * max(len(g), len(b))
    vecs, labels = zip(*(interleave(items, n) for items in (g, b)))
    return list(vecs), list(labels), [RSModel(v) for v in vecs]


@functools.lru_cache(maxsize=None)
def corpus_set(flat):
    return bm.PackedSet.pack(corpus()[0], gap_flat=flat)


FORMS = pytest.mark.parametrize("flat", [True, False], ids=["flat", "raw"])


# ------------------------------------------------------------------ mismatch reports

def where(labels, kind, p):
    nb, off = p >> 16, p & 0xFFFF
    if nb >= len(kind):
        return f"pos {p} (past the end)"
    lab = labels[nb] if labels is not None else KIND[int(kind[nb])]
    return f"pos {p}: block {nb} [{lab}] offset {off} window {off >> 9} fine group {off >> 13}"


def check_rank(got, want, pos, bv, labels=None, what=""):
    bad = np.flatnonzero(got != want)
    if bad.size:
        lines = [f"{where(labels, bv.kind, int(pos[i]))}: got {int(got[i])} want {int(want[i])}" for i in bad[:8]]
        pytest.fail(f"{what}: {bad.size} wrong ranks\n" + "\n".join(lines))


def check_select(got, want, ranks, m, labels=None, what=""):
    (gp, gf), (wp, wf) = got, want
    bad = np.flatnonzero((gf != wf) | (gp != wp))
    if bad.size:
        lines = []
        for i in bad[:8]:
            r = int(ranks[i])
            at = where(labels, m.bv.kind, int(wp[i])) if wf[i] else "not found"
            lines.append(f"rank {r} (block {int(wp[i]) >> 16}, rank in block {r - int(m.pre[int(wp[i]) >> 16]) if wf[i] else '-'}): "
                         f"got pos {int(gp[i])} found {bool(gf[i])}, want {at}")
        pytest.fail(f"{what}: {bad.size} wrong selects\n" + "\n".join(lines))


def check_export(rs, ps, v, m):
    bc, sc, sb = rs.export()
    obc, osc, osb = orclib.oracle_rs_build(ps, v)
    assert np.array_equal(bc, obc) and np.array_equal(bc.astype(U64), m.cnt), "bcount"
    assert np.array_equal(sc, osc), f"sub_count differs in blocks {np.flatnonzero(sc != osc)[:8]}"
    assert np.array_equal(sb, osb) and np.array_equal(sb, m.sb_count()), "sb_count"
    assert rs.total() == m.total


def past_end(n):
    return np.array([n * BB, n * BB + 1, n * BB + BB, 2**40, 2**63], U64)


# ------------------------------------------------------------------ GPU 1, 2: every position and every rank of the corpus

@gpu
@FORMS
def test_rank_at_every_position(ctx, flat):
    """All 65536 offsets of every corpus block, and positions past the end."""
    _, labels, models = corpus()
    ps = corpus_set(flat)
    dset = bm.DeviceSet.upload(ctx, ps)
    for v, m in enumerate(models):
        rs = bm.DeviceRS(ctx, dset, v)
        check_export(rs, ps, v, m)
        pos = np.concatenate([np.arange(m.n * BB, dtype=U64), past_end(m.n)])
        want = np.concatenate([m.block_rank(nb) for nb in range(m.n)] + [np.full(5, m.total, U64)])
        check_rank(rs.rank(pos), want, pos, m.bv, labels[v], f"vector {v}")
        rs.free()
    dset.free()


@gpu
@FORMS
def test_select_at_every_rank(ctx, flat):
    """select(r) for every r in 0 .. total + 1, then rank(select(r)) == r and select(rank(p)) == p for every set bit p."""
    _, labels, models = corpus()
    dset = bm.DeviceSet.upload(ctx, corpus_set(flat))
    for v, m in enumerate(models):
        rs = bm.DeviceRS(ctx, dset, v)
        ranks = np.arange(m.total + 2, dtype=U64)
        want = m.select(ranks)
        got = rs.select(ranks)
        check_select(got, want, ranks, m, labels[v], f"vector {v}")
        ones = got[0][1:m.total + 1]                                      # every set bit, in order
        check_rank(rs.rank(ones), ranks[1:m.total + 1], ones, m.bv, labels[v], f"vector {v}: rank(select(r)) != r")
        p, f = rs.select(rs.rank(ones))
        assert f.all() and np.array_equal(p, ones), f"vector {v}: select(rank(p)) != p at {ones[p != ones][:8]}"
        rs.free()
    dset.free()


# ------------------------------------------------------------------ GPU 3: superblock layouts

SB_SIZES = [1, 255, 256, 257, 4097]


def superblock_vectors(n):
    """Vectors whose superblocks are, in turn, all FULL (total 2^24), one 16-block group of corpus blocks, empty, and every
    17th block a corpus block; each vector starts the cycle at another layout.  Vector 3 holds only its first and last block."""
    pool = [d for _, d in gap_corpus()[::3]] + [d for _, d in bit_corpus()]
    vecs = []
    for shift in (0, 1, 3):
        bv = bm.BVector(n)
        for s in range((n + 255) // 256):
            lo, hi = 256 * s, min(256 * s + 256, n)
            kind = (s + shift) % 4
            if kind == 0:
                blocks = range(lo, hi)
            elif kind == 1:
                g = lo + 16 * ((5 * s + 3) % 16)
                blocks = range(g, min(g + 16, hi))
            elif kind == 2:
                blocks = range(0)
            else:
                blocks = range(lo, hi, 17)
            for nb in blocks:
                if kind == 0:
                    bv.set_full(nb)
                else:
                    d = pool[(nb + s) % len(pool)]
                    (bv.set_gap if d.dtype == np.uint16 else bv.set_bits)(nb, d)
        vecs.append(bv)
    bv = bm.BVector(n)
    bv.set_gap(0, pool[0])
    bv.set_full(n - 1)
    vecs.append(bv)
    return vecs


def edge_queries(m, n_sample=48):
    """positions: every block base -1/0/+1, every window start -1/0 of a sample of non-NULL blocks, past the end;
    ranks: base, base + 1 and base + count of every block (group and superblock edges are block edges), 0, total + 1"""
    bases = np.arange(m.n, dtype=np.int64) * BB
    live = np.flatnonzero(m.bv.kind != bm.BLK_NULL)
    sample = live[np.linspace(0, live.size - 1, min(n_sample, live.size)).astype(int)] if live.size else live
    wins = (sample[:, None] * BB + np.arange(0, BB, WIN)[None, :]).ravel()
    pos = np.concatenate([bases - 1, bases, bases + 1, wins - 1, wins, [m.n * BB - 1]])
    pos = np.concatenate([np.unique(pos[pos >= 0]).astype(U64), past_end(m.n)])
    ranks = np.unique(np.concatenate([m.pre[:-1], m.pre[:-1] + U64(1), m.pre[1:], [0, m.total + 1]]).astype(U64))
    return pos, ranks


@gpu
@pytest.mark.parametrize("n", SB_SIZES)
def test_superblock_layouts(ctx, n):
    vecs = superblock_vectors(n)
    ps = bm.PackedSet.pack(vecs)
    dset = bm.DeviceSet.upload(ctx, ps)
    for v, bv in enumerate(vecs):
        m = RSModel(bv)
        rs = bm.DeviceRS(ctx, dset, v)
        check_export(rs, ps, v, m)
        pos, ranks = edge_queries(m)
        check_rank(rs.rank(pos), m.rank(pos), pos, bv, None, f"n={n} vector {v}")
        check_select(rs.select(ranks), m.select(ranks), ranks, m, None, f"n={n} vector {v}")
        rs.free()
    dset.free()


# ------------------------------------------------------------------ GPU 4: more than 1024 superblocks

def sparse_vector(n):
    """1 to 3 non-NULL blocks per superblock, cycling through corpus shapes and FULL; the blocks around 2^32 bits, around the
    start of the second 1024-superblock pass and the last block are always non-NULL."""
    g, b = [d for _, d in gap_corpus()], [d for _, d in bit_corpus()]
    pool = [g[0], b[-1], None, g[-2], b[5], b[0], g[-9]]                # None = FULL
    bv = bm.BVector(n)

    def put(nb, d):
        if d is None:
            bv.set_full(nb)
        else:
            (bv.set_gap if d.dtype == np.uint16 else bv.set_bits)(nb, d)

    for s in range((n + 255) // 256):
        offs = ((37 * s) % 256, (101 * s + 7) % 256, (173 * s + 11) % 256)[: 1 + s % 3]
        for j, o in enumerate(offs):
            if 256 * s + o < n:
                put(256 * s + o, pool[(3 * s + j) % len(pool)])
    forced = {65535: b[1], 65536: g[1], 262143: g[0], 262144: b[-3], n - 1: g[-1]}
    for nb, d in forced.items():
        if nb < n:
            put(nb, d)
    return bv, sorted(nb for nb in forced if nb < n)


@gpu
@pytest.mark.parametrize("n", [262144, 262145, 300037])
def test_more_than_1024_superblocks(ctx, n):
    bv, exhaustive = sparse_vector(n)
    m = RSModel(bv)
    ps = bm.PackedSet.pack([bv])
    dset = bm.DeviceSet.upload(ctx, ps)
    rs = bm.DeviceRS(ctx, dset, 0)
    nsb = (n + 255) // 256
    assert nsb >= 1024 and rs.total() == m.total
    check_export(rs, ps, 0, m)
    sb = m.sb_count()
    bases = np.arange(nsb, dtype=U64) * U64(256 * BB)
    pos = np.concatenate([bases[1:] - U64(1), bases, bases + U64(1), past_end(n)])
    got = rs.rank(pos)
    check_rank(got, m.rank(pos), pos, bv, None, f"n={n} superblock bases")
    assert np.array_equal(got, orclib.oracle_rank(ps, 0, pos))
    nz = np.flatnonzero(sb[1:] > sb[:-1])
    ranks = np.concatenate([sb[nz] + U64(1), sb[nz + 1], [0, m.total + 1]]).astype(U64)
    sel = rs.select(ranks)
    check_select(sel, m.select(ranks), ranks, m, None, f"n={n} first and last rank of every superblock")
    for nb in exhaustive:
        p = np.arange(nb * BB, (nb + 1) * BB, dtype=U64)
        check_rank(rs.rank(p), m.block_rank(nb), p, bv, None, f"n={n} block {nb}")
    if orclib.have_ref(True):                                            # the real BM64ADDR reference on a sample
        rp, rr = pos[::7], ranks[::7]
        r_rank, r_pos, r_found, _ = orclib.ref_rank_select(ps, 0, rp, rr, addr64=True)
        assert np.array_equal(r_rank, got[::7])
        assert np.array_equal(r_found, sel[1][::7]) and np.array_equal(r_pos[r_found], sel[0][::7][r_found])
    rs.free(); dset.free()


# ------------------------------------------------------------------ GPU 5: the device entry points

@gpu
def test_device_entry_points_past_one_grid_trip():
    """rank_dev / select_dev on CUDA int64 tensors, on torch's current stream; 5 M queries take several trips of the capped grid
    (sm_count * 32 CTAs of 256 threads).  Answers == the host entry points == the model."""
    import torch
    _, labels, models = corpus()
    m = models[0]
    dev = torch.device("cuda", 0)
    c2 = bm.Context(0)
    c2.set_stream(torch.cuda.current_stream(dev).cuda_stream)
    sms = c2.device_info().get("sm_count", 132)
    big = 5_000_000
    assert big > 4 * sms * 32 * 256
    rng = np.random.default_rng(55)
    dset = bm.DeviceSet.upload(c2, corpus_set(True))
    rs = bm.DeviceRS(c2, dset, 0)
    try:
        for n in (1, 255, 257, big):
            pos = rng.integers(0, (m.n + 1) * BB, n, dtype=np.int64)
            ranks = rng.integers(0, m.total + 2, n, dtype=np.int64)
            tpos, trk = torch.from_numpy(pos).to(dev), torch.from_numpy(ranks).to(dev)
            out = torch.empty_like(tpos)
            tp, tf = torch.empty_like(trk), torch.empty(n, dtype=torch.uint8, device=dev)
            rs.rank_dev(tpos.data_ptr(), n, out.data_ptr())
            rs.select_dev(trk.data_ptr(), n, tp.data_ptr(), tf.data_ptr())
            got_rank = out.cpu().numpy().view(U64)
            got_sel = (tp.cpu().numpy().view(U64), tf.cpu().numpy().astype(bool))
            upos, urk = pos.view(U64), ranks.view(U64)
            check_rank(got_rank, m.rank(upos), upos, m.bv, labels[0], f"rank_dev n={n}")
            assert np.array_equal(got_rank, rs.rank(upos))
            check_select(got_sel, m.select(urk), urk, m, labels[0], f"select_dev n={n}")
            hp, hf = rs.select(urk)
            assert np.array_equal(hf, got_sel[1]) and np.array_equal(hp, got_sel[0])
    finally:
        torch.cuda.synchronize(dev)
        rs.free(); dset.free()                                            # before the context they belong to
        c2.close()


# ------------------------------------------------------------------ GPU 6: rebuild after the bits change

def rewritten(words, i):
    """new contents for bit-block i of the pool: its complement, or its words rotated"""
    return ~words if i % 2 == 0 else np.roll(words, 37 * i + 1) ^ np.uint32(0x0F0F0F0F * (i % 3))


@gpu
def test_rebuild_after_the_bits_change(ctx):
    """An adopted, torch-owned set: the index is built, bit-block words are overwritten in place (kinds and descriptors stay),
    rs.rebuild() must then answer for the new bits.  Vector 1 is all NULL: total 0, every rank 0, no select found."""
    import torch
    from bitmagic_b200 import capi
    vecs, labels, models = corpus()
    bvec = vecs[1]
    ps = bm.PackedSet.pack([bvec, bm.BVector(bvec.n_blocks)])
    dev = torch.device("cuda", 0)

    def up(a, pad=0):
        t = torch.zeros(a.nbytes + pad, dtype=torch.uint8, device=dev)
        t[: a.nbytes] = torch.from_numpy(a.view(np.uint8)).to(dev)
        return t
    t_desc, t_bb, t_gb = up(ps.desc), up(ps.bit_base), up(ps.gap_base)
    t_bp, t_gp = up(ps.bit_pool, 512), up(ps.gap_pool, 512)               # caller-owned pools need the 512-byte read slack
    c = capi.PackedSetC(ps.n_vec, ps.n_blocks, t_desc.data_ptr(), t_bb.data_ptr(), t_gb.data_ptr(), t_bp.data_ptr(), t_gp.data_ptr())
    h = ctypes.c_void_p(0)
    torch.cuda.synchronize(dev)                                            # the pools are written on torch's stream, read on the context's
    ctx.check(capi.lib().bmb200_set_adopt_device(ctx._h, ctypes.byref(c), ctypes.byref(h)), "set_adopt_device")
    dset = capi.DeviceSet(ctx, h)
    rs, rs0 = bm.DeviceRS(ctx, dset, 0), bm.DeviceRS(ctx, dset, 1)
    pos = np.arange(bvec.n_blocks * BB, dtype=U64)
    check_rank(rs.rank(pos), models[1].rank(pos), pos, bvec, labels[1], "before the rewrite")

    new_pool = np.concatenate([rewritten(w, i) for i, w in enumerate(ps.bit_pool.reshape(-1, 2048))])
    ctx.sync()
    t_bp[: new_pool.nbytes] = torch.from_numpy(new_pool.view(np.uint8)).to(dev)
    torch.cuda.synchronize(dev)
    rs.rebuild(); rs0.rebuild()
    ps2 = bm.PackedSet(ps.n_vec, ps.n_blocks, ps.desc, ps.bit_base, ps.gap_base, new_pool, ps.gap_pool)
    nv = ps2.vector(0)
    m = RSModel(nv)
    assert m.total != models[1].total
    check_export(rs, ps2, 0, m)
    check_rank(rs.rank(pos), m.rank(pos), pos, nv, labels[1], "after the rewrite")
    ranks = np.arange(m.total + 2, dtype=U64)
    check_select(rs.select(ranks), m.select(ranks), ranks, m, labels[1], "after the rewrite")

    assert rs0.total() == 0 and not rs0.export()[2].any()
    q = np.concatenate([pos[::4099], past_end(bvec.n_blocks)])
    assert not rs0.rank(q).any()
    p, f = rs0.select(np.array([0, 1, 2, 65536, 2**40], U64))
    assert not f.any() and not p.any()
    rs.free(); rs0.free(); dset.free()
    assert bool((t_bp[: new_pool.nbytes].cpu().numpy().view(np.uint32) == new_pool).all())      # the adopted pool stays torch's


# ------------------------------------------------------------------ CPU: the model against the oracle and the reference

def boundary_sample(m):
    """positions: in every block, 0, 1, the word and window edges, 512k-1 / 512k / 512k+1, the rs3 and aux borders +-1, 65535,
    and past the end; ranks: in every non-NULL block, the ones before each window (+0, +1), the block's last rank, 0, total + 1"""
    offs = [0, 1, 31, 32, 33, 511, 512, 513, BB - 2, BB - 1]
    offs += [b + d for b in RS3 + AUX for d in (-1, 0, 1)]
    offs += (np.arange(1, 128)[:, None] * WIN + np.array([-1, 0, 1])[None, :]).ravel().tolist()
    offs = np.unique(offs)
    pos = (np.arange(m.n, dtype=U64)[:, None] * U64(BB) + offs.astype(U64)[None, :]).ravel()
    pos = np.concatenate([pos, past_end(m.n)])
    ranks = [np.array([0, m.total, m.total + 1], U64)]
    for nb in np.flatnonzero(m.bv.kind != bm.BLK_NULL):
        br = m.block_rank(nb)
        before = np.concatenate([[m.pre[nb]], br[WIN - 1::WIN]])         # ones before window k, k = 0 .. 128
        ranks += [before, before + U64(1)]
    ranks = np.unique(np.concatenate(ranks))
    return pos, ranks[ranks <= U64(m.total + 1)]


@FORMS
def test_model_matches_oracle(flat):
    """On the boundary sample of every corpus vector and every superblock layout, the model == orc_rank_batch / orc_select_batch,
    and the model's block counts and superblock totals == orc_rs_build."""
    models = corpus()[2]
    sets = [(corpus_set(flat), models)]
    for n in SB_SIZES:
        sv = superblock_vectors(n)
        sets.append((bm.PackedSet.pack(sv, gap_flat=flat), [RSModel(v) for v in sv]))
    for ps, ms in sets:
        for v, m in enumerate(ms):
            pos, ranks = boundary_sample(m)
            assert np.array_equal(m.rank(pos), orclib.oracle_rank(ps, v, pos)), (ps.n_blocks, v)
            wp, wf = m.select(ranks)
            op, of = orclib.oracle_select(ps, v, ranks)
            assert np.array_equal(wf, of) and np.array_equal(wp[wf], op[of]), (ps.n_blocks, v)
            bc, sc, sb = orclib.oracle_rs_build(ps, v)
            assert np.array_equal(bc.astype(U64), m.cnt) and np.array_equal(sb, m.sb_count()), (ps.n_blocks, v)


def test_model_for_sparse_vectors_matches_oracle():
    """The model built from per-block counts, on a vector of 262145 blocks, == the oracle at every superblock base."""
    bv, _ = sparse_vector(262145)
    m = RSModel(bv)
    ps = bm.PackedSet.pack([bv])
    pos = np.concatenate([np.arange(1026, dtype=U64) * U64(256 * BB) + U64(d) for d in (0, 1, 65535)])
    assert np.array_equal(m.rank(pos), orclib.oracle_rank(ps, 0, pos))
    sb = m.sb_count()
    ranks = np.concatenate([sb + U64(1), sb, [0]]).astype(U64)
    wp, wf = m.select(ranks)
    op, of = orclib.oracle_select(ps, 0, ranks)
    assert np.array_equal(wf, of) and np.array_equal(wp[wf], op[of])
    assert np.array_equal(orclib.oracle_rs_build(ps, 0)[2], sb)


@needs_ref_answers
def test_model_matches_reference():
    """On the boundary sample of every corpus vector, the model == the reference's count_to / select and its rs_index block
    counts and superblock totals (bvector::build_rs_index)."""
    models = corpus()[2]
    ps = corpus_set(True)
    for v, m in enumerate(models):
        pos, ranks = boundary_sample(m)
        r_rank, r_pos, r_found, _ = orclib.ref_rank_select(ps, v, pos, ranks)
        assert np.array_equal(r_rank, m.rank(pos)), v
        wp, wf = m.select(ranks)
        assert np.array_equal(r_found, wf) and np.array_equal(r_pos[wf], wp[wf]), v
        bc, sc, sb, tot = orclib.ref_rs_build(ps, v)
        assert tot == m.total and np.array_equal(bc.astype(U64), m.cnt) and np.array_equal(sb, m.sb_count()), v
        assert np.array_equal(sc, orclib.oracle_rs_build(ps, v)[1]), v
