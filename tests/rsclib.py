"""Checkers of the rank-select compressed sparse vector path (test infrastructure):

* a plain numpy restatement of bm::rank_compressor (src/bmalgo.h:498-644) on dense bit arrays;
* ctypes access to oracle/_ref/libbmref_rsc.so (oracle/ref_rsc_shim.cpp: the unmodified reference's rsc_sparse_vector,
  sparse_vector_scanner<rsc_sparse_vector> and rank_compressor), with its answers recorded under tests/golden/ref like
  orclib's (BMB200_RECORD_REF=1 rewrites them where the library is built; elsewhere the recorded answers stand in)."""
from __future__ import annotations

import ctypes as C
import functools
import hashlib
import os

import numpy as np

import orclib
from bitmagic_b200.capi import BLOCK_BITS, BLOCK_WORDS, SCAN_RANGE, ptr

REF_RSC = orclib.ORACLE_DIR / "_ref" / "libbmref_rsc.so"
_lib = None


# ---- numpy restatement ----
def bits_of(words) -> np.ndarray:
    return np.unpackbits(np.ascontiguousarray(words, dtype="<u4").view(np.uint8), bitorder="little")


def words_of(bits, n_cols: int) -> np.ndarray:
    b = np.zeros(n_cols * BLOCK_BITS, np.uint8)
    b[:min(len(bits), b.size)] = np.asarray(bits, np.uint8)[:b.size]
    return np.packbits(b, bitorder="little").view("<u4").astype(np.uint32)


def np_rank_compress(nn_bits, src_bits) -> np.ndarray:
    """bit r = src at the position of the (r+1)-th set bit of NN (src & NN for a source that is not a subset)"""
    pos = np.flatnonzero(nn_bits)
    s = np.zeros(max(len(nn_bits), len(src_bits)), np.uint8); s[:len(src_bits)] = src_bits
    return s[pos].astype(np.uint8)


def np_rank_decompress(nn_bits, comp_bits) -> np.ndarray:
    """bit p = NN[p] and compressed bit rank_NN(p) - 1; compressed bits at or past count(NN) are never read"""
    pos = np.flatnonzero(nn_bits)
    c = np.zeros(pos.size, np.uint8); n = min(pos.size, len(comp_bits)); c[:n] = np.asarray(comp_bits, np.uint8)[:n]
    out = np.zeros(len(nn_bits), np.uint8)
    out[pos] = c
    return out


# ---- the reference ----
def have_ref_rsc() -> bool:
    return REF_RSC.exists()


def ref_rsc() -> C.CDLL:
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(REF_RSC))
    return _lib


def _recorded(fn):
    """orclib._recorded, keyed on libbmref_rsc.so"""
    @functools.wraps(fn)
    def call(*args, **kw):
        h = hashlib.sha256(fn.__name__.encode())
        orclib._hash_arg(args, h); orclib._hash_arg(sorted(kw.items()), h)
        path = orclib.GOLDEN_REF / f"{fn.__name__}_{h.hexdigest()[:20]}.npz"
        if have_ref_rsc():
            out = fn(*args, **kw)
            if os.environ.get("BMB200_RECORD_REF"):
                orclib._save_answer(path, out)
            elif path.exists():
                assert orclib._same_answer(out, orclib._load_answer(path)), f"{path.name} differs from the reference's answer; re-record it"
            return out
        if not path.exists():
            raise FileNotFoundError(f"reference library not built and no recorded answer {path.name} for this {fn.__name__} call")
        return orclib._load_answer(path)
    return call


def _n_cols(n: int) -> int:
    return max(1, (n + BLOCK_BITS - 1) // BLOCK_BITS)


@_recorded
def ref_rsc_planes(values, nulls, max_planes=32):
    """The real rsc_sparse_vector built from the nullable sparse vector -> (effective_size, planes[n_planes][words], nn[words])"""
    v = np.ascontiguousarray(values, dtype=np.uint32); nl = np.ascontiguousarray(nulls, dtype=np.uint8)
    nc = _n_cols(v.size)
    words = np.zeros((max_planes + 1) * nc * BLOCK_WORDS, np.uint32)
    npl, eff = C.c_uint32(0), C.c_uint64(0)
    rc = ref_rsc().ref_rsc_planes(ptr(v), ptr(nl), C.c_uint64(v.size), C.c_uint32(nc), C.c_uint32(max_planes), C.byref(npl),
                                  C.byref(eff), ptr(words))
    assert rc == 0, f"ref_rsc_planes rc={rc}"
    w = words.reshape(max_planes + 1, nc * BLOCK_WORDS)
    return int(eff.value), w[:npl.value].copy(), w[npl.value].copy()


@_recorded
def ref_rsc_scan(values, nulls, pred, search):
    """The real sparse_vector_scanner<rsc_sparse_vector<unsigned>> -> counts[n_search], words[n_search][n_cols * 2048]"""
    v = np.ascontiguousarray(values, dtype=np.uint32); nl = np.ascontiguousarray(nulls, dtype=np.uint8)
    sv = np.ascontiguousarray(search, dtype=np.uint32)
    ns = sv.shape[0] if pred == SCAN_RANGE else sv.size
    nc = _n_cols(v.size)
    counts = np.zeros(ns, np.uint64); words = np.zeros((ns, nc * BLOCK_WORDS), np.uint32)
    rc = ref_rsc().ref_rsc_scan(ptr(v), ptr(nl), C.c_uint64(v.size), int(pred), ptr(sv), C.c_uint32(ns), C.c_uint32(nc),
                                ptr(counts), ptr(words))
    assert rc == 0, f"ref_rsc_scan rc={rc}"
    return counts, words


def _ref_rank(name, idx_words, src_words, n_out_cols):
    i = np.ascontiguousarray(idx_words, dtype=np.uint32); s = np.ascontiguousarray(src_words, dtype=np.uint32)
    assert i.size == s.size and i.size % BLOCK_WORDS == 0
    out = np.zeros(n_out_cols * BLOCK_WORDS, np.uint32); cnt = C.c_uint64(0)
    rc = getattr(ref_rsc(), name)(ptr(i), ptr(s), C.c_uint32(i.size // BLOCK_WORDS), C.c_uint32(n_out_cols), ptr(out), C.byref(cnt))
    assert rc == 0, f"{name} rc={rc}"
    return int(cnt.value), out


@_recorded
def ref_rank_compress(idx_words, src_words, n_out_cols):
    """The real rank_compressor<bvector<>>::compress (src must be a subset of idx) -> (count, target words)"""
    return _ref_rank("ref_rank_compress", idx_words, src_words, n_out_cols)


@_recorded
def ref_rank_decompress(idx_words, src_words, n_out_cols):
    """The real rank_compressor<bvector<>>::decompress (src below count(idx)) -> (count, target words)"""
    return _ref_rank("ref_rank_decompress", idx_words, src_words, n_out_cols)
