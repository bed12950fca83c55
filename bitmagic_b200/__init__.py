"""bitmagic_b200 -- H100 (sm_90a) block-level set algebra + rank/select for BitMagic-format bit-vectors.

Product code: csrc/ (CUDA kernels + the C ABI of include/bmb200.h, built into libbmb200.so) and a thin
host-side mirror of the reference operator surface (aggregator.py, scanner.py, hostfmt.py, capi.py).
There is no CPU fallback: importing works anywhere, computing needs libbmb200.so and an H100.
"""
from .capi import (BLK_BIT, BLK_FULL, BLK_GAP, BLK_NULL, F_COUNT_ONLY, F_OPT_COMPRESS, F_OPT_NONE, F_OR_TARGET, OP_AND,
                   OP_AND_SUB, OP_OR, OP_XOR, OP_SHIFT_R_AND, BMB200Error, Context, DeviceResult, DeviceRS, DeviceSet,
                   aggregate, aggregate_batch, aggregate_host, default_context, scan, rank_compress, rank_decompress,
                   SCAN_EQ, SCAN_GE, SCAN_GT, SCAN_LE, SCAN_LT, SCAN_RANGE, NO_UNIVERSE)
from .hostfmt import BVector, PackedSet, result_to_bvector
from .scanner import RscSparseVector, SparseVector, SparseVectorScanner
from .aggregator import (OPT_COMPRESS, OPT_NONE, Aggregator, Pipeline, RSIndex, bit_and, bit_or, bit_or_and, bit_sub, bit_xor, merge,
                         build_rs_index, count_and, count_or, count_sub, count_xor)

__all__ = [n for n in dir() if not n.startswith("_")]
