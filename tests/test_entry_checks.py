"""Argument checks of the result-producing entry points: the return code of a bad column range, plane range or universe, and
which check wins when two fail at once.  A refused call leaves no result behind."""
from __future__ import annotations

import numpy as np
import pytest

import bitmagic_b200 as bm
from bitmagic_b200.capi import ERR_BADARG, ERR_RANGE

gpu = pytest.mark.gpu

NB, NV = 3, 8          # the set: 8 vectors of 3 blocks


def _scan(ctx, dset, res, pred=bm.SCAN_EQ, values=(1,), plane0=0, n_planes=4, universe=bm.NO_UNIVERSE, flags=0, nb_from=0, nb_to=0):
    if pred in (bm.SCAN_RANGE, bm.SCAN_RANGE_OPEN):
        values = [[v, v] for v in values]
    bm.scan(ctx, dset, pred, values, plane0, n_planes, universe, flags, nb_from, nb_to, result=res)


def _binop(ctx, dset, res, op=bm.OP_AND, va=0, vb=1, flags=0, nb_from=0, nb_to=0):
    bm.capi.binop(ctx, dset, op, va, vb, flags, nb_from, nb_to, result=res)


def _batch(ctx, dset, res, op=bm.OP_OR, groups=(([0, 1], None),), flags=0, nb_from=0, nb_to=0):
    bm.aggregate_batch(ctx, dset, op, list(groups), flags, nb_from, nb_to, result=res)


def _mismatch(ctx, dset, res, **kw):
    a = dict(plane0_a=0, n_planes_a=2, plane0_b=2, n_planes_b=2)
    a.update(kw)
    bm.capi.sv_mismatch(ctx, dset, bm.capi.mismatch_args(**a), result=res)


CASES = [
    # bmb200_scan: column range, plane range, universe
    ("scan nb_from == nb_to", _scan, dict(nb_from=NB), ERR_RANGE),
    ("scan nb_from > nb_to", _scan, dict(nb_from=2, nb_to=1), ERR_RANGE),
    ("scan nb_to past the set", _scan, dict(nb_to=NB + 1), ERR_RANGE),
    ("scan planes past the set", _scan, dict(plane0=NV - 3), ERR_RANGE),
    ("scan universe past the set", _scan, dict(universe=NV), ERR_RANGE),
    ("scan signed gt planes past the set", _scan, dict(pred=bm.SCAN_GT, flags=bm.F_SIGNED, plane0=NV - 3), ERR_RANGE),
    ("scan float range nb_to past the set", _scan, dict(pred=bm.SCAN_RANGE, flags=bm.F_FLOAT, nb_to=NB + 1), ERR_RANGE),
    ("scan too many planes before the range", _scan, dict(n_planes=65, nb_from=NB), ERR_BADARG),
    ("scan float eq before the planes", _scan, dict(flags=bm.F_FLOAT, plane0=NV), ERR_BADARG),
    ("scan_in nb_to past the set", _scan, dict(pred=bm.SCAN_IN, nb_to=NB + 1), ERR_RANGE),
    ("scan_in planes past the set", _scan, dict(pred=bm.SCAN_IN, plane0=NV - 3), ERR_RANGE),
    # bmb200_binop: column range, vectors, flags
    ("binop nb_from == nb_to", _binop, dict(nb_from=NB), ERR_RANGE),
    ("binop nb_from > nb_to", _binop, dict(nb_from=2, nb_to=1), ERR_RANGE),
    ("binop nb_to past the set", _binop, dict(nb_to=NB + 1), ERR_RANGE),
    ("binop vector past the set", _binop, dict(vb=NV), ERR_RANGE),
    ("binop count-only before the range", _binop, dict(flags=bm.F_COUNT_ONLY, nb_from=NB), ERR_BADARG),
    # bmb200_aggregate_batch: column range, members, op
    ("batch nb_from == nb_to", _batch, dict(nb_from=NB), ERR_RANGE),
    ("batch nb_from > nb_to", _batch, dict(nb_from=2, nb_to=1), ERR_RANGE),
    ("batch nb_to past the set", _batch, dict(nb_to=NB + 1), ERR_RANGE),
    ("batch shift nb_to past the set", _batch, dict(op=bm.OP_SHIFT_R_AND, nb_to=NB + 1), ERR_RANGE),
    ("batch member past the set", _batch, dict(groups=(([0, NV], None),)), ERR_RANGE),
    ("batch bad op before the range", _batch, dict(op=99, nb_from=NB), ERR_BADARG),
    # bmb200_sv_mismatch: planes outside the set are a bad argument, the column range a range error
    ("mismatch planes past the set", _mismatch, dict(plane0_b=NV - 1), ERR_BADARG),
    ("mismatch not-null past the set", _mismatch, dict(not_null_a=NV), ERR_BADARG),
    ("mismatch nb_to past the set", _mismatch, dict(nb_to=NB + 1), ERR_RANGE),
    ("mismatch planes before the range", _mismatch, dict(plane0_a=NV, nb_from=NB), ERR_BADARG),
]


@pytest.fixture(scope="module")
def dset(ctx):
    rng = np.random.default_rng(5)
    ds = bm.DeviceSet.upload(ctx, bm.PackedSet.pack([bm.BVector.random(NB, 0.3, rng) for _ in range(NV)]))
    yield ds
    ds.free()


@gpu
@pytest.mark.parametrize("call, kw, code", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_entry_point_refuses(ctx, dset, call, kw, code):
    res = bm.capi.DeviceResult(ctx)
    with pytest.raises(bm.BMB200Error) as e:
        call(ctx, dset, res, **kw)
    assert e.value.code == code
    assert not res._h.value
