"""Argument checks of the residual-batch Fp that run before any device work (CPU): ``fastfp_pack_set_residuals`` and
``fastfp_fp_sweep_residuals`` through ctypes, the shape checks of ``FastFp.calculate_Fp_batch``, and the pass-size
rule for more realisations than one pass takes."""
import ctypes

import numpy as np
import pytest

import fastfp_b200
from fastfp_b200 import _cabi, synth
from fastfp_b200.fastfp import _tile_cost, batch_pass_rows

NOT_A_PACK = ctypes.c_void_p(1)  # never dereferenced: every case below is refused on its arguments alone


def test_symbols_are_exported():
    lib = _cabi.load()
    for name in ("fastfp_pack_set_residuals", "fastfp_fp_sweep_residuals"):
        assert name in _cabi.SYMBOLS
        assert getattr(lib, name) is not None


def test_set_residuals_rejects_null_and_negative_arguments():
    lib = _cabi.load()
    one = np.zeros(4)
    arr = _cabi._ptr_array([one])
    assert lib.fastfp_pack_set_residuals(None, 1, arr, None) == -1
    assert lib.fastfp_pack_set_residuals(NOT_A_PACK, -1, arr, None) == -1
    assert lib.fastfp_pack_set_residuals(NOT_A_PACK, 2, None, None) == -1
    assert lib.fastfp_last_error().decode() == "fastfp_pack_set_residuals: null argument or negative R"


@pytest.mark.parametrize("F,freqs,out", [(-1, True, True), (3, False, True), (3, True, False)])
def test_sweep_residuals_rejects_null_and_negative_arguments(F, freqs, out):
    lib = _cabi.load()
    f, o = np.ones(3), np.empty(3)
    vp = lambda a: ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    assert lib.fastfp_fp_sweep_residuals(NOT_A_PACK, vp(f) if freqs else None, F, vp(o) if out else None, 0,
                                         None) == -1
    assert lib.fastfp_last_error().decode() == "fastfp_fp_sweep_residuals: null argument or negative F"
    assert lib.fastfp_fp_sweep_residuals(None, vp(f), 3, vp(o), 0, None) == -1


def test_front_end_rejects_residuals_of_the_wrong_shape():
    pta = synth.make_pta(3, [40, 57, 33], n_tm=3, ncomps=2)
    fp = fastfp_b200.FastFp(pta.psrs)
    a = (None, None, None)
    good = [np.zeros((4, n)) for n in (40, 57, 33)]
    cases = {
        "wrong R": [good[0], np.zeros((5, 57)), good[2]],
        "wrong n_p": [good[0], good[1], np.zeros((4, 34))],
        "1-D": [good[0], good[1], np.zeros(33)],
        "no rows": [np.zeros((0, n)) for n in (40, 57, 33)],
    }
    for what, res in cases.items():
        with pytest.raises(ValueError, match="residuals"):
            fp.calculate_Fp_batch(1e-8, *a, res)
    with pytest.raises(ValueError, match="one per pulsar"):
        fp.calculate_Fp_batch(1e-8, *a, good[:2])


def test_limit_and_pass_rule():
    # a pulsar takes roundup8(m) + roundup8(R) of the kernel's 640 G rows
    assert _cabi.max_residual_rows([72]) == 568
    assert _cabi.max_residual_rows([12, 72, 65]) == 568
    assert _cabi.max_residual_rows([12]) == 624
    assert _cabi.max_residual_rows([73]) == 560
    for R in (1, 248, 249):  # one pass where the library takes them all and splitting models no cheaper
        assert batch_pass_rows(R, [72]) == R
    for m, R in ((72, 568), (72, 569), (72, 1000), (12, 624), (12, 5000), (300, 340)):
        rows = batch_pass_rows(R, [m])
        assert 1 <= rows <= _cabi.max_residual_rows([m])
        assert rows * (-(-R // rows) - 1) < R  # evened out: the last pass is not empty


def _plan_cost(R, m, rows):
    return -(-R // rows) * _tile_cost(-(-m // 8) * 8 + -(-rows // 8) * 8)


@pytest.mark.parametrize("m", [200, 256, 296, 304, 305, 312, 313, 320])
def test_wide_bases_never_split_into_a_costlier_plan(m):
    """Near m = 300 the 16-frequency family leaves room for a few rows only: a pass rule keyed on that family alone would
    sweep R = 328 at m = 312 in 41 passes of 8 rows where the library takes all of them in one."""
    rmax = _cabi.max_residual_rows([m])
    for R in sorted({1, 8, 9, 24, 100, rmax // 2, rmax, rmax + 1, 3 * rmax}):
        rows = batch_pass_rows(R, [m])
        assert rows <= rmax
        if R <= rmax:  # never worse than the one library pass
            assert _plan_cost(R, m, rows) <= _plan_cost(R, m, R), (m, R, rows)
    assert batch_pass_rows(328, [312]) == 328
    assert batch_pass_rows(24, [304]) == 24  # one 384-row pass, measured cheaper than two 320-row ones
