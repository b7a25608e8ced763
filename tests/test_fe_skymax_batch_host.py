"""Argument checks of the residual-batch sky-maximised Fe that run before any device work (CPU):
``fastfp_fe_skymax_residuals`` through ctypes and the shape checks of ``FastFe.calculate_Fe_skymax_batch``."""
import ctypes

import numpy as np
import pytest

import fastfp_b200
from fastfp_b200 import _cabi, synth

NOT_A_PACK = ctypes.c_void_p(1)  # never dereferenced: every case below is refused on its arguments alone
MSG = "fastfp_fe_skymax_residuals: null argument or negative size"


def test_symbol_is_exported():
    assert "fastfp_fe_skymax_residuals" in _cabi.SYMBOLS
    assert _cabi.load().fastfp_fe_skymax_residuals is not None


def _vp(a):
    return ctypes.c_void_p(a.ctypes.data)


@pytest.mark.parametrize("drop", ["pack", "freqs", "fplus", "fcross", "fe_max", "sky_index"])
def test_rejects_null_arguments(drop):
    lib = _cabi.load()
    a = dict(pack=NOT_A_PACK, freqs=_vp(np.ones(3)), fplus=_vp(np.ones(4)), fcross=_vp(np.ones(4)),
             fe_max=_vp(np.empty(3)), sky_index=_vp(np.empty(3, dtype=np.int64)))
    a[drop] = None
    assert lib.fastfp_fe_skymax_residuals(a["pack"], a["freqs"], 3, a["fplus"], a["fcross"], 2, a["fe_max"],
                                          a["sky_index"], 0, None) == -1
    assert lib.fastfp_last_error().decode() == MSG


@pytest.mark.parametrize("F,S", [(-1, 2), (3, -1), (-1, -1)])
def test_rejects_negative_sizes(F, S):
    lib = _cabi.load()
    f, p, o, i = np.ones(3), np.ones(4), np.empty(3), np.empty(3, dtype=np.int64)
    assert lib.fastfp_fe_skymax_residuals(NOT_A_PACK, _vp(f), F, _vp(p), _vp(p), S, _vp(o), _vp(i), 0, None) == -1
    assert lib.fastfp_last_error().decode() == MSG


def test_front_end_rejects_bad_residuals_and_sky_grids():
    pta = synth.make_pta(3, [40, 57, 33], n_tm=3, ncomps=2)
    fe = fastfp_b200.FastFe(pta.psrs)
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
            fe.calculate_Fe_skymax_batch(1e-8, 0.5, 1.0, *a, res)
    with pytest.raises(ValueError, match="one per pulsar"):
        fe.calculate_Fe_skymax_batch(1e-8, 0.5, 1.0, *a, good[:2])
    for th, ph in ((np.zeros(3), np.zeros(4)), (np.zeros((2, 3)), np.zeros((2, 3)))):
        with pytest.raises(ValueError, match="broadcast to one shape"):
            fe.calculate_Fe_skymax_batch(1e-8, th, ph, *a, good)
