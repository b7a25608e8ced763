"""Argument checks of the sky-maximised Fe-statistic that run before any device work (CPU): ``fastfp_fe_skymax``
through ctypes and the sky-grid check of ``FastFe.calculate_Fe_skymax``."""
import ctypes

import numpy as np
import pytest

import fastfp_b200
from fastfp_b200 import _cabi, synth

NOT_A_PACK = ctypes.c_void_p(1)  # never dereferenced: every case below is refused on its arguments alone


def _call(F, S, fe_max=True, sky_index=True):
    lib = _cabi.load()
    f = np.ones(max(F, 1))
    fp = np.ones(max(S, 1) * 2)
    out = np.empty(max(F, 1))
    idx = np.empty(max(F, 1), dtype=np.int64)
    vp = lambda a: ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    return lib.fastfp_fe_skymax(NOT_A_PACK, vp(f), F, vp(fp), vp(fp), S, vp(out) if fe_max else None,
                                vp(idx) if sky_index else None, 0, None)


@pytest.mark.parametrize("which", ["fe_max", "sky_index"])
def test_null_outputs_are_rejected(which):
    assert _call(3, 2, fe_max=which != "fe_max", sky_index=which != "sky_index") == -1
    assert _cabi.load().fastfp_last_error().decode() == "fastfp_fe_skymax: null argument or negative size"


@pytest.mark.parametrize("F,S", [(-1, 2), (3, -1), (-1, -1)])
def test_negative_sizes_are_rejected(F, S):
    assert _call(F, S) == -1
    assert _cabi.load().fastfp_last_error().decode() == "fastfp_fe_skymax: null argument or negative size"


def test_null_pack_is_rejected():
    lib = _cabi.load()
    assert lib.fastfp_fe_skymax(None, None, 1, None, None, 1, None, None, 0, None) == -1


def test_front_end_rejects_a_sky_grid_that_does_not_broadcast():
    psrs = synth.make_pta(2, 24, n_tm=3, ncomps=2).psrs
    fe = fastfp_b200.FastFe(psrs)
    for th, ph in [(np.zeros(3), np.zeros(4)), (np.zeros((2, 3)), np.zeros(3))]:
        with pytest.raises(ValueError, match="broadcast"):
            fe.calculate_Fe_skymax(1e-8, th, ph, None, None, None)
