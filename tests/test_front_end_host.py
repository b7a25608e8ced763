"""The host-input contract of the ``FastFp`` / ``FastFe`` front ends (CPU): with a stub in place of the device pack,
which records what each method hands the pack and fills the outputs with values derived from their positions, check
what ``calculate_Fp``, ``calculate_Fp_batch``, ``calculate_Fe``, ``calculate_Fe_skymax`` and
``calculate_Fe_skymax_batch`` return for scalar, ``(F,)`` and ``(2, 3)`` frequencies and scalar or array skies, and
how the batch methods split and cache their realisations. The CUDA-tensor forms run in the GPU suite."""
import numpy as np
import pytest

import fastfp_b200
from fastfp_b200.fastfp import FastFp, batch_pass_rows
from fastfp_b200.fe import antenna_pattern

N = [5, 7]
POS = np.array([[1.0, 0.0, 0.0], [0.0, 0.6, 0.8]])


class _Psr:
    def __init__(self, n, pos):
        self.toas = np.linspace(0.0, 1e8, n)
        self.residuals = np.zeros(n)
        self.pos = pos


class StubPack:
    """Records every call; outputs are freqs (+ the row's residual tag res[0][k, 0], + the sky's pattern sums)."""

    def __init__(self, m):
        self.P, self.m, self.n = len(N), list(m), list(N)
        self.calls, self.res = [], None

    def close(self):
        pass

    def _fill(self, out, shape, value, dtype=np.float64):
        if out is None:
            return np.asarray(value, dtype=dtype).reshape(shape)
        assert isinstance(out, np.ndarray) and out.shape == shape and out.dtype == dtype and out.flags.c_contiguous
        out[...] = value
        return None

    def _freqs(self, name, freqs, stream, **extra):
        assert isinstance(freqs, np.ndarray) and freqs.ndim == 1 and freqs.dtype == np.float64
        self.calls.append(dict(name=name, freqs=freqs.copy(), stream=stream, **extra))
        return freqs

    def fp_sweep(self, freqs, out=None, stream=0, terms=False):
        f = self._freqs("fp_sweep", freqs, stream, terms=terms)
        return self._fill(out, f.shape, f)

    def fe_sweep(self, freqs, fplus, fcross, out=None, stream=0):
        f = self._freqs("fe_sweep", freqs, stream, S=fplus.shape[0])
        sky = fplus.sum(axis=1) + 10.0 * fcross.sum(axis=1)
        return self._fill(out, (fplus.shape[0], f.shape[0]), sky[:, None] + f[None, :])

    def fe_skymax(self, freqs, fplus, fcross, out=None, index_out=None, stream=0):
        f = self._freqs("fe_skymax", freqs, stream, S=fplus.shape[0])
        S = fplus.shape[0]
        best = self._fill(out, f.shape, f + S)
        idx = self._fill(index_out, f.shape, 7 * np.arange(f.shape[0]) + S, np.int64)
        return best, idx

    def set_residuals(self, residuals, stream=0):
        self.calls.append(dict(name="set_residuals", rows=residuals[0].shape[0], stream=stream))
        self.res = [np.array(r) for r in residuals]
        self.R = self.res[0].shape[0]

    def _tags(self):
        return self.res[0][:, 0]

    def fp_sweep_residuals(self, freqs, out=None, stream=0):
        f = self._freqs("fp_sweep_residuals", freqs, stream)
        return self._fill(out, (self.R, f.shape[0]), self._tags()[:, None] + f[None, :])

    def fe_skymax_residuals(self, freqs, fplus, fcross, out=None, index_out=None, stream=0):
        f = self._freqs("fe_skymax_residuals", freqs, stream, S=fplus.shape[0])
        S, shape = fplus.shape[0], (self.R, f.shape[0])
        best = self._fill(out, shape, self._tags()[:, None] + f[None, :] + S)
        idx = self._fill(index_out, shape, 100 * self._tags()[:, None].astype(np.int64) + np.arange(f.shape[0]) + S,
                         np.int64)
        return best, idx


@pytest.fixture
def stub(monkeypatch):
    """A ``FastFe`` whose pack builder returns a recording stub (``FastFe`` inherits the front ends of ``FastFp``)."""
    built = []

    def build(self, lists):
        built.append(StubPack(self.stub_m))
        return built[-1]

    monkeypatch.setattr(FastFp, "_build_pack", build)
    fe = fastfp_b200.FastFe([_Psr(n, p) for n, p in zip(N, POS)])
    fe.stub_m = [12, 20]
    fe.built = built
    return fe


LISTS = ([np.ones(n) for n in N], [np.ones((n, 2)) for n in N], [np.eye(2) for _ in N])
FGWS = {"scalar": 3e-9, "(F,)": np.array([1e-9, 2e-9, 5e-9, 7e-9]), "(2, 3)": np.arange(1.0, 7.0).reshape(2, 3) * 1e-9}


def _residuals(R):
    """Residuals whose row k carries the tag 10 k in its first entry."""
    res = [np.zeros((R, n)) for n in N]
    res[0][:, 0] = 10.0 * np.arange(R)
    return res


def _sweep_calls(fe, name):
    calls = [c for c in fe.built[-1].calls if c["name"] == name]
    for c in calls:
        assert c["stream"] == 0
    return calls


@pytest.mark.parametrize("fgw", FGWS.values(), ids=FGWS.keys())
def test_calculate_Fp(stub, fgw):
    res = stub.calculate_Fp(fgw, *LISTS)
    f = np.asarray(fgw, dtype=np.float64)
    if f.ndim == 0:
        assert type(res) is np.float64 and res == f
    else:
        assert type(res) is np.ndarray and res.dtype == np.float64 and res.shape == f.shape
        np.testing.assert_array_equal(res, f)
    (call,) = _sweep_calls(stub, "fp_sweep")
    np.testing.assert_array_equal(call["freqs"], f.reshape(-1))
    assert call["terms"] is False


SKIES = {"scalar": (0.3, 1.1), "(S,)": (np.array([0.3, 0.9, 2.0]), np.array([1.1, 4.0, 5.5]))}


@pytest.mark.parametrize("sky", SKIES.values(), ids=SKIES.keys())
@pytest.mark.parametrize("fgw", FGWS.values(), ids=FGWS.keys())
def test_calculate_Fe(stub, fgw, sky):
    res = stub.calculate_Fe(fgw, *sky, *LISTS)
    f = np.asarray(fgw, dtype=np.float64)
    fp, fx = antenna_pattern(POS, *np.broadcast_arrays(np.atleast_1d(sky[0]), np.atleast_1d(sky[1])))
    full = (fp.sum(axis=1) + 10.0 * fx.sum(axis=1))[:, None] + f.reshape(-1)[None, :]  # (S, F)
    want = full if f.ndim else full[:, 0]
    want = want if np.ndim(sky[0]) else want[0]
    if np.ndim(want) == 0:
        assert type(res) is np.float64
    else:
        assert type(res) is np.ndarray and res.dtype == np.float64
    assert np.shape(res) == np.shape(want)  # a (2, 3) fgw is not reshaped: (S, 6) or (6,)
    np.testing.assert_array_equal(res, want)
    (call,) = _sweep_calls(stub, "fe_sweep")
    np.testing.assert_array_equal(call["freqs"], f.reshape(-1))
    assert call["S"] == fp.shape[0]


@pytest.mark.parametrize("sky", SKIES.values(), ids=SKIES.keys())
@pytest.mark.parametrize("fgw", FGWS.values(), ids=FGWS.keys())
def test_calculate_Fe_skymax(stub, fgw, sky):
    best, idx = stub.calculate_Fe_skymax(fgw, *sky, *LISTS)
    f = np.asarray(fgw, dtype=np.float64)
    S = np.size(sky[0])
    if f.ndim == 0:
        assert type(best) is float and type(idx) is int
        assert best == f + S and idx == S
    else:
        assert type(best) is np.ndarray and best.dtype == np.float64 and best.shape == f.shape
        assert type(idx) is np.ndarray and idx.dtype == np.int64 and idx.shape == f.shape
        np.testing.assert_array_equal(best, f + S)
        np.testing.assert_array_equal(idx, (7 * np.arange(f.size) + S).reshape(f.shape))
    (call,) = _sweep_calls(stub, "fe_skymax")
    np.testing.assert_array_equal(call["freqs"], f.reshape(-1))
    assert call["S"] == S


# (basis widths of the stub pack, R): one pass, and 50 realisations in passes of at most 40 rows at m = 600
PLANS = {"one pass": ([12, 20], 6), "passes": ([12, 600], 50)}


def _check_passes(fe, name, m, R, f, calls_before=0):
    rows = batch_pass_rows(R, m)
    want = [min(rows, R - lo) for lo in range(0, R, rows)]
    assert [c["rows"] for c in _sweep_calls(fe, "set_residuals")[calls_before:]] == want
    sweeps = _sweep_calls(fe, name)
    assert len(sweeps) == len(fe.built[-1].calls) - len(_sweep_calls(fe, "set_residuals"))
    for c in sweeps:
        np.testing.assert_array_equal(c["freqs"], f.reshape(-1))
    return len(want)


@pytest.mark.parametrize("plan", PLANS.values(), ids=PLANS.keys())
@pytest.mark.parametrize("fgw", FGWS.values(), ids=FGWS.keys())
def test_calculate_Fp_batch(stub, fgw, plan):
    stub.stub_m, R = plan
    f = np.asarray(fgw, dtype=np.float64)
    res = stub.calculate_Fp_batch(fgw, *LISTS, _residuals(R))
    assert type(res) is np.ndarray and res.dtype == np.float64 and res.shape == (R,) + f.shape
    want = 10.0 * np.arange(R).reshape((R,) + (1,) * f.ndim) + f
    np.testing.assert_array_equal(res, want)
    npass = _check_passes(stub, "fp_sweep_residuals", stub.stub_m, R, f)
    assert len(_sweep_calls(stub, "fp_sweep_residuals")) == npass
    again = stub.calculate_Fp_batch(fgw, *LISTS, _residuals(R))
    np.testing.assert_array_equal(again, want)
    assert len(stub.built) == 1
    if npass == 1:  # the pack still holds the set: it is not uploaded again
        assert len(_sweep_calls(stub, "set_residuals")) == 1
    else:           # it holds the last pass only: every pass is uploaded again
        _check_passes(stub, "fp_sweep_residuals", stub.stub_m, R, f, calls_before=npass)
    assert len(_sweep_calls(stub, "fp_sweep_residuals")) == 2 * npass


@pytest.mark.parametrize("sky", SKIES.values(), ids=SKIES.keys())
@pytest.mark.parametrize("plan", PLANS.values(), ids=PLANS.keys())
@pytest.mark.parametrize("fgw", FGWS.values(), ids=FGWS.keys())
def test_calculate_Fe_skymax_batch(stub, fgw, plan, sky):
    stub.stub_m, R = plan
    f = np.asarray(fgw, dtype=np.float64)
    S = np.size(sky[0])
    best, idx = stub.calculate_Fe_skymax_batch(fgw, *sky, *LISTS, _residuals(R))
    assert type(best) is np.ndarray and best.dtype == np.float64 and best.shape == (R,) + f.shape
    assert type(idx) is np.ndarray and idx.dtype == np.int64 and idx.shape == (R,) + f.shape
    tag = np.arange(R).reshape((R,) + (1,) * f.ndim)
    np.testing.assert_array_equal(best, 10.0 * tag + f + S)
    np.testing.assert_array_equal(idx, 1000 * tag + np.arange(f.size).reshape(f.shape) + S)
    npass = _check_passes(stub, "fe_skymax_residuals", stub.stub_m, R, f)
    assert [c["S"] for c in _sweep_calls(stub, "fe_skymax_residuals")] == [S] * npass
    stub.calculate_Fe_skymax_batch(fgw, *sky, *LISTS, _residuals(R))
    assert len(_sweep_calls(stub, "set_residuals")) == (1 if npass == 1 else 2 * npass)
    assert len(_sweep_calls(stub, "fe_skymax_residuals")) == 2 * npass
