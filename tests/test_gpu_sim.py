"""Residual batches drawn on the device (``calculate_Fp_simulated``, ``calculate_Fe_skymax_simulated``,
``fastfp_pack_simulate_residuals*``) on the GPU, all with fixed seeds:

* route equivalence: every row against the longdouble truth of the explicit realisations of fastfp_b200/sim.py, which
  pins the device's random stream and the Woodbury identity it sweeps through, for a diagonal N, GP-basis ECORR and
  kernel ECORR, with a signal injected;
* the null distribution: 2 Fp ~ chi^2_2P and 2 Fe ~ chi^2_4 at one sky position under each noise model;
* injections: the noiseless statistic is 1/2 a^T M a, and with noise 2 Fe is non-central chi^2_4;
* the exact properties, the pass split, the refusals and the memory a simulated set holds."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
from scipy import stats

import fastfp_b200
from fastfp_b200 import _cabi, sim, synth
from fastfp_b200.fe import antenna_pattern
from oracle import truth
from test_gpu_blockn_batch import _assert_rows
from test_gpu_fe_skymax_batch import _assert_skymax_near, _row_truth
from test_gpu_fp_batch import assert_rows_near_truth

pytestmark = pytest.mark.gpu


def _model(pta, kind):
    """``(Nvecs, Ts, sigmas, phiinvs, tblocks)`` of noise model ``kind`` on ``pta`` (made with ``epoch > 1`` for the
    ECORR kinds): "diag", "gp_ecorr" (epoch-indicator basis columns, diagonal N) or "kernel_ecorr" (block N)."""
    if kind == "diag":
        Nvecs, Ts, TNTs, phis = pta.Nvecs, pta.Ts, pta.TNTs, pta.phis
    else:
        Nvecs, Ts, TNTs, phis = synth.with_ecorr(pta, kernel=kind == "kernel_ecorr")
    sig = [TNT + np.diag(1.0 / phi) for TNT, phi in zip(TNTs, phis)]
    tblocks = None
    if kind == "kernel_ecorr":
        tblocks = [(B.nvec, [(s.start, s.stop) for s in B.slices], B.jvec) for B in Nvecs]
    return Nvecs, Ts, sig, [1.0 / phi for phi in phis], tblocks


def _ragged(seed):
    pta = synth.make_pta(3, [300, 411, 257], n_tm=[12, 8, 5], ncomps=10, epoch=4, seed=seed)
    freqs = np.concatenate((synth.fp_freqs(40), np.array([1.0, 2.5, 7.0]) / pta.Tspan))
    return pta, freqs


def _signal(R, P, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(1e-8, 1e-7, R), rng.normal(size=(R, P, 2)) * 3e-7


@pytest.mark.parametrize("kind", ["diag", "gp_ecorr", "kernel_ecorr"])
def test_every_row_meets_the_truth_of_the_host_realisations(kind):
    pta, freqs = _ragged(seed=71)
    Nvecs, Ts, sig, phiinvs, tblocks = _model(pta, kind)
    R, seed = 12, 2024
    signal = _signal(R, pta.P, seed=5)
    fp = fastfp_b200.FastFp(pta.psrs)
    got = fp.calculate_Fp_simulated(freqs, Nvecs, Ts, sig, phiinvs, R, seed, signal=signal)
    assert got.shape == (R, freqs.shape[0]) and np.all(np.isfinite(got))
    res = sim.simulate_residuals(pta.toas, Nvecs, Ts, phiinvs, R, seed, signal=signal)
    if tblocks is None:
        assert_rows_near_truth(got, range(R), SimpleNamespace(toas=pta.toas, Nvecs=Nvecs, Ts=Ts, sigmas=sig), res, freqs)
    else:
        _assert_rows(got, range(R), freqs, pta, res, tblocks, sig, f"{kind}, simulated")


@pytest.mark.parametrize("kind", ["diag", "kernel_ecorr"])
def test_fe_skymax_rows_meet_the_truth(kind):
    pta, freqs = _ragged(seed=72)
    Nvecs, Ts, sig, phiinvs, tblocks = _model(pta, kind)
    pos = np.stack([q.pos for q in pta.psrs])
    rng = np.random.default_rng(3)
    th, ph = np.arccos(rng.uniform(-1, 1, 24)), rng.uniform(0, 2 * np.pi, 24)
    fplus, fcross = antenna_pattern(pos, th, ph)
    R, seed = 6, 77
    signal = _signal(R, pta.P, seed=6)
    fe = fastfp_b200.FastFe(pta.psrs)
    best, idx = fe.calculate_Fe_skymax_simulated(freqs, th, ph, Nvecs, Ts, sig, phiinvs, R, seed, signal=signal)
    assert best.shape == idx.shape == (R, freqs.shape[0])
    res = sim.simulate_residuals(pta.toas, Nvecs, Ts, phiinvs, R, seed, signal=signal)
    ns = SimpleNamespace(toas=pta.toas, Nvecs=Nvecs, Ts=Ts, sigmas=sig)
    for k in range(R):
        if tblocks is None:
            fet, cond, E = _row_truth(freqs, ns, [r[k] for r in res], fplus, fcross)
            _assert_skymax_near(best[k], idx[k], fet, cond, E, f"row {k}", rel=1e-9)
        else:  # test_gpu_blockn_batch.py::test_fe_skymax_batch's bar
            fet, cond = truth.fe_truth(freqs, fplus, fcross, pta.toas, [r[k] for r in res], None, Ts, sig,
                                       blocks=tblocks)
            fet = fet.astype(float)
            tol = 1e-9 * np.abs(fet) + 1024 * np.finfo(float).eps * cond
            defined = _defined(fet, cond)
            cols = np.arange(freqs.shape[0])
            at = (idx[k], cols)
            assert np.all(np.where(defined[at], np.abs(best[k] - fet[at]) <= tol[at], True)), k
            am = np.nanargmax(fet, axis=0)
            srt = np.sort(np.where(np.isnan(fet), -np.inf, fet), axis=0)
            clear = defined[am, cols] & (srt[-1] - srt[-2] > tol[am, cols] + tol[idx[k], cols])
            assert np.all(np.where(clear, idx[k] == am, True)), k


def _defined(tv, cond):
    """bins where the reference formula carries digits at all"""
    return np.finfo(float).eps * cond < 0.05 * np.abs(tv)


def _null_pta():
    pta = synth.make_pta(6, [300, 411, 257, 350, 280, 330], n_tm=[6, 8, 5, 7, 6, 8], ncomps=10, epoch=4, seed=81)
    # a dozen frequencies half-way between the red-noise bins k / Tspan, away from 1/yr (~15 / Tspan) and 2/yr
    freqs = (np.arange(16, 28) + 0.5) / pta.Tspan
    yr = 365.25 * 86400.0
    assert np.all(np.abs(freqs - 1 / yr) > 0.4 / pta.Tspan) and np.all(np.abs(freqs - 2 / yr) > 0.4 / pta.Tspan)
    return pta, freqs


@pytest.mark.parametrize("kind", ["diag", "gp_ecorr", "kernel_ecorr"])
def test_null_distribution(kind):
    pta, freqs = _null_pta()
    Nvecs, Ts, sig, phiinvs, _ = _model(pta, kind)
    P, R = pta.P, 512
    fp = fastfp_b200.FastFp(pta.psrs)
    got = fp.calculate_Fp_simulated(freqs, Nvecs, Ts, sig, phiinvs, R, seed=1000 + len(kind))
    assert got.shape == (R, freqs.shape[0])
    for f in range(freqs.shape[0]):
        pv = stats.kstest(2 * got[:, f], "chi2", args=(2 * P,)).pvalue
        assert pv >= 1e-4, (kind, f, pv)
        assert abs(got[:, f].mean() - P) <= 4 * np.sqrt(P / R), (kind, f, got[:, f].mean())
    fe = fastfp_b200.FastFe(pta.psrs)
    best, idx = fe.calculate_Fe_skymax_simulated(freqs, 1.1, 2.3, Nvecs, Ts, sig, phiinvs, R, seed=2000 + len(kind))
    assert np.all(idx == 0)
    for f in range(freqs.shape[0]):
        pv = stats.kstest(2 * best[:, f], "chi2", args=(4,)).pvalue
        assert pv >= 1e-4, (kind, "Fe", f, pv)


def test_injection():
    pta, freqs = _null_pta()
    Nvecs, Ts, sig, phiinvs, _ = _model(pta, "diag")
    f0, th0, ph0 = float(freqs[5]), 0.9, 4.0
    fe = fastfp_b200.FastFe(pta.psrs)
    inner = truth.sweep_inner_truth(np.array([f0]), pta.toas, pta.residuals, Nvecs, Ts, sig)
    Mp = np.stack([[inner["Mss"][:, 0], inner["Msc"][:, 0]], [inner["Msc"][:, 0], inner["Mcc"][:, 0]]]).astype(float)
    fplus, fcross = antenna_pattern(fe.pos, th0, ph0)
    M = np.zeros((4, 4))
    for p in range(pta.P):
        w = np.array([[fplus[p] ** 2, fplus[p] * fcross[p]], [fplus[p] * fcross[p], fcross[p] ** 2]])
        M += np.kron(w, Mp[:, :, p])
    a = np.array([1.0, -2.0, 0.5, 3.0])
    a *= np.sqrt(20.0 / (a @ M @ a))  # non-centrality a^T M a = 20
    lam = a @ M @ a
    signal = fe.cw_signal(f0, th0, ph0, a)
    # noiseless: Fe at the injected position is 1/2 a^T M a, Fp the sum of 1/2 x_p^T M_p x_p
    best, idx = fe.calculate_Fe_skymax_simulated(f0, th0, ph0, Nvecs, Ts, sig, phiinvs, 3, seed=5, signal=signal,
                                                 noise=False)
    assert np.all(idx == 0)
    np.testing.assert_allclose(best, 0.5 * lam, rtol=1e-9)
    fp_want = sum(0.5 * signal[1][p] @ Mp[:, :, p] @ signal[1][p] for p in range(pta.P))
    got = fe.calculate_Fp_simulated(f0, Nvecs, Ts, sig, phiinvs, 3, seed=5, signal=signal, noise=False)
    np.testing.assert_allclose(got, fp_want, rtol=1e-9)
    # with noise: 2 Fe ~ non-central chi^2_4 with non-centrality a^T M a
    R = 512
    best, idx = fe.calculate_Fe_skymax_simulated(f0, th0, ph0, Nvecs, Ts, sig, phiinvs, R, seed=6, signal=signal)
    pv = stats.kstest(2 * best, stats.ncx2(4, lam).cdf).pvalue
    assert pv >= 1e-4, pv


def _small(seed=91):
    pta = synth.make_pta(3, [300, 411, 257], n_tm=[12, 8, 5], ncomps=10, seed=seed)
    freqs = np.concatenate((synth.fp_freqs(40), np.array([1.0, 2.5, 7.0]) / pta.Tspan))
    return pta, freqs, (pta.Nvecs, pta.Ts, pta.sigmas), [1.0 / phi for phi in pta.phis]


def test_exact_properties():
    pta, freqs, a, phi = _small()
    fp = fastfp_b200.FastFp(pta.psrs)
    amp = np.random.default_rng(1).normal(size=(pta.P, 2)) * 3e-7
    sig = (3e-8, amp)
    base = fp.calculate_Fp_simulated(freqs, *a, phi, 8, seed=11, signal=sig)
    assert np.all(np.isfinite(base))
    # repeatable, on the cached set and after drawing it again
    np.testing.assert_array_equal(fp.calculate_Fp_simulated(freqs, *a, phi, 8, seed=11, signal=sig), base)
    fp._res_key = None
    np.testing.assert_array_equal(fp.calculate_Fp_simulated(freqs, *a, phi, 8, seed=11, signal=sig), base)
    # first shifts the rows bit for bit at equal R; another seed is another draw
    shifted = fp.calculate_Fp_simulated(freqs, *a, phi, 8, seed=11, first=5, signal=sig)
    np.testing.assert_array_equal(shifted[:3], base[5:])
    assert not np.array_equal(fp.calculate_Fp_simulated(freqs, *a, phi, 8, seed=12, signal=sig)[0], base[0])
    # an uploaded set and a simulated set of the same pack never share the cache: the simulated set is drawn again
    res = sim.simulate_residuals(pta.toas, pta.Nvecs, pta.Ts, phi, 8, seed=11, signal=sig)
    up = fp.calculate_Fp_batch(freqs, *a, res)
    assert not np.array_equal(up, base)
    np.testing.assert_array_equal(fp.calculate_Fp_simulated(freqs, *a, phi, 8, seed=11, signal=sig), base)
    # noiseless: doubling the amplitudes gives exactly 4x; no signal gives exactly 0
    one = fp.calculate_Fp_simulated(freqs, *a, phi, 8, seed=11, signal=sig, noise=False)
    two = fp.calculate_Fp_simulated(freqs, *a, phi, 8, seed=11, signal=(3e-8, 2 * amp), noise=False)
    assert np.all(one > 0)
    np.testing.assert_array_equal(two, 4 * one)
    zero = fp.calculate_Fp_simulated(freqs, *a, phi, 8, seed=11, noise=False)
    assert np.all(zero == 0.0)
    # a NaN in one realisation's signal makes only that row NaN
    f8, amp8 = np.full(8, 3e-8), np.broadcast_to(amp, (8, pta.P, 2)).copy()
    amp8[6, 1, 0] = np.nan
    bad = fp.calculate_Fp_simulated(freqs, *a, phi, 8, seed=11, signal=(f8, amp8))
    assert np.all(np.isnan(bad[6]))
    np.testing.assert_array_equal(np.delete(bad, 6, 0), np.delete(base, 6, 0))
    f8[2] = np.nan
    amp8[6, 1, 0] = amp[1, 0]
    bad = fp.calculate_Fp_simulated(freqs, *a, phi, 8, seed=11, signal=(f8, amp8))
    assert np.all(np.isnan(bad[2]))
    np.testing.assert_array_equal(np.delete(bad, 2, 0), np.delete(base, 2, 0))
    # the Fe sky maximum is repeatable and shifts with first alike
    fe = fastfp_b200.FastFe(pta.psrs)
    b0, i0 = fe.calculate_Fe_skymax_simulated(freqs, [0.3, 1.2], [1.0, 5.0], *a, phi, 8, seed=11, signal=sig)
    b1, i1 = fe.calculate_Fe_skymax_simulated(freqs, [0.3, 1.2], [1.0, 5.0], *a, phi, 8, seed=11, first=5, signal=sig)
    np.testing.assert_array_equal(b1[:3], b0[5:])
    np.testing.assert_array_equal(i1[:3], i0[5:])


@pytest.mark.parametrize("kind", ["diag", "kernel_ecorr"])
def test_more_rows_than_one_pass(kind):
    pta = synth.make_pta(2, [300, 257], n_tm=12, ncomps=30, epoch=4, seed=92)
    Nvecs, Ts, sig, phi, tblocks = _model(pta, kind)
    freqs = synth.fp_freqs(20)
    blockn = kind == "kernel_ecorr"
    rmax = _cabi.max_residual_rows([72, 72], blockn)
    R = rmax + 1
    fp = fastfp_b200.FastFp(pta.psrs)
    got = fp.calculate_Fp_simulated(freqs, Nvecs, Ts, sig, phi, R, seed=3)
    assert got.shape == (R, 20) and np.all(np.isfinite(got))
    rows = [0, rmax // 2, R - 1]
    res = sim.simulate_residuals(pta.toas, Nvecs, Ts, phi, R, seed=3)
    if tblocks is None:
        assert_rows_near_truth(got, rows, SimpleNamespace(toas=pta.toas, Nvecs=Nvecs, Ts=Ts, sigmas=sig), res, freqs,
                               well_conditioned=False)
    else:
        _assert_rows(got, rows, freqs, pta, res, tblocks, sig, "split R", well=False)
    # the library refuses a single set above the limit
    pack = fp.prepare(Nvecs, Ts, sig)
    call = pack.simulate_residuals_blockn if blockn else pack.simulate_residuals
    with pytest.raises(_cabi.FastFpError, match=rf"error -3: .*limit of {rmax} "):
        call(R, 3, phi)


def test_cuda_tensor_on_a_non_default_stream():
    import torch

    pta, freqs, a, phi = _small(seed=93)
    sig = (3e-8, np.ones((pta.P, 2)) * 1e-7)
    want = fastfp_b200.FastFp(pta.psrs).calculate_Fp_simulated(freqs[:40], *a, phi, 10, seed=4, signal=sig)
    fp = fastfp_b200.FastFp(pta.psrs)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        f = torch.tensor(freqs[:40].reshape(5, 8), dtype=torch.float64, device="cuda")
        got = fp.calculate_Fp_simulated(f, *a, phi, 10, seed=4, signal=sig)
    s.synchronize()
    assert got.is_cuda and got.shape == (10, 5, 8)
    np.testing.assert_array_equal(got.cpu().numpy().reshape(10, 40), want)


def test_refusals_and_memory():
    lib = _cabi.load()
    pta, freqs, a, phi = _small(seed=94)
    pack = fastfp_b200.FastFp(pta.psrs).prepare(*a)
    phis = _cabi._ptr_array([_cabi.as_f64(p) for p in phi])
    # bad priors, seeds, flags and half a signal, at the library
    for bad in (np.nan, -1.0, np.inf):
        worse = [p.copy() for p in phi]
        worse[2][3] = bad
        assert lib.fastfp_pack_simulate_residuals(pack._h, 4, 1, 0, _cabi._ptr_array(worse), None, None, 0, None) == -1
        assert "must be finite and >= 0" in lib.fastfp_last_error().decode()
    freq = np.ones(4)
    for args in ((4, -1, 0, phis, None, None, 0), (4, 1, -2, phis, None, None, 0), (4, 1, 0, phis, None, None, 2),
                 (4, 1, 0, phis, C.c_void_p(freq.ctypes.data), None, 0)):
        assert lib.fastfp_pack_simulate_residuals(pack._h, *args, None) == -1
    # memory: the same packets as an uploaded set of the same R, and the staging is freed
    base, dev0 = pack.nbytes, _cabi.device_bytes()
    res = sim.simulate_residuals(pta.toas, pta.Nvecs, pta.Ts, phi, 40, seed=1)
    pack.set_residuals(res)
    up_bytes, up_dev = pack.nbytes, _cabi.device_bytes()
    pack.simulate_residuals(40, 1, phi)
    assert pack.nbytes == up_bytes > base and pack.R == 40
    assert _cabi.device_bytes() == up_dev
    pack.simulate_residuals(0, 1, phi)  # R = 0 releases the set
    assert pack.nbytes == base and _cabi.device_bytes() == dev0
    # nmfp pack
    nm = _cabi.Pack.create(pta.toas, pta.residuals, pta.Nvecs, pta.Ts, pta.TNTs, m_fix=pta.n_tm,
                           phiinv_fix=[p[:k] ** -1 for p, k in zip(pta.phis, pta.n_tm)])
    assert lib.fastfp_pack_simulate_residuals(nm._h, 4, 1, 0, phis, None, None, 0, None) == -1
    # the wrong pack kind, both ways
    ep = synth.make_pta(2, 96, n_tm=4, ncomps=5, epoch=4, seed=95)
    Nvecs, Ts, sig, ephi, _ = _model(ep, "kernel_ecorr")
    bpack = fastfp_b200.FastFp(ep.psrs).prepare(Nvecs, Ts, sig)
    assert bpack.blockn
    ephis = _cabi._ptr_array([_cabi.as_f64(p) for p in ephi])
    assert lib.fastfp_pack_simulate_residuals(bpack._h, 2, 1, 0, ephis, None, None, 0, None) == -3
    with pytest.raises(_cabi.FastFpError, match="diagonal-N"):
        bpack.simulate_residuals(2, 1, ephi)
    with pytest.raises(_cabi.FastFpError, match="block-diagonal N pack"):
        pack.simulate_residuals_blockn(2, 1, phi)
    # block-N memory: as an uploaded set of the same R
    bbase, bdev0 = bpack.nbytes, _cabi.device_bytes()
    bpack.set_residuals_blockn(sim.simulate_residuals(ep.toas, Nvecs, Ts, ephi, 24, seed=2))
    bup, bdev = bpack.nbytes, _cabi.device_bytes()
    bpack.simulate_residuals_blockn(24, 2, ephi)
    assert bpack.nbytes == bup > bbase and _cabi.device_bytes() == bdev
    bpack.simulate_residuals_blockn(0, 2, ephi)
    assert bpack.nbytes == bbase and _cabi.device_bytes() == bdev0
