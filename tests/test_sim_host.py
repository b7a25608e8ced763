"""The host reference of the device-drawn residual batches (fastfp_b200/sim.py) and the argument checks of
``calculate_Fp_simulated`` / ``calculate_Fe_skymax_simulated`` (CPU): the Philox stream against NumPy's, the normals,
the independence of a realisation from the batch that drew it, and ``FastFe.cw_signal``."""
import numpy as np
import pytest

import fastfp_b200
from fastfp_b200 import blockn, sim, synth
from fastfp_b200.fe import antenna_pattern


@pytest.mark.parametrize("seed", [0, 1, 987654321, 2 ** 63 - 1])
def test_philox_matches_numpy_word_for_word(seed):
    rng = np.random.default_rng(seed % 1000)
    for q, k, p, tag in [(1, 0, 0, 0), (2, 5, 3, 2), (1 << 40, 1 << 33, 67, 1)] + \
            [tuple(int(v) for v in rng.integers(1, 2 ** 62, size=4)) for _ in range(5)]:
        want = np.random.Philox(key=[seed, 0], counter=[q - 1, k, p, tag]).random_raw(4)
        got = sim.philox4x64((q, k, p, tag), (seed, 0))
        assert [int(w) for w in got] == [int(w) for w in want], (seed, q, k, p, tag)
    # vectorised over counters: the same words as one at a time
    q = np.arange(1, 9, dtype=np.uint64)
    words = sim.philox4x64((q, 7, 2, 1), (seed, 0))
    for i, qi in enumerate(q):
        want = np.random.Philox(key=[seed, 0], counter=[int(qi) - 1, 7, 2, 1]).random_raw(4)
        assert [int(w[i]) for w in words] == [int(w) for w in want]


def test_normals_have_no_zero_uniform_and_sensible_moments():
    # no word maps to 0, so ln u0 is finite; the largest rounds to exactly 1 (2^53 - 0.5 is not a double), where
    # Box-Muller gives a finite 0
    u = [((np.uint64(x) >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0 ** -53 for x in (0, 2 ** 11, 2 ** 64 - 1)]
    assert u == [2.0 ** -54, 1.5 * 2.0 ** -53, 1.0]
    N = 1 << 20
    z = sim.normals(12345, np.uint64(0), 0, 0, np.arange(N))
    assert np.all(np.isfinite(z))
    se = 1.0 / np.sqrt(N)
    assert abs(z.mean()) < 5 * se
    assert abs(z.var() - 1.0) < 5 * np.sqrt(2.0) * se
    assert abs(np.mean(z ** 3)) < 5 * np.sqrt(15.0) * se
    assert abs(np.mean(z ** 4) - 3.0) < 5 * np.sqrt(96.0) * se
    # the two normals of each Box-Muller pair are uncorrelated, and so are neighbouring counter blocks
    assert abs(np.mean(z[0::2] * z[1::2])) < 5 * np.sqrt(2.0) * se
    assert abs(np.mean(z[:-4] * z[4:])) < 5 * se
    # other tags, pulsars, realisations and seeds are other streams
    for args in ((12345, 1, 0, 0), (12345, 0, 1, 0), (12345, 0, 0, 1), (12346, 0, 0, 0)):
        w = sim.normals(args[0], np.uint64(args[1]), args[2], args[3], np.arange(4096))
        assert abs(np.corrcoef(w, z[:4096])[0, 1]) < 0.1


def _pta_and_noise():
    pta = synth.make_pta(3, [40, 57, 33], n_tm=4, ncomps=3, epoch=4, seed=7)
    Nvecs, Ts, TNTs, phis = synth.with_ecorr(pta, kernel=True)
    return pta, Nvecs, Ts, [1.0 / phi for phi in phis]


def test_a_realisation_does_not_depend_on_the_batch_that_drew_it():
    pta, Nvecs, Ts, phiinvs = _pta_and_noise()
    assert any(blockn.is_block(N) for N in Nvecs)
    rng = np.random.default_rng(0)
    freqs8, amp8 = rng.uniform(1e-8, 1e-7, 8), rng.normal(size=(8, 3, 2)) * 1e-7
    for Nv in (Nvecs, pta.Nvecs):  # kernel ECORR and diagonal N
        a = sim.simulate_residuals(pta.toas, Nv, Ts, phiinvs, 8, seed=99, signal=(freqs8, amp8))
        b = sim.simulate_residuals(pta.toas, Nv, Ts, phiinvs, 3, seed=99, first=5, signal=(freqs8[5:], amp8[5:]))
        for p in range(3):
            np.testing.assert_array_equal(a[p][5:], b[p])
        c = sim.simulate_residuals(pta.toas, Nv, Ts, phiinvs, 3, seed=100, first=5)
        assert not np.array_equal(b[0], c[0])


def test_the_parts_of_a_realisation():
    pta, Nvecs, Ts, phiinvs = _pta_and_noise()
    R, seed = 4, 3
    k = np.arange(R, dtype=np.uint64)[:, None]
    sig = (2e-8, np.full((3, 2), 1e-7))
    only = sim.simulate_residuals(pta.toas, Nvecs, Ts, phiinvs, R, seed, signal=sig, noise=False)
    full = sim.simulate_residuals(pta.toas, Nvecs, Ts, phiinvs, R, seed, signal=sig)
    plain = sim.simulate_residuals(pta.toas, Nvecs, Ts, phiinvs, R, seed)
    for p in range(3):
        t = pta.toas[p]
        ph = (sim.TWO_PI * 2e-8) * t
        np.testing.assert_array_equal(only[p], np.broadcast_to(1e-7 * np.sin(ph) + 1e-7 * np.cos(ph), (R, t.size)))
        np.testing.assert_allclose(full[p], plain[p] + only[p], rtol=0, atol=1e-20)
        ep = blockn.epochs(Nvecs[p], t.size)
        white = np.sqrt(ep.nvec) * sim.normals(seed, k, p, 0, np.arange(t.size)[None, :])
        eta = np.sqrt(ep.jvec) * sim.normals(seed, k, p, 1, np.arange(len(ep.slices))[None, :])
        cols = np.nonzero(phiinvs[p] > 1e-30)[0]
        assert cols.size == Ts[p].shape[1] - pta.n_tm[p]  # the timing-model columns are not drawn explicitly
        basis = (sim.normals(seed, k, p, 2, cols[None, :]) / np.sqrt(phiinvs[p][cols])) @ Ts[p][:, cols].T
        ecorr = np.zeros_like(white)
        for e, (a, b) in enumerate(ep.slices):
            ecorr[:, a:b] = eta[:, e:e + 1]
        np.testing.assert_allclose(plain[p], white + ecorr + basis, rtol=1e-12, atol=1e-22)


def _fe_psrs():
    return synth.make_pta(4, 30, n_tm=3, ncomps=2, seed=8).psrs


def test_cw_signal_is_the_fe_template():
    psrs = _fe_psrs()
    fe = fastfp_b200.FastFe(psrs)
    th, ph = 1.1, 4.2
    fplus, fcross = antenna_pattern(fe.pos, th, ph)
    a = np.array([1.0, -2.0, 0.5, 3.0]) * 1e-7
    f, amp = fe.cw_signal(3e-8, th, ph, a)
    assert float(f) == 3e-8 and amp.shape == (4, 2)
    np.testing.assert_array_equal(amp[:, 0], a[0] * fplus + a[2] * fcross)
    np.testing.assert_array_equal(amp[:, 1], a[1] * fplus + a[3] * fcross)
    # the injected residuals are the Fe templates [F+ s, F+ c, Fx s, Fx c] weighted by a
    res = sim.simulate_residuals([q.toas for q in psrs], [np.ones(30)] * 4, [np.ones((30, 1))] * 4, [np.ones(1)] * 4,
                                 1, 0, signal=(f, amp), noise=False)
    for p, q in enumerate(psrs):
        s, c = np.sin((sim.TWO_PI * 3e-8) * q.toas), np.cos((sim.TWO_PI * 3e-8) * q.toas)
        tmpl = np.stack((fplus[p] * s, fplus[p] * c, fcross[p] * s, fcross[p] * c))
        np.testing.assert_allclose(res[p][0], a @ tmpl, rtol=1e-13, atol=1e-22)
    # one amplitude set per realisation
    aR = np.stack((a, 2 * a, -a))
    fR, ampR = fe.cw_signal(np.array([1e-8, 2e-8, 3e-8]), th, ph, aR)
    assert ampR.shape == (3, 4, 2)
    np.testing.assert_array_equal(ampR[1], fe.cw_signal(2e-8, th, ph, 2 * a)[1])
    with pytest.raises(ValueError, match="shape"):
        fe.cw_signal(3e-8, th, ph, np.ones(3))
    with pytest.raises(ValueError, match="one sky position"):
        fe.cw_signal(3e-8, [th, th], [ph, ph], a)


def _bad_calls():
    pta = synth.make_pta(2, [30, 41], n_tm=3, ncomps=2, seed=9)
    phi = [1.0 / p for p in pta.phis]
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    nan = [phi[0].copy(), phi[1]]
    nan[0][4] = np.nan
    neg = [phi[0], -phi[1]]
    return pta, phi, [
        (dict(phiinvs=phi, R=0, seed=1), "R must be"),
        (dict(phiinvs=phi, R=2.5, seed=1), "R must be"),
        (dict(phiinvs=phi, R=4, seed=-1), "seed"),
        (dict(phiinvs=phi, R=4, seed=1.0), "seed"),
        (dict(phiinvs=phi, R=4, seed=1, first=-3), "first"),
        (dict(phiinvs=phi, R=4, seed=1, first=2 ** 63 - 2), "first"),
        (dict(phiinvs=nan, R=4, seed=1), r"phiinvs\[0\] must be finite"),
        (dict(phiinvs=neg, R=4, seed=1), r"phiinvs\[1\] must be finite and >= 0"),
        (dict(phiinvs=phi[:1], R=4, seed=1), "list of 2"),
        (dict(phiinvs=[phi[0], phi[1][:-1]], R=4, seed=1), r"phiinvs\[1\] must have shape"),
        (dict(phiinvs=phi, R=4, seed=1, signal=(np.ones(3), np.ones((2, 2)))), "signal frequencies"),
        (dict(phiinvs=phi, R=4, seed=1, signal=(1e-8, np.ones((4, 3, 2)))), "signal amplitudes"),
        (dict(phiinvs=phi, R=4, seed=1, signal=1e-8), "pair"),
    ], a


def test_argument_errors_are_raised_before_any_device_work():
    pta, phi, cases, a = _bad_calls()
    fp = fastfp_b200.FastFp(pta.psrs)
    fe = fastfp_b200.FastFe(pta.psrs)
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            fp.calculate_Fp_simulated(np.array([1e-8]), *a, **kw)
        with pytest.raises(ValueError, match=msg):
            fe.calculate_Fe_skymax_simulated(np.array([1e-8]), 0.3, 1.0, *a, **kw)
    assert fp._pack is None and fe._pack is None  # nothing was built
    with pytest.raises(ValueError, match="seed"):
        sim.simulate_residuals(pta.toas, pta.Nvecs, pta.Ts, phi, 2, seed=-4)
