"""The extended-precision Fe-statistic truth (oracle/truth.fe_truth) against the float64 Fe oracle, the Fp truth and
the GP-basis form of a block-diagonal N (CPU). tests/test_gpu_fe_truth.py measures the CUDA Fe paths against it."""
import numpy as np

from conftest import EPS
from fastfp_b200 import synth
from fastfp_b200.fe import antenna_pattern
from oracle import fe_oracle
from oracle import fp_oracle as o
from oracle import truth

EPS_LD = float(np.finfo(np.longdouble).eps)


def _sky(pos):
    """Two random positions, the north pole, and one 0.03 rad from pulsar 0, where both the numerators and the
    denominator 1 + Omega.p of its antenna patterns are small."""
    th0, ph0 = np.arccos(pos[0, 2]), np.arctan2(pos[0, 1], pos[0, 0]) % (2 * np.pi)
    th, ph = np.array([0.3, 1.2, 0.0, th0 + 0.03]), np.array([0.1, 3.0, 0.0, ph0])
    om = -np.stack((np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)), axis=-1)
    assert 1 + om[3] @ pos[0] < 1e-3
    return th, ph


def test_float64_oracle_within_the_conditioning_envelope():
    """fe_oracle (float64, the published statistic on the reference's get_xCy) lies within 4 E eps cond of the truth,
    E >= 1 the float64 Fp oracle's own worst distance from the Fp truth in units of eps cond (the calibration of
    conftest.term_tolerance). In the red-noise bins its error is a visible fraction of that envelope."""
    pta = synth.make_pta(3, [300, 257, 411], n_tm=[6, 8, 5], ncomps=10, seed=12)
    freqs = np.concatenate((synth.fp_freqs(40)[8::8], np.array([1.0, 2.5, 7.0]) / pta.Tspan))
    pos = np.stack([q.pos for q in pta.psrs])
    th, ph = _sky(pos)
    fp, fx = antenna_pattern(pos, th, ph)
    args = (pta.toas, pta.residuals, pta.Nvecs, pta.Ts, pta.sigmas)
    fe, cond = truth.fe_truth(freqs, fp, fx, *args)
    fe = fe.astype(float)
    want = np.array([[fe_oracle.calculate_Fe(f, t, p_, pta.toas, pta.residuals, pos, *args[2:]) for f in freqs]
                     for t, p_ in zip(th, ph)])
    tt, tc = truth.fp_sweep_truth(freqs, *args)
    E = max(1.0, (np.abs(o.fp_sweep(freqs, *args, per_pulsar=True) - tt.astype(float)) / (EPS * tc)).max())
    defined = EPS * cond < 0.05 * np.abs(fe)
    assert defined.mean() > 0.9
    ratio = np.where(defined, np.abs(want - fe) / (4 * E * EPS * cond), 0.0)
    assert ratio.max() <= 1, (ratio.max(), E)
    red = freqs < 10.0 / pta.Tspan
    assert ratio[:, red].max() > 1e-2, ratio  # the envelope is not vacuous


def test_a_pair_of_pure_patterns_is_the_sum_of_two_fp_terms():
    """Pulsar i at (F+, Fx) = (1, 0), pulsar j at (0, 1), every other pulsar at (0, 0): M is block diagonal and Fe is
    the Fp term of i plus the Fp term of j."""
    pta = synth.make_pta(4, [200, 257, 180, 233], n_tm=[5, 7, 6, 4], ncomps=8, seed=21)
    freqs = np.concatenate((synth.fp_freqs(30)[::6], np.array([1.0, 2.5]) / pta.Tspan))
    args = (pta.toas, pta.residuals, pta.Nvecs, pta.Ts, pta.sigmas)
    pairs = [(i, j) for i in range(4) for j in range(4) if i != j]
    fp, fx = np.zeros((len(pairs), 4)), np.zeros((len(pairs), 4))
    for k, (i, j) in enumerate(pairs):
        fp[k, i], fx[k, j] = 1.0, 1.0
    fe, cond = truth.fe_truth(freqs, fp, fx, *args)
    tt, tc = truth.fp_sweep_truth(freqs, *args)
    for k, (i, j) in enumerate(pairs):
        want = tt[i] + tt[j]
        assert np.all(np.abs((fe[k] - want).astype(float)) <= 64 * EPS_LD * (tc[i] + tc[j])), (i, j)
        np.testing.assert_allclose(cond[k], tc[i] + tc[j], rtol=1e-12)


def test_block_n_fe_truth_equals_the_gp_basis_truth():
    """With ``blocks`` the truth applies N^-1 by Sherman-Morrison; on the widened GP basis [T | U] (epoch-indicator
    columns U, diagonal N, Sigma extended by 1/jvec) the plain truth evaluates the same Fe, as in
    test_oracle_golden.py::test_block_n_truth_equals_the_gp_basis_truth. Both Sigmas are formed in longdouble."""
    LDt = np.longdouble
    pta = synth.make_pta(3, [203, 160, 177], n_tm=[4, 5, 3], ncomps=6, seed=3)
    rng = np.random.default_rng(1)
    blocks, sig, Text, sig_ext = [], [], [], []
    for p in range(3):
        nvec, T, n = pta.Nvecs[p], pta.Ts[p], pta.psrs[p].toas.size
        sl = [(a, a + 4) for a in range(0, n - 40, 4)] + [(n - 30, n - 21)]
        jv = rng.uniform(0.3, 3.0, len(sl)) * 1e-13
        blocks.append((nvec, sl, jv))
        ninv = 1 / nvec.astype(LDt)
        NT = T.astype(LDt) * ninv[:, None]  # N^-1 T by Sherman-Morrison, epoch by epoch
        for (a, b), j in zip(sl, jv):
            NT[a:b] -= ninv[a:b, None] * (LDt(j) / (1 + LDt(j) * ninv[a:b].sum()) * NT[a:b].sum(0))[None, :]
        sig.append(T.astype(LDt).T @ NT + np.diag(1 / pta.phis[p].astype(LDt)))
        U = np.zeros((n, len(sl)))
        for e, (a, b) in enumerate(sl):
            U[a:b, e] = 1.0
        Te = np.concatenate((T, U), axis=1)
        Text.append(Te)
        sig_ext.append(Te.astype(LDt).T @ (Te.astype(LDt) * ninv[:, None])
                       + np.diag(1 / np.concatenate((pta.phis[p], jv)).astype(LDt)))
    freqs = np.concatenate((synth.fp_freqs(7), np.array([1.0, 2.5]) / pta.Tspan))
    pos = np.stack([q.pos for q in pta.psrs])
    fp, fx = antenna_pattern(pos, *_sky(pos))
    fb, cb = truth.fe_truth(freqs, fp, fx, pta.toas, pta.residuals, None, pta.Ts, sig, blocks=blocks)
    fg, cg = truth.fe_truth(freqs, fp, fx, pta.toas, pta.residuals, pta.Nvecs, Text, sig_ext)
    assert np.isfinite(fb.astype(float)).all()
    # two longdouble evaluations of one quantity: a small multiple of the longdouble rounding times the conditioning
    assert np.all(np.abs((fb - fg).astype(float)) <= 1e-14 * np.abs(fg.astype(float)) + 1e4 * EPS_LD * np.maximum(cb, cg))


def test_non_positive_frequencies_give_nan():
    pta = synth.make_pta(2, [120, 90], n_tm=4, ncomps=4, seed=5)
    pos = np.stack([q.pos for q in pta.psrs])
    fp, fx = antenna_pattern(pos, np.array([0.4, 2.0]), np.array([1.0, 4.0]))
    freqs = np.array([0.0, -1e-8, -5e-8, 3e-8])
    fe, cond = truth.fe_truth(freqs, fp, fx, pta.toas, pta.residuals, pta.Nvecs, pta.Ts, pta.sigmas)
    assert np.isnan(fe[:, :3].astype(float)).all() and np.isnan(cond[:, :3]).all()
    assert np.isfinite(fe[:, 3].astype(float)).all() and np.all(fe[:, 3] > 0)
