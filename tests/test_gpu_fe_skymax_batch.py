"""Sky-maximised Fe of a batch of residual realisations (``FastFe.calculate_Fe_skymax_batch``,
``fastfp_fe_skymax_residuals``) on the GPU: every row against the sky maximum of the longdouble Fe truth for that row's
residuals, row 0 against ``calculate_Fe_skymax``, the exact properties the formulation guarantees (repeatability,
row isolation, scaling, permutation, NaN isolation, f <= 0, the tensor-kernel setting), independence of the sky,
frequency-batch and pass splits, pure antenna patterns against the Fp batch, every row family, and the interface."""
import ctypes as C

import numpy as np
import pytest

import fastfp_b200
from conftest import EPS, term_tolerance
from fastfp_b200 import _cabi, synth
from fastfp_b200.fastfp import batch_pass_rows
from fastfp_b200.fe import antenna_pattern
from oracle import fp_oracle as o
from oracle import truth
from test_gpu_fp_batch import FAMILY_CASES, assert_rows_near_truth, realisations

pytestmark = pytest.mark.gpu


def _pos(pta):
    return np.stack([q.pos for q in pta.psrs])


def _grid(pos, n, seed):
    """n sky positions: n - 2 random, the north pole, and one 0.03 rad from pulsar 0."""
    rng = np.random.default_rng(seed)
    th0, ph0 = np.arccos(pos[0, 2]), np.arctan2(pos[0, 1], pos[0, 0]) % (2 * np.pi)
    th = np.concatenate((np.arccos(rng.uniform(-1, 1, n - 2)), [0.0, th0 + 0.03]))
    ph = np.concatenate((rng.uniform(0, 2 * np.pi, n - 2), [0.0, ph0]))
    return th, ph


def _freqs(pta):
    """73 bins including the 1, 2.5 and 7 / Tspan red-noise bins."""
    return np.concatenate((synth.fp_freqs(70), np.array([1.0, 2.5, 7.0]) / pta.Tspan))


def _row_truth(freqs, pta, res_k, fp, fx):
    """Fe truth (S, F), its cond and E (test_gpu_fe_truth's tolerance) for one realisation."""
    args = (pta.toas, res_k, pta.Nvecs, pta.Ts, pta.sigmas)
    inner = truth.sweep_inner_truth(freqs, *args)
    fe, cond = truth.fe_truth_from_inner(inner, freqs, fp, fx)
    tt, tc = truth.terms_truth(inner)
    E = (term_tolerance(tt.astype(float), tc, o.fp_sweep(freqs, *args, per_pulsar=True), k_oracle=1.0, rel=0.0)
         / (EPS * tc)).max()
    return fe.astype(float), cond, E


def _assert_skymax_near(best, idx, fe, cond, E, what, rel=1e-10):
    """best / idx (F,) against the sky maximum of the truth fe (S, F), with test_gpu_fe_truth._assert_near's tolerance
    (relative part ``rel``): the value is the truth at the returned position within that position's tolerance and the
    truth's maximum within the tolerances at both positions; the index is the truth's argmax wherever the truth's top
    two are further apart than their tolerances."""
    tol = rel * np.abs(fe) + 4 * E * EPS * cond
    am = np.nanargmax(fe, axis=0)
    cols = np.arange(fe.shape[1])
    tmax, tolm = fe[am, cols], tol[am, cols]
    defined = EPS * cond[am, cols] < 0.05 * np.abs(tmax)
    assert defined.mean() >= 0.9, (what, defined.mean())
    assert np.all(idx >= 0), what
    at, tola = fe[idx, cols], tol[idx, cols]
    ok = defined & (EPS * cond[idx, cols] < 0.05 * np.abs(at))
    assert np.all(np.where(ok, np.abs(best - at) <= tola, True)), (what, np.max(np.where(ok, np.abs(best - at) / tola, 0)))
    assert np.all(np.where(ok, np.abs(best - tmax) <= tolm + tola, True)), what
    order = np.argsort(np.where(np.isnan(fe), -np.inf, fe), axis=0)
    second = order[-2] if fe.shape[0] > 1 else am
    clear = defined & (tmax - fe[second, cols] > tolm + tol[second, cols])
    assert np.all(np.where(clear, idx == am, True)), (what, np.flatnonzero(clear & (idx != am)))


def _case(P=4, R=12, seed=41, S=30):
    ns = [300, 411, 257, 350, 222][:P]
    pta = synth.make_pta(P, ns, n_tm=[12, 8, 5, 9, 7][:P], ncomps=10, seed=seed)
    th, ph = _grid(_pos(pta), S, seed)
    return pta, realisations(pta, R, seed=seed), th, ph


def test_every_row_against_truth_and_row0_against_calculate_Fe_skymax():
    pta, res, th, ph = _case()
    freqs = _freqs(pta)
    fe = fastfp_b200.FastFe(pta.psrs)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    best, idx = fe.calculate_Fe_skymax_batch(freqs, th, ph, *a, res)
    assert best.shape == idx.shape == (12, 73) and idx.dtype == np.int64 and np.all(np.isfinite(best))
    fp, fx = antenna_pattern(_pos(pta), th, ph)
    truths = []
    for k in range(12):
        t = _row_truth(freqs, pta, [r[k] for r in res], fp, fx)
        truths.append(t)
        _assert_skymax_near(best[k], idx[k], *t, f"row {k}")
    # row 0 holds the pulsars' own residuals: calculate_Fe_skymax on its own pack, to twice the tolerance
    b0, i0 = fe.calculate_Fe_skymax(freqs, th, ph, *a)
    fe0, cond0, E0 = truths[0]
    _assert_skymax_near(b0, i0, fe0, cond0, E0, "calculate_Fe_skymax")
    tol = 2 * (1e-10 * np.abs(fe0) + 4 * E0 * EPS * cond0)[i0, np.arange(73)]
    assert np.all(np.abs(best[0] - b0) <= tol)
    srt = np.sort(fe0, axis=0)
    clear = srt[-1] - srt[-2] > tol
    assert np.all(np.where(clear, idx[0] == i0, True))


def test_exact_properties():
    pta, res, th, ph = _case(seed=42)
    freqs = _freqs(pta)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    fe = fastfp_b200.FastFe(pta.psrs)
    best, idx = fe.calculate_Fe_skymax_batch(freqs, th, ph, *a, res)
    # repeated calls and a fresh upload give the same bits
    for b2, i2 in (fe.calculate_Fe_skymax_batch(freqs, th, ph, *a, res),
                   fastfp_b200.FastFe(pta.psrs).calculate_Fe_skymax_batch(freqs, th, ph, *a, res)):
        np.testing.assert_array_equal(b2, best)
        np.testing.assert_array_equal(i2, idx)
    # an in-place edit of one realisation changes only its row
    res[1][5] *= 1.5
    b3, i3 = fe.calculate_Fe_skymax_batch(freqs, th, ph, *a, res)
    keep = np.arange(12) != 5
    np.testing.assert_array_equal(b3[keep], best[keep])
    np.testing.assert_array_equal(i3[keep], idx[keep])
    assert np.any(b3[5] != best[5])
    # 2r gives exactly 4x with the same indices; a permutation permutes the rows bit for bit
    perm = np.random.default_rng(3).permutation(12)
    res2 = [np.concatenate((r[perm], 2 * r[:1])) for r in res]
    b4, i4 = fe.calculate_Fe_skymax_batch(freqs, th, ph, *a, res2)
    np.testing.assert_array_equal(b4[:12], b3[perm])
    np.testing.assert_array_equal(i4[:12], i3[perm])
    np.testing.assert_array_equal(b4[12], 4 * b3[0])
    np.testing.assert_array_equal(i4[12], i3[0])
    # a NaN in one realisation gives (NaN, -1) in that row only
    res3 = [r.copy() for r in res]
    res3[2][7, 11] = np.nan
    b5, i5 = fe.calculate_Fe_skymax_batch(freqs, th, ph, *a, res3)
    assert np.all(np.isnan(b5[7])) and np.all(i5[7] == -1)
    keep = np.arange(12) != 7
    np.testing.assert_array_equal(b5[keep], b3[keep])
    # f <= 0 gives (NaN, -1) in every row
    fneg = np.concatenate((freqs[:5], [0.0, -1e-8, -5e-8]))
    b6, i6 = fe.calculate_Fe_skymax_batch(fneg, th, ph, *a, res)
    assert np.all(np.isnan(b6[:, 5:])) and np.all(i6[:, 5:] == -1)
    np.testing.assert_array_equal(b6[:, :5], b3[:, :5])
    # a prefer-i8 pack gives the same bits (the residual batch always runs the fp64 kernel)
    b7, i7 = fastfp_b200.FastFe(pta.psrs, path="prefer-i8").calculate_Fe_skymax_batch(freqs, th, ph, *a, res)
    np.testing.assert_array_equal(b7, b3)
    np.testing.assert_array_equal(i7, i3)


def _merge(parts):
    """fe_better merge of (best, idx) parts whose indices are already offset, in order."""
    best, idx = parts[0][0].copy(), parts[0][1].copy()
    for b, i in parts[1:]:
        better = ~np.isnan(b) & (np.isnan(best) | (b > best) | ((b == best) & (i < idx)))
        best, idx = np.where(better, b, best), np.where(better, i, idx)
    return best, idx


def _assert_sky_split(pack, freqs, fp, fx, cut):
    best, idx = pack.fe_skymax_residuals(freqs, fp, fx)
    b1, i1 = pack.fe_skymax_residuals(freqs, fp[:cut], fx[:cut])
    b2, i2 = pack.fe_skymax_residuals(freqs, fp[cut:], fx[cut:])
    mb, mi = _merge([(b1, i1), (b2, np.where(i2 >= 0, i2 + cut, -1))])
    np.testing.assert_array_equal(best, mb)
    np.testing.assert_array_equal(idx, mi)
    return best, idx


def test_sky_frequency_and_pulsar_splits():
    pta, res, th, ph = _case(seed=43, S=200)
    fp, fx = antenna_pattern(_pos(pta), th, ph)
    pack = fastfp_b200.FastFe(pta.psrs).prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    pack.set_residuals(res)
    _assert_sky_split(pack, _freqs(pta), fp, fx, 77)
    # few frequencies, many positions: the sky is split across CTAs and merged
    few = _freqs(pta)[60:63]
    thb, phb = _grid(_pos(pta), 5000, 9)
    fpb, fxb = antenna_pattern(_pos(pta), thb, phb)
    best, idx = _assert_sky_split(pack, few, fpb, fxb, 2345)
    # row 0 against calculate_Fe_skymax's kernel on the same grid
    b0, i0 = pack.fe_skymax(few, fpb, fxb)
    assert np.all(np.abs(best[0] - b0) <= 1e-8 * np.abs(b0))
    # S > 65 535
    thc, phc = _grid(_pos(pta), 70000, 10)
    fpc, fxc = antenna_pattern(_pos(pta), thc, phc)
    pack.set_residuals([r[:3] for r in res])
    _assert_sky_split(pack, few[:2], fpc, fxc, 65536)
    # a frequency range of several batches equals the per-batch calls: 2^27 / ((2R + 3) P) = 3111 at R = 566, P = 38
    big = synth.make_pta(38, 64, n_tm=3, ncomps=2, seed=44)
    pk = fastfp_b200.FastFe(big.psrs).prepare(big.Nvecs, big.Ts, big.sigmas)
    rb = realisations(big, 566, seed=4)
    pk.set_residuals(rb)
    fb = 2 ** 27 // ((2 * 566 + 3) * 38)
    freqs = np.linspace(1e-9, 3e-7, 2 * fb + 100)
    thd, phd = _grid(_pos(big), 40, 11)
    fpd, fxd = antenna_pattern(_pos(big), thd, phd)
    best, idx = pk.fe_skymax_residuals(freqs, fpd, fxd)
    for lo in range(0, freqs.shape[0], fb):
        b, i = pk.fe_skymax_residuals(freqs[lo:lo + fb], fpd, fxd)
        np.testing.assert_array_equal(b, best[:, lo:lo + fb])
        np.testing.assert_array_equal(i, idx[:, lo:lo + fb])


def test_more_pulsars_than_one_shared_memory_chunk():
    pta = synth.make_pta(50, [120 + 7 * p for p in range(50)], n_tm=4, ncomps=4, seed=45)
    res = realisations(pta, 20, seed=45)
    th, ph = _grid(_pos(pta), 70, 12)
    fp, fx = antenna_pattern(_pos(pta), th, ph)
    freqs = synth.fp_freqs(40)
    pack = fastfp_b200.FastFe(pta.psrs).prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    pack.set_residuals(res)
    best, idx = _assert_sky_split(pack, freqs, fp, fx, 33)
    for k in (0, 19):
        fe, cond, E = _row_truth(freqs, pta, [r[k] for r in res], fp, fx)
        _assert_skymax_near(best[k], idx[k], fe, cond, E, f"P = 50, row {k}")


def test_pure_patterns_equal_the_fp_batch():
    pta = synth.make_pta(2, [300, 257], n_tm=[12, 8], ncomps=10, seed=46)
    res = realisations(pta, 9, seed=46)
    freqs = _freqs(pta)
    pack = fastfp_b200.FastFe(pta.psrs).prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    pack.set_residuals(res)
    best, idx = pack.fe_skymax_residuals(freqs, np.array([[1.0, 0.0]]), np.array([[0.0, 1.0]]))
    assert np.all(idx == 0)
    assert_rows_near_truth(best, range(9), pta, res, freqs)
    fpb = pack.fp_sweep_residuals(freqs)
    for k in range(9):
        args = (freqs, pta.toas, [r[k] for r in res], pta.Nvecs, pta.Ts, pta.sigmas)
        tt, cond = truth.fp_sweep_truth(*args)
        tol = term_tolerance(tt.astype(float), cond, o.fp_sweep(*args, per_pulsar=True)).sum(axis=0)
        assert np.all(np.abs(best[k] - fpb[k]) <= 2 * tol), k


@pytest.mark.parametrize("m,R,fam", FAMILY_CASES)
def test_every_row_family(m, R, fam):
    if m == 12:
        pta = synth.make_pta(2, [300, 257], n_tm=12, white_only=True, seed=50 + R)
    else:
        pta = synth.make_pta(2, [300, 257], n_tm=12, ncomps=30, seed=50 + R)
    freqs = np.concatenate((synth.fp_freqs(30), np.array([1.0, 2.5, 7.0]) / pta.Tspan))
    res = realisations(pta, R, seed=R)
    th, ph = _grid(_pos(pta), 12, R)
    fp, fx = antenna_pattern(_pos(pta), th, ph)
    pack = fastfp_b200.FastFe(pta.psrs).prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    pack.set_residuals(res)
    best, idx = pack.fe_skymax_residuals(freqs, fp, fx)
    assert best.shape == (R, 33)
    for k in sorted({0, R // 2, R - 1}):
        fe, cond, E = _row_truth(freqs, pta, [r[k] for r in res], fp, fx)
        _assert_skymax_near(best[k], idx[k], fe, cond, E, f"m={m} R={R} ({fam}) row {k}")


def test_more_rows_than_one_pass_are_split():
    pta = synth.make_pta(2, [300, 257], n_tm=12, ncomps=30, seed=60)
    freqs = synth.fp_freqs(20)
    res = realisations(pta, 569, seed=5)
    th, ph = _grid(_pos(pta), 10, 60)
    fe = fastfp_b200.FastFe(pta.psrs)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    best, idx = fe.calculate_Fe_skymax_batch(freqs, th, ph, *a, res)
    assert best.shape == (569, 20) and np.all(np.isfinite(best))
    fp, fx = antenna_pattern(_pos(pta), th, ph)
    pack = fe.prepare(*a)
    rows = batch_pass_rows(569, [72, 72])
    assert rows < 569
    for lo in range(0, 569, rows):
        hi = min(569, lo + rows)
        pack.set_residuals([r[lo:hi] for r in res])
        b, i = pack.fe_skymax_residuals(freqs, fp, fx)
        np.testing.assert_array_equal(b, best[lo:hi])
        np.testing.assert_array_equal(i, idx[lo:hi])


def test_cuda_tensor_on_a_non_default_stream():
    import torch

    pta, res, th, ph = _case(seed=47, R=10)
    freqs = _freqs(pta)[:40]
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    want_b, want_i = fastfp_b200.FastFe(pta.psrs).calculate_Fe_skymax_batch(freqs, th, ph, *a, res)
    fe2 = fastfp_b200.FastFe(pta.psrs)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        f = torch.tensor(freqs.reshape(5, 8), dtype=torch.float64, device="cuda")
        got_b, got_i = fe2.calculate_Fe_skymax_batch(f, th, ph, *a, res)
    s.synchronize()
    assert got_b.is_cuda and got_b.shape == (10, 5, 8) and got_i.dtype == torch.int64
    np.testing.assert_array_equal(got_b.cpu().numpy().reshape(10, 40), want_b)
    np.testing.assert_array_equal(got_i.cpu().numpy().reshape(10, 40), want_i)
    b1, i1 = fe2.calculate_Fe_skymax_batch(freqs[3], th, ph, *a, res)  # a scalar fgw gives (R,)
    assert b1.shape == i1.shape == (10,)
    np.testing.assert_array_equal(b1, want_b[:, 3])


def test_refusals():
    lib = _cabi.load()
    pta, res, th, ph = _case(seed=48, R=4)
    freqs = _freqs(pta)
    fp, fx = antenna_pattern(_pos(pta), th, ph)
    F, S = freqs.shape[0], fp.shape[0]
    out, iout = np.empty((4, F)), np.empty((4, F), dtype=np.int64)
    vp = lambda x: C.c_void_p(x.ctypes.data)  # noqa: E731

    def call(pk, F=F, S=S):
        return lib.fastfp_fe_skymax_residuals(pk._h, vp(freqs), F, vp(fp), vp(fx), S, vp(out), vp(iout), 0, None)

    pack = fastfp_b200.FastFe(pta.psrs).prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    assert call(pack) == -1
    assert lib.fastfp_last_error().decode() == \
        "fastfp_fe_skymax_residuals: no residual realisations set (fastfp_pack_set_residuals)"
    pack.set_residuals(res)
    assert call(pack, S=0) == -1
    assert lib.fastfp_last_error().decode() == "fastfp_fe_skymax_residuals needs at least one sky position"
    out[:], iout[:] = 7.0, 7
    assert call(pack, F=0) == 0 and call(pack, F=0, S=0) == 0  # F = 0 writes nothing
    assert np.all(out == 7.0) and np.all(iout == 7)
    assert call(pack) == 0 and np.all(np.isfinite(out)) and np.all((iout >= 0) & (iout < S))
    nm = _cabi.Pack.create(pta.toas, pta.residuals, pta.Nvecs, pta.Ts, pta.TNTs, m_fix=pta.n_tm,
                           phiinv_fix=[phi[:k] ** -1 for phi, k in zip(pta.phis, pta.n_tm)])
    assert call(nm) == -1
    assert lib.fastfp_last_error().decode() == "fastfp_fe_skymax_residuals needs a plain-Fp pack (fastfp_pack_create)"
    # block-N packs cannot hold realisations
    ep = synth.make_pta(2, 96, n_tm=4, ncomps=5, epoch=4, seed=34)
    Nvecs, Ts, TNTs, phis = synth.with_ecorr(ep, kernel=True)
    bpack = fastfp_b200.FastFe(ep.psrs).prepare(Nvecs, Ts, [T + np.diag(1.0 / phi) for T, phi in zip(TNTs, phis)])
    assert bpack.blockn
    fpe, fxe = antenna_pattern(_pos(ep), th, ph)
    assert lib.fastfp_fe_skymax_residuals(bpack._h, vp(freqs), F, vp(fpe), vp(fxe), S, vp(out), vp(iout), 0, None) == -1
    assert "no residual realisations set" in lib.fastfp_last_error().decode()
