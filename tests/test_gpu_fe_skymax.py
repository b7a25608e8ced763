"""Sky-maximised Fe-statistic (``FastFe.calculate_Fe_skymax``, ``fastfp_fe_skymax``) on the GPU, on both sweep
kernels: bit for bit against the reduction rule applied to ``calculate_Fe``'s (S, F) map, and against
oracle/fe_oracle.py."""
import numpy as np
import pytest

import fastfp_b200
from fastfp_b200 import _cabi, synth
from fastfp_b200.fe import antenna_pattern
from oracle import fe_oracle

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("sweep_path")]


def rule(fe_map):
    """The documented reduction over the sky axis of an (S, F) map: NaN loses, the lowest index wins a tie, an
    all-NaN column gives (NaN, -1)."""
    fe_map = np.asarray(fe_map)
    nan = np.isnan(fe_map)
    best = np.where(nan, -np.inf, fe_map).max(axis=0)
    hit = (fe_map == best[None, :]) & ~nan
    some = hit.any(axis=0)
    idx = np.where(some, np.argmax(hit, axis=0), -1).astype(np.int64)
    val = np.where(some, fe_map[np.maximum(idx, 0), np.arange(fe_map.shape[1])], np.nan)
    return val, idx


def _equal(got, want):
    np.testing.assert_array_equal(got[0], want[0])
    np.testing.assert_array_equal(got[1], want[1])
    assert got[0].dtype == np.float64 and got[1].dtype == np.int64


def _grid(n_rand, n_th, n_ph, seed):
    rng = np.random.default_rng(seed)
    th = np.concatenate((np.arccos(rng.uniform(-1, 1, n_rand)), np.repeat(np.linspace(0.05, np.pi - 0.05, n_th), n_ph)))
    ph = np.concatenate((rng.uniform(0, 2 * np.pi, n_rand), np.tile(np.linspace(0, 2 * np.pi, n_ph, endpoint=False), n_th)))
    return th, ph


def test_bit_identity_with_the_map():
    pta = synth.make_pta(5, [300, 257, 411, 350, 280], n_tm=[6, 8, 5, 7, 6], ncomps=10, seed=21)
    yr = 365.25 * 86400.0
    freqs = np.concatenate((synth.fp_freqs(190), np.arange(1, 9) / pta.Tspan, [1.0 / yr, 2.0 / yr]))
    th, ph = _grid(260, 12, 20, seed=5)  # 500 positions
    fe = fastfp_b200.FastFe(pta.psrs)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    fe_map = fe.calculate_Fe(freqs, th, ph, *a)
    got = fe.calculate_Fe_skymax(freqs, th, ph, *a)
    _equal(got, rule(fe_map))
    assert np.all(got[1] >= 0)
    # scalar frequency -> (float, int)
    one = fe.calculate_Fe_skymax(float(freqs[7]), th, ph, *a)
    assert type(one[0]) is float and type(one[1]) is int
    assert (one[0], one[1]) == (got[0][7], got[1][7])


def test_against_the_oracle():
    pta = synth.make_pta(4, [300, 257, 411, 350], n_tm=[6, 8, 5, 7], ncomps=10, seed=12)
    freqs = np.concatenate((synth.fp_freqs(40)[10::7], [7.0 / pta.Tspan]))[:6]
    th, ph = _grid(12, 3, 4, seed=9)  # 24 positions
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    val, idx = fastfp_b200.FastFe(pta.psrs).calculate_Fe_skymax(freqs, th, ph, *a)
    pos = [q.pos for q in pta.psrs]
    want = np.array([[fe_oracle.calculate_Fe(f, t, p_, pta.toas, pta.residuals, pos, *a) for f in freqs]
                     for t, p_ in zip(th, ph)])
    well = freqs > 40.0 / pta.Tspan
    assert well.sum() >= 4
    top = np.max(want, axis=0)
    assert np.abs(val[well] / top[well] - 1).max() < 1e-9
    srt = np.sort(want, axis=0)
    clear = (srt[-1] - srt[-2]) > 1e-8 * np.abs(srt[-1])
    assert clear.sum() >= 3
    np.testing.assert_array_equal(idx[clear], np.argmax(want, axis=0)[clear])


def test_more_sky_positions_than_the_map_allows():
    pta = synth.make_pta(3, 120, n_tm=4, ncomps=4, seed=33)
    fe = fastfp_b200.FastFe(pta.psrs)
    pack = fe.prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    th, ph = _grid(70001, 0, 0, seed=1)
    fp, fx = antenna_pattern(fe.pos, th, ph)
    freqs = synth.fp_freqs(64)
    with pytest.raises(_cabi.FastFpError, match="65535"):
        pack.fe_sweep(freqs, fp, fx)
    fe_map = np.concatenate([pack.fe_sweep(freqs, fp[lo:lo + 65535], fx[lo:lo + 65535])
                             for lo in range(0, th.size, 65535)])
    got = pack.fe_skymax(freqs, fp, fx)
    _equal(got, rule(fe_map))


def test_many_frequencies_few_positions():
    P = 68
    pta = synth.make_pta(P, 40, n_tm=3, ncomps=2, seed=44)
    F = 400_000
    assert F > (1 << 27) // (5 * P)  # two frequency batches
    freqs = np.linspace(1e-9, 4e-7, F)
    th, ph = _grid(16, 0, 0, seed=2)
    fe = fastfp_b200.FastFe(pta.psrs)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    _equal(fe.calculate_Fe_skymax(freqs, th, ph, *a), rule(fe.calculate_Fe(freqs, th, ph, *a)))


def test_pulsars_in_several_chunks_and_several_sky_passes():
    """P = 40 takes two pulsar chunks of shared memory, so the inner products are reloaded for every pass of 16 sky
    positions while the accumulators carry across the chunks; S = 101 makes several passes per CTA with a partial last
    one, and F = 1000 leaves a partial last frequency tile."""
    pta = synth.make_pta(40, 60, n_tm=3, ncomps=3, seed=99)
    freqs = np.linspace(3e-9, 2.5e-7, 1000)
    th, ph = _grid(101, 0, 0, seed=6)
    fe = fastfp_b200.FastFe(pta.psrs)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    fe_map = fe.calculate_Fe(freqs, th, ph, *a)
    assert np.isfinite(fe_map).all()
    _equal(fe.calculate_Fe_skymax(freqs, th, ph, *a), rule(fe_map))


def test_ties_and_nan():
    pta = synth.make_pta(5, 200, n_tm=5, ncomps=6, seed=55)
    pack = fastfp_b200.FastFe(pta.psrs).prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    rng = np.random.default_rng(3)
    R, X = rng.uniform(-1, 1, (6, 5)), rng.uniform(-1, 1, (6, 5))
    freqs = np.concatenate((synth.fp_freqs(30), [0.0, -5e-8]))
    base = pack.fe_skymax(freqs, R, X)
    _equal(base, rule(pack.fe_sweep(freqs, R, X)))
    # the maximum of every column appears three times: the lowest index wins
    _equal(pack.fe_skymax(freqs, np.vstack((R, R, R)), np.vstack((X, X, X))), base)
    # every row the same: index 0 wherever a value exists
    same = pack.fe_skymax(freqs, np.repeat(R[2:3], 40, axis=0), np.repeat(X[2:3], 40, axis=0))
    col = pack.fe_sweep(freqs, R[2:3], X[2:3])[0]
    np.testing.assert_array_equal(same[0], col)
    np.testing.assert_array_equal(same[1], np.where(np.isnan(col), -1, 0))
    # all-zero rows give NaN (M = 0), which loses to every value
    Z = np.zeros((3, 5))
    zp, zx = np.vstack((Z, R, Z)), np.vstack((Z, X, Z))
    zmap = pack.fe_sweep(freqs, zp, zx)
    assert np.isnan(zmap[:3]).all() and np.isnan(zmap[-3:]).all()
    got = pack.fe_skymax(freqs, zp, zx)
    _equal(got, rule(zmap))
    ok = base[1] >= 0
    np.testing.assert_array_equal(got[1][ok], base[1][ok] + 3)
    # no position has a value: (NaN, -1) at every frequency, and at the frequencies where the map is all NaN
    v, i = pack.fe_skymax(freqs, Z, Z)
    assert np.isnan(v).all() and (i == -1).all()
    for k in (-2, -1):  # f = 0 and f < 0
        assert np.isnan(zmap[:, k]).all() and np.isnan(base[0][k]) and base[1][k] == -1
        assert np.isnan(got[0][k]) and got[1][k] == -1


def test_device_resident_calls():
    import torch

    pta = synth.make_pta(3, 300, n_tm=6, ncomps=8, seed=66)
    f = synth.fp_freqs(90)
    th, ph = _grid(40, 0, 0, seed=4)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    fe = fastfp_b200.FastFe(pta.psrs)
    host = fe.calculate_Fe_skymax(f, th, ph, *a)
    ft = torch.tensor(f, dtype=torch.float64, device="cuda")
    v, i = fe.calculate_Fe_skymax(ft, th, ph, *a)
    assert v.is_cuda and i.is_cuda and v.dtype == torch.float64 and i.dtype == torch.int64
    _equal((v.cpu().numpy(), i.cpu().numpy()), host)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        v2, i2 = fe.calculate_Fe_skymax(ft, th, ph, *a)
    s.synchronize()
    _equal((v2.cpu().numpy(), i2.cpu().numpy()), host)


def test_block_n_pack():
    pta = synth.make_pta(3, 240, n_tm=6, ncomps=8, seed=77, epoch=4)
    Nvecs, Ts, TNTs, phis = synth.with_ecorr(pta, kernel=True)
    sig = [TNT + np.diag(1.0 / phi) for TNT, phi in zip(TNTs, phis)]
    freqs = synth.fp_freqs(60)
    th, ph = _grid(50, 0, 0, seed=8)
    fe = fastfp_b200.FastFe(pta.psrs)
    fe_map = fe.calculate_Fe(freqs, th, ph, Nvecs, Ts, sig)
    assert np.isfinite(fe_map).all()
    _equal(fe.calculate_Fe_skymax(freqs, th, ph, Nvecs, Ts, sig), rule(fe_map))


def test_errors():
    from fastfp_b200.nmfp import NMFP, RN_container

    pta = synth.make_pta(2, 100, n_tm=4, ncomps=3, seed=88)
    fe = fastfp_b200.FastFe(pta.psrs)
    pack = fe.prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    freqs = synth.fp_freqs(8)
    with pytest.raises(_cabi.FastFpError, match="at least one sky position"):
        pack.fe_skymax(freqs, np.zeros((0, 2)), np.zeros((0, 2)))
    v, i = pack.fe_skymax(np.zeros(0), np.ones((3, 2)), np.ones((3, 2)))
    assert v.shape == (0,) and i.shape == (0,)
    v, i = fe.calculate_Fe_skymax(np.zeros(0), [0.3, 1.0], [0.2, 2.0], pta.Nvecs, pta.Ts, pta.sigmas)
    assert v.shape == (0,) and i.shape == (0,) and i.dtype == np.int64
    nm = NMFP(pta.psrs, [RN_container(q, ncomps=3) for q in pta.psrs]).prepare(pta.Nvecs, pta.Ts, pta.TNTs)
    with pytest.raises(_cabi.FastFpError, match="plain-Fp pack"):
        nm.fe_skymax(freqs, np.ones((3, 2)), np.ones((3, 2)))
