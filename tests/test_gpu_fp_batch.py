"""Fp of a batch of residual realisations (``FastFp.calculate_Fp_batch``, ``fastfp_fp_sweep_residuals``) on the GPU:
every row against the longdouble truth of oracle/truth.py for that row's residuals, the exact properties the
formulation guarantees (scaling, permutation, NaN isolation, repeatability, frequency batches, the tensor-kernel
setting), every kernel family at the bottom and top of its row range, and the refusals."""
import ctypes as C

import numpy as np
import pytest

import fastfp_b200
from conftest import EPS, term_tolerance
from fastfp_b200 import _cabi, synth
from fastfp_b200.fastfp import batch_pass_rows
from oracle import fp_oracle as o
from oracle import truth
from test_blockn_layout_host import family_of

pytestmark = pytest.mark.gpu


def realisations(pta, R, seed):
    """R residual vectors per pulsar: row 0 the pulsars' own residuals, then seeded white noise plus red noise drawn
    from the basis' prior, with the timing model projected out (what a false-alarm calibration simulates)."""
    rng = np.random.default_rng(seed)
    out = []
    for p, q in enumerate(pta.psrs):
        n, ntm = q.toas.shape[0], pta.n_tm[p]
        res = np.empty((R, n))
        res[0] = q.residuals
        for k in range(1, R):
            r = np.sqrt(pta.Nvecs[p]) * rng.standard_normal(n)
            phi_rn = pta.phis[p][ntm:]
            if phi_rn.size:
                r = r + pta.Ts[p][:, ntm:] @ (np.sqrt(phi_rn) * rng.standard_normal(phi_rn.size))
            res[k] = r - q.Mmat @ (q.Mmat.T @ r)
        out.append(res)
    return out


def assert_rows_near_truth(got, rows, pta, res, freqs, well_conditioned=True):
    """Each listed row against the ordered pulsar sum of the longdouble truth for that row's residuals, within the sum
    of the per-pulsar ``term_tolerance``; bins whose conditioning figure leaves all digits at plain 1e-10."""
    for k in rows:
        rk = [r[k] for r in res]
        args = (freqs, pta.toas, rk, pta.Nvecs, pta.Ts, pta.sigmas)
        tt, cond = truth.fp_sweep_truth(*args)
        tt = tt.astype(float)
        tol = term_tolerance(tt, cond, o.fp_sweep(*args, per_pulsar=True)).sum(axis=0)
        want = tt.sum(axis=0)
        defined = EPS * cond.sum(axis=0) < 0.05 * np.abs(want)
        assert defined.mean() > 0.9, k
        err = np.abs(got[k] - want)
        assert np.all(np.where(defined, err <= tol, True)), (k, float(np.max(np.where(defined, err / tol, 0))))
        if well_conditioned:
            good = EPS * cond.sum(axis=0) < 1e-13 * np.abs(want)
            assert good.any(), k
            assert np.all(np.where(good, err <= 1e-10 * np.abs(want), True)), k


def _small(seed=31):
    pta = synth.make_pta(3, [300, 411, 257], n_tm=[12, 8, 5], ncomps=10, seed=seed)
    freqs = np.concatenate((synth.fp_freqs(40), np.array([1.0, 2.5, 7.0]) / pta.Tspan))
    return pta, freqs


def test_parity_every_row_against_truth_and_row0_against_calculate_Fp():
    pta, freqs = _small()
    assert [T.shape[1] for T in pta.Ts] == [32, 28, 25]  # ragged m_p and n_p in one pack
    res = realisations(pta, 12, seed=1)
    fp = fastfp_b200.FastFp(pta.psrs)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    got = fp.calculate_Fp_batch(freqs, *a, res)
    assert got.shape == (12, freqs.shape[0]) and np.all(np.isfinite(got))
    assert_rows_near_truth(got, range(12), pta, res, freqs)
    # row 0 holds the pulsars' own residuals: what calculate_Fp computes (not bit for bit: (s|r) comes from the MMA)
    one = fp.calculate_Fp(freqs, *a)
    args = (freqs, pta.toas, pta.residuals, *a)
    tt, cond = truth.fp_sweep_truth(*args)
    tol = term_tolerance(tt.astype(float), cond, o.fp_sweep(*args, per_pulsar=True)).sum(axis=0)
    assert np.all(np.abs(got[0] - one) <= 2 * tol)
    # scalar and 2-D frequency arguments
    assert fp.calculate_Fp_batch(freqs[7], *a, res).shape == (12,)
    np.testing.assert_array_equal(fp.calculate_Fp_batch(freqs[7], *a, res), got[:, 7])
    np.testing.assert_array_equal(fp.calculate_Fp_batch(freqs[:40].reshape(5, 8), *a, res),
                                  got[:, :40].reshape(12, 5, 8))


def test_exact_properties():
    pta, freqs = _small(seed=32)
    freqs = np.concatenate((freqs, [0.0, -1e-8]))
    res = realisations(pta, 16, seed=2)
    fp = fastfp_b200.FastFp(pta.psrs)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    base = fp.calculate_Fp_batch(freqs, *a, res)
    assert np.all(np.isnan(base[:, -2:])) and np.all(np.isfinite(base[:, :-2]))  # f <= 0 gives NaN
    # repeated calls, on the cached set and after a fresh upload, are bit-identical
    np.testing.assert_array_equal(fp.calculate_Fp_batch(freqs, *a, res), base)
    fp._res_key = None
    np.testing.assert_array_equal(fp.calculate_Fp_batch(freqs, *a, res), base)
    # an edit in place is seen
    res[1][5, 3] += 1e-7
    edited = fp.calculate_Fp_batch(freqs, *a, res)
    assert not np.array_equal(edited[5, :-2], base[5, :-2])
    np.testing.assert_array_equal(np.delete(edited, 5, 0), np.delete(base, 5, 0))
    res[1][5, 3] -= 1e-7
    # a row holding 2 r is exactly 4 x the row holding r
    dbl = [r.copy() for r in res]
    for r in dbl:
        r[9] = 2.0 * r[4]
    got = fp.calculate_Fp_batch(freqs, *a, dbl)
    np.testing.assert_array_equal(got[9], 4.0 * base[4])
    # permuting the realisations permutes the rows bit for bit
    perm = np.random.default_rng(3).permutation(16)
    np.testing.assert_array_equal(fp.calculate_Fp_batch(freqs, *a, [r[perm] for r in res]), base[perm])
    # a NaN in one realisation of one pulsar makes only that row NaN
    bad = [r.copy() for r in res]
    bad[2][11, 100] = np.nan
    got = fp.calculate_Fp_batch(freqs, *a, bad)
    assert np.all(np.isnan(got[11]))
    np.testing.assert_array_equal(np.delete(got, 11, 0), np.delete(base, 11, 0))
    # the batch always runs the fp64 kernel on the same G packets, whatever the sweep path of the pack
    pre = fastfp_b200.FastFp(pta.psrs, path="prefer-i8")
    assert pre.prepare(*a).path in ("i8", "mixed")
    np.testing.assert_array_equal(pre.calculate_Fp_batch(freqs, *a, res), base)


def test_several_frequency_batches_equal_one():
    # R * P * F above the 2^27-double term budget: one pass of 624 rows x 40 pulsars x 12000 frequencies runs in
    # batches of 2^27 // (624 * 40) = 5377 frequencies, i.e. three batches of one sweep launch + one reduce launch
    pta = synth.make_pta(40, 100, n_tm=12, white_only=True, seed=41)
    res = realisations(pta, 624, seed=4)
    pack = fastfp_b200.FastFp(pta.psrs).prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    pack.set_residuals(res)
    freqs = synth.fp_freqs(12000)
    assert (1 << 27) // (624 * 40) == 5377
    before = _cabi.kernel_launches()
    full = pack.fp_sweep_residuals(freqs)
    assert _cabi.kernel_launches() - before == 2 * 3
    assert np.all(np.isfinite(full))
    for lo, hi in ((0, 5000), (5000, 10000), (10000, 12000)):  # one batch each
        before = _cabi.kernel_launches()
        np.testing.assert_array_equal(pack.fp_sweep_residuals(freqs[lo:hi]), full[:, lo:hi])
        assert _cabi.kernel_launches() - before == 2


# (m, R) -> the family of roundup8(m) + roundup8(R) G rows: bottom and top of each
FAMILY_CASES = [(12, 1, "w1"), (12, 24, "w1"), (72, 1, "w2"), (72, 8, "w2"), (72, 9, "w4"), (72, 88, "w4"),
                (72, 89, "wide"), (72, 248, "wide"), (72, 249, "xwide"), (72, 568, "xwide")]


PULSAR_META_BYTES = 104  # sizeof(ffp::PulsarMeta)


@pytest.mark.parametrize("m,R,fam", FAMILY_CASES)
def test_every_family(m, R, fam):
    rows = -(-m // 8) * 8 + -(-R // 8) * 8
    fam_, ci, mp = family_of(rows)
    assert fam_ == fam
    assert _cabi.load().fastfp_sweep_chunk_toas(rows, 0) == ci
    if m == 12:
        pta = synth.make_pta(2, [300, 257], n_tm=12, white_only=True, seed=50 + R)
    else:
        pta = synth.make_pta(2, [300, 257], n_tm=12, ncomps=30, seed=50 + R)
    assert [T.shape[1] for T in pta.Ts] == [m, m]
    freqs = np.concatenate((synth.fp_freqs(30), np.array([1.0, 2.5, 7.0]) / pta.Tspan))
    res = realisations(pta, R, seed=R)
    # all R rows in one pass of the library, so the configuration of `rows` is the one that runs: its packets take
    # ceil(n / CI) * CI * (4 + MP) doubles per pulsar
    pack = fastfp_b200.FastFp(pta.psrs).prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    base = pack.nbytes
    pack.set_residuals(res)
    assert pack.nbytes - base == sum(-(-n // ci) * ci * (4 + mp) * 8 for n in (300, 257)) + 2 * PULSAR_META_BYTES
    got = pack.fp_sweep_residuals(freqs)
    assert got.shape == (R, 33)
    assert_rows_near_truth(got, sorted({0, R // 2, R - 1}), pta, res, freqs, well_conditioned=m == 12)
    np.testing.assert_array_equal(pack.fp_sweep_residuals(freqs), got)


def test_more_rows_than_one_pass_are_split():
    pta = synth.make_pta(2, [300, 257], n_tm=12, ncomps=30, seed=60)
    freqs = synth.fp_freqs(20)
    res = realisations(pta, 569, seed=5)
    fp = fastfp_b200.FastFp(pta.psrs)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    pack = fp.prepare(*a)
    with pytest.raises(_cabi.FastFpError, match=r"limit of 568 .*widest pulsar 0 \(m = 72\)"):
        pack.set_residuals(res)
    got = fp.calculate_Fp_batch(freqs, *a, res)
    assert got.shape == (569, 20) and np.all(np.isfinite(got))
    # each pass of batch_pass_rows equals its rows swept alone in one library call
    rows = batch_pass_rows(569, [72, 72])
    assert rows < 569
    for lo in range(0, 569, rows):
        hi = min(569, lo + rows)
        pack.set_residuals([r[lo:hi] for r in res])
        np.testing.assert_array_equal(pack.fp_sweep_residuals(freqs), got[lo:hi])
    assert_rows_near_truth(got, [0, 300, 568], pta, res, freqs, well_conditioned=False)


def test_refusals_and_pack_bytes():
    lib = _cabi.load()
    pta, freqs = _small(seed=33)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    pack = fastfp_b200.FastFp(pta.psrs).prepare(*a)
    out = np.empty((4, freqs.shape[0]))
    vp = lambda x: C.c_void_p(x.ctypes.data)  # noqa: E731
    assert lib.fastfp_fp_sweep_residuals(pack._h, vp(freqs), freqs.shape[0], vp(out), 0, None) == -1
    assert "no residual realisations set" in lib.fastfp_last_error().decode()
    base = pack.nbytes
    res = realisations(pta, 4, seed=6)
    pack.set_residuals(res)
    assert pack.nbytes > base
    assert lib.fastfp_fp_sweep_residuals(pack._h, vp(freqs), 0, vp(out), 0, None) == 0  # F = 0 writes nothing
    assert pack.fp_sweep_residuals(freqs).shape == (4, freqs.shape[0])
    pack.set_residuals([r[:0] for r in res])  # R = 0 releases them
    assert pack.nbytes == base
    assert lib.fastfp_fp_sweep_residuals(pack._h, vp(freqs), freqs.shape[0], vp(out), 0, None) == -1
    # nmfp pack
    nm = _cabi.Pack.create(pta.toas, pta.residuals, pta.Nvecs, pta.Ts, pta.TNTs, m_fix=pta.n_tm,
                           phiinv_fix=[phi[:k] ** -1 for phi, k in zip(pta.phis, pta.n_tm)])
    assert lib.fastfp_pack_set_residuals(nm._h, 4, _cabi._ptr_array([_cabi.as_f64(r) for r in res]), None) == -1
    # block-N pack: refused by the library before it reads the arrays, and by the binding
    ep = synth.make_pta(2, 96, n_tm=4, ncomps=5, epoch=4, seed=34)
    Nvecs, Ts, TNTs, phis = synth.with_ecorr(ep, kernel=True)
    fb = fastfp_b200.FastFp(ep.psrs)
    bpack = fb.prepare(Nvecs, Ts, [T + np.diag(1.0 / phi) for T, phi in zip(TNTs, phis)])
    assert bpack.blockn
    rows = [np.zeros((2, n)) for n in bpack.n]
    assert lib.fastfp_pack_set_residuals(bpack._h, 2, _cabi._ptr_array(rows), None) == -3
    with pytest.raises(_cabi.FastFpError, match="diagonal-N"):
        bpack.set_residuals(rows)


def test_cuda_tensor_on_a_non_default_stream():
    import torch

    pta, freqs = _small(seed=35)
    res = realisations(pta, 10, seed=7)
    fp = fastfp_b200.FastFp(pta.psrs)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    want = fp.calculate_Fp_batch(freqs[:40], *a, res)
    fp2 = fastfp_b200.FastFp(pta.psrs)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        f = torch.tensor(freqs[:40].reshape(5, 8), dtype=torch.float64, device="cuda")
        got = fp2.calculate_Fp_batch(f, *a, res)
    s.synchronize()
    assert got.is_cuda and got.shape == (10, 5, 8)
    np.testing.assert_array_equal(got.cpu().numpy().reshape(10, 40), want)
