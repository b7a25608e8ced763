"""GPU parity tests for the plain Fp path: the CUDA sweep (through the C ABI) against the golden
vectors of the reference source, the oracle and the longdouble truth. Run with -m gpu on an H100."""
import numpy as np
import pytest

import fastfp_b200
from conftest import EPS, Psr, term_tolerance
from fastfp_b200 import _cabi, synth
from oracle import fp_oracle as o
from oracle import truth

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("sweep_path")]


def _args(g):
    return g.lst("Nvec"), g.lst("T"), g.lst("sigma")


@pytest.mark.parametrize("name", ["fp_white", "fp_red"])
def test_sweep_matches_reference_goldens(golden, name):
    g = golden(name)
    fp = fastfp_b200.FastFp(g.psrs)
    got_terms = fp.per_pulsar_terms(g["freqs"], *_args(g))
    ora_terms = o.fp_sweep(g["freqs"], g.lst("toas"), g.lst("res"), *_args(g), per_pulsar=True)
    tol = term_tolerance(g["truth_terms"], g["cond"], ora_terms)
    # (1) no further from the extended-precision truth than the reference formula's own envelope
    assert np.all(np.abs(got_terms - g["truth_terms"]) <= tol)
    # (2) the summed statistic against the reference source's output: 1e-10 relative, plus the
    #     conditioning allowance where the reference itself is only defined to eps*kappa
    got = fp(g["freqs"], *_args(g))
    assert got.shape == g["ref_fp"].shape
    assert np.all(np.abs(got - g["ref_fp"]) <= 1e-10 * np.abs(g["ref_fp"]) + 2 * tol.sum(0))
    # well-conditioned points must meet the plain 1e-10 (north-star tolerance)
    well = g["cond"].sum(0) * EPS < 1e-12 * np.abs(g["ref_fp"])
    assert well.any()
    assert np.all(np.abs(got[well] / g["ref_fp"][well] - 1) <= 1e-10)


def test_white_noise_config_c1_is_tight(golden):
    """C1 (examples/run_fp.py path, T = timing model only) is well conditioned everywhere."""
    g = golden("fp_white")
    got = fastfp_b200.FastFp(g.psrs)(g["freqs"], *_args(g))
    assert np.abs(got / g["ref_fp"] - 1).max() < 1e-12


def test_scalar_call_and_aliases(golden):
    g = golden("fp_white")
    fp = fastfp_b200.FastFp(g.psrs, pta="unused")
    f0 = float(g["freqs"][0])
    v = fp.calculate_Fp(f0, *_args(g))
    assert np.ndim(v) == 0 and abs(v / g["ref_fp"][0] - 1) < 1e-12
    assert fp.compute_Fp(f0, *_args(g)) == v == fp(f0, *_args(g))
    fn = fastfp_b200.vmap(fp.calculate_Fp, in_axes=(0, None, None, None))  # examples/run_fp.py:63
    np.testing.assert_array_equal(fn(g["freqs"], *_args(g)), fp(g["freqs"], *_args(g)))


def test_get_xcy_matches_reference(golden):
    g = golden("fp_white")
    for p in range(g.P):
        v = fastfp_b200.get_xCy(g[f"Nvec_{p}"], g[f"T_{p}"], g[f"sigma_{p}"], g[f"x_{p}"], g[f"y_{p}"])
        tv, cond = truth.get_xCy_truth(g[f"Nvec_{p}"], g[f"T_{p}"], g[f"sigma_{p}"], g[f"x_{p}"], g[f"y_{p}"])
        assert abs(v - g["ref_xcy"][p]) <= 1e-10 * abs(g["ref_xcy"][p]) + 64 * EPS * cond


def test_get_xcy_general_sigma_uses_pivoted_lu():
    """jnp.linalg.solve semantics: Sigma need not be positive definite (utils.py:54)."""
    rng = np.random.default_rng(5)
    n, m = 200, 9
    T, Nvec = rng.standard_normal((n, m)), rng.uniform(0.5, 2, n)
    sigma = rng.standard_normal((m, m))  # indefinite, non-symmetric
    x, y = rng.standard_normal(n), rng.standard_normal(n)
    want = o.get_xCy(Nvec, T, sigma, x, y)
    assert abs(fastfp_b200.get_xCy(Nvec, T, sigma, x, y) - want) < 1e-9 * abs(want) + 1e-9


# every kernel configuration family: m <= 40, <= 80, <= 160, <= 320, <= 640 (fp_sweep.cu::sweep_config)
@pytest.mark.parametrize("n_tm,ncomps", [(2, 0), (5, 3), (12, 30), (20, 30), (9, 45), (40, 55), (150, 45), (230, 40),
                                         (340, 30), (500, 60)])
def test_every_kernel_family_against_oracle(n_tm, ncomps):
    m_ = n_tm + 2 * ncomps
    # ragged, not multiples of the chunk size; comfortably more TOAs than basis columns
    ns = [333, 64, 1000] if m_ <= 40 else ([333, 300, 1000] if m_ <= 160 else ([2500, 1801, 3000] if m_ <= 320
                                                                          else [4000, 3001, 5000]))
    if ncomps == 0:
        pta = synth.make_pta(3, ns, n_tm=n_tm, white_only=True, seed=77)
    else:
        pta = synth.make_pta(3, ns, n_tm=n_tm, ncomps=ncomps, seed=77)
    m = pta.Ts[0].shape[1]
    k = np.array([1.0, 2.5, 7.0])
    freqs = np.concatenate((synth.fp_freqs(70), k / pta.Tspan))  # 73: not a multiple of any tile
    fp = fastfp_b200.FastFp(pta.psrs)
    got = fp.per_pulsar_terms(freqs, pta.Nvecs, pta.Ts, pta.sigmas)
    args = (freqs, pta.toas, pta.residuals, pta.Nvecs, pta.Ts, pta.sigmas)
    ora = o.fp_sweep(*args, per_pulsar=True)
    tt, cond = truth.fp_sweep_truth(*args)
    tol = term_tolerance(tt.astype(float), cond, ora)
    assert got.shape == (3, 73), m
    ratio = np.abs(got - tt.astype(float)) / tol
    # a bin whose conditioning figure times eps reaches the size of the term itself carries no digits in the
    # reference formula either (the 2x2 system is numerically singular there: the wide-basis cases put a red-noise
    # Fourier frequency on top of ~600 fitted columns); the linear error envelope does not apply to it
    defined = EPS * cond < 0.05 * np.abs(tt.astype(float))
    assert defined.mean() > 0.9
    ratio = np.where(defined, ratio, 0.0)
    worst = np.unravel_index(np.argmax(ratio), ratio.shape)
    assert np.all(ratio <= 1), (f"m={m}: worst |got - truth| / tol = {ratio.max():.3g} at (pulsar, bin) {worst}: got "
                                f"{got[worst]:.6g}, truth {float(tt[worst]):.6g}, oracle {ora[worst]:.6g}, cond {cond[worst]:.3g}")
    np.testing.assert_allclose(fp(freqs, pta.Nvecs, pta.Ts, pta.sigmas), got[0] + got[1] + got[2], rtol=1e-15)


def test_mixed_widths_in_one_pack_and_pulsar_order_of_the_sum():
    pta = synth.make_pta(4, [100, 257, 64, 500], n_tm=[3, 12, 30, 8], ncomps=30, seed=5)
    assert len({T.shape[1] for T in pta.Ts}) == 4
    freqs = synth.fp_freqs(9)
    fp = fastfp_b200.FastFp(pta.psrs)
    terms = fp.per_pulsar_terms(freqs, pta.Nvecs, pta.Ts, pta.sigmas)
    acc = np.zeros(9)
    for p in range(4):  # sequential pulsar sum starting from 0 (fastfp.py:71,90)
        acc = acc + terms[p]
    np.testing.assert_array_equal(fp(freqs, pta.Nvecs, pta.Ts, pta.sigmas), acc)
    ora = o.fp_sweep(freqs, pta.toas, pta.residuals, pta.Nvecs, pta.Ts, pta.sigmas)
    assert np.abs(acc / ora - 1).max() < 1e-7  # loose sanity; tight checks are per family above


def test_edge_cases_nan_semantics_and_large_phase():
    pta = synth.make_pta(2, [48, 100], n_tm=4, ncomps=6, seed=9)
    fp = fastfp_b200.FastFp(pta.psrs)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    out = fp(np.array([0.0, -1e-8, 1e-8]), *a)
    assert np.isnan(out[0]) and np.isnan(out[1]) and np.isfinite(out[2])  # f <= 0 -> NaN like f**(1/3)
    assert fp(np.zeros(0), *a).shape == (0,)
    one = fp(np.array([3e-8]), *a)
    assert one.shape == (1,) and one[0] == fp(3e-8, *a)
    # phases beyond the Cody-Waite range (|phi| > 1e5 rad) take the library sincos path
    fbig = np.array([5e-5, 1.2345e-4])
    ora = o.fp_sweep(fbig, pta.toas, pta.residuals, *a)
    assert np.abs(fp(fbig, *a) / ora - 1).max() < 1e-9
    # NaN in the data propagates silently (no exception), as in the reference
    bad = [r.copy() for r in pta.residuals]
    bad[0][3] = np.nan
    psrs = [Psr(q.toas, r) for q, r in zip(pta.psrs, bad)]
    assert np.isnan(fastfp_b200.FastFp(psrs)(1e-8, *a))


def test_device_resident_call_and_determinism():
    import torch

    pta = synth.make_pta(3, 700, n_tm=12, ncomps=30, seed=21)
    fp = fastfp_b200.FastFp(pta.psrs)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    f = synth.fp_freqs(257)
    host = fp(f, *a)
    dev = fp(torch.tensor(f, dtype=torch.float64, device="cuda"), *a)
    assert dev.is_cuda and dev.dtype == torch.float64
    np.testing.assert_array_equal(dev.cpu().numpy(), host)  # same kernels, same bits
    np.testing.assert_array_equal(fp(f, *a), host)  # run-to-run deterministic
    with pytest.raises(TypeError):
        fp(torch.tensor(f, dtype=torch.float32, device="cuda"), *a)
    assert _cabi.kernel_launches() > 0


@pytest.mark.parametrize("cfg,F", [("C2", 4096)])
def test_full_size_properties(cfg, F):
    """At BASELINE config size the oracle is too slow for every bin: size-independent properties
    plus an oracle/truth spot check."""
    pta = synth.make_config(cfg)
    freqs = synth.fp_freqs(10_000)[:: 10_000 // F][:F]
    fp = fastfp_b200.FastFp(pta.psrs)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    base = fp(freqs, *a)
    assert np.all(np.isfinite(base)) and base.min() > 0  # M is positive definite: Fp > 0
    # quadratic in the residuals: r -> 2 r gives exactly 4 Fp (power-of-two scaling is exact)
    psr2 = [Psr(q.toas, 2.0 * q.residuals) for q in pta.psrs]
    np.testing.assert_array_equal(fastfp_b200.FastFp(psr2)(freqs, *a), 4.0 * base)
    # noise-only data: 2 Fp ~ chi^2 with 2P degrees of freedom (examples/run_fp.ipynb:136-140),
    # checked on the part of the grid above the red-noise band
    hi = freqs > 35.0 / pta.Tspan
    mean = 2.0 * base[hi].mean()
    assert abs(mean - 2 * pta.P) < 0.15 * 2 * pta.P
    # spot check against oracle + truth on a few bins of three pulsars
    idx = np.array([0, 1, 17, F // 2, F - 1])
    sub = slice(10, 13)
    args = (freqs[idx], pta.toas[sub], pta.residuals[sub], pta.Nvecs[sub], pta.Ts[sub], pta.sigmas[sub])
    ora = o.fp_sweep(*args, per_pulsar=True)
    tt, cond = truth.fp_sweep_truth(*args)
    got = fp.per_pulsar_terms(freqs[idx], *a)[sub]
    assert np.all(np.abs(got - tt.astype(float)) <= term_tolerance(tt.astype(float), cond, ora))


@pytest.mark.parametrize("n,m", [(37, 3), (1000, 72), (5003, 150)])
def test_device_tnt_and_sigma(n, m):
    """T^T N^-1 T (+ diag phiinv) on the device (SURVEY 8f-f2) against NumPy; deterministic."""
    rng = np.random.default_rng(n + m)
    T, Nvec = rng.standard_normal((n, m)), rng.uniform(0.5, 2.0, n) * 1e-13
    ph = rng.uniform(1.0, 1e6, m)
    want = T.T @ (T / Nvec[:, None])
    scale = np.sqrt(np.outer(np.diag(want), np.diag(want)))
    got = fastfp_b200.compute_TNTs([Nvec], [T])[0]
    assert np.abs(got - want).max() <= 64 * EPS * scale.max()
    np.testing.assert_array_equal(got, got.T)
    np.testing.assert_array_equal(got, fastfp_b200.compute_TNTs([Nvec], [T])[0])
    sig = fastfp_b200.compute_sigmas([Nvec], [T], [ph])[0]
    np.testing.assert_array_equal(sig, got + np.diag(ph))


def test_pack_from_device_built_sigmas_matches_goldens(golden):
    """The whole precompute on the device: Sigma from the raw (Nvec, T, phiinv), then the sweep. Sigma
    differs from the golden one by summation-order rounding only, so the result stays inside the same
    envelope as the direct test above."""
    g = golden("fp_red")
    Nvecs, Ts, sigmas = _args(g)
    phiinvs = [np.diag(s) - np.diag(T.T @ (T / N[:, None])) for s, T, N in zip(sigmas, Ts, Nvecs)]
    sig = fastfp_b200.compute_sigmas(Nvecs, Ts, phiinvs)
    for a, b in zip(sig, sigmas):
        assert np.abs(a - b).max() <= 256 * EPS * np.abs(b).max()
    got = fastfp_b200.FastFp(g.psrs)(g["freqs"], Nvecs, Ts, sig)
    ora_terms = o.fp_sweep(g["freqs"], g.lst("toas"), g.lst("res"), Nvecs, Ts, sigmas, per_pulsar=True)
    tol = term_tolerance(g["truth_terms"], g["cond"], ora_terms)
    assert np.all(np.abs(got - g["ref_fp"]) <= 1e-10 * np.abs(g["ref_fp"]) + 4 * tol.sum(0))


def test_in_place_edit_of_the_inputs_rebuilds_the_pack():
    """ADVICE r1: the reference is a pure function of its arguments; an in-place change of ANY entry of the
    lists must be seen (the cache key hashes every byte), not answered from a stale device pack."""
    pta = synth.make_pta(2, [500, 700], n_tm=6, ncomps=10, seed=2)
    f = synth.fp_freqs(40)
    fp = fastfp_b200.FastFp(pta.psrs)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    base = fp(f, *a)
    np.testing.assert_array_equal(fp(f, *a), base)
    pta.Nvecs[1][123] *= 1.5  # one TOA re-weighted in place: misses any sparse content sample
    pta.sigmas[1][:] = pta.Ts[1].T @ (pta.Ts[1] / pta.Nvecs[1][:, None]) + np.diag(1.0 / pta.phis[1])
    edited = fp(f, *a)
    fresh = fastfp_b200.FastFp(pta.psrs)(f, *a)
    np.testing.assert_array_equal(edited, fresh)
    assert np.abs(edited / base - 1).max() > 1e-6
    fp.invalidate()
    np.testing.assert_array_equal(fp(f, *a), fresh)
    np.testing.assert_array_equal(fp.prepare(*a, force=True).fp_sweep(f), fresh)


def test_non_spd_sigma_is_reported_and_propagates_nan():
    """ADVICE r1: the sweep path factorises Sigma = L L^T; a Sigma that is not numerically SPD gives NaN for
    that pulsar (like a singular Sigma in the reference) and the pack says which pulsar and pivot."""
    pta = synth.make_pta(2, [300, 300], n_tm=4, ncomps=5, seed=6)
    bad = [pta.sigmas[0], pta.sigmas[1].copy()]
    bad[1][3, 3] = -abs(bad[1][3, 3])
    fp = fastfp_b200.FastFp(pta.psrs)
    with pytest.warns(RuntimeWarning, match=r"pulsar\(s\) 1 \(pivot 3\)"):
        out = fp.per_pulsar_terms(synth.fp_freqs(5), pta.Nvecs, pta.Ts, bad)
    assert np.all(np.isfinite(out[0])) and np.all(np.isnan(out[1]))
    assert fp.prepare(pta.Nvecs, pta.Ts, bad).factor_info() == [0, 4]
