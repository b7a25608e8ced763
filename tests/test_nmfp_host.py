"""Host-side containers of the noise-marginalised path against the reference goldens, and the truth figures its GPU
tests use (CPU)."""
import numpy as np
import pytest

import fastfp_b200
from conftest import Psr
from fastfp_b200 import NMFP, CURN_container, GPEcorr_container, RN_container, synth
from oracle import truth


def _samples(g):
    return {k[len("sample__"):]: g[k] for k in g.g.files if k.startswith("sample__")}


def test_containers_reproduce_reference_phi(golden):
    g = golden("nmfp")
    samples = _samples(g)
    pars0 = {k: v[0] for k, v in samples.items()}
    psrs = g.psrs
    curn = CURN_container(g["Ffreqs_curn"])
    np.testing.assert_array_equal(curn.get_phi_curn(pars0), g["ref_curn_phi0"])
    np.testing.assert_array_equal(curn.get_phiinv(pars0), 1.0 / g["ref_curn_phi0"])
    plain = [RN_container(q, Ffreqs=g["Ffreqs"]) for q in psrs]
    np.testing.assert_array_equal(np.concatenate([o.update_phi(pars0) for o in plain]), g["ref_phi0_plain"])
    with_curn = [RN_container(q, Ffreqs=g["Ffreqs"], add_curn=True, curn_container=curn) for q in psrs]
    np.testing.assert_array_equal(np.concatenate([o.get_phiinv(pars0) for o in with_curn]), g["ref_phiinv0"])
    assert plain[0].phi_fn == plain[0].get_phi_tm_rn and with_curn[0].phi_fn == with_curn[0].get_phi_tm_rn_curn
    # batched parameters give one row per draw
    batch = with_curn[1].get_phiinv(samples)
    assert batch.shape == (int(g["D"]), int(g["ntm_1"]) + g["Ffreqs"].shape[0])
    np.testing.assert_array_equal(batch[0], with_curn[1].get_phiinv(pars0))
    # default frequency grid from the pulsar's own span (nmfp.py:201-215)
    own = RN_container(psrs[0], ncomps=4)
    span = psrs[0].toas.max() - psrs[0].toas.min()
    np.testing.assert_array_equal(own.Ffreqs, np.repeat(np.arange(1, 5) / span, 2))


def test_gp_ecorr_layouts(golden):
    g = golden("nmfp")
    pars0 = {k: v[0] for k, v in _samples(g).items()}
    q = g.psrs[0]
    q.backend_flags = np.array(["A"] * 100 + ["B"] * (q.toas.size - 100))
    weights = [np.ones(int(k)) for k in g["ecorr_nw"]]
    wn = {f"{q.name}_basis_ecorr_A_log10_ecorr": float(g["ecorr_log10"][0]),
          f"{q.name}_basis_ecorr_B_log10_ecorr": float(g["ecorr_log10"][1])}
    ec = GPEcorr_container(q, weights, fix_wn_vals=wn)
    np.testing.assert_array_equal(ec.get_phi(pars0), g["ref_ecorr_phi"])
    curn = CURN_container(g["Ffreqs_curn"])
    a = RN_container(q, Ffreqs=g["Ffreqs"], gp_ecorr=True, ecorr_container=ec)
    b = RN_container(q, Ffreqs=g["Ffreqs"], gp_ecorr=True, ecorr_container=ec, add_curn=True, curn_container=curn)
    np.testing.assert_array_equal(a.update_phi(pars0), g["ref_phi_tm_ecorr_rn"])
    np.testing.assert_array_equal(b.update_phi(pars0), g["ref_phi_tm_ecorr_rn_curn"])
    assert a.fixed_phi().shape[0] == int(g["ntm_0"]) + int(g["ecorr_nw"].sum())


def test_get_sigmas_matches_reference(golden):
    g = golden("nmfp")
    pars0 = {k: v[0] for k, v in _samples(g).items()}
    curn = CURN_container(g["Ffreqs_curn"])
    sigs = [RN_container(q, Ffreqs=g["Ffreqs"], add_curn=True, curn_container=curn) for q in g.psrs]
    nm = NMFP(g.psrs, sigs)
    for p, s in enumerate(nm._get_sigmas(pars0, g.lst("TNT"))):
        np.testing.assert_array_equal(s, g[f"ref_sigma0_{p}"])


def test_layout_mismatch_is_reported_before_device_work(golden):
    g = golden("nmfp")
    sigs = [RN_container(q, Ffreqs=g["Ffreqs"][:-2]) for q in g.psrs]  # two entries short
    with pytest.raises(ValueError, match="basis has"):
        NMFP(g.psrs, sigs).prepare(g.lst("Nvec"), g.lst("T"), g.lst("TNT"))


def test_powerlaw_phiinv_truth_matches_reference_phiinv(golden):
    """The longdouble power-law truth against the reference's float64 ``get_phiinv`` (goldens): within a few ulp,
    each draw's row, with and without the common process on the leading entries."""
    g = golden("nmfp")
    samples = _samples(g)
    curn = CURN_container(g["Ffreqs_curn"])
    q = g.psrs[1]
    sig = RN_container(q, Ffreqs=g["Ffreqs"], add_curn=True, curn_container=curn)
    ntm = sig.tm_weights.shape[0]
    want = sig.get_phiinv(samples)[:, ntm:]
    got = truth.powerlaw_phiinv_truth(sig.Ffreqs, samples[sig.rn_A_name], samples[sig.rn_gam_name], curn.Ffreqs,
                                      samples["gw_log10_A"], samples["gw_gamma"])
    assert got.dtype == np.longdouble and got.shape == want.shape
    assert np.abs(got.astype(float) / want - 1).max() < 16 * 2.0**-52
    plain = truth.powerlaw_phiinv_truth(sig.Ffreqs, samples[sig.rn_A_name], samples[sig.rn_gam_name])
    want_plain = RN_container(q, Ffreqs=g["Ffreqs"]).get_phiinv(samples)[:, ntm:]
    assert np.abs(plain.astype(float) / want_plain - 1).max() < 16 * 2.0**-52
    # the common process only adds to the leading entries
    nc = curn.Ffreqs.shape[0]
    assert np.all(got[:, :nc] < plain[:, :nc])
    np.testing.assert_array_equal(got[:, nc:], plain[:, nc:])


def test_sigma_cond_truth_bounds_a_cholesky_backward_error():
    """``sigma_cond_truth`` is a first-order bound: replacing Sigma by Sigma + dSigma with |dSigma| = delta |L| |L^T|
    (random signs, symmetric) moves each longdouble term by at most delta * cond_Sigma, and the bound is not loose by
    orders of magnitude."""
    pta = synth.make_pta(2, [150, 170], ncomps=10, seed=5)
    freqs = np.concatenate((synth.nmfp_freqs(3, pta.Tspan), synth.fp_freqs(6)))
    args = (freqs, pta.toas, pta.residuals, pta.Nvecs, pta.Ts)
    base, _ = truth.fp_sweep_truth(*args, pta.sigmas)
    cs = truth.sigma_cond_truth(*args, pta.sigmas)
    delta, rng, worst = 1e-12, np.random.default_rng(0), np.zeros_like(cs)
    for _ in range(4):
        pert = []
        for S in pta.sigmas:
            L = np.linalg.cholesky(S)
            sgn = np.triu(rng.choice([-1.0, 1.0], S.shape))
            sgn = sgn + np.triu(sgn, 1).T
            pert.append(S.astype(np.longdouble) + delta * sgn * (np.abs(L) @ np.abs(L).T))
        moved, _ = truth.fp_sweep_truth(*args, pert)
        worst = np.maximum(worst, np.abs(moved - base).astype(float))
    assert np.all(worst <= 1.01 * delta * cs), (worst / (delta * cs)).max()
    assert (worst / (delta * cs)).max() > 1e-3
