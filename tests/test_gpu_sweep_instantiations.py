"""Every launchable instantiation of the fp64 sweep kernel on the GPU, against the longdouble truth of oracle/truth.py:
the 145 (mode, N kind, configuration) cases of tests/test_sweep_instantiations_host.py::CASES, one pulsar each, at
the flush edges of its TOA count, over one frequency grid with f <= 0, bins far past the Cody-Waite range and bins on
both sides of every pulsar's cold-path threshold inside one tile (sweep_freqs). Failures name the configuration, e.g.
"xwide/NMBW 8, m = 488, n = 1543". Run with -m gpu on an H100; each test prints the worst |got - truth| / tol of its
(mode, N kind) and the configuration it occurred at."""
from types import SimpleNamespace

import numpy as np
import pytest

import fastfp_b200
from conftest import EPS, term_tolerance
from fastfp_b200 import NMFP, RN_container, synth
from fastfp_b200.fe import antenna_pattern
from oracle import fp_oracle as o
from oracle import truth
from test_gpu_blockn_families import _blocks
from test_gpu_fp_batch import realisations
from test_sweep_instantiations_host import CASES, NNB, assert_near_threshold, label, split, sweep_freqs

pytestmark = pytest.mark.gpu

D = 2  # draws of every noise-marginalised case


def _set(cases, mode, seed):
    """One synthetic pulsar per case (its own TOAs, basis width c.m, c.n TOAs), as the lists of a PTA."""
    ptas = []
    for i, c in enumerate(cases):
        n_tm, nc = split(c.m, mode)
        pta = synth.make_pta(1, c.n, n_tm=n_tm, ncomps=max(nc, 1), white_only=nc == 0, seed=seed + 7 * i)
        assert pta.Ts[0].shape == (c.n, c.m), label(c)
        ptas.append(pta)
    s = SimpleNamespace(**{k: [getattr(p, k)[0] for p in ptas]
                           for k in ("psrs", "toas", "residuals", "Nvecs", "Ts", "TNTs", "phis", "sigmas", "n_tm")})
    s.Ffreqs = [p.Ffreqs for p in ptas]
    s.P = len(ptas)
    s.freqs = sweep_freqs(max(p.Tspan for p in ptas), [t.max() for t in s.toas])
    assert_near_threshold(s.freqs, [t.max() for t in s.toas], [c.fam for c in cases])
    s.pos = s.freqs > 0
    return s


def _ratio(got, tv, tol, cond):
    """|got - truth| / tol on the bins where the reference formula carries digits (0 elsewhere); at least 90% do."""
    defined = EPS * cond < 0.05 * np.abs(tv)
    assert defined.mean() > 0.9, defined.mean()
    return np.where(defined, np.abs(got - tv) / tol, 0.0)


def _report(what, ratios, labels):
    """Assert every case's worst ratio is at most 1, naming the configuration; print the worst of them all."""
    worst = [float(r.max()) for r in ratios]
    bad = [f"{lb}: {w:.3g}" for lb, w in zip(labels, worst) if not w <= 1]
    i = int(np.argmax(worst))
    print(f"\n[{what}] worst |got - truth| / tol = {worst[i]:.3g} at {labels[i]}")
    assert not bad, f"{what}: worst |got - truth| / tol above 1 at " + "; ".join(bad)


def _assert_nan_at_nonpositive(got, s, what):
    assert np.all(np.isnan(got[..., ~s.pos])), what
    assert np.all(np.isfinite(got[..., s.pos])), what


def _ordered_sum(rows):
    acc = np.zeros(rows[0].shape)
    for r in rows:  # pulsar order from 0 (fastfp.py:71,90)
        acc = acc + r
    return acc


# ---- Fp, diagonal N: one 26-pulsar pack --------------------------------------------------------------------------

@pytest.fixture(scope="module")
def fp_diag():
    cases = CASES[("fp", "diag")]
    s = _set(cases, "fp", seed=10_000)
    a = (s.Nvecs, s.Ts, s.sigmas)
    fp = fastfp_b200.FastFp(s.psrs, path="fp64")
    assert fp.prepare(*a).path == "fp64"
    got = fp.per_pulsar_terms(s.freqs, *a)
    inner = truth.sweep_inner_truth(s.freqs[s.pos], s.toas, s.residuals, *a)
    ora = o.fp_sweep(s.freqs[s.pos], s.toas, s.residuals, *a, per_pulsar=True)
    return SimpleNamespace(cases=cases, s=s, a=a, fp=fp, got=got, inner=inner, ora=ora)


def test_fp_diagonal_against_truth(fp_diag):
    d = fp_diag
    _assert_nan_at_nonpositive(d.got, d.s, "Fp, diagonal N")
    tt, cond = truth.terms_truth(d.inner)
    tv = tt.astype(float)
    ratio = _ratio(d.got[:, d.s.pos], tv, term_tolerance(tv, cond, d.ora), cond)
    _report("Fp, diagonal N", list(ratio), [label(c) for c in d.cases])


def test_fp_diagonal_bit_identities(fp_diag):
    """Each pulsar's row is that of the pulsar swept alone; the statistic is the ordered pulsar sum; a bin's value
    does not depend on where in a tile it lands (odd-shifted slices of the bins below every cold-path threshold)."""
    d = fp_diag
    s = d.s
    for p, c in enumerate(d.cases):
        one = fastfp_b200.FastFp([s.psrs[p]], path="fp64").per_pulsar_terms(
            s.freqs, [s.Nvecs[p]], [s.Ts[p]], [s.sigmas[p]])
        np.testing.assert_array_equal(one[0], d.got[p], err_msg=label(c))
    np.testing.assert_array_equal(d.fp(s.freqs, *d.a), _ordered_sum(d.got))
    for lo, hi in ((3, 70), (37, 38), (1, 88), (85, 88), (11, 44)):
        np.testing.assert_array_equal(d.fp.per_pulsar_terms(s.freqs[lo:hi], *d.a), d.got[:, lo:hi],
                                      err_msg=f"bins {lo}:{hi}")


def test_fe_diagonal_against_truth(fp_diag):
    """calculate_Fe at three sky positions: all five inner products of every configuration, through the Fe truth of
    the same longdouble inner products (rule of test_gpu_fe_truth.py)."""
    d = fp_diag
    s = d.s
    rng = np.random.default_rng(5)
    th, ph = np.arccos(rng.uniform(-1, 1, 3)), rng.uniform(0, 2 * np.pi, 3)
    got = fastfp_b200.FastFe(s.psrs, path="fp64").calculate_Fe(s.freqs, th, ph, *d.a)
    _assert_nan_at_nonpositive(got, s, "Fe")
    fplus, fcross = antenna_pattern(np.stack([q.pos for q in s.psrs]), th, ph)
    fe, cond = truth.fe_truth_from_inner(d.inner, s.freqs[s.pos], fplus, fcross)
    tt, tc = truth.terms_truth(d.inner)
    E = (term_tolerance(tt.astype(float), tc, d.ora, k_oracle=1.0, rel=0.0) / (EPS * tc)).max()
    tv = fe.astype(float)
    ratio = _ratio(got[:, s.pos], tv, 1e-10 * np.abs(tv) + 4 * E * EPS * cond, cond)
    _report("Fe, diagonal N", list(ratio), [f"sky position {k}" for k in range(3)])


# ---- Fp, block-diagonal N: one 24-pulsar pack --------------------------------------------------------------------

def _blockn_rule(tv, cond):
    return 1e-10 * np.abs(tv) + 256 * EPS * cond  # test_gpu_blockn_families.py::_assert_near_truth


def test_fp_block_n_against_truth():
    cases = CASES[("fp", "blockn")]
    s = _set(cases, "fp", seed=20_000)
    Nvecs, tblocks, TNTs = _blocks(s, np.random.default_rng(20))
    sig = [TNT + np.diag(1.0 / phi) for TNT, phi in zip(TNTs, s.phis)]
    fp = fastfp_b200.FastFp(s.psrs, path="fp64")
    assert fp.prepare(Nvecs, s.Ts, sig).blockn
    got = fp.per_pulsar_terms(s.freqs, Nvecs, s.Ts, sig)
    _assert_nan_at_nonpositive(got, s, "Fp, block-N")
    tt, cond = truth.fp_sweep_truth_blockn(s.freqs[s.pos], s.toas, s.residuals, tblocks, s.Ts, sigmas=sig)
    tv = tt.astype(float)
    ratio = _ratio(got[:, s.pos], tv, _blockn_rule(tv, cond), cond)
    _report("Fp, block-N", list(ratio), [label(c) for c in cases])
    np.testing.assert_array_equal(fp(s.freqs, Nvecs, s.Ts, sig), _ordered_sum(got))


# ---- residual batches: single-pulsar packs, then one pack of them all ------------------------------------------------

_RES = {}


def _res_set(kind):
    """The residual-batch pulsars of one N kind, their realisations and each one's calculate_Fp_batch alone."""
    if kind not in _RES:
        cases = CASES[("res", kind)]
        s = _set(cases, "res", seed=30_000 if kind == "diag" else 40_000)
        if kind == "blockn":
            s.Nvecs_in, s.tblocks, TNTs = _blocks(s, np.random.default_rng(40), diagonal=())
            s.sig = [TNT + np.diag(1.0 / phi) for TNT, phi in zip(TNTs, s.phis)]
        else:
            s.Nvecs_in, s.sig = s.Nvecs, s.sigmas
        s.res = realisations(s, cases[0].R, seed=31)
        s.single = [fastfp_b200.FastFp([s.psrs[p]], path="fp64").calculate_Fp_batch(
            s.freqs, [s.Nvecs_in[p]], [s.Ts[p]], [s.sig[p]], [s.res[p]]) for p in range(s.P)]
        _RES[kind] = (cases, s)
    return _RES[kind]


@pytest.mark.parametrize("fam", list(NNB))
@pytest.mark.parametrize("kind", ["diag", "blockn"])
def test_residual_batch_against_truth(kind, fam):
    """Every realisation row of every configuration of a family against the truth for that row's residuals (rules of
    test_gpu_fp_batch.py::assert_rows_near_truth and test_gpu_blockn_batch.py::_assert_rows)."""
    cases, s = _res_set(kind)
    ratios, labels = [], []
    for p, c in enumerate(cases):
        if c.fam != fam:
            continue
        got = s.single[p]
        assert got.shape == (c.R, s.freqs.shape[0])
        _assert_nan_at_nonpositive(got, s, label(c))
        for k in range(c.R):
            args = (s.freqs[s.pos], [s.toas[p]], [s.res[p][k]])
            if kind == "diag":
                a = args + ([s.Nvecs[p]], [s.Ts[p]], [s.sigmas[p]])
                tt, cond = truth.fp_sweep_truth(*a)
                tv = tt.astype(float)
                tol = term_tolerance(tv, cond, o.fp_sweep(*a, per_pulsar=True))
            else:
                tt, cond = truth.fp_sweep_truth_blockn(*args, [s.tblocks[p]], [s.Ts[p]], sigmas=[s.sig[p]])
                tv = tt.astype(float)
                tol = _blockn_rule(tv, cond)
            ratios.append(_ratio(got[k][s.pos], tv[0], tol[0], cond[0]))
            labels.append(f"{label(c)}, row {k}")
    _report(f"Res, {kind} N, {fam}", ratios, labels)


@pytest.mark.parametrize("kind", ["diag", "blockn"])
def test_residual_batch_pack_is_the_ordered_sum(kind):
    """A pack of all the pulsars returns the ordered pulsar sum, from 0.0, of their single-pulsar batches, bit for
    bit (reduce_terms_rows_kernel)."""
    cases, s = _res_set(kind)
    got = fastfp_b200.FastFp(s.psrs, path="fp64").calculate_Fp_batch(s.freqs, s.Nvecs_in, s.Ts, s.sig, s.res)
    np.testing.assert_array_equal(got, _ordered_sum(s.single))


# ---- noise-marginalised Fp: single-pulsar packs, two draws ---------------------------------------------------------

_NM = {}


def _nm_set(kind):
    if kind not in _NM:
        cases = CASES[("nmfp", kind)]
        s = _set(cases, "nmfp", seed=50_000 if kind == "diag" else 60_000)
        if kind == "blockn":
            s.Nvecs_in, s.tblocks, s.TNT_in = _blocks(s, np.random.default_rng(60), diagonal=())
        else:
            s.Nvecs_in, s.TNT_in = s.Nvecs, s.TNTs
        _NM[kind] = (cases, s)
    return _NM[kind]


@pytest.mark.parametrize("fam", list(NNB))
@pytest.mark.parametrize("kind", ["diag", "blockn"])
def test_nmfp_against_truth(kind, fam):
    """Both draws of every configuration of a family against the truth with that draw's Sigma (rule of
    test_gpu_blockn_families.py::test_block_n_nmfp_in_every_family); the timing model is the fixed block."""
    cases, s = _nm_set(kind)
    ratios, labels = [], []
    for p, c in enumerate(cases):
        if c.fam != fam:
            continue
        q = s.psrs[p]
        samples = synth.draw_samples(SimpleNamespace(psrs=[q]), D, seed=70 + p)
        nm = NMFP([q], [RN_container(q, Ffreqs=s.Ffreqs[p])], path="fp64")
        got = nm(s.freqs, samples, [s.Nvecs_in[p]], [s.Ts[p]], [s.TNT_in[p]])
        assert got.shape == (D, s.freqs.shape[0])
        assert nm.prepare([s.Nvecs_in[p]], [s.Ts[p]], [s.TNT_in[p]]).mvar_total == c.m - s.n_tm[p]
        _assert_nan_at_nonpositive(got, s, label(c))
        phi_args = [dict(psr_name=q.name, n_tm=s.n_tm[p], Ffreqs=s.Ffreqs[p])]
        for d in range(D):
            sig = o.get_sigmas({k: v[d] for k, v in samples.items()}, [s.TNT_in[p]], phi_args)
            args = (s.freqs[s.pos], [s.toas[p]], [s.residuals[p]])
            if kind == "diag":
                tt, cond = truth.fp_sweep_truth(*args, [s.Nvecs[p]], [s.Ts[p]], sig)
            else:
                tt, cond = truth.fp_sweep_truth_blockn(*args, [s.tblocks[p]], [s.Ts[p]], sigmas=sig)
            tv = tt[0].astype(float)
            ratios.append(_ratio(got[d][s.pos], tv, _blockn_rule(tv, cond[0]), cond[0]))
            labels.append(f"{label(c)}, draw {d}")
    _report(f"Nmfp, {kind} N, {fam}", ratios, labels)
