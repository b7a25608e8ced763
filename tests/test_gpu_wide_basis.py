"""Bases wider than one work item of the sweep kernel (640 G rows), swept as row groups of G and combined (DESIGN.md
section 5h), on the GPU: each width against the longdouble truth, the reference's GP-ECORR layout against the block-N
pack of the same model, mixed packs bit for bit against packs without the other pulsars, the Fe-statistic, the edge
cases and the refusals. Run with -m gpu on an H100."""
import numpy as np
import pytest

import fastfp_b200
from conftest import EPS, term_tolerance
from fastfp_b200 import _cabi, synth
from fastfp_b200.fe import antenna_pattern
from oracle import fp_oracle as o
from oracle import truth

pytestmark = pytest.mark.gpu

NCOMPS = 30


def _freqs(pta):
    """73 bins (a ragged tile) including the 1, 2.5 and 7 / Tspan red-noise bins."""
    return np.concatenate((synth.fp_freqs(70), np.array([1.0, 2.5, 7.0]) / pta.Tspan))


def _assert_terms(got, tt, cond, ora, what):
    """The rule of test_gpu_fp.py::test_every_kernel_family_against_oracle: within term_tolerance of the truth on every
    bin where the reference formula itself carries digits."""
    tv = tt.astype(float)
    tol = term_tolerance(tv, cond, ora)
    defined = EPS * cond < 0.05 * np.abs(tv)
    assert defined.mean() > 0.9, (what, defined.mean())
    ratio = np.where(defined, np.abs(got - tv) / tol, 0.0)
    worst = np.unravel_index(np.argmax(ratio), ratio.shape)
    assert np.all(ratio <= 1), (f"{what}: worst |got - truth| / tol = {ratio.max():.3g} at (pulsar, bin) {worst}: got "
                                f"{got[worst]:.6g}, truth {float(tt[worst]):.6g}, cond {cond[worst]:.3g}")


def _ordered_sum(terms):
    acc = np.zeros(terms.shape[1])
    for t in terms:  # pulsar order from 0 (fastfp.py:71,90)
        acc = acc + t
    return acc


# m = 641 (three groups), ~700 (three, ragged n over two pulsars), ~1000 (four), ~1300 (five), near the maximum (ten)
@pytest.mark.parametrize("n_tm,n", [(581, [900]), (640, [1000, 777]), (940, [1301]), (1240, [1611]),
                                    (2620, [2803])])
def test_widths_against_truth(n_tm, n):
    pta = synth.make_pta(len(n), n, n_tm=n_tm, ncomps=NCOMPS, seed=311)
    m = n_tm + 2 * NCOMPS
    assert pta.Ts[0].shape[1] == m and len(_cabi.row_groups(m)) >= 2
    freqs = _freqs(pta)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    fp = fastfp_b200.FastFp(pta.psrs, path="fp64")
    got = fp.per_pulsar_terms(freqs, *a)
    args = (freqs, pta.toas, pta.residuals, *a)
    tt, cond = truth.fp_sweep_truth(*args)
    _assert_terms(got, tt, cond, o.fp_sweep(*args, per_pulsar=True), f"m={m}")
    np.testing.assert_array_equal(fp(freqs, *a), _ordered_sum(got))


def _gp_and_kernel_ecorr():
    pta = synth.make_pta(2, [3200, 2403], n_tm=12, ncomps=NCOMPS, seed=71, epoch=4)
    Nk, Tk, TNTk, phik = synth.with_ecorr(pta, kernel=True)
    Ng, Tg, TNTg, phig = synth.with_ecorr(pta, kernel=False)
    return pta, (Nk, Tk, [t + np.diag(1.0 / f) for t, f in zip(TNTk, phik)]), \
        (Ng, Tg, [t + np.diag(1.0 / f) for t, f in zip(TNTg, phig)])


def test_reference_gp_ecorr_layout_and_its_block_n_pack():
    """The reference's ECORR model (initialize_pta(..., inc_ecorr=True)): epoch-indicator columns in T, m > 640, against
    the same model with a block-diagonal N; both meet the parity bar of the block-N truth."""
    pta, (Nk, Tk, Sk), (Ng, Tg, Sg) = _gp_and_kernel_ecorr()
    assert min(T.shape[1] for T in Tg) > 640 and max(T.shape[1] for T in Tk) <= 632
    freqs = _freqs(pta)
    wide = fastfp_b200.FastFp(pta.psrs).per_pulsar_terms(freqs, Ng, Tg, Sg)
    block = fastfp_b200.FastFp(pta.psrs).per_pulsar_terms(freqs, Nk, Tk, Sk)
    tblocks = [(pta.Nvecs[p], [(s.start, s.stop) for s in B.slices], np.asarray(B.jvec)) for p, B in enumerate(Nk)]
    tt, cond = truth.fp_sweep_truth_blockn(freqs, pta.toas, pta.residuals, tblocks, Tk, sigmas=Sk)
    ora = o.fp_sweep(freqs, pta.toas, pta.residuals, Ng, Tg, Sg, per_pulsar=True)
    _assert_terms(block, tt, cond, ora, "block-N pack")
    _assert_terms(wide, tt, cond, ora, "GP-ECORR basis")


@pytest.fixture(scope="module")
def mixed():
    """Narrow (m = 38, 70, 332) and wide (m = 760, 1130) pulsars, interleaved, ragged n."""
    pta = synth.make_pta(5, [400, 1500, 333, 1700, 901], n_tm=[8, 700, 10, 1070, 272], ncomps=NCOMPS, seed=808)
    return pta


def _sub(pta, idx):
    return ([pta.psrs[p] for p in idx], [pta.Nvecs[p] for p in idx], [pta.Ts[p] for p in idx],
            [pta.sigmas[p] for p in idx])


def test_mixed_pack_is_bit_identical_to_its_parts(mixed):
    pta = mixed
    freqs = _freqs(pta)
    terms = fastfp_b200.FastFp(pta.psrs).per_pulsar_terms(freqs, pta.Nvecs, pta.Ts, pta.sigmas)
    narrow = [p for p in range(pta.P) if pta.Ts[p].shape[1] <= 640]
    assert len(narrow) == 3
    psrs, N, T, S = _sub(pta, narrow)
    np.testing.assert_array_equal(terms[narrow], fastfp_b200.FastFp(psrs).per_pulsar_terms(freqs, N, T, S))
    for p in set(range(pta.P)) - set(narrow):
        psrs, N, T, S = _sub(pta, [p])
        np.testing.assert_array_equal(terms[p], fastfp_b200.FastFp(psrs).per_pulsar_terms(freqs, N, T, S)[0])
    np.testing.assert_array_equal(fastfp_b200.FastFp(pta.psrs)(freqs, pta.Nvecs, pta.Ts, pta.sigmas),
                                  _ordered_sum(terms))


def test_fe_against_truth_and_skymax_rule(mixed):
    from test_gpu_fe_skymax import rule

    pta = mixed
    freqs = _freqs(pta)
    rng = np.random.default_rng(12)
    th, ph = np.arccos(rng.uniform(-1, 1, 24)), rng.uniform(0, 2 * np.pi, 24)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    fe = fastfp_b200.FastFe(pta.psrs)
    fe_map = fe.calculate_Fe(freqs, th, ph, *a)
    fp_, fx_ = antenna_pattern(np.stack([q.pos for q in pta.psrs]), th, ph)
    args = (pta.toas, pta.residuals, *a)
    inner = truth.sweep_inner_truth(freqs, *args)
    want, cond = truth.fe_truth_from_inner(inner, freqs, fp_, fx_)
    tt, tc = truth.terms_truth(inner)
    ora = o.fp_sweep(freqs, *args, per_pulsar=True)
    E = (term_tolerance(tt.astype(float), tc, ora, k_oracle=1.0, rel=0.0) / (EPS * tc)).max()
    tv = want.astype(float)
    tol = 1e-10 * np.abs(tv) + 4 * E * EPS * cond
    defined = EPS * cond < 0.05 * np.abs(tv)
    assert defined.mean() >= 0.9
    assert np.all(np.where(defined, np.abs(fe_map - tv) / tol, 0.0) <= 1)
    got = fe.calculate_Fe_skymax(freqs, th, ph, *a)
    want_max = rule(fe_map)
    np.testing.assert_array_equal(got[0], want_max[0])
    np.testing.assert_array_equal(got[1], want_max[1])


def test_nan_at_nonpositive_frequency_and_repeatability(mixed):
    pta = mixed
    f = np.concatenate(([0.0, -1e-8], synth.fp_freqs(20)))
    pack = fastfp_b200.FastFp(pta.psrs).prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    terms = pack.fp_sweep(f, terms=True)
    assert np.all(np.isnan(terms[:, :2])) and np.all(np.isfinite(terms[:, 2:]))
    # the Fe-statistic reads the five inner products: NaN there, finite elsewhere
    rng = np.random.default_rng(3)
    fe = pack.fe_sweep(f, rng.uniform(-1, 1, (4, pta.P)), rng.uniform(-1, 1, (4, pta.P)))
    assert np.all(np.isnan(fe[:, :2])) and np.all(np.isfinite(fe[:, 2:]))
    np.testing.assert_array_equal(pack.fp_sweep(f, terms=True), terms)
    np.testing.assert_array_equal(pack.fp_sweep(f), pack.fp_sweep(f))


def test_results_do_not_depend_on_the_frequency_batch():
    """A pack of many small pulsars and a wide one: with the terms scratch (P doubles per frequency) and the row-group
    scratch (5 for the wide pulsar's group 0, 3 for each other group) the batches of fp_run hold 2^27 / (P + 5 + 3 (g - 1))
    frequencies, those of the Fe calls 2^27 / (5 P + 5 + 3 (g - 1)); bins on both sides of a boundary equal those of
    calls that take them in one batch."""
    P = 1200
    n = [64] * (P - 1) + [700]
    n_tm = [4] * (P - 1) + [590]
    pta = synth.make_pta(P, n, n_tm=n_tm, ncomps=NCOMPS, seed=4)
    g = len(_cabi.row_groups(pta.Ts[-1].shape[1]))
    FB = 2**27 // (P + 5 + 3 * (g - 1))
    F = FB + 700
    freqs = np.linspace(2e-9, 3e-7, F)
    pack = fastfp_b200.FastFp(pta.psrs).prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    full = pack.fp_sweep(freqs, terms=True)
    lo, hi = FB - 300, FB + 300
    part = pack.fp_sweep(freqs[lo:hi], terms=True)
    np.testing.assert_array_equal(full[:, lo:hi], part)
    np.testing.assert_array_equal(pack.fp_sweep(freqs)[lo:hi], pack.fp_sweep(freqs[lo:hi]))
    # the Fe sweep and its sky maximum, across their own boundary
    FB = 2**27 // (5 * P + 5 + 3 * (g - 1))
    f = freqs[: FB + 500]
    lo, hi = FB - 300, FB + 300
    rng = np.random.default_rng(8)
    fpl, fcr = rng.uniform(-1, 1, (3, P)), rng.uniform(-1, 1, (3, P))
    np.testing.assert_array_equal(pack.fe_sweep(f, fpl, fcr)[:, lo:hi], pack.fe_sweep(f[lo:hi], fpl, fcr))
    whole, part = pack.fe_skymax(f, fpl, fcr), pack.fe_skymax(f[lo:hi], fpl, fcr)
    np.testing.assert_array_equal(whole[0][lo:hi], part[0])
    np.testing.assert_array_equal(whole[1][lo:hi], part[1])


def test_cuda_tensor_frequencies_on_a_side_stream(mixed):
    import torch

    pta = mixed
    freqs = _freqs(pta)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    fp = fastfp_b200.FastFp(pta.psrs)
    host = fp(freqs, *a)
    ft = torch.tensor(freqs, dtype=torch.float64, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = fp(ft, *a)
    s.synchronize()
    assert got.is_cuda
    np.testing.assert_array_equal(got.cpu().numpy(), host)


def test_prefer_i8_pack_is_mixed_and_the_wide_pulsar_keeps_its_bits(mixed):
    pta = mixed
    freqs = _freqs(pta)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    pack = fastfp_b200.FastFp(pta.psrs, path="prefer-i8").prepare(*a)
    assert pack.path == "mixed"
    ref = fastfp_b200.FastFp(pta.psrs, path="fp64").per_pulsar_terms(freqs, *a)
    got = pack.fp_sweep(freqs, terms=True)
    wide = [p for p in range(pta.P) if pta.Ts[p].shape[1] > 640]
    np.testing.assert_array_equal(got[wide], ref[wide])
    with pytest.raises(_cabi.FastFpError, match="m > 639"):
        pack.set_path("i8")


def test_refusals():
    top = _cabi.MAX_M_WIDE
    pta = synth.make_pta(1, [top + 40], n_tm=top + 1 - 2 * NCOMPS, ncomps=NCOMPS, seed=2)
    with pytest.raises(ValueError, match=f"maximum {top}"):
        _cabi.Pack.create(pta.toas, pta.residuals, pta.Nvecs, pta.Ts, pta.sigmas)
    # the library refuses it as well, naming the limit
    import ctypes as C

    h = C.c_void_p()
    arr = lambda xs: _cabi._ptr_array([_cabi.as_f64(x) for x in xs])  # noqa: E731
    rc = _cabi.load().fastfp_pack_create(0, 1, _cabi._int64_array([top + 40]), _cabi._int64_array([top + 1]),
                                         arr(pta.toas), arr(pta.residuals), arr(pta.Nvecs), arr(pta.Ts),
                                         arr(pta.sigmas), None, C.byref(h))
    assert rc == -3 and f"maximum {top}".encode() in _cabi.load().fastfp_last_error()


def test_residual_and_simulated_batches_refuse_a_wide_pack(mixed):
    pta = mixed
    freqs = synth.fp_freqs(5)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    fp = fastfp_b200.FastFp(pta.psrs)
    res = [np.zeros((2, r.size)) for r in pta.residuals]
    with pytest.raises(ValueError, match="wider than 640"):
        fp.calculate_Fp_batch(freqs, *a, res)
    with pytest.raises(ValueError, match="wider than 640"):
        fp.calculate_Fp_simulated(freqs, *a, [1.0 / phi for phi in pta.phis], 4, seed=1)
    pack = fp.prepare(*a)
    with pytest.raises(_cabi.FastFpError, match="wider than 640"):
        pack.set_residuals(res)
