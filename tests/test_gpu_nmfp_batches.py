"""The two batch loops of the noise-marginalised sweep, and the corners of the noise prior (GPU).

``fastfp_b200/csrc/nmfp.cu`` splits one ``fastfp_nmfp_sweep`` in two host loops:

* draw batches (``nmfp_stage_b_impl``): the L^-1 fragment store is capped at 3 * 2^26 doubles (1.5 GiB), so one
  factor + stage-B launch pair handles ``DB`` draws; each batch offsets the phi^-1 rows by ``dd * mvar_total`` and the
  output rows by ``dd * out_ld``, and the last batch may hold fewer than the 8 draws of a stage-B CTA;
* frequency batches (``nmfp_sweep_impl``): stage-A output is capped at 2^27 doubles, so one stage A + factor + stage B
  handles ``FB`` frequencies, written at column ``f0`` of the ``(D, F)`` output with row stride ``F``.

Every boundary case asserts the launch-count difference that proves it crossed the boundary, so a change of either
budget makes these tests fail instead of quietly no longer crossing. Values are checked bit for bit against calls that
stay inside one batch, and against the longdouble truth of ``oracle/truth.py``.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import EPS, term_tolerance
from fastfp_b200 import NMFP, BlockNvec, CURN_container, RN_container, _cabi, parallel, synth
from oracle import fp_oracle as o
from oracle import truth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NB_DT = 8  # draws per stage-B CTA (nmfp.cu)


# ---- the batch sizes of fastfp_b200/csrc/nmfp.cu, restated --------------------------------------------------------
def _nmbv(mvar_max):
    """8-row blocks of the padded per-draw system (``nmfp_pack_finish``)."""
    return 4 if mvar_max <= 32 else 8 if mvar_max <= 64 else 12 if mvar_max <= 96 else 16


def _lfw(nmbv):
    """doubles per (pulsar, draw) in the L^-1 store: ``linv_blocks(NMBV) * 32 + 8 * NMBV``"""
    return sum(nmbv - kb // 2 for kb in range(2 * nmbv)) * 32 + 8 * nmbv


def draw_batch(P, mvar_max, D=1 << 40):
    """``DB`` of ``nmfp_stage_b_impl`` with the default (1.5 GiB) budget."""
    return max(NB_DT, min(D, (3 << 26) // (P * _lfw(_nmbv(mvar_max))) // NB_DT * NB_DT))


def draw_batch_lf_mb(P, mvar_max, D, F, lf_mb, num_sms):
    """``DB`` of ``nmfp_stage_b_impl`` under ``FASTFP_B200_NMFP_LF_MB=lf_mb``, and whether the wave rounding changed it."""
    per_draw = P * _lfw(_nmbv(mvar_max)) * 8
    groups = max(1, (lf_mb << 20) // (per_draw * NB_DT))
    pairs = (-(-F // 32) + 1) // 2
    unrounded = groups
    if pairs < num_sms:
        per_wave = max(1, num_sms // pairs)
        if groups >= per_wave:
            groups = groups // per_wave * per_wave
    cap = max(NB_DT, -(-D // NB_DT) * NB_DT)
    return min(max(NB_DT, groups * NB_DT), cap), groups != unrounded


def freq_batch(P, mvar_max):
    """``FB`` of ``nmfp_sweep_impl``: whole 32-frequency tiles of stage-A output within 2^27 doubles."""
    MV = 8 * _nmbv(mvar_max)
    return max(32, (1 << 27) // (P * (64 * MV + 160)) * 32)


# the figures these tests are built around
assert [draw_batch(68, mv) for mv in (32, 64, 96, 128)] == [4400, 1248, 576, 328]
assert [draw_batch(8, mv) for mv in (32, 64, 96, 128)] == [37448, 10624, 4944, 2848]
assert [freq_batch(68, mv) for mv in (32, 64, 96, 128)] == [28576, 14816, 10016, 7552]


# ---- cases --------------------------------------------------------------------------------------------------------
class Case:
    """A pulsar set with CURN, diagonal or block-diagonal N (epochs of 4 TOAs, as at C5), and what the truth needs."""

    def __init__(self, P, ncomps, n, seed, block=False):
        self.pta = pta = synth.make_pta(P, n, ncomps=ncomps, seed=seed)
        self.P, self.mvar = P, 2 * ncomps
        self.curn = CURN_container(pta.Ffreqs)
        self.phi_args = [dict(psr_name=q.name, n_tm=pta.n_tm[p], Ffreqs=pta.Ffreqs, add_curn=True,
                              curn_Ffreqs=self.curn.Ffreqs) for p, q in enumerate(pta.psrs)]
        self.tblocks = None
        if block:
            rng = np.random.default_rng(seed + 777)
            Nvecs, self.tblocks, TNTs = [], [], []
            for p in range(P):
                k = pta.toas[p].size
                sl = [slice(a, a + 4) for a in range(0, k - 3, 4)]
                jv = rng.uniform(0.3, 3.0, len(sl)) * 1e-13
                B = BlockNvec(pta.Nvecs[p], sl, jv)
                TNT = pta.Ts[p].T @ B.solve(pta.Ts[p])
                Nvecs.append(B)
                self.tblocks.append((pta.Nvecs[p], [(s.start, s.stop) for s in sl], jv))
                TNTs.append(0.5 * (TNT + TNT.T))
            self.mats = (Nvecs, pta.Ts, TNTs)
        else:
            self.mats = (pta.Nvecs, pta.Ts, pta.TNTs)

    def nmfp(self):
        sigs = [RN_container(q, Ffreqs=self.pta.Ffreqs, add_curn=True, curn_container=self.curn)
                for q in self.pta.psrs]
        return NMFP(self.pta.psrs, sigs)

    def freqs(self, F):
        """ragged grid: the first red-noise Fourier bins (the worst-conditioned points), then the plain-Fp grid"""
        return np.concatenate((synth.nmfp_freqs(5, self.pta.Tspan), synth.fp_freqs(F - 5)))

    def truth(self, freqs, sigmas):
        """``(sum over pulsars of the terms, sum of cond)`` for one draw's Sigma matrices"""
        pta = self.pta
        if self.tblocks is None:
            tt, cond = truth.fp_sweep_truth(freqs, pta.toas, pta.residuals, pta.Nvecs, pta.Ts, sigmas)
        else:
            tt, cond = truth.fp_sweep_truth_blockn(freqs, pta.toas, pta.residuals, self.tblocks, pta.Ts,
                                                   sigmas=sigmas)
        return tt.sum(0).astype(float), cond.sum(0)


# name -> (P, ncomps, n, seed, block N, D): D = DB + tail; every per-draw family, tails of 2, 3, 8 and 1 draws
DRAW_CASES = {
    "c5_nmbv8": (68, 30, [300 + 4 * (p % 7) for p in range(68)], 51, True, 1248 + 2),
    "nmbv4": (68, 13, [200 + 3 * (p % 11) for p in range(68)], 52, False, 4400 + 3),
    "nmbv12": (68, 45, [220 + 5 * (p % 5) for p in range(68)], 53, False, 576 + 8),
    "nmbv16": (68, 61, [240 + 2 * (p % 13) for p in range(68)], 54, False, 328 + 1),
}
_CASES, _TRUTH = {}, {}


def _case(name):
    if name not in _CASES:
        P, ncomps, n, seed, block, _ = DRAW_CASES[name]
        _CASES[name] = Case(P, ncomps, n, seed, block)
    return _CASES[name]


def _draw_truth(name, case, freqs, samples, d):
    """truth for draw d of a case (cached: it does not depend on the sweep kernel)"""
    key = (name, d, freqs.tobytes())
    if key not in _TRUTH:
        pars = {k: v[d] for k, v in samples.items()}
        _TRUTH[key] = case.truth(freqs, o.get_sigmas(pars, case.mats[2], case.phi_args))
    return _TRUTH[key]


def _rows(samples, sl):
    return {k: v[sl] for k, v in samples.items()}


def _launches(fn):
    before = _cabi.kernel_launches()
    out = fn()
    return out, _cabi.kernel_launches() - before


def _tol(tv, cond):
    return 1e-10 * np.abs(tv) + 256 * EPS * cond


# ---- 1. draw batches ----------------------------------------------------------------------------------------------
@pytest.mark.usefixtures("sweep_path")
@pytest.mark.parametrize("name", list(DRAW_CASES))
def test_draw_batch_boundary(name):
    case = _case(name)
    D = DRAW_CASES[name][5]
    DB = draw_batch(case.P, case.mvar)
    assert DB < D <= 2 * DB
    nm = case.nmfp()
    F = 45  # not a multiple of the 32-frequency tile
    freqs = case.freqs(F)
    samples = synth.draw_samples(case.pta, D)
    mats = case.mats
    nm(freqs, _rows(samples, slice(0, NB_DT)), *mats)  # builds the pack
    # launch counts: D = 8 and D = DB are one batch, D = DB + 1 and D are two (one more factor + stage-B pair)
    _, n8 = _launches(lambda: nm(freqs, _rows(samples, slice(0, NB_DT)), *mats))
    _, ndb = _launches(lambda: nm(freqs, _rows(samples, slice(0, DB)), *mats))
    _, ndb1 = _launches(lambda: nm(freqs, _rows(samples, slice(0, DB + 1)), *mats))
    full, nfull = _launches(lambda: nm(freqs, samples, *mats))
    assert (ndb, ndb1, nfull) == (n8, n8 + 2, n8 + 2), (name, n8, ndb, ndb1, nfull)
    assert full.shape == (D, F) and np.all(np.isfinite(full)) and full.min() > 0
    # each of these calls stays inside one batch
    np.testing.assert_array_equal(nm(freqs, _rows(samples, slice(0, DB)), *mats), full[:DB])
    np.testing.assert_array_equal(nm(freqs, _rows(samples, slice(DB, D)), *mats), full[DB:])
    for d in (DB - 1, DB):
        np.testing.assert_array_equal(nm(freqs, _rows(samples, slice(d, d + 1)), *mats), full[d:d + 1])
    # reversed draw order moves draws across the boundary
    np.testing.assert_array_equal(nm(freqs, _rows(samples, slice(None, None, -1)), *mats), full[::-1])
    for d in (DB - 1, DB, D - 1):
        tv, cond = _draw_truth(name, case, freqs, samples, d)
        assert np.all(np.abs(full[d] - tv) <= _tol(tv, cond)), (name, d, (np.abs(full[d] - tv) / _tol(tv, cond)).max())


@pytest.mark.usefixtures("sweep_path")
def test_c5_two_dimensional_stage_b_crosses_the_draw_batch():
    """What C5 runs on each of 8 ranks: stage A in 8 frequency blocks (``parallel.tile_blocks``; one GPU stands in for
    the ranks), then ``nmfp_stage_b`` for 1250 draws = a 1248-draw batch and a 2-draw batch. Bit for bit the combined
    call."""
    import torch

    name = "c5_nmbv8"
    case = _case(name)
    D, world = DRAW_CASES[name][5], 8
    assert draw_batch(case.P, case.mvar) == 1248 and D == 1250
    F = 455  # 15 tiles: 8 blocks of 2, the last one padding only
    f = torch.from_numpy(case.freqs(F)).cuda()
    samples = synth.draw_samples(case.pta, D)
    nm = case.nmfp()
    want = nm(f, samples, *case.mats)
    pack = nm.prepare(*case.mats)
    nt, per = parallel.tile_blocks(F, world)
    assert (nt, per) == (15, 2)
    zt, at = pack.nmfp_tile_sizes()
    zall = torch.full((world * per * zt,), float("nan"), dtype=torch.float64, device="cuda")
    aall = torch.full((world * per * at,), float("nan"), dtype=torch.float64, device="cuda")
    for r in range(world):
        idx = torch.arange(32 * r * per, 32 * (r + 1) * per, device="cuda").clamp_(max=F - 1)
        floc = f[idx].contiguous()
        pack.nmfp_stage_a(floc.data_ptr(), 32 * per, zall[r * per * zt:].data_ptr(), aall[r * per * at:].data_ptr())
    _, A, G, cA, cG, _, _ = nm._draw_arrays(samples)
    phiinv = torch.empty((D, pack.mvar_total), dtype=torch.float64, device="cuda")
    pack.powerlaw_phiinv([s.Ffreqs for s in nm.rn_sigs], A, G, case.curn.Ffreqs, cA, cG, phiinv.data_ptr())
    out = torch.full((D, F), float("nan"), dtype=torch.float64, device="cuda")
    _, n = _launches(lambda: pack.nmfp_stage_b(f.data_ptr(), F, zall.data_ptr(), aall.data_ptr(), per,
                                               phiinv.data_ptr(), D, out.data_ptr()))
    torch.cuda.synchronize()
    assert n == 2 * 2  # two factor + stage-B pairs
    assert torch.equal(out.view(torch.int64), want.view(torch.int64))


# ---- 2. frequency batches -----------------------------------------------------------------------------------------
_FB_CASE = {}


def _fb_case():
    if not _FB_CASE:
        _FB_CASE["c"] = Case(68, 64, [200 + 3 * (p % 9) for p in range(68)], 61)
    return _FB_CASE["c"]


@pytest.mark.usefixtures("sweep_path")
def test_frequency_batch_boundary():
    import torch

    case = _fb_case()
    assert case.mvar == 128
    FB = freq_batch(case.P, case.mvar)
    assert FB == 7552
    F, D = FB + 45, 9  # 9 draws: the second 8-draw CTA holds one
    freqs = np.linspace(2e-9, 3e-7, F)
    # f <= 0 where the other batch's frequency at the same position is positive: stage A in nmfp mode does not mask
    # f <= 0, stage B does from its own frequency pointer, and Fp is even in f -- only a negative f shows a wrong offset
    freqs[FB + 7], freqs[FB + 20], freqs[33] = 0.0, -freqs[FB + 20], -freqs[33]
    bad = np.zeros(F, dtype=bool)
    bad[[FB + 7, FB + 20, 33]] = True
    assert np.all(freqs[[7, 20, FB + 33]] > 0)
    samples = synth.draw_samples(case.pta, D)
    nm = case.nmfp()
    mats = case.mats
    nm(freqs[:64], samples, *mats)  # builds the pack
    pack = nm.prepare(*mats)
    zt, at = pack.nmfp_tile_sizes()

    def stage_a_launches(Fa):
        nt = -(-Fa // 32)
        z = torch.empty(nt * zt, dtype=torch.float64, device="cuda")
        a = torch.empty(nt * at, dtype=torch.float64, device="cuda")
        fa = torch.from_numpy(np.abs(freqs[:Fa]) + 1e-9).cuda()
        _, n = _launches(lambda: pack.nmfp_stage_a(fa.data_ptr(), Fa, z.data_ptr(), a.data_ptr()))
        torch.cuda.synchronize()
        return n

    a_fb, a_tail = stage_a_launches(FB), stage_a_launches(45)
    # one phi^-1 launch, then per frequency batch a stage A and a factor + stage-B pair
    _, n_fb = _launches(lambda: nm(freqs[:FB], samples, *mats))
    full, n_full = _launches(lambda: nm(freqs, samples, *mats))
    assert n_fb == 1 + a_fb + 2, (n_fb, a_fb)
    assert n_full == n_fb + a_tail + 2, (n_full, n_fb, a_tail)

    assert full.shape == (D, F)
    assert np.all(np.isnan(full[:, bad])) and np.all(np.isfinite(full[:, ~bad]))
    np.testing.assert_array_equal(np.concatenate((nm(freqs[:FB], samples, *mats), nm(freqs[FB:], samples, *mats)),
                                                 axis=1), full)
    # CUDA-tensor frequencies: the device-output path, the same bits
    fd = torch.from_numpy(freqs).cuda()
    got = nm(fd, samples, *mats)
    assert torch.equal(got.cpu().view(torch.int64), torch.from_numpy(full).view(torch.int64))
    halves = torch.cat((nm(fd[:FB], samples, *mats), nm(fd[FB:], samples, *mats)), dim=1)
    assert torch.equal(halves.cpu().view(torch.int64), torch.from_numpy(full).view(torch.int64))
    # the columns either side of the boundary and the last one, two draws, against the truth
    cols = np.array([FB - 1, FB, F - 1])
    for d in (0, D - 1):
        pars = {k: v[d] for k, v in samples.items()}
        key = ("fb", d)
        if key not in _TRUTH:
            _TRUTH[key] = case.truth(freqs[cols], o.get_sigmas(pars, mats[2], case.phi_args))
        tv, cond = _TRUTH[key]
        assert np.all(np.abs(full[d, cols] - tv) <= _tol(tv, cond)), (d, full[d, cols], tv)


# ---- 3. the L2-resident draw batches ------------------------------------------------------------------------------
_CHILD = r"""
import sys
import numpy as np
sys.path.insert(0, {tests!r})
import test_gpu_nmfp_batches as t
from fastfp_b200 import _cabi, synth
out, F = sys.argv[1], int(sys.argv[2])
name = "c5_nmbv8"
case = t._case(name)
nm = case.nmfp()
freqs = case.freqs(F)
samples = synth.draw_samples(case.pta, t.DRAW_CASES[name][5])
nm(freqs, t._rows(samples, slice(0, 8)), *case.mats)
got, n = t._launches(lambda: nm(freqs, samples, *case.mats))
np.save(out, np.append(got.reshape(-1), float(n)))
"""


@pytest.mark.usefixtures("sweep_path")
@pytest.mark.parametrize("lf_mb", [1, 64])
def test_l2_resident_draw_batches_equal_the_default(lf_mb, tmp_path):
    """``FASTFP_B200_NMFP_LF_MB`` is read once per process, so the budgeted sweep runs in a child process; its draw
    batches (whole CTA waves under the budget) must give the default's bits. The grid has fewer frequency-tile pairs
    than SMs, so the rounding to whole waves applies."""
    import torch

    name = "c5_nmbv8"
    case = _case(name)
    D = DRAW_CASES[name][5]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pairs = sms // 5              # 5 draw groups of 8 per wave
    F = 64 * pairs - 13
    DB, rounded = draw_batch_lf_mb(case.P, case.mvar, D, F, lf_mb, sms)
    assert rounded == (lf_mb == 64), (lf_mb, DB)
    nm = case.nmfp()
    freqs = case.freqs(F)
    samples = synth.draw_samples(case.pta, D)
    nm(freqs, _rows(samples, slice(0, NB_DT)), *case.mats)
    want, n_def = _launches(lambda: nm(freqs, samples, *case.mats))
    out = tmp_path / "nmfp.npy"
    env = dict(os.environ, FASTFP_B200_NMFP_LF_MB=str(lf_mb), PYTHONDONTWRITEBYTECODE="1")
    r = subprocess.run([sys.executable, "-c", _CHILD.format(tests=os.path.join(ROOT, "tests")), str(out), str(F)],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = np.load(out)
    got, n = res[:-1].reshape(D, F), int(res[-1])
    # the default runs two draw batches (1248 + 2); the budgeted one ceil(D / DB) of them
    assert n == n_def - 2 * 2 + 2 * -(-D // DB), (n, n_def, DB)
    np.testing.assert_array_equal(got, want)


# ---- 4. the corners of the noise prior ----------------------------------------------------------------------------
CORNERS = [(-20.0, 0.0), (-20.0, 7.0), (-11.0, 0.0), (-11.0, 7.0)]  # (log10_A, gamma) of the usual prior's box
_CORNER_CASES = {}


def _corner_case(ncomps):
    """4 pulsars; 16 draws = every (CURN corner, red-noise corner) pair, each draw giving the pulsars all four
    red-noise corners"""
    if ncomps not in _CORNER_CASES:
        case = Case(4, ncomps, [300, 333, 287, 310], 71 + ncomps)
        D = 16
        samples = {}
        for p, q in enumerate(case.pta.psrs):
            c = np.array([CORNERS[(d + p) % 4] for d in range(D)])
            samples[f"{q.name}_red_noise_log10_A"], samples[f"{q.name}_red_noise_gamma"] = c[:, 0], c[:, 1]
        c = np.array([CORNERS[d // 4] for d in range(D)])
        samples["gw_log10_A"], samples["gw_gamma"] = c[:, 0], c[:, 1]
        _CORNER_CASES[ncomps] = (case, samples)
    return _CORNER_CASES[ncomps]


def _device_phiinv(nm, case, samples):
    import torch

    pack = nm.prepare(*case.mats)
    _, A, G, cA, cG, D, _ = nm._draw_arrays(samples)
    out = torch.empty((D, pack.mvar_total), dtype=torch.float64, device="cuda")
    pack.powerlaw_phiinv([s.Ffreqs for s in nm.rn_sigs], A, G, case.curn.Ffreqs, cA, cG, out.data_ptr())
    torch.cuda.synchronize()
    return out.cpu().numpy(), A, G, cA, cG


@pytest.mark.parametrize("ncomps", [30, 64])
def test_powerlaw_phiinv_at_prior_corners(ncomps):
    """``powerlaw_phiinv_kernel`` against the longdouble power law within 16 eps relative (16 ulp at 1.0). Budget, in
    eps relative: three CUDA ``pow`` calls at 2 ulp each (CUDA Math API), the amplitude's 2 doubled by squaring: 8;
    the float64 ``fyr`` (0.5, raised to |gamma - 3| <= 4: 2) and ``pi^2`` (0.5) constants: 2.5; six multiplications
    / divisions and the reciprocal at 0.5 each: 3.5; the CURN sum of two positive terms: 0.5. Total 14.5.
    ``gamma - 3`` is exact at the corners."""
    case, samples = _corner_case(ncomps)
    nm = case.nmfp()
    dev, A, G, cA, cG = _device_phiinv(nm, case, samples)
    assert np.all(np.isfinite(dev)) and dev.min() > 0
    m = case.mvar
    for p in range(case.P):
        want = truth.powerlaw_phiinv_truth(case.pta.Ffreqs, A[:, p], G[:, p], case.curn.Ffreqs, cA, cG)
        rel = np.abs(dev[:, p * m:(p + 1) * m] / want.astype(float) - 1)
        assert rel.max() <= 16 * EPS, (p, rel.max() / EPS)
    # the range the corners span: the prior hardly constrains the system at one end and dominates it at the other
    assert dev.min() < 1e5 and dev.max() > 1e29, (dev.min(), dev.max())


@pytest.mark.usefixtures("sweep_path")
@pytest.mark.parametrize("ncomps", [30, 64])
def test_nmfp_at_prior_corners_against_truth(ncomps):
    """``calculate_nmfp`` at the corner draws in the NMBV = 8 and 16 families against the truth of each draw's Sigma,
    built from the device's own phi^-1 (checked above), so that the factorisation is what is measured.

    Near gamma = 7 with a loud red process Sigma ~ T^T N^-1 T is itself badly conditioned (kappa ~ 1e13 here), and
    any float64 factorisation of it then errs by far more than the inner-product figure ``cond`` allows: the device and
    the float64 oracle reach 1.9e8 and 1e7 eps cond. ``cond`` is therefore extended by ``truth.sigma_cond_truth``, the
    first-order effect of a Cholesky backward error of Sigma. The allowance is the oracle-relative one of
    ``conftest.term_tolerance`` on that figure: 1e-10 |truth| + 4 E eps (cond + cond_Sigma), with E the float64
    oracle's own worst normalised error for that draw."""
    case, samples = _corner_case(ncomps)
    assert _nmbv(case.mvar) == (8 if ncomps == 30 else 16)
    nm = case.nmfp()
    F = 40
    freqs = case.freqs(F)
    got = nm(freqs, samples, *case.mats)
    D = got.shape[0]
    assert got.shape == (16, F) and np.all(np.isfinite(got))
    key = ("corners", ncomps)
    if key not in _TRUTH:
        dev = _device_phiinv(nm, case, samples)[0]
        pta, m = case.pta, case.mvar
        tv, cond, ora = np.empty((D, F)), np.empty((D, F)), np.empty((D, F))
        for d in range(D):
            sig = []
            for p in range(case.P):
                ntm = pta.n_tm[p]
                phiinv = np.concatenate((1.0 / np.full(ntm, 1e40), dev[d, p * m:(p + 1) * m]))
                sig.append(case.mats[2][p] + np.diag(phiinv))
            tv[d], cond[d] = case.truth(freqs, sig)
            cond[d] += truth.sigma_cond_truth(freqs, pta.toas, pta.residuals, pta.Nvecs, pta.Ts, sig).sum(0)
            ora[d] = o.fp_sweep(freqs, pta.toas, pta.residuals, pta.Nvecs, pta.Ts, sig)
        _TRUTH[key] = tv, cond, ora
    tv, cond, ora = _TRUTH[key]
    tol = term_tolerance(tv, cond, ora)
    dev_ = np.abs(got - tv)
    assert np.all(dev_ <= tol), (ncomps, np.unravel_index(np.argmax(dev_ / tol), tol.shape), (dev_ / tol).max())
