"""The tensor-core sweep (fp_sweep_i8.cu) in every launch geometry, against the longdouble truth of oracle/truth.py:
the packs of tests/test_i8_geometry_host.py (every G-ring depth, every row-group count with every last-group size, the
w row alone in its group, odd and even stage counts, nst = 1, narrow pulsars on a wide pulsar's ring, several items
per CTA), then data the format finds hard, on both sweep kernels. Run with -m gpu on an H100.

* Fp: every pulsar of every pack on a grid with red-noise bins, f <= 0 (NaN), bins past the Cody-Waite range, a
  ragged last tile and one tile whose producer warps take both sincos paths; in the multi-item packs, the whole tiles
  of every item the first and the last CTA sweep. Fe at three sky positions against the Fe truth of the same inner
  products. Failures name the geometry ("rows 224, 2 groups, last 96, gst 5, nst 14").
* Exact identities (the integer sums are exact and the producers' two partial sums are added commutatively): a
  pulsar's row equals that pulsar swept alone (on the ring its own width gives), a bin does not depend on its tile
  position, on F or on the items its CTA swept before it, and the statistic is the ordered pulsar sum.
* Noise-marginalised stage A against the truth of each draw's Sigma, per-draw blocks straddling row groups.
* A pulsar the routing sends to the fp64 kernel returns the all-fp64 bits.
* Data edges on both kernels: N over six decades with a few TOAs 10^3 x more precise than the rest, epoch-clustered
  TOAs with seasonal gaps and a cluster where cos(omega t) ~ 0 at every precise TOA, a 10^4 sigma outlier, all-zero
  residuals (terms exactly 0) and a basis column with no TOAs."""
from types import SimpleNamespace

import numpy as np
import pytest

import fastfp_b200
from conftest import EPS, term_tolerance
from fastfp_b200 import NMFP, RN_container, synth
from fastfp_b200.fe import antenna_pattern
from oracle import fp_oracle as o
from oracle import truth
from test_gpu_sweep_instantiations import _assert_nan_at_nonpositive, _ordered_sum, _ratio, _report
from test_i8_geometry_host import C, CASES, NM_CASES, label, pack_gst, psr_geometry
from test_sweep_instantiations_host import LO, LO8, SINCOS_FAST, sweep_freqs

pytestmark = pytest.mark.gpu

NF = C["NF"]
D = 2  # draws of every noise-marginalised pack


def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _assert_straddle(freqs, tabs):
    """Every pulsar has a fast bin (LO) and a library-sincos bin (LO + 1) in one 16-bin tile, in different producer
    warps of 4 bins; the same for the pair at LO8."""
    fast = np.abs(2 * np.pi * freqs)[None, :] * np.asarray(tabs)[:, None] <= SINCOS_FAST
    for lo in (LO, LO8):
        assert np.all(fast[:, lo]) and not np.any(fast[:, lo + 1])
        assert lo // NF == (lo + 1) // NF and (lo % NF) // 4 != ((lo + 1) % NF) // 4


def _build(pack, seed):
    """One synthetic pulsar per entry of the pack (its own TOAs and basis), as the lists of a PTA, and its grid."""
    ptas = []
    for i, (n_tm, nc, n) in enumerate(pack.psrs):
        pta = synth.make_pta(1, n, n_tm=n_tm, ncomps=max(nc, 1), white_only=nc == 0, seed=seed + 7 * i)
        assert pta.Ts[0].shape == (n, n_tm + 2 * nc), label(pack, i)
        ptas.append(pta)
    s = SimpleNamespace(**{k: [getattr(p, k)[0] for p in ptas]
                           for k in ("psrs", "toas", "residuals", "Nvecs", "Ts", "TNTs", "phis", "sigmas", "n_tm")})
    s.Ffreqs = [p.Ffreqs for p in ptas]
    s.P = len(ptas)
    s.Tspan = max(p.Tspan for p in ptas)
    s.a = (s.Nvecs, s.Ts, s.sigmas)
    return s


# ---- Fp and Fe over the geometry packs ---------------------------------------------------------------------------

_FP = {}


def _fp_pack(name):
    """The pack's sweep on the tensor path, the (pulsar, bin) entries checked against the truth and their truth."""
    if name in _FP:
        return _FP[name]
    k = [c.name for c in CASES].index(name)
    pack = CASES[k]
    s = _build(pack, seed=80_000 + 1000 * k)
    if pack.F == 131:
        s.freqs = sweep_freqs(s.Tspan, [t.max() for t in s.toas])
        _assert_straddle(s.freqs, [t.max() for t in s.toas])
    else:
        s.freqs = np.linspace(1e-8, 9e-7, pack.F)  # all bins on the fast sincos path, above the lowest red-noise bins
    s.pos = s.freqs > 0
    fp = fastfp_b200.FastFp(s.psrs, path="i8")
    assert fp.prepare(*s.a).path == "i8", pack.name
    got = fp.per_pulsar_terms(s.freqs, *s.a)
    assert got.shape == (s.P, pack.F)
    _assert_nan_at_nonpositive(got, s, pack.name)
    ntile = -(-pack.F // NF)
    nwork = s.P * ntile
    grid = min(nwork, _sms())
    if pack.F == 131:
        tiles = [(p, t) for p in range(s.P) for t in range(ntile)]
    else:  # every item of the first and the last CTA: several items each, row groups and parities carried over
        items = sorted({b + j * grid for b in (0, grid - 1) for j in range(-(-nwork // grid))})
        tiles = [(i // ntile, i % ntile) for i in items if i < nwork]
    checked = {p: sorted({b for q, t in tiles if q == p for b in range(NF * t, min(NF * t + NF, pack.F))})
               for p in range(s.P)}
    checked = {p: np.array([b for b in bins if s.pos[b]], dtype=int) for p, bins in checked.items() if bins}
    inner, tt, cond, ora = {}, {}, {}, {}
    for p, bins in checked.items():
        args = (s.freqs[bins], [s.toas[p]], [s.residuals[p]], [s.Nvecs[p]], [s.Ts[p]], [s.sigmas[p]])
        inner[p] = truth.sweep_inner_truth(*args)
        tt[p], cond[p] = truth.terms_truth(inner[p])
        ora[p] = o.fp_sweep(*args, per_pulsar=True)
    r = SimpleNamespace(pack=pack, s=s, fp=fp, got=got, tiles=tiles, checked=checked, inner=inner, tt=tt, cond=cond,
                        ora=ora, grid=grid, ntile=ntile, nwork=nwork)
    _FP[name] = r
    return r


FP_NAMES = [c.name for c in CASES]


@pytest.mark.parametrize("name", FP_NAMES)
def test_fp_against_truth(name):
    d = _fp_pack(name)
    if d.pack.F != 131:
        assert -(-d.nwork // d.grid) >= 5, (name, d.nwork, d.grid)  # several items per CTA
    ratios, labels = [], []
    for p, bins in d.checked.items():
        tv = d.tt[p].astype(float)
        ratios.append(_ratio(d.got[p, bins], tv[0], term_tolerance(tv, d.cond[p], d.ora[p])[0], d.cond[p][0]))
        labels.append(label(d.pack, p))
        print(f"\n[i8 Fp] gst {pack_gst(d.pack)}, last {psr_geometry(d.pack.psrs[p])['last']}: worst "
              f"{ratios[-1].max():.3g} ({labels[-1]})", end="")
    _report(f"Fp, {name}", ratios, labels)


@pytest.mark.parametrize("name", [c.name for c in CASES if c.F == 131 and len(c.psrs) > 1])
def test_fe_against_truth(name):
    """calculate_Fe at three sky positions: all five inner products of every pulsar through the Fe truth of the same
    longdouble inner products (rule of test_gpu_fe_truth.py). Not on the one-pulsar pack of 31 TOAs: a single short
    pulsar leaves too few Fe bins with digits in any float64 formulation."""
    d = _fp_pack(name)
    s = d.s
    rng = np.random.default_rng(len(name))
    th, ph = np.arccos(rng.uniform(-1, 1, 3)), rng.uniform(0, 2 * np.pi, 3)
    fe_obj = fastfp_b200.FastFe(s.psrs, path="i8")
    assert fe_obj.prepare(*s.a).path == "i8"
    got = fe_obj.calculate_Fe(s.freqs, th, ph, *s.a)
    _assert_nan_at_nonpositive(got, s, f"Fe, {name}")
    inner = {k: np.concatenate([d.inner[p][k] for p in range(s.P)]) for k in d.inner[0]}
    fplus, fcross = antenna_pattern(np.stack([q.pos for q in s.psrs]), th, ph)
    fe, cond = truth.fe_truth_from_inner(inner, s.freqs[s.pos], fplus, fcross)
    tc = np.concatenate([d.cond[p] for p in range(s.P)])
    tt = np.concatenate([d.tt[p] for p in range(s.P)]).astype(float)
    ora = np.concatenate([d.ora[p] for p in range(s.P)])
    E = (term_tolerance(tt, tc, ora, k_oracle=1.0, rel=0.0) / (EPS * tc)).max()
    tv = fe.astype(float)
    ratio = _ratio(got[:, s.pos], tv, 1e-10 * np.abs(tv) + 4 * E * EPS * cond, cond)
    print(f"\n[i8 Fe] gst {pack_gst(d.pack)}: worst {ratio.max():.3g} ({name})", end="")
    _report(f"Fe, {name}", list(ratio), [f"{name}, sky position {k}" for k in range(3)])


@pytest.mark.parametrize("name", FP_NAMES)
def test_fp_bit_identities(name):
    """Each pulsar alone (its own ring depth) gives its row of the pack; the statistic is the ordered pulsar sum; a bin
    does not depend on its tile position or on F: odd-shifted slices of fast-path bins (in the multi-item packs,
    around every checked tile, which the full launch swept after other items of its CTA)."""
    d = _fp_pack(name)
    s, pack = d.s, d.pack
    for p in range(s.P):
        one = fastfp_b200.FastFp([s.psrs[p]], path="i8")
        assert one.prepare([s.Nvecs[p]], [s.Ts[p]], [s.sigmas[p]]).path == "i8"
        got1 = one.per_pulsar_terms(s.freqs, [s.Nvecs[p]], [s.Ts[p]], [s.sigmas[p]])
        np.testing.assert_array_equal(got1[0], d.got[p], err_msg=f"alone: {label(pack, p)}")
    np.testing.assert_array_equal(d.fp(s.freqs, *s.a), _ordered_sum(d.got), err_msg=name)
    if pack.F == 131:
        slices = ((3, 70), (37, 38), (1, 88), (85, 88), (11, 44))
    else:
        slices = sorted({(max(0, NF * t - 5), min(pack.F, NF * t + NF + 3)) for _, t in d.tiles})
    for lo, hi in slices:
        np.testing.assert_array_equal(d.fp.per_pulsar_terms(s.freqs[lo:hi], *s.a), d.got[:, lo:hi],
                                      err_msg=f"{name}: bins {lo}:{hi}")


# ---- noise-marginalised stage A -------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", [c.name for c in NM_CASES])
def test_nmfp_against_truth(name):
    """Two draws against the truth of each draw's Sigma; ``cond`` extended by ``truth.sigma_cond_truth`` and the
    oracle-relative allowance of ``conftest.term_tolerance`` (rule of test_gpu_nmfp_batches.py). The per-draw rows
    mfix .. m - 1 leave the kernel as z' rows, the others enter its b-sums."""
    k = [c.name for c in NM_CASES].index(name)
    pack = NM_CASES[k]
    s = _build(pack, seed=90_000 + 1000 * k)
    freqs = np.concatenate((np.linspace(2e-9, 3e-7, 36), np.array([1.0, 2.5]) / s.Tspan, [0.0, 5e-5]))
    s.pos = freqs > 0
    samples = synth.draw_samples(SimpleNamespace(psrs=s.psrs), D, seed=95 + k)
    nm = NMFP(s.psrs, [RN_container(q, Ffreqs=ff) for q, ff in zip(s.psrs, s.Ffreqs)], path="i8")
    pk = nm.prepare(s.Nvecs, s.Ts, s.TNTs)
    assert pk.path == "i8" and pk.mvar_total == sum(2 * q[1] for q in pack.psrs), name
    got = nm(freqs, samples, s.Nvecs, s.Ts, s.TNTs)
    assert got.shape == (D, freqs.shape[0])
    _assert_nan_at_nonpositive(got, s, name)
    phi_args = [dict(psr_name=q.name, n_tm=s.n_tm[p], Ffreqs=s.Ffreqs[p]) for p, q in enumerate(s.psrs)]
    f = freqs[s.pos]
    tv, cond, ora = np.empty((D, f.shape[0])), np.empty((D, f.shape[0])), np.empty((D, f.shape[0]))
    for dd in range(D):
        sig = o.get_sigmas({key: v[dd] for key, v in samples.items()}, s.TNTs, phi_args)
        args = (f, s.toas, s.residuals, s.Nvecs, s.Ts, sig)
        tt, c = truth.fp_sweep_truth(*args)
        tv[dd], cond[dd] = tt.sum(0).astype(float), c.sum(0) + truth.sigma_cond_truth(*args).sum(0)
        ora[dd] = o.fp_sweep(*args)
    tol = term_tolerance(tv, cond, ora)
    ratio = np.abs(got[:, s.pos] - tv) / tol
    geo = "; ".join(label(pack, p) + f", per-draw rows {q[0]}..{q[0] + 2 * q[1] - 1}" for p, q in enumerate(pack.psrs))
    print(f"\n[i8 Nmfp] gst {pack_gst(pack)}, last {psr_geometry(pack.psrs[-1])['last']}: worst {ratio.max():.3g} "
          f"({geo})", end="")
    worst = np.unravel_index(np.argmax(ratio), ratio.shape)
    assert np.all(ratio <= 1), f"{geo}: worst |got - truth| / tol = {ratio.max():.3g} at (draw, bin) {worst}"


# ---- routing: what the tensor path does not take runs on the fp64 kernel, bit for bit ------------------------------

def test_routing_sends_the_rest_to_the_fp64_kernel():
    """One pulsar the tensor path takes, and one each past n = 16384, past m + 1 = 640, with a non-finite w (a NaN
    residual) and with a failed factor: ``prefer-i8`` sweeps them as a mixed pack, and every pulsar the routing sends
    to the fp64 kernel returns the bits of an all-fp64 pack."""
    pack = SimpleNamespace(name="routing", psrs=((12, 30, 500), (7, 10, 16385), (520, 60, 700), (12, 30, 300),
                                                 (12, 30, 301)))
    s = _build(pack, seed=99_000)
    s.psrs[3].residuals = s.psrs[3].residuals.copy()
    s.psrs[3].residuals[17] = np.nan
    s.sigmas[4] = s.sigmas[4].copy()
    s.sigmas[4][5, 5] = -abs(s.sigmas[4][5, 5])
    freqs = np.concatenate((synth.fp_freqs(30), np.array([1.0, 2.5]) / s.Tspan, [0.0]))
    with pytest.warns(RuntimeWarning, match="not numerically symmetric positive definite"):
        mixed = fastfp_b200.FastFp(s.psrs, path="prefer-i8")
        assert mixed.prepare(*s.a).path == "mixed"
        tm = mixed.per_pulsar_terms(freqs, *s.a)
        all64 = fastfp_b200.FastFp(s.psrs, path="fp64")
        assert all64.prepare(*s.a).path == "fp64"
        t64 = all64.per_pulsar_terms(freqs, *s.a)
    for p in (1, 2, 3, 4):
        np.testing.assert_array_equal(tm[p], t64[p], err_msg=f"pulsar {p}")
    assert np.all(np.isnan(tm[3])) and np.all(np.isnan(tm[4]))
    one = fastfp_b200.FastFp([s.psrs[0]], path="i8").per_pulsar_terms(freqs, [s.Nvecs[0]], [s.Ts[0]], [s.sigmas[0]])
    np.testing.assert_array_equal(tm[0], one[0])
    assert not np.array_equal(tm[0, :30], t64[0, :30])  # pulsar 0 did run on the tensor kernel


# ---- data edges, on both kernels ----------------------------------------------------------------------------------

EDGES = ["N over six decades", "seasons, aligned precise cluster", "10^4 sigma outlier", "zero residuals",
         "basis column with no TOAs"]
N_TM, NCOMPS = 12, 30


def _edge_pulsar(name, t, sig, rng, r=None, dmx=()):
    """One pulsar on TOAs ``t`` with TOA errors ``sig``, the recipe of synth.make_pta (timing model, 30 Fourier
    components, red noise injected, timing model fitted out), optionally with DMX-like range columns ``dmx`` ((lo, hi)
    time ranges, prior variance 1e-12 s^2) in front of the basis."""
    U = synth._timing_basis(t, N_TM)
    Tspan = t.max() - t.min()
    Ff = np.repeat(np.arange(1, NCOMPS + 1) / Tspan, 2)
    F = np.empty((t.size, 2 * NCOMPS))
    arg = 2.0 * np.pi * t[:, None] * Ff[None, ::2]
    F[:, ::2], F[:, 1::2] = np.sin(arg), np.cos(arg)
    phi_rn = synth.powerlaw_phi(Ff, -14.0, 13.0 / 3.0)
    if r is None:
        r = sig * rng.standard_normal(t.size) + F @ (rng.standard_normal(2 * NCOMPS) * np.sqrt(phi_rn))
        r = r - U @ (U.T @ r)
    X = np.stack([((t >= lo) & (t < hi)).astype(float) for lo, hi in dmx], axis=1) if dmx else np.zeros((t.size, 0))
    T = np.ascontiguousarray(np.concatenate((X, U, F), axis=1))
    phi = np.concatenate((np.full(len(dmx), 1e-12), np.full(N_TM, 1e40), phi_rn))
    Nvec = sig**2
    TNT = T.T @ (T / Nvec[:, None])
    TNT = 0.5 * (TNT + TNT.T)
    psr = SimpleNamespace(name=name, toas=t, residuals=r, Mmat=U, backend_flags=np.array(["synth"] * t.size),
                          pos=synth._sky_position(rng))
    return psr, Nvec, T, TNT + np.diag(1.0 / phi)


def _seasons(rng, nep, per_epoch, t0):
    """``nep`` epochs of ``per_epoch`` TOAs 0.2 s apart, observed in the 8 months of each year away from the Sun
    (the other 4 months are a gap), over 15 years from ``t0``."""
    yr = 365.25 * 86400.0
    year = rng.integers(0, 15, nep)
    day = rng.uniform(0.0, 8.0 / 12.0 * yr, nep)
    ep = np.sort(t0 + year * yr + day)
    ep = ep + 10.0 * np.arange(nep)
    return (ep[:, None] + 0.2 * np.arange(per_epoch)[None, :]).reshape(-1)


ALIGNED_K = (23, 61, 97, 150)  # cos((2 pi f) t) ~ 0 at the precise cluster for f = (k + 1/4) / t_c
ALIGNED_BINS = (10, 30, 50, 65)


@pytest.fixture(scope="module")
def edges():
    rng = np.random.default_rng(4711)
    t0 = synth.MJD0_SECONDS
    yr = 365.25 * 86400.0
    out = []
    # 1. N from 1e-18 to 1e-12: errors 1e-7..1e-6 s, four TOAs at 1e-9 s (10^3 x the least precise)
    t = t0 + np.sort(rng.uniform(0.0, 15 * yr, 700))
    sig = 10.0 ** rng.uniform(-7.0, -6.0, t.size)
    sig[[50, 300, 301, 620]] = 1e-9
    out.append(_edge_pulsar("J0001+0000", t, sig, rng))
    # 2. epochs of 8 TOAs with seasonal gaps; the precise TOAs are one whole epoch, at t_c
    t = _seasons(rng, 90, 8, t0)
    sig = 10.0 ** rng.uniform(-7.0, -6.0, t.size)
    c = 8 * 41
    sig[c:c + 8] = 1e-9
    t_c = float(t[c + 4])
    out.append(_edge_pulsar("J0002+0000", t, sig, rng))
    # 3. one residual 10^4 sigma off
    t = t0 + np.sort(rng.uniform(0.0, 15 * yr, 640))
    sig = rng.uniform(1e-7, 1e-6, t.size)
    q = _edge_pulsar("J0003+0000", t, sig, rng)
    q[0].residuals = q[0].residuals.copy()
    q[0].residuals[333] += 1e4 * sig[333]
    out.append(q)
    # 4. all-zero residuals
    t = t0 + np.sort(rng.uniform(0.0, 15 * yr, 500))
    out.append(_edge_pulsar("J0004+0000", t, rng.uniform(1e-7, 1e-6, t.size), rng, r=np.zeros(t.size)))
    # 5. DMX ranges of 2 years, the first one (column 0: an exactly zero G row) inside a gap without TOAs
    t = t0 + np.sort(np.concatenate((rng.uniform(2.5 * yr, 15 * yr, 600), rng.uniform(0.0, 0.4 * yr, 20))))
    dmx = [(t0 + 0.5 * yr, t0 + 2.5 * yr), (t0 + 2.5 * yr, t0 + 4.5 * yr), (t0 + 9.0 * yr, t0 + 11.0 * yr)]
    out.append(_edge_pulsar("J0005+0000", t, rng.uniform(1e-7, 1e-6, t.size), rng, dmx=dmx))
    assert not np.any(out[4][2][:, 0]) and np.all(np.any(out[4][2][:, 1:], axis=0))
    s = SimpleNamespace(psrs=[q[0] for q in out], Nvecs=[q[1] for q in out], Ts=[q[2] for q in out],
                        sigmas=[q[3] for q in out], P=len(out))
    s.toas = [q.toas for q in s.psrs]
    s.residuals = [q.residuals for q in s.psrs]
    s.a = (s.Nvecs, s.Ts, s.sigmas)
    tspan = max(t.max() for t in s.toas) - min(t.min() for t in s.toas)
    s.freqs = sweep_freqs(tspan, [t.max() for t in s.toas])
    for b, k in zip(ALIGNED_BINS, ALIGNED_K):
        s.freqs[b] = (k + 0.25) / t_c
    _assert_straddle(s.freqs, [t.max() for t in s.toas])
    precise = slice(c, c + 8)
    ph = (2 * np.pi * s.freqs[list(ALIGNED_BINS)])[:, None] * s.toas[1][None, precise]
    assert np.abs(np.cos(ph)).max() < 1e-6  # cos(omega t) ~ 0 at every precise TOA of the aligned bins
    s.pos = s.freqs > 0
    f = s.freqs[s.pos]
    tt, s.cond = truth.fp_sweep_truth(f, s.toas, s.residuals, *s.a)
    s.tv = tt.astype(float)
    s.tol = term_tolerance(s.tv, s.cond, o.fp_sweep(f, s.toas, s.residuals, *s.a, per_pulsar=True))
    return s


@pytest.mark.parametrize("path", ["i8", "fp64"])
def test_data_edges(edges, path):
    s = edges
    fp = fastfp_b200.FastFp(s.psrs, path=path)
    assert fp.prepare(*s.a).path == path
    got = fp.per_pulsar_terms(s.freqs, *s.a)
    _assert_nan_at_nonpositive(got[[0, 1, 2, 4]], s, path)
    assert np.all(np.isnan(got[3, ~s.pos])) and np.all(got[3, s.pos] == 0.0), "zero residuals: terms exactly 0"
    aligned = np.searchsorted(np.flatnonzero(s.pos), ALIGNED_BINS)
    ratios, labels = [], []
    for p in (0, 1, 2, 4):
        r = _ratio(got[p, s.pos], s.tv[p], s.tol[p], s.cond[p])
        ratios.append(r)
        labels.append(f"{path}: {EDGES[p]}")
        extra = f", aligned bins {r[aligned].max():.3g}" if p == 1 else ""
        print(f"\n[edges, {path}] {EDGES[p]}: worst {r.max():.3g}{extra}", end="")
    _report(f"data edges, {path}", ratios, labels)
