"""The Fe-statistic on the GPU against the longdouble truth (oracle/truth.fe_truth) on every sweep path: each family of
the fp64 DMMA kernel, the INT8 tensor-core kernel at its limits, a pack that mixes the two, the frequency batches of
fastfp_fe_sweep, the library sincos path, block-diagonal N in the wide families, and f <= 0. Plus identities that hold
exactly or to a few roundings on the kernels' own inner products: a pair of pure antenna patterns reduces Fe to two Fp
terms, power-of-two pattern scaling and sky permutations change nothing.

Tolerance: ``1e-10 |truth| + 4 E eps cond`` with ``cond`` the first-order conditioning figure of the truth and
``E >= 1`` the float64 Fp oracle's own worst distance from the Fp truth over the case's pulsars, in units of eps cond:
the float64 error of the same inner products (fe_oracle itself is too slow at these widths). Bins whose eps cond
reaches 5% of the value carry no digits in any float64 formulation and are left out; at least 90% must qualify."""
import numpy as np
import pytest

import fastfp_b200
from conftest import EPS, term_tolerance
from fastfp_b200 import _cabi, synth
from fastfp_b200.fe import antenna_pattern
from oracle import fp_oracle as o
from oracle import truth
from test_blockn_layout_host import family_of
from test_gpu_blockn_families import _case as blockn_case
from test_gpu_blockn_families import _config as blockn_config

pytestmark = pytest.mark.gpu

NAN_F = np.array([0.0, -1e-8, -5e-8])


def _sky(pos, seed):
    """Six positions: four random, the north pole, and one 0.03 rad from pulsar 0 (1 + Omega.p ~ 5e-4: both the
    numerators and the denominator of its antenna patterns are small)."""
    rng = np.random.default_rng(seed)
    th0, ph0 = np.arccos(pos[0, 2]), np.arctan2(pos[0, 1], pos[0, 0]) % (2 * np.pi)
    th = np.concatenate((np.arccos(rng.uniform(-1, 1, 4)), [0.0, th0 + 0.03]))
    ph = np.concatenate((rng.uniform(0, 2 * np.pi, 4), [0.0, ph0]))
    return antenna_pattern(pos, th, ph)


def _freqs(pta):
    """73 bins (a ragged tile) including the 1, 2.5 and 7 / Tspan red-noise bins."""
    return np.concatenate((synth.fp_freqs(70), np.array([1.0, 2.5, 7.0]) / pta.Tspan))


def _pos(pta):
    return np.stack([q.pos for q in pta.psrs])


def _truth(freqs, pta, fp, fx):
    """Fe truth, its cond, E (see the module docstring) and the Fp truth's cond, from one longdouble pass over the
    inner products."""
    args = (pta.toas, pta.residuals, pta.Nvecs, pta.Ts, pta.sigmas)
    inner = truth.sweep_inner_truth(freqs, *args)
    fe, cond = truth.fe_truth_from_inner(inner, freqs, fp, fx)
    tt, tc = truth.terms_truth(inner)
    ora = o.fp_sweep(freqs, *args, per_pulsar=True)
    E = (term_tolerance(tt.astype(float), tc, ora, k_oracle=1.0, rel=0.0) / (EPS * tc)).max()
    return fe, cond, E, tc


def _assert_near(got, fe, cond, E, what):
    tv = np.asarray(fe, dtype=np.float64)
    tol = 1e-10 * np.abs(tv) + 4 * E * EPS * cond
    defined = EPS * cond < 0.05 * np.abs(tv)
    assert defined.mean() >= 0.9, (what, defined.mean())
    ratio = np.where(defined, np.abs(got - tv) / tol, 0.0)
    worst = tuple(int(i) for i in np.unravel_index(np.argmax(ratio), ratio.shape))
    assert np.all(ratio <= 1), (f"{what}: worst |got - truth| / tol = {ratio.max():.3g} at (sky, bin) {worst}: got "
                                f"{got[worst]:.6g}, truth {tv[worst]:.6g}, cond {cond[worst]:.3g}, E {E:.3g}")


def _fe_pack(pta, path):
    return fastfp_b200.FastFe(pta.psrs, path=path).prepare(pta.Nvecs, pta.Ts, pta.sigmas)


# ---- 1. every family of the fp64 kernel at its bottom and top width (test_gpu_fp.py) ---------------------------------
FAMILY_CASES = {(2, 0): "w1", (5, 3): "w1", (12, 30): "w2", (20, 30): "w2", (9, 45): "w4", (40, 55): "w4",
                (150, 45): "wide", (230, 40): "wide", (340, 30): "xwide", (500, 60): "xwide"}


@pytest.mark.parametrize("n_tm,ncomps", list(FAMILY_CASES))
def test_fe_in_every_fp64_family(n_tm, ncomps):
    m = n_tm + 2 * ncomps
    fam, ci, _ = family_of(m)
    assert fam == FAMILY_CASES[(n_tm, ncomps)] and _cabi.load().fastfp_sweep_chunk_toas(m, 0) == ci
    ns = [333, 64, 1000] if m <= 40 else ([333, 300, 1000] if m <= 160 else ([2500, 1801, 3000] if m <= 320
                                                                        else [4000, 3001, 5000]))
    pta = synth.make_pta(3, ns, n_tm=n_tm, ncomps=ncomps, white_only=ncomps == 0, seed=77)
    pack = _fe_pack(pta, "fp64")
    assert pack.path == "fp64" and pack.m == [m] * 3
    freqs = _freqs(pta)
    fp, fx = _sky(_pos(pta), seed=m)
    got = pack.fe_sweep(freqs, fp, fx)
    _assert_near(got, *_truth(freqs, pta, fp, fx)[:3], f"m={m} ({fam}, CI={ci})")


# ---- 2. the INT8 kernel at its limits (test_gpu_i8_limits.py) --------------------------------------------------------
I8_CASES = {
    "m=127, n=16384": (dict(P=2, ns=[16384, 4099], n_tm=[7, 7], ncomps=60, seed=31), 127),
    "m=128": (dict(P=2, ns=[1500, 901], n_tm=8, ncomps=60, seed=34), 128),
    "m=256": (dict(P=2, ns=[1500, 901], n_tm=136, ncomps=60, seed=34), 256),
    "m=639": (dict(P=2, ns=[2600, 1901], n_tm=519, ncomps=60, seed=34), 639),
    "m=1, n=33/32/7": (dict(P=3, ns=[33, 32, 7], n_tm=1, ncomps=0, seed=33), 1),
}


@pytest.mark.parametrize("case", list(I8_CASES))
def test_fe_on_the_int8_kernel_at_its_limits(case):
    kw, m = I8_CASES[case]
    pta = synth.make_pta(kw["P"], kw["ns"], n_tm=kw["n_tm"], ncomps=kw["ncomps"], white_only=kw["ncomps"] == 0,
                         seed=kw["seed"])
    pack = _fe_pack(pta, "i8")
    assert pack.path == "i8" and pack.m[0] == m and pack.n == kw["ns"]
    freqs = _freqs(pta)
    fp, fx = _sky(_pos(pta), seed=m)
    got = pack.fe_sweep(freqs, fp, fx)
    _assert_near(got, *_truth(freqs, pta, fp, fx)[:3], f"i8 {case}")


# ---- 3. a mixed pack: the INT8 kernel and the fp64 rest_only sweep write parts of one inner-product array ---------------
def test_fe_on_a_mixed_pack():
    pta = synth.make_pta(3, [16385, 300, 1207], n_tm=[7, 7, 9], ncomps=60, seed=32)
    pack = _fe_pack(pta, "prefer-i8")
    assert pack.path == "mixed"
    freqs = _freqs(pta)
    fp, fx = _sky(_pos(pta), seed=3)
    fe, cond, E, tc = _truth(freqs, pta, fp, fx)
    _assert_near(pack.fe_sweep(freqs, fp, fx), fe, cond, E, "mixed pack")
    # pulsar 0 (one TOA beyond the INT8 exactness bound) is swept by the fp64 kernel: its Fp term is that of an
    # all-fp64 pack bit for bit, and Fe of a pure pattern pair built on its inner products is that term plus the other
    t64 = _fe_pack(pta, "fp64").fp_sweep(freqs, terms=True)
    tm = pack.fp_sweep(freqs, terms=True)
    np.testing.assert_array_equal(tm[0], t64[0])
    pairs = [(0, 1), (2, 0)]
    got = pack.fe_sweep(freqs, *_pair_patterns(pairs, 3))
    for k, (i, j) in enumerate(pairs):
        want = (t64 if i == 0 else tm)[i] + (t64 if j == 0 else tm)[j]
        assert np.all(np.abs(got[k] - want) <= 8 * EPS * (tc[i] + tc[j])), (i, j)


# ---- 4. a pair of pure patterns: Fe is the sum of two Fp terms on the same inner-product bits ---------------------------
def _pair_patterns(pairs, P):
    fp, fx = np.zeros((len(pairs), P)), np.zeros((len(pairs), P))
    for k, (i, j) in enumerate(pairs):
        fp[k, i], fx[k, j] = 1.0, 1.0
    return fp, fx


def test_pair_identity_routes_every_inner_product(sweep_path):
    """Pulsar i at (F+, Fx) = (1, 0), pulsar j at (0, 1), every other pulsar at (0, 0): M is block diagonal and Fe =
    term_i + term_j. Both sides come from the same inner products and differ only in the 2x2 and 4x4 solves, so a
    swapped or mis-indexed inner product (wrong pulsar, wrong frequency row, a missing -b term) fails far below any
    truth tolerance."""
    pta = synth.make_pta(5, [300, 257, 411, 350, 180], n_tm=[3, 12, 30, 8, 70], ncomps=10, seed=41)
    ms = [T.shape[1] for T in pta.Ts]
    assert len({family_of(m)[0] for m in ms}) == 3
    pack = fastfp_b200.FastFe(pta.psrs).prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    assert pack.path == {"auto": "i8", "fp64": "fp64"}[sweep_path]
    freqs = _freqs(pta)
    pairs = [(i, j) for i in range(5) for j in range(5) if i != j]
    got = pack.fe_sweep(freqs, *_pair_patterns(pairs, 5))
    terms = pack.fp_sweep(freqs, terms=True)
    _, tc = truth.fp_sweep_truth(freqs, pta.toas, pta.residuals, pta.Nvecs, pta.Ts, pta.sigmas)
    for k, (i, j) in enumerate(pairs):
        diff = np.abs(got[k] - (terms[i] + terms[j]))
        tol = 8 * EPS * (tc[i] + tc[j])
        assert np.all(diff <= tol), f"pair {(i, j)}: worst diff / tol {(diff / tol).max():.3g}"


# ---- 5. exact properties ---------------------------------------------------------------------------------------------
def test_pattern_scaling_and_sky_permutation_are_exact(sweep_path):
    """Fe is homogeneous of degree 0 in (F+, Fx): a power-of-two scaling is exact in every step of the combine, so the
    map and the sky maximum are unchanged bit for bit. Each sky row is computed on its own: permuting the rows
    permutes the map, and the sky maximum follows the permutation."""
    pta = synth.make_pta(5, [300, 257, 411, 350, 280], n_tm=[6, 8, 5, 7, 6], ncomps=10, seed=51)
    pack = fastfp_b200.FastFe(pta.psrs).prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    assert pack.path == {"auto": "i8", "fp64": "fp64"}[sweep_path]
    rng = np.random.default_rng(5)
    fp, fx = antenna_pattern(_pos(pta), np.arccos(rng.uniform(-1, 1, 40)), rng.uniform(0, 2 * np.pi, 40))
    freqs = _freqs(pta)
    base = pack.fe_sweep(freqs, fp, fx)
    bmax, bidx = pack.fe_skymax(freqs, fp, fx)
    assert np.all(np.isfinite(base)) and np.all(bidx >= 0)
    for k in (-3, 5):
        s = 2.0 ** k
        np.testing.assert_array_equal(pack.fe_sweep(freqs, s * fp, s * fx), base)
        v, i = pack.fe_skymax(freqs, s * fp, s * fx)
        np.testing.assert_array_equal(v, bmax)
        np.testing.assert_array_equal(i, bidx)
    perm = rng.permutation(40)
    np.testing.assert_array_equal(pack.fe_sweep(freqs, fp[perm], fx[perm]), base[perm])
    v, i = pack.fe_skymax(freqs, fp[perm], fx[perm])
    np.testing.assert_array_equal(v, bmax)
    unique = (base == bmax[None, :]).sum(0) == 1
    assert unique.all()
    np.testing.assert_array_equal(perm[i], bidx)


# ---- 6. frequency batches of fastfp_fe_sweep ---------------------------------------------------------------------------
def test_frequency_batches(sweep_path):
    """P = 200 short pulsars: fastfp_fe_sweep takes FB = 2^27 / (5 P) = 134217 frequencies per sweep, so F = 150000
    spans two batches. Split calls give the full call's bits; bins on both sides of the boundary match the truth."""
    P, F = 200, 150_000
    pta = synth.make_pta(P, 40, n_tm=3, ncomps=2, seed=61)
    FB = (1 << 27) // (5 * P)
    assert FB < F < 2 * FB
    pack = fastfp_b200.FastFe(pta.psrs).prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    assert pack.path == {"auto": "i8", "fp64": "fp64"}[sweep_path]
    freqs = np.linspace(1e-9, 4e-7, F)
    fp, fx = (a[:4] for a in _sky(_pos(pta), seed=6))
    full = pack.fe_sweep(freqs, fp, fx)
    assert full.shape == (4, F) and np.all(np.isfinite(full))
    for cut in (FB, 70_001):
        split = np.concatenate((pack.fe_sweep(freqs[:cut], fp, fx), pack.fe_sweep(freqs[cut:], fp, fx)), axis=1)
        np.testing.assert_array_equal(split, full)
    idx = np.array([0, 1, FB - 2, FB - 1, FB, FB + 1, F - 1])
    _assert_near(full[:, idx], *_truth(freqs[idx], pta, fp, fx)[:3], "bins around the batch boundary")


# ---- 7. the library sincos path ----------------------------------------------------------------------------------------
def test_library_sincos_path(sweep_path):
    """Phases beyond the Cody-Waite range (|phi| > 1e5 rad) take the library sincos path."""
    pta = synth.make_pta(3, [300, 257, 411], n_tm=[6, 8, 5], ncomps=10, seed=71)
    pack = fastfp_b200.FastFe(pta.psrs).prepare(pta.Nvecs, pta.Ts, pta.sigmas)
    assert pack.path == {"auto": "i8", "fp64": "fp64"}[sweep_path]
    freqs = np.array([5e-5, 1.2345e-4])
    assert (2 * np.pi * freqs[0] * np.concatenate(pta.toas)).max() > 1e5
    fp, fx = _sky(_pos(pta), seed=7)
    _assert_near(pack.fe_sweep(freqs, fp, fx), *_truth(freqs, pta, fp, fx)[:3], "library sincos")


# ---- 8. block-diagonal N in the wide families ------------------------------------------------------------------------
@pytest.mark.parametrize("m,family", [(153, "wide"), (313, "xwide")])
def test_block_n_fe_in_the_wide_families(m, family):
    """Against the Sherman-Morrison truth with the block-N allowance of test_gpu_blockn_families.py (256 eps cond:
    there is no float64 block-N oracle to measure E against)."""
    fam, ci = blockn_config(m)
    assert fam == family
    pta, Nvecs, tblocks, _, sig = blockn_case(m, seed=800)
    pack = fastfp_b200.FastFe(pta.psrs).prepare(Nvecs, pta.Ts, sig)
    assert pack.path == "fp64" and pack.m == [m] * 3 and all(n % ci == 0 for n in pack.n)
    freqs = _freqs(pta)
    fp, fx = _sky(_pos(pta), seed=m)
    inner = truth.sweep_inner_truth_blockn(freqs, pta.toas, pta.residuals, tblocks, pta.Ts, sigmas=sig)
    fe, cond = truth.fe_truth_from_inner(inner, freqs, fp, fx)
    _assert_near(pack.fe_sweep(freqs, fp, fx), fe, cond, 64.0, f"block-N m={m} ({fam}, CI={ci})")


# ---- 9. f <= 0 ---------------------------------------------------------------------------------------------------------
def test_non_positive_frequencies_give_nan(sweep_path):
    """f <= 0 gives NaN, as f**(1/3) does in the reference convention and as Fp does. Fe is even in f (s flips sign
    with f), so the inner products themselves must be masked, not only the Fp term."""
    pta = synth.make_pta(4, [300, 257, 411, 350], n_tm=[6, 8, 5, 7], ncomps=10, seed=91)
    fe = fastfp_b200.FastFe(pta.psrs)
    a = (pta.Nvecs, pta.Ts, pta.sigmas)
    assert fe.prepare(*a).path == {"auto": "i8", "fp64": "fp64"}[sweep_path]
    pos_f = synth.fp_freqs(40)[10:13]
    freqs = np.concatenate((NAN_F, pos_f))
    th, ph = np.array([0.3, 1.2, 2.6]), np.array([0.1, 3.0, 5.5])
    got = fe.calculate_Fe(freqs, th, ph, *a)
    assert np.isnan(got[:, :3]).all()
    np.testing.assert_array_equal(got[:, 3:], fe.calculate_Fe(pos_f, th, ph, *a))
    for f in NAN_F:
        assert np.isnan(fe.calculate_Fe(float(f), 0.7, 2.0, *a))
        assert np.isnan(fe.calculate_Fe_skymax(float(f), th, ph, *a)[0])
        assert fe.calculate_Fe_skymax(float(f), th, ph, *a)[1] == -1
    v, i = fe.calculate_Fe_skymax(freqs, th, ph, *a)
    assert np.isnan(v[:3]).all() and (i[:3] == -1).all()
    w, j = fe.calculate_Fe_skymax(pos_f, th, ph, *a)
    np.testing.assert_array_equal(v[3:], w)
    np.testing.assert_array_equal(i[3:], j)
    # Fp of the same pack is unchanged: NaN at f <= 0, the same bits elsewhere
    fp = fe.calculate_Fp(freqs, *a)
    assert np.isnan(fp[:3]).all()
    np.testing.assert_array_equal(fp[3:], fe.calculate_Fp(pos_f, *a))
    np.testing.assert_array_equal(fp, fastfp_b200.FastFp(pta.psrs)(freqs, *a))
