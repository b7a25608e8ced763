"""Block-diagonal N (kernel ECORR) in every kernel family of the fp64 sweep, and on the edges of the epoch-slot
machinery. Block-N pulsars run on their own instantiations, fp_sweep_kernel<C, NMFP, ECORR = true>: 8 epoch-slot rows
at MP-8 .. MP-1 of the G tile (behind zero padding where the family rounds MP up), a slot warp (the last warp row)
that folds beta_e A^x A^y into the b-sums when an epoch ends, and open epoch sums kept in registers across the
level-2 flushes. Every case is checked against the longdouble Sherman-Morrison truth (oracle/truth.py), which
tests/test_oracle_golden.py pins to the GP-basis formulation the reference implements."""
import ctypes as C

import numpy as np
import pytest

import fastfp_b200
from conftest import EPS
from fastfp_b200 import NMFP, BlockNvec, RN_container, _cabi, blockn, synth
from oracle import fe_oracle
from oracle import fp_oracle as o
from oracle import truth
from test_blockn_layout_host import (BLOCKN_MAX_M, assert_edge_layout, blockn_rows, edge_blocks, edge_epochs,
                                     family_of, random_epochs)

pytestmark = pytest.mark.gpu

# the bottom and the top width of every family: m -> (family, timing-model columns, Fourier components)
WIDTHS = {1: ("w1", 1, 0), 32: ("w1", 12, 10), 33: ("w2", 13, 10), 72: ("w2", 12, 30), 73: ("w4", 13, 30),
          152: ("w4", 92, 30), 153: ("wide", 93, 30), 312: ("wide", 252, 30), 313: ("xwide", 253, 30),
          632: ("xwide", 572, 30)}


def _config(m):
    """The kernel configuration a block-N pulsar of width m gets: (family, CI), checked against the library."""
    fam, ci, _ = family_of(blockn_rows(m))
    assert _cabi.load().fastfp_sweep_chunk_toas(m, 1) == ci, m
    return fam, ci


def _blocks(pta, rng, diagonal=(2,), long_at=1):
    """Random epochs of 1-8 TOAs with gaps on every pulsar but those in ``diagonal`` (plain vector N), one 70-TOA epoch
    on pulsar ``long_at``. Returns the Nvecs to pass, the truth's (nvec, spans, jvec) and the block-N TNTs."""
    Nvecs, tblocks, TNTs = [], [], []
    for p, (nvec, T) in enumerate(zip(pta.Nvecs, pta.Ts)):
        sl = [] if p in diagonal else random_epochs(nvec.shape[0], rng, long_at=4 if p == long_at else None)
        jv = rng.uniform(0.3, 3.0, len(sl)) * 1e-13
        B = BlockNvec(nvec, sl, jv)
        Nvecs.append(nvec if p in diagonal else B)
        tblocks.append((nvec, [(s.start, s.stop) for s in sl], jv))
        TNT = T.T @ B.solve(T)
        TNTs.append(0.5 * (TNT + TNT.T))
    return Nvecs, tblocks, TNTs


def _case(m, seed, inc_cp=True):
    fam, n_tm, ncomps = WIDTHS[m]
    pta = synth.make_pta(3, [m + 301, m + 433, m + 377], n_tm=n_tm, ncomps=ncomps, white_only=ncomps == 0,
                         inc_cp=inc_cp, seed=seed + m)
    assert [T.shape[1] for T in pta.Ts] == [m] * 3
    Nvecs, tblocks, TNTs = _blocks(pta, np.random.default_rng(seed + m))
    sig = [TNT + np.diag(1.0 / phi) for TNT, phi in zip(TNTs, pta.phis)]
    return pta, Nvecs, tblocks, TNTs, sig


def _freqs(pta):
    # 73 bins, not a multiple of any tile; as in test_gpu_fp.py::test_every_kernel_family_against_oracle, enough of
    # them lie above the band a wide timing model spans (its high polynomial orders absorb the lowest bins)
    return np.concatenate((synth.fp_freqs(70), np.array([1.0, 2.5, 7.0]) / pta.Tspan))


def _assert_near_truth(got, tt, cond, what):
    """|got - truth| <= 1e-10 |truth| + 256 eps cond wherever the reference formula carries digits at all."""
    tv = np.asarray(tt, dtype=np.float64)
    tol = 1e-10 * np.abs(tv) + 256 * EPS * cond
    # a bin whose conditioning figure times eps reaches the size of the term carries no digits in the reference
    # formula either (test_gpu_fp.py::test_every_kernel_family_against_oracle)
    defined = EPS * cond < 0.05 * np.abs(tv)
    assert defined.mean() > 0.9, what
    ratio = np.where(defined, np.abs(got - tv) / tol, 0.0)
    worst = tuple(int(i) for i in np.unravel_index(np.argmax(ratio), ratio.shape))
    assert np.all(ratio <= 1), (f"{what}: worst |got - truth| / tol = {ratio.max():.3g} at {worst}: got "
                                f"{got[worst]:.6g}, truth {tv[worst]:.6g}, cond {cond[worst]:.3g}")


@pytest.mark.parametrize("m", sorted(WIDTHS))
def test_block_n_fp_in_every_family(m):
    fam, ci = _config(m)
    assert fam == WIDTHS[m][0]
    pta, Nvecs, tblocks, _, sig = _case(m, seed=100)
    freqs = _freqs(pta)
    fp = fastfp_b200.FastFp(pta.psrs, path="auto")
    got = fp.per_pulsar_terms(freqs, Nvecs, pta.Ts, sig)
    pack = fp.prepare(Nvecs, pta.Ts, sig)
    assert pack.m == [m] * 3 and all(n % ci == 0 for n in pack.n) and pack.path == "fp64"
    tt, cond = truth.fp_sweep_truth_blockn(freqs, pta.toas, pta.residuals, tblocks, pta.Ts, sigmas=sig)
    _assert_near_truth(got, tt, cond, f"m={m} ({fam}, CI={ci}), (pulsar, bin)")
    # deterministic, and the summed statistic is the ordered pulsar sum
    np.testing.assert_array_equal(fp.per_pulsar_terms(freqs, Nvecs, pta.Ts, sig), got)
    np.testing.assert_array_equal(fp(freqs, Nvecs, pta.Ts, sig), (got[0] + got[1]) + got[2])
    # the tensor kernel takes no block-N pulsar: "prefer-i8" falls back to the same fp64 kernel, "i8" refuses
    pre = fastfp_b200.FastFp(pta.psrs, path="prefer-i8")
    np.testing.assert_array_equal(pre.per_pulsar_terms(freqs, Nvecs, pta.Ts, sig), got)
    assert pre.prepare(Nvecs, pta.Ts, sig).path == "fp64"
    with pytest.raises(_cabi.FastFpError):
        fastfp_b200.FastFp(pta.psrs, path="i8").prepare(Nvecs, pta.Ts, sig)


@pytest.mark.parametrize("m", [1, 33, 73, 153, 313])
def test_block_n_bins_do_not_depend_on_their_tile(m):
    """A bin's value does not depend on where in a frequency tile it lands: a block of bins, then odd-shifted slices
    of it swept alone (tiles of 128 / 64 / 32 / 16 / 8 frequencies)."""
    _config(m)
    pta, Nvecs, _, _, sig = _case(m, seed=200)
    grid = synth.fp_freqs(2000)
    fp = fastfp_b200.FastFp(pta.psrs)
    base = fp.per_pulsar_terms(grid[100:401], Nvecs, pta.Ts, sig)
    assert np.all(np.isfinite(base))
    np.testing.assert_array_equal(fp.per_pulsar_terms(grid[137:238], Nvecs, pta.Ts, sig), base[:, 37:138])
    np.testing.assert_array_equal(fp.per_pulsar_terms(grid[105:110], Nvecs, pta.Ts, sig), base[:, 5:10])
    np.testing.assert_array_equal(fp.per_pulsar_terms(grid[400:401], Nvecs, pta.Ts, sig), base[:, 300:])


def test_mixed_families_in_one_block_n_pack():
    """One pulsar of each family (m = 26, 60, 73, 153, 313: CI = 16, 32, 16, 16, 8) plus a diagonal-N pulsar in one
    block-N pack: several kernel groups and per-chunk mask offsets across pulsars of different CI."""
    n_tm = [6, 40, 53, 133, 293, 12]
    pta = synth.make_pta(6, [400, 613, 700, 900, 1100, 500], n_tm=n_tm, ncomps=10, seed=300)
    ms = [T.shape[1] for T in pta.Ts]
    assert [_config(m)[0] for m in ms[:5]] == ["w1", "w2", "w4", "wide", "xwide"]
    Nvecs, tblocks, TNTs = _blocks(pta, np.random.default_rng(300), diagonal=(5,), long_at=3)
    sig = [TNT + np.diag(1.0 / phi) for TNT, phi in zip(TNTs, pta.phis)]
    freqs = _freqs(pta)
    fp = fastfp_b200.FastFp(pta.psrs)
    got = fp.per_pulsar_terms(freqs, Nvecs, pta.Ts, sig)
    for p in range(5):
        one = fastfp_b200.FastFp([pta.psrs[p]]).per_pulsar_terms(freqs, [Nvecs[p]], [pta.Ts[p]], [sig[p]])
        np.testing.assert_array_equal(one[0], got[p], err_msg=f"pulsar {p} (m={ms[p]})")
    tt, cond = truth.fp_sweep_truth_blockn(freqs, pta.toas, pta.residuals, tblocks, pta.Ts, sigmas=sig)
    _assert_near_truth(got, tt, cond, "mixed pack, (pulsar, bin)")
    acc = np.zeros(freqs.shape[0])
    for p in range(6):  # sequential pulsar sum starting from 0 (fastfp.py:71,90)
        acc = acc + got[p]
    np.testing.assert_array_equal(fp(freqs, Nvecs, pta.Ts, sig), acc)


@pytest.mark.parametrize("m,ci", [(20, 16), (72, 32), (400, 8)])
def test_block_n_epoch_slot_edges(m, ci):
    """The layouts of test_blockn_layout_host.py::edge_epochs: all slots closing in one chunk, epochs across, ending at
    and starting at a level-2 flush, a 700-TOA epoch open through a flush, single-TOA epochs, a pulsar whose TOAs are
    all in epochs with an ECORR 1e3 x the white noise (beta_e sum 1/nvec -> 1: the correction cancels the diagonal
    part almost entirely)."""
    assert _config(m)[1] == ci
    n_tm, ncomps = {20: (6, 7), 72: (12, 30), 400: (340, 30)}[m]
    pta = synth.make_pta(3, [n for n, _, _ in edge_epochs()], n_tm=n_tm, ncomps=ncomps, seed=400 + m)
    assert [T.shape[1] for T in pta.Ts] == [m] * 3
    blocks = edge_blocks(pta)
    assert_edge_layout([blockn.prepare(q.toas, q.residuals, B, T, ci)
                        for q, B, T in zip(pta.psrs, blocks, pta.Ts)], ci)
    sig = []
    for B, T, phi in zip(blocks, pta.Ts, pta.phis):
        TNT = T.T @ B.solve(T)
        sig.append(0.5 * (TNT + TNT.T) + np.diag(1.0 / phi))
    freqs = _freqs(pta)
    got = fastfp_b200.FastFp(pta.psrs).per_pulsar_terms(freqs, blocks, pta.Ts, sig)
    tblocks = [(B.nvec, [(s.start, s.stop) for s in B.slices], B.jvec) for B in blocks]
    tt, cond = truth.fp_sweep_truth_blockn(freqs, pta.toas, pta.residuals, tblocks, pta.Ts, sigmas=sig)
    layouts = ["all slots closing in one chunk, epochs across / at level-2 flushes", "single-TOA epochs",
               "every TOA in an epoch, large ECORR"]
    for p, what in enumerate(layouts):
        _assert_near_truth(got[p], tt[p], cond[p], f"m={m} (CI={ci}), pulsar {p} ({what}), bin")


# one width per family for the noise-marginalised path (per-draw block 2 * ncomps <= 128 columns); wide and xwide
# carry a wide timing model as the draw-independent block
NMFP_WIDTHS = [32, 72, 73, 153, 313, 632]


@pytest.mark.parametrize("m", NMFP_WIDTHS)
def test_block_n_nmfp_in_every_family(m):
    _config(m)
    pta, Nvecs, tblocks, TNTs, sig = _case(m, seed=500, inc_cp=False)
    sigs = [RN_container(q, Ffreqs=pta.Ffreqs) for q in pta.psrs]
    D = 5
    samples = synth.draw_samples(pta, D)
    freqs = np.concatenate((synth.nmfp_freqs(3, pta.Tspan) * 1.0071, synth.fp_freqs(70)))  # 73 bins
    nm = NMFP(pta.psrs, sigs)
    got = nm(freqs, samples, Nvecs, pta.Ts, TNTs)
    assert got.shape == (D, freqs.shape[0])
    assert nm.prepare(Nvecs, pta.Ts, TNTs).mvar_total == 3 * 2 * WIDTHS[m][2]  # m_fix = the timing model
    phi_args = [dict(psr_name=q.name, n_tm=pta.n_tm[p], Ffreqs=pta.Ffreqs) for p, q in enumerate(pta.psrs)]
    for d in (0, D - 1):
        pars = {k: v[d] for k, v in samples.items()}
        tt, cond = truth.fp_sweep_truth_blockn(freqs, pta.toas, pta.residuals, tblocks, pta.Ts,
                                               sigmas=o.get_sigmas(pars, TNTs, phi_args))
        _assert_near_truth(got[d], tt.sum(0), cond.sum(0), f"m={m}, draw {d}, bin")
    # a draw equal to the fixed noise values is the plain-Fp sweep with the block-N Sigma
    fixed = nm(freqs, pta.noise, Nvecs, pta.Ts, TNTs)
    plain = fastfp_b200.FastFp(pta.psrs)(freqs, Nvecs, pta.Ts, sig)
    well = freqs > 40.0 / pta.Tspan
    assert well.sum() >= 10
    assert np.abs(fixed[well] / plain[well] - 1).max() < 1e-9


@pytest.mark.parametrize("n_tm,ncomps", [(6, 10), (13, 30)])
def test_block_n_fe_against_gp_basis_oracle(n_tm, ncomps):
    """Fe-statistic on a block-N pack (w1: m = 26, w4: m = 73) against oracle/fe_oracle.py on the widened GP basis
    [T | U] (epoch-indicator columns U, diagonal N, phi extended with jvec)."""
    pta = synth.make_pta(3, [300, 257, 411], n_tm=n_tm, ncomps=ncomps, seed=600)
    m = pta.Ts[0].shape[1]
    assert _config(m)[0] == {26: "w1", 73: "w4"}[m]
    Nvecs, tblocks, TNTs = _blocks(pta, np.random.default_rng(600))
    sig = [TNT + np.diag(1.0 / phi) for TNT, phi in zip(TNTs, pta.phis)]
    Text, sig_ext = [], []
    for (nvec, spans, jv), T, phi in zip(tblocks, pta.Ts, pta.phis):
        U = np.zeros((nvec.shape[0], len(spans)))
        for e, (a, b) in enumerate(spans):
            U[a:b, e] = 1.0
        Te = np.ascontiguousarray(np.concatenate((T, U), axis=1))
        Text.append(Te)
        sig_ext.append(Te.T @ (Te / nvec[:, None]) + np.diag(1.0 / np.concatenate((phi, jv))))
    freqs = np.concatenate((synth.fp_freqs(40)[8::4], np.array([2.5, 7.0]) / pta.Tspan))
    th, ph = np.array([0.3, 2.6]), np.array([0.1, 5.5])
    got = fastfp_b200.FastFe(pta.psrs).calculate_Fe(freqs, th, ph, Nvecs, pta.Ts, sig)
    pos = [q.pos for q in pta.psrs]
    want = np.array([[fe_oracle.calculate_Fe(f, t, p_, pta.toas, pta.residuals, pos, pta.Nvecs, Text, sig_ext)
                      for f in freqs] for t, p_ in zip(th, ph)])
    well = freqs > 40.0 / pta.Tspan
    assert well.sum() >= 6
    assert np.abs(got[:, well] / want[:, well] - 1).max() < 1e-9


def test_get_xcy_block_n_wider_than_the_thread_block():
    """m = 300 basis columns: more than the 256 threads of xcy_kernel, so every per-column loop wraps; n = 1001."""
    rng = np.random.default_rng(7)
    n, m = 1001, 300
    T, nvec = rng.standard_normal((n, m)), rng.uniform(0.5, 2.0, n)
    sl = random_epochs(n, rng, long_at=4)
    B = BlockNvec(nvec, sl, rng.uniform(0.2, 3.0, len(sl)))
    phi = rng.uniform(0.1, 3.0, m)
    x, y = rng.standard_normal(n), rng.standard_normal(n)
    sigma = T.T @ B.solve(T) + np.diag(1.0 / phi)
    Cy = np.linalg.solve(B.dense() + T @ np.diag(phi) @ T.T, y)  # dense known answer
    want = x @ Cy
    got = fastfp_b200.get_xCy(B, T, sigma, x, y)
    assert abs(got - want) < 1e-10 * (np.abs(x) @ np.abs(Cy)), (got, want)


def test_block_n_width_limit():
    """632 columns is the widest block-N basis (640 kernel rows less 8 epoch-slot rows; m = 632 sweeps in
    test_block_n_fp_in_every_family). 633 is refused by the Python layer and by the C ABI."""
    m, n = BLOCKN_MAX_M + 1, 1000
    pta = synth.make_pta(1, n, n_tm=3, white_only=True, seed=700)
    rng = np.random.default_rng(700)
    T = rng.standard_normal((n, m))
    sl = random_epochs(n, rng)
    B = BlockNvec(pta.Nvecs[0], sl, rng.uniform(0.3, 3.0, len(sl)) * 1e-13)
    sigma = T.T @ B.solve(T) + np.eye(m)
    with pytest.raises(ValueError, match="basis width 633"):
        fastfp_b200.FastFp(pta.psrs)(synth.fp_freqs(3), [B], [T], [sigma])
    # the C ABI, with a layout made at the chunk size of the widest kernel
    d = blockn.prepare(pta.psrs[0].toas, pta.psrs[0].residuals, B, T, 8)
    lib = _cabi.load()
    arr = {k: _cabi.as_f64(d[k]) for k in ("toas", "res", "res_w", "Nvec", "T", "slot_val")}
    sidx, done = np.ascontiguousarray(d["slot_idx"]), np.ascontiguousarray(d["done_mask"])
    h = C.c_void_p()
    rc = lib.fastfp_pack_create_blockn(
        0, 1, _cabi._int64_array([d["toas"].shape[0]]), _cabi._int64_array([m]),
        *[_cabi._ptr_array([arr[k]]) for k in ("toas", "res", "res_w", "Nvec", "T")], _cabi._ptr_array([sigma]),
        (C.POINTER(C.c_int32) * 1)(sidx.ctypes.data_as(C.POINTER(C.c_int32))), _cabi._ptr_array([arr["slot_val"]]),
        (C.POINTER(C.c_ubyte) * 1)(done.ctypes.data_as(C.POINTER(C.c_ubyte))), None, None, C.c_void_p(0),
        C.byref(h))
    assert rc == -3 and not h.value  # FASTFP_ERR_UNSUPPORTED, no pack
    msg = lib.fastfp_last_error().decode()
    assert "m=633" in msg and "block-N maximum 632" in msg, msg
