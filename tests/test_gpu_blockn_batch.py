"""Residual batches on block-diagonal N packs on the GPU (``Pack.set_residuals_blockn``,
``fastfp_pack_set_residuals_blockn``; ``calculate_Fp_batch`` / ``calculate_Fe_skymax_batch`` with a ``BlockNvec``).
The realisations run on fp_sweep_kernel<C, Res, ECORR = true>: basis rows, w_1 .. w_R, then the 8 epoch-slot rows last,
in the TOA layout of the residual configuration's chunk size, which often differs from the pack's. Every case is
checked against the longdouble Sherman-Morrison truth for that row's residuals."""
import numpy as np
import pytest

import fastfp_b200
from conftest import EPS, Psr
from fastfp_b200 import _cabi, synth
from fastfp_b200.fe import antenna_pattern
from oracle import truth
from test_blockn_layout_host import edge_blocks, edge_epochs, family_of
from test_gpu_blockn_families import _assert_near_truth, _blocks, _freqs
from test_gpu_fe_skymax_batch import _grid, _pos
from test_gpu_fp_batch import realisations

pytestmark = pytest.mark.gpu


def _ci(m, R=0):
    """chunk size of a block-N pulsar of width m with R realisation rows (R = 0: the pack's)"""
    return _cabi.load().fastfp_sweep_chunk_toas(-(-m // 8) * 8 + -(-R // 8) * 8, 1)


def _pta(ns, n_tm, ncomps, seed, diagonal=(2,), long_at=1, white=False):
    pta = synth.make_pta(len(ns), list(ns), n_tm=n_tm, ncomps=ncomps, white_only=white, seed=seed)
    Nvecs, tblocks, TNTs = _blocks(pta, np.random.default_rng(seed), diagonal=diagonal, long_at=long_at)
    sig = [TNT + np.diag(1.0 / phi) for TNT, phi in zip(TNTs, pta.phis)]
    return pta, Nvecs, tblocks, sig


def _truth_row(freqs, pta, res, k, tblocks, sig):
    tt, cond = truth.fp_sweep_truth_blockn(freqs, pta.toas, [r[k] for r in res], tblocks, pta.Ts, sigmas=sig)
    return tt.sum(0).astype(float), cond.sum(0)


def _assert_rows(got, rows, freqs, pta, res, tblocks, sig, what, well=True):
    for k in rows:
        tv, cond = _truth_row(freqs, pta, res, k, tblocks, sig)
        _assert_near_truth(got[k], tv, cond, f"{what}, row {k}")
        if well:  # well-conditioned bins: 1e-10
            good = EPS * cond < 1e-13 * np.abs(tv)
            assert good.any() and np.all(np.abs(got[k] - tv)[good] <= 1e-10 * np.abs(tv[good])), (what, k)


def _ragged():
    """test_gpu_blockn.py's layouts: epochs of 1-8 TOAs, a 70-TOA epoch, free TOAs, a diagonal-N pulsar (m = 72, 70,
    68: the pack's chunk is 32 TOAs, with R = 12 the residual layout's 16)."""
    pta, Nvecs, tblocks, sig = _pta([400, 613, 300], [12, 10, 8], 30, seed=17)
    return pta, Nvecs, tblocks, sig, _freqs(pta)


def test_every_row_against_truth_and_calculate_Fp():
    pta, Nvecs, tblocks, sig, freqs = _ragged()
    assert [T.shape[1] for T in pta.Ts] == [72, 70, 68] and _ci(72) == 32 and _ci(72, 12) == 16
    R = 12
    res = realisations(pta, R, seed=3)
    fp = fastfp_b200.FastFp(pta.psrs)
    got = fp.calculate_Fp_batch(freqs, Nvecs, pta.Ts, sig, res)
    assert got.shape == (R, freqs.shape[0]) and np.all(np.isfinite(got))
    _assert_rows(got, range(R), freqs, pta, res, tblocks, sig, "ragged block-N PTA")
    for k in (0, 5, R - 1):  # row k against a block-N FastFp built with residuals r_k: the parity bar, not the bits
        one = fastfp_b200.FastFp([Psr(q.toas, r[k]) for q, r in zip(pta.psrs, res)])(freqs, Nvecs, pta.Ts, sig)
        tv, cond = _truth_row(freqs, pta, res, k, tblocks, sig)
        defined = EPS * cond < 0.05 * np.abs(tv)
        assert np.all(np.where(defined, np.abs(got[k] - one) <= 2 * (1e-10 * np.abs(tv) + 256 * EPS * cond), True)), k
    np.testing.assert_array_equal(fp.calculate_Fp_batch(freqs[7], Nvecs, pta.Ts, sig, res), got[:, 7])


def test_exact_properties():
    pta, Nvecs, tblocks, sig, freqs = _ragged()
    R = 12
    res = realisations(pta, R, seed=4)
    fp = fastfp_b200.FastFp(pta.psrs)
    a = (Nvecs, pta.Ts, sig)
    got = fp.calculate_Fp_batch(freqs, *a, res)
    np.testing.assert_array_equal(fp.calculate_Fp_batch(freqs, *a, res), got)  # repeatable
    two = [r.copy() for r in res]
    for r in two:
        r[3] = 2 * r[1]
    np.testing.assert_array_equal(fp.calculate_Fp_batch(freqs, *a, two)[3], 4 * got[1])  # 2r: exactly 4x
    perm = np.random.default_rng(0).permutation(R)
    np.testing.assert_array_equal(fp.calculate_Fp_batch(freqs, *a, [r[perm] for r in res]), got[perm])
    bad = [r.copy() for r in res]
    bad[1][6, 17] = np.nan
    gb = fp.calculate_Fp_batch(freqs, *a, bad)
    assert np.all(np.isnan(gb[6])) and np.all(np.isfinite(np.delete(gb, 6, axis=0)))
    np.testing.assert_array_equal(np.delete(gb, 6, axis=0), np.delete(got, 6, axis=0))
    # no dependence on the frequency tiles or batches: halves of the grid swept alone, and a grid of several batches
    h = freqs.shape[0] // 2 + 3
    np.testing.assert_array_equal(fp.calculate_Fp_batch(freqs[h:], *a, res), got[:, h:])
    big = np.concatenate((synth.fp_freqs(2 ** 27 // (R * 3) + 500), freqs))
    np.testing.assert_array_equal(fp.calculate_Fp_batch(big, *a, res)[:, -freqs.shape[0]:], got)
    # an in-place edit of the realisations is seen
    for r in res:
        r[4] *= 2.0
    np.testing.assert_array_equal(fp.calculate_Fp_batch(freqs, *a, res)[4], 4 * got[4])
    # R = 0 releases the set: pack.nbytes returns to its value before
    pack = fp.prepare(*a)
    pack.set_residuals_blockn([r[:0] for r in res])
    before = pack.nbytes
    pack.set_residuals_blockn([r[:5] for r in res])
    assert pack.nbytes > before and pack.R == 5
    pack.set_residuals_blockn([r[:0] for r in res])
    assert pack.nbytes == before
    fp._res_pack = None


# (m, n_tm, ncomps, R): the bottom and top of each family's Res+ECORR row range roundup8(m) + roundup8(R) + 8, with
# the pack's and the residual layout's chunk size
FAMILY_CASES = [
    (1, 1, 0, 1),      # 24 rows: w1 (CI 16 -> 16)
    (16, 6, 5, 16),    # 40: top of w1
    (26, 6, 10, 8),    # 48: w2, CI 16 -> 32
    (26, 6, 10, 40),   # 80: top of w2
    (72, 12, 30, 8),   # 88: w4, CI 32 -> 16
    (72, 12, 30, 80),  # 160: top of w4
    (72, 12, 30, 88),  # 168: wide
    (72, 12, 30, 240),  # 320: top of wide
    (72, 12, 30, 248),  # 328: xwide, CI 32 -> 8
]


@pytest.mark.parametrize("m,n_tm,ncomps,R", FAMILY_CASES)
def test_every_family(m, n_tm, ncomps, R):
    rows = -(-m // 8) * 8 + -(-R // 8) * 8 + 8
    fam, ci, _ = family_of(rows)
    assert _ci(m, R) == ci
    pta, Nvecs, tblocks, sig = _pta([m + 301, m + 433, m + 377], n_tm, ncomps, seed=800 + m, white=ncomps == 0)
    assert [T.shape[1] for T in pta.Ts] == [m] * 3
    res = realisations(pta, R, seed=m + R)
    freqs = _freqs(pta)
    got = fastfp_b200.FastFp(pta.psrs).calculate_Fp_batch(freqs, Nvecs, pta.Ts, sig, res)
    _assert_rows(got, sorted({0, R // 2, R - 1}), freqs, pta, res, tblocks, sig,
                 f"m={m}, R={R}: {rows} rows ({fam}, CI {_ci(m)} -> {ci})", well=ncomps > 0)


@pytest.mark.parametrize("m,R", [(72, 8), (72, 248), (20, 24)])
def test_epoch_slot_edges(m, R):
    """test_blockn_layout_host.py::edge_epochs in the residual layout: all 8 slots closing in one chunk, epochs across,
    ending at and starting at a level-2 flush, single-TOA epochs, every TOA in an epoch with a large ECORR."""
    n_tm, ncomps = {20: (6, 7), 72: (12, 30)}[m]
    pta = synth.make_pta(3, [n for n, _, _ in edge_epochs()], n_tm=n_tm, ncomps=ncomps, seed=400 + m)
    blocks = edge_blocks(pta)
    sig = []
    for B, T, phi in zip(blocks, pta.Ts, pta.phis):
        TNT = T.T @ B.solve(T)
        sig.append(0.5 * (TNT + TNT.T) + np.diag(1.0 / phi))
    tblocks = [(B.nvec, [(s.start, s.stop) for s in B.slices], B.jvec) for B in blocks]
    res = realisations(pta, R, seed=9)
    freqs = _freqs(pta)
    got = fastfp_b200.FastFp(pta.psrs).calculate_Fp_batch(freqs, blocks, pta.Ts, sig, res)
    for k in sorted({0, R - 1}):
        tt, cond = truth.fp_sweep_truth_blockn(freqs, pta.toas, [r[k] for r in res], tblocks, pta.Ts, sigmas=sig)
        tv = tt.astype(float)
        # per pulsar: the terms of one row are the Fp of that row with the other pulsars' terms, so compare the sum
        _assert_near_truth(got[k], tv.sum(0), cond.sum(0), f"m={m}, R={R} (CI {_ci(m, R)}), row {k}")


def test_the_row_limit():
    """R = 632 - roundup8(m) runs in one pass; one more is refused by the library; calculate_Fp_batch splits it."""
    pta, Nvecs, tblocks, sig = _pta([300, 257, 411], [12, 12, 12], 30, seed=900, diagonal=(1,), long_at=0)
    freqs = _freqs(pta)[::3]
    rmax = 632 - 72
    assert _cabi.max_residual_rows([T.shape[1] for T in pta.Ts], blockn=True) == rmax
    res = realisations(pta, rmax + 1, seed=10)
    fp = fastfp_b200.FastFp(pta.psrs)
    pack = fp.prepare(Nvecs, pta.Ts, sig)
    pack.set_residuals_blockn([r[:rmax] for r in res])
    one = pack.fp_sweep_residuals(freqs)
    assert one.shape == (rmax, freqs.shape[0])
    with pytest.raises(_cabi.FastFpError, match=r"error -3: .*limit of 560 .*widest pulsar 0 \(m = 72\)"):
        pack.set_residuals_blockn(res)
    got = fp.calculate_Fp_batch(freqs, Nvecs, pta.Ts, sig, res)  # passes of batch_pass_rows rows
    _assert_rows(got, [0, rmax // 2, rmax], freqs, pta, res, tblocks, sig, "split R = 561", well=False)
    for k in (0, 123, rmax - 1):
        tv, cond = _truth_row(freqs, pta, res, k, tblocks, sig)
        defined = EPS * cond < 0.05 * np.abs(tv)
        tol = 2 * (1e-10 * np.abs(tv) + 256 * EPS * cond)
        assert np.all(np.where(defined, np.abs(got[k] - one[k]) <= tol, True)), k


def test_fe_skymax_batch():
    pta, Nvecs, tblocks, sig = _pta([300, 411, 257], [8, 8, 8], 10, seed=41)
    freqs = np.concatenate((synth.fp_freqs(24), np.array([2.5, 7.0]) / pta.Tspan))
    pos = _pos(pta)
    th, ph = _grid(pos, 30, seed=5)
    assert th[-2] == 0.0  # the pole
    R = 6
    res = realisations(pta, R, seed=12)
    fe = fastfp_b200.FastFe(pta.psrs)
    best, idx = fe.calculate_Fe_skymax_batch(freqs, th, ph, Nvecs, pta.Ts, sig, res)
    assert best.shape == idx.shape == (R, freqs.shape[0])
    fplus, fcross = antenna_pattern(pos, th, ph)
    cols = np.arange(freqs.shape[0])
    b0, i0 = fastfp_b200.FastFe(pta.psrs).calculate_Fe_skymax(freqs, th, ph, Nvecs, pta.Ts, sig)
    for k in range(R):
        fet, cond = truth.fe_truth(freqs, fplus, fcross, pta.toas, [r[k] for r in res], None, pta.Ts, sig,
                                   blocks=tblocks)
        fet = fet.astype(float)
        tol = 1e-9 * np.abs(fet) + 1024 * EPS * cond
        defined = EPS * cond < 0.05 * np.abs(fet)
        at = (idx[k], cols)
        assert np.all(np.where(defined[at], np.abs(best[k] - fet[at]) <= tol[at], True)), k
        am = np.nanargmax(fet, axis=0)
        srt = np.sort(np.where(np.isnan(fet), -np.inf, fet), axis=0)
        clear = defined[am, cols] & (srt[-1] - srt[-2] > tol[am, cols] + tol[idx[k], cols])
        assert np.all(np.where(clear, idx[k] == am, True)), k
        if k == 0:  # the pulsars' own residuals: calculate_Fe_skymax on its own block-N pack, within the parity bar
            same = defined[at] & (i0 == idx[0])
            assert same.mean() > 0.8 and np.all(np.where(same, np.abs(best[0] - b0) <= 2 * tol[at], True))


def test_pure_patterns_equal_the_fp_batch():
    """Pulsar 0 with (F+, Fx) = (1, 0), pulsar 1 with (0, 1): Fe decouples into the two pulsars' Fp terms."""
    pta, Nvecs, tblocks, sig = _pta([300, 257], [12, 8], 10, seed=46, diagonal=(), long_at=0)
    res = realisations(pta, 9, seed=46)
    freqs = _freqs(pta)
    pack = fastfp_b200.FastFe(pta.psrs).prepare(Nvecs, pta.Ts, sig)
    pack.set_residuals_blockn(res)
    best, idx = pack.fe_skymax_residuals(freqs, np.array([[1.0, 0.0]]), np.array([[0.0, 1.0]]))
    assert np.all(idx == 0)
    fpb = pack.fp_sweep_residuals(freqs)
    for k in range(9):
        tv, cond = _truth_row(freqs, pta, res, k, tblocks, sig)
        _assert_near_truth(best[k], tv, cond, f"pure patterns, row {k}")
        defined = EPS * cond < 0.05 * np.abs(tv)
        tol = 2 * (1e-10 * np.abs(tv) + 256 * EPS * cond)
        assert np.all(np.where(defined, np.abs(best[k] - fpb[k]) <= tol, True)), k


def test_cuda_tensor_on_a_non_default_stream():
    import torch

    pta, Nvecs, tblocks, sig, freqs = _ragged()
    res = realisations(pta, 9, seed=13)
    fp = fastfp_b200.FastFp(pta.psrs)
    host = fp.calculate_Fp_batch(freqs, Nvecs, pta.Ts, sig, res)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        dev = fp.calculate_Fp_batch(torch.from_numpy(freqs).cuda(), Nvecs, pta.Ts, sig, res)
        out = dev.cpu()
    assert dev.is_cuda
    np.testing.assert_array_equal(out.numpy(), host)
