"""Every pack gives back all the device memory it took: after a pack of each kind is built, used so that each of its
scratch buffers grows, and destroyed, the library holds exactly the device bytes it held before
(``fastfp_device_bytes``, counted at every allocation and release, unaffected by other work on the device). Builds
that fail part-way give theirs back too. Run with -m gpu on an H100."""
import gc

import numpy as np
import pytest

from fastfp_b200 import BlockNvec, _cabi, synth

pytestmark = pytest.mark.gpu

NCOMPS = 10  # Fourier components: 2 * NCOMPS per-draw columns of an nmfp pack


def _sky(P, S=48, seed=5):
    rng = np.random.default_rng(seed)
    return rng.uniform(-1, 1, (S, P)), rng.uniform(-1, 1, (S, P))


def _plain(pta, path=None):
    pack = _cabi.Pack.create(pta.toas, pta.residuals, pta.Nvecs, pta.Ts, pta.sigmas)
    if path:
        pack.set_path(path)
        assert pack.path == path
    return pack


def _blockn_lists(pta, seed=17):
    """A block-diagonal N (epochs of 1-8 TOAs) for every pulsar, and the sigmas and TNTs that go with it."""
    rng = np.random.default_rng(seed)
    blocks, sigmas, TNTs = [], [], []
    for p, N in enumerate(pta.Nvecs):
        n, sl, a = N.shape[0], [], 0
        while a < n - 8:
            ln = int(rng.integers(1, 9))
            sl.append(slice(a, a + ln))
            a += ln + int(rng.integers(0, 2))
        B = BlockNvec(N, sl, rng.uniform(0.3, 3.0, len(sl)) * 1e-13)
        T = pta.Ts[p]
        TNT = T.T @ B.solve(T)
        TNT = 0.5 * (TNT + TNT.T)
        blocks.append(B)
        TNTs.append(TNT)
        sigmas.append(TNT + np.diag(1.0 / pta.phis[p]))
    return blocks, sigmas, TNTs


def _nmfp(pta, Nvecs, TNTs, ncomps=NCOMPS):
    m_fix = [T.shape[1] - 2 * ncomps for T in pta.Ts]
    return _cabi.Pack.create(pta.toas, pta.residuals, Nvecs, pta.Ts, TNTs, m_fix=m_fix,
                             phiinv_fix=[np.full(k, 1e-40) for k in m_fix])


def _exercise_fp(pack, residuals=None):
    """Every sweep of a plain-Fp pack, at sizes that grow each of its scratch buffers."""
    freqs = synth.fp_freqs(300)
    fplus, fcross = _sky(pack.P)
    assert pack.fp_sweep(freqs).shape == (freqs.size,)
    assert pack.fp_sweep(freqs, terms=True).shape == (pack.P, freqs.size)
    assert pack.fe_sweep(freqs, fplus, fcross).shape == (fplus.shape[0], freqs.size)
    fe, idx = pack.fe_skymax(freqs, fplus, fcross)
    assert fe.shape == idx.shape == (freqs.size,)
    if residuals is None:
        return
    rng = np.random.default_rng(9)
    for R in (8, 40):  # the second set replaces the first
        pack.set_residuals([r + 1e-7 * rng.standard_normal((R, r.size)) for r in residuals])
        assert _cabi.device_bytes() >= pack.nbytes
        assert pack.fp_sweep_residuals(freqs).shape == (R, freqs.size)
        fe, idx = pack.fe_skymax_residuals(freqs, fplus, fcross)
        assert fe.shape == idx.shape == (R, freqs.size)
    pack.set_residuals([np.zeros((0, r.size)) for r in residuals])


def _exercise_nmfp(pack, pta, ncomps=NCOMPS):
    """The device power law with a growing draw count, then the sweep with host parameters and stage timing."""
    import torch

    rng = np.random.default_rng(3)
    Ff = [pta.Ffreqs[: 2 * ncomps]] * pack.P
    phiinv = None
    for D in (4, 9, 24):
        A, G = rng.uniform(-15, -13, (D, pack.P)), rng.uniform(2, 5, (D, pack.P))
        out = torch.empty((D, pack.mvar_total), dtype=torch.float64, device="cuda")
        pack.powerlaw_phiinv(Ff, A, G, None, None, None, out.data_ptr())
        torch.cuda.synchronize()
        phiinv = out.cpu().numpy()
    pack.stage_timing(True)
    got = pack.nmfp_sweep(synth.nmfp_freqs(70, pta.Tspan), phiinv, phiinv.shape[0])
    assert got.shape == (phiinv.shape[0], 70)
    assert all(ms >= 0 for ms in pack.stage_ms())


def _gives_back_everything(build, exercise):
    gc.collect()
    before = _cabi.device_bytes()
    pack = build()
    assert _cabi.device_bytes() - before >= pack.nbytes > 0
    exercise(pack)
    assert _cabi.device_bytes() - before >= pack.nbytes
    del pack
    gc.collect()
    assert _cabi.device_bytes() == before


def test_plain_pack_on_the_tensor_path():
    pta = synth.make_pta(3, [900, 1203, 517], n_tm=[8, 10, 7], ncomps=NCOMPS, seed=41)
    _gives_back_everything(lambda: _plain(pta, "i8"), lambda pk: _exercise_fp(pk, pta.residuals))


def test_mixed_pack():
    # pulsar 0 is beyond the tensor kernel's 16 384 TOAs: the fp64 kernel sweeps it, the tensor kernel the other
    pta = synth.make_pta(2, [16385, 700], n_tm=[7, 9], ncomps=NCOMPS, seed=42)
    _gives_back_everything(lambda: _plain(pta, "mixed"), lambda pk: _exercise_fp(pk, pta.residuals))


def test_block_n_pack():
    pta = synth.make_pta(3, [400, 613, 300], n_tm=[8, 12, 10], ncomps=NCOMPS, seed=43)
    blocks, sigmas, _ = _blockn_lists(pta)
    _gives_back_everything(lambda: _cabi.Pack.create(pta.toas, pta.residuals, blocks, pta.Ts, sigmas), _exercise_fp)


def test_nmfp_pack():
    pta = synth.make_pta(3, [700, 1203, 333], n_tm=[8, 12, 5], ncomps=NCOMPS, seed=44)
    _gives_back_everything(lambda: _nmfp(pta, pta.Nvecs, pta.TNTs), lambda pk: _exercise_nmfp(pk, pta))


def test_block_n_nmfp_pack():
    pta = synth.make_pta(3, [400, 613, 300], n_tm=[8, 12, 10], ncomps=NCOMPS, seed=45)
    blocks, _, TNTs = _blockn_lists(pta)
    _gives_back_everything(lambda: _nmfp(pta, blocks, TNTs), lambda pk: _exercise_nmfp(pk, pta))


def test_failed_builds_give_back_what_they_took():
    gc.collect()
    before = _cabi.device_bytes()
    # 66 Fourier components = 132 per-draw columns: refused after the pack's core buffers exist
    wide = synth.make_pta(2, [300, 200], n_tm=[8, 6], ncomps=66, seed=46)
    with pytest.raises(_cabi.FastFpError, match="more than 128 per-draw columns"):
        _nmfp(wide, wide.Nvecs, wide.TNTs, ncomps=66)
    assert _cabi.device_bytes() == before
    # a residual batch above the row limit is refused and leaves the pack as it was
    pta = synth.make_pta(2, [300, 200], n_tm=[8, 6], ncomps=NCOMPS, seed=47)
    pack = _plain(pta)
    held = _cabi.device_bytes()
    R = _cabi.max_residual_rows(pack.m) + 1
    with pytest.raises(_cabi.FastFpError, match="exceeds the limit"):
        pack.set_residuals([np.zeros((R, r.size)) for r in pta.residuals])
    assert _cabi.device_bytes() == held
    del pack
    gc.collect()
    assert _cabi.device_bytes() == before
