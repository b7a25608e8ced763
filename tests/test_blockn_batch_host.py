"""Host side of residual batches on block-diagonal N packs (no GPU): the epoch layout's prefix property the packet
builder relies on, the factored layout and R-row Sherman-Morrison against ``blockn.prepare``, the block-N row limit and
pass rule, and the refusals of ``fastfp_pack_set_residuals_blockn`` and the front ends that need no pack."""
import numpy as np
import pytest

import fastfp_b200
from conftest import Psr
from fastfp_b200 import BlockNvec, _cabi, blockn
from fastfp_b200.fastfp import _tile_cost, batch_pass_rows


def _pulsar(seed=0, n=900, m=7):
    """Epochs of 1-8 TOAs with gaps (free TOAs), one of 70 TOAs (longer than any chunk), free TOAs at the end."""
    rng = np.random.default_rng(seed)
    sl, a = [], 0
    while a < n - 120:
        ln = 70 if len(sl) == 5 else int(rng.integers(1, 9))
        sl.append(slice(a, a + ln))
        a += ln + int(rng.integers(0, 3))
    nvec = rng.uniform(0.5, 2.0, n) * 1e-12
    B = BlockNvec(nvec, sl, rng.uniform(0.3, 3.0, len(sl)) * 1e-13)
    toas = np.sort(rng.uniform(0.0, 3e8, n))
    return B, toas, rng.standard_normal(n) * 1e-6, rng.standard_normal((n, m))


@pytest.mark.parametrize("seed", [0, 1])
def test_layouts_agree_on_every_real_toa(seed):
    B, toas, res, T = _pulsar(seed)
    preps = {ci: blockn.prepare(toas, res, B, T, ci) for ci in (8, 16, 32)}
    orders = {ci: blockn.layout(blockn.epochs(B, toas.shape[0]), ci)["order"] for ci in preps}
    last = max(int(np.flatnonzero(o >= 0).max()) for o in orders.values())
    for ci, o in orders.items():
        assert o.shape[0] % ci == 0 and o.shape[0] == preps[ci]["toas"].shape[0]
        np.testing.assert_array_equal(o[:last + 1], orders[8][:last + 1])  # every real TOA at the same position
        assert np.all(o[last + 1:] == -1)  # past it, padding only
        for k in ("toas", "res", "res_w", "Nvec", "T"):
            np.testing.assert_array_equal(preps[ci][k][:last + 1], preps[8][k][:last + 1])
    assert sorted(orders[8][orders[8] >= 0]) == list(range(toas.shape[0]))


@pytest.mark.parametrize("ci", [8, 16, 32])
def test_layout_reproduces_prepare(ci):
    B, toas, res, T = _pulsar(2)
    d = blockn.prepare(toas, res, B, T, ci)
    lay = blockn.layout(blockn.epochs(B, toas.shape[0]), ci)
    for k in ("slot_idx", "slot_val", "done_mask"):
        assert lay[k].dtype == d[k].dtype
        np.testing.assert_array_equal(lay[k], d[k])
    np.testing.assert_array_equal(blockn.relay(lay["order"], toas), d["toas"])
    np.testing.assert_array_equal(blockn.relay(lay["order"], res), d["res"])


def test_r_row_sherman_morrison_is_prepare_row_by_row():
    """Bit for bit: solve_rows reduces each epoch along the TOA axis in the same order for one row and for many."""
    B, toas, res, T = _pulsar(3)
    ep = blockn.epochs(B, toas.shape[0])
    X = np.random.default_rng(4).standard_normal((17, toas.shape[0])) * 1e-6
    X[0] = res
    W = blockn.solve_rows(ep, X)
    for k in range(X.shape[0]):
        want = blockn.prepare(toas, X[k], B, T, 16)
        np.testing.assert_array_equal(blockn.relay(blockn.layout(ep, 16)["order"], W[k]), want["res_w"])
    # and it is N^-1 X (times nvec)
    np.testing.assert_allclose(W / B.nvec, B.solve(X.T).T, rtol=1e-12, atol=0)
    # a diagonal N: no correction
    np.testing.assert_array_equal(blockn.solve_rows(blockn.epochs(B.nvec, toas.shape[0]), X), X)


def test_block_n_row_limit_and_pass_rule():
    assert _cabi.max_residual_rows([72], blockn=True) == 560
    assert _cabi.max_residual_rows([12], blockn=True) == 616
    assert _cabi.max_residual_rows([12, 72, 30], blockn=True) == 560
    for m in ([12], [72], [300]):  # the defaults are the diagonal-N rule
        assert _cabi.max_residual_rows(m) == _cabi.max_residual_rows(m, blockn=False)
        for R in (1, 8, 200, 600):
            assert batch_pass_rows(R, m) == batch_pass_rows(R, m, blockn=False)
    for m in ([12], [72], [300]):
        rmax = _cabi.max_residual_rows(m, blockn=True)
        mr = -(-max(m) // 8) * 8 + 8
        for R in list(range(1, 80)) + [248, 249, 300, rmax, rmax + 1, 1500]:
            rows = batch_pass_rows(R, m, blockn=True)
            npass = -(-R // rows)
            assert 1 <= rows <= rmax and rows == -(-R // npass), (m, R, rows)  # passes evened out
            cost = npass * _tile_cost(mr + -(-rows // 8) * 8)
            for cap in range(8, min(R, rmax) + 1, 8):  # no even split the library takes is modelled cheaper
                k = -(-R // cap)
                assert cost <= k * _tile_cost(mr + -(-(-(-R // k)) // 8) * 8)
    # m = 72: 8 slot rows more than the diagonal rule, so the one-pass range ends earlier
    assert batch_pass_rows(240, [72], blockn=True) == 240  # 72 + 240 + 8 = 320 rows: the top of the 16-frequency family
    assert batch_pass_rows(560, [72], blockn=True) == 280  # 2 x 384-row passes model cheaper than one 640-row pass
    assert batch_pass_rows(561, [72], blockn=True) <= 560


def test_set_residuals_blockn_refusals_without_a_pack():
    lib = _cabi.load()
    z = _cabi._ptr_array([np.zeros(8)])
    i32 = (_cabi.C.POINTER(_cabi.C.c_int32) * 1)()
    u8 = (_cabi.C.POINTER(_cabi.C.c_ubyte) * 1)()
    n = _cabi._int64_array([8])
    assert lib.fastfp_pack_set_residuals_blockn(None, 1, n, z, z, i32, z, u8, None) == -1
    assert "null argument or negative R" in lib.fastfp_last_error().decode()
    assert lib.fastfp_pack_set_residuals_blockn(None, -1, None, None, None, None, None, None, None) == -1
    assert lib.fastfp_pack_set_residuals_blockn(None, 0, None, None, None, None, None, None, None) == -1


def _stub_pack(block, n, m, epochs=None):
    pack = object.__new__(_cabi.Pack)
    pack._h, pack.P, pack.nmfp, pack.n, pack.m = None, len(n), False, list(n), list(m)
    pack.blockn, pack.epochs = block, epochs
    return pack


def test_front_end_shape_checks_for_block_n_inputs():
    B, toas, res, T = _pulsar(5, n=300)
    ep = blockn.epochs(B, 300)
    pack = _stub_pack(True, [320], [7], [ep])
    with pytest.raises(ValueError, match=r"shape \(R, 300\)"):  # rows in the original TOA order, not the pack's 320
        pack.set_residuals_blockn([np.zeros((3, 320))])
    with pytest.raises(ValueError, match="one per pulsar"):
        pack.set_residuals_blockn([np.zeros((3, 300))] * 2)
    with pytest.raises(_cabi.FastFpError, match="set_residuals_blockn"):
        pack.set_residuals([np.zeros((3, 320))])
    with pytest.raises(_cabi.FastFpError, match="takes set_residuals"):
        _stub_pack(False, [300], [7]).set_residuals_blockn([np.zeros((3, 300))])
    # FastFp / FastFe check the realisations against the pulsars' own TOA counts before any pack exists
    psr = Psr(toas, res)
    psr.pos = np.array([0.0, 0.0, 1.0])
    sig = [T.T @ B.solve(T) + np.eye(7)]
    fp, fe = fastfp_b200.FastFp([psr]), fastfp_b200.FastFe([psr])
    for call in (lambda r: fp.calculate_Fp_batch(np.array([1e-8]), [B], [T], sig, r),
                 lambda r: fe.calculate_Fe_skymax_batch(np.array([1e-8]), 0.5, 1.0, [B], [T], sig, r)):
        with pytest.raises(ValueError, match=r"residuals\[0\] must have shape \(R, 300\)"):
            call([np.zeros((2, 320))])
        with pytest.raises(ValueError, match="at least one realisation"):
            call([np.zeros((0, 300))])
