"""Row groups of bases wider than one sweep work item (DESIGN.md section 5h), without a GPU: the split rule at its edges,
the row-to-group map, and the refusals the Python side makes before any device work."""
import numpy as np
import pytest

from fastfp_b200 import _cabi, synth
from fastfp_b200.fastfp import batch_pass_rows


def test_split_rule_at_the_edges():
    assert _cabi.MAX_M == 640 and _cabi.MAX_M_WIDE == 2688
    assert _cabi.row_groups(1) == [(0, 1)]
    assert _cabi.row_groups(640) == [(0, 640)]
    assert _cabi.row_groups(641) == [(0, 216), (216, 432), (432, 641)]
    assert _cabi.row_groups(864) == [(0, 288), (288, 576), (576, 864)]
    assert len(_cabi.row_groups(865)) == 4
    assert _cabi.row_groups(2688) == [(272 * k, 272 * (k + 1)) for k in range(6)] + [(1632 + 264 * k, 1896 + 264 * k)
                                                                                   for k in range(4)]
    assert len(_cabi.row_groups(2572)) == 9  # the C5 GP-ECORR pulsar
    for m in (0, -3, 2689, 10_000):
        with pytest.raises(ValueError, match="2688"):
            _cabi.row_groups(m)


@pytest.mark.parametrize("m", [641, 647, 700, 768, 863, 864, 865, 1000, 1280, 1281, 1300, 1536, 2000, 2572, 2687, 2688])
def test_row_to_group_map(m):
    groups = _cabi.row_groups(m)
    assert len(groups) == -(-m // 288)
    assert groups[0][0] == 0 and groups[-1][1] == m
    assert all(a[1] == b[0] for a, b in zip(groups, groups[1:]))  # every row in exactly one group, in order
    assert all(lo % 8 == 0 for lo, _ in groups)  # whole blocks of 8 rows
    padded = [-(-(hi - lo) // 8) * 8 for lo, hi in groups]
    assert max(padded) - min(padded) <= 8  # near-equal widths
    assert max(padded) <= 640  # each group fits one work item of the kernel


def test_python_refusals():
    top = _cabi.MAX_M_WIDE
    n = 8
    toas, res, N = [np.arange(n) * 1e5], [np.zeros(n)], [np.ones(n)]
    with pytest.raises(ValueError, match=f"maximum {top}"):
        _cabi.Pack.create(toas, res, N, [np.zeros((n, top + 1))], [np.eye(top + 1)])
    with pytest.raises(ValueError, match="maximum 640 of a noise-marginalised pack"):
        _cabi.Pack.create(toas, res, N, [np.zeros((n, 641))], [np.eye(641)], m_fix=[600], phiinv_fix=[np.ones(600)])
    # residual batches keep one work item per pulsar: a basis wider than 640 gets a message, not a negative limit
    assert _cabi.max_residual_rows([640]) == 0
    for fn in (lambda: _cabi.max_residual_rows([72, 700]), lambda: batch_pass_rows(8, [72, 700]),
               lambda: _cabi.max_residual_rows([700], blockn=True)):
        with pytest.raises(ValueError, match="pulsar 1 has a basis wider than 640|pulsar 0 has a basis wider than 640"):
            fn()


def test_headline_gp_ecorr_layout_is_within_the_maximum():
    """The C5 GP-ECORR shape (10^4 TOAs in 2 500 epochs of 4): 12 + 2 500 + 60 = 2 572 columns."""
    assert 12 + 2500 + 2 * 30 == 2572 <= _cabi.MAX_M_WIDE
    pta = synth.make_pta(1, 400, n_tm=12, ncomps=30, seed=5, epoch=4)
    _, Ts, _, _ = synth.with_ecorr(pta, kernel=False)
    assert Ts[0].shape[1] == 12 + 100 + 60
