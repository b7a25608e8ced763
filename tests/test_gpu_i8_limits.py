"""GPU tests at the limits of the tensor-core sweep (fp_sweep_i8.cu): the widest basis and the longest pulsar it
takes in one pass (m = 127 -> all 128 operand rows, n = 16384 -> the int32 accumulators' exactness bound), wider
bases in row groups up to m = 639, the narrowest one, and the hand-over to the fp64 kernel just outside. Run with -m gpu on an H100."""
import numpy as np
import pytest

import fastfp_b200
from conftest import EPS, term_tolerance
from fastfp_b200 import _cabi, synth
from oracle import fp_oracle as o
from oracle import truth

pytestmark = pytest.mark.gpu


def _against_truth(pta, freqs, path, expect=None):
    mats = (pta.Nvecs, pta.Ts, pta.sigmas)
    fp = fastfp_b200.FastFp(pta.psrs, path=path)
    assert fp.prepare(*mats).path == (expect or path)
    got = fp.per_pulsar_terms(freqs, *mats)
    args = (freqs, pta.toas, pta.residuals, *mats)
    ora = o.fp_sweep(*args, per_pulsar=True)
    tt, cond = truth.fp_sweep_truth(*args)
    tol = term_tolerance(tt.astype(float), cond, ora)
    defined = EPS * cond < 0.05 * np.abs(tt.astype(float))
    assert defined.mean() > 0.9
    ratio = np.where(defined, np.abs(got - tt.astype(float)) / tol, 0.0)
    assert np.all(ratio <= 1), f"{path}: worst |got - truth| / tol = {ratio.max():.3g}"
    return got, np.where(defined, tol, np.inf)


def test_widest_basis_and_longest_pulsar_the_tensor_path_takes():
    # m = 7 + 2 * 60 = 127 columns (+ the C^-1 r row = 128 operand rows); 16384 TOAs = 512 stages
    pta = synth.make_pta(2, [16384, 4099], n_tm=[7, 7], ncomps=60, seed=31)
    assert pta.Ts[0].shape == (16384, 127)
    freqs = np.concatenate((synth.fp_freqs(30), np.array([1.0, 17.5, 60.0]) / pta.Tspan))  # 33 bins: ragged tile
    t8, tol = _against_truth(pta, freqs, "i8")
    t64, _ = _against_truth(pta, freqs, "fp64")
    assert np.all(np.abs(t8 - t64) <= 2 * tol)  # the same statistic from both kernels


def test_one_toa_too_many_goes_to_the_fp64_kernel_pulsar_by_pulsar():
    # pulsar 0 is one TOA beyond the exactness bound of the int32 accumulators: the fp64 kernel sweeps it, the tensor
    # kernel the other two, in the same call
    pta = synth.make_pta(3, [16385, 300, 1207], n_tm=[7, 7, 9], ncomps=60, seed=32)
    mats = (pta.Nvecs, pta.Ts, pta.sigmas)
    assert fastfp_b200.FastFp(pta.psrs).prepare(*mats).path == "fp64"         # auto: the DMMA kernel
    assert fastfp_b200.FastFp(pta.psrs, path="prefer-i8").prepare(*mats).path == "mixed"
    with pytest.raises(_cabi.FastFpError):
        fastfp_b200.FastFp(pta.psrs, path="i8").prepare(*mats)
    freqs = np.concatenate((synth.fp_freqs(30), np.array([1.0, 17.5, 60.0]) / pta.Tspan))
    tm, tol = _against_truth(pta, freqs, "prefer-i8", expect="mixed")
    t64, _ = _against_truth(pta, freqs, "fp64")
    np.testing.assert_array_equal(tm[0], t64[0])            # pulsar 0 ran on the fp64 kernel: the same bits
    assert np.all(np.abs(tm - t64) <= 2 * tol)
    # the noise-marginalised stage A mixes the same way: the (D, F) result against the all-fp64 run
    from fastfp_b200 import NMFP, RN_container

    sigs = [RN_container(q, Ffreqs=pta.Ffreqs) for q in pta.psrs]
    samples = {k: v for k, v in synth.draw_samples(pta, 3).items() if not k.startswith("gw_")}
    fn = synth.nmfp_freqs(40, pta.Tspan) * 1.003
    a = NMFP(pta.psrs, sigs, path="prefer-i8")(fn, samples, pta.Nvecs, pta.Ts, pta.TNTs)
    b = NMFP(pta.psrs, sigs, path="fp64")(fn, samples, pta.Nvecs, pta.Ts, pta.TNTs)
    np.testing.assert_allclose(a, b, rtol=1e-6)


@pytest.mark.parametrize("n_tm,ncomps", [(8, 60), (68, 60), (136, 60), (140, 60), (519, 60)])
def test_row_groups_of_wide_bases(n_tm, ncomps):
    """m = 128 (the w row alone in a second group), 188, 256 (two full groups + the w row), 260 and 639 (five groups):
    one pass over the TOAs per group of 128 operand rows, b-sums added up across the passes."""
    m = n_tm + 2 * ncomps
    pta = synth.make_pta(2, [1500, 901] if m < 300 else [2600, 1901], n_tm=n_tm, ncomps=ncomps, seed=34)
    assert pta.Ts[0].shape[1] == m
    freqs = np.concatenate((synth.fp_freqs(40), np.array([1.0, 9.5]) / pta.Tspan))
    t8, tol = _against_truth(pta, freqs, "i8")
    t64, _ = _against_truth(pta, freqs, "fp64")
    assert np.all(np.abs(t8 - t64) <= 2 * tol)  # the same statistic from both kernels, inside the envelope


def test_narrowest_basis_and_shortest_pulsars():
    # one timing-model column, white noise only: 2 real operand rows of 128; 33 and 1 TOAs: a partial first stage
    pta = synth.make_pta(3, [33, 32, 7], n_tm=1, white_only=True, seed=33)
    freqs = synth.fp_freqs(65)
    _against_truth(pta, freqs, "i8")
