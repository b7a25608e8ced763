"""Every instantiation of the fp64 sweep kernel, on the host (CPU): the configurations the five fp_sweep_*.cu files
compile, read from their FFP_SWEEP_CASE lists; the configurations sweep_config can hand each (mode, N kind); and
``CASES``, one pulsar per reachable (mode, N kind, configuration), which tests/test_gpu_sweep_instantiations.py sweeps
against the longdouble truth. A configuration added to the sources without a case, or a case that no longer lands on
its configuration, fails here.

Each configuration (family, NMBW: row blocks of 8 per consumer warp) is its own pipeline: NMBW sets the accumulator
and fragment arrays and the epilogue reductions, and through the shared-memory budget the depth GST of the G-tile ring,
on which the mbarrier phase parity (k / GST) & 1 depends. So each one needs a launch of its own."""
import os
import re
from collections import namedtuple

import numpy as np

from fastfp_b200 import _cabi
from test_blockn_layout_host import BLOCKN_MAX_M, FAMILIES, family_of

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "fastfp_b200", "csrc")
FILES = ["fp_sweep_w1.cu", "fp_sweep_w2.cu", "fp_sweep_w4.cu", "fp_sweep_wide.cu", "fp_sweep_xwide.cu"]

# fp_sweep.cu::sweep_config per family: frequency blocks of 4 per consumer warp (NNB) and the NMBW it takes
NNB = {"w1": 4, "w2": 2, "w4": 2, "wide": 2, "xwide": 2}
FLUSH = 512  # relaid TOAs per level-1 block (ffp_internal.cuh FLUSH_TOAS)
MAX_M = 640
R_RES = 3  # realisations of every residual-batch case
MODES = [("fp", "diag"), ("fp", "blockn"), ("nmfp", "diag"), ("nmfp", "blockn"), ("res", "diag"), ("res", "blockn")]


def config_of(rows):
    """``(family, NMBW)`` of the kernel a pulsar needing ``rows`` G rows runs on."""
    fam, _, mp = family_of(rows)
    wmw = {name: w for _, name, _, w in FAMILIES}[fam]
    return fam, mp // (8 * wmw)


def cfg_tuple(fam, nmbw):
    """``(NMBW, NNB, WMW, CI)``: the arguments of the configuration's FFP_SWEEP_CASE."""
    _, _, ci, wmw = next(f for f in FAMILIES if f[1] == fam)
    return nmbw, NNB[fam], wmw, ci


def row_range(fam, nmbw):
    """The G-row counts (multiples of 8) that land on a configuration: ``(MP - 8 WMW, MP]``."""
    wmw = cfg_tuple(fam, nmbw)[2]
    mp = 8 * nmbw * wmw
    return list(range(mp - 8 * wmw + 8, mp + 1, 8))


def compiled():
    """The ``(NMBW, NNB, WMW, CI)`` of every FFP_SWEEP_CASE / FFP_SWEEP_CASE_W2 use in the five files."""
    out = []
    for name in FILES:
        with open(os.path.join(CSRC, name)) as fh:
            src = fh.read()
        out += [tuple(int(v) for v in g) for g in re.findall(r"FFP_SWEEP_CASE\((\d+),\s*(\d+),\s*(\d+),\s*(\d+)\)", src)]
        d = re.search(r"#define FFP_SWEEP_CASE_W2\(NMBWv\)\s+FFP_SWEEP_CASE_W\(NMBWv,\s*(\d+),\s*(\d+),\s*(\d+)", src)
        uses = re.findall(r"FFP_SWEEP_CASE_W2\((\d+)\)", src)
        assert not uses or d, name
        out += [(int(u),) + tuple(int(v) for v in d.groups()) for u in uses]
    return out


def extra_rows(mode, kind):
    """G rows beyond roundup8(m): R_RES realisations for residual batches, 8 epoch slots for block-N packs."""
    return (8 if mode == "res" else 0) + (8 if kind == "blockn" else 0)


def reachable(mode, kind):
    """The configurations sweep_config can return for a (mode, N kind): every multiple of 8 G rows from the fewest
    the mode needs (8 basis rows, plus 8 for one or more realisations, plus 8 epoch slots) to 640."""
    first = 8 + (8 if mode == "res" else 0) + (8 if kind == "blockn" else 0)
    return {config_of(r) for r in range(first, MAX_M + 1, 8)}


def split(m, mode):
    """``(n_tm, ncomps)`` of a case of width m: white noise only up to 12 columns (Fp, residual batches), else up to 30
    Fourier components. The noise-marginalised path needs at least one per-draw column and at most 128."""
    if mode != "nmfp" and m <= 12:
        return m, 0
    nc = max(1, min(30, (m - 1) // 4))
    return m - 2 * nc, nc


def flush_edges(m, ci):
    """TOA counts on the edges of the level-2 flush for a pulsar of width m, with j the smallest count of 512-TOA
    blocks holding 3m TOAs: no flush at the last block (512 j), a flush then a one-TOA chunk (512 j + 1), a flush
    then a chunk one TOA short (512 j + CI - 1), and 1024 j + 1 (capped at 2049 >= 3 * 640, so the widest family stays
    near 2 000 TOAs)."""
    j = max(1, -(-3 * m // FLUSH))
    return [FLUSH * j, FLUSH * j + 1, FLUSH * j + ci - 1, min(2 * FLUSH * j, 4 * FLUSH) + 1]


Case = namedtuple("Case", "fam nmbw m n R")


def _cases(mode, kind):
    out, i = [], 0
    R = R_RES if mode == "res" else 0
    for fam in NNB:
        nmbws = sorted({nb for f, nb in reachable(mode, kind) if f == fam})
        for nmbw in nmbws:
            rows = row_range(fam, nmbw)
            # bottom, middle, top of the configuration's rows; the last basis row block full or partly padding
            r = rows[[0, len(rows) // 2, -1][i % 3]] - extra_rows(mode, kind)
            m = r - 5 if i % 2 and r > 8 else r
            if mode == "nmfp" and m < 3:
                m = 3
            n = flush_edges(m, cfg_tuple(fam, nmbw)[3])[i % 4]
            out.append(Case(fam, nmbw, m, n, R))
            i += 1
    if ("w1", 1) in reachable(mode, kind):
        out.append(Case("w1", 1, 3, 11, R))  # fewer TOAs than one chunk of 16: a single chunk, mostly padding
    return out


CASES = {mk: _cases(*mk) for mk in MODES}


def label(c):
    return f"{c.fam}/NMBW {c.nmbw}, m = {c.m}, n = {c.n}" + (f", R = {c.R}" if c.R else "")


# ---- tests -----------------------------------------------------------------------------------------------------------

def test_compiled_set_is_what_sweep_config_returns():
    got = compiled()
    assert len(got) == len(set(got)), "an FFP_SWEEP_CASE is listed twice"
    want = {cfg_tuple(*c) for c in reachable("fp", "diag")}
    assert set(got) == want and len(want) == 25


def test_family_mirror_against_the_library():
    lib = _cabi.load()
    for m in range(1, MAX_M + 1):
        assert lib.fastfp_sweep_chunk_toas(m, 0) == cfg_tuple(*config_of(_cabi.sweep_rows(m)))[3], m
    for m in range(1, BLOCKN_MAX_M + 1):
        assert lib.fastfp_sweep_chunk_toas(m, 1) == cfg_tuple(*config_of(_cabi.sweep_rows(m, 0, True)))[3], m


def test_unreachable_instantiations():
    """5 of the 150 kernels (25 configurations x {Fp, Nmfp, Res} x {diagonal, block-diagonal N}) are compiled but
    can never launch: one realisation or the 8 epoch slots already take 16 G rows, two of them 24."""
    every = {config_of(r) for r in range(8, MAX_M + 1, 8)}
    missing = {(mode, kind, c) for mode, kind in MODES for c in every - reachable(mode, kind)}
    assert missing == {("res", "diag", ("w1", 1)), ("res", "blockn", ("w1", 1)), ("res", "blockn", ("w1", 2)),
                       ("fp", "blockn", ("w1", 1)), ("nmfp", "blockn", ("w1", 1))}
    assert sum(len(reachable(*mk)) for mk in MODES) == 145


def test_cases_cover_every_reachable_configuration():
    for (mode, kind), cases in CASES.items():
        blockn = kind == "blockn"
        assert {(c.fam, c.nmbw) for c in cases} == reachable(mode, kind), (mode, kind)
        for c in cases:
            rows = _cabi.sweep_rows(c.m, c.R, blockn)
            assert config_of(rows) == (c.fam, c.nmbw), (mode, kind, label(c))
            ci = cfg_tuple(c.fam, c.nmbw)[3]
            assert c.n in flush_edges(c.m, ci) or (c.n < ci and (c.fam, c.nmbw) == ("w1", 1)), (mode, kind, label(c))
            assert c.m <= c.n <= 2100 and c.R == (R_RES if mode == "res" else 0)
            n_tm, nc = split(c.m, mode)
            assert n_tm >= 1 and n_tm + 2 * nc == c.m and (mode != "nmfp" or 1 <= 2 * nc <= 128)
        # the cases alternate between the bottom, middle and top rows of their configuration, and between a full and
        # a partly padded last basis row block
        assert any(c.m % 8 for c in cases) and any(c.m % 8 == 0 for c in cases)
        # every flush edge appears
        edges = {flush_edges(c.m, cfg_tuple(c.fam, c.nmbw)[3]).index(c.n) for c in cases if c.n >= FLUSH}
        assert edges == {0, 1, 2, 3}, (mode, kind)
    assert sum(len({(c.fam, c.nmbw) for c in cs}) for cs in CASES.values()) == 145
    assert any(c.n < 16 for c in CASES[("fp", "diag")])


# ---- the frequency grid every mode sweeps --------------------------------------------------------------------------

SINCOS_FAST = 0.999e5  # the sweep evaluates sin/cos by Cody-Waite reduction while |2 pi f| max|t| <= 0.999 FFP_SINCOS_MAX
KF = {"w1": 128, "w2": 64, "w4": 32, "wide": 16, "xwide": 8}  # frequencies per tile
LO, LO8 = 87, 91  # the below-threshold bins of the two near-threshold pairs


def sweep_freqs(Tspan, tabs):
    """131 bins (not a multiple of 8, more than one 128-bin tile): the 73-bin grid with the 1, 2.5 and 7 / Tspan
    red-noise bins, f = 0 and f < 0, two bins far past the Cody-Waite range, and two pairs of bins on both sides of
    the cold-path threshold 0.999e5 / (2 pi max|t|) of every pulsar (``tabs``: their max|t|). The first pair ends one
    group of 8 frequencies and starts the next inside one tile of every family but the 8-frequency one, so that tile
    has producer warps on the fast and on the library-sincos path; the second pair shares a group of 8."""
    thr = SINCOS_FAST / (2 * np.pi * np.asarray(tabs, dtype=np.float64))
    lo, hi = thr.min() * (1 - 1e-6), thr.max() * (1 + 1e-6)
    f = np.concatenate((np.linspace(2e-9, 3e-7, 70), np.array([1.0, 2.5, 7.0]) / Tspan, np.linspace(3.05e-7, 9e-7, 58)))
    f[LO], f[LO + 1], f[LO8], f[LO8 + 1] = lo, hi, lo * (1 - 1e-6), hi * (1 + 1e-6)
    f[95], f[97] = 0.0, -1e-8
    f[100], f[130] = 5e-5, 1.7e-3
    return f


def assert_near_threshold(freqs, tabs, fams):
    """Every pulsar p (family ``fams[p]``, max|t| ``tabs[p]``) has bins on both sides of its own threshold inside one
    tile, and (families of 16 or more frequencies per tile) one fast group of 8 before a cold one in that tile."""
    om = np.abs(2 * np.pi * freqs)
    for t, fam in zip(tabs, fams):
        fast = om * t <= SINCOS_FAST
        kf = KF[fam]
        for lo in (LO, LO8) if kf >= 16 else (LO8,):
            assert fast[lo] and not fast[lo + 1] and lo // kf == (lo + 1) // kf, (fam, lo)
        if kf >= 16:  # the group of 8 ending at LO is all fast, the next one holds a cold bin
            assert LO % 8 == 7 and np.all(fast[LO - 7:LO + 1]) and np.all(freqs[LO - 7:LO + 1] > 0)
        assert LO8 // 8 == (LO8 + 1) // 8


def test_frequency_grid():
    tabs = 53000.0 * 86400.0 + np.array([4.7e8, 4.3e8, 4.73e8])
    f = sweep_freqs(4.7e8, tabs)
    assert f.shape[0] == 131 and f.shape[0] % 8 and f.shape[0] > 128
    assert np.unique(f).shape[0] == 131
    for fam in KF:
        assert_near_threshold(f, tabs, [fam] * 3)
    fast = np.abs(2 * np.pi * f) * tabs.max() <= SINCOS_FAST
    assert not fast[100] and not fast[130] and (f <= 0).sum() == 2
    assert np.all(fast[:LO + 1]) and np.all(f[:LO] < f[LO])
