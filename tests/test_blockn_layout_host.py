"""Block-diagonal N (kernel ECORR) on the host, per kernel family: which chunk size a block-N pulsar gets, and the
epoch-slot layout of fastfp_b200.blockn at every chunk size, including layouts built to sit on the edges of the slot
machinery (CPU). tests/test_gpu_blockn_families.py runs the same layouts on the GPU and asserts them as preconditions
with the helpers defined here."""
import numpy as np
import pytest

from fastfp_b200 import _cabi, blockn, synth

# fp_sweep.cu::sweep_config, by the number of G rows a pulsar needs: (largest rows, family, TOAs per chunk, warp rows
# WMW). The padded width MP rounds the rows up to 8 * WMW; a block-N pulsar needs roundup8(m) + 8 rows, the last 8
# of MP hold the epoch slots.
FAMILIES = [(40, "w1", 16, 1), (80, "w2", 32, 1), (160, "w4", 16, 2), (320, "wide", 16, 4), (640, "xwide", 8, 8)]
BLOCKN_MAX_M = 632


def blockn_rows(m):
    return -(-m // 8) * 8 + 8


def family_of(rows):
    """``(family, CI, MP)`` of a pulsar needing ``rows`` G rows, or None if no kernel takes it."""
    if rows < 1:
        return None
    for top, name, ci, wmw in FAMILIES:
        if rows <= top:
            return name, ci, -(-rows // (8 * wmw)) * 8 * wmw
    return None


def test_family_table_reaches_every_family_at_its_edges():
    """The widths the GPU tests sweep: bottom and top of every family, with the slot rows behind zero padding where
    the family rounds MP up to more than 8 rows."""
    want = {1: (16, "w1", 16), 32: (40, "w1", 40), 33: (48, "w2", 48), 72: (80, "w2", 80), 73: (88, "w4", 96),
            152: (160, "w4", 160), 153: (168, "wide", 192), 312: (320, "wide", 320), 313: (328, "xwide", 384),
            632: (640, "xwide", 640)}
    for m, (rows, name, mp) in want.items():
        fam = family_of(blockn_rows(m))
        assert (blockn_rows(m), fam[0], fam[2]) == (rows, name, mp), m


def test_chunk_toas_follow_the_family_table():
    lib = _cabi.load()
    for m in range(-1, 642):
        fam = family_of(blockn_rows(m)) if m >= 1 else None
        assert lib.fastfp_sweep_chunk_toas(m, 1) == (fam[1] if fam else 0), m
        fam = family_of(m) if m >= 1 else None
        assert lib.fastfp_sweep_chunk_toas(m, 0) == (fam[1] if fam else 0), m
    # block-N: the 8 slot rows leave 632 basis columns of the widest kernel's 640
    assert lib.fastfp_sweep_chunk_toas(BLOCKN_MAX_M, 1) == 8
    assert all(lib.fastfp_sweep_chunk_toas(m, 1) == 0 for m in range(BLOCKN_MAX_M + 1, 641))
    assert lib.fastfp_sweep_chunk_toas(640, 0) == 8


# ---- layout invariants -------------------------------------------------------------------------------------------

def relaid_spans(slices):
    """Where blockn.prepare puts each epoch: epochs in slice order, each padded to a multiple of 4 TOAs."""
    spans, a = [], 0
    for s in slices:
        b = a + -(-(s.stop - s.start) // 4) * 4
        spans.append((a, b))
        a = b
    return spans


def epoch_spans(d, ci):
    """The epochs as the kernel sees them, read back from the slot indices and per-chunk done masks alone: a slot opens
    at the first k-block that carries it and closes at the end of the chunk whose mask has its bit. Returns the relaid
    ``(start, stop)`` of every epoch, ordered by start."""
    kb_slot = d["slot_idx"].reshape(-1, 4).max(axis=1)
    kb = ci // 4
    open_, spans = {}, []
    for k, s in enumerate(kb_slot):
        if s >= 0:
            open_.setdefault(int(s), [k, k])[1] = k
        if (k + 1) % kb == 0:
            mask = int(d["done_mask"][k // kb])
            for s2 in range(8):
                if (mask >> s2) & 1:
                    assert s2 in open_, f"chunk {k // kb} closes slot {s2}, which holds no epoch"
                    a, b = open_.pop(s2)
                    spans.append((4 * a, 4 * (b + 1)))
    assert not open_, f"slots {sorted(open_)} are never closed"
    return sorted(spans)


def check_layout(q, B, T, ci):
    """Every invariant of ``blockn.prepare(..., ci)`` for one pulsar; returns its output."""
    n = q.toas.shape[0]
    d = blockn.prepare(q.toas, q.residuals, B, T, ci)
    n2 = d["toas"].shape[0]
    assert n2 % ci == 0 and d["done_mask"].shape[0] == n2 // ci
    real = np.isfinite(d["Nvec"])
    assert real.sum() == n  # every TOA appears exactly once, padding has infinite variance
    np.testing.assert_array_equal(np.sort(d["toas"][real]), np.sort(q.toas))
    assert np.all(d["T"][~real] == 0) and np.all(d["slot_val"][~real] == 0) and np.all(d["slot_idx"][~real] == -1)
    # every group of 4 TOAs carries at most one slot, slots are 0..7, and a chunk holds at most KB epochs
    g = d["slot_idx"].reshape(-1, 4)
    for row in g:
        s = set(row[row >= 0])
        assert len(s) <= 1 and all(0 <= v < 8 for v in s)
    assert max(bin(int(v)).count("1") for v in d["done_mask"]) <= ci // 4
    # the slots describe exactly the epochs, where the layout puts them
    assert epoch_spans(d, ci) == relaid_spans(B.slices)
    # the quadratic form x^T N^-1 x is the diagonal part minus the folded slot sums
    x = np.random.default_rng(2).standard_normal(n)
    pos = np.searchsorted(q.toas, d["toas"][real])  # toas are sorted and unique: map by value
    xs = np.zeros(n2)
    xs[real] = x[pos]
    ninv = np.where(real, 1.0 / d["Nvec"], 0.0)
    diag = (xs * xs * ninv).sum()
    corr, run = 0.0, np.zeros(8)
    for c in range(n2 // ci):
        sl = slice(c * ci, (c + 1) * ci)
        for s in range(8):
            sel = d["slot_idx"][sl] == s
            run[s] += (d["slot_val"][sl][sel] * xs[sl][sel]).sum()
            if (d["done_mask"][c] >> s) & 1:
                corr += run[s] ** 2
                run[s] = 0.0
    assert np.all(run == 0.0)  # every epoch was closed
    want = x @ B.solve(x)
    assert abs((diag - corr) - want) < 1e-12 * (diag + corr)
    # Sherman-Morrison applied to T and r in the "(N^-1 x) * nvec" form (absolute error: a large ECORR cancels most of
    # the diagonal part x / nvec)
    for got, x_ in (((d["T"] * ninv[:, None])[real], T), ((d["res_w"] * ninv)[real], q.residuals)):
        scale = np.abs(x_ / (B.nvec if x_.ndim == 1 else B.nvec[:, None])).max()
        np.testing.assert_allclose(got, B.solve(x_)[pos], rtol=1e-10, atol=1e-12 * scale)
    return d


def random_epochs(n, rng, long_at=None):
    """Epochs of 1-8 TOAs with 0-2 TOAs outside any epoch after each; epoch ``long_at`` has 70 TOAs."""
    slices, a = [], 0
    while a < n - 70:
        ln = 70 if len(slices) == long_at else int(rng.integers(1, 9))
        slices.append(slice(a, a + ln))
        a += ln + int(rng.integers(0, 3))
    return slices


@pytest.mark.parametrize("ci", [8, 16, 32])
def test_layout_invariants_with_random_epochs(ci):
    pta = synth.make_pta(1, 613, n_tm=6, ncomps=4, seed=ci)
    rng = np.random.default_rng(ci)
    sl = random_epochs(613, rng, long_at=5)
    B = blockn.BlockNvec(pta.Nvecs[0], sl, rng.uniform(0.2, 3.0, len(sl)) * 1e-13)
    check_layout(pta.psrs[0], B, pta.Ts[0], ci)


# ---- layouts on the edges of the slot machinery --------------------------------------------------------------------

FLUSH = 512  # fp_sweep kernel: relaid TOAs per level-1 block (ffp_internal.cuh FLUSH_TOAS)


def _place(lens, rng, gap):
    """Epochs of the given lengths in TOA order, each followed by ``rng.integers(*gap)`` TOAs outside any epoch."""
    slices, a = [], 0
    for ln in lens:
        slices.append(slice(a, a + int(ln)))
        a += int(ln) + int(rng.integers(*gap))
    return a, slices


def edge_epochs(seed=0):
    """Three pulsars' epochs, ``[(n, slices, large_ecorr)]``, laid out (in relaid TOAs, which do not depend on the chunk
    size) so that
      0. eight 4-TOA epochs open and close in the first 32 TOAs (one chunk at CI = 32: all 8 slots end there); one
         epoch straddles relaid TOA 512 (a level-2 flush), one ends exactly at 1024 and the next starts there; that
         one has 700 TOAs, so its open slot sum stays in registers across the flush at 1536;
      1. every epoch is a single TOA (1 real TOA + 3 padding per k-block);
      2. every TOA is in an epoch, so the last epoch closes in the last chunk; its ECORR is 1e3 x the white noise."""
    rng = np.random.default_rng(seed)
    lens, pos = [4] * 8, 32

    def add(ln):
        nonlocal pos
        lens.append(int(ln))
        pos += -(-int(ln) // 4) * 4

    def fill(upto):
        while pos < upto:
            add(rng.integers(1, 9))

    fill(FLUSH - 32)
    add(FLUSH - pos + 21)           # relaid [pos, 536): across 512
    fill(2 * FLUSH - 24)
    add(2 * FLUSH - pos)            # ends at 1024 (pos is a multiple of 4)
    add(700)                        # [1024, 1724): across 1536
    fill(3 * FLUSH + 300)
    lens_full, pos_full = [], 0
    while pos_full < 3 * FLUSH + 200:
        lens_full.append(int(rng.integers(1, 13)))
        pos_full += -(-lens_full[-1] // 4) * 4
    return [_place(lens, rng, (0, 3)) + (False,),
            _place([1] * 420, rng, (0, 3)) + (False,),
            _place(lens_full, rng, (0, 1)) + (True,)]


def edge_blocks(pta, seed=0):
    """``BlockNvec`` of the :func:`edge_epochs` layouts on the pulsars of ``pta`` (made with their TOA counts)."""
    rng = np.random.default_rng(seed + 1)
    out = []
    for (n, sl, large), nvec in zip(edge_epochs(seed), pta.Nvecs):
        assert nvec.shape == (n,)
        jv = (1e3 * np.array([nvec[s].mean() for s in sl]) if large
              else rng.uniform(0.3, 3.0, len(sl)) * 1e-13)
        out.append(blockn.BlockNvec(nvec, sl, jv))
    return out


def assert_edge_layout(preps, ci):
    """The :func:`edge_epochs` layouts, as ``blockn.prepare`` made them at chunk size ``ci``, are where they are meant
    to be: checked on the slot indices and done masks the kernel reads."""
    kb = ci // 4
    d0, d1, d2 = preps
    for d in preps:
        assert d["toas"].shape[0] >= 3 * FLUSH
    pop = [bin(int(v)).count("1") for v in d0["done_mask"]]
    assert max(pop) == kb
    if ci == 32:
        assert d0["done_mask"][0] == 0xFF  # all 8 slots close in one chunk
    spans = epoch_spans(d0, ci)
    assert any(a < FLUSH < b for a, b in spans)
    assert any(b == 2 * FLUSH for a, b in spans) and any(a == 2 * FLUSH for a, b in spans)
    assert any(b - a >= 700 and a < 3 * FLUSH < b for a, b in spans)
    # 1: every slotted k-block holds exactly one real TOA
    g = d1["slot_idx"].reshape(-1, 4)
    real = np.isfinite(d1["Nvec"]).reshape(-1, 4)
    slotted = (g >= 0).any(axis=1)
    assert slotted.sum() >= 3 * FLUSH // 4 and np.all(real[slotted].sum(axis=1) == 1)
    assert all(b - a == 4 for a, b in epoch_spans(d1, ci))
    # 2: no TOA outside an epoch; the last epoch ends in the last chunk
    assert not np.any(np.isfinite(d2["Nvec"]) & (d2["slot_idx"] < 0))
    nch = d2["done_mask"].shape[0]
    assert d2["done_mask"][-1] != 0 and epoch_spans(d2, ci)[-1][1] > (nch - 1) * ci


@pytest.mark.parametrize("ci", [8, 16, 32])
def test_edge_layouts(ci):
    ns = [n for n, _, _ in edge_epochs()]
    pta = synth.make_pta(3, ns, n_tm=5, ncomps=3, seed=3)
    blocks = edge_blocks(pta)
    preps = [check_layout(q, B, T, ci) for q, B, T in zip(pta.psrs, blocks, pta.Ts)]
    assert_edge_layout(preps, ci)
