"""Lane-level NumPy emulation of the fp64 sweep kernel's producer mapping (csrc/fp_sweep_kernel.cuh, producer_loop) for
the m <= 80 family, which runs 8 producer warps (SweepCfg<..., 8, 8, ...>) where the other families run 16. It checks
that every S-tile element of a chunk is stored exactly once, at the address the consumers' A-fragment loads read
(tests/test_sweep_fragment_layout.py), and that the five scalar sums of every frequency come out bit for bit as under
16 producer warps: the same partial sums over the same k-block ranges, folded into the level-2 slab at the same chunk
boundaries, reduced over the same lanes and added in the same order in the epilogue (the emulation rounds the products
of the kernel's fmas separately, the same way for both orders). Runs on the CPU."""
import numpy as np
import pytest

LANE = np.arange(32)
G8, T4 = LANE >> 2, LANE & 3
NWC, NWP_DEFAULT = 8, 16
FLUSH_TOAS = 512


def cfg(nmbw, nnb, wmw, ci, nwp, pregs):  # SweepCfg's derived producer sizes (csrc/ffp_internal.cuh)
    kf = (NWC // wmw) * nnb * 4
    nx, kb = kf // 8, ci // 4
    xw = nx // nwp if nx >= nwp else 1
    ksplit = 1 if nx >= NWP_DEFAULT else min(NWP_DEFAULT // nx, kb)
    wpg = 1 if nx >= nwp else min(nwp // nx, ksplit)
    kbw = kb // ksplit
    c = dict(KF=kf, NX=nx, KB=kb, XW=xw, KSPLIT=ksplit, KBW=kbw, WPG=wpg, SPW=ksplit // wpg, NWP=nwp,
             NACTIVE=nwp if nx >= nwp else nx * wpg, NV=kbw * xw if pregs >= 72 else 1, FLUSH=FLUSH_TOAS // ci)
    assert kb % ksplit == 0 and ksplit % wpg == 0 and c["NACTIVE"] <= nwp and (kbw * xw) % c["NV"] == 0
    return c


def elements(c, pw):
    """(partial sum, [(k-block, frequency group)] in the order the warp's threads evaluate and sum them)"""
    bx0 = pw * c["XW"] if c["NX"] >= c["NWP"] else pw % c["NX"]
    bsplit = 0 if c["NX"] >= c["NWP"] else (pw // c["NX"]) * c["SPW"]
    out = []
    for sp in range(c["SPW"]):
        kb0 = (bsplit + sp) * c["KBW"]
        els = []
        for e0 in range(0, c["KBW"] * c["XW"], c["NV"]):  # NV chains in lockstep, summed in element order
            for v in range(c["NV"]):
                e = e0 + v
                els.append((kb0 + e // c["XW"], bx0 + e % c["XW"]))
        out.append((bsplit + sp, els))
    return out


W2 = [(nmbw, 2, 1, 32) for nmbw in range(6, 11)]
OTHERS = [(1, 4, 1, 16), (5, 4, 1, 16), (7, 2, 2, 16), (10, 2, 2, 16), (8, 2, 4, 16), (6, 2, 8, 8), (10, 2, 8, 8)]


@pytest.mark.parametrize("fam", W2)
def test_w2_split(fam):
    c = cfg(*fam, nwp=8, pregs=88)
    # one warp per frequency group, both halves of the chunk, four lockstep chains per half
    assert (c["NACTIVE"], c["XW"], c["KSPLIT"], c["SPW"], c["KBW"], c["NV"]) == (8, 1, 2, 2, 4, 4)
    # slab slots per producer thread x threads: within sweep_max_slab_doubles()'s producer share (10 x 512)
    assert 5 * c["SPW"] * c["XW"] * 32 * c["NWP"] <= 10 * 512


@pytest.mark.parametrize("fam", W2 + OTHERS)
def test_default_split_unchanged(fam):
    """with 16 producer warps a warp keeps one partial sum and evaluates one pair at a time, as before"""
    c = cfg(*fam, nwp=16, pregs=56)
    assert c["SPW"] == 1 and c["NV"] == 1 and c["WPG"] == c["KSPLIT"]
    for pw in range(c["NACTIVE"]):
        bx0 = pw * c["XW"] if c["NX"] >= 16 else pw % c["NX"]
        bkb0 = 0 if c["NX"] >= 16 else (pw // c["NX"]) * c["KBW"]
        ((bs, els),) = elements(c, pw)
        assert bs == (0 if c["NX"] >= 16 else pw // c["NX"])
        assert els == [(bkb0 + kk, bx0 + xx) for kk in range(c["KBW"]) for xx in range(c["XW"])]


@pytest.mark.parametrize("fam", W2)
def test_w2_stores_once(fam):
    c = cfg(*fam, nwp=8, pregs=88)
    NX, KB = c["NX"], c["KB"]
    S = np.full(KB * NX * 64, np.nan)
    tag = lambda f, i: 1000.0 * f + i  # noqa: E731
    for pw in range(c["NWP"]):
        for _, els in elements(c, pw):
            for kb, x in els:
                f, i = 8 * x + G8, 4 * kb + T4
                o = (kb * NX + x) * 64 + 2 * LANE
                assert np.isnan(S[o]).all() and np.isnan(S[o + 1]).all()
                S[o], S[o + 1] = tag(f, i), -tag(f, i) - 1
    assert not np.isnan(S).any()
    # the consumers' A fragment of frequency tile x, k-block kb: lane (g, t) loads (sin, cos) of (8x + g, 4kb + t)
    for kb in range(KB):
        for x in range(NX):
            a = S[(kb * NX + x) * 64 + 2 * LANE + np.array([[0], [1]])]
            assert np.array_equal(a[0], tag(8 * x + G8, 4 * kb + T4))
            assert np.array_equal(a[1], -tag(8 * x + G8, 4 * kb + T4) - 1)


def producer_sums(c, nch, s, cs, ni, wv):
    """redA[KSPLIT][KF][5] as the producers leave it; s, cs: [KF][n] sin/cos, ni, wv: [n] 1/N and w"""
    ci = 4 * c["KB"]
    red = np.full((c["KSPLIT"], c["KF"], 5), np.nan)
    for pw in range(c["NACTIVE"]):
        parts = elements(c, pw)
        acc = np.zeros((len(parts), 5, 32))
        slab = np.zeros((len(parts), 5, 32))
        flushed = False
        for ch in range(nch):
            for p, (_, els) in enumerate(parts):
                for kb, x in els:
                    f, i = 8 * x + G8, ch * ci + 4 * kb + T4
                    sv, cv = s[f, i], cs[f, i]
                    sn, cn = sv * ni[i], cv * ni[i]
                    acc[p] = acc[p] + np.stack([sn * sv, sn * cv, cn * cv, sv * wv[i], cv * wv[i]])
            if (ch + 1) % c["FLUSH"] == 0 and ch + 1 < nch:
                slab = slab + acc if flushed else acc.copy()
                acc[:] = 0.0
                flushed = True
        for p, (bsplit, els) in enumerate(parts):
            v = acc[p] + slab[p] if flushed else acc[p]
            for sh in (1, 2):
                v = v + v[:, LANE ^ sh]
            x = els[0][1]
            lead = T4 == 0
            red[bsplit, 8 * x + G8[lead]] = v[:, lead].T
    assert not np.isnan(red).any()
    return red


def epilogue(red):
    a = np.zeros(red.shape[1:])
    for g in range(red.shape[0]):
        a = a + red[g]
    return a


@pytest.mark.parametrize("fam", [(9, 2, 1, 32), (6, 2, 1, 32)])
def test_w2_sums_bitwise(fam):
    new, old = cfg(*fam, nwp=8, pregs=88), cfg(*fam, nwp=16, pregs=56)
    ci = 4 * new["KB"]
    nch = 2 * new["FLUSH"] + 5  # two level-2 folds and an open tail
    n = nch * ci
    rng = np.random.default_rng(20261018)
    t = rng.uniform(-4.6e8, 4.6e8, n)
    f = rng.uniform(1e-9, 1e-6, new["KF"])
    ph = (2 * np.pi * f)[:, None] * t[None, :]
    s, cs = np.sin(ph), np.cos(ph)
    ni, wv = 1.0 / rng.uniform(1e-14, 1e-12, n), rng.standard_normal(n) * 1e6
    r_new, r_old = producer_sums(new, nch, s, cs, ni, wv), producer_sums(old, nch, s, cs, ni, wv)
    assert np.array_equal(r_new, r_old)
    assert np.array_equal(epilogue(r_new), epilogue(r_old))
    # the partition matters: one running sum per frequency over the whole chunk rounds differently
    single = np.zeros((new["KF"], 5))
    for i in range(n):
        sn, cn = s[:, i] * ni[i], cs[:, i] * ni[i]
        single = single + np.stack([sn * s[:, i], sn * cs[:, i], cn * cs[:, i], s[:, i] * wv[i], cs[:, i] * wv[i]], 1)
    np.testing.assert_allclose(epilogue(r_new), single, rtol=1e-9)
    assert not np.array_equal(epilogue(r_new), single)
