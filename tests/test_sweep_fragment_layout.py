"""Lane-level NumPy emulation of one chunk of the fp64 sweep kernel (csrc/fp_sweep_kernel.cuh): the producers' S-tile
stores, the consumers' A (sin/cos) and B (G packet) fragment loads, mma.m16n8k4.f64 under the PTX fragment layout, the
accumulator ownership, the b-sum lanes, the nmfp z' addresses, the block-N slot indices and the residual rows. Runs on
the CPU: it pins the index algebra the CUDA kernel is written from (the kernel itself is covered by the GPU tests)."""
import numpy as np
import pytest

LANE = np.arange(32)
G8, T4 = LANE >> 2, LANE & 3  # groupID, threadID_in_group
NWC, NWP = 8, 16


def g_frag_index(il, j, nmb):  # csrc/ffp_internal.cuh: the packet's G part
    return (((il >> 2) * nmb + (j >> 3)) << 5) + (((j & 7) << 2) | (il & 3))


def dmma16(d, a0, a1, b):
    """mma.m16n8k4.f64: A[g][t] = a0, A[g+8][t] = a1, B[t][g] = b; D[g][2t+e] = d[e], D[g+8][2t+e] = d[2+e]"""
    A, B = np.zeros((16, 4)), np.zeros((4, 8))
    A[G8, T4], A[G8 + 8, T4] = a0, a1
    B[T4, G8] = b
    D = A @ B
    return d + np.stack([D[G8, 2 * T4], D[G8, 2 * T4 + 1], D[G8 + 8, 2 * T4], D[G8 + 8, 2 * T4 + 1]])


def cfg(nmbw, nnb, wmw, ci):  # SweepCfg's derived sizes
    wnw = NWC // wmw
    kf = wnw * nnb * 4
    nx, kb = kf // 8, ci // 4
    xw = nx // NWP if nx >= NWP else 1
    ksplit = 1 if nx >= NWP else min(NWP // nx, kb)
    return dict(WNW=wnw, KF=kf, NX=nx, KB=kb, NMB=nmbw * wmw, MP=8 * nmbw * wmw, XW=xw, KBW=kb // ksplit,
                NACTIVE=NWP if nx >= NWP else nx * ksplit)


FAMILIES = [(1, 4, 1, 16), (5, 4, 1, 16), (6, 2, 1, 32), (9, 2, 1, 32), (10, 2, 1, 32), (7, 2, 2, 16), (10, 2, 2, 16),
            (8, 2, 4, 16), (6, 2, 8, 8), (10, 2, 8, 8)]


@pytest.mark.parametrize("nmbw,nnb,wmw,ci", FAMILIES)
def test_one_chunk(nmbw, nnb, wmw, ci):
    c = cfg(nmbw, nnb, wmw, ci)
    KF, NX, KB, NMB, MP = c["KF"], c["NX"], c["KB"], c["NMB"], c["MP"]
    NMT = nnb // 2
    rng = np.random.default_rng(nmbw * 100 + wmw * 10 + ci)
    G = rng.standard_normal((MP, ci))  # basis rows x TOAs of the chunk
    Ssin, Scos = rng.standard_normal((KF, ci)), rng.standard_normal((KF, ci))  # frequency x TOA
    pkt = np.full(ci * MP, np.nan)
    for j in range(MP):
        for il in range(ci):
            pkt[g_frag_index(il, j, NMB)] = G[j, il]
    assert not np.isnan(pkt).any()

    # producers: warp pw, lane (bf8, bk) stores the (sin, cos) pair of (frequency 8x + bf8, TOA 4kb + bk) with one
    # 16-byte store at (kb*NX + x)*64 + 2*lane
    S = np.full(KB * NX * 64, np.nan)
    bf8, bk = G8, T4
    for pw in range(c["NACTIVE"]):
        bx0 = pw * c["XW"] if NX >= NWP else pw % NX
        bkb0 = 0 if NX >= NWP else (pw // NX) * c["KBW"]
        for kk in range(c["KBW"]):
            kb = bkb0 + kk
            for xx in range(c["XW"]):
                f, i = 8 * (bx0 + xx) + bf8, 4 * kb + bk
                o = (kb * NX + bx0 + xx) * 64 + 2 * LANE
                assert np.isnan(S[o]).all() and np.isnan(S[o + 1]).all()
                S[o], S[o + 1] = Ssin[f, i], Scos[f, i]
    assert not np.isnan(S).any()
    ofs = 2 * LANE  # one warp's 128-bit loads: a quarter-warp covers 8 distinct 16-byte bank groups
    assert all(len(set(((ofs[8 * h:8 * h + 8] // 2) % 8).tolist())) == 8 for h in range(4))

    Ysin, Ycos = Ssin @ G.T, Scos @ G.T  # [KF][MP]
    mfix = MP - 5  # rows from mfix on: per-draw block (nmfp) / residual realisations
    bsum = np.zeros((KF, 3))
    z = {}
    slots = {}
    res_rows = {}
    for cw in range(NWC):
        wm, wn = cw // c["WNW"], cw % c["WNW"]
        acc = np.zeros((nmbw, NMT, 4, 32))
        for kb in range(KB):
            b = [pkt[(kb * NMB + wm * nmbw + r) * 32 + LANE] for r in range(nmbw)]
            a = [S[(kb * NX + wn * NMT + q) * 64 + 2 * LANE + np.array([[0], [1]])] for q in range(NMT)]
            for r in range(nmbw):
                for q in range(NMT):
                    acc[r, q] = dmma16(acc[r, q], a[q][0], a[q][1], b[r])
        for r in range(nmbw):
            for q in range(NMT):
                f = 8 * (wn * NMT + q) + G8
                for e in range(2):
                    j = 8 * (wm * nmbw + r) + 2 * T4 + e
                    np.testing.assert_allclose(acc[r, q, e], Ysin[f, j], rtol=1e-12, atol=1e-12)
                    np.testing.assert_allclose(acc[r, q, 2 + e], Ycos[f, j], rtol=1e-12, atol=1e-12)
        # b-sums: one chain per row residue 2t + e over the row blocks, the two added in registers, then reduced over
        # the four t-lanes (shfl_xor 1, 2)
        for q in range(NMT):
            p = np.zeros((2, 3, 32))
            for r in range(nmbw):
                for e in range(2):
                    j = 8 * (wm * nmbw + r) + 2 * T4 + e
                    ys, yc = acc[r, q, e], acc[r, q, 2 + e]
                    p[e] += np.where(j < mfix, np.stack([ys * ys, ys * yc, yc * yc]), 0.0)
                    f = 8 * (wn * NMT + q) + G8
                    for ln in np.nonzero(j >= mfix)[0]:  # z' of the per-draw rows, stage-B tile address
                        jr, fi = j[ln] - mfix, f[ln] & 31
                        addr = ((jr >> 2) * 8 + (fi >> 2)) * 32 + 4 * (fi & 3) + (jr & 3)
                        assert (f[ln] >> 5, addr) not in z
                        z[(f[ln] >> 5, addr)] = ys[ln]
                        z[(f[ln] >> 5, addr + 16)] = yc[ln]
                        res_rows[(j[ln] - mfix, f[ln])] = (ys[ln], yc[ln])
            p = p[0] + p[1]
            for s in (1, 2):
                p = p + p[:, LANE ^ s]
            lead = T4 == 0
            bsum[8 * (wn * NMT + q) + G8[lead]] += p[:, lead].T
            # the same rounding as the m8n8k4 layout, where lane (row residue rr, frequency) kept one chain over the
            # row blocks and the shuffles paired residues rr^1, rr^2, rr^4: the frequency's sums are bit for bit equal
            rows = 8 * (wm * nmbw + np.arange(nmbw))[:, None] + np.arange(8)[None, :]  # [r][residue]
            ys8, yc8 = np.zeros((nmbw, 8, 8)), np.zeros((nmbw, 8, 8))  # [r][residue][frequency in the tile]
            for r in range(nmbw):
                for e in range(2):
                    ys8[r, 2 * T4 + e, G8] = acc[r, q, e]
                    yc8[r, 2 * T4 + e, G8] = acc[r, q, 2 + e]
            old = np.zeros((8, 3, 8))  # [residue][sum][frequency in the tile]
            for r in range(nmbw):
                on = (rows[r] < mfix)[:, None]
                old[:, 0] += np.where(on, ys8[r] * ys8[r], 0.0)
                old[:, 1] += np.where(on, ys8[r] * yc8[r], 0.0)
                old[:, 2] += np.where(on, yc8[r] * yc8[r], 0.0)
            for s in (1, 2, 4):
                old = old + old[np.arange(8) ^ s]
            assert np.array_equal(old[0].T, p[:, lead].T)
        if wm == wmw - 1:  # block-N slot warp: the last row block holds 8 epoch slots, lane (g, t) owns 2t and 2t+1
            for q in range(NMT):
                for e in range(2):
                    slot = 2 * T4 + e
                    for ln in range(32):
                        slots[(slot[ln], 8 * (wn * NMT + q) + G8[ln])] = acc[nmbw - 1, q, e, ln]
    # every frequency's b-sums over the fixed rows, across the warp rows
    want = np.stack([(Ysin[:, :mfix] ** 2).sum(1), (Ysin[:, :mfix] * Ycos[:, :mfix]).sum(1),
                     (Ycos[:, :mfix] ** 2).sum(1)], 1)
    np.testing.assert_allclose(bsum, want, rtol=1e-12)
    # z': the canonical [k-block][freq block][16*sc + 4*(f%4) + row%4] tile, every element written once
    for f in range(KF):
        for jr in range(MP - mfix):
            fi = f & 31
            addr = ((jr >> 2) * 8 + (fi >> 2)) * 32 + 4 * (fi & 3) + (jr & 3)
            assert z[(f >> 5, addr)] == pytest.approx(Ysin[f, mfix + jr], rel=1e-12, abs=1e-12)
            assert z[(f >> 5, addr + 16)] == pytest.approx(Ycos[f, mfix + jr], rel=1e-12, abs=1e-12)
            assert res_rows[(jr, f)] == pytest.approx((Ysin[f, mfix + jr], Ycos[f, mfix + jr]), rel=1e-12, abs=1e-12)
    # slot s of frequency f is row 8*(NMB-1) + s
    assert len(slots) == 8 * KF
    for (s, f), v in slots.items():
        assert v == pytest.approx(Ysin[f, 8 * (NMB - 1) + s], rel=1e-12, abs=1e-12)
