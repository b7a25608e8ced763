"""Residual batches on a block-diagonal N pack (kernel ECORR) against one pack and one calculate_Fp per realisation, at
the shapes of tools/time_blockn.py (C2: 45 pulsars x 5000 TOAs in 1250 epochs of 4, F = 10^4), plus one
calculate_Fe_skymax_batch line. usage: time_blockn_batch.py [P N F]"""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import fastfp_b200
from fastfp_b200 import BlockNvec, synth
from fastfp_b200.fe import antenna_pattern

P, n, F = (int(v) for v in sys.argv[1:4]) if len(sys.argv) > 3 else (45, 5000, 10_000)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print(f"card: {card}")
pta = synth.make_pta(P, n)
rng = np.random.default_rng(5)
blocks, sig = [], []
for p in range(P):
    sl = [slice(a, a + 4) for a in range(0, n - 3, 4)]
    B = BlockNvec(pta.Nvecs[p], sl, rng.uniform(0.3, 3.0, len(sl)) * 1e-13)
    TNT = pta.Ts[p].T @ B.solve(pta.Ts[p])
    blocks.append(B)
    sig.append(0.5 * (TNT + TNT.T) + np.diag(1.0 / pta.phis[p]))
freqs = synth.fp_freqs(F)
fr = torch.tensor(freqs, dtype=torch.float64, device="cuda")
m = pta.Ts[0].shape[1]


def sim(R, seed):
    g = np.random.default_rng(seed)
    return [np.sqrt(nv)[None, :] * g.standard_normal((R, n)) for nv in pta.Nvecs]


def events(fn, reps=2):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


# separate route: a fresh block-N pack and one calculate_Fp per realisation, two realisations, scaled
res2 = sim(2, 1)
sep = []
for k in range(2):
    psrs = [type("Psr", (), {"toas": q.toas, "residuals": r[k]})() for q, r in zip(pta.psrs, res2)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fastfp_b200.FastFp(psrs)(fr, blocks, pta.Ts, sig)
    torch.cuda.synchronize()
    sep.append(time.perf_counter() - t0)
sep_ms = 1e3 * sep[1]  # the second one: no first-launch costs
fp = fastfp_b200.FastFp(pta.psrs)
pack = fp.prepare(blocks, pta.Ts, sig)
one = events(lambda: pack.fp_sweep(fr, out=torch.empty(F, dtype=torch.float64, device="cuda")))
print(f"C2 block N: {P} x {n}, m = {m}, F = {F}; one sweep {one:.1f} ms, separate {sep_ms:.1f} ms per realisation")
print("| R | set_residuals_blockn | fp_sweep_residuals | per realisation | separate (scaled) | speed-up | evals/s |")
for R in (1, 8, 64, 248):
    res = sim(R, 10 + R)
    pack.set_residuals_blockn(res)  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pack.set_residuals_blockn(res)
    torch.cuda.synchronize()
    t_set = 1e3 * (time.perf_counter() - t0)
    out = torch.empty((R, F), dtype=torch.float64, device="cuda")
    call = events(lambda: pack.fp_sweep_residuals(fr, out=out))
    assert bool(torch.isfinite(out).all())
    print(f"| {R} | {t_set:.1f} ms | {call:.1f} ms | {call / R:.2f} ms | {sep_ms * R / 1e3:.2f} s | "
          f"{sep_ms * R / call:.1f}x | {R * P * F / call * 1e3:.3g} |")
S, R = 768, 64
pos = np.stack([q.pos for q in pta.psrs])
g = np.random.default_rng(7)
th, ph = np.arccos(g.uniform(-1, 1, S)), g.uniform(0, 2 * np.pi, S)
fplus, fcross = antenna_pattern(pos, th, ph)
pack.set_residuals_blockn(sim(R, 99))
bo = torch.empty((R, F), dtype=torch.float64, device="cuda")
io = torch.empty((R, F), dtype=torch.int64, device="cuda")
ms = events(lambda: pack.fe_skymax_residuals(fr, fplus, fcross, out=bo, index_out=io))
print(f"fe_skymax_residuals: S = {S}, R = {R}: {ms:.1f} ms per call, {ms / R:.2f} ms per realisation")
pack.close()
