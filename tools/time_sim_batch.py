"""Residual batches drawn on the device (Pack.simulate_residuals*, DESIGN.md section 5g) against the host route they
replace (NumPy draws as tests/test_gpu_fp_batch.py::realisations makes them, then set_residuals / set_residuals_blockn),
with the sweep of the set, at C2 (45 x 5000, F = 10^4), C4 (68 x 10^4 TOAs, F = 10^3: the sweep of the full C4 grid
takes seconds per realisation) and C2 with kernel ECORR (1250 epochs of 4), for R = 8, 64, 248 and the one-pass maximum.
The simulated set-up and the sweep are timed with CUDA events, the host route by the host clock around work that ends in
a synchronise. ``--profile`` instead runs one simulated set-up at C2, R = 248, under torch.profiler and prints the CUDA
time of each kernel it launches; with ``--trace FILE`` it also writes the Chrome trace there.

usage: time_sim_batch.py [C2|C4|C2E ...] [--profile [--trace FILE]]"""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import fastfp_b200
from fastfp_b200 import BlockNvec, _cabi, synth

SHAPES = {"C2": (45, 5000, 10_000, False), "C4": (68, 10_000, 1000, False), "C2E": (45, 5000, 10_000, True)}


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


def setup(P, n, blockn):
    pta = synth.make_pta(P, n)
    Nvecs, sig = pta.Nvecs, pta.sigmas
    if blockn:
        rng = np.random.default_rng(5)
        Nvecs, sig = [], []
        for p in range(P):
            B = BlockNvec(pta.Nvecs[p], [slice(a, a + 4) for a in range(0, n - 3, 4)],
                          rng.uniform(0.3, 3.0, n // 4) * 1e-13)
            TNT = pta.Ts[p].T @ B.solve(pta.Ts[p])
            Nvecs.append(B)
            sig.append(0.5 * (TNT + TNT.T) + np.diag(1.0 / pta.phis[p]))
    pack = fastfp_b200.FastFp(pta.psrs).prepare(Nvecs, pta.Ts, sig)
    return pta, Nvecs, pack, [1.0 / phi for phi in pta.phis]


def host_draw(pta, Nvecs, R, seed):
    """the host route's realisations: white noise (+ the ECORR epoch draws), plus the non-timing-model basis columns
    drawn from their prior, one realisation and pulsar at a time"""
    g = np.random.default_rng(seed)
    out = []
    for p, q in enumerate(pta.psrs):
        n, ntm = q.toas.shape[0], pta.n_tm[p]
        res = np.empty((R, n))
        nvec = Nvecs[p].nvec if hasattr(Nvecs[p], "nvec") else Nvecs[p]
        for k in range(R):
            r = np.sqrt(nvec) * g.standard_normal(n)
            if hasattr(Nvecs[p], "nvec"):
                r += np.repeat(np.sqrt(Nvecs[p].jvec) * g.standard_normal(n // 4), 4)
            phi_rn = pta.phis[p][ntm:]
            res[k] = r + pta.Ts[p][:, ntm:] @ (np.sqrt(phi_rn) * g.standard_normal(phi_rn.size))
        out.append(res)
    return out


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


def run(name):
    P, n, F, blockn = SHAPES[name]
    pta, Nvecs, pack, phi = setup(P, n, blockn)
    m = max(pack.m)
    simulate = pack.simulate_residuals_blockn if blockn else pack.simulate_residuals
    upload = pack.set_residuals_blockn if blockn else pack.set_residuals
    fr = torch.tensor(synth.fp_freqs(F), dtype=torch.float64, device="cuda")
    rmax = _cabi.max_residual_rows(pack.m, blockn)
    print(f"{name}: {P} x {n}{' in epochs of 4 (kernel ECORR)' if blockn else ''}, m = {m}, F = {F}; card: {card()}")
    print("| R | simulated set-up | host route: draws + upload | sweep call | simulated per realisation | "
          "host route per realisation |")
    print("|---|---|---|---|---|---|")
    for R in (8, 64, 248, rmax):
        t_sim = events(lambda: simulate(R, 1, phi))
        out = torch.empty((R, F), dtype=torch.float64, device="cuda")
        call = events(lambda: pack.fp_sweep_residuals(fr, out=out))
        assert bool(torch.isfinite(out).all())
        try:
            t0 = time.perf_counter()
            res = host_draw(pta, Nvecs, R, seed=R)
            upload(res)
            torch.cuda.synchronize()
            t_host = 1e3 * (time.perf_counter() - t0)
            del res
            host, host_per = f"{t_host:.1f} ms", f"{(t_host + call) / R:.2f} ms"
        except MemoryError:
            host, host_per = "not measured (host memory)", "not measured"
        print(f"| {R} | {t_sim:.1f} ms | {host} | {call:.1f} ms | {(t_sim + call) / R:.2f} ms | {host_per} |")
    pack.close()


def profile(trace=None):
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile as tprof

    P, n, _, _ = SHAPES["C2"]
    pta, Nvecs, pack, phi = setup(P, n, False)
    pack.simulate_residuals(248, 1, phi)
    torch.cuda.synchronize()
    with tprof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for seed in (2, 3):
            pack.simulate_residuals(248, seed, phi)
        torch.cuda.synchronize()
    print(f"C2, R = 248, two simulated set-ups; card: {card()}")
    print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=12))
    if trace:
        prof.export_chrome_trace(trace)
    pack.close()


if __name__ == "__main__":
    if "--profile" in sys.argv:
        profile(sys.argv[sys.argv.index("--trace") + 1] if "--trace" in sys.argv[:-1] else None)
    else:
        for name in [a for a in sys.argv[1:] if a in SHAPES] or list(SHAPES):
            run(name)
