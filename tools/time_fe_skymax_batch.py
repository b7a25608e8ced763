"""Timing of the sky-maximised Fe over a batch of residual realisations against one pack and one sky maximum per
realisation.

usage: time_fe_skymax_batch.py [--cases C2,C4] [--R 1,8,64,248] [--sky 768,3072,12288] [--reps 1]

For each PTA shape (C2: 45 pulsars x 5000 TOAs, F = 10^4; C4: 68 x 10^4, F = 10^5), each R and each sky grid size S it
prints: the set_residuals time (host clock around a synchronised call), the fe_skymax_residuals call time (CUDA events
after a warm-up, outputs on the device) and the time per realisation; the per-realisation route (a fresh pack built
with that realisation's residuals, then one calculate_Fe_skymax, host clock; timed for rows 0 and R-1 and scaled to R);
the fe_skymax_res_kernel time from torch.profiler next to fe_skymax_kernel's time for one realisation in the same
process, and the combine kernel's rate (8 R S P F flop of the N GEMM, from the shapes) against fastfp_fp64_peak kinds 0
(DFMA) and 1 (DMMA) measured in the same process; and the agreement of rows 0 and R-1 with calculate_Fe_skymax on their
own packs (largest relative difference, share of equal indices).
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from fastfp_b200 import _cabi, synth  # noqa: E402
from fastfp_b200.fe import FastFe, antenna_pattern  # noqa: E402

CASES = {"C2": ("C2", 10_000), "C4": ("C4", 100_000)}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        pl = "unknown"
    return name, pl


def timed(fn, reps):
    fn()  # warm-up
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_ms(fn, name):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(e.device_time_total for e in prof.key_averages() if name in e.key) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="C2,C4")
    ap.add_argument("--R", default="1,8,64,248")
    ap.add_argument("--sky", default="768,3072,12288")
    ap.add_argument("--reps", type=int, default=1)
    args = ap.parse_args()
    name, pl = card()
    dfma, _ = _cabi.fp64_peak(0)
    dmma, _ = _cabi.fp64_peak(1)
    print(f"card: {name}, power limit {pl}; fastfp_fp64_peak kind 0 (DFMA) {dfma:.2f} TFLOP/s, kind 1 (DMMA) "
          f"{dmma:.2f} TFLOP/s", flush=True)
    rng = np.random.default_rng(7)
    for case in args.cases.split(","):
        cfg, F = CASES[case]
        pta = synth.make_config(cfg)
        P = pta.P
        a = (pta.Nvecs, pta.Ts, pta.sigmas)
        fe = FastFe(pta.psrs)
        pack = fe.prepare(*a)
        freqs = np.linspace(2e-9, 3e-7, F)
        f = torch.tensor(freqs, dtype=torch.float64, device="cuda")
        fa = (f.data_ptr(), F)
        st = torch.cuda.current_stream().cuda_stream
        Rmax = max(int(r) for r in args.R.split(","))
        noise = [np.sqrt(N) * rng.standard_normal((Rmax, N.shape[0])) for N in pta.Nvecs]
        for S in (int(s) for s in args.sky.split(",")):
            th, ph = np.arccos(rng.uniform(-1, 1, S)), rng.uniform(0, 2 * np.pi, S)
            fpl, fcr = antenna_pattern(fe.pos, th, ph)
            b1 = torch.empty(F, dtype=torch.float64, device="cuda")
            i1 = torch.empty(F, dtype=torch.int64, device="cuda")
            pack.fe_skymax(fa, fpl, fcr, out=b1.data_ptr(), index_out=i1.data_ptr(), stream=st)  # warm-up
            one_ms = kernel_ms(lambda: pack.fe_skymax(fa, fpl, fcr, out=b1.data_ptr(), index_out=i1.data_ptr(),
                                                      stream=st), "fe_skymax_kernel")
            route, route_rows = None, {}
            for R in (int(r) for r in args.R.split(",")):
                res = [n[:R] for n in noise]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                pack.set_residuals(res)
                torch.cuda.synchronize()
                t_set = (time.perf_counter() - t0) * 1e3
                best = torch.empty((R, F), dtype=torch.float64, device="cuda")
                idx = torch.empty((R, F), dtype=torch.int64, device="cuda")

                def call():
                    pack.fe_skymax_residuals(fa, fpl, fcr, out=best.data_ptr(), index_out=idx.data_ptr(), stream=st)

                t_call = timed(call, args.reps)
                k_ms = kernel_ms(call, "fe_skymax_res_kernel")
                # the per-realisation route for rows 0 and R-1: a pack of their own, one calculate_Fe_skymax each
                ts = []
                for k in sorted({0, R - 1}):
                    fk = FastFe(pta.psrs)
                    fk.residuals = [n[k] for n in noise]
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    bk, ik = fk.calculate_Fe_skymax(freqs, th, ph, *a)
                    ts.append((time.perf_counter() - t0) * 1e3)
                    fk.invalidate()
                    route_rows[k] = (bk, ik)
                route = float(np.mean(ts))
                got_b, got_i = best.cpu().numpy(), idx.cpu().numpy()
                rel = max(float(np.max(np.abs(got_b[k] / route_rows[k][0] - 1.0))) for k in sorted({0, R - 1}))
                same = min(float(np.mean(got_i[k] == route_rows[k][1])) for k in sorted({0, R - 1}))
                if not k_ms:  # the profiler recorded no launch of the kernel
                    k_ms = float("nan")
                tf = 8.0 * R * S * P * F / (k_ms * 1e-3) / 1e12
                print(f"{case} P={P} F={F} S={S} R={R}: set_residuals {t_set:.1f} ms | call {t_call:.1f} ms, "
                      f"{t_call / R:.2f} ms per realisation | per-realisation route {route:.1f} ms per realisation, "
                      f"{route * R:.0f} ms scaled, speed-up {route * R / (t_set + t_call):.1f}x end to end | "
                      f"fe_skymax_res_kernel {k_ms:.2f} ms = {k_ms / R:.3f} ms per realisation vs fe_skymax_kernel "
                      f"{one_ms:.2f} ms ({one_ms * R / k_ms:.1f}x), {tf:.2f} TFLOP/s = {100 * tf / dfma:.0f}% of kind "
                      f"0, {100 * tf / dmma:.0f}% of kind 1 | rows 0, R-1 vs calculate_Fe_skymax: max rel diff "
                      f"{rel:.1e}, equal indices {100 * same:.2f}%", flush=True)
                del best, idx
            pack.set_residuals([n[:0] for n in noise])
            torch.cuda.empty_cache()
        del pack
        fe.invalidate()


if __name__ == "__main__":
    main()
