"""Timing of the residual-batch Fp (``fastfp_fp_sweep_residuals``) against one sweep per realisation.

usage: time_fp_batch.py [--cases C2,C4,m12,m304] [--R <counts, default per case>] [--reps 2]

For each PTA shape (C2: 45 pulsars x 5000 TOAs, F = 10^4; C4: 68 x 10^4, F = 10^5; m12 / m304: C2's size with basis
widths 12 and 304) it prints:
  * one ``fastfp_fp_sweep`` of the pack (CUDA events after a warm-up call);
  * the cost per realisation of the separate route -- build a pack with that realisation's residuals
    (``fastfp_pack_create``, host clock) and sweep it -- timed for two realisations and scaled linearly in R;
  * per R: the one-time ``set_residuals`` (host clock, it ends in a synchronise), one ``fastfp_fp_sweep_residuals``
    (CUDA events), the speed-up over R separate builds + sweeps, and Fp evaluations per second, one evaluation being
    one (realisation, pulsar, frequency); plus the time per realisation, which decides the pass size for large R.
The realisations are white noise at the pulsars' own levels; their values do not change the work.
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
from fastfp_b200.fastfp import FastFp  # noqa: E402

# name -> (PTA, F, default realisation counts). The counts at m = 72 put the tile at the top of each family (R = 8, 88,
# 248, 568: 80, 160, 320, 640 rows), which calibrates the per-row costs calculate_Fp_batch chooses its passes with
# (R = 284 is one of the two passes it makes of 568 at C2);
# "m12" does the same for the m <= 40 family (R = 24: 40 rows), "m304" checks the choice for a wide basis.
CASES = {
    "C2": (lambda: synth.make_config("C2"), 10_000, "1,8,64,88,248,284,568"),
    "C4": (lambda: synth.make_config("C4"), 100_000, "1,8,64,88,248,568"),
    "m12": (lambda: synth.make_pta(45, 5000, n_tm=12, white_only=True), 10_000, "1,24,64,304"),
    "m304": (lambda: synth.make_pta(45, 5000, n_tm=12, ncomps=146), 10_000, "8,16,24,336"),
}


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="C2,C4,m12,m304")
    ap.add_argument("--R", default=None)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    name, pl = card()
    print(f"card: {name}, power limit {pl}", flush=True)
    for case in args.cases.split(","):
        make, F, Rdef = CASES[case]
        Rs = [int(r) for r in (args.R or Rdef).split(",")]
        pta = make()
        P = pta.P
        pack = FastFp(pta.psrs).prepare(pta.Nvecs, pta.Ts, pta.sigmas)
        f = torch.tensor(np.linspace(2e-9, 3e-7, F), dtype=torch.float64, device="cuda")
        fa = (f.data_ptr(), F)
        st = torch.cuda.current_stream().cuda_stream
        one = torch.empty(F, dtype=torch.float64, device="cuda")
        t_sweep = timed(lambda: pack.fp_sweep(fa, out=one.data_ptr(), stream=st), args.reps)
        rng = np.random.default_rng(11)
        res = [np.sqrt(N) * rng.standard_normal((max(Rs), N.shape[0])) for N in pta.Nvecs]
        t_sep = []
        for k in range(2):  # the separate route: a pack per realisation, then its sweep
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pk = _cabi.Pack.create(pta.toas, [r[k] for r in res], pta.Nvecs, pta.Ts, pta.sigmas)
            t_build = (time.perf_counter() - t0) * 1e3
            t_sep.append(t_build + timed(lambda: pk.fp_sweep(fa, out=one.data_ptr(), stream=st), args.reps))
            pk.close()
        t_sep = float(np.mean(t_sep))
        print(f"{case} P={P} m={pta.Ts[0].shape[1]} F={F}: fp_sweep {t_sweep:.1f} ms | separate route per realisation (pack build + sweep, "
              f"mean of 2) {t_sep:.1f} ms", flush=True)
        for R in Rs:
            out = torch.empty((R, F), dtype=torch.float64, device="cuda")
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pack.set_residuals([r[:R] for r in res])
            t_set = (time.perf_counter() - t0) * 1e3
            t_b = timed(lambda: pack.fp_sweep_residuals(fa, out=out.data_ptr(), stream=st), args.reps)
            evals = R * P * F / (t_b * 1e-3)
            mp = (-(-pta.Ts[0].shape[1] // 8) + -(-R // 8)) * 8
            print(f"  R={R:4d} ({mp} rows): set_residuals {t_set:8.1f} ms | fp_sweep_residuals {t_b:8.1f} ms "
                  f"({t_b / R:7.3f} ms per realisation, {t_b / t_sweep:6.2f} x one fp_sweep) | R separate "
                  f"(scaled) {R * t_sep:9.1f} ms -> {R * t_sep / t_b:6.1f} x | {evals:.3g} Fp evaluations/s",
                  flush=True)
            del out
        pack.close()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
