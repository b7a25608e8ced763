"""Timing of the sky-maximised Fe-statistic against the full map.

usage: time_fe_skymax.py [--cases C2,C4] [--sky 768,3072,12288] [--reps 2]

For each PTA shape (C2: 45 pulsars x 5000 TOAs, F = 10^4; C4: 68 x 10^4, a slice of F = 10^5) and each sky grid size S
it prints, from CUDA events after a warm-up call: the Fp sweep alone, fe_skymax end to end, and fe_sweep followed by
an on-device max / argmax over the (S, F) map (where the map fits in device memory); then the fe_skymax kernel time
from torch.profiler in a separate run, and its DFMA rate (14 DFMA per (sky, frequency, pulsar), from the shapes) next
to the DFMA peak (fastfp_fp64_peak kind 0) measured in the same process. The two Fe results are compared bit for bit.
"""
import argparse
import os
import subprocess
import sys

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="C2,C4")
    ap.add_argument("--sky", default="768,3072,12288")
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    name, pl = card()
    peak, _ = _cabi.fp64_peak(0)
    print(f"card: {name}, power limit {pl}; DFMA peak (fastfp_fp64_peak kind 0) {peak:.2f} TFLOP/s")
    free = torch.cuda.mem_get_info()[0]
    rng = np.random.default_rng(7)
    for case in args.cases.split(","):
        cfg, F = CASES[case]
        pta = synth.make_config(cfg)
        fe = FastFe(pta.psrs)
        pack = fe.prepare(pta.Nvecs, pta.Ts, pta.sigmas)
        P = pta.P
        f = torch.tensor(np.linspace(2e-9, 3e-7, F), dtype=torch.float64, device="cuda")
        fa = (f.data_ptr(), F)
        st = torch.cuda.current_stream().cuda_stream
        fp_out = torch.empty(F, dtype=torch.float64, device="cuda")
        t_fp = timed(lambda: pack.fp_sweep(fa, out=fp_out.data_ptr(), stream=st), args.reps)
        for S in (int(s) for s in args.sky.split(",")):
            th, ph = np.arccos(rng.uniform(-1, 1, S)), rng.uniform(0, 2 * np.pi, S)
            fpl, fcr = antenna_pattern(fe.pos, th, ph)
            best = torch.empty(F, dtype=torch.float64, device="cuda")
            idx = torch.empty(F, dtype=torch.int64, device="cuda")

            def skymax():
                pack.fe_skymax(fa, fpl, fcr, out=best.data_ptr(), index_out=idx.data_ptr(), stream=st)

            t_sky = timed(skymax, args.reps)
            line = f"{case} P={P} F={F} S={S}: fp_sweep {t_fp:.1f} ms | fe_skymax {t_sky:.1f} ms"
            if S * F * 8 < 0.6 * free:
                fe_map = torch.empty((S, F), dtype=torch.float64, device="cuda")
                res = {}

                def via_map():
                    pack.fe_sweep(fa, fpl, fcr, out=fe_map.data_ptr(), stream=st)
                    res["v"], res["i"] = torch.max(torch.nan_to_num(fe_map, nan=-np.inf), dim=0)

                t_map = timed(via_map, args.reps)
                # the rule on the map: NaN loses, the lowest index wins a tie, an all-NaN column is (NaN, -1)
                m = torch.nan_to_num(fe_map, nan=-np.inf)
                top = m.max(dim=0).values
                hit = (m == top[None, :]) & ~torch.isnan(fe_map)
                some = hit.any(dim=0)
                want_i = torch.where(some, hit.to(torch.int8).argmax(dim=0), torch.full_like(idx, -1))
                same_i = bool(torch.equal(want_i, idx))
                want_v = torch.where(some, top, torch.full_like(top, float("nan")))
                same_v = bool(torch.equal(torch.nan_to_num(want_v, nan=0.0), torch.nan_to_num(best, nan=0.0))) and \
                    bool(torch.equal(torch.isnan(want_v), torch.isnan(best)))
                line += f" | fe_sweep + max {t_map:.1f} ms | bit-identical values {same_v}, indices {same_i}"
                del fe_map, m, hit
                torch.cuda.empty_cache()
            else:
                line += " | map does not fit"
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                skymax()
                torch.cuda.synchronize()
            k_us = sum(e.device_time_total for e in prof.key_averages() if "fe_skymax_kernel" in e.key)
            tf = 2.0 * 14 * P * S * F / (k_us * 1e-6) / 1e12 if k_us else float("nan")
            line += f" | kernel {k_us / 1e3:.1f} ms, {tf:.2f} TFLOP/s = {100 * tf / peak:.0f}% of the DFMA peak"
            print(line, flush=True)
        del pack
        fe.invalidate()


if __name__ == "__main__":
    main()
