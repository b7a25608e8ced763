"""Cost of bases wider than one sweep work item (row groups, DESIGN.md section 5h), on the GPU.

usage: time_wide_basis.py [P n F] [--no-split]   (default 45 5000 10000; --no-split: skip the split-rule comparison)

Per width m (640, 704, 1280, 2572): the pack build and its kernels (chol_kernel, or for a wide basis the blocked
chol_diag_kernel / chol_panel_kernel / chol_update_kernel, then build_packets_kernel, ur_kernel, w_kernel; from
torch.profiler), the peak of fastfp_device_bytes during the build (polled from a second thread), the sweep
(fastfp_fp_sweep with device frequencies, CUDA events) and the end-to-end FastFp.calculate_Fp, which also hashes every
byte of the inputs. Then, at two widths, the library's split against ceil(m/640) and ceil(m/320) groups, emulated by
packs of P x g narrow pulsars whose widths are those groups' (the same sweep work without the combine step). Every
pulsar of a pack shares one TOA set, basis and Sigma (the host arrays are the same objects), so the host set-up stays
small; the device work is that of P distinct pulsars. Prints the card's name and power limit first."""
import os
import subprocess
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import fastfp_b200  # noqa: E402
from fastfp_b200 import _cabi, synth  # noqa: E402

ARGS = [a for a in sys.argv[1:] if not a.startswith("--")]
P, n, F = (int(a) for a in ARGS[:3]) if len(ARGS) >= 3 else (45, 5000, 10_000)
SPLIT = "--no-split" not in sys.argv
NCOMPS = 30
BUILD_KERNELS = ("chol_kernel", "chol_diag_kernel", "chol_panel_kernel", "chol_update_kernel",
                 "build_packets_kernel", "ur_kernel", "w_kernel")


def card():
    q = "name,power.limit,clocks.max.sm"
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


def lists(m, P):
    one = synth.make_pta(1, n, n_tm=m - 2 * NCOMPS, ncomps=NCOMPS, seed=5)
    q = one.psrs[0]
    return [q] * P, [one.Nvecs[0]] * P, [one.Ts[0]] * P, [one.sigmas[0]] * P


def build(psrs, N, T, S, profile=False):
    """Pack build: wall time, peak device bytes, kernel times (ms) when profiled."""
    peak, stop = [_cabi.device_bytes()], threading.Event()

    def poll():
        while not stop.is_set():
            peak[0] = max(peak[0], _cabi.device_bytes())
            time.sleep(1e-4)

    th = threading.Thread(target=poll)
    th.start()
    kern = {}
    t0 = time.perf_counter()
    if profile:
        from torch.profiler import ProfilerActivity, profile as prof

        with prof(activities=[ProfilerActivity.CUDA]) as pr:
            pack = _cabi.Pack.create([q.toas for q in psrs], [q.residuals for q in psrs], N, T, S)
            torch.cuda.synchronize()
        for ev in pr.key_averages():
            for k in BUILD_KERNELS:
                if ev.key.startswith(k) or f"::{k}" in ev.key:
                    kern[k] = kern.get(k, 0.0) + ev.device_time_total / 1e3
    else:
        pack = _cabi.Pack.create([q.toas for q in psrs], [q.residuals for q in psrs], N, T, S)
        torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    stop.set()
    th.join()
    return pack, wall, peak[0], kern


def sweep_ms(pack, fr, reps=3):
    pack.fp_sweep(fr)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        pack.fp_sweep(fr)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def split(m, g):
    """near-equal groups in whole blocks of 8 rows (the library's rule, with g given)"""
    nb = -(-m // 8)
    st = [min(m, 8 * (k * (nb // g) + min(k, nb % g))) for k in range(g + 1)]
    return [b - a for a, b in zip(st, st[1:])]


def main():
    print(f"card: {card()}", flush=True)
    print(f"P={P} n={n} F={F}", flush=True)
    fr = torch.tensor(synth.fp_freqs(F), dtype=torch.float64, device="cuda")
    for m in (640, 704, 1280, 2572):
        psrs, N, T, S = lists(m, P)
        base = _cabi.device_bytes()
        pack, wall, peak, kern = build(psrs, N, T, S, profile=True)
        held = _cabi.device_bytes() - base
        ms = sweep_ms(pack, fr)
        groups = len(_cabi.row_groups(m))
        print(f"m={m:4d} groups={groups}: build {wall:7.2f} s (kernels, ms: "
              + ", ".join(f"{k} {kern.get(k, float('nan')):.1f}" for k in BUILD_KERNELS)
              + f"); device bytes held {held / 1e9:.2f} GB, peak during the build {(peak - base) / 1e9:.2f} GB",
              flush=True)
        print(f"   sweep {ms:9.2f} ms = {ms * 1e6 / (F * P * m):.4f} ns per (frequency, pulsar, G row)", flush=True)
        fp = fastfp_b200.FastFp(psrs, path="fp64")
        fp(fr, N, T, S)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fp(fr, N, T, S)
        torch.cuda.synchronize()
        print(f"   calculate_Fp end to end (content hash included) {(time.perf_counter() - t0) * 1e3:9.2f} ms",
              flush=True)
        del pack, fp
        if SPLIT and m in (1280, 2572):
            for label, g in (("library rule", groups), ("ceil(m/640)", -(-m // 640)), ("ceil(m/320)", -(-m // 320))):
                widths = split(m, g)
                lst = [[], [], [], []]
                for w in widths:
                    for x, y in zip(lst, lists(w, P)):
                        x.extend(y)
                pk, _, _, _ = build(*lst)
                print(f"   emulated {label:12s}: {g} groups of {sorted(set(widths))} rows: "
                      f"sweep {sweep_ms(pk, fr):9.2f} ms", flush=True)
                del pk
    print("GP-ECORR C5-shape pulsar against its kernel-ECORR pack: not measured", flush=True)


if __name__ == "__main__":
    main()
