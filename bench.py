#!/usr/bin/env python
"""Benchmark of the Fp frequency-sweep hot path (BASELINE.json metric: Fp evals/s).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--workload C4|C2|C3|C5] [--impl ours|reference]
                    [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...

Default workload = the configuration the metric is quoted on (BASELINE.json north_star / configs[3]):

  C4 (default)  Fp sweep, 68 pulsars x 10 000 TOAs, m = 72, F = 1 000 000 frequencies IN TOTAL, sharded over
                the N ranks (STRONG scaling: N = 1 sweeps all 1e6 bins on one GPU), one NCCL all-gather of
                the per-bin values at the end.
  C2            Fp sweep, 45 x 5000, m = 72, 10 000 frequencies PER GPU (configs[1]; weak scaling)
  C3            noise-marginalised Fp, 45 x 5000, 1000 frequencies x 1000 draws PER GPU (configs[2]; the
                draw axis is sharded; weak scaling)
  C5            noise-marginalised Fp with a block-diagonal (kernel-ECORR) N: 68 x 10 000 TOAs in 2500
                epochs of 4, 10 000 frequencies x 10 000 draws IN TOTAL, draws sharded (configs[4]; strong)
  T             tiny, contract tests only

One "step" = one pass of the hot path over the rank's shard through the public API (`FastFp.calculate_Fp`
/ `NMFP.calculate_nmfp`) followed for N > 1 by the single NCCL all-gather. With the default workload the
JSON line also carries `secondary.C2` and `secondary.C3` (same fields, a few steps each) unless
`--no-secondary` is given.

Timing: a clock spin-up, W >= 3 untimed warm-up steps, then exactly K steps, each bracketed by CUDA events
on the launching stream with an L2 flush (a 256 MiB buffer written) between steps outside the brackets;
barrier + synchronize on both sides; max over ranks. `e2e` repeats the measurement through the same public
call with HOST buffers (pinned): host->device copy of the step's inputs and device->host copy of the result
inside the timed region, including the host-side content hash that guards the cached device pack.

Checks recorded in the line (`checks`): (1) the NCCL-gathered output equals what a single GPU computes for
the same bins, bit for bit (every rank recomputes a slice of ANOTHER rank's shard); (2) an untimed oracle
spot check of bins of the timed result. `--impl reference` times the CPU restatement of the reference
(oracle/, NumPy + threaded pieces, all host cores) on a bounded sample of the same workload; together with
`cpu_baseline` and the spot check it is the only place outside tests/ and smoke() that executes oracle/.

`--dump-outputs DIR` writes what the last timed step of the primary workload returned (rank 0, after the timing)
as DIR/<name>.npy in float64: `fp.npy`, the (F,) Fp values of a plain sweep, or `nmfp.npy`, the (D, F) values of
a noise-marginalised one. An output above 64 MB is replaced by a fixed, seeded sample of its rows
(`nmfp_rows.npy` holds their indices as float64). The inputs are seeded, so two builds run with the same arguments
can be compared output for output.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

WORKLOADS = {
    "C4": dict(kind="fp", P=68, n=10_000, F_total=1_000_000, scaling="strong"),
    "C2": dict(kind="fp", P=45, n=5000, F_per_gpu=10_000, scaling="weak"),
    "C3": dict(kind="nmfp", P=45, n=5000, F=1_000, D_per_gpu=1_000, scaling="weak"),
    "C5": dict(kind="nmfp", P=68, n=10_000, F=10_000, D_total=10_000, blockn=True, epoch=4, scaling="strong"),
    # wide bases (SURVEY 7.3-H3: real pulsars reach several hundred columns): 12 timing-model + 2 x 149 Fourier columns
    "W": dict(kind="fp", P=16, n=5000, F_per_gpu=4096, ncomps=149, scaling="weak"),
    "T": dict(kind="fp", P=3, n=300, F_per_gpu=256, scaling="weak"),  # tiny: tests/test_bench_contract.py
    "TN": dict(kind="nmfp", P=3, n=300, F=64, D_per_gpu=16, scaling="weak"),
}
M_BASIS = 72


def m_of(wl):
    """basis width of a workload: 12 timing-model columns + 2 per Fourier component (30 unless the workload says otherwise)"""
    return 12 + 2 * wl.get("ncomps", 30)

M_VAR = 60  # per-draw (red-noise) block of the basis: 30 Fourier components
METRIC = "Fp evals/sec (freqs x pulsars x draws)"


def total_F(wl, world):
    return wl["F_total"] if "F_total" in wl else wl["F_per_gpu"] * world


def total_D(wl, world):
    return wl["D_total"] if "D_total" in wl else wl["D_per_gpu"] * world


def bytes_per_eval(n, m):
    """Algorithmic bytes of the streaming model (SURVEY.md section 8d): t, Nvec, r, T, Sigma."""
    return 8.0 * (n * (m + 3) + m * m)


def flops_per_eval(n, m):
    """fp64 flops of the hoisted formulation: Y = G [s c] (4 m n) + five weighted sums (10 n)."""
    return (4.0 * m + 10.0) * n


def nmfp_flops_per_eval(n, m, mv, F, D):
    """fp64 flops per (pulsar, frequency, draw) of the noise-marginalised path: stage B applies the
    lower-triangular L^-1 (mv^2/2 entries) to the two columns of z' (2 mv^2) and forms five length-mv
    sums (10 mv); the per-draw factorisation + inversion (~2/3 mv^3) is shared by F frequencies and the
    per-frequency stage A sweep ((4m+10) n) by D draws. Returns (total, stage-B-only)."""
    stage_b = 2.0 * mv * mv + 10.0 * mv
    return stage_b + (2.0 / 3.0) * mv ** 3 / F + flops_per_eval(n, m) / D, stage_b


def measured_traffic(workload):
    """DRAM bytes of one launch of the dominant kernel of this workload, from the committed ncu captures
    (profiles/r*_dram_traffic.json: dram__bytes_read.sum + dram__bytes_write.sum); newest round first."""
    for name in ("r2_dram_traffic.json", "r1_dram_traffic.json"):
        try:
            with open(os.path.join(ROOT, "profiles", name)) as f:
                d = json.load(f)[workload]
            return float(d["dram_bytes_per_launch"]), f"profiles/{name}: {d.get('kernel', 'dominant kernel')}, per launch, " \
                                                      f"{d.get('shard', 'one GPU shard')}"
        except (OSError, KeyError, ValueError):
            continue
    return None, None


def measured_peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        with open(path) as f:
            d = json.load(f)
        return float(d["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    return 3350.0, "H100 SXM data sheet (HBM3)"


def config_of(key, wl, gpus):
    """The workload-defining part of the line: identical for `--impl ours` and `--impl reference`."""
    if wl["kind"] == "nmfp":
        D = total_D(wl, gpus)
        ec = f" in {wl['n'] // wl['epoch']} epochs of {wl['epoch']} TOAs (block-diagonal kernel-ECORR N)" if wl.get("blockn") else ""
        per = "in total, draws sharded" if "D_total" in wl else f"= {wl['D_per_gpu']} per GPU"
        name = (f"{key}: noise-marginalised Fp, {wl['P']} pulsars x {wl['n']} TOAs{ec}, m={M_BASIS} (12 timing-model + "
                f"60 red-noise/CURN Fourier), {wl['F']} frequencies x {D} noise draws {per}, {gpus} GPU(s), fp64")
        return {"workload": name, "P": wl["P"], "n_toas": wl["n"], "m": M_BASIS, "F": wl["F"], "D": D,
                "n_gpus": gpus, "scaling": wl["scaling"]}
    F = total_F(wl, gpus)
    per = "in total, sharded over the GPUs" if "F_total" in wl else f"= {wl['F_per_gpu']} per GPU"
    name = (f"{key}: Fp sweep, {wl['P']} pulsars x {wl['n']} TOAs, m={m_of(wl)} (12 timing-model + {m_of(wl) - 12} Fourier), "
            f"{F} frequencies {per}, {gpus} GPU(s), red+white Woodbury C, fp64")
    return {"workload": name, "P": wl["P"], "n_toas": wl["n"], "m": m_of(wl), "F": F, "D": 1, "n_gpus": gpus,
            "scaling": wl["scaling"]}


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region (read-only queries)."""

    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.proc, self.lines = index, None, []

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", "-i", str(self.index), f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                 "-lms", "100"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
        except OSError:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        self.thread.join(timeout=2)
        sm, smax, pw, reasons = [], [], [], set()
        for line in self.lines:
            parts = [p.strip() for p in line.split(",")]
            if len(parts) < 7:
                continue
            try:
                sm.append(float(parts[0])); smax.append(float(parts[1]))
                pw.append(float(parts[2]))
            except ValueError:
                continue
            for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), parts[3:7]):
                if val == "Active":
                    reasons.add(name)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(smax) if smax else None,
                "power_w_max": max(pw) if pw else None, "samples": len(sm), "reasons": sorted(reasons)}


# ---------------------------------------------------------------------------------------------------
# the reference's CPU path (oracle port) -- cpu_baseline and --impl reference
# ---------------------------------------------------------------------------------------------------
def cpu_reference_rate(wl, world=1, steps=1, warmup=0, target_s=12.0):
    """Plain Fp: the vmapped program's formulas, batched over frequency, spread over all host cores, on a
    bounded sample of the workload (all pulsars x a calibrated number of the grid's frequencies, spread
    evenly over the grid) sized for ~target_s seconds per step. Returns evals/s and metadata."""
    from fastfp_b200 import synth
    from oracle import fp_oracle

    cores = os.cpu_count() or 1
    pta = synth.make_pta(wl["P"], wl["n"], ncomps=wl.get("ncomps", 30))
    F_all = total_F(wl, world)
    grid = synth.fp_freqs(F_all)
    common = (pta.toas, pta.residuals, pta.Nvecs, pta.Ts, pta.sigmas)
    chunk = 64
    fcal = min(F_all, max(chunk, chunk * (-(-cores // wl["P"]))))  # enough pieces to occupy every core
    fp_oracle.fp_sweep_mt(grid[:fcal], *common, workers=cores, chunk=chunk)  # warm-up
    t0 = time.perf_counter()
    fp_oracle.fp_sweep_mt(grid[:fcal], *common, workers=cores, chunk=chunk)
    t_cal = time.perf_counter() - t0
    Fs = int(min(F_all, max(fcal, fcal * target_s / max(t_cal, 1e-3))))
    Fs = max(min(chunk, F_all), Fs // chunk * chunk)
    freqs = grid[:: max(1, F_all // Fs)][:Fs]
    for _ in range(warmup):
        fp_oracle.fp_sweep_mt(freqs, *common, workers=cores, chunk=chunk)
    times = []
    for _ in range(max(1, steps)):
        t0 = time.perf_counter()
        fp_oracle.fp_sweep_mt(freqs, *common, workers=cores, chunk=chunk)
        times.append(time.perf_counter() - t0)
    evals = wl["P"] * len(freqs)
    return evals / statistics.median(times), {
        "cores": cores, "kind": "port",
        "sample": f"{wl['P']} pulsars x {wl['n']} TOAs x {len(freqs)} of the {F_all} frequencies, evenly spaced over "
                  f"the grid ({evals} evals per step, median of {max(1, steps)} step(s)); NumPy/SciPy restatement of the "
                  f"reference formulas, (pulsar, 64-frequency) pieces on a {cores}-thread pool, 1 BLAS thread each",
        "ms_per_step": statistics.median(times) * 1e3,
    }


def nmfp_problem(wl):
    """Inputs of an nmfp workload: (pta, containers, Nvecs-or-BlockNvecs, TNTs)."""
    from fastfp_b200 import BlockNvec, CURN_container, RN_container, synth

    pta = synth.make_pta(wl["P"], wl["n"], ncomps=wl.get("ncomps", 30))
    curn = CURN_container(pta.Ffreqs)
    sigs = [RN_container(q, Ffreqs=pta.Ffreqs, add_curn=True, curn_container=curn) for q in pta.psrs]
    if not wl.get("blockn"):
        return pta, sigs, pta.Nvecs, pta.TNTs
    # kernel ECORR: epochs of `epoch` consecutive TOAs, j_e ~ (0.3 .. 3) x 1e-13 s^2 (seeded)
    rng = np.random.default_rng(20240607 + 777)
    ep = wl["epoch"]
    Nblk, TNTs = [], []
    for p in range(wl["P"]):
        n = wl["n"]
        slices = [slice(a, a + ep) for a in range(0, n - ep + 1, ep)]
        B = BlockNvec(pta.Nvecs[p], slices, rng.uniform(0.3, 3.0, len(slices)) * 1e-13)
        TNT = pta.Ts[p].T @ B.solve(pta.Ts[p])
        Nblk.append(B)
        TNTs.append(0.5 * (TNT + TNT.T))
    return pta, sigs, Nblk, TNTs


def cpu_reference_rate_nmfp(wl, world=1, steps=1, warmup=0, target_s=12.0):
    """nmfp: per draw ``_get_sigmas`` and the frequency sweep of calculate_Fp over all pulsars, on all host
    cores; sample = a calibrated number of draws x (all, or for large F an evenly spaced subset of) the
    frequencies. A block-diagonal N has no reference implementation (fastfp/utils.py:29-31): the port then
    runs the diagonal-N program on the same shapes (a LOWER bound on what a CPU implementation would cost)."""
    from fastfp_b200 import synth
    from oracle import fp_oracle

    cores = os.cpu_count() or 1
    pta = synth.make_pta(wl["P"], wl["n"], ncomps=wl.get("ncomps", 30))
    F_all = wl["F"]
    Fs = min(F_all, 1024)
    freqs = synth.nmfp_freqs(F_all, pta.Tspan)[:: max(1, F_all // Fs)][:Fs]
    phi_args = [dict(psr_name=q.name, n_tm=ntm, Ffreqs=pta.Ffreqs, add_curn=True, curn_Ffreqs=pta.Ffreqs)
                for q, ntm in zip(pta.psrs, pta.n_tm)]
    common = (pta.toas, pta.residuals, pta.Nvecs, pta.Ts)

    def run(samples, nd):
        for d in range(nd):
            pars = {k: v[d] for k, v in samples.items()}
            sigmas = fp_oracle.get_sigmas(pars, pta.TNTs, phi_args)
            fp_oracle.fp_sweep_mt(freqs, *common, sigmas, workers=cores, chunk=64)

    D_all = total_D(wl, world)
    samples = synth.draw_samples(pta, min(64, D_all))
    run(samples, 1)  # warm-up
    t0 = time.perf_counter()
    run(samples, 1)
    t1 = time.perf_counter() - t0
    nd = int(max(1, min(64, D_all, target_s / max(t1, 1e-3))))
    for _ in range(warmup):
        run(samples, nd)
    times = []
    for _ in range(max(1, steps)):
        t0 = time.perf_counter()
        run(samples, nd)
        times.append(time.perf_counter() - t0)
    evals = wl["P"] * len(freqs) * nd
    return evals / statistics.median(times), {
        "cores": cores, "kind": "port",
        "sample": f"{wl['P']} pulsars x {wl['n']} TOAs x {len(freqs)} of the {F_all} frequencies x {nd} of the "
                  f"{D_all} draws ({evals} evals per step, median of {max(1, steps)} step(s)); NumPy/SciPy "
                  f"restatement of NMFP.calculate_nmfp (per draw: _get_sigmas, then the Fp sweep in (pulsar, "
                  f"64-frequency) pieces on a {cores}-thread pool, 1 BLAS thread each)"
                  + ("; diagonal-N program on the same shapes (the reference has no block-diagonal N)" if wl.get("blockn") else ""),
        "ms_per_step": statistics.median(times) * 1e3,
    }


def run_reference(args, key, wl, rank, world):
    if rank != 0:
        return
    fn = cpu_reference_rate_nmfp if wl["kind"] == "nmfp" else cpu_reference_rate
    rate, meta = fn(wl, world=args.gpus, steps=args.steps, warmup=min(args.warmup, 1),
                    target_s=min(12.0, 120.0 / max(1, args.steps + min(args.warmup, 1))))
    emit({
        "impl": "reference", "metric": METRIC, "value": rate, "unit": "evals/s",
        "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": meta["ms_per_step"],
        "higher_is_better": True, "scaling": wl["scaling"], "vs_baseline": None, "dtype": "f64", "data": "synthetic",
        "config": config_of(key, wl, args.gpus),
        "run": {"parallelism": "cpu-host, all cores", "note": "each step = the bounded sample in cpu_baseline.sample"},
        "cpu_baseline": {"value": rate, "unit": "evals/s", "cores": meta["cores"], "kind": meta["kind"],
                         "sample": meta["sample"]},
        "e2e": {"value": rate, "unit": "evals/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    })


# ---------------------------------------------------------------------------------------------------
# GPU arm
# ---------------------------------------------------------------------------------------------------
class Ctx:
    """Per-process CUDA / NCCL context shared by the primary and the secondary workloads."""

    def __init__(self, rank, world, local):
        import torch
        import torch.distributed as dist

        if not torch.cuda.is_available():
            raise SystemExit("bench.py needs a CUDA device (the Fp hot path has no CPU fallback)")
        self.torch, self.dist = torch, dist
        self.rank, self.world, self.local = rank, world, local
        torch.cuda.set_device(local)
        self.dev = torch.device("cuda", local)
        if world > 1:
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            os.environ.setdefault("NCCL_DEBUG", "WARN")  # keep NCCL's version banner off stdout (one JSON line)
            dist.init_process_group("nccl", device_id=self.dev)
        self.flush_buf = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device=self.dev)
        self.last = None  # what the last timed step returned
        self.dump_dir = None  # --dump-outputs: set for the primary workload only

    def barrier(self):
        if self.world > 1:
            self.dist.barrier()
        self.torch.cuda.synchronize()

    def timed(self, fn, steps):
        """sum over `steps` of the CUDA-event time of fn(), L2 flushed before each; max over ranks (ms)"""
        torch = self.torch
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        self.barrier()
        for a, b in ev:
            self.flush_buf.fill_(1.0)  # L2 flush, outside the timed bracket
            a.record()
            self.last = fn()
            b.record()
        self.barrier()
        t = torch.tensor([sum(a.elapsed_time(b) for a, b in ev)], dtype=torch.float64, device=self.dev)
        if self.world > 1:
            self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX)
        return float(t.item())

    def all_ok(self, ok):
        t = self.torch.tensor([1 if ok else 0], dtype=self.torch.int32, device=self.dev)
        if self.world > 1:
            self.dist.all_reduce(t, op=self.dist.ReduceOp.MIN)
        return bool(t.item())

    def close(self):
        if self.world > 1:
            self.dist.destroy_process_group()


DUMP_MAX_BYTES = 64 * 2**20


def dump_output(ctx, name, out):
    """--dump-outputs: the last timed step's result as DIR/<name>.npy (float64); a (D, F) result above 64 MB keeps a
    seeded sample of its rows, whose indices go to DIR/<name>_rows.npy"""
    if ctx.dump_dir is None or ctx.rank != 0:
        return
    os.makedirs(ctx.dump_dir, exist_ok=True)
    a = out.detach().to("cpu", ctx.torch.float64).numpy()
    if a.nbytes > DUMP_MAX_BYTES:
        keep = max(1, DUMP_MAX_BYTES // (2 * a[0].nbytes))
        rows = np.sort(np.random.default_rng(20240607).choice(a.shape[0], size=keep, replace=False))
        a = a[rows]
        np.save(os.path.join(ctx.dump_dir, f"{name}_rows.npy"), rows.astype(np.float64))
    np.save(os.path.join(ctx.dump_dir, f"{name}.npy"), np.ascontiguousarray(a))


def same_bits(torch, a, b):
    """bitwise equality of two float64 tensors (NaN payloads included)"""
    return bool(torch.equal(a.contiguous().view(torch.int64), b.contiguous().view(torch.int64)))


def e2e_steps_for(steps, ms_step):
    """the end-to-end leg repeats the K steps unless that alone would take more than ~30 s"""
    if ms_step * steps <= 30_000.0:
        return steps
    return max(3, int(30_000.0 / ms_step))


def spot_bins(F, Tspan, freqs):
    """bins of the timed result that are checked against the oracle: the grid ends, two interior bins and
    (when the grid reaches down there) the bins next to the first red-noise Fourier frequencies"""
    idx = sorted({0, 1, F // 3, F // 2, F - 2, F - 1} & set(range(F)))
    return np.array(idx, dtype=np.int64)


def run_fp(key, wl, ctx, steps, warmup, with_cpu_baseline):
    """Plain-Fp workload: frequency axis sharded across ranks, pulsar arrays replicated."""
    import fastfp_b200
    from fastfp_b200 import _cabi, parallel, synth

    torch, rank, world, dev = ctx.torch, ctx.rank, ctx.world, ctx.dev
    pta = synth.make_pta(wl["P"], wl["n"], ncomps=wl.get("ncomps", 30))
    m_basis = m_of(wl)
    F_total = total_F(wl, world)
    freqs_np = synth.fp_freqs(F_total)
    freqs_host = torch.from_numpy(freqs_np).pin_memory()
    fp = fastfp_b200.FastFp(pta.psrs, device=ctx.local)
    mats = (pta.Nvecs, pta.Ts, pta.sigmas)
    t0 = time.perf_counter()
    pack = fp.prepare(*mats)
    torch.cuda.synchronize()
    pack_ms = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    fp.prepare(*mats)  # steady state: the content hash of the three lists (every byte), no rebuild
    hash_ms = (time.perf_counter() - t0) * 1e3
    freqs_dev = freqs_host.to(dev)
    lo, hi, per = parallel.shard_bounds(F_total, rank, world)

    def step_device():
        """inputs resident in HBM: sweep the shard, all-gather the bins"""
        return parallel.sharded_sweep(lambda f: fp.calculate_Fp(f, *mats), freqs_dev)

    out_pinned = torch.empty(F_total, dtype=torch.float64).pin_memory()

    def step_e2e():
        """public API with host buffers: H2D of the shard's frequencies, sweep, gather, D2H of Fp"""
        f = freqs_host[lo:hi].to(dev, non_blocking=True)
        full = parallel.sharded_sweep(lambda _: fp.calculate_Fp(f, *mats), freqs_dev)
        out_pinned.copy_(full, non_blocking=True)
        return out_pinned

    # clock spin-up (the SM clock needs ~0.4 s of load to leave its idle state), then W warm-ups. The
    # spin-up is wall-clock bounded, so it must stay rank-local: no collective inside.
    shard0 = freqs_dev[lo:min(hi, lo + 16384)].contiguous()
    t_spin = time.perf_counter()
    while time.perf_counter() - t_spin < 1.5:
        fp.calculate_Fp(shard0, *mats)
        torch.cuda.synchronize()
    ctx.barrier()
    for _ in range(warmup):
        step_device()
    sampler = ClockSampler(ctx.local)
    if rank == 0:
        sampler.start()
    launches0 = _cabi.kernel_launches()
    total_ms = ctx.timed(step_device, steps)
    launches = _cabi.kernel_launches() - launches0
    clocks = sampler.stop() if rank == 0 else None
    dump_output(ctx, "fp", ctx.last)
    ms_step = total_ms / steps
    ne2e = e2e_steps_for(steps, ms_step)
    for _ in range(2 if ms_step < 1000.0 else 1):
        step_e2e()
    e2e_ms = ctx.timed(step_e2e, ne2e) / ne2e

    # ---- checks (untimed) -----------------------------------------------------------------------
    full = step_device()
    torch.cuda.synchronize()
    checks = {}
    # (1) what the gather delivered for ANOTHER rank's shard == what this GPU computes alone for those bins
    nb = (rank + 1) % world
    lo2, hi2, _ = parallel.shard_bounds(F_total, nb, world)
    if world == 1:  # one GPU: a slice from the middle of the grid recomputed as its own call
        lo2 = F_total // 2
        hi2 = F_total
    k = min(4096, hi2 - lo2)
    again = fp.calculate_Fp(freqs_dev[lo2:lo2 + k].contiguous(), *mats)
    ok = same_bits(torch, again, full[lo2:lo2 + k])
    nonfinite = torch.nonzero(~torch.isfinite(full)).flatten()
    checks["gathered_equals_single_gpu"] = {
        "ok": ctx.all_ok(ok), "bins_per_rank": int(k),
        "non_finite_bins": {"count": int(nonfinite.numel()),
                            "freqs_hz": [float(freqs_np[i]) for i in nonfinite[:8].cpu().numpy().tolist()],
                            "note": "bins where M = [[(s|s),(s|c)],[(c|s),(c|c)]] is numerically singular: the synthetic "
                                    "timing model holds yearly and half-yearly sinusoids with phi = 1e40, so at f = 1/yr "
                                    "and 2/yr (to ~1e-5 relative) the Earth-term basis lies inside span(T) and the "
                                    "reference formula itself returns rounding noise there (NaN compares equal to NaN "
                                    "in this check)"},
        "how": ("every rank recomputes the first bins of the next rank's shard alone and compares them with the "
                "NCCL-gathered output bit for bit" if world > 1 else
                "one GPU: a slice from the middle of the grid recomputed as a separate call, bit for bit")}
    # (2) oracle spot check of the timed result (rank 0)
    if rank == 0:
        from oracle import fp_oracle

        idx = spot_bins(F_total, pta.Tspan, freqs_np)
        want = fp_oracle.fp_sweep(freqs_np[idx], pta.toas, pta.residuals, *mats)
        got = full[torch.from_numpy(idx).to(dev)].cpu().numpy()
        rel = np.abs(got / want - 1.0)
        well = freqs_np[idx] > 40.0 / pta.Tspan  # above the red-noise band: the plain 1e-10 applies
        checks["oracle_spot"] = {
            "bins": idx.tolist(), "max_rel_dev": float(rel.max()),
            "max_rel_dev_well_conditioned": float(rel[well].max()) if well.any() else None,
            "n_well_conditioned": int(well.sum()), "tolerance_well_conditioned": 1e-10,
            "ok": bool((rel[well] <= 1e-10).all() and (rel <= 1e-6).all()),
            "how": "oracle/fp_oracle.fp_sweep (NumPy restatement of fastfp/fastfp.py:69-92) on these bins of the "
                   "gathered result of an untimed repeat of the step; bins inside the red-noise band (f < 40/Tspan) "
                   "are ill-conditioned in the reference formula itself and held to 1e-6 here (tests/ bound them "
                   "against the longdouble truth)"}

    # dominant kernel alone, this rank's shard (for the roofline)
    ks, ke = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    shard = freqs_dev[lo:hi].contiguous()
    nk = 3 if ms_step < 1000.0 else 1
    t_spin = time.perf_counter()
    while time.perf_counter() - t_spin < 0.6 and ms_step < 1000.0:  # the checks above ran on the host: clocks back up
        fp.calculate_Fp(shard, *mats)
        torch.cuda.synchronize()
    fp.calculate_Fp(shard[:1024], *mats)
    torch.cuda.synchronize()
    ks.record()
    for _ in range(nk):
        fp.calculate_Fp(shard, *mats)
    ke.record()
    torch.cuda.synchronize()
    kern_ms = ks.elapsed_time(ke) / nk
    pack_bytes = pack.nbytes
    sweep_path = pack.path
    fp.invalidate()  # free this workload's device pack before the next one is built

    if rank != 0:
        return None
    evals_step = float(F_total) * wl["P"]
    evals_kernel = float(hi - lo) * wl["P"]
    hbm_peak, peak_src = measured_peaks()
    ach_gbs = evals_kernel * bytes_per_eval(wl["n"], m_basis) / (kern_ms * 1e-3) / 1e9
    traffic, traffic_src = measured_traffic(key)
    fp64_peak, _ = _cabi.fp64_peak(1, 20000, device=ctx.local)  # DMMA loop, same pipe as DFMA
    ach_tf = evals_kernel * flops_per_eval(wl["n"], m_basis) / (kern_ms * 1e-3) / 1e12
    if sweep_path == "i8":
        # The contraction runs on the INT8 tensor path: Y = G [s c] as 28 products of 8-bit digit planes
        # (wgmma .s32.s8.s8, exact int32 accumulation). Algorithmic integer ops per eval: 28 plane products
        # x 2 (multiply, add) x 2 columns (sin, cos) x (m + 1) rows (basis + the C^-1 r row) x n TOAs.
        i8_peak, _ = _cabi.fp64_peak(17, 2000, device=ctx.local)
        i8_shape, _ = _cabi.fp64_peak(18, 4000, device=ctx.local)
        ops_eval = 28.0 * 2.0 * 2.0 * (m_basis + 1) * wl["n"]
        ach_top = evals_kernel * ops_eval / (kern_ms * 1e-3) / 1e12
        nst = -(-wl["n"] // 32)
        rows_pad = 32 * -(-(m_basis + 1) // 32)
        passes = -(-rows_pad // 128)  # row groups of 128 operand rows: one pass over the TOAs each
        items = wl["P"] * -(-(hi - lo) // 16) * passes
        exec_top = items * nst * 28.0 * 2.0 * 128 * 32 * 32 / (kern_ms * 1e-3) / 1e12
        smem_stage = 28.0 * 2 * 3072 + 7.0 * min(rows_pad, 128) * 32 + 7168
        sm_count = torch.cuda.get_device_properties(ctx.local).multi_processor_count
        smem_peak = 128.0 * sm_count * (clocks["sm_mhz"] if clocks and clocks.get("sm_mhz") else 1965.0) * 1e6 / 1e9
        roofline = {
            "bound": "tensor", "pipe": "INT8 tensor path (wgmma .s32.s8.s8, int32 accumulators in registers)",
            "achieved": ach_top, "peak": i8_peak, "unit": "TOP/s", "frac": ach_top / i8_peak,
            "traffic": traffic, "traffic_source": traffic_src,
            "peak_source": "measured live on this GPU: fastfp_fp64_peak kind 17 (back-to-back s8 wgmmas, m64n256k32, "
                           "two warpgroups per SM); MEASURED_PEAKS.json holds a bf16 figure only",
            "kernel": "fp_sweep_i8_kernel (persistent, warp-specialised: TMA / wgmma issue + epilogue / sincos producers)",
            "kernel_ms": kern_ms, "ops_per_eval": ops_eval,
            "shape_bound": {"achieved": exec_top, "peak": i8_shape, "unit": "TOP/s", "frac": exec_top / i8_shape,
                            "note": "executed MMA work (128-row operands, m + 1 real rows in all) against the "
                                    "same 28-product stage issued back to back (kind 18): each m64n32k32 wgmma reads 3 KB "
                                    "of operands from shared memory; the 7 accumulators of a 128 x 32 tile take 112 "
                                    "registers per consumer thread, so N cannot grow"},
            "smem_bound": {
                "achieved": items * nst * smem_stage / (kern_ms * 1e-3) / 1e9, "peak": smem_peak, "unit": "GB/s",
                "frac": items * nst * smem_stage / (kern_ms * 1e-3) / 1e9 / smem_peak, "bytes_per_stage": smem_stage,
                "note": "shared-memory traffic of one 32-TOA x 16-frequency stage (2 x 28 wgmmas x 3 KB of operand reads, "
                        "the TMA write of the G planes, the producers' 7 KB of sin/cos planes) against 128 B/clk/SM at the "
                        "sampled SM clock: the floor of this formulation; the rest of the step is the fp64 sin/cos work"},
            "fp64_equivalent": {"achieved": ach_tf, "unit": "TFLOP/s", "fp64_pipe_peak": fp64_peak,
                                "ratio": ach_tf / fp64_peak,
                                "note": "the same statistic in fp64 flops (4m+10)n per eval against the fp64 pipe peak the "
                                        "DMMA kernel is bound by"},
            "note": "algorithmic INT8 ops = 112 (m+1) n per eval; padding rows of the 128-row operand and the producers' "
                    "fp64 sincos work are not counted"}
    else:
        roofline = {"bound": "tensor", "pipe": "fp64 tensor path (DMMA; DFMA shares the pipe)",
                    "achieved": ach_tf, "peak": fp64_peak, "unit": "TFLOP/s", "frac": ach_tf / fp64_peak,
                    "traffic": traffic, "traffic_source": traffic_src,
                    "peak_source": "measured live on this GPU: fastfp_fp64_peak (mma.sync.m8n8k4.f64 loop); "
                                   "MEASURED_PEAKS.json holds no fp64 figure",
                    "kernel": "fp_sweep_kernel (persistent, warp-specialised)", "kernel_ms": kern_ms,
                    "flops_per_eval": flops_per_eval(wl["n"], m_basis),
                    "note": "algorithmic flops (4m+10)n per eval: Y = G[s c] and the five weighted sums; the "
                            "sincos generation that must also run on this pipe is not counted"}
    line = {
        "metric": METRIC, "value": evals_step / ms_step * 1e3, "unit": "evals/s",
        "n_gpus": world, "steps": steps, "warmup": warmup, "ms_per_step": ms_step,
        "higher_is_better": True, "scaling": wl["scaling"], "vs_baseline": None, "dtype": "f64", "data": "synthetic",
        "config": config_of(key, wl, world),
        "run": {"parallelism": f"freq-shard x{world} ({hi - lo} bins on rank 0), pulsar arrays replicated, one NCCL "
                               "all-gather of the bins",
                "l2": "256 MiB buffer written between timed steps (L2 flush); packed inputs are "
                      f"{pack_bytes / 2**20:.0f} MiB per GPU",
                "pack_ms_one_time": pack_ms, "content_hash_ms_per_call": hash_ms,
                "sweep_kernel": {"i8": "INT8 tensor-core kernel (wgmma)", "fp64": "fp64 DMMA kernel"}[sweep_path],
                "freqs_total": F_total, "evals_per_step": evals_step},
        "e2e": {"value": evals_step / e2e_ms * 1e3, "unit": "evals/s", "ms_per_step": e2e_ms, "steps": ne2e,
                "h2d_bytes_per_step": int(8 * F_total), "d2h_bytes_per_step": int(8 * F_total * world),
                "cold": {"value": evals_step / (e2e_ms + pack_ms) * 1e3, "unit": "evals/s",
                         "note": "first call of a process: one-time pack (upload + Cholesky + G build) + one step"}},
        "gpu_launches": int(launches),
        "clocks": clocks,
        "checks": checks,
        "roofline": roofline,
        "roofline_hbm": {"bound": "hbm", "achieved": ach_gbs, "peak": hbm_peak, "unit": "GB/s",
                         "frac": ach_gbs / hbm_peak, "traffic": traffic, "peak_source": peak_src,
                         "note": "algorithmic bytes 8(n(m+3)+m^2) per eval (the reference's streaming model); "
                                 "every input is frequency-independent and L2-resident and tiles are reused "
                                 "across the frequencies of a tile, so this effective figure exceeds 1 by "
                                 "construction -- HBM is not the bound, measured DRAM traffic per launch is `traffic`"},
    }
    if with_cpu_baseline and world == 1:
        rate, meta = cpu_reference_rate(wl, world=world, steps=1)
        line["cpu_baseline"] = {"value": rate, "unit": "evals/s", "cores": meta["cores"], "kind": meta["kind"],
                                "sample": meta["sample"]}
    return line


def run_nmfp(key, wl, ctx, steps, warmup, with_cpu_baseline):
    """nmfp workload: NMFP.calculate_nmfp over (draws x frequencies); draws sharded across ranks."""
    import fastfp_b200
    from fastfp_b200 import _cabi, parallel, synth

    torch, rank, world, dev = ctx.torch, ctx.rank, ctx.world, ctx.dev
    pta, sigs, Nvecs, TNTs = nmfp_problem(wl)
    F, D_total = wl["F"], total_D(wl, world)
    nm = fastfp_b200.NMFP(pta.psrs, sigs, device=ctx.local)
    mats = (Nvecs, pta.Ts, TNTs)
    t0 = time.perf_counter()
    pack = nm.prepare(*mats)
    torch.cuda.synchronize()
    pack_ms = (time.perf_counter() - t0) * 1e3
    samples = synth.draw_samples(pta, D_total)
    freqs_np = synth.nmfp_freqs(F, pta.Tspan)
    freqs_host = torch.from_numpy(freqs_np).pin_memory()
    freqs_dev = freqs_host.to(dev)
    lo, hi, _ = parallel.shard_bounds(D_total, rank, world)
    mine = {k: v[lo:hi] for k, v in samples.items()}  # this rank's draws (the reference's host dict)

    def step_device():
        return parallel.sharded_draws(lambda a, b: nm.calculate_nmfp_2d(freqs_dev, mine, *mats), D_total)

    out_pinned = torch.empty((D_total, F), dtype=torch.float64).pin_memory()

    def step_e2e():
        f = freqs_host.to(dev, non_blocking=True)
        full = parallel.sharded_draws(lambda a, b: nm.calculate_nmfp_2d(f, mine, *mats), D_total)
        out_pinned.copy_(full, non_blocking=True)
        return out_pinned

    few = {k: v[lo:min(hi, lo + 32)] for k, v in samples.items()}
    t_spin = time.perf_counter()
    while time.perf_counter() - t_spin < 1.5:  # rank-local spin-up (no collective: wall-clock bounded)
        nm(freqs_dev, few, *mats)
        torch.cuda.synchronize()
    ctx.barrier()
    for _ in range(warmup):
        step_device()
    sampler = ClockSampler(ctx.local)
    if rank == 0:
        sampler.start()
    launches0 = _cabi.kernel_launches()
    total_ms = ctx.timed(step_device, steps)
    launches = _cabi.kernel_launches() - launches0
    clocks = sampler.stop() if rank == 0 else None
    dump_output(ctx, "nmfp", ctx.last)
    ms_step = total_ms / steps
    ne2e = e2e_steps_for(steps, ms_step)
    for _ in range(2 if ms_step < 1000.0 else 1):
        step_e2e()
    e2e_ms = ctx.timed(step_e2e, ne2e) / ne2e

    # ---- checks (untimed) -----------------------------------------------------------------------
    full = step_device()
    torch.cuda.synchronize()
    checks = {}
    nb = (rank + 1) % world
    lo2, hi2, _ = parallel.shard_bounds(D_total, nb, world)
    if world == 1:
        lo2 = D_total // 2
    k = min(8, hi2 - lo2)
    again = nm(freqs_dev, {kk: v[lo2:lo2 + k] for kk, v in samples.items()}, *mats)
    ok = same_bits(torch, again, full[lo2:lo2 + k])
    checks["gathered_equals_single_gpu"] = {
        "ok": ctx.all_ok(ok), "draws_per_rank": int(k), "non_finite": int((~torch.isfinite(full)).sum().item()),
        "how": ("every rank recomputes the first draws of the next rank's shard alone and compares the rows with "
                "the NCCL-gathered (D, F) output bit for bit" if world > 1 else
                "one GPU: draws from the middle of the batch recomputed as a separate call, bit for bit")}
    if rank == 0 and not wl.get("blockn"):
        from oracle import fp_oracle

        phi_args = [dict(psr_name=q.name, n_tm=ntm, Ffreqs=pta.Ffreqs, add_curn=True, curn_Ffreqs=pta.Ffreqs)
                    for q, ntm in zip(pta.psrs, pta.n_tm)]
        bins = np.array(sorted({0, min(F - 1, 45), F // 2, F - 2, F - 1} & set(range(F))), dtype=np.int64)
        draws = sorted({0, D_total - 1})
        sub = {kk: v[draws] for kk, v in samples.items()}
        want = fp_oracle.nmfp_sweep(freqs_np[bins], sub, pta.toas, pta.residuals, pta.Nvecs, pta.Ts, pta.TNTs, phi_args)
        got = full[draws][:, torch.from_numpy(bins).to(dev)].cpu().numpy()
        rel = np.abs(got / want - 1.0)
        well = freqs_np[bins] > 40.0 / pta.Tspan
        checks["oracle_spot"] = {
            "draws": draws, "bins": bins.tolist(), "max_rel_dev": float(rel.max()),
            "max_rel_dev_well_conditioned": float(rel[:, well].max()) if well.any() else None,
            "tolerance_well_conditioned": 1e-10,
            "ok": bool((rel[:, well] <= 1e-10).all() and (rel <= 1e-5).all()),
            "how": "oracle/fp_oracle.nmfp_sweep (restatement of fastfp/nmfp.py:57-119) on these (draw, bin) entries of "
                   "the gathered result of an untimed repeat; the nmfp grid sits exactly on the red-noise Fourier "
                   "frequencies k/Tspan, so bins with k < 40 are ill-conditioned in the reference formula itself"}
    elif rank == 0:
        checks["oracle_spot"] = {"ok": None, "how": "block-diagonal N: no reference implementation to restate "
                                 "(fastfp/utils.py:29-31); parity of this path is pinned by tests/test_gpu_blockn.py and "
                                 "the C5-shape test through the equivalent GP-basis formulation"}

    # per-stage kernel times of this rank's shard (events inside the library, on the launching stream)
    pack.stage_timing(True)
    stage = np.zeros(3)
    nrep = 3 if ms_step < 1000.0 else 1
    for _ in range(nrep):
        nm(freqs_dev, mine, *mats)
        stage += np.array(pack.stage_ms())
    stage /= nrep
    pack.stage_timing(False)
    nm.invalidate()  # free this workload's device pack before the next one is built

    if rank != 0:
        return None
    evals_step = float(F) * D_total * wl["P"]
    evals_rank = float(F) * (hi - lo) * wl["P"]
    fl_total, fl_b = nmfp_flops_per_eval(wl["n"], M_BASIS, M_VAR, F, hi - lo)
    fp64_peak, _ = _cabi.fp64_peak(1, 20000, device=ctx.local)
    hbm_peak, peak_src = measured_peaks()
    ach_b = evals_rank * fl_b / (stage[2] * 1e-3) / 1e12
    ach_all = evals_rank * fl_total / (stage.sum() * 1e-3) / 1e12
    ach_gbs = evals_rank * bytes_per_eval(wl["n"], M_BASIS) / (stage.sum() * 1e-3) / 1e9
    traffic, traffic_src = measured_traffic(key)
    line = {
        "metric": METRIC, "value": evals_step / ms_step * 1e3,
        "unit": "evals/s", "n_gpus": world, "steps": steps, "warmup": warmup, "ms_per_step": ms_step,
        "higher_is_better": True, "scaling": wl["scaling"], "vs_baseline": None, "dtype": "f64", "data": "synthetic",
        "config": config_of(key, wl, world),
        "run": {"parallelism": f"draw-shard x{world} ({hi - lo} draws on rank 0), pulsar arrays replicated, one NCCL "
                               f"all-gather of the (D, F) rows ({8 * F * (hi - lo) / 1e6:.1f} MB per rank)" +
                               ("; the draw-independent stage A is sharded over the frequency tiles and its outputs "
                                "all-gathered (two NCCL all-gathers per step) instead of being repeated on every rank"
                                if world > 1 else ""),
                "l2": "256 MiB buffer written between timed steps (L2 flush)",
                "inputs": "frequencies resident in HBM; the noise draws are the reference's host dict of "
                          f"(D,) arrays ({8 * (2 * wl['P'] + 2) * (hi - lo)} bytes per GPU), uploaded inside "
                          "every step of both timings",
                "pack_ms_one_time": pack_ms, "draws_total": D_total, "evals_per_step": evals_step},
        "e2e": {"value": evals_step / e2e_ms * 1e3, "unit": "evals/s", "ms_per_step": e2e_ms, "steps": ne2e,
                "h2d_bytes_per_step": int(8 * F + 8 * (2 * wl["P"] + 2) * (hi - lo)) * world,
                "d2h_bytes_per_step": int(8 * F * D_total * world)},
        "gpu_launches": int(launches),
        "clocks": clocks,
        "checks": checks,
        "roofline": {"bound": "tensor", "pipe": "fp64 tensor path (DMMA; DFMA shares the pipe)",
                     "kernel": "nmfp_stageB_kernel", "achieved": ach_b, "peak": fp64_peak, "unit": "TFLOP/s",
                     "frac": ach_b / fp64_peak, "kernel_ms": float(stage[2]), "flops_per_eval": fl_b,
                     "traffic": traffic, "traffic_source": traffic_src,
                     "all_stages": {"achieved": ach_all, "frac": ach_all / fp64_peak,
                                    "flops_per_eval": fl_total, "ms": float(stage.sum())},
                     "stage_ms": {"stage_A_sweep": float(stage[0]), "factor": float(stage[1]),
                                  "stage_B": float(stage[2])},
                     "peak_source": "measured live on this GPU: fastfp_fp64_peak (mma.sync.m8n8k4.f64 loop); "
                                    "MEASURED_PEAKS.json holds no fp64 figure",
                     "note": "algorithmic flops 2 mv^2 + 10 mv per eval for stage B (exact triangle, mv = 60)"},
        "roofline_hbm": {"bound": "hbm", "achieved": ach_gbs, "peak": hbm_peak, "unit": "GB/s",
                         "frac": ach_gbs / hbm_peak, "peak_source": peak_src,
                         "note": "algorithmic bytes 8(n(m+3)+m^2) per eval (the reference re-streams every input "
                                 "for each (frequency, draw)); here they are read once per frequency (stage A) "
                                 "and the per-draw work runs on mv x mv blocks, so this effective figure exceeds "
                                 "1 by construction -- HBM is not the bound"},
    }
    if with_cpu_baseline and world == 1:
        rate, meta = cpu_reference_rate_nmfp(wl, world=world, steps=1)
        line["cpu_baseline"] = {"value": rate, "unit": "evals/s", "cores": meta["cores"], "kind": meta["kind"],
                                "sample": meta["sample"]}
    return line


_JSON_OUT = None


def emit(line):
    """The one JSON line goes to the process's original stdout; everything else that libraries write to
    fd 1 (NCCL prints its version banner there) was redirected to stderr in main()."""
    out = _JSON_OUT or sys.stdout
    out.write(json.dumps(line) + "\n")
    out.flush()


def main():
    global _JSON_OUT
    _JSON_OUT = os.fdopen(os.dup(1), "w")
    os.dup2(2, 1)
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workload", choices=sorted(WORKLOADS), default=None)
    ap.add_argument("--impl", choices=["ours", "reference"], default="ours")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-secondary", action="store_true")
    ap.add_argument("--sweep-path", choices=["auto", "fp64", "i8", "prefer-i8"], default=None,
                    help="kernel of the plain-Fp sweep (default auto: the fp64 DMMA kernel)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed step's output of the primary workload to DIR/<name>.npy (float64)")
    args = ap.parse_args()
    if args.steps < 1:
        raise SystemExit("--steps must be >= 1")
    args.warmup = max(args.warmup, 3) if args.impl == "ours" else args.warmup
    key = args.workload or "C4"
    wl = WORKLOADS[key]
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))

    if args.impl == "reference":
        run_reference(args, key, wl, rank, world)
        return
    if os.environ.get("FASTFP_DBG") and not os.environ.get("FASTFP_BENCH_ALLOW_DBG"):
        raise SystemExit("FASTFP_DBG is set: it only acts on developer builds that can switch work off; unset it")
    if os.environ.get("FASTFP_B200_NVCC_FLAGS") and not os.environ.get("FASTFP_BENCH_ALLOW_DBG"):
        raise SystemExit("FASTFP_B200_NVCC_FLAGS is set: bench.py only measures the library as shipped")

    if args.sweep_path:
        os.environ["FASTFP_B200_PATH"] = args.sweep_path
    ctx = Ctx(rank, world, local)
    runner = run_nmfp if wl["kind"] == "nmfp" else run_fp
    ctx.dump_dir = args.dump_outputs
    line = runner(key, wl, ctx, args.steps, args.warmup, not args.no_cpu_baseline)
    ctx.dump_dir = None
    if args.workload is None and not args.no_secondary:
        sec = {}
        for k2 in ("C2", "C3", "W"):
            w2 = WORKLOADS[k2]
            r2 = run_nmfp if w2["kind"] == "nmfp" else run_fp
            res = r2(k2, w2, ctx, min(args.steps, 10), 3, False)
            if res is not None:
                sec[k2] = res
        if line is not None:
            line["secondary"] = sec
    if line is not None:
        bad = [name for name, c in line.get("checks", {}).items() if c.get("ok") is False]
        for k2, l2 in line.get("secondary", {}).items():
            bad += [f"{k2}.{name}" for name, c in l2.get("checks", {}).items() if c.get("ok") is False]
        line["checks_failed"] = bad
        # tuning switches of the library that change the schedule, never the results: recorded when set
        knobs = {k: os.environ[k] for k in ("FASTFP_B200_PATH", "FASTFP_B200_NMFP_LF_MB")
                 if k in os.environ}
        if knobs:
            line["env"] = knobs
        emit(line)
        if bad:
            print(f"bench.py: result checks FAILED: {bad}", file=sys.stderr)
            ctx.close()
            raise SystemExit(3)
    ctx.close()


if __name__ == "__main__":
    main()
