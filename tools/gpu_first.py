"""First GPU contact: golden parity, a C2-sized timing and the fp64 pipe peaks."""
import json, os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import fastfp_b200
from fastfp_b200 import synth, _cabi

out = {}
EPS = 2.2e-16
def L(g, k): return [g[f"{k}_{p}"] for p in range(int(g["P"]))]
class Psr:  # duck-typed pulsar
    def __init__(s, t, r): s.toas, s.residuals = t, r
for name in ["fp_white", "fp_red"]:
    g = np.load(f"tests/golden/{name}.npz")
    psrs = [Psr(t, r) for t, r in zip(L(g, "toas"), L(g, "res"))]
    fp = fastfp_b200.FastFp(psrs)
    got = fp(g["freqs"], L(g, "Nvec"), L(g, "T"), L(g, "sigma"))
    ref, tr, cond = g["ref_fp"], g["truth_fp"], g["cond"].sum(0)
    out[name] = dict(
        max_rel_vs_ref=float(np.abs(got / ref - 1).max()),
        max_rel_vs_truth=float(np.abs(got / tr - 1).max()),
        ref_rel_vs_truth=float(np.abs(ref / tr - 1).max()),
        allow_ratio_vs_ref=float((np.abs(got - ref) / (1e-10 * np.abs(ref) + 16 * EPS * cond)).max()),
        err_over_epscond=float((np.abs(got - tr) / (EPS * cond)).max()),
        ref_err_over_epscond=float((np.abs(ref - tr) / (EPS * cond)).max()),
    )
    print(name, out[name], flush=True)
    if name == "fp_white":
        xs = [float(fastfp_b200.get_xCy(g[f"Nvec_{p}"], g[f"T_{p}"], g[f"sigma_{p}"], g[f"x_{p}"], g[f"y_{p}"])) for p in range(int(g["P"]))]
        out["xcy_max_rel"] = float(np.abs(np.array(xs) / g["ref_xcy"] - 1).max())
        print("xcy", out["xcy_max_rel"])

for kind, nm in [(0, "dfma"), (1, "dmma"), (2, "mixed")]:
    tf, ms = _cabi.fp64_peak(kind, 40000)
    out[f"peak_{nm}_tflops"] = tf
    print(nm, tf, "TFLOP/s", ms, "ms", flush=True)

t0 = time.time(); pta = synth.make_config("C2"); print("synth C2", time.time() - t0, flush=True)
fp = fastfp_b200.FastFp(pta.psrs)
t0 = time.time(); fp.prepare(pta.Nvecs, pta.Ts, pta.sigmas); torch.cuda.synchronize(); out["c2_pack_s"] = time.time() - t0
F = 10000
fr = torch.tensor(synth.fp_freqs(F), dtype=torch.float64, device="cuda")
for _ in range(2): res = fp(fr, pta.Nvecs, pta.Ts, pta.sigmas)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(3): res = fp(fr, pta.Nvecs, pta.Ts, pta.sigmas)
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / 3
evals = F * pta.P
flops = sum(2.0 * (2 * m + 5) * n for n, m in zip(fp._pack.n, fp._pack.m)) * F
out["c2"] = dict(ms=ms, evals_per_s=evals / ms * 1e3, dfma_tflops=flops / ms / 1e9)
print("C2", out["c2"], flush=True)
# spot-check C2 against the oracle on a few frequencies
from oracle import fp_oracle
idx = np.array([0, 1, 17, 100, 2500, 9999])
ora = fp_oracle.fp_sweep(synth.fp_freqs(F)[idx], pta.toas, pta.residuals, pta.Nvecs, pta.Ts, pta.sigmas)
got = res.cpu().numpy()[idx]
out["c2_rel_vs_oracle"] = [float(v) for v in np.abs(got / ora - 1)]
print("C2 vs oracle", out["c2_rel_vs_oracle"], got[:3], ora[:3])
out_dir = os.environ.get("OUT_DIR", ".")
os.makedirs(out_dir, exist_ok=True)
json.dump(out, open(os.path.join(out_dir, "gpu_first.json"), "w"), indent=1)
