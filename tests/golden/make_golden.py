"""Generate the golden fixtures in this directory by executing the UNMODIFIED reference
source (a checkout of gabefreedman/fastfp, ``fastfp/*.py``) on seeded synthetic inputs.

JAX and ``enterprise`` are not installable in the build image (no network), so the reference
modules are imported with two stand-ins placed in ``sys.modules`` first:

* ``jax`` / ``jax.numpy`` -> a thin NumPy-backed shim (``jit`` = identity, ``vmap`` = Python
  loop, ``x.at[i].set/add`` = functional copy-update, everything else forwarded to NumPy
  in float64). The reference's *formulas, argument order and operation order* therefore
  execute exactly as written; only the primitive kernels (XLA's sin/cos/dot/LU) are NumPy's.
* ``enterprise*`` -> empty stub modules (they are imported at the top of
  ``fastfp/utils.py`` but never touched by the hot path).

Run with the reference checkout named by FASTFP_REFERENCE:
    FASTFP_REFERENCE=<path to fastfp> python tests/golden/make_golden.py
Outputs: tests/golden/fp_white.npz, fp_red.npz, nmfp.npz  (inputs + reference outputs +
longdouble truth), all small enough to commit. Nothing here runs on the GPU.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REFERENCE = os.environ.get("FASTFP_REFERENCE", "")


# --------------------------------------------------------------------------------------
# NumPy-backed jax shim
# --------------------------------------------------------------------------------------
class ShimArray(np.ndarray):
    @property
    def at(self):
        return _At(self)


class _At:
    def __init__(self, arr):
        self.arr = arr

    def __getitem__(self, idx):
        return _AtIdx(self.arr, idx)


class _AtIdx:
    def __init__(self, arr, idx):
        self.arr, self.idx = arr, idx

    def set(self, v):
        out = np.array(self.arr, copy=True).view(ShimArray)
        out[self.idx] = v
        return out

    def add(self, v):
        out = np.array(self.arr, copy=True).view(ShimArray)
        out[self.idx] = out[self.idx] + v
        return out


def _wrap(x):
    if isinstance(x, np.ndarray) and not isinstance(x, ShimArray):
        return x.view(ShimArray)
    return x


class _JnpModule(types.ModuleType):
    pi = np.pi

    def __getattr__(self, name):
        target = getattr(np, name)
        if callable(target) and not isinstance(target, type):

            def f(*a, **k):
                return _wrap(target(*a, **k))

            return f
        return target


def _vmap(fn, in_axes):
    def mapped(*args):
        n = None
        for a, ax in zip(args, in_axes):
            if ax is not None:
                n = len(next(iter(a.values()))) if isinstance(a, dict) else np.shape(a)[ax]
        outs = []
        for i in range(n):
            call = []
            for a, ax in zip(args, in_axes):
                if ax is None:
                    call.append(a)
                elif isinstance(a, dict):
                    call.append({k: v[i] for k, v in a.items()})
                else:
                    call.append(np.take(a, i, axis=ax))
            outs.append(fn(*call))
        return _wrap(np.stack([np.asarray(o) for o in outs]))

    return mapped


def install_shims():
    jax = types.ModuleType("jax")
    jnp = _JnpModule("jax.numpy")
    jnp.linalg = types.SimpleNamespace(solve=lambda a, b: _wrap(np.linalg.solve(a, b)))
    jax.numpy = jnp
    jax.jit = lambda f: f
    jax.vmap = _vmap
    jax.Array = ShimArray
    jax.config = types.SimpleNamespace(update=lambda *a, **k: None)
    jax.default_backend = lambda: "numpy-shim"
    tree_util = types.ModuleType("jax.tree_util")
    tree_util.register_pytree_node_class = lambda c: c
    jax.tree_util = tree_util
    sys.modules.update({"jax": jax, "jax.numpy": jnp, "jax.tree_util": tree_util})
    for name, attrs in {
        "enterprise": [],
        "enterprise.signals": [],
        "enterprise.signals.parameter": ["Constant"],
        "enterprise.signals.white_signals": ["MeasurementNoise"],
        "enterprise.signals.gp_signals": ["TimingModel"],
        "enterprise.signals.signal_base": ["PTA"],
        "enterprise_extensions": [],
        "enterprise_extensions.model_utils": ["get_tspan"],
        "enterprise_extensions.blocks": ["red_noise_block", "common_red_noise_block", "white_noise_block"],
    }.items():
        mod = types.ModuleType(name)
        for a in attrs:
            setattr(mod, a, None)
        sys.modules[name] = mod


# --------------------------------------------------------------------------------------
def main():
    if not REFERENCE:
        raise SystemExit("set FASTFP_REFERENCE to a checkout of the reference fastfp source")
    install_shims()
    sys.path.insert(0, REFERENCE)
    sys.path.insert(0, REPO)
    import fastfp.fastfp as ref_fastfp  # noqa: E402  (the reference package)
    import fastfp.nmfp as ref_nmfp  # noqa: E402
    import fastfp.utils as ref_utils  # noqa: E402
    import jax  # the shim

    assert ref_fastfp.__file__.startswith(REFERENCE), ref_fastfp.__file__
    from fastfp_b200 import synth
    from oracle import truth

    def pack_inputs(pta):
        d = {"P": pta.P, "Tspan": pta.Tspan}
        for p in range(pta.P):
            d[f"toas_{p}"] = pta.psrs[p].toas
            d[f"res_{p}"] = pta.psrs[p].residuals
            d[f"Nvec_{p}"] = pta.Nvecs[p]
            d[f"T_{p}"] = pta.Ts[p]
            d[f"TNT_{p}"] = pta.TNTs[p]
            d[f"sigma_{p}"] = pta.sigmas[p]
            d[f"ntm_{p}"] = pta.n_tm[p]
            d[f"name_{p}"] = pta.psrs[p].name
        return d

    def run_fp(pta, freqs):
        obj = ref_fastfp.FastFp(pta.psrs, None)
        fn = jax.vmap(obj.calculate_Fp, in_axes=(0, None, None, None))  # examples/run_fp.py:63
        fps = np.asarray(fn(freqs, pta.Nvecs, pta.Ts, pta.sigmas), dtype=np.float64)
        toas = [q.toas for q in pta.psrs]
        res = [q.residuals for q in pta.psrs]
        tt, cond = truth.fp_sweep_truth(freqs, toas, res, pta.Nvecs, pta.Ts, pta.sigmas)
        return fps, tt.sum(0).astype(np.float64), tt.astype(np.float64), cond

    # ---- fp_white: config C1 (10 psr x 1000 TOAs, T = timing model only) ---------------
    pta = synth.make_config("C1")
    freqs = np.concatenate((synth.fp_freqs(1), np.linspace(2e-9, 3e-7, 7)))
    fps, tr, trp, cond = run_fp(pta, freqs)
    # one get_xCy golden per pulsar on generic vectors
    rng = np.random.default_rng(7)
    xs = [rng.standard_normal(q.toas.size) for q in pta.psrs]
    ys = [rng.standard_normal(q.toas.size) for q in pta.psrs]
    xcy = np.array(
        [float(ref_utils.get_xCy(pta.Nvecs[p], pta.Ts[p], pta.sigmas[p], xs[p], ys[p])) for p in range(pta.P)]
    )
    d = pack_inputs(pta)
    d.update(freqs=freqs, ref_fp=fps, truth_fp=tr, truth_terms=trp, cond=cond, ref_xcy=xcy)
    for p in range(pta.P):
        d[f"x_{p}"], d[f"y_{p}"] = xs[p], ys[p]
    np.savez_compressed(os.path.join(HERE, "fp_white.npz"), **d)
    print("fp_white", fps[:3], np.abs(fps - tr).max() / np.abs(tr).max())

    # ---- fp_red: ragged red+white Woodbury case ----------------------------------------
    pta = synth.make_pta(3, [250, 300, 347], n_tm=[8, 12, 15], ncomps=30, seed=synth.SEED0 + 1000)
    k = np.array([1, 2, 5, 30])
    freqs = np.concatenate((np.linspace(2e-9, 3e-7, 16), k / pta.Tspan, (k + 1e-3) / pta.Tspan))
    fps, tr, trp, cond = run_fp(pta, freqs)
    d = pack_inputs(pta)
    d.update(freqs=freqs, ref_fp=fps, truth_fp=tr, truth_terms=trp, cond=cond)
    np.savez_compressed(os.path.join(HERE, "fp_red.npz"), **d)
    print("fp_red", fps[:3], (np.abs(fps - tr) / np.abs(tr)).max())

    # ---- nmfp: containers + _get_sigmas + calculate_nmfp under the double vmap ---------
    P, D, F = 3, 4, 6
    pta = synth.make_pta(P, [260, 300, 333], n_tm=[9, 12, 14], ncomps=30, seed=synth.SEED0 + 2000)
    Ff_rn = np.asarray(pta.Ffreqs).view(ShimArray)
    ngwb = 5
    Ff_curn = np.repeat(np.arange(1, ngwb + 1) / pta.Tspan, 2).view(ShimArray)
    curn = ref_nmfp.CURN_container(Ff_curn)
    rn_objs = [ref_nmfp.RN_container(q, Ffreqs=Ff_rn, add_curn=True, curn_container=curn) for q in pta.psrs]
    rn_plain = [ref_nmfp.RN_container(q, Ffreqs=Ff_rn) for q in pta.psrs]
    samples = synth.draw_samples(pta, D)
    freqs = synth.nmfp_freqs(F, pta.Tspan)
    nm = ref_nmfp.NMFP(pta.psrs, rn_objs)
    vmap_f = jax.vmap(nm, in_axes=(0, None, None, None, None))  # examples/run_nmfp.py:265
    vmap_g = jax.vmap(vmap_f, in_axes=(None, 0, None, None, None))  # :266
    vals = np.asarray(vmap_g(freqs, samples, pta.Nvecs, pta.Ts, pta.TNTs), dtype=np.float64)
    nm2 = ref_nmfp.NMFP(pta.psrs, rn_plain)
    vals_plain = np.asarray(
        jax.vmap(jax.vmap(nm2, in_axes=(0, None, None, None, None)), in_axes=(None, 0, None, None, None))(
            freqs, samples, pta.Nvecs, pta.Ts, pta.TNTs
        ),
        dtype=np.float64,
    )
    pars0 = {k_: v[0] for k_, v in samples.items()}
    phiinv0 = [np.asarray(o.get_phiinv(pars0), dtype=np.float64) for o in rn_objs]
    phi0_plain = [np.asarray(o.update_phi(pars0), dtype=np.float64) for o in rn_plain]
    curn_phi0 = np.asarray(curn.get_phi_curn(pars0), dtype=np.float64)
    sig0 = [np.asarray(s, dtype=np.float64) for s in nm._get_sigmas(pars0, pta.TNTs)]
    # GP-ECORR layouts: the hot path only needs phi (the T columns are the caller's business)
    q0 = pta.psrs[0]
    q0.backend_flags = np.array(["A"] * 100 + ["B"] * (q0.toas.size - 100))
    weights = [np.ones(11).view(ShimArray), np.ones(17).view(ShimArray)]
    wn = {f"{q0.name}_basis_ecorr_A_log10_ecorr": -6.3, f"{q0.name}_basis_ecorr_B_log10_ecorr": -7.1}
    ec = ref_nmfp.GPEcorr_container(q0, weights, fix_wn_vals=wn)
    rn_ec = ref_nmfp.RN_container(q0, Ffreqs=Ff_rn, gp_ecorr=True, ecorr_container=ec)
    rn_ec_cu = ref_nmfp.RN_container(
        q0, Ffreqs=Ff_rn, gp_ecorr=True, ecorr_container=ec, add_curn=True, curn_container=curn
    )
    # truth for the nmfp grid
    toas = [q.toas for q in pta.psrs]
    res = [q.residuals for q in pta.psrs]
    tr = np.empty((D, F))
    cond = np.empty((D, F))
    for dd in range(D):
        pars = {k_: v[dd] for k_, v in samples.items()}
        sig = [np.asarray(s, dtype=np.float64) for s in nm._get_sigmas(pars, pta.TNTs)]
        tt, cc = truth.fp_sweep_truth(freqs, toas, res, pta.Nvecs, pta.Ts, sig)
        tr[dd], cond[dd] = tt.sum(0).astype(np.float64), cc.sum(0)
    d = pack_inputs(pta)
    d.update(
        freqs=freqs,
        D=D,
        ngwb=ngwb,
        Ffreqs=np.asarray(pta.Ffreqs),
        Ffreqs_curn=np.asarray(Ff_curn),
        ref_nmfp_curn=vals,
        ref_nmfp_plain=vals_plain,
        truth_nmfp_curn=tr,
        cond_curn=cond,
        ref_phiinv0=np.concatenate(phiinv0),
        ref_phi0_plain=np.concatenate(phi0_plain),
        ref_curn_phi0=curn_phi0,
        ref_ecorr_phi=np.asarray(ec.get_phi(pars0), dtype=np.float64),
        ref_phi_tm_ecorr_rn=np.asarray(rn_ec.update_phi(pars0), dtype=np.float64),
        ref_phi_tm_ecorr_rn_curn=np.asarray(rn_ec_cu.update_phi(pars0), dtype=np.float64),
        ecorr_log10=np.array([-6.3, -7.1]),
        ecorr_nw=np.array([11, 17]),
    )
    for p in range(P):
        d[f"ref_sigma0_{p}"] = sig0[p]
    for k_, v in samples.items():
        d["sample__" + k_] = v
    np.savez_compressed(os.path.join(HERE, "nmfp.npz"), **d)
    print("nmfp", vals[0, :3], (np.abs(vals - tr) / np.abs(tr)).max())


if __name__ == "__main__":
    main()
