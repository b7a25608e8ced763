# -*- coding: utf-8 -*-
"""Noise-marginalised Fp with the fastfp_b200 engine: the counterpart of the reference's ``examples/run_nmfp.py``
(same flow and flags; output ``res/<savefile>.npy`` holding the ``(nsamples, ncwfreqs)`` array, draw-major).

Two ways to get the inputs:
  * ``psrfile noisefile chainfile savefile`` -- a pickle of ``enterprise`` pulsars, a noise JSON and a PTMCMC text
    chain, exactly as the reference script takes them; the PTA is then built by ``fastfp_b200.utils.initialize_pta``
    (a pass-through to ``enterprise``, which must be installed) and everything after it runs on the GPU;
  * ``--synthetic P NTOA`` -- seeded synthetic pulsars and a stand-in chain written in the PTMCMC layout
    (no ``enterprise`` needed).
``--inc_ecorr`` models ECORR as a Gaussian process on the epoch basis like the reference (``GPEcorr_container``);
``--kernel_ecorr`` (synthetic runs) uses the block-diagonal ``N`` instead -- the reference's to-do
(``fastfp/utils.py:29-31``) -- and gives the same statistic with a basis that stays 72 columns wide.
All draws go to the GPU in one call; ``--batch_size`` reproduces the reference's host loop over draw batches
(``run_nmfp.py:256-270``), which here only bounds the size of the host-side output.
"""
import argparse
import json
import logging
import os
import pickle
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fastfp_b200 import chains, get_mats_nmfp, model, vmap  # noqa: E402


def main(psrfile=None, noisefile=None, chainfile=None, savefile="nmfp_out", synthetic=None, inc_ecorr=False,
         kernel_ecorr=False, inc_cp=False, nrncomps=30, ngwbcomps=30, ncwfreqs=100, nsamples=1000, batch_size=None,
         seed=None, outdir="res"):
    logging.basicConfig(format="%(levelname)s: %(message)s", level=logging.INFO)
    logger = logging.getLogger(__name__)
    logger.info(f"number of CW frequencies: {ncwfreqs}")
    logger.info(f"number of samples: {nsamples}")
    logger.info(f"batch_size: {batch_size}")
    os.makedirs(outdir, exist_ok=True)
    rng = np.random.default_rng(seed)

    if synthetic:
        from fastfp_b200 import synth

        ecorr = inc_ecorr or kernel_ecorr
        pta = synth.make_pta(synthetic[0], synthetic[1], ncomps=nrncomps, inc_cp=inc_cp, epoch=4 if ecorr else 0)
        psrs, noise, Tspan = pta.psrs, pta.noise, pta.Tspan
        t_start = time.perf_counter()
        if ecorr:
            Nvecs, Ts, TNTs, _ = synth.with_ecorr(pta, kernel=kernel_ecorr)
        else:
            TNTs, Nvecs, Ts = get_mats_nmfp(pta, noise)
        names = model.param_names(psrs, inc_cp)
        if chainfile is None:  # stand-in MCMC chain, written in the PTMCMC text layout and read back
            chainfile = os.path.join(outdir, f"{savefile}_chain_1.txt")
            chains.write_chain(chainfile, synth.draw_samples(pta, max(2 * nsamples, 8)), names)
    else:
        from fastfp_b200.utils import initialize_pta  # pass-through to enterprise (must be installed)

        if kernel_ecorr:
            raise SystemExit("--kernel_ecorr needs a PTA built with EcorrKernelNoise; with enterprise data use --inc_ecorr")
        with open(psrfile, "rb") as f:
            psrs = pickle.load(f)
        with open(noisefile, "r") as f:
            noise = json.load(f)
        # the CURN keys must exist in the noise dictionary; their values come from the chain (run_nmfp.py:224-230)
        noise["gw_gamma"] = 13 / 3
        noise["gw_log10_A"] = np.log10(2e-15)
        Tspan = model.get_tspan(psrs)
        pta = initialize_pta(psrs, noise, inc_cp=inc_cp, rn_comps=nrncomps, gwb_comps=ngwbcomps, inc_ecorr=inc_ecorr)
        t_start = time.perf_counter()
        TNTs, Nvecs, Ts = get_mats_nmfp(pta, noise)
        names = [p.name for p in pta.params]
    logger.info(f"Precompute matrix wall time: {time.perf_counter() - t_start:.2f} s")

    nmfp = model.setup_fp_model(psrs, noise, Tspan=Tspan, add_ecorr=inc_ecorr and not kernel_ecorr, add_curn=inc_cp,
                                nrncomps=nrncomps, ngwbcomps=ngwbcomps)
    freqs = np.arange(1, ncwfreqs + 1) / Tspan  # CW grid = red-noise Fourier grid (run_nmfp.py:247)
    samples, rows = chains.draws_from_chain(chainfile, names, nsamples, rng=rng)  # 25 % burn-in, distinct rows

    t_start = time.perf_counter()
    vmap_f = vmap(nmfp, in_axes=(0, None, None, None, None))
    vmap_g = vmap(vmap_f, in_axes=(None, 0, None, None, None))
    if batch_size:
        nmfp_vals = np.vstack([np.asarray(vmap_g(freqs, part, Nvecs, Ts, TNTs))
                               for part in chains.draw_batches(samples, batch_size)])
    else:
        nmfp_vals = np.asarray(vmap_g(freqs, samples, Nvecs, Ts, TNTs))
    logger.info(f"Noise marginalized Fp-statistic wall time: {time.perf_counter() - t_start:.2f} s")

    with open(os.path.join(outdir, f"{savefile}.npy"), "wb") as f:
        np.save(f, nmfp_vals)
    np.save(os.path.join(outdir, f"{savefile}_rows.npy"), rows)  # which chain rows were drawn (reproducibility)
    return nmfp_vals


if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument("psrfile", nargs="?", type=str, help="filepath for pulsars pickle object")
    parser.add_argument("noisefile", nargs="?", type=str, help="filepath for noise dictionary")
    parser.add_argument("chainfile", nargs="?", type=str, help="filepath for MCMC chain (PTMCMC text; last 4 columns = sampler metadata)")
    parser.add_argument("savefile", nargs="?", type=str, default="nmfp_out", help="name of the output Fp values array")
    parser.add_argument("--synthetic", nargs=2, type=int, metavar=("P", "NTOA"), help="use seeded synthetic pulsars")
    parser.add_argument("--save", type=str, default=None, help="output name (alternative to the positional savefile)")
    parser.add_argument("--inc_ecorr", action="store_true", help="include ECORR (Gaussian process on the epoch basis)")
    parser.add_argument("--kernel_ecorr", action="store_true", help="ECORR as a block-diagonal N (synthetic runs)")
    parser.add_argument("--inc_cp", action="store_true", help="include CURN process")
    parser.add_argument("--nrncomps", type=int, default=30, help="number of intrinsic red noise components")
    parser.add_argument("--ngwbcomps", type=int, default=30, help="number of CURN components")
    parser.add_argument("--ncwfreqs", type=int, default=100, help="number of CW frequencies to calculate at")
    parser.add_argument("--nsamples", type=int, default=1000, help="number of red noise draws from the MCMC chain")
    parser.add_argument("--batch_size", type=int, default=None, help="draws per call (host-side output batches)")
    parser.add_argument("--seed", type=int, default=None, help="seed of the row selection (the reference's is unseeded)")
    parser.add_argument("--outdir", type=str, default="res")
    kwargs = vars(parser.parse_args())
    save = kwargs.pop("save")
    if save:
        kwargs["savefile"] = save
    if not kwargs["synthetic"] and not (kwargs["psrfile"] and kwargs["noisefile"] and kwargs["chainfile"]):
        parser.error("give psrfile noisefile chainfile [savefile], or --synthetic P NTOA")
    main(**kwargs)
