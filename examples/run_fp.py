# -*- coding: utf-8 -*-
"""Fp-statistic frequency scan with the fastfp_b200 engine: the counterpart of the reference's
``examples/run_fp.py`` (same flow, same output file: a JSON dictionary ``{frequency: Fp}``).

Two ways to get the inputs:
  * ``--synthetic P N``: seeded synthetic pulsars (no ``enterprise`` needed);
  * ``psrfile noisefile``: a pickle of ``enterprise`` pulsars and a noise JSON, exactly as the
    reference script takes them -- model construction goes through ``fastfp_b200.utils.initialize_pta``
    (a pass-through to ``enterprise``, which must be installed); ``FastFp``, ``get_mats_fp`` and ``vmap``
    come from ``fastfp_b200``.
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
from fastfp_b200 import FastFp, get_mats_fp, vmap  # noqa: E402


def main(psrfile=None, noisefile=None, savefile="fp_out", synthetic=None, nfreqs=200):
    logging.basicConfig(format="%(levelname)s: %(message)s", level=logging.INFO)
    logger = logging.getLogger(__name__)
    if synthetic:
        from fastfp_b200 import synth

        pta = synth.make_pta(synthetic[0], synthetic[1])
        psrs, noise = pta.psrs, pta.noise
    else:
        from fastfp_b200.utils import initialize_pta  # pass-through to enterprise (must be installed)

        with open(psrfile, "rb") as f:
            psrs = pickle.load(f)
        with open(noisefile, "rb") as f:
            noise = json.load(f)
        noise["gw_gamma"] = 13 / 3
        noise["gw_log10_A"] = np.log10(2e-15)
        pta = initialize_pta(psrs, noise, inc_cp=True, gwb_comps=30)

    t_start = time.perf_counter()
    Nvecs, Ts, sigmas = get_mats_fp(pta, noise)
    logger.info("Precompute matrix wall time: {0:.4f} s".format(time.perf_counter() - t_start))

    Fp_obj = FastFp(psrs, pta)
    freqs = np.linspace(2e-9, 3e-7, nfreqs)

    t_start = time.perf_counter()
    fn = vmap(Fp_obj.calculate_Fp, in_axes=(0, None, None, None))  # one kernel launch for the grid
    fps = fn(freqs, Nvecs, Ts, sigmas)
    logger.info("Fp-statistic wall time (incl. one-time packing): {0:.4f} s".format(time.perf_counter() - t_start))

    res = {freq: float(fp) for freq, fp in zip(freqs, fps)}
    with open("{}.json".format(savefile), "w") as f:
        json.dump(res, f)


if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument("psrfile", nargs="?", type=str, help="filename for pulsars pickle object")
    parser.add_argument("noisefile", nargs="?", type=str, help="filename for noise dictionary")
    parser.add_argument("savefile", nargs="?", default="fp_out", type=str, help="filename for resulting Fp dictionary")
    parser.add_argument("--synthetic", nargs=2, type=int, metavar=("P", "NTOA"), help="use synthetic pulsars")
    parser.add_argument("--nfreqs", type=int, default=200)
    parser.add_argument("--save", type=str, default=None, help="output name (alternative to the positional savefile)")
    kwargs = vars(parser.parse_args())
    save = kwargs.pop("save")
    if save:
        kwargs["savefile"] = save
    if not kwargs["synthetic"] and not (kwargs["psrfile"] and kwargs["noisefile"]):
        parser.error("give psrfile noisefile [savefile], or --synthetic P NTOA")
    main(**kwargs)
