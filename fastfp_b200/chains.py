"""MCMC-chain plumbing of the noise-marginalised driver (reference ``examples/run_nmfp.py``).

The reference script reads a PTMCMC text chain (one row per step; the trailing four columns are
sampler bookkeeping, ``run_nmfp.py:254``), discards the first quarter as burn-in (``:221``), picks
``nsamples`` distinct rows at random (``:253``) and turns the ``(n_params, nsamples)`` block into the
``{parameter name: (nsamples,) array}`` dict that ``NMFP`` consumes (``map_params``, ``:174-186``).
These helpers do the same on plain NumPy arrays; parameter names are passed in explicitly (the
reference takes them from ``pta.params``), so no ``enterprise`` object is needed.
"""
from __future__ import annotations

from typing import Dict, Sequence, Tuple

import numpy as np

N_META_COLUMNS = 4  # lnpost, lnlike, acceptance rate, PT swap rate


def map_params(param_names: Sequence[str], xs) -> Dict[str, np.ndarray]:
    """``xs`` of shape ``(n_params,)`` -> ``{name: scalar}``; ``(n_params, D)`` -> ``{name: (D,)}``
    (row ``i`` belongs to ``param_names[i]``; reference ``run_nmfp.py:174-186``)."""
    xs = np.asarray(xs, dtype=np.float64)
    if xs.shape[0] != len(param_names):
        raise ValueError(f"{xs.shape[0]} parameter rows for {len(param_names)} names")
    if xs.ndim > 2:
        raise ValueError("xs must be (n_params,) or (n_params, D)")
    return {name: xs[i] for i, name in enumerate(param_names)}


def draws_from_chain(chain, param_names: Sequence[str], nsamples: int, burn_frac: float = 0.25, rng=None,
                     n_meta: int = N_META_COLUMNS) -> Tuple[Dict[str, np.ndarray], np.ndarray]:
    """``nsamples`` distinct post-burn-in rows of ``chain`` (array or path of a text chain) as the
    ``samples`` dict, plus the chosen row indices."""
    if isinstance(chain, (str, bytes)) or hasattr(chain, "__fspath__"):
        chain = np.loadtxt(chain)
    chain = np.atleast_2d(np.asarray(chain, dtype=np.float64))
    npar = chain.shape[1] - n_meta
    if npar != len(param_names):
        raise ValueError(f"chain has {npar} parameter columns, {len(param_names)} names given")
    burn = int(burn_frac * chain.shape[0])
    if nsamples > chain.shape[0] - burn:
        raise ValueError(f"asked for {nsamples} draws, the chain holds {chain.shape[0] - burn} after burn-in")
    rng = np.random.default_rng() if rng is None else rng
    idxs = rng.choice(np.arange(burn, chain.shape[0]), nsamples, replace=False)
    block = chain[idxs, :npar].T  # (n_params, nsamples), the layout of rns_full (run_nmfp.py:252-254)
    return map_params(param_names, block), idxs


def draw_batches(samples: Dict[str, np.ndarray], batch_size: int):
    """The draw-batch loop of the reference (``run_nmfp.py:256-270``) as a generator of sub-dicts; the
    engine batches draws internally, so this is only needed to bound the ``(D, F)`` output."""
    D = len(next(iter(samples.values())))
    for start in range(0, D, batch_size):
        yield {k: v[start:start + batch_size] for k, v in samples.items()}


def write_chain(path, samples: Dict[str, np.ndarray], param_names: Sequence[str]) -> None:
    """A text chain in the layout above from a samples dict (synthetic runs and tests)."""
    cols = np.stack([np.asarray(samples[n], dtype=np.float64) for n in param_names], axis=1)
    meta = np.zeros((cols.shape[0], N_META_COLUMNS))
    np.savetxt(path, np.hstack([cols, meta]))
