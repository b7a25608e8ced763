"""Noise-marginalised Fp -- drop-in for the reference's ``fastfp/nmfp.py``.

``NMFP``, ``RN_container``, ``CURN_container`` and ``GPEcorr_container`` keep the reference's
constructor and method signatures (``fastfp/nmfp.py:45, 161-170, 355, 434``). The containers are
small host-side objects (NumPy float64) describing how the prior variances ``phi`` depend on the
noise parameters; the hot path -- ``NMFP.calculate_nmfp`` over a batch of frequencies and a batch
of draws -- runs on the GPU through the C ABI:

* ``phi`` of the per-draw block (the power laws of ``nmfp.py:226-234`` and the CURN add of
  ``:247/275``) is evaluated by a device kernel for all draws at once (``fastfp_powerlaw_phiinv``);
* ``Sigma = TNT + diag(phiinv)`` (``nmfp.py:58-74``) is never materialised per draw: the
  draw-independent columns (timing model ``1e40``, fixed GP-ECORR) are eliminated once per pulsar and
  only the ``2*ncomps``-square per-draw system is factorised per (pulsar, draw) (DESIGN.md §5).

Batching: ``fgw`` may be a scalar or ``(F,)``; the values of ``samples`` may be scalars or ``(D,)``
arrays (what ``map_params`` builds, ``examples/run_nmfp.py:174-186``). Both batched gives
``(D, F)``, draw-major, as the reference's nested ``vmap`` (``run_nmfp.py:265-270``).
"""
from __future__ import annotations

import numpy as np

from . import constants as const
from ._cabi import _is_cuda_tensor
from .fastfp import _PackCache


def _powerlaw(Ffreqs, log10_A, gamma):
    """Power-law PSD (reference ``nmfp.py:226-234`` / ``:373-381``), same operation order.
    ``log10_A`` / ``gamma`` may be scalars or ``(D,)`` arrays (then the result is ``(D, m)``)."""
    Ffreqs = np.asarray(Ffreqs, dtype=np.float64)
    df = np.diff(np.concatenate((np.array([0.0]), Ffreqs[::2])))
    A, g = np.asarray(log10_A, dtype=np.float64), np.asarray(gamma, dtype=np.float64)
    if A.ndim or g.ndim:
        A, g = np.atleast_1d(A)[:, None], np.atleast_1d(g)[:, None]
    return Ffreqs ** (-g) * (10**A) ** 2 / 12.0 / np.pi**2 * const.fyr ** (g - 3) * np.repeat(df, 2)


def _cat(parts):
    """concatenate along the last axis, broadcasting unbatched parts against batched ones"""
    nb = max(np.ndim(p) for p in parts)
    if nb == 1:
        return np.concatenate(parts)
    D = max(p.shape[0] for p in parts if np.ndim(p) == 2)
    return np.concatenate([p if np.ndim(p) == 2 else np.broadcast_to(p, (D, p.shape[0])) for p in parts], axis=1)


class CURN_container(object):
    """Common uncorrelated red-noise process (reference ``nmfp.py:344-417``).

    :param Ffreqs: ``repeat(k / Tspan, 2)`` of the common process"""

    def __init__(self, Ffreqs):
        self.rn_A_name = "gw_log10_A"
        self.rn_gam_name = "gw_gamma"
        self.Ffreqs = np.asarray(Ffreqs, dtype=np.float64)
        self.phi_fn = self.get_phi_curn

    def _powerlaw(self, pars):
        return _powerlaw(self.Ffreqs, pars[self.rn_A_name], pars[self.rn_gam_name])

    def get_phi_curn(self, pars):
        return self._powerlaw(pars)

    def update_phi(self, pars):
        return self.phi_fn(pars)

    def get_phiinv(self, pars):
        return 1.0 / self.update_phi(pars)

    def tree_flatten(self):
        return (self.Ffreqs,), ()

    @classmethod
    def tree_unflatten(cls, aux_data, children):
        return cls(*aux_data, *children)


class GPEcorr_container(object):
    """Fixed ECORR modelled as a Gaussian process (reference ``nmfp.py:420-477``): per backend
    ``weights_i * 10**(2*log10_ecorr_i)``, looked up as
    ``"{psr}_basis_ecorr_{backend}_log10_ecorr"`` in ``fix_wn_vals`` (``:447-450``)."""

    def __init__(self, psr, weights, fix_wn_vals=None):
        self.psr = psr
        self.weights = weights
        self.fix_wn_vals = fix_wn_vals
        self._select_by_backend(psr, fix_wn_vals)
        self._init_phi()

    def _select_by_backend(self, psr, fix_wn_vals):
        backends = np.unique(psr.backend_flags)
        self.ecorrs = np.array(
            [fix_wn_vals["_".join([psr.name, "basis", "ecorr", val, "log10_ecorr"])] for val in backends],
            dtype=np.float64,
        )

    def _init_phi(self):
        self._phi = np.concatenate(
            [np.asarray(self.weights[i], dtype=np.float64) * 10 ** (2 * ecorr) for i, ecorr in enumerate(self.ecorrs)]
        )
        self._get_phi = self.get_phi

    def get_phi(self, pars):
        return self._phi

    def tree_flatten(self):
        return (), (self.psr, self.weights, self.fix_wn_vals)

    @classmethod
    def tree_unflatten(cls, aux_data, children):
        return cls(*aux_data, *children)


class RN_container(object):
    """Per-pulsar red-noise prior (reference ``nmfp.py:131-341``); the eight ``get_phi_*`` layouts of
    ``:239-292`` and the selector of ``:188-199`` are kept. The column order must match the basis
    ``T``: timing model, (basis ECORR), Fourier."""

    def __init__(self, psr, Ffreqs=None, ncomps=30, gp_ecorr=False, ecorr_container=None, add_curn=False,
                 curn_container=None):
        self.psr = psr
        self.ncomps = ncomps
        self.gp_ecorr = gp_ecorr
        self.ecorr_container = ecorr_container
        self.add_curn = add_curn
        self.curn_container = curn_container
        self.rn_A_name = f"{psr.name}_red_noise_log10_A"
        self.rn_gam_name = f"{psr.name}_red_noise_gamma"
        # the reference keeps a supplied array and otherwise derives the grid from the pulsar's span
        self.Ffreqs = np.asarray(Ffreqs, dtype=np.float64) if Ffreqs is not None else self._create_freqarray(psr, ncomps)
        self.tm_weights = np.ones(psr.Mmat.shape[1])
        if add_curn:
            self.phi_fn = self.get_phi_tm_ecorr_rn_curn if gp_ecorr else self.get_phi_tm_rn_curn
        else:
            self.phi_fn = self.get_phi_tm_ecorr_rn if gp_ecorr else self.get_phi_tm_rn

    def _create_freqarray(self, psr, ncomps=30):
        Tspan = np.max(psr.toas) - np.min(psr.toas)
        return np.repeat(1.0 * np.arange(1, ncomps + 1) / Tspan, 2)

    def _powerlaw(self, pars):
        return _powerlaw(self.Ffreqs, pars[self.rn_A_name], pars[self.rn_gam_name])

    def _rn_curn(self, pars):
        rn_phi = np.array(self._powerlaw(pars), copy=True)
        curn_phi = self.curn_container.get_phi_curn(pars)
        rn_phi[..., : curn_phi.shape[-1]] += curn_phi
        return rn_phi

    # the eight layouts (reference nmfp.py:239-292)
    def get_phi_rn(self, pars):
        return self._powerlaw(pars)

    def get_phi_rn_curn(self, pars):
        return self._rn_curn(pars)

    def get_phi_ecorr_rn(self, pars):
        return _cat((self.ecorr_container.get_phi(pars), self._powerlaw(pars)))

    def get_phi_ecorr_rn_curn(self, pars):
        return _cat((self.ecorr_container.get_phi(pars), self._rn_curn(pars)))

    def get_phi_tm_rn(self, pars):
        return _cat((self.tm_weights * 1e40, self._powerlaw(pars)))

    def get_phi_tm_rn_curn(self, pars):
        return _cat((self.tm_weights * 1e40, self._rn_curn(pars)))

    def get_phi_tm_ecorr_rn(self, pars):
        return _cat((self.tm_weights * 1e40, self.ecorr_container.get_phi(pars), self._powerlaw(pars)))

    def get_phi_tm_ecorr_rn_curn(self, pars):
        return _cat((self.tm_weights * 1e40, self.ecorr_container.get_phi(pars), self._rn_curn(pars)))

    def update_phi(self, pars):
        return self.phi_fn(pars)

    def get_phiinv(self, pars):
        return 1.0 / self.update_phi(pars)

    # what the device path needs: the draw-independent leading block and the size of the rest
    def fixed_phi(self):
        parts = [self.tm_weights * 1e40]
        if self.gp_ecorr:
            parts.append(np.asarray(self.ecorr_container.get_phi({}), dtype=np.float64))
        return np.concatenate(parts)

    def tree_flatten(self):
        return (self.Ffreqs,), (self.psr, self.ncomps, self.gp_ecorr, self.ecorr_container, self.add_curn,
                                self.curn_container)

    @classmethod
    def tree_unflatten(cls, aux_data, children):
        psr, ncomps, gp_ecorr, ecorr_container, add_curn, curn_container = aux_data
        (Ffreqs,) = children
        return cls(psr, Ffreqs, ncomps, gp_ecorr, ecorr_container, add_curn, curn_container)


class NMFP(_PackCache):
    """Noise-marginalised Fp-statistic (reference ``nmfp.py:22-128``).

    :param psrs: objects with ``.toas`` / ``.residuals`` (``nmfp.py:50-51``)
    :param rn_sigs: one :class:`RN_container` per pulsar
    :param device: CUDA device ordinal (extension; default ``LOCAL_RANK`` or 0)
    :param path: kernel of the draw-independent stage A, like :class:`FastFp`'s ``path`` (``"auto"`` / ``"fp64"`` /
        ``"i8"`` / ``"prefer-i8"``; default from ``FASTFP_B200_PATH``)"""

    def __init__(self, psrs, rn_sigs, device=None, path=None):
        self.psrs = psrs
        self.rn_sigs = rn_sigs
        super().__init__(psrs, device, path)

    def __call__(self, fgw, samples, Nvecs, Ts, TNTs):
        return self.calculate_nmfp(fgw, samples, Nvecs, Ts, TNTs)

    def _get_sigmas(self, pars, TNTs):
        """``Sigma = TNT + diag(phiinv)`` per pulsar (reference ``nmfp.py:57-74``), host arrays.
        (API parity; the device path never forms these per draw.)"""
        sigmas = []
        for rn_sig, TNT in zip(self.rn_sigs, TNTs):
            phiinv = rn_sig.get_phiinv(pars)
            sigmas.append(np.asarray(TNT, dtype=np.float64) + np.diag(phiinv))
        return sigmas

    def prepare(self, Nvecs, Ts, TNTs, force=False):
        """Cached like :meth:`FastFp.prepare`: keyed on a hash of every byte of the three lists."""
        return self._ensure((Nvecs, Ts, TNTs), force=force)

    def _build_pack(self, lists):
        Nvecs, Ts, TNTs = lists
        fixed = [sig.fixed_phi() for sig in self.rn_sigs]
        m_fix = [f.shape[0] for f in fixed]
        for p, (sig, T) in enumerate(zip(self.rn_sigs, Ts)):
            if m_fix[p] + sig.Ffreqs.shape[0] != np.shape(T)[1]:
                raise ValueError(
                    f"pulsar {p}: basis has {np.shape(T)[1]} columns but the RN_container describes "
                    f"{m_fix[p]} fixed + {sig.Ffreqs.shape[0]} red-noise entries"
                )
        return self._create_pack(Nvecs, Ts, TNTs, m_fix, [1.0 / f for f in fixed])

    def _curn_setup(self):
        flags = {bool(sig.add_curn) for sig in self.rn_sigs}
        if flags == {False}:
            return None
        if flags != {True}:
            raise ValueError("either every RN_container carries the common process or none does")
        c0 = self.rn_sigs[0].curn_container
        for sig in self.rn_sigs[1:]:
            c = sig.curn_container
            if c is not c0 and not (c.rn_A_name == c0.rn_A_name and c.rn_gam_name == c0.rn_gam_name
                                    and np.array_equal(c.Ffreqs, c0.Ffreqs)):
                raise ValueError("the common process must be the same CURN_container for every pulsar")
        return c0

    def _draw_arrays(self, samples):
        """The sample dictionary of the reference (``nmfp.py:82-92``) as ``(D, P)`` arrays of the red-noise
        parameters, the common-process ones as ``(D,)`` (or None), the draw count and whether a draw axis was given."""
        P = len(self.rn_sigs)
        curn = self._curn_setup()
        names = [(s.rn_A_name, s.rn_gam_name) for s in self.rn_sigs]
        vals = [np.asarray(samples[k], dtype=np.float64) for pair in names for k in pair]
        if curn is not None:
            vals += [np.asarray(samples[curn.rn_A_name], dtype=np.float64),
                     np.asarray(samples[curn.rn_gam_name], dtype=np.float64)]
        batched = any(v.ndim > 0 for v in vals)
        D = max([v.shape[0] for v in vals if v.ndim > 0], default=1)
        col = lambda v: np.broadcast_to(v, (D,)) if v.ndim == 0 else v
        A = np.stack([col(vals[2 * p]) for p in range(P)], axis=1)       # (D, P)
        G = np.stack([col(vals[2 * p + 1]) for p in range(P)], axis=1)   # (D, P)
        cA = col(vals[2 * P]) if curn is not None else None
        cG = col(vals[2 * P + 1]) if curn is not None else None
        return curn, A, G, cA, cG, D, batched

    def calculate_nmfp_2d(self, fgw, samples, Nvecs, Ts, TNTs, group=None):
        """``calculate_nmfp`` for THIS rank's draws when the draws are sharded over the ranks of ``group`` (one process
        per GPU): the stage that depends on the frequency but not on the draw (``nmfp.py:103-113``) is computed for a
        slice of the frequency grid per rank and exchanged with one all-gather, instead of being repeated on every
        rank; the per-draw factorisation and contraction then run locally for all frequencies. ``fgw``: 1-D float64
        CUDA tensor (the same on every rank); returns this rank's ``(D_local, F)`` tensor, bit-identical to
        ``calculate_nmfp`` (tiles are computed independently of how they are grouped)."""
        import torch
        import torch.distributed as dist

        from . import parallel

        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            out = self.calculate_nmfp(fgw, samples, Nvecs, Ts, TNTs)
            return out if out.dim() == 2 else out[None]
        if not _is_cuda_tensor(fgw) or fgw.dtype != torch.float64 or fgw.dim() != 1 or fgw.device.index != self.device:
            raise TypeError("calculate_nmfp_2d needs a 1-D float64 CUDA tensor of frequencies on the pack's device")
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        curn, A, G, cA, cG, D, _ = self._draw_arrays(samples)
        dev = torch.device("cuda", self.device)
        stream = torch.cuda.current_stream(dev).cuda_stream
        f = fgw.contiguous()
        F = int(f.shape[0])
        nt, per = parallel.tile_blocks(F, world)
        out = torch.empty((D, F), dtype=torch.float64, device=dev)

        def run(pack):
            zt, at = pack.nmfp_tile_sizes()
            # this rank's tiles: frequencies [32 * rank * per, 32 * (rank + 1) * per), the tail repeated (padding tiles
            # are computed like any other and never read)
            idx = torch.arange(32 * rank * per, 32 * (rank + 1) * per, device=dev).clamp_(max=F - 1)
            floc = f[idx].contiguous()
            zloc = torch.empty(per * zt, dtype=torch.float64, device=dev)
            aloc = torch.empty(per * at, dtype=torch.float64, device=dev)
            pack.nmfp_stage_a(floc.data_ptr(), 32 * per, zloc.data_ptr(), aloc.data_ptr(), stream=stream)
            zall = torch.empty(world * per * zt, dtype=torch.float64, device=dev)
            aall = torch.empty(world * per * at, dtype=torch.float64, device=dev)
            dist.all_gather_into_tensor(zall, zloc, group=group)
            dist.all_gather_into_tensor(aall, aloc, group=group)
            if D == 0:  # more ranks than draws: this rank only contributes its stage-A tiles
                return out
            phiinv = torch.empty((D, pack.mvar_total), dtype=torch.float64, device=dev)
            pack.powerlaw_phiinv([s.Ffreqs for s in self.rn_sigs], A, G, None if curn is None else curn.Ffreqs,
                                 cA, cG, phiinv.data_ptr(), stream=stream)
            pack.nmfp_stage_b(f.data_ptr(), F, zall.data_ptr(), aall.data_ptr(), per, phiinv.data_ptr(), D,
                              out.data_ptr(), stream=stream)
            return out

        return self._run_verified((Nvecs, Ts, TNTs), run, asynchronous=True)

    def calculate_nmfp(self, fgw, samples, Nvecs, Ts, TNTs):
        """Fp at ``fgw`` for the noise parameters ``samples`` (reference ``nmfp.py:76-119``)."""
        import torch

        lists = (Nvecs, Ts, TNTs)
        curn, A, G, cA, cG, D, batched = self._draw_arrays(samples)

        dev = torch.device("cuda", self.device)
        on_dev = _is_cuda_tensor(fgw)
        if on_dev:
            f, stream = self._device_freqs(fgw)
            out = torch.empty((D, f.shape[0]), dtype=torch.float64, device=dev)
        else:
            f = np.asarray(fgw, dtype=np.float64)
            stream = torch.cuda.current_stream(dev).cuda_stream

        def run(pack):
            phiinv = torch.empty((D, pack.mvar_total), dtype=torch.float64, device=dev)
            pack.powerlaw_phiinv([s.Ffreqs for s in self.rn_sigs], A, G, None if curn is None else curn.Ffreqs,
                                 cA, cG, phiinv.data_ptr(), stream=stream)
            if on_dev:
                pack.nmfp_sweep((f.data_ptr(), f.shape[0]), phiinv.data_ptr(), D, out=out.data_ptr(), stream=stream)
                return out
            return pack.nmfp_sweep(f.reshape(-1), phiinv.data_ptr(), D, stream=stream)  # (D, F) on the host

        res = self._run_verified(lists, run, asynchronous=on_dev)
        if on_dev:
            return res if batched else res[0]
        if f.ndim == 0:
            res = res[:, 0]
        if not batched:
            res = res[0]
        return np.float64(res) if np.ndim(res) == 0 else res

    def tree_flatten(self):
        return (), (self.psrs, self.rn_sigs)

    @classmethod
    def tree_unflatten(cls, aux_data, children):
        return cls(*aux_data, *children)
