"""``FastFe`` -- the Fe-statistic on the fastfp_b200 engine.

The reference lists the Fe-statistic as a to-do (``README.md:23``); ``enterprise_extensions.frequentist.FeStat`` is the
implementation users have today. Fe (Ellis, Siemens & Creighton 2012) is the coherent Earth-term counterpart of Fp: for
a sky position ``(gwtheta, gwphi)`` the four templates of pulsar ``p`` are ``[F+ s, F+ c, Fx s, Fx c]`` with the same
``s, c = sin, cos(((2 pi) f) t)`` as ``FastFp.calculate_Fp`` (``fastfp/fastfp.py:78-79``) and the antenna patterns
``F+_p, Fx_p``; the statistic is ``1/2 N^T M^-1 N`` with the 4-vector ``N`` and the 4x4 matrix ``M`` summed over
pulsars. Every entry is one of the five inner products the Fp sweep already forms per (pulsar, frequency), so a sky
scan costs one sweep plus a small combine kernel (``fastfp_fe_sweep``).
"""
from __future__ import annotations

import numpy as np

from .fastfp import FastFp


def antenna_pattern(pos, gwtheta, gwphi):
    """``(F+, Fx)`` of a pulsar at unit vector ``pos`` for a source at polar angle ``gwtheta`` and azimuth ``gwphi``
    (the convention of ``enterprise.signals.utils.create_gw_antenna_pattern``). ``gwtheta`` / ``gwphi`` may be
    arrays (broadcast); ``pos`` is ``(3,)`` or ``(P, 3)`` -> result ``(..., P)``."""
    pos = np.atleast_2d(np.asarray(pos, dtype=np.float64))
    th, ph = np.broadcast_arrays(np.asarray(gwtheta, dtype=np.float64), np.asarray(gwphi, dtype=np.float64))
    m = np.stack((np.sin(ph), -np.cos(ph), np.zeros_like(ph)), axis=-1)
    n = np.stack((-np.cos(th) * np.cos(ph), -np.cos(th) * np.sin(ph), np.sin(th)), axis=-1)
    om = np.stack((-np.sin(th) * np.cos(ph), -np.sin(th) * np.sin(ph), -np.cos(th)), axis=-1)
    mp, npos, op = m @ pos.T, n @ pos.T, om @ pos.T
    fplus = 0.5 * (mp ** 2 - npos ** 2) / (1.0 + op)
    fcross = mp * npos / (1.0 + op)
    return fplus, fcross


class FastFe(FastFp):
    """Fe-statistic for a list of pulsars; the pulsars additionally need ``.pos`` (unit vector, as
    ``enterprise.pulsar.Pulsar`` provides). Same packing and caching as :class:`FastFp`."""

    def __init__(self, psrs, pta=None, device=None, path=None):
        super().__init__(psrs, pta=pta, device=device, path=path)
        self.pos = np.stack([np.asarray(psr.pos, dtype=np.float64) for psr in psrs])

    def calculate_Fe(self, fgw, gwtheta, gwphi, Nvecs, Ts, sigmas):
        """Fe at frequency ``fgw`` (scalar or ``(F,)``, host array or CUDA tensor) and sky position(s)
        ``gwtheta``, ``gwphi`` (scalars or ``(S,)``): returns a scalar, ``(F,)``, ``(S,)`` or ``(S, F)``. A frequency
        ``f <= 0`` gives NaN, as in :meth:`calculate_Fp` (the reference's ``f^(-1/3)``)."""
        sky_batched = np.ndim(gwtheta) > 0 or np.ndim(gwphi) > 0
        fplus, fcross = self._sky_grid(gwtheta, gwphi)
        f, empty, stream, on_device = self._front_end(fgw)
        out = empty((fplus.shape[0], f.shape[0]))

        def run(pack):
            pack.fe_sweep(f, fplus, fcross, out=out, stream=stream)
            return out

        res = self._run_verified((Nvecs, Ts, sigmas), run, asynchronous=on_device)
        res = res if np.ndim(fgw) else res[:, 0]
        return res if sky_batched else res[0]

    compute_Fe = calculate_Fe

    def calculate_Fe_skymax(self, fgw, gwtheta, gwphi, Nvecs, Ts, sigmas):
        """The loudest position of the sky grid ``gwtheta``, ``gwphi`` (broadcast to ``(S,)``) at each frequency
        ``fgw``, without forming the ``(S, F)`` map of :meth:`calculate_Fe` (``fastfp_fe_skymax``). Returns
        ``(fe_max, sky_index)``: ``(float, int)`` for a scalar ``fgw``, ``float64`` and ``int64`` arrays of
        ``fgw``'s shape for an array, CUDA tensors on its device (enqueued on torch's current stream) for a float64
        CUDA tensor. Each value equals the corresponding entry of :meth:`calculate_Fe`'s map bit for bit; NaN loses,
        ties go to the lowest index, and a frequency with no finite value gives ``(nan, -1)``."""
        fplus, fcross = self._sky_grid(gwtheta, gwphi)
        f, empty, stream, on_device = self._front_end(fgw)
        best, idx = empty(f.shape[0]), empty(f.shape[0], np.int64)

        def run(pack):
            pack.fe_skymax(f, fplus, fcross, out=best, index_out=idx, stream=stream)
            return best, idx

        best, idx = self._run_verified((Nvecs, Ts, sigmas), run, asynchronous=on_device)
        if not on_device and np.ndim(fgw) == 0:
            return float(best[0]), int(idx[0])
        return best.reshape(np.shape(fgw)), idx.reshape(np.shape(fgw))

    def calculate_Fe_skymax_batch(self, fgw, gwtheta, gwphi, Nvecs, Ts, sigmas, residuals):
        """:meth:`calculate_Fe_skymax` for each of ``R`` realisations of the residuals, with the pulsars, noise model
        and basis of ``Nvecs, Ts, sigmas``: the scan of simulated noise that calibrates an all-sky search's false-alarm
        threshold (the maximum over correlated sky positions has no closed-form distribution), or of injected signals
        for its detection probability. ``residuals`` is a list of ``P`` arrays ``(R, n_p)`` as for
        :meth:`calculate_Fp_batch`, validated, cached and split into passes the same way. Returns ``(fe_max,
        sky_index)``: ``(R,)`` for a scalar ``fgw``, ``(R, *fgw.shape)`` for an array, CUDA tensors on torch's current
        stream for a float64 CUDA tensor. Row ``k`` is the sky maximum of Fe with residuals ``residuals[p][k]``, under
        the same rule (NaN loses, ties go to the lowest index, ``(nan, -1)`` where no position is finite). Values meet
        the parity bar of :meth:`calculate_Fe_skymax` but are not bit-identical to it (``fastfp_fe_skymax_residuals``,
        DESIGN.md section 5e). One sky position is a targeted search at a known position. A block-diagonal N among
        the ``Nvecs`` works as in :meth:`calculate_Fp_batch`."""
        fplus, fcross = self._sky_grid(gwtheta, gwphi)
        R, passes = self._residual_passes(residuals)
        return self._skymax_passes(fgw, fplus, fcross, Nvecs, Ts, sigmas, R, passes)

    def calculate_Fe_skymax_simulated(self, fgw, gwtheta, gwphi, Nvecs, Ts, sigmas, phiinvs, R, seed, first=0,
                                      signal=None, noise=True):
        """:meth:`calculate_Fe_skymax_batch` on ``R`` realisations of the noise model drawn on the device, with the
        arguments, stream and signal of :meth:`calculate_Fp_simulated`: the all-sky scan of simulated noise that
        calibrates the search's false-alarm threshold, or of injected signals (:meth:`cw_signal`) for its detection
        probability. Returns ``(fe_max, sky_index)`` shaped as for :meth:`calculate_Fe_skymax_batch`."""
        fplus, fcross = self._sky_grid(gwtheta, gwphi)
        R, passes = self._simulated_passes(Ts, phiinvs, R, seed, first, signal, noise)
        return self._skymax_passes(fgw, fplus, fcross, Nvecs, Ts, sigmas, R, passes)

    def _skymax_passes(self, fgw, fplus, fcross, Nvecs, Ts, sigmas, R, passes):
        f, empty, stream, on_device = self._front_end(fgw)
        best, idx = empty((R, f.shape[0])), empty((R, f.shape[0]), np.int64)

        def run(pack):
            for lo, hi in passes(pack, stream):
                pack.fe_skymax_residuals(f, fplus, fcross, out=best[lo:hi], index_out=idx[lo:hi], stream=stream)
            return best, idx

        best, idx = self._run_verified((Nvecs, Ts, sigmas), run, asynchronous=on_device)
        shape = (R,) + np.shape(fgw)
        return best.reshape(shape), idx.reshape(shape)

    def cw_signal(self, fgw, gwtheta, gwphi, a):
        """The ``signal`` argument of :meth:`calculate_Fp_simulated` / :meth:`calculate_Fe_skymax_simulated` for an
        Earth-term source at frequency ``fgw`` (scalar or ``(R,)``) and sky position ``(gwtheta, gwphi)`` with the four
        Fe amplitudes ``a`` (``(4,)`` or ``(R, 4)``), the coefficients of the templates ``[F+ s, F+ c, Fx s, Fx c]``:
        ``A_s = a1 F+ + a3 Fx`` and ``A_c = a2 F+ + a4 Fx`` per pulsar (:func:`antenna_pattern`). Returns ``(fgw,
        amp)`` with ``amp`` ``(P, 2)`` or ``(R, P, 2)``."""
        a = np.asarray(a, dtype=np.float64)
        if a.shape[-1:] != (4,) or a.ndim > 2:
            raise ValueError("a must have shape (4,) or (R, 4)")
        fplus, fcross = antenna_pattern(self.pos, gwtheta, gwphi)
        if np.ndim(fplus) != 1:
            raise ValueError("cw_signal takes one sky position")
        a = a[..., None, :]
        amp = np.stack((a[..., 0] * fplus + a[..., 2] * fcross, a[..., 1] * fplus + a[..., 3] * fcross), axis=-1)
        return np.asarray(fgw, dtype=np.float64), amp

    def _sky_grid(self, gwtheta, gwphi):
        """Antenna patterns ``(F+, Fx)``, each ``(S, P)``, of the sky grid ``gwtheta``, ``gwphi`` broadcast to ``(S,)``."""
        try:
            th, ph = np.broadcast_arrays(np.atleast_1d(np.asarray(gwtheta, dtype=np.float64)),
                                         np.atleast_1d(np.asarray(gwphi, dtype=np.float64)))
        except ValueError:
            raise ValueError("gwtheta and gwphi must broadcast to one shape (S,)") from None
        if th.ndim != 1:
            raise ValueError("gwtheta and gwphi must broadcast to one shape (S,)")
        return antenna_pattern(self.pos, th, ph)
