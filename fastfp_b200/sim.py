"""Residual realisations of a PTA's own noise model, on the host (NumPy).

This is the reference for the residual batches the library draws on the device (``fastfp_pack_simulate_residuals``,
``FastFp.calculate_Fp_simulated``; DESIGN.md section 5g), and a way to get the realisations themselves. Both use one
random stream, so realisation ``k`` here is the realisation ``k`` the device sweeps:

* Philox4x64-10 with key ``(seed, 0)`` and counter ``(q, k, p, tag)``: ``k`` the global realisation index, ``p`` the
  pulsar, ``tag`` 0 for the white noise (normal number = the pulsar's original TOA index), 1 for the ECORR epoch draws
  (normal number = epoch, in the order of the ``BlockNvec``'s slices), 2 for the basis columns (normal number = column);
* counter block ``q`` gives normals ``4q .. 4q+3``: each 64-bit word ``x`` becomes the uniform
  ``((x >> 11) + 0.5) 2^-53`` in (0, 1] (never 0; the largest word rounds to 1), and Box-Muller maps ``(u0, u1)`` to
  ``sqrt(-2 ln u0) (cos, sin)(2 pi u1)`` and ``(u2, u3)`` likewise.

:func:`philox4x64` is word for word ``np.random.Philox(key=[seed, 0], counter=[q - 1, k, p, tag]).random_raw(4)``
(NumPy increments the counter before it generates).
"""
from __future__ import annotations

import numpy as np

_M0, _M1 = np.uint64(0xD2E7470EE14C6C93), np.uint64(0xCA5A826395121157)
_W0, _W1 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBB67AE8584CAA73B)
_LO32 = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)

TWO_PI = 6.283185307179586  # the double nearest 2 pi: the device's rounding of 2 pi u and of (2 pi) f


def _mulhilo(a, b):
    """``(hi, lo)`` 64-bit halves of the 128-bit products ``a * b`` (uint64 arrays)."""
    a_lo, a_hi, b_lo, b_hi = a & _LO32, a >> _S32, b & _LO32, b >> _S32
    p0, p1, p2, p3 = a_lo * b_lo, a_lo * b_hi, a_hi * b_lo, a_hi * b_hi
    mid = (p0 >> _S32) + (p1 & _LO32) + (p2 & _LO32)
    return p3 + (p1 >> _S32) + (p2 >> _S32) + (mid >> _S32), a * b


def philox4x64(counter, key):
    """Philox4x64-10 of the four counter words and two key words (uint64, broadcast against each other): the four
    output words."""
    c = [np.asarray(x, dtype=np.uint64) for x in np.broadcast_arrays(*(np.asarray(v, dtype=np.uint64) for v in counter))]
    k0, k1 = (np.asarray(v, dtype=np.uint64) for v in key)
    with np.errstate(over="ignore"):
        for _ in range(10):
            hi0, lo0 = _mulhilo(np.broadcast_to(_M0, c[0].shape), c[0])
            hi1, lo1 = _mulhilo(np.broadcast_to(_M1, c[2].shape), c[2])
            c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
            k0, k1 = k0 + _W0, k1 + _W1
    return c


def normals(seed, k, p, tag, j):
    """Normal number ``j`` of the stream ``(seed, k, p, tag)`` (all broadcast), float64."""
    j = np.asarray(j, dtype=np.int64)
    x = philox4x64((j >> 2, k, p, tag), (seed, 0))
    second = (j & 2) != 0
    a, b = np.where(second, x[2], x[0]), np.where(second, x[3], x[1])
    u0 = ((a >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0 ** -53
    u1 = ((b >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0 ** -53
    ang = TWO_PI * u1
    return np.sqrt(-2.0 * np.log(u0)) * np.where((j & 1) != 0, np.sin(ang), np.cos(ang))


def check_seed(seed, first=0):
    """``seed`` and ``first`` as non-negative ints (the stream's key and first realisation index)."""
    for name, v in (("seed", seed), ("first", first)):
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or v < 0 or v >= 2 ** 63:
            raise ValueError(f"{name} must be an integer in [0, 2^63)")
    return int(seed), int(first)


def check_phiinvs(phiinvs, m):
    """``phiinvs``, one array of ``m[p]`` prior inverse variances per pulsar, as float64; every entry finite and
    ``>= 0``."""
    if len(phiinvs) != len(m):
        raise ValueError(f"phiinvs must be a list of {len(m)} arrays (one per pulsar)")
    out = []
    for p, a in enumerate(phiinvs):
        a = np.ascontiguousarray(np.asarray(a, dtype=np.float64))
        if a.shape != (m[p],):
            raise ValueError(f"phiinvs[{p}] must have shape ({m[p]},); got {a.shape}")
        if not (np.all(np.isfinite(a)) and np.all(a >= 0.0)):
            raise ValueError(f"phiinvs[{p}] must be finite and >= 0")
        out.append(a)
    return out


def signal_arrays(signal, R, P):
    """``signal = (freqs, amp)`` as ``(freqs (R,), amp (R, P, 2))`` float64, or ``(None, None)`` for no signal.
    ``freqs`` is a scalar or ``(R,)``; ``amp`` is ``(P, 2)`` (every realisation) or ``(R, P, 2)``, the ``(A_s, A_c)``
    of each pulsar's Earth term ``A_s sin(2 pi f t) + A_c cos(2 pi f t)``."""
    if signal is None:
        return None, None
    try:
        freqs, amp = signal
    except (TypeError, ValueError):
        raise ValueError("signal must be a pair (freqs, amp)") from None
    freqs = np.asarray(freqs, dtype=np.float64)
    amp = np.asarray(amp, dtype=np.float64)
    if freqs.shape not in ((), (R,)):
        raise ValueError(f"signal frequencies must be a scalar or have shape ({R},); got {freqs.shape}")
    if amp.shape not in ((P, 2), (R, P, 2)):
        raise ValueError(f"signal amplitudes must have shape ({P}, 2) or ({R}, {P}, 2); got {amp.shape}")
    return (np.ascontiguousarray(np.broadcast_to(freqs, (R,))),
            np.ascontiguousarray(np.broadcast_to(amp, (R, P, 2))))


def simulate_residuals(toas, Nvecs, Ts, phiinvs, R, seed, first=0, signal=None, noise=True, columns=None):
    """Realisations ``first .. first + R - 1`` of the residuals, one ``(R, n_p)`` array per pulsar:
    ``sqrt(Nvec) z`` (white noise), plus ``sqrt(j_e) eta_e`` on every TOA of epoch ``e`` for a ``BlockNvec``-like
    ``Nvec`` (kernel ECORR), plus ``T[:, cols] (sqrt(phi) zeta)[cols]`` with ``phi = 1 / phiinv``, plus the signal
    (:func:`signal_arrays`); ``noise=False`` leaves the signal alone.

    ``columns[p]`` are the basis columns drawn; by default those with ``phiinv > 1e-30``. The timing-model columns
    (``phiinv = 1e-40``) are left out: drawn explicitly their ``1e20`` amplitudes would swamp float64, and the statistic
    projects them out. The device draws them with their true, negligible weight, which needs no such rule."""
    from . import blockn

    seed, first = check_seed(seed, first)
    P = len(toas)
    m = [np.shape(T)[1] for T in Ts]
    phiinvs = check_phiinvs(phiinvs, m)
    freqs, amp = signal_arrays(signal, R, P)
    k = (first + np.arange(R, dtype=np.int64))[:, None].astype(np.uint64)
    out = []
    for p in range(P):
        t = np.asarray(toas[p], dtype=np.float64)
        n = t.shape[0]
        r = np.zeros((R, n))
        if noise:
            ep = blockn.epochs(Nvecs[p], n)
            r += np.sqrt(ep.nvec)[None, :] * normals(seed, k, p, 0, np.arange(n)[None, :])
            if ep.slices:
                eta = normals(seed, k, p, 1, np.arange(len(ep.slices))[None, :]) * np.sqrt(ep.jvec)[None, :]
                for e, (a, b) in enumerate(ep.slices):
                    r[:, a:b] += eta[:, e:e + 1]
            cols = np.nonzero(phiinvs[p] > 1e-30)[0] if columns is None else np.asarray(columns[p], dtype=np.int64)
            if cols.size:
                zeta = normals(seed, k, p, 2, cols[None, :]) * np.sqrt(1.0 / phiinvs[p][cols])[None, :]
                r += zeta @ np.asarray(Ts[p], dtype=np.float64)[:, cols].T
        if freqs is not None:
            ph = (TWO_PI * freqs)[:, None] * t[None, :]
            r += amp[:, p, 0:1] * np.sin(ph) + amp[:, p, 1:2] * np.cos(ph)
        out.append(r)
    return out
