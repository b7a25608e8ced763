"""EXTENDED-PRECISION TRUTH -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The same quantities as ``oracle/fp_oracle.py`` evaluated in x87 ``np.longdouble`` (64-bit
mantissa, eps ~ 1.1e-19), plus a first-order *conditioning* figure for every output.

Why it exists (SURVEY.md §7.3 H1): near a red-noise Fourier frequency the Earth-term basis
lies almost inside span(T) and ``(x|y) = x^T N^-1 y - (T^T N^-1 x)^T Sigma^-1 (T^T N^-1 y)``
is the difference of two numbers up to 1e6-1e10 times larger than the result. There the
reference's own float64 output is only defined to ``eps * kappa``; two correct float64
implementations that differ in summation order differ by that much. Parity tests therefore
use ``|cuda - oracle| <= 1e-10*|oracle| + c*eps*cond`` with ``cond`` from this module, and
additionally check that the CUDA path is no further from this truth than the oracle is.

Definition of "truth": the float64 inputs are exact, and the float64-rounded phase
``fl(fl(2*pi*f)*t)`` of reference ``fastfp/fastfp.py:78-79`` is taken as exact input (the
reference defines the phase by that float64 expression); everything after that -- sin/cos,
N^-1 scaling, the T^T N^-1 x products, the Sigma solve, the 2x2 solve -- is done in longdouble.
"""
from __future__ import annotations

import numpy as np

LD = np.longdouble


def _chol_ld(S):
    """Lower Cholesky factor in longdouble (no LAPACK for this dtype)."""
    A = np.array(S, dtype=LD)
    m = A.shape[0]
    L = np.zeros_like(A)
    for j in range(m):
        d = A[j, j] - np.dot(L[j, :j], L[j, :j])
        L[j, j] = np.sqrt(d)
        if j + 1 < m:
            L[j + 1 :, j] = (A[j + 1 :, j] - L[j + 1 :, :j] @ L[j, :j]) / L[j, j]
    return L


def _fwd_ld(L, B):
    """Solve L X = B (lower triangular), longdouble, B: (m, k)."""
    m = L.shape[0]
    X = np.array(B, dtype=LD)
    for j in range(m):
        X[j] = (X[j] - L[j, :j] @ X[:j]) / L[j, j]
    return X


def sweep_inner_truth(freqs, toas, residuals, Nvecs, Ts, sigmas, chunk=128):
    """The five per-(pulsar, frequency) inner products of the sweep, ``(P, F)`` longdouble each: ``Mss, Msc, Mcc``
    = (s|s), (s|c), (c|c) and ``Ns, Nc`` = (s|r), (c|r), plus the magnitudes of their two cancelling parts (the
    diagonal-N part and the subtracted Woodbury part), ``A0, A1`` for ``Ns, Nc`` and ``B00, B01, B11`` for the
    three entries of M. :func:`fp_sweep_truth` and :func:`fe_truth` are formed from them."""
    freqs = np.atleast_1d(np.asarray(freqs, dtype=np.float64))
    F, P = freqs.shape[0], len(toas)
    out = {k: np.zeros((P, F), dtype=LD) for k in _INNER_KEYS}
    for p in range(P):
        toa = np.asarray(toas[p], dtype=np.float64)
        ninv = LD(1) / np.asarray(Nvecs[p], dtype=LD)
        T = np.asarray(Ts[p], dtype=LD)
        r = np.asarray(residuals[p], dtype=LD)
        L = _chol_ld(sigmas[p])
        G = _fwd_ld(L, (T * ninv[:, None]).T)  # (m, n): L^-1 T^T N^-1
        ur = G @ r
        rn = r * ninv
        for lo in range(0, F, chunk):
            f = freqs[lo : lo + chunk]
            # float64 phase exactly as the reference forms it: ((2*pi)*f)*t
            ph = ((2 * np.pi * f)[:, None] * toa[None, :]).astype(LD)
            S, C = np.sin(ph), np.cos(ph)
            US, UC = S @ G.T, C @ G.T  # (F, m)
            Sn, Cn = S * ninv, C * ninv
            sNs, sNc, cNc = (S * Sn).sum(1), (S * Cn).sum(1), (C * Cn).sum(1)
            sNr, cNr = S @ rn, C @ rn
            bss, bsc, bcc = (US * US).sum(1), (US * UC).sum(1), (UC * UC).sum(1)
            bsr, bcr = US @ ur, UC @ ur
            _store(out, p, slice(lo, lo + chunk), Mss=sNs - bss, Msc=sNc - bsc, Mcc=cNc - bcc, Ns=sNr - bsr,
                   Nc=cNr - bcr, A0=np.abs(sNr) + np.abs(bsr), A1=np.abs(cNr) + np.abs(bcr), B00=sNs + bss,
                   B01=np.abs(sNc) + np.abs(bsc), B11=cNc + bcc)
    return out


_INNER_KEYS = ("Mss", "Msc", "Mcc", "Ns", "Nc", "A0", "A1", "B00", "B01", "B11")


def _store(out, p, cols, **vals):
    for k, v in vals.items():
        out[k][p, cols] = v


def _solve_2x2(inner):
    Mss, Msc, Mcc, Ns, Nc = (inner[k] for k in ("Mss", "Msc", "Mcc", "Ns", "Nc"))
    det = Mss * Mcc - Msc * Msc
    return (Mcc * Ns - Msc * Nc) / det, (Mss * Nc - Msc * Ns) / det


def _first_order(x0, x1, A0, A1, B00, B01, B11):
    """``|x|^T A + 0.5 |x|^T B |x|``: the first-order change of ``0.5 N^T M^-1 N`` for changes of ``N`` bounded by
    ``A`` and of ``M`` by ``B``"""
    ax0, ax1 = np.abs(x0), np.abs(x1)
    return ax0 * A0 + ax1 * A1 + LD(0.5) * (ax0 * ax0 * B00 + 2 * ax0 * ax1 * B01 + ax1 * ax1 * B11)


def terms_truth(inner):
    """``(terms (P,F) longdouble, cond (P,F) float64)`` of :func:`fp_sweep_truth` from :func:`sweep_inner_truth`."""
    x0, x1 = _solve_2x2(inner)
    terms = LD(0.5) * (inner["Ns"] * x0 + inner["Nc"] * x1)
    c = _first_order(x0, x1, *(inner[k] for k in ("A0", "A1", "B00", "B01", "B11")))
    return terms, c.astype(np.float64)


def _bwd_ld(L, B):
    """Solve L^T X = B (L lower triangular), longdouble, B: (m, k)."""
    m = L.shape[0]
    X = np.array(B, dtype=LD)
    for j in range(m - 1, -1, -1):
        X[j] = (X[j] - L[j + 1 :, j] @ X[j + 1 :]) / L[j, j]
    return X


def sigma_cond_truth(freqs, toas, residuals, Nvecs, Ts, sigmas, chunk=128):
    """Conditioning of the per-pulsar terms of :func:`fp_sweep_truth` with respect to ``Sigma`` itself: ``(P, F)``
    float64.

    :func:`fp_sweep_truth`'s ``cond`` charges the rounding committed in the inner products for an exact ``Sigma``
    solve. A float64 Cholesky of ``Sigma = L L^T`` is instead the exact factor of ``Sigma + dSigma`` with
    ``|dSigma| <= gamma_(m+1) |L| |L^T|`` elementwise (Higham, *Accuracy and Stability of Numerical Algorithms*, Thm
    10.3), and a badly conditioned ``Sigma`` (a loud, steep red process leaves ``Sigma ~ T^T N^-1 T``) turns that into
    errors ``cond`` does not see. To first order ``d(x|y) = w_x^T dSigma w_y`` with ``w_x = Sigma^-1 T^T N^-1 x``, so
    ``|d(x|y)| <= gamma * v_x^T v_y`` with ``v_x = |L^T| |w_x|``; these bounds go through the 2x2 solve as in ``cond``.
    Returned in units of the rounding factor, like ``cond``."""
    freqs = np.atleast_1d(np.asarray(freqs, dtype=np.float64))
    F, P = freqs.shape[0], len(toas)
    out = np.zeros((P, F))
    for p in range(P):
        toa = np.asarray(toas[p], dtype=np.float64)
        ninv = LD(1) / np.asarray(Nvecs[p], dtype=LD)
        T = np.asarray(Ts[p], dtype=LD)
        r = np.asarray(residuals[p], dtype=LD)
        L = _chol_ld(sigmas[p])
        aLt = np.abs(L).T
        G = _fwd_ld(L, (T * ninv[:, None]).T)  # (m, n): L^-1 T^T N^-1
        ur = G @ r
        vr = aLt @ np.abs(_bwd_ld(L, ur[:, None])[:, 0])
        rn = r * ninv
        for lo in range(0, F, chunk):
            f = freqs[lo : lo + chunk]
            ph = ((2 * np.pi * f)[:, None] * toa[None, :]).astype(LD)
            S, C = np.sin(ph), np.cos(ph)
            US, UC = G @ S.T, G @ C.T  # (m, F)
            vs, vc = aLt @ np.abs(_bwd_ld(L, US)), aLt @ np.abs(_bwd_ld(L, UC))
            Sn, Cn = S * ninv, C * ninv
            inner = dict(Mss=(S * Sn).sum(1) - (US * US).sum(0), Msc=(S * Cn).sum(1) - (US * UC).sum(0),
                         Mcc=(C * Cn).sum(1) - (UC * UC).sum(0), Ns=S @ rn - US.T @ ur, Nc=C @ rn - UC.T @ ur)
            x0, x1 = _solve_2x2(inner)
            c = _first_order(x0, x1, vs.T @ vr, vc.T @ vr, (vs * vs).sum(0), (vs * vc).sum(0), (vc * vc).sum(0))
            out[p, lo : lo + chunk] = c.astype(np.float64)
    return out


def fp_sweep_truth(freqs, toas, residuals, Nvecs, Ts, sigmas, chunk=128):
    """Truth for ``fp_sweep``. Returns ``(terms (P,F) longdouble, cond (P,F) float64)``.

    ``cond[p, f]`` bounds (to first order, in units of the relative rounding error committed
    in each of the two cancelling parts of every inner product) the absolute change of the
    per-pulsar term ``0.5 * N^T M^-1 N``:
    ``|x|^T A + 0.5 |x|^T B |x|`` with ``x = M^-1 N`` and ``A_k``/``B_kl`` the sums of the
    magnitudes of the two parts of ``N_k``/``M_kl``."""
    return terms_truth(sweep_inner_truth(freqs, toas, residuals, Nvecs, Ts, sigmas, chunk))


def get_xCy_truth(Nvec, T, sigma, x, y):
    """Truth for one ``get_xCy`` (reference ``fastfp/utils.py:49-54``); returns
    ``(value longdouble, cond float64)`` with ``cond = |x N^-1 y| + |second term|``."""
    ninv = LD(1) / np.asarray(Nvec, dtype=LD)
    T = np.asarray(T, dtype=LD)
    x = np.asarray(x, dtype=LD)
    y = np.asarray(y, dtype=LD)
    L = _chol_ld(sigma)
    ux = _fwd_ld(L, (T.T @ (x * ninv))[:, None])[:, 0]
    uy = _fwd_ld(L, (T.T @ (y * ninv))[:, None])[:, 0]
    a = (x * ninv * y).sum()
    b = ux @ uy
    return a - b, float(np.abs(a) + np.abs(b))


def fp_sweep_truth_blockn(freqs, toas, residuals, blocks, Ts, phiinvs=None, chunk=64, sigmas=None):
    """Truth for a BLOCK-DIAGONAL white-noise matrix ``N = diag(nvec) + sum_e j_e 1_e 1_e^T`` (kernel ECORR).

    The reference has no implementation of this case (``fastfp/utils.py:29-31``); it is mathematically the
    GP-basis model ``C = diag(nvec) + U J U^T + T Phi T^T`` the reference does implement (epoch-indicator
    columns appended to ``T``, ``fastfp/nmfp.py:277-282``), whose extended-precision evaluation
    (:func:`fp_sweep_truth` on the widened basis) costs O((m + n_epoch)^3) longdouble operations without
    LAPACK -- minutes per pulsar at 2500 epochs. This function evaluates the SAME quantity with ``N^-1``
    applied by Sherman-Morrison in longdouble, ``Sigma = T^T N^-1 T + diag(phiinv)`` formed in longdouble;
    ``tests/test_oracle_golden.py`` pins it against :func:`fp_sweep_truth` on the widened basis at a size
    where both run. ``blocks[p]`` is ``(nvec, [(start, stop), ...], jvec)``. With ``sigmas`` given, those
    float64 matrices are taken as exact inputs (what the engine is handed), like :func:`fp_sweep_truth` does;
    otherwise ``Sigma`` is formed here from ``phiinvs``. Returns ``(terms, cond)`` like :func:`fp_sweep_truth`."""
    return terms_truth(sweep_inner_truth_blockn(freqs, toas, residuals, blocks, Ts, phiinvs, chunk, sigmas))


def sweep_inner_truth_blockn(freqs, toas, residuals, blocks, Ts, phiinvs=None, chunk=64, sigmas=None):
    """:func:`sweep_inner_truth` for a block-diagonal N (arguments as :func:`fp_sweep_truth_blockn`)."""
    freqs = np.atleast_1d(np.asarray(freqs, dtype=np.float64))
    F, P = freqs.shape[0], len(toas)
    out = {k: np.zeros((P, F), dtype=LD) for k in _INNER_KEYS}
    for p in range(P):
        toa = np.asarray(toas[p], dtype=np.float64)
        nvec, slices, jvec = blocks[p]
        ninv = LD(1) / np.asarray(nvec, dtype=LD)
        T = np.asarray(Ts[p], dtype=LD)
        r = np.asarray(residuals[p], dtype=LD)
        n = toa.shape[0]
        # epoch membership: eid[i] = epoch of TOA i or -1; beta_e = j_e / (1 + j_e sum_e 1/nvec)
        eid = np.full(n, -1, dtype=np.int64)
        for e, (a, b) in enumerate(slices):
            eid[a:b] = e
        ne = len(slices)
        member = eid >= 0
        ssum = np.zeros(ne, dtype=LD)
        np.add.at(ssum, eid[member], ninv[member])
        jv = np.asarray(jvec, dtype=LD)
        beta = jv / (LD(1) + jv * ssum)

        def nsolve(X):  # N^-1 X, X: (n,) or (n, k)
            Y = X * (ninv if X.ndim == 1 else ninv[:, None])
            acc = np.zeros((ne,) + Y.shape[1:], dtype=LD)
            np.add.at(acc, eid[member], Y[member])
            corr = (beta if X.ndim == 1 else beta[:, None]) * acc
            Y = Y.copy()
            Y[member] -= (ninv[member] if X.ndim == 1 else ninv[member][:, None]) * corr[eid[member]]
            return Y

        NT = nsolve(T)                       # N^-1 T   (n, m)
        if sigmas is not None:
            Sigma = np.asarray(sigmas[p], dtype=LD)
        else:
            Sigma = T.T @ NT + np.diag(np.asarray(phiinvs[p], dtype=LD))
        L = _chol_ld(Sigma)
        G = _fwd_ld(L, NT.T)                 # L^-1 T^T N^-1   (m, n)
        rn = nsolve(r)
        ur = G @ r
        for lo in range(0, F, chunk):
            f = freqs[lo : lo + chunk]
            ph = ((2 * np.pi * f)[:, None] * toa[None, :]).astype(LD)
            S, C = np.sin(ph), np.cos(ph)
            Sn, Cn = nsolve(S.T).T, nsolve(C.T).T
            US, UC = S @ G.T, C @ G.T
            sNs, sNc, cNc = (S * Sn).sum(1), (S * Cn).sum(1), (C * Cn).sum(1)
            sNr, cNr = S @ rn, C @ rn
            bss, bsc, bcc = (US * US).sum(1), (US * UC).sum(1), (UC * UC).sum(1)
            bsr, bcr = US @ ur, UC @ ur
            # conditioning: the diagonal-N part and the two subtracted parts (epoch correction, Woodbury)
            dS, dC = S * ninv, C * ninv
            pss, psc, pcc = (S * dS).sum(1), np.abs(S * dC).sum(1), (C * dC).sum(1)
            _store(out, p, slice(lo, lo + chunk), Mss=sNs - bss, Msc=sNc - bsc, Mcc=cNc - bcc, Ns=sNr - bsr,
                   Nc=cNr - bcr, A0=np.abs(S * (r * ninv)).sum(1) + np.abs(bsr),
                   A1=np.abs(C * (r * ninv)).sum(1) + np.abs(bcr), B00=2 * pss - sNs + bss, B01=psc + np.abs(bsc),
                   B11=2 * pcc - cNc + bcc)
    return out


def _solve_ld(M, b):
    """``M^-1 b`` for a batch of small systems, ``M (K, n, n)``, ``b (K, n)``, in longdouble (NumPy's LAPACK-backed
    solve has no longdouble): Gaussian elimination with partial pivoting, then back substitution."""
    A, y = np.array(M, dtype=LD), np.array(b, dtype=LD)
    K, n = y.shape
    ar = np.arange(K)
    for c in range(n):
        piv = c + np.argmax(np.abs(A[:, c:, c]), axis=1)
        A[ar, c], A[ar, piv] = A[ar, piv], A[ar, c].copy()
        y[ar, c], y[ar, piv] = y[ar, piv], y[ar, c].copy()
        for r in range(c + 1, n):
            l = A[:, r, c] / A[:, c, c]
            A[:, r, c:] -= l[:, None] * A[:, c, c:]
            y[:, r] -= l * y[:, c]
    x = np.zeros_like(y)
    for r in range(n - 1, -1, -1):
        x[:, r] = (y[:, r] - (A[:, r, r + 1 :] * x[:, r + 1 :]).sum(1)) / A[:, r, r]
    return x


def fe_truth_from_inner(inner, freqs, fplus, fcross):
    """The Fe-statistic ``0.5 N^T M^-1 N`` of ``S`` sky positions (antenna patterns ``fplus``, ``fcross``: ``(S, P)``)
    from the per-pulsar inner products of :func:`sweep_inner_truth`: returns ``(fe (S,F) longdouble, cond (S,F)
    float64)``, NaN at ``f <= 0`` (the ``f^(-1/3)`` prefactor of the reference convention).

    With the four templates ``[F+ s, F+ c, Fx s, Fx c]`` of every pulsar, ``N = sum_p [F+ N_p ; Fx N_p]`` and
    ``M = sum_p [[F+^2 M_p, F+ Fx M_p], [F+ Fx M_p, Fx^2 M_p]]``. ``cond`` generalises the figure of
    :func:`fp_sweep_truth`: ``|x|^T A + 0.5 |x|^T B |x|`` with ``x = M^-1 N``, ``A = sum_p [|F+| A_p ; |Fx| A_p]`` and
    ``B = sum_p [[F+^2 B_p, |F+ Fx| B_p], [|F+ Fx| B_p, Fx^2 B_p]]`` over the part magnitudes ``A_p``, ``B_p``."""
    freqs = np.atleast_1d(np.asarray(freqs, dtype=np.float64))
    fp, fx = np.asarray(fplus, dtype=LD), np.asarray(fcross, dtype=LD)
    S, F = fp.shape[0], freqs.shape[0]
    pp, px, xx = fp * fp, fp * fx, fx * fx
    g = {k: inner[k] for k in _INNER_KEYS}
    N = np.stack((fp @ g["Ns"], fp @ g["Nc"], fx @ g["Ns"], fx @ g["Nc"]), axis=-1)  # (S, F, 4)

    def quad(a, b, c, w_pp, w_px, w_xx):  # sum_p of the 4x4 weighting of the symmetric 2x2 [[a, b], [b, c]]
        m = np.empty((S, F, 4, 4), dtype=LD)
        for (i, j), w in (((0, 0), w_pp), ((0, 2), w_px), ((2, 0), w_px), ((2, 2), w_xx)):
            m[..., i, j], m[..., i, j + 1] = w @ a, w @ b
            m[..., i + 1, j], m[..., i + 1, j + 1] = w @ b, w @ c
        return m

    M = quad(g["Mss"], g["Msc"], g["Mcc"], pp, px, xx)
    with np.errstate(all="ignore"):
        x = _solve_ld(M.reshape(-1, 4, 4), N.reshape(-1, 4)).reshape(S, F, 4)
        fe = LD(0.5) * (N * x).sum(-1)
        afp, afx = np.abs(fp), np.abs(fx)
        A = np.stack((afp @ g["A0"], afp @ g["A1"], afx @ g["A0"], afx @ g["A1"]), axis=-1)
        B = quad(g["B00"], g["B01"], g["B11"], pp, np.abs(px), xx)
        ax = np.abs(x)
        cond = (ax * A).sum(-1) + LD(0.5) * np.einsum("sfk,sfkl,sfl->sf", ax, B, ax)
    bad = ~(freqs > 0)
    fe[:, bad] = np.nan
    cond[:, bad] = np.nan
    return fe, cond.astype(np.float64)


_PI = LD("3.14159265358979323846264338327950288")
_FYR = LD(1) / LD(31557600)


def _powerlaw_phi_ld(Ffreqs, log10_A, gamma):
    """``(D, m)`` longdouble power law of ``Ffreqs`` for ``(D,)`` parameters (see :func:`powerlaw_phiinv_truth`)."""
    f = np.asarray(Ffreqs, dtype=np.float64).astype(LD)
    df = np.repeat(np.diff(np.concatenate((np.zeros(1, dtype=LD), f[::2]))), 2)[: f.shape[0]]
    A = np.atleast_1d(np.asarray(log10_A, dtype=np.float64)).astype(LD)[:, None]
    g = np.atleast_1d(np.asarray(gamma, dtype=np.float64)).astype(LD)[:, None]
    amp = np.power(LD(10), A)
    return np.power(f, -g) * (amp * amp) / 12 / (_PI * _PI) * np.power(_FYR, g - 3) * df


def powerlaw_phiinv_truth(Ffreqs, log10_A, gamma, curn_Ffreqs=None, curn_log10_A=None, curn_gamma=None):
    """Truth for the per-draw block of ``RN_container.get_phiinv``: ``(D, m)`` longdouble ``1/phi``.

    ``phi = f^-gamma (10^log10_A)^2 / 12 / pi^2 fyr^(gamma - 3) df`` with ``df = repeat(diff([0, Ffreqs[::2]]), 2)``
    (reference ``fastfp/nmfp.py:226-234``), plus the common process's power law of ``curn_Ffreqs`` on the leading
    entries (``:247, 275``), then ``1/phi`` (``:315``). ``log10_A`` / ``gamma`` are ``(D,)`` (or scalars), the CURN
    ones ``(D,)``. The float64 inputs are exact; everything after them, ``gamma - 3``, ``pi`` and ``fyr = 1 / 31557600``
    included, is longdouble."""
    phi = _powerlaw_phi_ld(Ffreqs, log10_A, gamma)
    if curn_Ffreqs is not None and len(curn_Ffreqs):
        c = _powerlaw_phi_ld(curn_Ffreqs, curn_log10_A, curn_gamma)
        phi[:, : c.shape[1]] += c
    return LD(1) / phi


def fe_truth(freqs, fplus, fcross, toas, residuals, Nvecs, Ts, sigmas, blocks=None):
    """Truth for ``fastfp_fe_sweep``: ``(fe (S,F) longdouble, cond (S,F) float64)`` for the antenna patterns
    ``fplus``, ``fcross`` ``(S, P)`` (:func:`fe_truth_from_inner`). The inner products are those of
    :func:`fp_sweep_truth`; with ``blocks`` (as in :func:`fp_sweep_truth_blockn`, ``Nvecs`` then unused) ``N^-1`` is
    applied by Sherman-Morrison and ``sigmas`` are the exact block-N Sigma matrices."""
    if blocks is None:
        inner = sweep_inner_truth(freqs, toas, residuals, Nvecs, Ts, sigmas)
    else:
        inner = sweep_inner_truth_blockn(freqs, toas, residuals, blocks, Ts, sigmas=sigmas)
    return fe_truth_from_inner(inner, freqs, fplus, fcross)
