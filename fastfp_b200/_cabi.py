"""ctypes binding of ``libfastfp_b200.so`` (the C ABI of ``include/fastfp_b200.h``).

The product path is the CUDA library; there is deliberately **no CPU fallback**: if the
library is missing, or no CUDA device is visible, every compute entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Sequence

import numpy as np

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_lib", "libfastfp_b200.so")
_lib = None

c_double_p = C.POINTER(C.c_double)
c_int64_p = C.POINTER(C.c_int64)
c_double_pp = C.POINTER(c_double_p)

FREQS_ON_DEVICE = 1
OUT_ON_DEVICE = 2
PARAMS_ON_DEVICE = 4
SIM_NO_NOISE = 1

# every symbol include/fastfp_b200.h declares: name -> (restype, argtypes)
SYMBOLS = {
    "fastfp_last_error": (C.c_char_p, []),
    "fastfp_version": (C.c_int, []),
    "fastfp_device_count": (C.c_int, []),
    "fastfp_pack_create": (
        C.c_int,
        [C.c_int, C.c_int, c_int64_p, c_int64_p, c_double_pp, c_double_pp, c_double_pp, c_double_pp,
         c_double_pp, C.c_void_p, C.POINTER(C.c_void_p)],
    ),
    "fastfp_fp_sweep": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p]),
    "fastfp_fp_terms": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p]),
    "fastfp_fe_sweep": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                  C.c_int, C.c_void_p]),
    "fastfp_fe_skymax": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                   C.c_void_p, C.c_int, C.c_void_p]),
    "fastfp_pack_set_residuals": (C.c_int, [C.c_void_p, C.c_int64, c_double_pp, C.c_void_p]),
    "fastfp_pack_set_residuals_blockn": (
        C.c_int,
        [C.c_void_p, C.c_int64, c_int64_p, c_double_pp, c_double_pp, C.POINTER(C.POINTER(C.c_int32)), c_double_pp,
         C.POINTER(C.POINTER(C.c_ubyte)), C.c_void_p],
    ),
    "fastfp_pack_simulate_residuals": (
        C.c_int,
        [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, c_double_pp, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p],
    ),
    "fastfp_pack_simulate_residuals_blockn": (
        C.c_int,
        [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, c_double_pp, C.c_void_p, C.c_void_p, c_int64_p,
         C.POINTER(C.POINTER(C.c_int32)), c_double_pp, C.POINTER(C.POINTER(C.c_ubyte)),
         C.POINTER(C.POINTER(C.c_int32)), C.POINTER(C.POINTER(C.c_int32)), c_double_pp, c_double_pp, C.c_int,
         C.c_void_p],
    ),
    "fastfp_fp_sweep_residuals": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p]),
    "fastfp_fe_skymax_residuals": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                             C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "fastfp_nmfp_pack_create": (
        C.c_int,
        [C.c_int, C.c_int, c_int64_p, c_int64_p, c_double_pp, c_double_pp, c_double_pp, c_double_pp,
         c_double_pp, c_int64_p, c_double_pp, C.c_void_p, C.POINTER(C.c_void_p)],
    ),
    "fastfp_nmfp_tile_sizes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "fastfp_nmfp_stage_a": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "fastfp_nmfp_stage_b": (
        C.c_int,
        [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p],
    ),
    "fastfp_nmfp_sweep": (
        C.c_int,
        [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p],
    ),
    "fastfp_powerlaw_phiinv": (
        C.c_int,
        [C.c_void_p, c_double_pp, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
         C.c_void_p, C.c_void_p, C.c_void_p],
    ),
    "fastfp_sweep_chunk_toas": (C.c_int, [C.c_int64, C.c_int]),
    "fastfp_pack_create_blockn": (
        C.c_int,
        [C.c_int, C.c_int, c_int64_p, c_int64_p, c_double_pp, c_double_pp, c_double_pp, c_double_pp, c_double_pp,
         c_double_pp, C.POINTER(C.POINTER(C.c_int32)), c_double_pp, C.POINTER(C.POINTER(C.c_ubyte)), c_int64_p,
         c_double_pp, C.c_void_p, C.POINTER(C.c_void_p)],
    ),
    "fastfp_pack_destroy": (None, [C.c_void_p]),
    "fastfp_pack_bytes": (C.c_int64, [C.c_void_p]),
    "fastfp_pack_num_pulsars": (C.c_int, [C.c_void_p]),
    "fastfp_pack_mvar_total": (C.c_int64, [C.c_void_p]),
    "fastfp_pack_set_path": (C.c_int, [C.c_void_p, C.c_int]),
    "fastfp_pack_path": (C.c_int, [C.c_void_p]),
    "fastfp_pack_factor_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32)]),
    "fastfp_hash64": (C.c_uint64, [C.c_void_p, C.c_int64, C.c_uint64]),
    "fastfp_hash64_many": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "fastfp_kernel_launches": (C.c_int64, []),
    "fastfp_device_bytes": (C.c_int64, []),
    "fastfp_xcy": (
        C.c_int,
        [C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
         C.c_void_p, C.c_void_p],
    ),
    "fastfp_tnt": (
        C.c_int,
        [C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p],
    ),
    "fastfp_nmfp_stage_timing": (C.c_int, [C.c_void_p, C.c_int]),
    "fastfp_nmfp_stage_ms": (C.c_int, [C.c_void_p, c_double_p]),
    "fastfp_xcy_blockn": (
        C.c_int,
        [C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
         C.c_void_p, C.c_void_p],
    ),
    "fastfp_fp64_peak": (C.c_int, [C.c_int, C.c_int, C.c_int, c_double_p, c_double_p]),
    "fastfp_row_groups": (C.c_int, [C.c_int64, C.POINTER(C.c_int64)]),
}


MAX_M = 640  # G rows of the widest sweep kernel (csrc/ffp_internal.cuh)
MAX_M_WIDE = 2688  # widest basis of a diagonal-N Fp pack, swept as row groups of at most MAX_M rows (DESIGN.md 5h)


def row_groups(m: int):
    """The row groups the library sweeps a basis of width ``m`` in (``fastfp_row_groups``): a list of ``(start, stop)``
    row ranges, one for ``m <= MAX_M``. Raises ``ValueError`` outside ``1 .. MAX_M_WIDE``."""
    starts = (C.c_int64 * (m // 8 + 2))() if 1 <= m <= MAX_M_WIDE else None
    g = load().fastfp_row_groups(int(m), starts)
    if g < 1:
        raise ValueError(f"basis width m={m} is outside 1 .. {MAX_M_WIDE}")
    return [(starts[k], starts[k + 1]) for k in range(g)]


def sweep_rows(m: int, R: int = 0, blockn: bool = False) -> int:
    """G rows of the sweep kernel a pulsar of basis width ``m`` takes: its basis rows, then ``R`` residual realisations
    from row ``roundup8(m)`` on, then with a block-diagonal N the 8 epoch-slot rows (csrc/ffp_internal.cuh)."""
    return -(-m // 8) * 8 + -(-R // 8) * 8 + (8 if blockn else 0)


def max_residual_rows(m, blockn: bool = False) -> int:
    """Most residual realisations ``fastfp_pack_set_residuals`` takes for pulsars of basis widths ``m``: every pulsar
    needs :func:`sweep_rows` of the sweep kernel's ``MAX_M`` G rows. A block-diagonal N pack
    (``fastfp_pack_set_residuals_blockn``) needs 8 more, the epoch slots. Residual batches take no basis wider than
    ``MAX_M`` columns (row groups are for plain sweeps): ``ValueError`` for such a pulsar."""
    if max(m) > MAX_M:
        raise ValueError(f"residual batches need every basis to be at most {MAX_M} columns wide; pulsar "
                         f"{list(m).index(max(m))} has a basis wider than {MAX_M} (m = {max(m)})")
    return MAX_M - sweep_rows(max(m), 0, blockn)


def check_realisations(residuals, n):
    """``residuals``, a list of one ``(R, n[p])`` array per pulsar with the same ``R``, as float64 arrays, and ``R``."""
    if len(residuals) != len(n):
        raise ValueError(f"residuals must be a list of {len(n)} arrays (one per pulsar)")
    res = [as_f64(r) for r in residuals]
    R = res[0].shape[0] if res[0].ndim == 2 else -1
    for p, r in enumerate(res):
        if r.shape != (R, n[p]):
            raise ValueError(f"residuals[{p}] must have shape (R, {n[p]}) with the same R for every pulsar; got {r.shape}")
    return res, R


class FastFpError(RuntimeError):
    pass


def lib_path() -> str:
    return _LIB_PATH


def load():
    """Load the shared library (once). Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise FastFpError(
            f"{_LIB_PATH} is missing: build it with `python -m fastfp_b200.build` "
            "(there is no CPU fallback for the Fp hot path)"
        )
    lib = C.CDLL(_LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        msg = load().fastfp_last_error()
        raise FastFpError(f"fastfp_b200 error {rc}: {msg.decode() if msg else '?'}")


def require_device() -> int:
    n = load().fastfp_device_count()
    if n < 1:
        raise FastFpError("no CUDA device visible: the Fp hot path only runs on an H100 (no CPU fallback)")
    return n


def as_f64(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64))


def _ptr_array(arrs: Sequence[np.ndarray]):
    arr = (c_double_p * len(arrs))()
    for i, a in enumerate(arrs):
        arr[i] = a.ctypes.data_as(c_double_p)
    return arr


def _int64_array(vals: Sequence[int]):
    return (C.c_int64 * len(vals))(*[int(v) for v in vals])


def _is_cuda_tensor(x) -> bool:
    return type(x).__module__.startswith("torch") and getattr(x, "is_cuda", False)


def _vp(x) -> C.c_void_p:
    """host ndarray / CUDA tensor / integer device address -> void*"""
    if isinstance(x, np.ndarray):
        return C.c_void_p(x.ctypes.data)
    if _is_cuda_tensor(x):
        return C.c_void_p(x.data_ptr())
    return C.c_void_p(int(x))


def _check_lists(toas, residuals, Nvecs, Ts, mats, what):
    P = len(toas)
    if P < 1 or not (len(residuals) == len(Nvecs) == len(Ts) == len(mats) == P):
        raise ValueError(f"toas, residuals, Nvecs, Ts and {what} must be lists of equal length P >= 1")
    toas, residuals, Nvecs = [as_f64(a) for a in toas], [as_f64(a) for a in residuals], [as_f64(a) for a in Nvecs]
    Ts, mats = [as_f64(a) for a in Ts], [as_f64(a) for a in mats]
    n, m = [], []
    for p in range(P):
        if Ts[p].ndim != 2:
            raise ValueError(f"Ts[{p}] must be 2-D (ntoa, nbasis)")
        np_, mp_ = Ts[p].shape
        if toas[p].shape != (np_,) or residuals[p].shape != (np_,) or Nvecs[p].shape != (np_,):
            raise ValueError(
                f"pulsar {p}: toas/residuals/Nvec must have shape ({np_},) to match Ts "
                "(a diagonal N is required, as in the reference's get_xCy)"
            )
        if mats[p].shape != (mp_, mp_):
            raise ValueError(f"pulsar {p}: {what} must have shape ({mp_}, {mp_})")
        n.append(np_)
        m.append(mp_)
    return P, n, m, toas, residuals, Nvecs, Ts, mats


def hash64(a: np.ndarray, seed: int = 0) -> int:
    """64-bit hash of every byte of a C-contiguous host array (``fastfp_hash64``)."""
    return int(load().fastfp_hash64(C.c_void_p(a.ctypes.data), a.nbytes, C.c_uint64(seed & (2**64 - 1))))


def hash64_many(arrays, seeds) -> list:
    """``hash64`` of each C-contiguous host array in one library call (one thread pool over all of them)."""
    n = len(arrays)
    if n == 0:
        return []
    ptrs = (C.c_void_p * n)(*[a.ctypes.data for a in arrays])
    sizes = (C.c_int64 * n)(*[a.nbytes for a in arrays])
    sd = (C.c_uint64 * n)(*[s & (2**64 - 1) for s in seeds])
    out = (C.c_uint64 * n)()
    check(load().fastfp_hash64_many(ptrs, sizes, n, sd, out))
    return list(out)


class Pack:
    """Owner of one ``fastfp_pack_t*``: the device-resident packed pulsar array."""

    def __init__(self, handle, P: int, device: int, nmfp: bool, n, m):
        self._h, self.P, self.device, self.nmfp = handle, P, device, nmfp
        self.n, self.m = list(n), list(m)
        self._sim_layouts = {}  # block-N packs: simulate_residuals_blockn's layout arrays per tuple of chunk sizes
        self._warn_if_not_spd()

    PATHS = {"auto": 0, "fp64": 1, "i8": 2, "mixed": 3}
    blockn = False  # a block-diagonal N (set by create)
    epochs = None   # block-N packs: each pulsar's blockn.Epochs (its realisations are laid out with them)
    R = 0           # realisations set by set_residuals

    def set_path(self, path: str) -> None:
        """Kernel of the plain-Fp sweep: "auto" (default: the fp64 DMMA kernel), "fp64", "i8" (the INT8
        tensor-core kernel; raises unless every pulsar fits) or "mixed" (the tensor kernel for the pulsars it takes,
        the fp64 kernel for the others; raises if it takes none); ``path`` then reads "fp64", "i8" or "mixed"."""
        check(load().fastfp_pack_set_path(self._h, self.PATHS[path]))

    @property
    def path(self) -> str:
        return {1: "fp64", 2: "i8", 3: "mixed"}[load().fastfp_pack_path(self._h)]

    def factor_info(self):
        """Per-pulsar status of the one-time Cholesky (0 = fine, j+1 = pivot j not positive)."""
        info = (C.c_int32 * self.P)()
        rc = load().fastfp_pack_factor_info(self._h, info)
        if rc < 0:
            check(rc)
        return list(info)

    def _warn_if_not_spd(self):
        bad = [(p, v) for p, v in enumerate(self.factor_info()) if v]
        if bad:
            import warnings

            what = "Sigma" if not self.nmfp else "the draw-independent block of Sigma"
            warnings.warn(
                "fastfp_b200: " + what + " is not numerically symmetric positive definite for pulsar(s) "
                + ", ".join(f"{p} (pivot {v - 1})" for p, v in bad)
                + "; their terms are NaN. The sweep path factorises Sigma = L L^T (lower triangle); the "
                "reference's general LU solve is only available through get_xCy.", RuntimeWarning, stacklevel=3)

    @classmethod
    def create(cls, toas, residuals, Nvecs, Ts, mats, m_fix=None, phiinv_fix=None, device: int = 0,
               stream: int = 0) -> "Pack":
        """Pack the pulsar lists on ``device``. ``mats`` are the sigmas of a plain-Fp pack (``m_fix is None``) or the
        TNTs of an nmfp pack, whose ``m_fix[p]`` leading columns are draw-independent with prior ``phiinv_fix[p]``.
        A ``blockn`` object among the ``Nvecs`` (a block-diagonal N, kernel ECORR) makes the pack a block-N one."""
        from . import blockn

        block = any(blockn.is_block(N) for N in Nvecs)
        if block:
            P = len(toas)
            if P < 1 or not (len(residuals) == len(Nvecs) == len(Ts) == len(mats) == P):
                raise ValueError("toas, residuals, Nvecs, Ts and the matrices must be lists of equal length P >= 1")
            Ts, mats = [as_f64(T) for T in Ts], [as_f64(a) for a in mats]
            prep, n, m, epochs = [], [], [], []
            for p in range(P):
                if Ts[p].ndim != 2 or mats[p].shape != (Ts[p].shape[1],) * 2:
                    raise ValueError(f"pulsar {p}: Ts must be (ntoa, nbasis) and the matrix (nbasis, nbasis)")
                ci = load().fastfp_sweep_chunk_toas(Ts[p].shape[1], 1)
                if ci <= 0:
                    raise ValueError(f"pulsar {p}: basis width {Ts[p].shape[1]} is not supported with a block-diagonal N")
                prep.append(blockn.prepare(toas[p], residuals[p], Nvecs[p], Ts[p], ci))
                epochs.append(blockn.epochs(Nvecs[p], Ts[p].shape[0]))
                n.append(prep[-1]["toas"].shape[0])
                m.append(Ts[p].shape[1])
        else:
            what = "sigmas" if m_fix is None else "TNTs"
            P, n, m, toas, residuals, Nvecs, Ts, mats = _check_lists(toas, residuals, Nvecs, Ts, mats, what)
        nmfp, fixed = m_fix is not None, (None, None)
        top = MAX_M if nmfp else MAX_M_WIDE  # block-N widths are checked above
        for p, mp_ in enumerate(m):
            if not block and mp_ > top:
                raise ValueError(f"pulsar {p}: basis width {mp_} exceeds the maximum {top} of "
                                 + ("a noise-marginalised pack" if nmfp else "a diagonal-N pack"))
        if nmfp:
            if len(m_fix) != P or len(phiinv_fix) != P:
                raise ValueError("m_fix and phiinv_fix must have one entry per pulsar")
            pf = []
            for p in range(P):
                if not 0 <= int(m_fix[p]) <= m[p]:
                    raise ValueError(f"pulsar {p}: m_fix out of range")
                a = as_f64(phiinv_fix[p]).reshape(-1)
                if a.shape[0] != int(m_fix[p]):
                    raise ValueError(f"pulsar {p}: phiinv_fix must have m_fix entries")
                pf.append(a if a.size else np.zeros(1))
            fixed = (_int64_array(m_fix), _ptr_array(pf))
        lib = load()
        require_device()
        h = C.c_void_p()
        head = (device, P, _int64_array(n), _int64_array(m))
        tail = (C.c_void_p(stream), C.byref(h))
        if block:
            i32pp = (C.POINTER(C.c_int32) * P)(*[d["slot_idx"].ctypes.data_as(C.POINTER(C.c_int32)) for d in prep])
            u8pp = (C.POINTER(C.c_ubyte) * P)(*[d["done_mask"].ctypes.data_as(C.POINTER(C.c_ubyte)) for d in prep])
            arrays = [_ptr_array([d[k] for d in prep]) for k in ("toas", "res", "res_w", "Nvec", "T")]
            check(lib.fastfp_pack_create_blockn(*head, *arrays, _ptr_array(mats), i32pp,
                                                _ptr_array([d["slot_val"] for d in prep]), u8pp,
                                                *fixed, *tail))
        elif nmfp:
            check(lib.fastfp_nmfp_pack_create(*head, *map(_ptr_array, (toas, residuals, Nvecs, Ts, mats)), *fixed, *tail))
        else:
            check(lib.fastfp_pack_create(*head, *map(_ptr_array, (toas, residuals, Nvecs, Ts, mats)), *tail))
        pack = cls(h, P, device, nmfp, n, m)
        pack.blockn = block
        if block:
            pack.epochs = epochs
        return pack

    # -- sweeps -------------------------------------------------------------------------
    @staticmethod
    def _stage(freqs, out, rows=None):
        """``freqs``: host ndarray, contiguous CUDA tensor or ``(device_address, F)``; ``out``: None (a host array of
        shape ``(F,)`` or ``(rows, F)`` is allocated and returned), a host ndarray, a contiguous CUDA tensor, or an
        integer device address. Returns the frequency and output arguments (kept alive by the caller), ``F``, the array
        to return and the location flags."""
        flags = 0
        if isinstance(freqs, tuple):
            freqs, F = freqs
            flags |= FREQS_ON_DEVICE
        elif _is_cuda_tensor(freqs):
            F = freqs.numel()
            flags |= FREQS_ON_DEVICE
        else:
            freqs = as_f64(freqs).reshape(-1)
            F = freqs.shape[0]
        ret = None
        if out is None:
            out = ret = np.empty((F,) if rows is None else (rows, F), dtype=np.float64)
        elif not isinstance(out, np.ndarray):
            flags |= OUT_ON_DEVICE
        return freqs, out, F, ret, flags

    def _sky(self, fplus, fcross):
        fplus, fcross = as_f64(fplus), as_f64(fcross)
        if fplus.ndim != 2 or fplus.shape != fcross.shape or fplus.shape[1] != self.P:
            raise ValueError("fplus and fcross must both have shape (n_sky, n_pulsars)")
        return fplus, fcross, fplus.shape[0]

    def fp_sweep(self, freqs, out=None, stream: int = 0, terms: bool = False):
        """``freqs``: host ndarray, CUDA tensor or ``(device_address, F)``; ``out``: None (a host array is
        returned), a host ndarray, a CUDA tensor, or an integer device address."""
        freqs, out, F, ret, flags = self._stage(freqs, out, self.P if terms else None)
        fn = load().fastfp_fp_terms if terms else load().fastfp_fp_sweep
        check(fn(self._h, _vp(freqs), F, _vp(out), flags, C.c_void_p(stream)))
        return ret

    def fe_sweep(self, freqs, fplus, fcross, out=None, stream: int = 0):
        """Fe-statistic for ``S`` sky positions: ``fplus``, ``fcross`` host arrays ``(S, P)``; returns / fills
        ``(S, F)``. ``freqs`` / ``out`` as in :meth:`fp_sweep`."""
        fplus, fcross, S = self._sky(fplus, fcross)
        freqs, out, F, ret, flags = self._stage(freqs, out, S)
        check(load().fastfp_fe_sweep(self._h, _vp(freqs), F, _vp(fplus), _vp(fcross), S, _vp(out), flags,
                                     C.c_void_p(stream)))
        return ret

    def fe_skymax(self, freqs, fplus, fcross, out=None, index_out=None, stream: int = 0):
        """Loudest of ``S`` sky positions per frequency: ``fplus``, ``fcross`` host arrays ``(S, P)``. Returns / fills
        ``(fe_max, sky_index)``, ``(F,)`` float64 and int64. ``freqs`` / ``out`` as in :meth:`fp_sweep`; ``index_out``
        is a host int64 array when ``out`` is on the host, a CUDA tensor or device address when ``out`` is on the
        device."""
        return self._skymax(load().fastfp_fe_skymax, None, freqs, fplus, fcross, out, index_out, stream)

    def fe_skymax_residuals(self, freqs, fplus, fcross, out=None, index_out=None, stream: int = 0):
        """:meth:`fe_skymax` for each realisation set by :meth:`set_residuals`: ``(fe_max, sky_index)`` of shape
        ``(R, F)``. Always the fp64 kernel, whatever :attr:`path` says."""
        return self._skymax(load().fastfp_fe_skymax_residuals, self.R, freqs, fplus, fcross, out, index_out, stream)

    def _skymax(self, fn, rows, freqs, fplus, fcross, out, index_out, stream):
        fplus, fcross, S = self._sky(fplus, fcross)
        freqs, out, F, ret, flags = self._stage(freqs, out, rows)
        shape = (F,) if rows is None else (rows, F)
        iret = None
        if flags & OUT_ON_DEVICE:
            if index_out is None or isinstance(index_out, np.ndarray):
                raise ValueError("out is a device address, so index_out must be one too")
        elif index_out is None:
            index_out = iret = np.empty(shape, dtype=np.int64)
        elif not (isinstance(index_out, np.ndarray) and index_out.dtype == np.int64 and index_out.shape == shape
                  and index_out.flags.c_contiguous):
            raise ValueError("index_out must be a contiguous int64 host array of shape " + ("(F,)" if rows is None else "(R, F)"))
        check(fn(self._h, _vp(freqs), F, _vp(fplus), _vp(fcross), S, _vp(out), _vp(index_out), flags,
                 C.c_void_p(stream)))
        return ret, iret

    def set_residuals(self, residuals, stream: int = 0) -> None:
        """Realisations of the residuals for :meth:`fp_sweep_residuals`: ``residuals[p]`` is ``(R, n_p)`` (host); the
        pack keeps them until the next call. ``R`` is at most :func:`max_residual_rows` of the pack's widths; an
        empty list of rows (``R == 0``) releases them."""
        if self.blockn:  # its TOAs are re-laid out by epoch (blockn.prepare); the library refuses these packs too
            raise FastFpError("set_residuals needs a diagonal-N pack; this one has a block-diagonal N and takes its "
                              "realisations through set_residuals_blockn")
        res, R = check_realisations(residuals, self.n)
        check(load().fastfp_pack_set_residuals(self._h, R, _ptr_array(res), C.c_void_p(stream)))
        self.R = R

    def set_residuals_blockn(self, residuals, stream: int = 0) -> None:
        """:meth:`set_residuals` for a block-diagonal N pack: ``residuals[p]`` is ``(R, n_p)`` (host) in the caller's
        original TOA order, ``n_p`` the pulsar's TOA count before the epoch layout. The rows are laid out for the chunk
        size of the residual kernel (``blockn.layout``), the Sherman-Morrison ``N^-1 r_k`` is applied on the host
        (``blockn.solve_rows``) and ``fastfp_pack_set_residuals_blockn`` builds the packets. ``R`` is at most
        ``max_residual_rows(m, blockn=True)``; ``R == 0`` releases the set."""
        from . import blockn

        if not self.blockn:
            raise FastFpError("set_residuals_blockn needs a block-diagonal N pack; this one takes set_residuals")
        res, R = check_realisations(residuals, [ep.n for ep in self.epochs])
        lib = load()
        P = self.P
        i32pp, u8pp = C.POINTER(C.c_int32) * P, C.POINTER(C.c_ubyte) * P
        if R == 0 or R > max_residual_rows(self.m, blockn=True):  # nothing to lay out: the library releases or refuses
            check(lib.fastfp_pack_set_residuals_blockn(self._h, R, _int64_array(self.n), (c_double_p * P)(),
                                                       (c_double_p * P)(), i32pp(), (c_double_p * P)(), u8pp(),
                                                       C.c_void_p(stream)))
            self.R = 0
            return
        n, raw, rw, sidx, sval, dm = [], [], [], [], [], []
        for p in range(P):
            ci = lib.fastfp_sweep_chunk_toas(sweep_rows(self.m[p], R), 1)
            lay = blockn.layout(self.epochs[p], ci)
            order = lay["order"]
            n.append(order.shape[0])
            raw.append(blockn.relay(order, res[p]))
            rw.append(blockn.relay(order, blockn.solve_rows(self.epochs[p], res[p])))
            sidx.append(lay["slot_idx"])
            sval.append(lay["slot_val"])
            dm.append(lay["done_mask"])
        check(lib.fastfp_pack_set_residuals_blockn(
            self._h, R, _int64_array(n), _ptr_array(raw), _ptr_array(rw),
            i32pp(*[a.ctypes.data_as(C.POINTER(C.c_int32)) for a in sidx]), _ptr_array(sval),
            u8pp(*[a.ctypes.data_as(C.POINTER(C.c_ubyte)) for a in dm]), C.c_void_p(stream)))
        self.R = R

    def _sim_args(self, R, seed, first, phiinvs, signal, noise):
        """The arguments both simulate calls share, checked: seed, first, the priors, the signal and the flags."""
        from . import sim

        seed, first = sim.check_seed(seed, first)
        phi = sim.check_phiinvs(phiinvs, self.m)
        freqs, amp = sim.signal_arrays(signal, R, self.P)
        keep = (phi, freqs, amp)
        args = (R, seed, first, _ptr_array(phi), None if freqs is None else _vp(freqs), None if amp is None else _vp(amp))
        return args, (0 if noise else SIM_NO_NOISE), keep

    def simulate_residuals(self, R: int, seed: int, phiinvs, first: int = 0, signal=None, noise: bool = True,
                           stream: int = 0) -> None:
        """:meth:`set_residuals` with ``R`` realisations of the pack's own noise model drawn on the device
        (``fastfp_pack_simulate_residuals``): rows ``first .. first + R - 1`` of the stream of ``seed``, which
        :func:`fastfp_b200.sim.simulate_residuals` reproduces on the host. ``phiinvs[p]`` is the ``(m_p,)`` prior
        ``1/phi`` that went into ``sigma_p``; ``signal = (freqs, amp)`` as in :func:`fastfp_b200.sim.signal_arrays`;
        ``noise=False`` sets the signal alone. ``R == 0`` releases the set."""
        if self.blockn:
            raise FastFpError("simulate_residuals needs a diagonal-N pack; this one has a block-diagonal N and takes "
                              "simulate_residuals_blockn")
        args, flags, keep = self._sim_args(R, seed, first, phiinvs, signal, noise)
        check(load().fastfp_pack_simulate_residuals(self._h, *args, flags, C.c_void_p(stream)))
        self.R = R

    def simulate_residuals_blockn(self, R: int, seed: int, phiinvs, first: int = 0, signal=None, noise: bool = True,
                                  stream: int = 0) -> None:
        """:meth:`simulate_residuals` for a block-diagonal N pack (``fastfp_pack_simulate_residuals_blockn``): the
        draw adds the ECORR epoch terms and the device applies the Sherman-Morrison ``N^-1``. The layout arrays of
        :meth:`set_residuals_blockn` are built once per pulsar per call; nothing is done per realisation on the host."""
        from . import blockn

        if not self.blockn:
            raise FastFpError("simulate_residuals_blockn needs a block-diagonal N pack; this one takes "
                              "simulate_residuals")
        args, flags, keep = self._sim_args(R, seed, first, phiinvs, signal, noise)
        lib = load()
        P = self.P
        i32pp, u8pp = C.POINTER(C.c_int32) * P, C.POINTER(C.c_ubyte) * P
        i32 = lambda arrs: i32pp(*[a.ctypes.data_as(C.POINTER(C.c_int32)) for a in arrs])  # noqa: E731
        if R == 0 or R > max_residual_rows(self.m, blockn=True):  # nothing to lay out: the library releases or refuses
            check(lib.fastfp_pack_simulate_residuals_blockn(self._h, *args, _int64_array(self.n), i32pp(),
                                                            (c_double_p * P)(), u8pp(), i32pp(), i32pp(),
                                                            (c_double_p * P)(), (c_double_p * P)(), flags,
                                                            C.c_void_p(stream)))
            self.R = 0
            return
        cis = tuple(lib.fastfp_sweep_chunk_toas(sweep_rows(m, R), 1) for m in self.m)
        if cis not in self._sim_layouts:  # the layouts of these chunk sizes, kept for the next pass or call
            arrs = [[] for _ in range(8)]
            for ep, ci in zip(self.epochs, cis):
                lay = blockn.layout(ep, ci)
                order = lay["order"]
                ep_of = np.full(ep.n, -1, dtype=np.int32)
                for e, (a, b) in enumerate(ep.slices):
                    ep_of[a:b] = e
                eidx = np.where(order >= 0, ep_of[np.maximum(order, 0)], -1).astype(np.int32)
                for lst, a in zip(arrs, (order.shape[0], lay["slot_idx"], lay["slot_val"], lay["done_mask"],
                                         np.ascontiguousarray(order.astype(np.int32)), np.ascontiguousarray(eidx),
                                         as_f64(np.sqrt(ep.jvec)) if ep.slices else np.zeros(1),
                                         as_f64(ep.beta) if ep.slices else np.zeros(1))):
                    lst.append(a)
            self._sim_layouts[cis] = arrs
        n, sidx, sval, dm, tidx, eidx, sj, beta = self._sim_layouts[cis]
        check(lib.fastfp_pack_simulate_residuals_blockn(
            self._h, *args, _int64_array(n), i32(sidx), _ptr_array(sval),
            u8pp(*[a.ctypes.data_as(C.POINTER(C.c_ubyte)) for a in dm]), i32(tidx), i32(eidx), _ptr_array(sj),
            _ptr_array(beta), flags, C.c_void_p(stream)))
        self.R = R

    def fp_sweep_residuals(self, freqs, out=None, stream: int = 0):
        """Fp of each realisation set by :meth:`set_residuals`: ``(R, F)``. ``freqs`` / ``out`` as in
        :meth:`fp_sweep`. Always the fp64 kernel, whatever :attr:`path` says."""
        freqs, out, F, ret, flags = self._stage(freqs, out, self.R)
        check(load().fastfp_fp_sweep_residuals(self._h, _vp(freqs), F, _vp(out), flags, C.c_void_p(stream)))
        return ret

    def nmfp_sweep(self, freqs, phiinv_var, D: int, out=None, stream: int = 0):
        freqs, out, F, ret, flags = self._stage(freqs, out, D)
        if isinstance(phiinv_var, np.ndarray):
            phiinv_var = as_f64(phiinv_var)
        else:
            flags |= PARAMS_ON_DEVICE
        check(load().fastfp_nmfp_sweep(self._h, _vp(freqs), F, _vp(phiinv_var), D, _vp(out), flags,
                                       C.c_void_p(stream)))
        return ret

    # the two halves of nmfp_sweep as separate calls (device pointers only): parallel.py shards them in two dimensions
    def nmfp_tile_sizes(self):
        """doubles per 32-frequency tile (all pulsars) of the two stage-A outputs"""
        z, a = C.c_int64(0), C.c_int64(0)
        check(load().fastfp_nmfp_tile_sizes(self._h, C.byref(z), C.byref(a)))
        return int(z.value), int(a.value)

    def nmfp_stage_a(self, freqs_ptr: int, F: int, z_ptr: int, a_ptr: int, stream: int = 0):
        check(load().fastfp_nmfp_stage_a(self._h, C.c_void_p(freqs_ptr), F, C.c_void_p(z_ptr), C.c_void_p(a_ptr),
                                         C.c_void_p(stream)))

    def nmfp_stage_b(self, freqs_ptr: int, F: int, z_ptr: int, a_ptr: int, tiles_per_block: int, phiinv_ptr: int,
                     D: int, out_ptr: int, stream: int = 0):
        check(load().fastfp_nmfp_stage_b(self._h, C.c_void_p(freqs_ptr), F, C.c_void_p(z_ptr), C.c_void_p(a_ptr),
                                         tiles_per_block, C.c_void_p(phiinv_ptr), D, C.c_void_p(out_ptr),
                                         C.c_void_p(stream)))

    def powerlaw_phiinv(self, Ffreqs, log10_A, gamma, curn_Ffreqs, curn_log10_A, curn_gamma, out_dev, stream=0):
        """Device-side ``get_phiinv`` of the varying block for D draws (host params in)."""
        lib = load()
        Ff = [as_f64(a) for a in Ffreqs]
        A, G = as_f64(log10_A), as_f64(gamma)
        D = A.shape[0]
        if curn_Ffreqs is not None and len(curn_Ffreqs):
            cf, cA, cG = as_f64(curn_Ffreqs), as_f64(curn_log10_A), as_f64(curn_gamma)
            args = (_vp(cf), cf.shape[0], _vp(cA), _vp(cG))
        else:
            args = (C.c_void_p(0), 0, C.c_void_p(0), C.c_void_p(0))
        check(
            lib.fastfp_powerlaw_phiinv(
                self._h, _ptr_array(Ff), _vp(A), _vp(G), D, *args, C.c_void_p(int(out_dev)), C.c_void_p(stream)
            )
        )

    def stage_timing(self, enable: bool = True) -> None:
        """Bracket the three nmfp stages of later sweeps with CUDA events (measurement aid)."""
        check(load().fastfp_nmfp_stage_timing(self._h, int(bool(enable))))

    def stage_ms(self):
        """``(stage A, factor, stage B)`` milliseconds of the last timed nmfp sweep."""
        out = (C.c_double * 3)()
        check(load().fastfp_nmfp_stage_ms(self._h, out))
        return tuple(out)

    @property
    def mvar_total(self) -> int:
        return int(load().fastfp_pack_mvar_total(self._h))

    @property
    def nbytes(self) -> int:
        return int(load().fastfp_pack_bytes(self._h))

    def close(self):
        if self._h:
            load().fastfp_pack_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def tnt(Nvec, T, phiinv=None, device: int = 0, stream: int = 0) -> np.ndarray:
    """``T^T N^-1 T`` (``+ diag(phiinv)``) on the device; diagonal ``N`` given as the variance vector."""
    Nvec, T = as_f64(Nvec), as_f64(T)
    if T.ndim != 2 or Nvec.shape != (T.shape[0],):
        raise ValueError("tnt: shapes must be Nvec (n,), T (n, m)")
    ph = None
    if phiinv is not None:
        ph = as_f64(phiinv)
        if ph.shape != (T.shape[1],):
            raise ValueError("tnt: phiinv must have shape (m,)")
    lib = load()
    require_device()
    out = np.empty((T.shape[1], T.shape[1]))
    check(lib.fastfp_tnt(device, T.shape[0], T.shape[1], _vp(Nvec), _vp(T), _vp(ph) if ph is not None else None,
                         _vp(out), C.c_void_p(stream)))
    return out


def xcy(Nvec, T, sigma, x, y, device: int = 0, stream: int = 0) -> float:
    from . import blockn

    if blockn.is_block(Nvec):  # block-diagonal N: Sherman-Morrison on the host, same kernel
        nvec, T, sigma, x, y = as_f64(Nvec._nvec), as_f64(T), as_f64(sigma), as_f64(x), as_f64(y)
        if T.ndim != 2 or nvec.shape != (T.shape[0],) or x.shape != nvec.shape or y.shape != nvec.shape \
                or sigma.shape != (T.shape[1],) * 2:
            raise ValueError("get_xCy: shapes must be Nvec (n,), T (n,m), sigma (m,m), x (n,), y (n,)")
        B = blockn.BlockNvec(nvec, Nvec._slices, Nvec._jvec)
        xw, yw = as_f64(B.solve(x) * nvec), as_f64(B.solve(y) * nvec)
        lib = load()
        require_device()
        out = np.empty(1)
        check(lib.fastfp_xcy_blockn(device, T.shape[0], T.shape[1], _vp(nvec), _vp(T), _vp(sigma), _vp(x), _vp(xw),
                                    _vp(yw), _vp(out), C.c_void_p(stream)))
        return float(out[0])
    Nvec, T, sigma, x, y = as_f64(Nvec), as_f64(T), as_f64(sigma), as_f64(x), as_f64(y)
    if T.ndim != 2:
        raise ValueError("get_xCy: T must be 2-D (ntoa, nbasis)")
    n, m = T.shape
    if Nvec.shape != (n,) or x.shape != (n,) or y.shape != (n,) or sigma.shape != (m, m):
        raise ValueError("get_xCy: shapes must be Nvec (n,), T (n,m), sigma (m,m), x (n,), y (n,)")
    lib = load()
    require_device()
    out = np.empty(1)
    check(lib.fastfp_xcy(device, n, m, _vp(Nvec), _vp(T), _vp(sigma), _vp(x), _vp(y), _vp(out), C.c_void_p(stream)))
    return float(out[0])


def fp64_peak(kind: int = 0, iters: int = 20000, device: int = 0):
    lib = load()
    require_device()
    tf, ms = C.c_double(), C.c_double()
    check(lib.fastfp_fp64_peak(device, kind, iters, C.byref(tf), C.byref(ms)))
    return tf.value, ms.value


def kernel_launches() -> int:
    return int(load().fastfp_kernel_launches())


def device_bytes() -> int:
    """Device memory the library holds now, in bytes, over all packs and devices of this process."""
    return int(load().fastfp_device_bytes())
