"""``FastFp`` -- drop-in for the reference's ``fastfp.fastfp.FastFp`` (``fastfp/fastfp.py:22-101``).

Same constructor and call signatures; the JAX/XLA program behind ``calculate_Fp`` is replaced
by the sm_90a sweep kernel of ``libfastfp_b200.so`` reached through the C ABI. Differences a
caller can see, all additive:

* ``fgw`` may be a scalar (reference semantics, returns a float) **or** a 1-D array of
  frequencies (returns ``(F,)``) -- what the reference obtains with
  ``jax.vmap(calculate_Fp, in_axes=(0, None, None, None))`` (``examples/run_fp.py:63``);
  :func:`fastfp_b200.vmap` keeps that spelling working too.
* ``fgw`` may be a float64 CUDA ``torch.Tensor``; the result is then a CUDA tensor and nothing
  crosses PCIe (the sweep is enqueued on torch's current stream).
* ``compute_Fp`` is an alias of ``calculate_Fp`` (the name ``enterprise_extensions``' ``FpStat``
  uses, cited at ``fastfp/fastfp.py:27-28``).

No validation beyond shapes is added: NaN/Inf propagate silently exactly as in the reference.
"""
from __future__ import annotations

import os

import numpy as np

from . import _cabi
from ._cabi import _is_cuda_tensor


def _fingerprint(lists) -> tuple:
    """Content key of the caller's lists: shape + a 64-bit hash of EVERY byte of every array
    (``fastfp_hash64``: memory-bandwidth class, threaded for large arrays). The reference is a pure function
    of these arguments (``fastfp/fastfp.py:52``), so the cached device pack must be rebuilt whenever any
    entry changes -- including in-place edits, which an address- or sample-based key cannot see."""
    key, arrays, seeds, slots = [], [], [], []
    for lst in lists:
        key.append(len(lst))
        for a in lst:
            parts = [a._nvec, a._jvec, np.asarray([(s.start, s.stop) for s in a._slices], dtype=np.int64)] \
                if hasattr(a, "_nvec") else [a]
            for x in parts:
                x = np.ascontiguousarray(x)
                slots.append(len(key))
                seeds.append(len(key))
                arrays.append(x)
                key.append((x.shape, x.dtype.str))
    for slot, h in zip(slots, _cabi.hash64_many(arrays, seeds)):  # one call: all arrays share the hashing threads
        key[slot] = key[slot] + (h,)
    return tuple(key)


def _shape_key(lists) -> tuple:
    """Cheap structural key (lengths and shapes only): decides whether the cached pack can even be tried."""
    key = []
    for lst in lists:
        key.append(len(lst))
        for a in lst:
            key.append((np.shape(a._nvec), len(a._slices)) if hasattr(a, "_nvec") else np.shape(a))
    return tuple(key)


_HASHER = None


def _hasher():
    """One worker thread for the content hash (the ctypes calls release the GIL)."""
    global _HASHER
    if _HASHER is None:
        from concurrent.futures import ThreadPoolExecutor

        _HASHER = ThreadPoolExecutor(max_workers=1, thread_name_prefix="fastfp-hash")
    return _HASHER


class _PackCache:
    """The device pack is a CACHE of the caller's lists; the reference is a pure function of them. Every call
    hashes every byte of the lists. To keep that off the critical path the sweep is started on the cached pack
    right away while the hash runs on a worker thread (or, for asynchronous device-resident calls, on this thread
    after the launch); if the hash shows the inputs changed, the pack is rebuilt and the sweep repeated -- the
    caller never sees a result computed from stale data.

    It also holds what the front ends share: the pulsars' TOAs and residuals, the device (default ``LOCAL_RANK``
    or 0) and the sweep path (default ``FASTFP_B200_PATH`` or "auto"), resolved at construction."""

    _pack = None
    _pack_key = None
    _pack_shape = None

    def __init__(self, psrs, device=None, path=None):
        self.toas = [np.asarray(psr.toas, dtype=np.float64) for psr in psrs]
        self.residuals = [np.asarray(psr.residuals, dtype=np.float64) for psr in psrs]
        self.device = int(os.environ.get("LOCAL_RANK", "0")) if device is None else int(device)
        self.path = path if path is not None else os.environ.get("FASTFP_B200_PATH", "auto")
        if self.path not in ("auto", "fp64", "i8", "prefer-i8"):
            raise ValueError("path must be 'auto', 'fp64', 'i8' or 'prefer-i8'")

    def invalidate(self):
        """Drop the cached device pack (the next call rebuilds it)."""
        if self._pack is not None:
            self._pack.close()
        self._pack, self._pack_key, self._pack_shape = None, None, None

    def _build_pack(self, lists):  # -> _cabi.Pack
        raise NotImplementedError

    def _create_pack(self, Nvecs, Ts, mats, m_fix=None, phiinv_fix=None):
        """``_cabi.Pack.create`` on this object's pulsars and device, set to its sweep path."""
        pack = _cabi.Pack.create(self.toas, self.residuals, Nvecs, Ts, mats, m_fix, phiinv_fix, device=self.device)
        if self.path == "prefer-i8":  # the tensor kernel where the pack can take it, silently the fp64 one otherwise
            for p in ("i8", "mixed"):
                try:
                    pack.set_path(p)
                    break
                except _cabi.FastFpError:
                    pass
        elif self.path != "auto":
            pack.set_path(self.path)
        return pack

    def _device_freqs(self, fgw):
        """A CUDA-tensor ``fgw`` as a flat contiguous tensor on the pack's device, and torch's current stream there."""
        import torch

        if fgw.dtype != torch.float64:
            raise TypeError("fgw tensor must be float64 (the reference enables jax x64)")
        if fgw.device.index != self.device:
            raise ValueError(f"fgw is on {fgw.device}, the pack on cuda:{self.device}")
        return fgw.contiguous().reshape(-1), torch.cuda.current_stream(fgw.device).cuda_stream

    def _front_end(self, fgw):
        """What a front end hands the pack for ``fgw``: the flat float64 frequencies, ``empty(shape, dtype=float64)``
        for its outputs, the stream and whether the call is asynchronous. A CUDA tensor stays on its device: outputs
        from ``torch.empty`` there, torch's current stream, asynchronous. Host values: ``np.empty``, stream 0, and the
        call returns with the results on the host."""
        if _is_cuda_tensor(fgw):
            import torch

            f, stream = self._device_freqs(fgw)

            def empty(shape, dtype=np.float64):
                return torch.empty(shape, dtype=getattr(torch, np.dtype(dtype).name), device=f.device)

            return f, empty, stream, True
        return np.asarray(fgw, dtype=np.float64).reshape(-1), np.empty, 0, False

    def _ensure(self, lists, force=False, key=None):
        key = _fingerprint(lists) if key is None else key
        if force or self._pack is None or key != self._pack_key:
            if self._pack is not None:
                self._pack.close()
                self._pack = None
            self._pack = self._build_pack(lists)
            self._pack_key, self._pack_shape = key, _shape_key(lists)
        return self._pack

    def _run_verified(self, lists, run, asynchronous):
        """``run(pack)`` on a pack that is verified to match ``lists`` byte for byte."""
        if self._pack is None or _shape_key(lists) != self._pack_shape:
            return run(self._ensure(lists))
        if asynchronous:  # the launch returns at once: hash here while the GPU works
            res = run(self._pack)
            key = _fingerprint(lists)
        else:             # the call blocks until the result is on the host: hash on the worker meanwhile
            fut = _hasher().submit(_fingerprint, lists)
            try:
                res = run(self._pack)
            finally:
                key = fut.result()
        if key == self._pack_key:
            return res
        return run(self._ensure(lists, key=key))  # the inputs changed: rebuild, repeat


def _tile_cost(rows: int) -> float:
    """Modelled cost of one residual pass per (frequency, TOA): the padded width MP that ``sweep_config`` gives ``rows`` G
    rows, times a per-row factor. On an H100 a tile row costs about the same in every configuration measured (0.49-0.51
    ms per row at C2 shapes for 40 to 384 rows) except the 8-frequency family with 10 row blocks per warp (640 rows),
    which costs 1.3-1.5 times as much per row (DESIGN.md section 5d). That family was measured at 6 row blocks (384
    rows, no extra cost) and at 10; the 7 to 9 blocks in between were not measured and are given the 10-block factor.
    These costs were measured with a diagonal N; block-N passes (8 more rows, the epoch slots, folded per epoch) are
    modelled with the same factors, which is not measured."""
    for top, per_block in ((40, 8), (80, 8), (160, 16), (320, 32), (640, 64)):
        if rows <= top:
            nmbw = -(-rows // per_block)
            return nmbw * per_block * (1.4 if top == 640 and nmbw >= 7 else 1.0)
    raise ValueError(f"{rows} rows exceed the sweep kernel")


def batch_pass_rows(R: int, m, blockn: bool = False) -> int:
    """Realisations per pass of :meth:`FastFp.calculate_Fp_batch` for ``R`` realisations of pulsars of basis widths
    ``m``: of the even splits of ``R`` into passes the library takes (at most ``_cabi.max_residual_rows`` rows each),
    the one with the least modelled cost, passes x :func:`_tile_cost` of ``roundup8(max m) + roundup8(rows)`` rows
    (``+ 8``, the epoch slots, for a block-diagonal N pack: ``blockn=True``); among equal costs the fewest passes."""
    rmax = _cabi.max_residual_rows(m, blockn)
    best = None
    for cap in sorted({min(R, rmax)} | set(range(8, min(R, rmax), 8))):
        npass = -(-R // cap)
        rows = -(-R // npass)
        cost = npass * _tile_cost(_cabi.sweep_rows(max(m), rows, blockn))
        if best is None or (cost, npass) < best[:2]:
            best = (cost, npass, rows)
    return best[2]


class FastFp(_PackCache):
    """Fp-statistic (Ellis, Siemens & Creighton 2012) for a list of pulsars.

    :param psrs: objects with ``.toas`` and ``.residuals`` (seconds) -- all the reference reads
        (``fastfp/fastfp.py:44-45``)
    :param pta: stored and never used in compute, as in the reference (``fastfp.py:42``)
    :param device: CUDA device ordinal (extension; default 0 or ``LOCAL_RANK``)
    :param path: which kernel sweeps (extension): ``"auto"`` (default; also from ``FASTFP_B200_PATH``) = the
        fp64 DMMA kernel, the faster one on an H100; ``"prefer-i8"`` = the INT8 tensor-core kernel (``wgmma``,
        exact digit-plane product) for every pulsar that fits its tile, the fp64 kernel for the rest;
        ``"fp64"`` / ``"i8"`` force one (``"i8"`` raises if the pack cannot take it).
        Both meet the same parity bar; see DESIGN.md.
    """

    def __init__(self, psrs, pta=None, device=None, path=None):
        self.psrs = psrs
        self.pta = pta
        super().__init__(psrs, device, path)

    # -- packing (one-time, frequency-independent precompute on the device) -----------------
    def _build_pack(self, lists):
        return self._create_pack(*lists)

    def prepare(self, Nvecs, Ts, sigmas, force=False):
        """Upload and pre-reduce the per-pulsar arrays. The pack is cached and keyed on the full contents
        of the three lists (every byte is hashed on each call), so passing different arrays -- or the same
        arrays edited in place -- rebuilds it; ``force=True`` rebuilds unconditionally."""
        return self._ensure((Nvecs, Ts, sigmas), force=force)

    def __call__(self, fgw, Nvecs, Ts, sigmas):
        """Callable method (reference ``fastfp.py:47-49``)."""
        return self.calculate_Fp(fgw, Nvecs, Ts, sigmas)

    def calculate_Fp(self, fgw, Nvecs, Ts, sigmas):
        """Fp at ``fgw`` (reference ``fastfp.py:51-92``); see the module docstring for the
        batched forms of ``fgw``."""
        f, empty, stream, on_device = self._front_end(fgw)
        out = empty(f.shape[0])

        def run(pack):
            pack.fp_sweep(f, out=out, stream=stream)
            return out

        res = self._run_verified((Nvecs, Ts, sigmas), run, asynchronous=on_device)
        return res.reshape(np.shape(fgw))[()]  # a scalar fgw: a numpy scalar from host values, a 0-d tensor from a tensor

    compute_Fp = calculate_Fp

    def calculate_Fp_batch(self, fgw, Nvecs, Ts, sigmas, residuals):
        """Fp at ``fgw`` for each of ``R`` realisations of the residuals (simulated noise for a false-alarm
        calibration, injected signals for a detection study), with the pulsars, noise model and basis of
        ``Nvecs, Ts, sigmas``. ``residuals`` is a list of ``P`` arrays of shape ``(R, n_p)``; row ``k`` of the result
        is the Fp :meth:`calculate_Fp` gives with residuals ``residuals[p][k]``: ``(R,)`` for a scalar ``fgw``,
        ``(R, *fgw.shape)`` for an array, a CUDA tensor on torch's current stream for a float64 CUDA tensor (so
        ``parallel.sharded_sweep(..., lead_shape=(R,))`` spreads it over several GPUs).

        The realisations ride along as extra rows of the fp64 sweep kernel (``fastfp_fp_sweep_residuals``, whatever
        ``path`` says). Values meet the parity bar of :meth:`calculate_Fp` but are not bit-identical to it. The set is
        cached on the pack and uploaded again when any byte of ``residuals`` changes. A set of several passes is
        uploaded pass by pass on every call, and each upload synchronises the stream, so with a CUDA-tensor ``fgw``
        such a call returns only when its last pass has been launched and is not asynchronous; the content hash of
        ``residuals`` is also taken on the calling thread before the first launch. The library takes at most ``_cabi.max_residual_rows`` rows per pass (568
        at m = 72, 560 with a block-diagonal N); ``R`` is split into passes of :func:`batch_pass_rows` rows, the split with the least modelled
        sweep cost (measured per-row costs of the kernel configurations). The pass size selects the kernel configuration, so values can differ in the last bits
        between different ``R``; within one ``R`` every row is computed alike wherever it sits.

        A block-diagonal N (a ``BlockNvec`` or enterprise ``ShermanMorrison`` among the ``Nvecs``) works the same way:
        the realisations, in the pulsars' original TOA order, are laid out by epoch and given the Sherman-Morrison
        ``N^-1`` on the host (``_cabi.Pack.set_residuals_blockn``)."""
        R, passes = self._residual_passes(residuals)
        f, empty, stream, on_device = self._front_end(fgw)
        out = empty((R, f.shape[0]))

        def run(pack):
            for lo, hi in passes(pack, stream):
                pack.fp_sweep_residuals(f, out=out[lo:hi], stream=stream)
            return out

        return self._run_verified((Nvecs, Ts, sigmas), run, asynchronous=on_device).reshape((R,) + np.shape(fgw))

    def calculate_Fp_simulated(self, fgw, Nvecs, Ts, sigmas, phiinvs, R, seed, first=0, signal=None, noise=True):
        """:meth:`calculate_Fp_batch` on ``R`` realisations of the noise model of ``Nvecs, Ts, sigmas`` drawn on the
        device: row ``k`` is realisation ``first + k`` of the stream of ``seed``, the residuals ``n + T Phi^(1/2)
        zeta`` (white noise, ECORR epoch terms for a block-diagonal N, the basis with prior ``1/phiinvs``) plus an
        optional Earth-term signal. Nothing is drawn or uploaded per realisation on the host
        (``fastfp_pack_simulate_residuals``; DESIGN.md section 5g). :func:`fastfp_b200.sim.simulate_residuals` gives
        the same realisations on the host.

        ``phiinvs[p]`` is the ``(m_p,)`` prior ``1/phi`` that went into ``sigmas[p]`` (``pta.get_phiinv``); ``seed``
        and ``first`` are integers ``>= 0``. ``signal = (freqs, amp)``: ``freqs`` a scalar or ``(R,)``, ``amp``
        ``(P, 2)`` or ``(R, P, 2)``, each pulsar's ``(A_s, A_c)`` of ``A_s sin(2 pi f t) + A_c cos(2 pi f t)``
        (:meth:`FastFe.cw_signal` builds it from the Fe amplitudes); ``noise=False`` sweeps the signal alone. The
        result has the shape and device semantics of :meth:`calculate_Fp_batch`, and is computed in passes of
        :func:`batch_pass_rows` rows the same way; a realisation is the same whatever ``R``, ``first`` or pass split
        drew it."""
        R, passes = self._simulated_passes(Ts, phiinvs, R, seed, first, signal, noise)
        f, empty, stream, on_device = self._front_end(fgw)
        out = empty((R, f.shape[0]))

        def run(pack):
            for lo, hi in passes(pack, stream):
                pack.fp_sweep_residuals(f, out=out[lo:hi], stream=stream)
            return out

        return self._run_verified((Nvecs, Ts, sigmas), run, asynchronous=on_device).reshape((R,) + np.shape(fgw))

    def _residual_passes(self, residuals):
        """Checks the shapes of ``residuals`` (a list of ``P`` arrays ``(R, n_p)``) and returns ``(R, passes)`` of
        :meth:`_passes` that upload them."""
        res, R = _cabi.check_realisations(residuals, [t.shape[0] for t in self.toas])
        if R < 1:
            raise ValueError("residuals must hold at least one realisation")

        def upload(pack, lo, hi, stream):
            fn = pack.set_residuals_blockn if getattr(pack, "blockn", False) else pack.set_residuals
            fn([r[lo:hi] for r in res], stream=stream)

        return R, self._passes(R, ("uploaded", _fingerprint([res])), upload)

    def _simulated_passes(self, Ts, phiinvs, R, seed, first, signal, noise):
        """Checks the arguments of a simulated batch and returns ``(R, passes)`` of :meth:`_passes` that draw it."""
        from . import sim

        if isinstance(R, (bool, np.bool_)) or not isinstance(R, (int, np.integer)) or R < 1:
            raise ValueError("R must be an integer >= 1")
        R = int(R)
        seed, first = sim.check_seed(seed, first)
        if first > 2 ** 63 - 1 - R:
            raise ValueError("first + R must stay below 2^63")
        if len(Ts) != len(self.toas):
            raise ValueError(f"Ts must be a list of {len(self.toas)} arrays (one per pulsar)")
        phi = sim.check_phiinvs(phiinvs, [np.shape(T)[1] for T in Ts])
        freqs, amp = sim.signal_arrays(signal, R, len(self.toas))
        sig = [] if freqs is None else [freqs, amp]
        key = ("simulated", seed, first, bool(noise), freqs is None, _fingerprint([phi, sig]))

        def upload(pack, lo, hi, stream):
            fn = pack.simulate_residuals_blockn if getattr(pack, "blockn", False) else pack.simulate_residuals
            part = None if freqs is None else (freqs[lo:hi], amp[lo:hi])
            fn(hi - lo, seed, phi, first=first + lo, signal=part, noise=noise, stream=stream)

        return R, self._passes(R, key, upload)

    def _passes(self, R, key, upload):
        """``passes(pack, stream=0)`` yields the row ranges ``(lo, hi)`` of :func:`batch_pass_rows` passes with each
        pass's realisations set on ``pack`` by ``upload(pack, lo, hi, stream)``, again only when the pack or ``key``
        (the content of the set: an uploaded set and a simulated set never share one) changed."""

        def passes(pack, stream=0):
            blockn = getattr(pack, "blockn", False)  # a pack without the attribute has a diagonal N
            rows = batch_pass_rows(R, pack.m, blockn)
            for lo in range(0, R, rows):
                hi = min(R, lo + rows)
                if self._res_pack is not pack or self._res_key != (key, lo, hi):
                    self._res_pack, self._res_key = None, None
                    upload(pack, lo, hi, stream)
                    self._res_pack, self._res_key = pack, (key, lo, hi)
                yield lo, hi

        return passes

    _res_pack = None
    _res_key = None

    def per_pulsar_terms(self, fgw, Nvecs, Ts, sigmas):
        """``0.5 * N^T M^-1 N`` per pulsar, ``(P, F)`` -- the summands of ``fastfp.py:90``."""
        pack = self.prepare(Nvecs, Ts, sigmas)
        return pack.fp_sweep(np.atleast_1d(np.asarray(fgw, dtype=np.float64)), terms=True)

    # pytree protocol of the reference (fastfp.py:94-101), kept so code that flattens the
    # object keeps working; there is no tracing here.
    def tree_flatten(self):
        return (), (self.psrs, self.pta)

    @classmethod
    def tree_unflatten(cls, aux_data, children):
        return cls(*aux_data, *children)
