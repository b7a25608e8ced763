"""Block-diagonal white noise (``EcorrKernelNoise``) for the Fp hot path.

The reference's ``get_xCy`` "does not apply for the case where N is block-diagonal"
(``fastfp/utils.py:29-31``; README to-do). Here ``N = diag(nvec) + sum_e jvec[e] * 1_e 1_e^T`` over
contiguous TOA slices (the layout of ``enterprise``'s ``ShermanMorrison`` object: ``_nvec``,
``_jvec``, ``_slices``) is a first-class input: pass a :class:`BlockNvec` (or any object with those
three attributes) in place of a 1-D ``Nvec``.

Host-side preparation (NumPy, one time per pack), everything else runs in the CUDA kernels:

* Sherman-Morrison: ``(N^-1 x)_i = x_i/nvec_i - beta_e * (sum_{i' in e} x_i'/nvec_i') / nvec_i`` with
  ``beta_e = jvec_e / (1 + jvec_e * sum_e 1/nvec)`` -- applied to the columns of ``T`` and to ``r``;
* TOAs are re-laid in groups of 4 so that every group belongs to one epoch (zero-weight padding);
  chunks of ``CI`` TOAs then see at most 8 epochs, each bound to one of 8 *slot* rows appended to the
  G tile, carrying ``sqrt(beta_e)/nvec_i``; a per-chunk mask says which slots end there. The sweep
  kernel accumulates ``sqrt(beta_e) * sum_e x_i/nvec_i`` in the slot rows on the MMA path and folds
  ``beta_e * A_x * A_y`` into the ``x^T N^-1 y`` sums when an epoch ends.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Sequence

import numpy as np


@dataclass
class BlockNvec:
    """``N = diag(nvec) + sum_e jvec[e] * ones((len_e, len_e))`` on ``slices[e]``."""

    nvec: np.ndarray
    slices: Sequence[slice]
    jvec: np.ndarray

    @property
    def _nvec(self):
        return self.nvec

    @property
    def _slices(self):
        return self.slices

    @property
    def _jvec(self):
        return self.jvec

    def dense(self) -> np.ndarray:
        N = np.diag(np.asarray(self.nvec, dtype=np.float64))
        for sl, j in zip(self.slices, self.jvec):
            N[sl, sl] += j
        return N

    def solve(self, X: np.ndarray) -> np.ndarray:
        """``N^-1 X`` by Sherman-Morrison (X: (n,) or (n, k))."""
        nvec = np.asarray(self.nvec, dtype=np.float64)
        X = np.asarray(X, dtype=np.float64)
        out = X / (nvec if X.ndim == 1 else nvec[:, None])
        idx, eid, offs = _epoch_index(self.slices)
        if idx.size:
            ninv = 1.0 / nvec
            jv = np.asarray(self.jvec, dtype=np.float64)
            beta = jv / (1.0 + jv * np.add.reduceat(ninv[idx], offs))
            sums = np.add.reduceat(out[idx], offs, axis=0)  # per-epoch sums of N_d^-1 X
            corr = (beta * sums if X.ndim == 1 else beta[:, None] * sums)[eid]
            out[idx] -= ninv[idx] * corr if X.ndim == 1 else ninv[idx, None] * corr
        return out


def _epoch_index(slices):
    """Concatenated TOA indices of all epochs, the epoch id of each, and the start offsets."""
    if len(slices) == 0:
        z = np.zeros(0, dtype=np.int64)
        return z, z, z
    starts = np.asarray([int(s.start) for s in slices], dtype=np.int64)
    lens = np.asarray([int(s.stop) - int(s.start) for s in slices], dtype=np.int64)
    offs = np.cumsum(lens) - lens
    eid = np.repeat(np.arange(len(slices), dtype=np.int64), lens)
    idx = np.arange(int(lens.sum()), dtype=np.int64) - offs[eid] + starts[eid]
    return idx, eid, offs


def is_block(Nvec) -> bool:
    return all(hasattr(Nvec, a) for a in ("_nvec", "_jvec", "_slices"))


@dataclass
class Epochs:
    """One pulsar's block-diagonal N as the layout and the Sherman-Morrison need it: the white variances ``nvec``,
    the epochs ``slices`` as ``(start, stop)``, ``beta_e = jvec_e / (1 + jvec_e * sum_e 1/nvec)`` and the epoch
    variances ``jvec`` (what a draw of the noise needs). A diagonal N has no epochs."""

    nvec: np.ndarray
    slices: List[tuple]
    beta: np.ndarray
    jvec: np.ndarray

    @property
    def n(self) -> int:
        return self.nvec.shape[0]


def epochs(Nvec, n: int) -> Epochs:
    """The :class:`Epochs` of a :class:`BlockNvec`-like object or a 1-D array (no epochs) for ``n`` TOAs."""
    if is_block(Nvec):
        nvec = np.asarray(Nvec._nvec, dtype=np.float64)
        slices = [(int(s.start), int(s.stop)) for s in Nvec._slices]
        jvec = np.asarray(Nvec._jvec, dtype=np.float64)
    else:
        nvec, slices, jvec = np.asarray(Nvec, dtype=np.float64), [], np.zeros(0)
    if nvec.shape != (n,):
        raise ValueError("block N: nvec must have one entry per TOA")
    covered = np.zeros(n, dtype=bool)
    for (a, b) in slices:
        if not 0 <= a < b <= n or covered[a:b].any():
            raise ValueError("block N: slices must be non-empty, in range and disjoint")
        covered[a:b] = True
    beta = np.zeros(len(slices))
    if slices:
        idx, eid, offs = _epoch_index([slice(a, b) for a, b in slices])
        beta = jvec / (1.0 + jvec * np.add.reduceat(1.0 / nvec[idx], offs))
    return Epochs(nvec, slices, beta, jvec)


def solve_rows(ep: Epochs, X) -> np.ndarray:
    """Sherman-Morrison of the ``R`` rows of ``X`` (``(R, n)``) at once, expressed as ``(N^-1 x_k) * nvec`` so the
    kernels' ``x/N`` recovers ``N^-1 x_k``: the ``res_w`` of :func:`prepare`, row by row and bit for bit."""
    X = np.asarray(X, dtype=np.float64)
    out = X.copy()
    if ep.slices:
        idx, eid, offs = _epoch_index([slice(a, b) for a, b in ep.slices])
        ninv = 1.0 / ep.nvec
        out[:, idx] -= (ep.beta * np.add.reduceat(X[:, idx] * ninv[idx], offs, axis=1))[:, eid]
    return out


def layout(ep: Epochs, CI: int) -> dict:
    """The TOA order of a block-N pack whose kernel takes chunks of ``CI`` TOAs, and its epoch slots.

    TOAs are laid out as the epochs, each padded to a multiple of 4, then the TOAs outside any epoch, 4 at a time, then
    padding k-blocks up to a multiple of ``CI``. Only that padded tail depends on ``CI``: two layouts of one pulsar agree
    position by position on every real TOA (the residual batches of a block-N pack rely on it). Returns ``order``
    (original TOA index, -1 for padding), ``slot_idx`` (slot 0..7 of a TOA's epoch inside its chunk, -1 if none),
    ``slot_val`` (``sqrt(beta_e) / nvec_i``) and ``done_mask`` (per chunk, the slots whose epoch ends there)."""
    n, slices, beta, nvec = ep.n, ep.slices, ep.beta, ep.nvec
    covered = np.zeros(n, dtype=bool)
    for (a, b) in slices:
        covered[a:b] = True
    # groups of TOAs: epochs (padded to multiples of 4) then the uncovered TOAs, 4 at a time
    KB = CI // 4
    order: List[int] = []          # original TOA index or -1 (padding), length 4 * number of k-blocks
    kb_epoch: List[int] = []       # epoch of each k-block, -1 = none
    for e, (a, b) in enumerate(slices):
        idx = list(range(a, b))
        idx += [-1] * (-len(idx) % 4)
        order += idx
        kb_epoch += [e] * (len(idx) // 4)
    free = list(np.nonzero(~covered)[0])
    free += [-1] * (-len(free) % 4)
    order += free
    kb_epoch += [-1] * (len(free) // 4)
    pad_kb = -len(kb_epoch) % KB
    order += [-1] * (4 * pad_kb)
    kb_epoch += [-1] * pad_kb
    nkb = len(kb_epoch)
    nch = nkb // KB
    # slot assignment: an epoch keeps one slot for all its k-blocks, also across chunk boundaries
    slot_of_kb = np.full(nkb, -1, dtype=np.int32)
    done = np.zeros(nch, dtype=np.uint8)
    last_kb = {}
    for kbi, e in enumerate(kb_epoch):
        if e >= 0:
            last_kb[e] = kbi
    carry = {}  # epoch -> slot, for epochs that continue into the next chunk
    for c in range(nch):
        used = dict(carry)
        free_slots = [s for s in range(8) if s not in used.values()]
        for kbi in range(c * KB, (c + 1) * KB):
            e = kb_epoch[kbi]
            if e < 0:
                continue
            if e not in used:
                used[e] = free_slots.pop(0)
            slot_of_kb[kbi] = used[e]
        carry = {}
        for e, s in used.items():
            if last_kb[e] < (c + 1) * KB:
                done[c] |= np.uint8(1 << s)
            else:
                carry[e] = s
    order = np.asarray(order, dtype=np.int64)
    real = order >= 0
    slot_idx = np.repeat(slot_of_kb, 4).astype(np.int32)
    slot_idx[~real] = -1
    slot_val = np.zeros(order.shape[0])
    ep_of_toa = np.repeat(np.asarray(kb_epoch), 4)
    sel = real & (ep_of_toa >= 0)
    slot_val[sel] = np.sqrt(beta[ep_of_toa[sel]]) / nvec[order[sel]]
    slot_idx[~sel] = -1
    return dict(order=order, slot_idx=np.ascontiguousarray(slot_idx), slot_val=slot_val,
                done_mask=np.ascontiguousarray(done))


def relay(order, X) -> np.ndarray:
    """The columns of ``X`` (``(..., n)``) in the TOA order ``order`` of :func:`layout`, zero at padding."""
    X = np.asarray(X, dtype=np.float64)
    real = order >= 0
    out = np.zeros(X.shape[:-1] + order.shape)
    out[..., real] = X[..., order[real]]
    return out


def prepare(toas, res, Nvec, T, CI: int):
    """Lay one pulsar out for a block-N pack. ``Nvec`` is a :class:`BlockNvec`-like object or a
    1-D array (no epochs). Returns a dict of the arrays ``fastfp_pack_create_blockn`` takes."""
    toas, res, T = (np.asarray(a, dtype=np.float64) for a in (toas, res, T))
    n, m = T.shape
    ep = epochs(Nvec, n)
    nvec, ninv = ep.nvec, 1.0 / ep.nvec
    # Sherman-Morrison applied to T and r, expressed as (N^-1 x) * nvec so the kernels' x/N recovers it
    Tw = T.copy()
    if ep.slices:
        idx, eid, offs = _epoch_index([slice(a, b) for a, b in ep.slices])
        Tw[idx] -= (ep.beta[:, None] * np.add.reduceat(T[idx] * ninv[idx, None], offs, axis=0))[eid]
    rw = solve_rows(ep, res[None])[0]
    lay = layout(ep, CI)
    order = lay["order"]
    real = order >= 0
    out_n = np.full(order.shape[0], np.inf)
    out_n[real] = nvec[order[real]]
    out_T = np.zeros((order.shape[0], m))
    out_T[real] = Tw[order[real]]
    return dict(toas=relay(order, toas), res=relay(order, res), res_w=relay(order, rw), Nvec=out_n,
                T=np.ascontiguousarray(out_T), slot_idx=lay["slot_idx"], slot_val=lay["slot_val"],
                done_mask=lay["done_mask"])
