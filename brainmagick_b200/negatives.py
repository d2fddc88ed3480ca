"""Drop-in negative pool: the solver's `optim.negatives` / `optim.negative_pool_size` (bm/solver.py:152-164, 358-371),
kept on the device and scored in place by the CLIP kernels.

The reference keeps one CPU tensor per phase and, before every loss call whose batch holds fewer than `negatives` rows,
copies the batch to the host, gathers `negatives - B` random pool rows, copies them back to the device and writes a new
pool tensor.  Here the pool's rows live in one fp32 device buffer per phase, the logical pool is a host list of row slots,
and each call only writes the B new rows (`bm_scatter_rows`).  `complete` returns a `PooledCandidates` that the drop-in
`ClipLoss` scores where the rows lie (`bm_clip_loss_fwd_pooled` / `bm_clip_loss_bwd_pooled`), with no gather or `cat` copy.

Reference semantics kept: `torch.randperm(len(pool))` on the CPU default generator at the same point in the step; the
candidates `[output; pool[kept]]`; the new pool `[output; pool[kept]; old pool][:negative_pool_size]`, newest first, so
re-drawn rows are prepended again and may come back as duplicates; no gradient through the candidates whenever the pool
code runs (the reference's `cat` is under `torch.no_grad()`); `output` itself, with its gradient, when it already holds
`negatives` rows; no checkpointing (the reference's pool is not in the solver's stateful attributes).
"""
from __future__ import annotations

import typing as tp
import weakref

import numpy as np
import torch

from . import functional as BF

PHASES = ("train", "valid")


class PooledCandidates:
    """The candidates `[output; pool[kept]]` of one step, without the concatenation: the batch rows (the `output` tensor,
    read in place), the phase's device storage and an int32 device table of the drawn slots.  It answers like the
    reference's concatenated tensor for `shape`, `size()`, `len()`, `device`, `dtype` and `requires_grad` (False: the
    reference builds it under no_grad), and `materialize()` returns that tensor.  While it lives, and while an autograd
    graph that saved it has not run its backward, the slots it reads are never overwritten."""

    def __init__(self, batch: torch.Tensor, storage: torch.Tensor, slots: torch.Tensor, host_slots: np.ndarray):
        self.batch = batch
        self.storage = storage
        self.slots = slots
        self.host_slots = host_slots            # the same table on the host: the lease the pool reads
        self.shape = torch.Size((batch.shape[0] + len(host_slots),) + tuple(batch.shape[1:]))

    def size(self, dim: tp.Optional[int] = None):
        return self.shape if dim is None else self.shape[dim]

    def dim(self) -> int:
        return len(self.shape)

    def __len__(self) -> int:
        return self.shape[0]

    @property
    def device(self) -> torch.device:
        return self.batch.device

    @property
    def dtype(self) -> torch.dtype:
        return self.batch.dtype

    @property
    def requires_grad(self) -> bool:
        return False

    @property
    def row_elems(self) -> int:
        return self.batch[0].numel() if self.batch.shape[0] else int(np.prod(self.shape[1:]))

    def materialize(self) -> torch.Tensor:
        """The reference's `torch.cat([output, buf[kept]])`: the batch rows copied, the pool rows gathered on the device."""
        out = torch.empty(self.shape, dtype=self.dtype, device=self.device)
        bb = self.batch.shape[0]
        out[:bb].copy_(self.batch)
        n = len(self.host_slots)
        if n:
            BF.call("bm_gather_rows", BF.ptr(self.storage), BF.ptr(self.slots), n, self.row_elems, BF.ptr(out[bb:]),
                    BF.stream())
        return out


class _Phase:
    """One phase's pool: the device rows, the logical pool (slot ids, newest first, repeats allowed) and the live
    PooledCandidates whose slots must stay untouched."""

    def __init__(self):
        self.storage: tp.Optional[torch.Tensor] = None
        self.slots = np.empty(0, dtype=np.int32)
        self.leases: "weakref.WeakSet[PooledCandidates]" = weakref.WeakSet()

    def free_slots(self, keep: np.ndarray, n: int) -> np.ndarray:
        """n slots that neither `keep` nor a live PooledCandidates holds, lowest first; grows the storage (a reallocation
        and a device copy) when there are fewer."""
        cap = self.storage.shape[0]
        used = np.zeros(cap, dtype=bool)
        used[keep] = True
        for lease in list(self.leases):
            used[lease.host_slots[lease.host_slots < cap]] = True
        free = np.flatnonzero(~used)
        if len(free) < n:
            grown = torch.empty((cap + n - len(free),) + tuple(self.storage.shape[1:]), dtype=self.storage.dtype,
                                device=self.storage.device)
            grown[:cap].copy_(self.storage)
            self.storage = grown                # live PooledCandidates keep reading the old buffer
            free = np.concatenate([free, np.arange(cap, grown.shape[0])])
        return free[:n].astype(np.int32)


class NegativePool:
    """Drop-in for `Solver._make_negative_pool` (bm/solver.py:152-164) and the negatives block of `_run_one_epoch`
    (bm/solver.py:358-371):

        self.negative_pool = NegativePool(args.optim.negatives, args.optim.negative_pool_size)
        ...
        output = self.negative_pool.complete(output, training)
        loss = self.loss(estimate, output, features_mask)      # the drop-in ClipLoss

    Each phase's device storage holds `negative_pool_size + negatives - 1` rows, allocated on the phase's first pooled
    step: enough for the pool and one step's new rows, so the solver's loop never reallocates it.  Holding several
    PooledCandidates alive at once (two forwards before either backward) grows it.  The row shape is fixed by the first
    call; another shape raises the reference's `torch.cat` error.  Nothing here reads the device on the host."""

    def __init__(self, negatives: tp.Optional[int], negative_pool_size: tp.Optional[int] = None):
        if negatives is not None:
            if negative_pool_size is None:
                negative_pool_size = 2 * negatives
            assert negative_pool_size >= negatives, "Pool of negatives should be larger than the number of negatives"
        self.negatives = negatives
        self.negative_pool_size = negative_pool_size
        self._phases = {name: _Phase() for name in PHASES}
        self._row_shape: tp.Optional[tp.Tuple[int, ...]] = None

    def _check_rows(self, output: torch.Tensor) -> None:
        if self._row_shape is None:
            if output.dtype != torch.float32:
                raise TypeError(f"the negative pool holds fp32 rows for the ClipLoss kernels, got {output.dtype}")
            self._row_shape = tuple(output.shape[1:])
        elif tuple(output.shape[1:]) != self._row_shape or output.dtype != torch.float32:
            # what the reference's torch.cat([output, buf[kept]]) raises for these shapes
            torch.cat([torch.empty((0,) + tuple(output.shape[1:]), dtype=output.dtype),
                       torch.empty((1,) + self._row_shape)])
            raise TypeError(f"the negative pool holds fp32 rows, got {output.dtype}")

    def complete(self, output: torch.Tensor, training: bool):
        """`output` itself when no pool applies (negatives None, or at least `negatives` rows); otherwise the candidates
        `[output; pool[kept]]` as a PooledCandidates, after adding them to the phase's pool."""
        if self.negatives is None or len(output) >= self.negatives:
            return output
        if BF.capturing():
            raise RuntimeError("a negative pool step cannot be captured in a CUDA graph: the slot table is built on the "
                               "host and the candidate count grows while the pool fills")
        self._check_rows(output)
        phase = self._phases["train" if training else "valid"]
        batch = output.detach().contiguous()
        B = batch.shape[0]
        kept = torch.randperm(len(phase.slots))[:self.negatives - B].numpy()     # solver.py:365, the CPU generator
        kept_slots = phase.slots[kept]
        if phase.storage is None:
            phase.storage = torch.empty((self.negative_pool_size + self.negatives - 1,) + self._row_shape,
                                        dtype=torch.float32, device=batch.device)
        retained = np.concatenate([kept_slots, phase.slots])[:max(0, self.negative_pool_size - B)]
        new_slots = phase.free_slots(np.concatenate([retained, kept_slots]), B)
        phase.slots = np.concatenate([new_slots, retained])[:self.negative_pool_size]
        table = torch.from_numpy(np.concatenate([kept_slots, new_slots]).astype(np.int32))
        if batch.is_cuda:
            table = table.pin_memory().to(batch.device, non_blocking=True)
        storage = phase.storage
        if B:
            BF.call("bm_scatter_rows", BF.ptr(batch), BF.ptr(table[len(kept_slots):]), B, batch[0].numel(),
                    BF.ptr(storage), BF.stream())
        cand = PooledCandidates(batch, storage, table[:len(kept_slots)], kept_slots)
        phase.leases.add(cand)
        return cand

    def buffer(self, phase: str) -> torch.Tensor:
        """The reference's `negative_pool[phase]`: the pool's rows, newest first, as one tensor on the pool's device
        (the reference's empty `torch.Tensor([])` before the phase's first pooled step)."""
        p = self._phases[phase]
        if not len(p.slots):
            return torch.Tensor([])
        slots = torch.from_numpy(p.slots.astype(np.int32)).to(p.storage.device)
        out = torch.empty((len(p.slots),) + self._row_shape, dtype=torch.float32, device=p.storage.device)
        BF.call("bm_gather_rows", BF.ptr(p.storage), BF.ptr(slots), len(p.slots), out[0].numel(), BF.ptr(out),
                BF.stream())
        return out
