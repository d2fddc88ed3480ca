"""Multi-GPU plumbing (one process per GPU, torch.distributed/NCCL over NVLink).

The path shards by batch row (SURVEY.md 8(e)): each rank encodes its rows (BatchNorm statistics per rank, or over the
process group for layers converted with torch.nn.SyncBatchNorm.convert_sync_batchnorm, see functional.bn_sync_groups), then
  * `all_gather_candidates`: the ONE forward exchange -- NCCL all-gather of the candidate block so every rank
    scores its rows against the global batch (new semantic; the reference keeps negatives local, README.md:139-143);
  * `all_gather_candidates_with_grad`: the same exchange when a trainable feature model produced the candidates --
    its backward is the reduce-scatter(sum) of the candidate gradients;
  * `sync_gradients`: the reference's gradient all-reduce(avg) (flashy.distrib.sync_model, bm/solver.py:386),
    done on one flat bucket AFTER the backward pass: the backward's kernels fill every SM, so an NCCL
    kernel overlapped with them would push CTAs into a second round (see the candidate gather below), costing more
    than the ~0.3 ms the 36-80 MB all-reduce takes on its own.
"""
from __future__ import annotations

import os
import typing as tp

import torch
import torch.distributed as dist


def world_size() -> int:
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def rank() -> int:
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def gather_counts(n_local: int, device) -> tp.List[int]:
    """Rows every rank contributes.  The reference's loaders have no drop_last and ScaleReject / exclude_empty_features
    drop samples per rank (bm/norm.py:325-341), so per-rank batch sizes can differ: they are exchanged first (one tiny
    all-gather + a host read), unless the caller vouches for equal batches (`uniform=True`, e.g. drop_last loaders)."""
    W = world_size()
    if W == 1:
        return [n_local]
    mine = torch.tensor([n_local], dtype=torch.int64, device=device)
    allc = torch.empty(W, dtype=torch.int64, device=device)
    dist.all_gather_into_tensor(allc, mine)
    return [int(v) for v in allc.tolist()]


def _pad_rows(x: torch.Tensor, rows: int) -> torch.Tensor:
    if x.shape[0] == rows:
        return x.contiguous()
    out = x.new_zeros((rows,) + tuple(x.shape[1:]))
    out[:x.shape[0]] = x
    return out


def _compact(padded: torch.Tensor, counts: tp.List[int], block: int) -> torch.Tensor:
    """[W*block, ...] with rank r's rows at [r*block, r*block + counts[r]) -> [sum(counts), ...]"""
    if all(c == block for c in counts):
        return padded
    return torch.cat([padded[r * block:r * block + c] for r, c in enumerate(counts)], dim=0)


def all_gather_candidates(candidate: torch.Tensor, uniform: bool = False) -> tp.Tuple[torch.Tensor, int]:
    """[B_r, F, T] on rank r -> ([sum_r B_r, F, T], row of this rank's first candidate).  For candidates that carry no
    gradient (no feature_model); see `all_gather_candidates_with_grad` otherwise.  Ragged per-rank batches are padded to
    the largest for the exchange and the padding rows are dropped afterwards."""
    W = world_size()
    if W == 1:
        return candidate, 0
    n = candidate.shape[0]
    counts = [n] * W if uniform else gather_counts(n, candidate.device)
    block = max(counts)
    src = _pad_rows(candidate, block)
    out = torch.empty((W * block,) + tuple(candidate.shape[1:]), dtype=candidate.dtype, device=candidate.device)
    dist.all_gather_into_tensor(out, src)
    return _compact(out, counts, block), sum(counts[:rank()])


class _GatherWithGrad(torch.autograd.Function):
    """All-gather whose backward is the reduce-scatter(sum) SURVEY.md 8(e) asks for when the candidates carry a gradient
    (a trainable feature model, bm/solver.py:304-320): rank r's block of the gathered tensor feeds EVERY rank's loss term,
    so its gradient is the sum over ranks of that block of their gradients.  (Parameter gradients are then averaged by
    `sync_gradients` / flashy's sync_model like all others, which yields the gradient of the mean of the per-rank losses.)"""

    @staticmethod
    def forward(ctx, candidate, counts):
        W = world_size()
        block = max(counts)
        src = _pad_rows(candidate, block)
        out = torch.empty((W * block,) + tuple(candidate.shape[1:]), dtype=candidate.dtype, device=candidate.device)
        dist.all_gather_into_tensor(out, src)
        ctx.counts, ctx.block = counts, block
        return _compact(out, counts, block)

    @staticmethod
    def backward(ctx, dgathered):
        counts, block, r = ctx.counts, ctx.block, rank()
        n = counts[r]
        if any(c != block for c in counts):                     # back to the padded [W*block] layout of the exchange
            padded = dgathered.new_zeros((len(counts) * block,) + tuple(dgathered.shape[1:]))
            off = 0
            for i, c in enumerate(counts):
                padded[i * block:i * block + c] = dgathered[off:off + c]
                off += c
            dgathered = padded
        dgathered = dgathered.contiguous()
        if dist.get_backend() == "nccl":
            own = torch.empty((block,) + tuple(dgathered.shape[1:]), dtype=dgathered.dtype, device=dgathered.device)
            dist.reduce_scatter_tensor(own, dgathered, op=dist.ReduceOp.SUM)
            return own[:n].contiguous(), None
        total = dgathered.clone()              # gloo (CPU tests) has no reduce-scatter
        dist.all_reduce(total, op=dist.ReduceOp.SUM)
        return total[r * block:r * block + n].clone(), None


def all_gather_candidates_with_grad(candidate: torch.Tensor, uniform: bool = False) -> tp.Tuple[torch.Tensor, int]:
    """`all_gather_candidates` for candidates that require grad: differentiable (reduce-scatter in backward)."""
    W = world_size()
    if W == 1:
        return candidate, 0
    n = candidate.shape[0]
    counts = [n] * W if uniform else gather_counts(n, candidate.device)
    return _GatherWithGrad.apply(candidate, counts), sum(counts[:rank()])


# ---------------------------------------------------------------------------------------------------------------------
# Candidate all-gather over NVLink peer memory, driven by the COPY ENGINES (no SMs)
# ---------------------------------------------------------------------------------------------------------------------
# The conv / weight-gradient / CLIP kernels run one CTA per SM (all of the SM's shared memory) in waves sized to the SM
# count.  An NCCL all-gather kernel that runs beside them for milliseconds (3 GB at N = 8) takes a handful of SMs for that
# whole time, and every launch in that window finds fewer SMs than it was sized for: the leftover CTAs wait for a
# whole CTA to finish its tile -- a second round, up to 2x per kernel.  So the gather is done without SMs: every rank
# copies its block into a symmetric-memory buffer (torch.distributed._symmetric_memory: cuMem allocations mapped into
# every peer), and after a barrier PULLS the other ranks' blocks with cudaMemcpyAsync device-to-device copies, which the
# copy engines execute over NVLink.  A second barrier tells the owners that their buffer may be overwritten by the next
# step.  Anything missing (torch without symmetric memory, peers without P2P) falls back to the NCCL all-gather.
_symm_state: tp.Dict[tp.Any, tp.Any] = {}
USE_SYMMETRIC_GATHER = os.environ.get("BM_SYMM_GATHER", "1") != "0"      # BM_SYMM_GATHER=0: NCCL all-gather (A/B timing)


def _symm_buffers(shape: tp.Tuple[int, ...], device: torch.device):
    """One symmetric buffer + handle per (shape, device), created collectively on first use (None if unavailable)."""
    key = (tuple(shape), device)
    if key in _symm_state:
        return _symm_state[key]
    out = None
    try:
        import torch.distributed._symmetric_memory as symm_mem
        group = dist.group.WORLD
        buf = symm_mem.empty(*shape, dtype=torch.float32, device=device)
        hdl = symm_mem.rendezvous(buf, group.group_name)
        out = (buf, hdl, torch.cuda.Stream(device=device))
    except Exception as exc:                                   # pragma: no cover - depends on the installation
        import warnings
        warnings.warn(f"symmetric-memory candidate gather unavailable ({type(exc).__name__}: {exc}); using NCCL all-gather")
    # every rank must take the same branch: agree on availability
    flag = torch.tensor([1 if out is not None else 0], device=device)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if int(flag.item()) == 0:
        out = None
    _symm_state[key] = out
    return out


class CandidateGather:
    """The candidate all-gather started EARLY (it does not depend on the encoder): the blocks move over NVLink while the
    encoder's forward kernels run; `wait()` joins it on the current stream just before the contrastive matmul.
    Uniform per-rank batches on NCCL devices go through symmetric memory and the copy engines (above); ragged batches and
    other backends through the (padded) NCCL / gloo all-gather."""

    def __init__(self, candidate: torch.Tensor, uniform: bool = False):
        self.source = candidate
        W = world_size()
        n = candidate.shape[0]
        self.work = self.event = None
        if W == 1:
            self.out, self.offset, self.counts, self.block = candidate, 0, [n], n
            return
        self.counts = [n] * W if uniform else gather_counts(n, candidate.device)
        self.block = max(self.counts)
        self.offset = sum(self.counts[:rank()])
        ragged = any(c != self.block for c in self.counts)
        symm = None
        if USE_SYMMETRIC_GATHER and not ragged and candidate.is_cuda and candidate.dtype == torch.float32 \
                and dist.get_backend() == "nccl":
            symm = _symm_buffers(tuple(candidate.shape), candidate.device)
        if symm is not None:
            buf, hdl, side = symm
            r = rank()
            main = torch.cuda.current_stream()
            self.out = torch.empty((W * n,) + tuple(candidate.shape[1:]), dtype=candidate.dtype, device=candidate.device)
            side.wait_stream(main)
            with torch.cuda.stream(side):
                buf.copy_(candidate)                                   # my block, where the peers can read it
                hdl.barrier(channel=0)                                 # every rank's block is in place
                for step in range(1, W):
                    peer = (r - step) % W
                    self.out[peer * n:(peer + 1) * n].copy_(hdl.get_buffer(peer, candidate.shape, candidate.dtype))
                self.out[r * n:(r + 1) * n].copy_(candidate)
                hdl.barrier(channel=1)                                 # every rank has read my block: it may be reused
                self.event = torch.cuda.Event()
                self.event.record(side)
            self.out.record_stream(side)
            self._src = candidate
            return
        src = _pad_rows(candidate, self.block)
        self.out = torch.empty((W * self.block,) + tuple(candidate.shape[1:]), dtype=candidate.dtype,
                               device=candidate.device)
        self.work = dist.all_gather_into_tensor(self.out, src, async_op=True)
        self._src = src                        # keep the (possibly padded) source alive until the collective is joined

    def wait(self) -> tp.Tuple[torch.Tensor, int]:
        if self.event is not None:
            torch.cuda.current_stream().wait_event(self.event)
            self.event = None
            self._src = None
        if self.work is not None:
            self.work.wait()          # current stream waits for NCCL's stream; the host does not block
            self.work = None
            self._src = None
            self.out = _compact(self.out, self.counts, self.block)
        return self.out, self.offset


def sync_gradients(params: tp.Iterable[torch.nn.Parameter]) -> None:
    """all-reduce(avg) of every .grad through one flat fp32 bucket: one concatenation, one collective (NCCL averages in
    the reduction itself), one multi-tensor copy back -- three launches for the ~60 gradient tensors."""
    W = world_size()
    if W == 1:
        return
    grads = [p.grad for p in params if p.grad is not None]
    if not grads:
        return
    flat = torch.cat([g.reshape(-1) for g in grads])
    if dist.get_backend() == "nccl":
        dist.all_reduce(flat, op=dist.ReduceOp.AVG)
    else:
        dist.all_reduce(flat, op=dist.ReduceOp.SUM)
        flat.div_(W)
    views, off = [], 0
    for g in grads:
        n = g.numel()
        views.append(flat[off:off + n].view_as(g))
        off += n
    torch._foreach_copy_(grads, views)
