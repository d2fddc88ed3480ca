"""Drop-in test metrics (bm/metrics.py): `OnlineCorrelation`, `L1Reg`, `L2Reg` and `ClassificationAcc`, with the
reference's constructors, attributes, `update(left, right, mask) -> self`, `get()` and `reduce`, and the reference's
results, quirks included (DESIGN §4.9).

Each update adds its per-column sums over dim 0 into fp64 accumulators on the operands' device in one C-ABI call and
reads nothing on the host; `get()` runs one finalize kernel and reads one flag word.  The reference re-initialises its sums
while `_count.sum() == 0`; here a device word records whether any mask entry has been True, and an update overwrites the
sums while it is 0.  That word is read on the host only when an update's column shape, dtype or device differs from the
accumulators'.
"""
from __future__ import annotations

import typing as tp
from abc import ABC
from functools import partial

import torch

from . import functional as F


class TestMetric(ABC):
    def __init__(self, left_slice: slice, right_slice, name: str = "metric"):
        self.name = name
        self.left_slice = left_slice
        self.right_slice = right_slice

    @classmethod
    def get_constructor(cls, *args: tp.Any, **kwargs: tp.Any) -> tp.Callable[..., "TestMetric"]:
        return partial(cls, *args, **kwargs)

    def update(self, left: torch.Tensor, right: torch.Tensor, mask: torch.Tensor) -> "TestMetric":
        raise NotImplementedError()

    def get(self) -> torch.Tensor:
        raise NotImplementedError()

    @classmethod
    def reduce(cls, stats: tp.List[torch.Tensor]) -> torch.Tensor:
        return torch.stack(stats).mean().item()


class _Sums:
    """A metric's device accumulators: fp64 [planes, columns], the ping-pong "seen a True mask entry" word and the parity
    the next update reads, and the column shape, dtype and device of the update that initialised them."""

    def __init__(self, kind: int, shape: tp.Tuple[int, ...], dtype: torch.dtype, device: torch.device):
        cols = 1
        for s in shape:
            cols *= s
        self.acc = torch.zeros((F.metric_planes(kind), cols), dtype=torch.float64, device=device)
        self.seen = torch.zeros(2, dtype=torch.int32, device=device)
        self.parity = 0
        self.shape, self.dtype, self.device = shape, dtype, device

    def seen_true(self) -> bool:
        return bool(int(self.seen[self.parity]))


def _update(metric, kind: int, left: torch.Tensor, right: torch.Tensor, mask: torch.Tensor) -> None:
    if metric.dim != 0:
        raise NotImplementedError(f"brainmagick_b200 test metrics reduce over dim 0 only, got dim={metric.dim}")
    if left.is_complex() or right.is_complex():
        raise NotImplementedError("brainmagick_b200 test metrics take real operands (no CUDA model here is complex)")
    left = left[:, metric.left_slice]
    right = right[:, metric.right_slice]
    F.metric_operands(kind, left, right, mask)
    ref = left if kind == F.METRIC_CORRELATION else right
    shape, dtype, device = tuple(ref.shape[1:]), ref.dtype, ref.device
    sums = metric._sums
    if sums is None or (sums.shape, sums.dtype, sums.device) != (shape, dtype, device):
        # the reference re-initialises from this update while no mask entry has been True; afterwards it adds into the
        # sums it has (a later dtype is cast into them, another shape or device fails)
        if sums is None or not sums.seen_true():
            sums = metric._sums = _Sums(kind, shape, dtype, device)
        elif sums.shape != shape or sums.device != device:
            raise RuntimeError(f"{type(metric).__name__} '{metric.name}': an update of columns {shape} on {device} after "
                               f"columns {sums.shape} on {sums.device}")
    F.metric_update(kind, left, right, mask, sums.acc, sums.seen, sums.parity)
    sums.parity ^= 1


class OnlineCorrelation(TestMetric):
    def __init__(self, left_slice: slice, right_slice: slice,
                 name: str = "correlation", dim: int = 0, tol: float = 1e-8):
        """
        Online correlations between `left` and `right` along dim 0, per (channel, time) column: updates stream batches
        along that dimension.  Only dim 0 and real operands are ported.
        Args:
            dim (int): dimension along which to compute the correlation (0).
            tol (float): tolerance used for numerical stability.
        """
        super().__init__(left_slice, right_slice, name)
        self.dim = dim
        self.tol = tol
        assert tol >= 0
        self._sums: tp.Optional[_Sums] = None

    def update(self, left: torch.Tensor, right: torch.Tensor,
               mask: torch.Tensor) -> "OnlineCorrelation":
        _update(self, F.METRIC_CORRELATION, left, right, mask)
        return self

    def get(self) -> torch.Tensor:
        """
        Return the correlation tensor.
        """
        sums = self._sums
        if sums is None:
            raise AttributeError(f"OnlineCorrelation '{self.name}' has no sums: get() before any update()")
        if sums.acc.shape[1] == 0:                      # the reference's norm_squared.min() of an empty tensor
            raise RuntimeError(f"OnlineCorrelation '{self.name}': no columns (an empty slice or time crop)")
        out, flag = F.metric_finalize(F.METRIC_CORRELATION, sums.acc, sums.acc.shape[1], self.tol, sums.dtype)
        bits = int(flag.item())
        for side, unstable, nan in (("left", F.METRIC_LEFT_UNSTABLE, F.METRIC_LEFT_NAN),
                                    ("right", F.METRIC_RIGHT_UNSTABLE, F.METRIC_RIGHT_NAN)):
            # the reference's norm_squared.min() < -tol, which a NaN among the norms makes False
            if bits & unstable and not bits & nan:
                raise ValueError(f"Numerical instabilities when computing the correlation: a {side} norm squared "
                                 f"below -{self.tol}")
        assert not bits & F.METRIC_RESULT_NAN, "Tensor contain nans. Perhaps division by zero cause that?"
        return out.view(sums.shape)


class AccumulativeMetric(TestMetric):
    _kind: tp.Optional[int] = None

    def __init__(self,
                 left_slice: slice,
                 right_slice: slice,
                 name: str = "N/A", dim: int = 0):

        super().__init__(left_slice, right_slice, name)
        self.dim = dim
        self._sums: tp.Optional[_Sums] = None

    def update(self, left: torch.Tensor, right: torch.Tensor,
               mask: torch.Tensor) -> "AccumulativeMetric":
        if self._kind is None:
            raise NotImplementedError()
        _update(self, self._kind, left, right, mask)
        return self

    def get(self) -> torch.Tensor:
        sums = self._sums
        if sums is None:
            return torch.Tensor([0.])
        out, flag = F.metric_finalize(self._kind, sums.acc, sums.acc.shape[1], 0.0, sums.dtype)
        bits = int(flag.item())
        if not bits & F.METRIC_COUNTED:
            return torch.Tensor([0.])
        assert not bits & F.METRIC_RESULT_NAN, "Tensor contain nans. Perhaps division by zero cause that?"
        return out.view(sums.shape)


class L1Reg(AccumulativeMetric):
    """Σ |(left - right) · mask| / count per column"""
    _kind = F.METRIC_L1


class L2Reg(AccumulativeMetric):
    """Σ ((left - right) · mask)² / count per column"""
    _kind = F.METRIC_L2

    @classmethod
    def reduce(cls, stats: torch.Tensor) -> torch.Tensor:
        return torch.stack(stats).mean().sqrt().item()


class ClassificationAcc(AccumulativeMetric):
    """the share of masked (n, t) where the first argmax over the left slice's channels equals the target"""
    _kind = F.METRIC_ACCURACY
