"""Drop-in `FeatureDecodingLoss` (reference: bm/losses.py:117-173): same constructor `(used_features, scaler)`,
`forward(estimate, output, mask)`, the sum over the features of a masked MSE (regression features) or a class-weighted
cross-entropy (categorical ones), in CUDA through the C ABI (`functional.decoding_loss`); see the class.

Drop-in `L1Loss` / `L2Loss` (reference: bm/losses.py:11-26): no constructor arguments, `forward(estimate, output, mask)`,
the mean absolute / squared error over the entries where the broadcast mask is True, in CUDA through the C ABI
(`functional.masked_loss`) with no host read, so a step that uses them can be captured in a CUDA graph.

Drop-in `ClipLoss` (reference: bm/losses.py:29-114): same constructor, `forward(estimate, candidate, mask)`,
`get_scores`, `get_probabilities`, `trim_samples`.  Scores, softmax / cross-entropy and their gradients run in
CUDA through the C ABI (`functional.clip_loss`, `functional.clip_scores`, and `functional.clip_scores_grad` when the
scores are differentiated, e.g. for gradient-based attribution).

Reference semantics kept on purpose: only the CANDIDATES are L2-normalised (losses.py:91-94), no temperature,
the `linear` projection is constructed but never applied (losses.py:35,82), targets are the first B candidates.

Extension (SURVEY.md 8(e), not in the reference): `global_negatives=True` all-gathers the candidates over the
default process group before scoring, so every rank contrasts against the global batch; when the candidates require
grad (a trainable feature model) the gather is differentiable (reduce-scatter of the candidate gradients).
"""
from __future__ import annotations

import typing as tp
import weakref

import torch

from . import functional as BF
from . import distrib
from .negatives import PooledCandidates


def _wants_grad(estimates, candidates) -> bool:
    return torch.is_grad_enabled() and (estimates.requires_grad or candidates.requires_grad)


class _MaskedLoss(torch.nn.Module):
    _kind: int

    def forward(self, estimate, output, mask=None):
        return BF.masked_loss(self._kind, estimate, output, mask)


class L1Loss(_MaskedLoss):
    """torch.nn.L1Loss() over estimate[mask.expand_as(estimate)] and output[...] (bm/losses.py:17-20)"""
    _kind = BF.MASKED_L1


class L2Loss(_MaskedLoss):
    """torch.nn.MSELoss() over estimate[mask.expand_as(estimate)] and output[...] (bm/losses.py:23-26)"""
    _kind = BF.MASKED_L2


class _DecodedFeature(tp.NamedTuple):
    name: str
    categorical: bool
    est_start: int
    est_width: int          # the feature's output_dimension (K for a categorical feature)
    out_start: int
    out_width: int          # the feature's dimension


class FeatureDecodingLoss(torch.nn.Module):
    """Drop-in `FeatureDecodingLoss(used_features, scaler)` (bm/losses.py:117-173), the solver's `regression_classification`
    loss: per feature of `used_features`, in order, F.mse_loss over the masked entries of a regression feature or
    F.cross_entropy over the masked (b, t) of a categorical one -- weighted by `scaler.get_categorical_feature_weights(name)`
    when a scaler is given -- added up as `loss += ...`.

    `used_features` is duck-typed like the reference's FeaturesBuilder (`values()` of features with `name`, `categorical`,
    `dimension`, `output_dimension`; `get_slice(name, model_output)`, `dimension`, `output_dimension`) and `scaler` like
    its BatchScaler or this package's (`get_categorical_feature_weights`, and `feature_scalers[name].categories_count_`).
    The feature table is built once per device, the class weights once per device and again whenever a feature's
    `categories_count_` is replaced or changed in place.  An eager step reads one flag word to raise the reference's errors;
    a captured step reads nothing and reports them through `functional.check_tc_status()`."""

    def __init__(self, used_features, scaler):
        super().__init__()
        self.used_features = used_features
        self.scaler = scaler
        self._plan: tp.Optional[tp.List[_DecodedFeature]] = None
        self._tables: tp.Dict[torch.device, torch.Tensor] = {}
        self._weights: tp.Dict[torch.device, tp.Tuple[tp.Tuple, torch.Tensor]] = {}

    def _features(self) -> tp.List[_DecodedFeature]:
        if self._plan is None:
            plan = []
            for feature in self.used_features.values():
                est_sl = self.used_features.get_slice(feature.name, model_output=True)
                out_sl = self.used_features.get_slice(feature.name)
                plan.append(_DecodedFeature(feature.name, bool(feature.categorical), est_sl.start, est_sl.stop - est_sl.start,
                                            out_sl.start, out_sl.stop - out_sl.start))
            if not 1 <= len(plan) <= BF.DECODING_MAX_FEATURES:
                raise NotImplementedError(f"FeatureDecodingLoss takes 1 to {BF.DECODING_MAX_FEATURES} features, got "
                                          f"{len(plan)}")
            self._plan = plan
        return self._plan

    def _table(self, device) -> torch.Tensor:
        table = self._tables.get(device)
        if table is None:
            if BF.capturing():
                raise RuntimeError("FeatureDecodingLoss copies its feature table to the device on the first call: run one "
                                   "eager step on this device before capturing")
            rows, woff, slot = [], 0, 0
            for f in self._features():
                if f.categorical:
                    rows.append([BF.DECODING_CATEGORICAL, f.est_start, f.est_width, f.out_start,
                                 woff if self.scaler is not None else -1, slot])
                    woff, slot = woff + f.est_width, slot + 1
                else:
                    rows.append([BF.DECODING_REGRESSION, f.est_start, f.est_width, f.out_start, -1, -1])
            table = self._tables[device] = torch.tensor(rows, dtype=torch.int32).to(device)
        return table

    def _count_token(self, name):
        """what identifies the class counts the weights of feature `name` come from: the tensor and its version"""
        counts = getattr(getattr(self.scaler, "feature_scalers", {}).get(name), "categories_count_", None)
        return None if counts is None else (counts, counts._version)

    def _class_weights(self, device) -> tp.Optional[torch.Tensor]:
        if self.scaler is None:
            return None
        cats = [f for f in self._features() if f.categorical]
        tokens = tuple(self._count_token(f.name) for f in cats)
        cached = self._weights.get(device)
        if cached is not None and all(a is b or (a is not None and b is not None and a[0] is b[0] and a[1] == b[1])
                                      for a, b in zip(cached[0], tokens)):
            return cached[1]
        if BF.capturing():
            raise RuntimeError("FeatureDecodingLoss copies the class weights to the device when they are first used or "
                               "the scaler's category counts change: run one eager step before capturing")
        parts = []
        for f in cats:
            w = self.scaler.get_categorical_feature_weights(f.name)
            if w.dim() != 1 or w.numel() != f.est_width:     # F.cross_entropy's check
                raise RuntimeError(f"weight tensor should be defined either for all {f.est_width} classes or no classes "
                                   f"but got weight tensor of shape: {list(w.shape)}")
            parts.append(w.detach().to(device=device, dtype=torch.float32))
        weights = torch.cat(parts) if parts else torch.zeros(1, device=device)
        self._weights[device] = (tokens, weights)
        return weights

    def forward(self, estimate, output, mask=None):
        uf = self.used_features
        assert estimate.shape[1] == uf.output_dimension and output.shape[1] == uf.dimension, \
            "Invalid features dim received. Are you using the correct features for the loss?"
        if mask is None:
            raise TypeError("FeatureDecodingLoss needs a bool mask (bm/losses.py:141 expands it); got None")
        if estimate.dim() != 3 or output.dim() != 3:
            raise ValueError(f"FeatureDecodingLoss takes [B, C, T] operands, got {estimate.dim()} and {output.dim()} "
                             "dimensions")
        plan = self._features()
        for f in plan:                                       # the reference's shape errors, in its order
            feature_mask = mask.expand_as(estimate[:, f.est_start:f.est_start + f.est_width])    # RuntimeError
            if f.categorical:
                assert f.out_width == 1, "Supporting only single categorical cross entropy for now."
                if mask.dim() != 3 or mask.shape[1] != 1 or \
                        (mask.shape[0], mask.shape[2]) != (output.shape[0], output.shape[2]):
                    raise IndexError(f"The shape of the mask {list(mask.transpose(-1, -2).shape)} does not match the "
                                     f"shape of the indexed tensor {[output.shape[0], output.shape[2], 1]}")
            elif output[:, f.out_start:f.out_start + f.out_width].shape != feature_mask.shape:
                raise IndexError(f"The shape of the mask {list(feature_mask.shape)} does not match the shape of the "
                                 f"indexed tensor {list(output[:, f.out_start:f.out_start + f.out_width].shape)}")
        m = mask
        while m.dim() < 3:
            m = m.unsqueeze(0)
        m = m.expand(estimate.shape[0], m.shape[1], estimate.shape[2])
        device = estimate.device
        loss, flag = BF.decoding_loss(self._table(device), sum(f.categorical for f in plan), self._class_weights(device),
                                      estimate, output, m)
        if not BF.capturing():
            code = int(flag.item())                          # the one host read of an eager step
            if code:
                f = plan[code >> 16]
                raise BF._decoding_error(code & 0xFFFF, f"feature {f.name!r}, output_dim {f.est_width}")
        return loss


class ClipLoss(torch.nn.Module):
    def __init__(self, linear=None, twin=True, pool=False, tmin=None, tmax=None,
                 tmin_train=None, tmax_train=None, dset_args=None, center=False, global_negatives=False,
                 uniform_batches=False):
        super().__init__()
        self.linear = None                      # the reference never applies its projection (losses.py:35)
        self.pool = pool
        self.center = center
        if linear is not None:                  # kept for state_dict compatibility only
            self.linear_est = torch.nn.LazyLinear(linear)
            self.linear_gt = self.linear_est if twin else torch.nn.LazyLinear(linear)
        self.tmin, self.tmax = tmin, tmax
        self.tmin_train, self.tmax_train = tmin_train, tmax_train
        self.dset_args = dset_args
        self.global_negatives = global_negatives
        # global_negatives only: True = every rank holds the same number of rows each step (drop_last loaders, no
        # rejection), which saves the per-step exchange of the per-rank counts; False = counts are exchanged and ragged
        # batches are handled (the reference's loaders have no drop_last, and ScaleReject drops samples per rank)
        self.uniform_batches = uniform_batches
        self._prefetched = None
        self._mask_ok = None

    # -- time cropping (losses.py:50-75) ---------------------------------------------------------------
    def _window(self, n_samples: int):
        use_train = self.training and (self.tmin_train is not None or self.tmax_train is not None)
        tmin, tmax = (self.tmin_train, self.tmax_train) if use_train else (self.tmin, self.tmax)
        start, stop = 0, n_samples
        if tmin is not None or tmax is not None:
            assert self.dset_args is not None and self.dset_args.tmin is not None
            origin, rate = self.dset_args.tmin, self.dset_args.sample_rate
            if tmin is not None:
                assert tmin >= origin, 'clip.tmin should be above dset.tmin'
                start = int((tmin - origin) * rate)
            if tmax is not None:
                stop = int((tmax - origin) * rate)
        return start, stop

    def trim_samples(self, estimates, candidates):
        start, stop = self._window(estimates.shape[-1])
        return estimates[..., start:stop], candidates[..., start:stop]

    def _prepare(self, estimates, candidates):
        estimates, candidates = self.trim_samples(estimates, candidates)
        if self.pool:                            # losses.py:85-87
            estimates = estimates.mean(dim=2, keepdim=True)
            candidates = candidates.mean(dim=2, keepdim=True)
        if self.center:                          # losses.py:88-90
            estimates = estimates - estimates.mean(dim=(1, 2), keepdim=True)
            candidates = candidates - candidates.mean(dim=(1, 2), keepdim=True)
        return estimates, candidates

    def get_scores(self, estimates: torch.Tensor, candidates: torch.Tensor):
        """[B, C, T] x [B', C, T] -> [B, B'] matching scores.  Differentiable when an input requires grad (gradient-based
        attribution); otherwise no autograd node is recorded."""
        estimates, candidates = self._prepare(estimates, candidates)
        if _wants_grad(estimates, candidates):
            return BF.clip_scores_grad(estimates, candidates)
        return BF.clip_scores(estimates, candidates)

    def get_probabilities(self, estimates, candidates):
        estimates, candidates = self._prepare(estimates, candidates)
        if _wants_grad(estimates, candidates):
            return BF.clip_scores_grad(estimates, candidates, want_probs=True)
        return BF.clip_scores(estimates, candidates, want_probs=True)

    def prefetch_candidates(self, candidate: torch.Tensor) -> None:
        """Optional (multi-GPU, global_negatives): start the candidate all-gather now -- e.g. right after the batch reaches
        the device, before the encoder forward -- so that it overlaps compute.  `forward` picks it up when it is called
        with the same tensor; without this call the gather simply happens inside `forward`."""
        if self.global_negatives and distrib.world_size() > 1 and not candidate.requires_grad \
                and not (self.pool or self.center) \
                and self._window(candidate.shape[-1]) == (0, candidate.shape[-1]):
            self._prefetched = distrib.CandidateGather(candidate, self.uniform_batches)

    def _check_mask(self, mask) -> None:
        """losses.py:110 `assert mask.all()`: on a CUDA mask that is a device->host sync per call.  The verdict is kept per
        mask tensor OBJECT (weak reference + version counter), so a caller that reuses one all-true mask pays it once; a fresh
        mask per batch (what bm/solver.py passes) is checked every time, exactly like the reference.

        While the step is captured in a CUDA graph the host cannot read the mask, and a replay changes its content without
        running any Python: the check is then enqueued on the device on every call (`functional.check_all_true`), and a
        False entry raises at the next `functional.check_tc_status()`."""
        if BF.capturing():
            BF.check_all_true(mask)
            return
        seen = self._mask_ok
        if seen is not None and seen[0]() is mask and seen[1] == mask._version:
            return
        assert mask.all(), "mask is not supported for now"
        self._mask_ok = (weakref.ref(mask), mask._version)

    def forward(self, estimate, candidate, mask=None):
        if isinstance(candidate, PooledCandidates):
            if self.global_negatives and distrib.world_size() > 1:
                raise NotImplementedError("ClipLoss(global_negatives=True) over a negative pool: the reference's pool is "
                                          "local to each GPU, and mixing pools across ranks has no reference meaning")
            if BF.capturing():
                raise RuntimeError("ClipLoss over a negative pool cannot be captured in a CUDA graph: the slot table is "
                                   "built on the host and the candidate count grows while the pool fills")
            if self._window(estimate.shape[-1]) == (0, estimate.shape[-1]) and not (self.pool or self.center) \
                    and BF.clip_pooled_supported(candidate.row_elems):
                self._check_mask(mask)
                assert estimate.size(0) <= candidate.size(0), "need at least as many targets as estimates"
                return BF.clip_loss_pooled(estimate, candidate)
            candidate = candidate.materialize()
        if self.global_negatives and BF.capturing() and distrib.world_size() > 1:
            raise RuntimeError("ClipLoss(global_negatives=True) all-gathers the candidates over the ranks, which a CUDA graph "
                               "capture of the step cannot hold; capture on one rank or without global_negatives")
        self._check_mask(mask)
        assert estimate.size(0) <= candidate.size(0), "need at least as many targets as estimates"
        pre, self._prefetched = self._prefetched, None
        if candidate.requires_grad and torch.is_grad_enabled() and self.global_negatives and distrib.world_size() > 1:
            # a trainable feature model made the candidates: differentiable gather (reduce-scatter of dC in backward)
            estimate, candidate = self._prepare(estimate, candidate)
            candidate, offset = distrib.all_gather_candidates_with_grad(candidate, self.uniform_batches)
            return BF.clip_loss(estimate, candidate, offset)
        if pre is not None and pre.source is candidate:
            estimate, _ = self._prepare(estimate, candidate)
            candidate, offset = pre.wait()
            return BF.clip_loss(estimate, candidate, offset)
        estimate, candidate = self._prepare(estimate, candidate)
        offset = 0
        if self.global_negatives and distrib.world_size() > 1:
            candidate, offset = distrib.all_gather_candidates(candidate, self.uniform_batches)
        return BF.clip_loss(estimate, candidate, offset)
