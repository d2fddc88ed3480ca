"""TEST INFRASTRUCTURE ONLY -- stores what the verbatim reference FeatureDecodingLoss (bm/losses.py:117-173, plain PyTorch
autograd) computes, so that tests/test_decoding_loss_cpu.py can hold the drop-in loss to it wherever the tests run (the
reference tree is needed only to regenerate them).

    python oracle/make_decoding_loss_golden.py      # writes tests/golden/decoding_*.npz

The loss gets a small stand-in for bm.features.FeaturesBuilder (features with `name`, `dimension`, `cardinality`; the
builder's `get_slice`, `dimension`, `output_dimension`) and, for the weighted cases, class weights from the reference's own
`BatchScaler.get_categorical_feature_weights` over `NoOpCategoryCountScaler`s fitted on class ids (bm/norm.py:124-147,
289-308).

Each file holds one case: `est`, `out`, `mask` and `limit` (> 0: the loss takes est[..., limit:] and the same crop of out
and mask, as the solver's time crops); the features as `names`, `dims` (dimension) and `cards` (cardinality, 0 for a
regression feature); `weighted`; per categorical feature i, `counts<i>` and `weights<i>`; and `loss`, `d_est`, `d_out`: the
loss and its gradients with respect to the full `est` and `out` tensors (zeros where autograd gives none).

  decoding_cat_k2            one categorical feature with K = 2, a ragged [B, 1, T] mask
  decoding_mixed             [regression 3, categorical 5, regression 1, categorical 7], fractional targets (.long()
                             truncates), unweighted
  decoding_mixed_weighted    the same, weighted
  decoding_all_true          the same, weighted, an all-true mask
  decoding_zero_count        weighted, masked targets in a class that never occurred in the fit (weight 0)
  decoding_ignore_index      weighted, masked targets of -100 and -100.5 (ignore_index after .long())
  decoding_time_crop         weighted, est[..., limit:] at an odd element offset
  decoding_zero_weight_only  every masked target of a categorical feature is in a zero-weight class: that term and its
                             gradients are NaN, as torch computes them
"""
from __future__ import annotations

import os
import sys
from collections import OrderedDict

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_loader  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
B, T = 3, 13
MIXED = [("mel", 3, None), ("phoneme", 1, 5), ("env", 1, None), ("pos", 1, 7)]


class _Feature:
    def __init__(self, name, dimension, cardinality):
        self.name, self.dimension, self.cardinality = name, dimension, cardinality

    @property
    def categorical(self):
        return self.cardinality is not None

    @property
    def output_dimension(self):
        return self.dimension if self.cardinality is None else self.cardinality


class _Builder(OrderedDict):
    """bm.features.FeaturesBuilder's slicing surface (bm/features/base.py:128-173)"""

    def get_slice(self, name, model_output=False):
        start = 0
        for key, feature in self.items():
            width = feature.output_dimension if model_output else feature.dimension
            if key == name:
                return slice(start, start + width)
            start += width
        raise KeyError(name)

    @property
    def dimension(self):
        return sum(f.dimension for f in self.values())

    @property
    def output_dimension(self):
        return sum(f.output_dimension for f in self.values())


class _ScalerStub:
    def __init__(self, feature_scalers):
        self.feature_scalers = feature_scalers


def _ragged(gen, t):
    mask = torch.ones(B, 1, t, dtype=torch.bool)
    for b in range(B):
        start = int(torch.randint(0, t - 4, (1,), generator=gen))
        mask[b, 0, start:start + 2 + b] = False
    return mask


def _inputs(gen, spec, t, frac=False):
    builder = _Builder((name, _Feature(name, dim, card)) for name, dim, card in spec)
    est = torch.randn(B, builder.output_dimension, t, generator=gen) * 2
    out = torch.randn(B, builder.dimension, t, generator=gen)
    for name, _, card in spec:
        if card is not None:
            ids = torch.randint(0, card, (B, t), generator=gen).float()
            if frac:
                ids = ids + 0.9 * torch.rand(B, t, generator=gen)
            out[:, builder.get_slice(name).start] = ids
    return builder, est, out


def cases():
    gen = torch.Generator().manual_seed(2024)
    builder, est, out = _inputs(gen, [("word_segment", 1, 2)], T)
    yield "cat_k2", builder, est, out, _ragged(gen, T), 0, None
    builder, est, out = _inputs(gen, MIXED, T, frac=True)
    mask = _ragged(gen, T)
    yield "mixed", builder, est, out, mask, 0, None
    yield "mixed_weighted", builder, est, out, mask, 0, {}
    yield "all_true", builder, est, out, torch.ones(B, 1, T, dtype=torch.bool), 0, {}
    builder, est, out = _inputs(gen, MIXED, T)
    out[:, 3, :4] = 3.0                                   # class 3 of `phoneme` never occurs in its fit
    yield "zero_count", builder, est, out, _ragged(gen, T), 0, {"phoneme": 3}
    builder, est, out = _inputs(gen, MIXED, T)
    out[:, 3, 1::3] = -100.0
    out[:, 5, 2::4] = -100.5
    yield "ignore_index", builder, est, out, _ragged(gen, T), 0, {}
    limit = 3
    builder, est, out = _inputs(gen, MIXED, T + limit)
    yield "time_crop", builder, est, out, _ragged(gen, T + limit), limit, {}
    builder, est, out = _inputs(gen, MIXED, T)
    out[:, 5] = 4.0                                       # every `pos` target is class 4, which never occurs in its fit
    yield "zero_weight_only", builder, est, out, _ragged(gen, T), 0, {"pos": 4}


def _fitted_scaler(norm, builder, gen, absent):
    scalers = OrderedDict()
    for name, feature in builder.items():
        if not feature.categorical:
            continue
        K = feature.cardinality
        ids = torch.randint(0, K, (200,), generator=gen).float()
        ids[0], ids[1] = 0.0, K - 1.0
        if name in absent:
            ids[ids == absent[name]] = 0.0 if absent[name] != 0 else 1.0
        scalers[name] = norm.NoOpCategoryCountScaler(K).fit(ids, torch.ones(200, dtype=torch.bool))
    return _ScalerStub(scalers)


def main():
    torch.set_num_threads(1)
    _, _, losses = ref_loader.load_reference()
    norm = ref_loader.load_reference_norm()
    gen = torch.Generator().manual_seed(7)
    for name, builder, est, out, mask, limit, absent in cases():
        scaler = None if absent is None else _fitted_scaler(norm, builder, gen, absent)
        if scaler is not None:
            scaler.get_categorical_feature_weights = \
                lambda n, s=scaler: norm.BatchScaler.get_categorical_feature_weights(s, n)
        e, o = est.clone().requires_grad_(True), out.clone().requires_grad_(True)
        loss = losses.FeatureDecodingLoss(builder, scaler)(e[..., limit:], o[..., limit:], mask[..., limit:])
        loss.backward()
        feats = list(builder.values())
        arrays = dict(est=est.numpy(), out=out.numpy(), mask=mask.numpy(), limit=np.int64(limit),
                      names=np.array([f.name for f in feats]), dims=np.array([f.dimension for f in feats]),
                      cards=np.array([f.cardinality or 0 for f in feats]), weighted=np.bool_(scaler is not None),
                      loss=loss.detach().numpy(), d_est=e.grad.numpy(),
                      d_out=(o.grad if o.grad is not None else torch.zeros_like(out)).numpy())
        if scaler is not None:
            for i, (fname, s) in enumerate(scaler.feature_scalers.items()):
                arrays[f"counts{i}"] = s.categories_count_.numpy()
                arrays[f"weights{i}"] = scaler.get_categorical_feature_weights(fname).numpy()
        path = os.path.join(OUT, f"decoding_{name}.npz")
        np.savez_compressed(path, **arrays)
        print(path, os.path.getsize(path), float(loss.detach()))


if __name__ == "__main__":
    main()
