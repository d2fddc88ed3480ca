"""TEST INFRASTRUCTURE ONLY -- stores what the verbatim reference `svd_penalty` (bm/svd.py over torch.svd_lowrank, plain
PyTorch on the CPU) computes, so that tests/test_svd_penalty_cpu.py can hold the drop-in to it wherever the tests run (the
reference tree is needed only to regenerate them).  bm/svd.py is loaded by file path; it imports only random and torch.

    python oracle/make_svd_golden.py      # writes tests/golden/svd_*.npz

Each file holds one model and a sequence of calls `svd_penalty(model, min_size, proba=proba)`, each after
`torch.manual_seed(seed_c)`, with the reference's `penalty_rng` reset to Random(1234) before the first call:
  model:   `model` (JSON: the module class under brainmagick_b200 or torch.nn and its kwargs), `w_{i}` the conv / linear
           weights in named_modules() order (every one, selected or not), `frozen` the indices of weights that do not
           require grad
  call c:  `seed_{c}`, `value_{c}` (nan: the call returned the float 0. without drawing), `draws_{c}` the number of
           torch.randn draws it made, `r_{c}_{k}` draw k, `g_{c}_{i}` the gradient of the value on weight i (zeros where
           it is frozen or not selected)
  `min_size`, `proba`, `calls`

  svd_clip_conv    a small clip_conv SimpleConv: [C, C*3] encoder and GLU convs, the 1x1 merger linear and the head's
                   Conv1d and ConvTranspose1d (wide: transposed), default min_size
  svd_residual     a ConvSequence with rewrite, LayerScale and post_skip: the depthwise [C, 1, 1] post_skip weights
                   (n = 1 < q) and the [C, C, 1] rewrite convs, min_size 0.01 so that none is skipped
  svd_layers       nn.Linear [50, 30], nn.ConvTranspose1d [24, 40, 3] (m < n), a Conv1d [60, 8, 5], a [16, 16] square
                   Linear (n = q) and two weights min_size skips
  svd_frozen       svd_layers with two weights frozen: their estimates count, they get no gradient
  svd_proba        svd_layers at proba = 0.5 over 8 calls: the reference's skip pattern and the 1 / proba scale
"""
from __future__ import annotations

import importlib.util
import json
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def _load_svd():
    spec = importlib.util.spec_from_file_location("ref_bm_svd", os.path.join(ref_loader.REF, "svd.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def model_from_spec(spec):
    """the module a fixture's `model` JSON describes, built with the drop-in package or torch.nn (the same module walk as
    the reference's)"""
    kind, kw = spec["kind"], spec["kwargs"]
    if kind == "SimpleConv":
        import brainmagick_b200 as bb
        return bb.SimpleConv(**kw)
    if kind == "ConvSequence":
        import brainmagick_b200 as bb
        return bb.ConvSequence(**kw)
    layers = []
    for name, args in kw["layers"]:
        layers.append(getattr(torch.nn, name)(*args))
    return torch.nn.Sequential(*layers)


def walk(model):
    return [m.weight for _, m in model.named_modules()
            if isinstance(m, (torch.nn.modules.conv._ConvNd, torch.nn.Linear))]


LAYERS = dict(kind="Sequential", kwargs=dict(layers=[["Linear", [30, 50]], ["ConvTranspose1d", [24, 40, 3]],
                                                     ["Conv1d", [8, 60, 5]], ["Linear", [16, 16]], ["Linear", [4, 4]],
                                                     ["Conv1d", [3, 5, 1]]]))
CASES = {
    "clip_conv": (dict(kind="SimpleConv", kwargs=dict(
        in_channels=dict(meg=20), out_channels=48, n_subjects=3,
        **ref_loader.clip_conv_kwargs(hidden=40, depth=4, merger_channels=24, initial_linear=24, merger_pos_dim=32))),
        1.0, 1, [], [11, 12]),
    "residual": (dict(kind="ConvSequence", kwargs=dict(channels=[24, 24, 24, 24], kernel=3, stride=1, skip=True,
                                                       rewrite=True, post_skip=True, scale=0.1, batch_norm=True)),
                 0.01, 1, [], [21]),
    "layers": (LAYERS, 1.0, 1, [], [31, 32]),
    "frozen": (LAYERS, 1.0, 1, [0, 2], [41]),
    "proba": (LAYERS, 1.0, 0.5, [], [51 + c for c in range(8)]),
}


def reference_model(spec):
    """the same module built by the verbatim reference (bm/models) or torch.nn"""
    common, sc, _ = ref_loader.load_reference()
    if spec["kind"] == "SimpleConv":
        return sc.SimpleConv(**spec["kwargs"])
    if spec["kind"] == "ConvSequence":
        return common.ConvSequence(**spec["kwargs"])
    return model_from_spec(spec)


def make(name):
    spec, min_size, proba, frozen, seeds = CASES[name]
    ref = _load_svd()
    torch.manual_seed(7)
    model = reference_model(spec)
    weights = walk(model)
    for i in frozen:
        weights[i].requires_grad_(False)
    out = dict(model=np.array(json.dumps(spec)), min_size=np.array(min_size), proba=np.array(float(proba)),
               frozen=np.array(frozen, dtype=np.int64), calls=np.array(len(seeds)))
    for i, w in enumerate(weights):
        out[f"w_{i}"] = w.detach().numpy().copy()
    ref.penalty_rng = random.Random(1234)
    randn = torch.randn
    for c, seed in enumerate(seeds):
        draws = []

        def recording_randn(*a, **k):
            t = randn(*a, **k)
            draws.append(t.detach().clone())
            return t
        torch.manual_seed(seed)
        torch.randn = recording_randn
        try:
            value = ref.svd_penalty(model, min_size=min_size, proba=proba)
        finally:
            torch.randn = randn
        grads = [torch.zeros_like(w) for w in weights]
        if isinstance(value, torch.Tensor):
            live = [w for w in weights if w.requires_grad]
            gs = torch.autograd.grad(value, live, allow_unused=True)
            for w, g in zip(live, gs):
                if g is not None:
                    grads[next(i for i, x in enumerate(weights) if x is w)] = g
            out[f"value_{c}"] = np.array(float(value))
        else:
            out[f"value_{c}"] = np.array(float("nan"))
        out[f"seed_{c}"] = np.array(seed)
        out[f"draws_{c}"] = np.array(len(draws))
        for k, r in enumerate(draws):
            out[f"r_{c}_{k}"] = r.numpy()
        for i, g in enumerate(grads):
            out[f"g_{c}_{i}"] = g.numpy()
    np.savez_compressed(os.path.join(OUT, f"svd_{name}.npz"), **out)
    print(name, [float(out[f"value_{c}"]) for c in range(len(seeds))])


if __name__ == "__main__":
    for name in CASES:
        make(name)
