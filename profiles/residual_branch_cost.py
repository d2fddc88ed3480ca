"""What ConvSequence's residual-branch options cost in a SimpleConv training step, at cfg2 (B = 256, 208 sensors, T = 360,
F = 1024; bench.py's model and optimizer):

  baseline     clip_conv as bench.py builds it
  scale        + LayerScale(0.1) on every layer that keeps its width (scale=0.1)
  post_skip    + the depthwise 1x1 gain (post_skip=True)
  rewrite      + a 320 -> 320 1x1 conv and LeakyReLU in every residual branch (rewrite=True)
  all          the three together

Every model is built from the same seed; their steps (forward, ClipLoss, backward, Adam) are timed in alternating rounds so
that drift on a shared machine hits all of them.

    python profiles/residual_branch_cost.py [--steps 20] [--rounds 3] [--out result.json]

Prints one JSON line; the card's name and power limit are part of it.  Needs cuda:0.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
import brainmagick_b200 as bb  # noqa: E402
from brainmagick_b200 import functional as BF, synthetic  # noqa: E402
from profiles.input_grad_cost import card, timed_ms  # noqa: E402

VARIANTS = {"baseline": {}, "scale": dict(scale=0.1), "post_skip": dict(post_skip=True), "rewrite": dict(rewrite=True),
            "all": dict(scale=0.1, post_skip=True, rewrite=True)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/residual_branch_cost.py measures on cuda:0"
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    cfg = bench.CONFIGS["cfg2"]
    B, C, T, F, S = 256, cfg["C"], cfg["T"], cfg["F"], cfg["S"]
    positions = synthetic.normalised_positions(S, C, seed=7)
    recs = [synthetic.SyntheticRecording(s, positions[s]) for s in range(S)]
    meg, feats, subj = (t.to(dev) for t in bench.make_host_batch(cfg, B, 2036))
    batch = synthetic.SyntheticBatch(meg, subj, [recs[s] for s in subj.tolist()])
    mask = torch.ones(B, 1, T, dtype=torch.bool, device=dev)
    clip = bb.ClipLoss().to(dev).train()

    def step_of(extra):
        torch.manual_seed(2036)
        kw = {k: (dict(v) if isinstance(v, dict) else v) for k, v in bench.CLIP_CONV.items()}
        kw.update(extra)
        model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, n_subjects=S, **kw).to(dev).train()
        opt = torch.optim.Adam(model.parameters(), lr=3e-4, betas=(0.9, 0.999), fused=True)

        def fn():
            opt.zero_grad(set_to_none=True)
            clip(model(dict(meg=meg), batch), feats, mask).backward()
            opt.step()
        return fn

    runs = {k: step_of(v) for k, v in VARIANTS.items()}
    for _ in range(args.warmup):
        for fn in runs.values():
            fn()
    times = {k: [] for k in runs}
    for _ in range(args.rounds):
        for k, fn in runs.items():
            times[k].append(timed_ms(fn, args.steps))
    BF.check_tc_status()
    best = {k: min(v) for k, v in times.items()}
    res = dict(card=card(), config="cfg2", batch=B, steps_per_round=args.steps)
    res.update({k + "_ms": [round(v, 2) for v in vs] for k, vs in times.items()})
    res.update({k + "_over_baseline": round(best[k] / best["baseline"] - 1, 4) for k in runs if k != "baseline"})
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
