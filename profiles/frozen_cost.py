"""What a backward costs when part of the model is frozen, at cfg2 (B = 256, 208 sensors, T = 360, F = 1024; bench.py's model
and optimizer), each timed in alternating rounds so that drift on a shared machine hits all of them:

  full_step        forward, ClipLoss, backward, Adam with every parameter trainable
  head_step        the same with only the head (final.*) trainable: linear probing / head-only fine-tuning
  subject_step     only subject_layers.weights trainable: adapting a trained model to new subjects
  attribution      a frozen model in eval mode: forward, get_scores, backward of the true candidates' scores to meg
  eval_forward     the same forward under torch.no_grad()

and the peak memory (torch.cuda.max_memory_allocated above what was allocated before) of each.

    python profiles/frozen_cost.py [--steps 20] [--rounds 3] [--out result.json]

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/frozen_cost.py measures on cuda:0"
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    cfg = bench.CONFIGS["cfg2"]
    B, C, T, F, S = 256, cfg["C"], cfg["T"], cfg["F"], cfg["S"]
    torch.manual_seed(2036)
    model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, n_subjects=S,
                          **{k: (dict(v) if isinstance(v, dict) else v) for k, v in bench.CLIP_CONV.items()}).to(dev)
    clip = bb.ClipLoss().to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=3e-4, betas=(0.9, 0.999), fused=True)
    positions = synthetic.normalised_positions(S, C, seed=7)
    recs = [synthetic.SyntheticRecording(s, positions[s]) for s in range(S)]
    meg, feats, subj = (t.to(dev) for t in bench.make_host_batch(cfg, B, 2036))
    subj_h = subj.tolist()
    mask = torch.ones(B, 1, T, dtype=torch.bool, device=dev)

    def batch_of(x):
        return synthetic.SyntheticBatch(x, subj, [recs[s] for s in subj_h])

    def trainable(which):
        for name, p in model.named_parameters():
            p.requires_grad_(which == "full" or (which == "head" and name.startswith("final.")) or
                             (which == "subject" and name == "subject_layers.weights"))

    def step(which):
        def fn():
            trainable(which)
            opt.zero_grad(set_to_none=True)
            clip(model(dict(meg=meg), batch_of(meg)), feats, mask).backward()
            opt.step()
        return fn

    def attribution():
        x = meg.detach().requires_grad_(True)
        scores = clip.get_scores(model(dict(meg=x), batch_of(x.detach())), feats)
        scores.diagonal().sum().backward()

    def eval_forward():
        with torch.no_grad():
            model(dict(meg=meg), batch_of(meg))

    def peak_mb(fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fn()
        torch.cuda.synchronize()
        return round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)

    train_runs = {"full_step": step("full"), "head_step": step("head"), "subject_step": step("subject")}
    model.train()
    clip.train()
    for _ in range(args.warmup):
        for fn in train_runs.values():
            fn()
    times = {k: [] for k in list(train_runs) + ["attribution", "eval_forward"]}
    peaks = {k: peak_mb(fn) for k, fn in train_runs.items()}
    for _ in range(args.rounds):
        for k, fn in train_runs.items():
            times[k].append(timed_ms(fn, args.steps))

    model.eval().requires_grad_(False)
    clip.eval()
    eval_runs = {"attribution": attribution, "eval_forward": eval_forward}
    for _ in range(args.warmup):
        for fn in eval_runs.values():
            fn()
    peaks.update({k: peak_mb(fn) for k, fn in eval_runs.items()})
    for _ in range(args.rounds):
        for k, fn in eval_runs.items():
            times[k].append(timed_ms(fn, args.steps))
    BF.check_tc_status()
    res = dict(card=card(), config="cfg2", batch=B, steps_per_round=args.steps)
    res.update({k + "_ms": [round(v, 2) for v in vs] for k, vs in times.items()})
    res.update({k + "_peak_mb": v for k, v in peaks.items()})
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
