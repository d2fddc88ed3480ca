"""What backpropagating to `meg` costs at cfg2 (B = 256, 208 sensors, T = 360, F = 1024; bench.py's model and optimizer):

  step            one training step (forward, ClipLoss, backward, Adam) with meg.requires_grad False, then True; the two
                  are timed in alternating rounds so that drift on a shared machine hits both
  attribution     a frozen model (requires_grad_(False)) in eval mode: forward, get_scores, backward of the true
                  candidates' scores to meg -- the gradient-based attribution pass
  eval_forward    the same forward under torch.no_grad(), for scale

The input gradient adds the sensor-mix data gradient, about 2*T*Op*Cp = 2*360*320*256 = 59 MFLOP per segment.

    python profiles/input_grad_cost.py [--steps 20] [--rounds 3] [--out result.json]

Prints one JSON line; the card's name and power limit are part of it.  Needs cuda:0.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
import brainmagick_b200 as bb  # noqa: E402
from brainmagick_b200 import functional as BF, synthetic  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def timed_ms(fn, n):
    """Mean device time per call of fn over n calls (CUDA events around the whole window)."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/input_grad_cost.py measures on cuda:0"
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

    def step(meg_grad):
        x = meg.detach().requires_grad_(meg_grad)
        opt.zero_grad(set_to_none=True)
        clip(model(dict(meg=x), batch_of(x.detach())), feats, mask).backward()
        opt.step()

    model.train()
    clip.train()
    for _ in range(args.warmup):
        step(False)
        step(True)
    plain, with_grad = [], []
    for _ in range(args.rounds):
        plain.append(timed_ms(lambda: step(False), args.steps))
        with_grad.append(timed_ms(lambda: step(True), args.steps))

    model.eval().requires_grad_(False)
    clip.eval()

    def attribution():
        x = meg.detach().requires_grad_(True)
        scores = clip.get_scores(model(dict(meg=x), batch_of(x.detach())), feats)
        scores.diagonal().sum().backward()

    def eval_forward():
        with torch.no_grad():
            model(dict(meg=meg), batch_of(meg))

    for _ in range(args.warmup):
        attribution()
        eval_forward()
    attr, fwd = [], []
    for _ in range(args.rounds):
        attr.append(timed_ms(attribution, args.steps))
        fwd.append(timed_ms(eval_forward, args.steps))
    BF.check_tc_status()
    res = dict(card=card(), config="cfg2", batch=B, steps_per_round=args.steps,
               step_ms=[round(v, 2) for v in plain], step_meg_grad_ms=[round(v, 2) for v in with_grad],
               attribution_ms=[round(v, 2) for v in attr], eval_forward_ms=[round(v, 2) for v in fwd],
               added_mflop_per_segment=round(2 * T * 320 * 256 / 1e6, 1))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
