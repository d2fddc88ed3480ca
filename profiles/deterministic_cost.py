"""What torch.use_deterministic_algorithms(True) costs a training step (forward, ClipLoss, backward, Adam; bench.py's model and
optimizer) at cfg2 and cfg4, B = 256:

  off         the default call stream (atomic reductions)
  on          the deterministic forms, with torch's NaN fill of torch.empty (torch.utils.deterministic.
              fill_uninitialized_memory, on by default under the flag)
  on_nofill   the deterministic forms without the fill

The three modes are timed in alternating rounds in one process so that drift on a shared machine hits all of them.

    python profiles/deterministic_cost.py [--steps 20] [--rounds 3] [--out result.json]

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
import torch.utils.deterministic  # noqa: E402

import bench  # noqa: E402
import brainmagick_b200 as bb  # noqa: E402
from brainmagick_b200 import functional as BF, synthetic  # noqa: E402
from profiles.input_grad_cost import card, timed_ms  # noqa: E402

MODES = {"off": (False, True), "on": (True, True), "on_nofill": (True, False)}   # (flag, NaN fill)


def set_mode(mode):
    flag, fill = MODES[mode]
    torch.use_deterministic_algorithms(flag)
    torch.utils.deterministic.fill_uninitialized_memory = fill


def measure(cfg_name, B, args, dev):
    cfg = bench.CONFIGS[cfg_name]
    C, T, F, S = cfg["C"], cfg["T"], cfg["F"], cfg["S"]
    torch.manual_seed(2036)
    model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, n_subjects=S,
                          **{k: (dict(v) if isinstance(v, dict) else v) for k, v in bench.CLIP_CONV.items()}).to(dev)
    clip = bb.ClipLoss().to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=3e-4, betas=(0.9, 0.999), fused=True)
    positions = synthetic.normalised_positions(S, C, seed=7)
    recs = [synthetic.SyntheticRecording(s, positions[s]) for s in range(S)]
    meg, feats, subj = (t.to(dev) for t in bench.make_host_batch(cfg, B, 2036))
    batch = synthetic.SyntheticBatch(meg, subj, [recs[s] for s in subj.tolist()])
    mask = torch.ones(B, 1, T, dtype=torch.bool, device=dev)

    def step():
        opt.zero_grad(set_to_none=True)
        clip(model(dict(meg=meg), batch), feats, mask).backward()
        opt.step()

    model.train()
    clip.train()
    for mode in MODES:
        set_mode(mode)
        for _ in range(args.warmup):
            step()
    times = {m: [] for m in MODES}
    for _ in range(args.rounds):
        for mode in MODES:
            set_mode(mode)
            times[mode].append(round(timed_ms(step, args.steps), 2))
    set_mode("off")
    BF.check_tc_status()
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/deterministic_cost.py measures on cuda:0"
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = dict(card=card(), batch=args.batch, steps_per_round=args.steps)
    for cfg_name in ("cfg2", "cfg4"):
        res[cfg_name + "_step_ms"] = measure(cfg_name, args.batch, args, dev)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
