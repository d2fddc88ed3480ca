"""Where the device time of one training step goes, per kernel: bench.py's model and optimizer at cfg2 (or --config), B = 256,
warmed up, then `--steps` steps under torch.profiler (CUDA activity).  Sums the device time of every kernel launch by kernel
name and prints one JSON line: the card, the profiled steps' summed kernel time (kernels on the side streams overlap the
main stream, so this exceeds the step's wall time) and the `--top` names with their total ms per step and launch count.
A profiled run is slower than bench.py's timed steps: take times from bench.py, the split from here.

    python profiles/step_kernels.py [--lib PATH] [--config cfg2] [--steps 2] [--top 25] [--out result.json]
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from brainmagick_b200 import _lib  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default="", help="path of the libbm_b200.so to load (default: the in-tree build)")
    ap.add_argument("--config", default="cfg2")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--top", type=int, default=25)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    assert torch.cuda.is_available(), "profiles/step_kernels.py profiles on cuda:0"
    import bench
    import brainmagick_b200 as bb
    from brainmagick_b200 import functional as BF, synthetic
    from profiles.input_grad_cost import card
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    cfg = bench.CONFIGS[args.config]
    B = args.batch
    C, T, F, S = cfg["C"], cfg["T"], cfg["F"], cfg["S"]
    torch.manual_seed(2036)
    model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, n_subjects=S,
                          **{k: (dict(v) if isinstance(v, dict) else v) for k, v in bench.CLIP_CONV.items()}).to(dev)
    clip = bb.ClipLoss().to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=3e-4, betas=(0.9, 0.999), fused=True)
    positions = synthetic.normalised_positions(S, C, n_valid=cfg["n_valid"], seed=7)
    recs = [synthetic.SyntheticRecording(s, positions[s]) for s in range(S)]
    meg, feats, subj = (t.to(dev) for t in bench.make_host_batch(cfg, B, 2036))
    batch = synthetic.SyntheticBatch(meg, subj, [recs[s] for s in subj.tolist()])
    mask = torch.ones(B, 1, T, dtype=torch.bool, device=dev)
    model.train()
    clip.train()

    def step():
        opt.zero_grad(set_to_none=True)
        clip(model(dict(meg=meg), batch), feats, mask).backward()
        opt.step()
    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    BF.check_tc_status()
    total_us, count = collections.Counter(), collections.Counter()
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and ev.device_time > 0:
            name = ev.name if len(ev.name) <= 160 else ev.name[:157] + "..."
            total_us[name] += ev.device_time
            count[name] += 1
    summed = sum(total_us.values()) / 1e3 / args.steps
    top = [dict(kernel=n, ms_per_step=round(us / 1e3 / args.steps, 3), launches_per_step=count[n] / args.steps)
           for n, us in total_us.most_common(args.top)]
    res = dict(card=card(), lib=_lib.LIB_PATH, config=args.config, batch=B, steps=args.steps,
               kernel_ms_per_step=round(summed, 3), top=top)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
