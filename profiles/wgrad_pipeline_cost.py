"""The conv weight gradients of the cfg2 training step (bm_tc_wgrad_conv and its `_tf32` form) at B = 256, T = 360:

  K3    320 -> 320, k = 3, dilation 4  (10 per step)
  K4    320 -> 640, k = 3              (the GLU convs, 5 per step)
  head  1024 -> 640, k = 1             (one per step)

each timed as bench._time_kernel does (CUDA events around back-to-back launches over rotating operand sets larger than L2),
in `--rounds` rounds; then the cfg2 and cfg4 training steps (bench.py's model and optimizer, 3xTF32).  `--lib PATH` loads
that build of libbm_b200.so instead of the in-tree one, so that one GPU command can alternate two builds in separate
processes.  `--dump DIR` also writes dW of seeded operands at the three shapes, both pass counts, as DIR/<shape><form>.npy,
for a bitwise comparison of two builds.

    python profiles/wgrad_pipeline_cost.py [--lib PATH] [--rounds 3] [--steps 20] [--dump DIR] [--out result.json]

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

from brainmagick_b200 import _lib  # noqa: E402

SHAPES = {  # name: dy channels, x channels, taps, dilation
    "k3": (320, 320, 3, 4),
    "k4": (640, 320, 3, 1),
    "head": (640, 1024, 1, 1),
}
NSETS = 3


def kernels(args, dev):
    from brainmagick_b200._lib import call, ptr, stream
    import bench
    lib = _lib.load()
    B, T = args.batch, 360
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    res = {}
    for name, (M, N, Kw, dil) in SHAPES.items():
        g = torch.Generator(device=dev).manual_seed(17)
        sets = [(torch.randn(B, T, M, device=dev, generator=g), torch.randn(B, T, N, device=dev, generator=g))
                for _ in range(NSETS)]
        ws = torch.empty(int(lib.bm_tc_wgrad_conv_workspace(B, T, M, N, Kw)), device=dev)
        dw = torch.empty(M, N, Kw, device=dev)

        def fns(suffix):
            return [lambda dy=dy, x=x: call("bm_tc_wgrad_conv" + suffix, ptr(dy), ptr(x), B, T, M, N, N, Kw, dil, ptr(ws),
                                            ptr(dw), ptr(status), stream()) for dy, x in sets]
        times = {"3xtf32": [], "tf32": []}
        for _ in range(args.rounds):
            for form, suffix in (("3xtf32", ""), ("tf32", "_tf32")):
                times[form].append(round(bench._time_kernel(fns(suffix), iters=args.iters), 4))
        res[name] = dict(ms=times, gflop=2.0 * M * N * Kw * B * T / 1e9)
        if args.dump:
            os.makedirs(args.dump, exist_ok=True)
            dy, x = sets[0]
            for suffix in ("", "_tf32"):
                call("bm_tc_wgrad_conv" + suffix, ptr(dy), ptr(x), B, T, M, N, N, Kw, dil, ptr(ws), ptr(dw), ptr(status),
                     stream())
                torch.cuda.synchronize()
                import numpy as np
                np.save(os.path.join(args.dump, name + suffix + ".npy"), dw.cpu().numpy())
        del sets, ws, dw
        torch.cuda.empty_cache()
    torch.cuda.synchronize()
    assert int(status.item()) == 0, f"pipeline status {int(status.item())}"
    return res


def step_ms(cfg_name, args, dev):
    import bench
    import brainmagick_b200 as bb
    from brainmagick_b200 import functional as BF, synthetic
    from profiles.input_grad_cost import timed_ms
    cfg = bench.CONFIGS[cfg_name]
    B = args.batch
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
    model.train()
    clip.train()

    def step():
        opt.zero_grad(set_to_none=True)
        clip(model(dict(meg=meg), batch), feats, mask).backward()
        opt.step()
    for _ in range(args.warmup):
        step()
    out = [round(timed_ms(step, args.steps), 2) for _ in range(args.rounds)]
    BF.check_tc_status()
    del model, clip, opt
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default="", help="path of the libbm_b200.so to load (default: the in-tree build)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=24)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--no-steps", action="store_true", help="time the kernels only")
    ap.add_argument("--dump", default="")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    assert torch.cuda.is_available(), "profiles/wgrad_pipeline_cost.py measures on cuda:0"
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    from profiles.input_grad_cost import card
    res = dict(card=card(), lib=_lib.LIB_PATH, batch=args.batch)
    res["kernels"] = kernels(args, dev)
    if not args.no_steps:
        res["step_ms"] = {c: step_ms(c, args, dev) for c in ("cfg2", "cfg4")}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
