"""What torch.autocast(dtype=torch.bfloat16) buys (the `_bf16` entry points) against the two existing forms, 3xTF32 (the
default) and single-pass TF32 (torch.set_float32_matmul_precision("high")), at cfg2 and cfg4, B = 256, with bench.py's model
and optimizer:

  step_ms    training step (forward and ClipLoss under the mode, backward, fused Adam)
  eval_ms    eval forward (no_grad)

and, with CUDA events over repeated launches at cfg2 sizes:

  conv_fwd_ms     one 320 -> 320, k = 3 conv forward at B = 256, T = 360 (bm_tc_conv1d_persistent[_tf32 | _bf16])
  conv_wgrad_ms   its weight gradient (bm_tc_wgrad_conv[_tf32 | _bf16])
  clip_scores_ms  the CLIP scores, 256 x 256 over F * T = 368 640 (bm_clip_scores[_tf32 | _bf16])

Each round runs in a process of its own (module loads, allocator and clocks start afresh) and alternates the three modes
inside it, so that drift on a shared machine hits all three; the rounds' spread is the noise to compare a difference with.

    python profiles/bf16_cost.py [--steps 20] [--rounds 3] [--out result.json]

Prints one JSON line; the card's name and power limit are part of it.  Needs cuda:0.
"""
from __future__ import annotations

import argparse
import contextlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

MODES = ("3xtf32", "tf32", "bf16")
SUFFIX = {"3xtf32": "", "tf32": "_tf32", "bf16": "_bf16"}


@contextlib.contextmanager
def mode_ctx(mode):
    from brainmagick_b200 import _lib
    torch.set_float32_matmul_precision("high" if mode == "tf32" else "highest")
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "bf16"):
        assert _lib.tf32() == (mode == "tf32") and _lib.bf16() == (mode == "bf16")
        yield
    torch.set_float32_matmul_precision("highest")


def measure(cfg_name, B, args, dev):
    import bench
    import brainmagick_b200 as bb
    from brainmagick_b200 import functional as BF, synthetic
    from profiles.input_grad_cost import timed_ms
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

    def step(mode):
        opt.zero_grad(set_to_none=True)
        with mode_ctx(mode):
            loss = clip(model(dict(meg=meg), batch), feats, mask)
        loss.backward()
        opt.step()

    def evaluate(mode):
        with mode_ctx(mode), torch.no_grad():
            model(dict(meg=meg), batch)

    res = {}
    for name, fn, train in (("step_ms", step, True), ("eval_ms", evaluate, False)):
        model.train(train)
        clip.train(train)
        for mode in MODES:
            for _ in range(args.warmup):
                fn(mode)
        res[name] = {mode: round(timed_ms(lambda: fn(mode), args.steps), 2) for mode in MODES}
    BF.check_tc_status()
    return res


def kernels(args, dev):
    """Single entry points at cfg2 sizes in each form."""
    from brainmagick_b200 import _lib, functional as BF
    from brainmagick_b200._lib import call, ptr, stream
    from profiles.input_grad_cost import timed_ms
    lib = _lib.load()
    B, T, H, Kw, KT = 256, 360, 320, 3, 1024 * 360
    g = torch.Generator(device=dev).manual_seed(5)
    x, dy = torch.randn(B, T, H, device=dev, generator=g), torch.randn(B, T, H, device=dev, generator=g)
    w = torch.randn(H, H, Kw, device=dev, generator=g) / (H * Kw) ** 0.5
    f = torch.empty(Kw, H, H, device=dev)
    call("bm_tc_weight_split", ptr(w), H, H, Kw, ptr(f), None, None, None, stream())
    y = torch.empty(B, T, H, device=dev)
    status = BF.tc_status_tensor(dev)
    ws = torch.empty(int(lib.bm_tc_wgrad_conv_workspace(B, T, H, H, Kw)), device=dev)
    dw = torch.empty(H, H, Kw, device=dev)
    est, cand = torch.randn(256, KT, device=dev, generator=g), torch.randn(256, KT, device=dev, generator=g)
    inv, sc = torch.empty(256, device=dev), torch.empty(256, 256, device=dev)
    cws = torch.empty(int(lib.bm_clip_workspace(256, 256, KT)), device=dev)
    fns = {
        "conv_fwd_ms": lambda s: call("bm_tc_conv1d_persistent" + s, ptr(x), ptr(f), None, 0, B, T, H, H, Kw, 4, 1, 0, 0, 0,
                                      ptr(y), None, None, None, ptr(status), stream()),
        "conv_wgrad_ms": lambda s: call("bm_tc_wgrad_conv" + s, ptr(dy), ptr(x), B, T, H, H, H, Kw, 4, ptr(ws), ptr(dw),
                                        ptr(status), stream()),
        "clip_scores_ms": lambda s: call("bm_clip_scores" + s, ptr(est), ptr(cand), 256, 256, KT, 0, ptr(inv), ptr(sc), None,
                                         ptr(cws), cws.numel(), ptr(status), stream()),
    }
    res = {}
    for name, fn in fns.items():
        for mode in MODES:
            for _ in range(3):
                fn(SUFFIX[mode])
        res[name] = {mode: round(timed_ms(lambda: fn(SUFFIX[mode]), 4 * args.steps), 3) for mode in MODES}
    BF.check_tc_status()
    return res


def one_round(args):
    """One round, in this process: every mode of every measurement."""
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {cfg_name: measure(cfg_name, args.batch, args, dev) for cfg_name in ("cfg2", "cfg4")}
    res["kernels_cfg2"] = kernels(args, dev)
    return res


def merge(rounds):
    """[{group: {name: {mode: ms}}}] -> {group: {name: {mode: [ms per round]}}}"""
    out = {}
    for r in rounds:
        for group, names in r.items():
            for name, modes in names.items():
                for mode, ms in modes.items():
                    out.setdefault(group, {}).setdefault(name, {}).setdefault(mode, []).append(ms)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--out", default="")
    ap.add_argument("--one-round", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/bf16_cost.py measures on cuda:0"
    if args.one_round:
        print(json.dumps(one_round(args)))
        return
    from profiles.input_grad_cost import card
    rounds = []
    for _ in range(args.rounds):
        cmd = [sys.executable, os.path.abspath(__file__), "--one-round", "--steps", str(args.steps), "--warmup",
               str(args.warmup), "--batch", str(args.batch)]
        out = subprocess.run(cmd, check=True, capture_output=True, text=True, cwd=ROOT).stdout
        rounds.append(json.loads(out.strip().splitlines()[-1]))
    res = dict(card=card(), batch=args.batch, steps_per_round=args.steps, rounds=args.rounds, **merge(rounds))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
