"""What an encoding training step costs (bm/train.py:61-67, bm/solver.py:283-294: SimpleConv over `meg` and `features`,
trained with an L1 loss against the MEG itself), next to the decoding step of bench.py's cfg2, at B = 256:

  decode_step        cfg2: 208 sensors, T = 360, F = 1024, ClipLoss, fused Adam (bench.py's model and optimizer)
  encode_step        meg 208 + features 120 (mel), hidden 320 per stream, complex_out, out_channels 208, torch's L1 loss
                     on the output, fused Adam
  encode_linear_step the same with linear_out
  encode_concat_step the same as encode_step with concatenate: one encoder over the joined streams (hidden 640)

each timed in alternating rounds so that drift on a shared machine hits all of them.  Then, for encode_step:
  join_split_ms      device time of the channel join / split kernels in one step (torch.profiler, CUDA kernels named
                     channel_join_kernel), and their share of the step
  head_ms            the complex_out head (forward + backward) timed alone at the step's shapes with CUDA events; at
                     out_channels 208 its convs miss the tensor-core gates and it runs the FP32-FMA `fma` form
  linear_head_ms     the same for linear_out's single 1x1 ConvTranspose (FP32-FMA `_Conv`s at 208 outputs)
and the bytes the join / split move per step.

    python profiles/encode_cost.py [--steps 10] [--rounds 3] [--out result.json]

Prints one JSON line; the card's name and power limit are part of it.  Needs cuda:0.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
import brainmagick_b200 as bb  # noqa: E402
from brainmagick_b200 import functional as BF, synthetic  # noqa: E402
from oracle.encode_oracle import EncodeVariant  # noqa: E402
from profiles.input_grad_cost import card, timed_ms  # noqa: E402

FEATURES, HIDDEN = 120, 320


def join_split_bytes(B, T, F_in, hidden):
    """Bytes the join / split kernels read and write in one encoding step (fp32): the features stream into its encoder's
    padded input (read C, write the padded width), the two encoder outputs into the head's input (read and write 2H), the
    head input gradient split back (2H both ways), and features.grad is not asked for in training."""
    pad = BF._round_up(F_in, 64)
    rows = B * T
    return 4 * rows * ((F_in + pad) + 2 * (2 * hidden) + 2 * (2 * hidden))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/encode_cost.py measures on cuda:0"
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    cfg = bench.CONFIGS["cfg2"]
    B, C, T, F, S = 256, cfg["C"], cfg["T"], cfg["F"], cfg["S"]
    positions = synthetic.normalised_positions(S, C, seed=7)
    recs = [synthetic.SyntheticRecording(s, positions[s]) for s in range(S)]
    meg, feats, subj = (t.to(dev) for t in bench.make_host_batch(cfg, B, 2036))
    subj_h = subj.tolist()
    mask = torch.ones(B, 1, T, dtype=torch.bool, device=dev)
    mel_full = torch.randn(B, FEATURES, T + 60, device=dev)
    mel = mel_full[:, :, 30:30 + T]                              # the solver's offset crop: a view

    def batch_of(x):
        return synthetic.SyntheticBatch(x, subj, [recs[s] for s in subj_h])

    torch.manual_seed(2036)
    dec = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, n_subjects=S,
                        **{k: (dict(v) if isinstance(v, dict) else v) for k, v in bench.CLIP_CONV.items()}).to(dev).train()
    clip = bb.ClipLoss().to(dev).train()
    dec_opt = torch.optim.Adam(dec.parameters(), lr=3e-4, betas=(0.9, 0.999), fused=True)

    def encoder(linear, concatenate=False):
        v = EncodeVariant(in_channels=dict(meg=C, features=FEATURES), hidden=dict(meg=HIDDEN, features=HIDDEN),
                          out_channels=C, n_subjects=S, linear_out=linear, complex_out=not linear, concatenate=concatenate)
        torch.manual_seed(2036)
        model = bb.SimpleConv(**v.kwargs()).to(dev).train()
        return model, torch.optim.Adam(model.parameters(), lr=3e-4, betas=(0.9, 0.999), fused=True)
    enc, enc_opt = encoder(False)
    lin, lin_opt = encoder(True)
    cat, cat_opt = encoder(False, concatenate=True)

    def decode_step():
        dec_opt.zero_grad(set_to_none=True)
        clip(dec(dict(meg=meg), batch_of(meg)), feats, mask).backward()
        dec_opt.step()

    def encode_step(model, opt):
        def fn():
            opt.zero_grad(set_to_none=True)
            out = model(dict(meg=meg, features=mel), batch_of(meg))
            torch.nn.functional.l1_loss(out, meg).backward()
            opt.step()
        return fn

    runs = {"decode_step": decode_step, "encode_step": encode_step(enc, enc_opt),
            "encode_linear_step": encode_step(lin, lin_opt), "encode_concat_step": encode_step(cat, cat_opt)}
    for _ in range(args.warmup):
        for fn in runs.values():
            fn()
    times = {k: [] for k in runs}
    for _ in range(args.rounds):
        for k, fn in runs.items():
            times[k].append(timed_ms(fn, args.steps))

    # the join / split kernels inside one encode step
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            runs["encode_step"]()
        torch.cuda.synchronize()
    join_us = sum(e.self_device_time_total for e in prof.key_averages() if "channel_join_kernel" in e.key)
    join_ms = join_us / 1000 / args.steps

    # the heads alone, at the step's shapes
    status = BF.tc_status_tensor(dev)
    plan = types.SimpleNamespace(act_code=BF.ACT_GELU, act_slope=0.0, use_tensor_cores=True)
    nd = types.SimpleNamespace(head=(True,) * 4, below=[True])
    H = 2 * HIDDEN
    x = torch.randn(B, T, H, device=dev)
    dest = torch.randn(B, C, T, device=dev)
    side = BF._side_stream(dev)

    def head_params(module, linear):
        if linear:
            return None, None, module.weight, module.bias
        return module[0].weight, module[0].bias, module[2].weight, module[2].bias

    def head_step(module, linear):
        params = head_params(module, linear)

        def fn():
            _, rec = BF.head_forward(plan, x, *params, nd, True, B, T, status)
            BF.head_backward(plan, rec, dest, nd.head, B, T, status, side, [])
            torch.cuda.current_stream().wait_stream(side)
        return fn, BF.head_forward(plan, x, *params, nd, True, B, T, status)[1]["form"]

    head_fn, head_form = head_step(enc.final, False)
    lin_fn, lin_form = head_step(lin.final, True)
    for _ in range(args.warmup):
        head_fn()
        lin_fn()
    head_ms = min(timed_ms(head_fn, args.steps) for _ in range(args.rounds))
    lin_ms = min(timed_ms(lin_fn, args.steps) for _ in range(args.rounds))
    BF.check_tc_status()

    enc_ms = min(times["encode_step"])
    res = dict(card=card(), batch=B, T=T, meg=C, features=FEATURES, hidden=HIDDEN, steps_per_round=args.steps)
    res.update({k + "_ms": [round(v, 2) for v in vs] for k, vs in times.items()})
    res.update(join_split_ms=round(join_ms, 3), join_split_share=round(join_ms / enc_ms, 4),
               join_split_bytes=join_split_bytes(B, T, FEATURES, HIDDEN),
               join_split_gbps=round(join_split_bytes(B, T, FEATURES, HIDDEN) / (join_ms * 1e-3) / 1e9, 1),
               head_form=head_form, head_ms=round(head_ms, 2), head_share=round(head_ms / enc_ms, 4),
               linear_head_form=lin_form, linear_head_ms=round(lin_ms, 2),
               linear_head_share=round(lin_ms / min(times["encode_linear_step"]), 4))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
