"""What nn.SyncBatchNorm costs a two-rank training step (forward, ClipLoss, backward, gradient all-reduce, Adam; bench.py's
model and optimizer) at cfg3 with B = 64 per rank, over NCCL, one GPU per rank:

  plain       SimpleConv as constructed (per-rank BatchNorm statistics)
  sync        the same model after torch.nn.SyncBatchNorm.convert_sync_batchnorm (two all-reduces of 2C + 1 fp64 per
              BatchNorm layer and step)

The two are timed in alternating rounds in one run so that drift on a shared machine hits both.  With fewer than two GPUs
visible nothing is measured: NCCL needs one GPU per rank, and two gloo ranks sharing one GPU time the host copies of gloo,
not the step.

    python profiles/syncbn_cost.py [--steps 20] [--rounds 3] [--out result.json]

Prints one JSON line; the card's name and power limit are part of it.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
import torch.multiprocessing as mp  # noqa: E402

from profiles.input_grad_cost import card, timed_ms  # noqa: E402

WORLD, BATCH = 2, 64


def _rank(rank, args, init, ret):
    sys.path.insert(0, ROOT)
    import bench
    import brainmagick_b200 as bb
    from brainmagick_b200 import distrib, functional as BF, synthetic
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", init_method=init, rank=rank, world_size=WORLD)
    try:
        cfg = bench.CONFIGS["cfg3"]
        C, T, F, S = cfg["C"], cfg["T"], cfg["F"], cfg["S"]
        positions = synthetic.normalised_positions(S, C, seed=7)
        recs = [synthetic.SyntheticRecording(s, positions[s]) for s in range(S)]
        meg, feats, subj = (t.to(dev) for t in bench.make_host_batch(cfg, BATCH, 2036 + rank))
        batch = synthetic.SyntheticBatch(meg, subj, [recs[s] for s in subj.tolist()])
        mask = torch.ones(BATCH, 1, T, dtype=torch.bool, device=dev)
        clip = bb.ClipLoss().to(dev).train()
        steps = {}
        for mode in ("plain", "sync"):
            torch.manual_seed(2036)
            model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, n_subjects=S,
                                  **{k: (dict(v) if isinstance(v, dict) else v) for k, v in bench.CLIP_CONV.items()})
            if mode == "sync":
                model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
            model = model.to(dev).train()
            opt = torch.optim.Adam(model.parameters(), lr=3e-4, betas=(0.9, 0.999), fused=True)

            def step(model=model, opt=opt):
                opt.zero_grad(set_to_none=True)
                clip(model(dict(meg=meg), batch), feats, mask).backward()
                distrib.sync_gradients(model.parameters())
                opt.step()
            steps[mode] = step
        for fn in steps.values():
            for _ in range(args.warmup):
                fn()
        times = {m: [] for m in steps}
        for _ in range(args.rounds):
            for mode, fn in steps.items():
                dist.barrier()
                times[mode].append(round(timed_ms(fn, args.steps), 2))
        BF.check_tc_status()
        ret[rank] = times
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/syncbn_cost.py measures on CUDA devices"
    res = dict(card=card(), config="cfg3", batch_per_rank=BATCH, ranks=WORLD, steps_per_round=args.steps)
    if torch.cuda.device_count() < WORLD:
        res["step_ms"] = f"not measured: {torch.cuda.device_count()} GPU visible, NCCL needs one per rank"
    else:
        with tempfile.TemporaryDirectory() as tmp, mp.Manager() as mgr:
            ret = mgr.dict()
            mp.spawn(_rank, args=(args, f"file://{os.path.join(tmp, 'store')}", ret), nprocs=WORLD, join=True)
            res["step_ms"] = {f"rank{r}": ret[r] for r in range(WORLD)}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
