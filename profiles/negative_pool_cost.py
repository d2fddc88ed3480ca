"""What does the solver's negative pool (`optim.negatives`, bm/solver.py:358-371; DESIGN §4.11) cost per training step?

cfg2 training steps (bench.py's workload: SimpleConv + ClipLoss + fused Adam at B = `--batch`) in three arms, alternating
in one process, for each `negatives` in `--negatives` with the default pool (2 * negatives):
  * none:  ClipLoss against the batch's own candidates;
  * pool:  the drop-in `NegativePool.complete` (device storage, pooled CLIP entry points);
  * host:  the reference's host pool block (oracle/negative_pool_oracle.py) at one CPU thread (bm/train.py:182), its
           concatenated candidates fed to the drop-in ClipLoss.
Before timing, with torch.use_deterministic_algorithms(True), each pool is filled and then, for 3 steps, the pool and host
arms score the same model estimate from the same CPU generator state: the losses and the estimate gradients must be
bitwise equal (B >= 192: both backwards run the same GEMM).  Prints one JSON line: median ms per step over the
rounds with the min and max, and the card's name and power limit.  Needs cuda:0.
    python profiles/negative_pool_cost.py [--negatives 512 1024] [--steps 3] [--rounds 3] [--batch 256] [--out FILE]"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import brainmagick_b200 as bb  # noqa: E402
from brainmagick_b200 import synthetic  # noqa: E402
from oracle.negative_pool_oracle import HostNegativePool  # noqa: E402
from profiles.graph_cost import card, make  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--negatives", type=int, nargs="+", default=[512, 1024])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/negative_pool_cost.py needs cuda:0"
    torch.set_num_threads(1)                         # bm/train.py:182
    dev = torch.device("cuda:0")
    cfg = bench.CONFIGS["cfg2"]
    B, C, T, S = args.batch, cfg["C"], cfg["T"], cfg["S"]
    model, clip, opt = make(cfg, B, dev)
    positions = synthetic.normalised_positions(S, C, n_valid=cfg["n_valid"], seed=7)
    recs = [synthetic.SyntheticRecording(s, positions[s]) for s in range(S)]
    host = []
    for seed in range(4):
        meg, feats, subj = bench.make_host_batch(cfg, B, seed)
        meg = meg.to(dev)
        host.append((meg, feats.to(dev), synthetic.SyntheticBatch(meg, subj, [recs[s] for s in subj.tolist()])))
    mask = torch.ones(B, 1, T, dtype=torch.bool, device=dev)

    def step(i, pool):
        meg, feats, batch = host[i % len(host)]
        opt.zero_grad(set_to_none=True)
        cand = feats if pool is None else pool.complete(feats, True)
        clip(model(dict(meg=meg), batch), cand, mask).backward()
        opt.step()

    def timed(pool):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for i in range(args.steps):
            step(i, pool)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    results = {}
    for neg in args.negatives:
        arms = {"none": None, "pool": bb.NegativePool(neg), "host": HostNegativePool(neg)}
        fill = 2 * neg // B + 1
        torch.use_deterministic_algorithms(True)
        for i in range(fill + 3):               # one estimate, the same draws: bitwise-equal losses and gradients
            meg, feats, batch = host[i % len(host)]
            est = model(dict(meg=meg), batch).detach().requires_grad_(True)
            rng = torch.get_rng_state()
            got = []
            for name in ("pool", "host"):
                torch.set_rng_state(rng)
                loss = clip(est, arms[name].complete(feats, True), mask)
                got.append((loss.detach(), torch.autograd.grad(loss, est)[0]))
            if i >= fill:
                assert torch.equal(got[0][0], got[1][0]), (neg, i, got[0][0].item(), got[1][0].item())
                assert torch.equal(got[0][1], got[1][1]), (neg, i)
        torch.use_deterministic_algorithms(False)
        for name, pool in arms.items():
            step(0, pool)
        samples = {name: [] for name in arms}
        for _ in range(args.rounds):
            for name, pool in arms.items():
                samples[name].append(timed(pool))
        results[str(neg)] = {name: dict(median=round(statistics.median(v), 3), min=round(min(v), 3),
                                        max=round(max(v), 3)) for name, v in samples.items()}
    name, limit = card()
    out = dict(card=name, power_limit=limit, batch=B, F=cfg["F"], T=T, ms_per_step=results, rounds=args.rounds,
               steps=args.steps, threads=1)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
