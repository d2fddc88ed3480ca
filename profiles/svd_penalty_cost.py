"""What does the drop-in spectral penalty (bm/svd.py: svd_penalty; DESIGN §4.10) cost, and what does it save?

  * the penalty alone on the 18 weights of a BASELINE-width clip_conv SimpleConv (dim 16, niters 2): the value, and the
    value plus its backward, timed with CUDA events over `--iters` calls; against a torch restatement of the reference
    (torch.svd_lowrank per weight, summed, backward through autograd) on the same weights.  Both draw their own R from
    the CUDA generator, as the reference does.
  * a cfg2 training step (bench.py's workload: SimpleConv + ClipLoss + fused Adam at B = `--batch`) without the penalty,
    with the drop-in (`loss += 0.1 * svd_penalty(model)`) and with the restatement, in alternating rounds, median ms/step.
Prints one JSON line; the card's name and power limit are part of it.  Needs cuda:0.
    python profiles/svd_penalty_cost.py [--iters 50] [--steps 20] [--rounds 5] [--batch 256] [--out FILE]"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from brainmagick_b200 import svd as S, synthetic  # noqa: E402
from profiles.graph_cost import card, make  # noqa: E402
from profiles.regression_loss_cost import _events_ms  # noqa: E402


def torch_penalty(model, min_size=1., dim=16, niters=2):
    """the reference's svd_penalty with proba 1 (its body, on torch.svd_lowrank)"""
    total = 0
    for _, m in model.named_modules():
        if not isinstance(m, (torch.nn.modules.conv._ConvNd, torch.nn.Linear)):
            continue
        p = m.weight
        if p.numel() / 2**8 < min_size:
            continue
        total += torch.svd_lowrank(p.view(p.shape[0], -1), dim, niters)[1][0].pow(2)
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/svd_penalty_cost.py needs cuda:0"
    dev = torch.device("cuda:0")
    cfg = bench.CONFIGS["cfg2"]
    B, C, T, F, Sb = args.batch, cfg["C"], cfg["T"], cfg["F"], cfg["S"]
    model, clip, opt = make(cfg, B, dev)
    S.penalty_rng.seed(1234)

    def drop_fwd():
        S.svd_penalty(model)

    def drop_both():
        S.svd_penalty(model).backward()

    def torch_fwd():
        with torch.no_grad():
            torch_penalty(model)

    def torch_both():
        torch_penalty(model).backward()

    penalty = {}
    for name, fn in (("drop_in_value", drop_fwd), ("drop_in_value_and_grad", drop_both), ("torch_value", torch_fwd),
                     ("torch_value_and_grad", torch_both)):
        _events_ms(fn, 3)
        penalty[name] = round(_events_ms(fn, args.iters), 4)
    model.zero_grad(set_to_none=True)

    positions = synthetic.normalised_positions(Sb, C, n_valid=cfg["n_valid"], seed=7)
    recs = [synthetic.SyntheticRecording(s, positions[s]) for s in range(Sb)]
    host = []
    for seed in range(4):
        meg, feats, subj = bench.make_host_batch(cfg, B, seed)
        meg = meg.to(dev)
        host.append((meg, feats.to(dev), synthetic.SyntheticBatch(meg, subj, [recs[s] for s in subj.tolist()])))
    mask = torch.ones(B, 1, T, dtype=torch.bool, device=dev)
    terms = {"no_penalty": lambda: 0., "drop_in": lambda: S.svd_penalty(model), "torch": lambda: torch_penalty(model)}

    def step(i, term):
        meg, feats, batch = host[i % len(host)]
        opt.zero_grad(set_to_none=True)
        loss = clip(model(dict(meg=meg), batch), feats, mask)
        loss = loss + 0.1 * terms[term]()
        loss.backward()
        opt.step()

    def timed(term):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for i in range(args.steps):
            step(i, term)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for term in terms:
        for i in range(3):
            step(i, term)
    samples = {term: [] for term in terms}
    for _ in range(args.rounds):
        for term in terms:
            samples[term].append(timed(term))
    steps = {term: round(statistics.median(v), 3) for term, v in samples.items()}
    name, limit = card()
    out = dict(card=name, power_limit=limit, weights=18, dim=16, niters=2, penalty_ms=penalty,
               cfg2_step_ms=dict(batch=B, **steps), rounds=args.rounds, steps=args.steps)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
