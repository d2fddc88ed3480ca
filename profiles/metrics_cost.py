"""What do the drop-in test metrics (bm/metrics.py; DESIGN §4.9) cost, and what do they save?

  * kernels: one update of each metric timed with CUDA events over `--iters` updates, fp64 operands as
    play.get_test_metrics passes them, ragged [B, 1, T] masks:
      encode  corr_meg at B = 256, C = 208, T = 324 (a crop of 360)
      decode  L2Reg and the correlation on a 120-channel mel slice and ClassificationAcc over 41 classes, B = 256,
              T = 342
    Bytes are the left and right slices and the mask read once, plus the accumulators read and written; achieved bytes/s
    is given over the H100 SXM data sheet's 3.35 TB/s.  Each is set against a torch restatement of the reference update
    (bm/metrics.py: the `_count.sum() == 0` host read, then the masked products and sums on the fp64 tensors).
  * the test-stage loop: an encoding SimpleConv (meg 208 + features 120, complex_out) in eval mode under no_grad, over
    `--batches` batches of B = 64, each forward followed by the crop, the fp64 casts and corr_meg's update, then get();
    the drop-in against the restatement in alternating rounds, median ms per loop.
Prints one JSON line; the card's name and power limit are part of it.  Needs cuda:0.
    python profiles/metrics_cost.py [--iters 200] [--batches 20] [--rounds 5] [--out FILE]"""
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
from brainmagick_b200 import functional as BF, metrics as BM, synthetic  # noqa: E402
from profiles.graph_cost import card  # noqa: E402
from profiles.regression_loss_cost import LIMIT, _events_ms  # noqa: E402

HBM = 3.35e12


class TorchCorrelation:
    """torch restatement of the reference OnlineCorrelation's update (dim 0, real operands) and get()"""

    def __init__(self, ls, rs):
        self.ls, self.rs = ls, rs
        self.count = torch.zeros(1)

    def update(self, left, right, mask):
        left, right = left[:, self.ls], right[:, self.rs]
        if self.count.sum() == 0:                         # a host read per update
            self.dot, self.sl, self.sr, self.sll, self.srr, self.count = (torch.zeros_like(left[0]) for _ in range(6))
        self.dot += (left * right * mask).sum(0)
        self.sl += (left * mask).sum(0)
        self.sr += (right * mask).sum(0)
        self.sll += (left * mask).abs().pow(2).sum(0)
        self.srr += (right * mask).abs().pow(2).sum(0)
        self.count += mask.sum(0)
        return self

    def get(self):
        nl = (self.sll - self.sl ** 2 / self.count).clamp(0, float("inf")).sqrt()
        nr = (self.srr - self.sr ** 2 / self.count).clamp(0, float("inf")).sqrt()
        corr = (self.dot - self.sl * self.sr / self.count) / (nl * nr).clamp(1e-8, float("inf"))
        assert not torch.isnan(corr).any()
        return corr


class TorchAccumulative:
    """torch restatement of the reference AccumulativeMetric's update for L2Reg and ClassificationAcc"""

    def __init__(self, ls, rs, kind):
        self.ls, self.rs, self.kind = ls, rs, kind
        self.count = torch.zeros(1)

    def update(self, left, right, mask):
        left, right = left[:, self.ls], right[:, self.rs]
        if self.count.sum() == 0:
            self.acc, self.count = torch.zeros_like(right[0]), torch.zeros_like(right[0])
        if self.kind == "l2":
            self.acc += (((left - right) * mask) ** 2).sum(0)
        else:
            preds = left.argmax(1, keepdim=True)
            expected = right.clone()
            preds[~mask], expected[~mask] = -1, -2
            self.acc += (preds == expected).sum(0)
        self.count += mask.sum(0)
        return self


def _ragged(B, T, dev, g):
    mask = torch.arange(T, device=dev)[None, None] < torch.randint(T // 2, T + 1, (B, 1, 1), device=dev, generator=g)
    mask[0] = True
    return mask


def kernels(iters, dev):
    g = torch.Generator(device=dev).manual_seed(11)
    out = {}
    B, C, T = 256, 208, 360
    meg = torch.randn(B, C, T, device=dev, dtype=torch.float64, generator=g)
    est = 0.5 * meg + torch.randn(B, C, T, device=dev, dtype=torch.float64, generator=g)
    e, m, mask = est[..., T - 324:], meg[..., T - 324:], _ragged(B, 324, dev, g)
    cases = [("encode.corr", BM.OnlineCorrelation(slice(None), slice(None)), TorchCorrelation(slice(None), slice(None)),
              (e, m, mask), 2 * B * C * 324 * 8 + B * 324 + 2 * 6 * C * 324 * 8)]
    est = torch.randn(B, 161, 342, device=dev, dtype=torch.float64, generator=g)
    gt = torch.randn(B, 121, 342, device=dev, dtype=torch.float64, generator=g)
    gt[:, 120] = torch.randint(0, 41, (B, 342), device=dev, generator=g).double()
    dmask = _ragged(B, 342, dev, g)
    mel, cls = slice(0, 120), slice(120, 161)
    reg_bytes = 2 * B * 120 * 342 * 8 + B * 342
    cases += [("decode.l2", BM.L2Reg(mel, mel), TorchAccumulative(mel, mel, "l2"), (est, gt, dmask),
               reg_bytes + 2 * 2 * 120 * 342 * 8),
              ("decode.corr", BM.OnlineCorrelation(mel, mel), TorchCorrelation(mel, mel), (est, gt, dmask),
               reg_bytes + 2 * 6 * 120 * 342 * 8),
              ("decode.acc", BM.ClassificationAcc(cls, slice(120, 121)), TorchAccumulative(cls, slice(120, 121), "acc"),
               (est, gt, dmask), B * 41 * 342 * 8 + B * 342 * 8 + B * 342 + 2 * 2 * 342 * 8)]
    for tag, drop, ref, args, nbytes in cases:
        ms = _events_ms(lambda: drop.update(*args), iters)
        ref_ms = _events_ms(lambda: ref.update(*args), max(iters // 10, 5))
        out[tag] = dict(ms=round(ms, 4), tb_s=round(nbytes / ms / 1e9, 3), of_peak=round(nbytes / ms / 1e9 / 3.35, 3),
                        bound_ms=round(nbytes / HBM * 1e3, 4), mb=round(nbytes / 1e6, 1), torch_ms=round(ref_ms, 3))
        drop.get()
    return out


def test_stage(batches, rounds, dev):
    cfg = dict(bench.CONFIGS["cfg2"], F=120, S=4)
    C, T, F, S = cfg["C"], cfg["T"], cfg["F"], cfg["S"]
    B = 64
    positions = synthetic.normalised_positions(S, C, seed=7)
    recs = [synthetic.SyntheticRecording(s, positions[s]) for s in range(S)]
    host = []
    for seed in range(4):
        meg, feats, subj = bench.make_host_batch(cfg, B, seed)
        meg = meg.to(dev)
        host.append((meg, feats.to(dev), synthetic.SyntheticBatch(meg, subj, [recs[s] for s in subj.tolist()])))
    g = torch.Generator(device=dev).manual_seed(5)
    masks = [_ragged(B, T, dev, g) for _ in range(4)]
    in_mask = torch.zeros(T, device=dev)
    in_mask[:LIMIT] = 1
    torch.manual_seed(2036)
    kw = {k: (dict(v) if isinstance(v, dict) else v) for k, v in bench.CLIP_CONV.items()}
    kw["hidden"] = dict(meg=320, features=320)
    model = bb.SimpleConv(in_channels=dict(meg=C, features=F), out_channels=C, n_subjects=S, **kw).to(dev).eval()

    def loop(make_metric):
        metric = make_metric()
        with torch.no_grad():
            for i in range(batches):
                meg, feats, batch = host[i % len(host)]
                est = model(dict(meg=in_mask * meg, features=feats), batch)
                metric.update(est[..., LIMIT:].double(), meg[..., LIMIT:].double(), masks[i % 4][..., LIMIT:])
        return metric.get()

    variants = dict(torch_metric=lambda: TorchCorrelation(slice(None), slice(None)),
                    drop_in=lambda: BM.OnlineCorrelation(slice(None), slice(None), "corr_meg"))
    results = {name: loop(fn) for name, fn in variants.items()}      # warm-up, and the two agree
    diff = (results["drop_in"] - results["torch_metric"]).abs().max().item()
    times = {name: [] for name in variants}
    for _ in range(rounds):
        for name, fn in variants.items():
            times[name].append(_events_ms(lambda fn=fn: loop(fn), 1))
    BF.check_tc_status()
    out = {name: dict(median_ms=round(statistics.median(t), 2), min_ms=round(min(t), 2), max_ms=round(max(t), 2))
           for name, t in times.items()}
    out["max_abs_diff"] = diff
    out["batches"], out["B"] = batches, B
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profiles/metrics_cost.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    name, limit = card()
    row = dict(card=name, power_limit=limit, kernels=kernels(args.iters, dev))
    torch.cuda.empty_cache()
    row["test_stage"] = test_stage(args.batches, args.rounds, dev)
    line = json.dumps(row)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
