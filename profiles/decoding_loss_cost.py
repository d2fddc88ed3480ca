"""What does the drop-in FeatureDecodingLoss cost, and what does it save?

  * kernels: bm_decoding_loss_fwd (partials + finalize) and bm_decoding_loss_bwd (d_estimate only, the targets being
    fixed) timed with CUDA events over `--iters` launches at B = 256, T = 342, for the decoding feature set [120 mel
    (regression), 41 classes, 2 classes] and for one feature of 1025 classes, both weighted, with a ragged [B, 1, T] mask;
    against a torch restatement of the reference loss (bm/losses.py:117-173: mask.any(), the per-feature max() asserts,
    the weights copied to the device, boolean-mask indexing, F.mse_loss / F.cross_entropy; its forward includes those host
    reads).  Bytes are computed from the shapes: the forward reads the estimate, the regression outputs, the target rows
    and the mask once and writes the log-sum-exp; the backward reads the same, the log-sum-exp, and writes d_estimate.
    Achieved bytes/s is given over the H100 SXM data sheet's 3.35 TB/s.
  * the decoding training step (clip_conv SimpleConv, C = 208, T = 342, 163 outputs, Adam) at B = 32, 64 and 256: eager
    with the torch loss, eager with the drop-in, and the drop-in step captured in a CUDA graph and replayed, in alternating
    rounds of `--steps` steps each timed with CUDA events; the median per-step time is reported.
Prints one JSON line; the card's name and power limit are part of it.  Needs cuda:0.
    python profiles/decoding_loss_cost.py [--iters 200] [--steps 10] [--rounds 5] [--out FILE]"""
import argparse
import json
import os
import statistics
import sys
from collections import OrderedDict

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import brainmagick_b200 as bb  # noqa: E402
from brainmagick_b200 import _lib, functional as BF, synthetic  # noqa: E402
from profiles.graph_cost import card  # noqa: E402
from profiles.regression_loss_cost import _events_ms  # noqa: E402

HBM = 3.35e12
T_DEC = 342


class _Feature:
    def __init__(self, name, dimension, cardinality=None):
        self.name, self.dimension, self.cardinality = name, dimension, cardinality
        self.categorical = cardinality is not None
        self.output_dimension = dimension if cardinality is None else cardinality


class _Builder(OrderedDict):
    def get_slice(self, name, model_output=False):
        start = 0
        for key, f in self.items():
            width = f.output_dimension if model_output else f.dimension
            if key == name:
                return slice(start, start + width)
            start += width

    @property
    def dimension(self):
        return sum(f.dimension for f in self.values())

    @property
    def output_dimension(self):
        return sum(f.output_dimension for f in self.values())


class _Scaler:
    """norm.py:289-308 weights over fixed counts (one empty class per feature)"""

    def __init__(self, builder):
        g = torch.Generator().manual_seed(3)
        self.weights = {}
        for name, f in builder.items():
            if f.categorical:
                counts = torch.randint(1, 100, (f.cardinality,), generator=g).float()
                counts[-1] = 0
                p = counts / counts.sum()
                w = 1 / torch.sqrt(p)
                w[p == 0] = 0
                self.weights[name] = w / torch.sqrt(p).sum()

    def get_categorical_feature_weights(self, name):
        return self.weights[name]


def _features(tag):
    spec = [("mel", 120, None), ("hash", 1, 41), ("seg", 1, 2)] if tag == "decoding" else [("cls", 1, 1025)]
    builder = _Builder((n, _Feature(n, d, c)) for n, d, c in spec)
    return builder, _Scaler(builder)


class TorchDecodingLoss(torch.nn.Module):
    """bm/losses.py:127-173 restated with torch ops"""

    def __init__(self, used_features, scaler):
        super().__init__()
        self.used_features, self.scaler = used_features, scaler

    def forward(self, estimate, output, mask):
        assert mask.any()
        loss = 0
        for feature in self.used_features.values():
            sl, sl_out = self.used_features.get_slice(feature.name), self.used_features.get_slice(feature.name, True)
            fe, fo = estimate[:, sl_out], output[:, sl]
            fm = mask.expand_as(fe)
            if feature.categorical:
                assert feature.output_dimension > output[:, sl.start].max()
                w = self.scaler.get_categorical_feature_weights(feature.name).to(output)
                loss += F.cross_entropy(fe.transpose(1, 2)[fm.transpose(1, 2)].reshape(-1, sl_out.stop - sl_out.start),
                                        fo.transpose(1, 2).long()[mask.transpose(1, 2)], w)
            else:
                loss += F.mse_loss(fe[fm], fo[fm])
        return loss


def _data(builder, B, T, dev, seed=11):
    g = torch.Generator(device=dev).manual_seed(seed)
    est = torch.randn(B, builder.output_dimension, T, generator=g, device=dev)
    out = torch.randn(B, builder.dimension, T, generator=g, device=dev)
    for name, f in builder.items():
        if f.categorical:
            out[:, builder.get_slice(name).start] = torch.randint(0, f.cardinality, (B, T), generator=g, device=dev).float()
    mask = torch.arange(T, device=dev) < (T - torch.randint(0, 90, (B, 1, 1), generator=g, device=dev))
    return est, out, mask


def kernels(tag, iters, dev):
    builder, scaler = _features(tag)
    B, T = 256, T_DEC
    est, out, mask = _data(builder, B, T, dev)
    loss_fn = bb.FeatureDecodingLoss(builder, scaler)
    table, weights = loss_fn._table(dev), loss_fn._class_weights(dev)
    Fn, Ce, Co = table.shape[0], est.shape[1], out.shape[1]
    n_cat = sum(f.categorical for f in builder.values())
    st = _lib.c_void_p(torch.cuda.current_stream().cuda_stream)
    loss, scale, gout = torch.ones(1, device=dev), torch.ones(Fn, device=dev), torch.ones(1, device=dev)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    lse = torch.empty(n_cat * B * T, device=dev)
    ws = torch.empty(max(int(_lib.load().bm_decoding_loss_workspace(B, T, Fn)), 2), device=dev)
    d_est = torch.empty(B, Ce, T, device=dev)
    ops = [BF._view_ptr(est), est.stride(0), est.stride(1), BF._view_ptr(out), out.stride(0), out.stride(1),
           BF._view_ptr(mask), *BF._mask_strides(mask), B, T]
    fwd_ms = _events_ms(lambda: _lib.call("bm_decoding_loss_fwd", *ops, _lib.ptr(table), Fn, _lib.ptr(weights),
                                          _lib.ptr(lse), _lib.ptr(ws), ws.numel(), _lib.ptr(loss), _lib.ptr(scale),
                                          _lib.ptr(flag), None, st), iters)
    bwd_ms = _events_ms(lambda: _lib.call("bm_decoding_loss_bwd", _lib.ptr(gout), _lib.ptr(scale), _lib.ptr(lse), *ops,
                                          Ce, Co, _lib.ptr(table), Fn, _lib.ptr(weights), _lib.ptr(d_est), None, st), iters)
    ref = TorchDecodingLoss(builder, scaler)
    e_req = est.detach().requires_grad_(True)
    torch_fwd_ms = _events_ms(lambda: ref(est, out, mask), iters)

    def torch_step():
        e_req.grad = None
        ref(e_req, out, mask).backward()
    torch_fwd_bwd_ms = _events_ms(torch_step, iters)
    n_reg = sum(f.dimension for f in builder.values() if not f.categorical)
    read = 4 * B * T * (Ce + n_reg + n_cat) + B * T           # estimate, regression outputs, target rows, mask
    fwd_bytes, bwd_bytes = read + 4 * n_cat * B * T, read + 4 * n_cat * B * T + 4 * B * Ce * T
    return dict(shape=dict(B=B, T=T, est_C=Ce, out_C=Co), fwd_ms=round(fwd_ms, 4), bwd_ms=round(bwd_ms, 4),
                fwd_tbps=round(fwd_bytes / fwd_ms / 1e9, 3), bwd_tbps=round(bwd_bytes / bwd_ms / 1e9, 3),
                fwd_share_of_hbm=round(fwd_bytes / fwd_ms * 1e3 / HBM, 3),
                bwd_share_of_hbm=round(bwd_bytes / bwd_ms * 1e3 / HBM, 3),
                torch_fwd_ms=round(torch_fwd_ms, 4), torch_fwd_bwd_ms=round(torch_fwd_bwd_ms, 4))


def decoding_step(B, steps, rounds, dev):
    cfg = dict(bench.CONFIGS["cfg2"], T=T_DEC, S=4)
    C, T, S = cfg["C"], cfg["T"], cfg["S"]
    builder, scaler = _features("decoding")
    positions = synthetic.normalised_positions(S, C, seed=7)
    recs = [synthetic.SyntheticRecording(s, positions[s]) for s in range(S)]
    host = []
    for seed in range(4):
        meg, _, subj = bench.make_host_batch(dict(cfg, F=1), B, seed)
        meg = meg.to(dev)
        _, out, mask = _data(builder, B, T, dev, seed=seed)
        host.append((meg, out, mask, synthetic.SyntheticBatch(meg, subj, [recs[s] for s in subj.tolist()])))

    def make(capturable=False):
        torch.manual_seed(2036)
        kw = {k: (dict(v) if isinstance(v, dict) else v) for k, v in bench.CLIP_CONV.items()}
        model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=builder.output_dimension, n_subjects=S,
                              **kw).to(dev).train()
        return model, torch.optim.Adam(model.parameters(), lr=3e-4, fused=True, capturable=capturable)

    def one(model, opt, loss_fn, meg, out, mask, batch):
        opt.zero_grad(set_to_none=True)
        est = model(dict(meg=meg), batch)
        loss_fn(est, out, mask).backward()
        opt.step()

    variants = {}
    for name, loss_fn in (("eager_torch_loss", TorchDecodingLoss(builder, scaler)),
                          ("eager_drop_in", bb.FeatureDecodingLoss(builder, scaler))):
        model, opt = make()
        variants[name] = (lambda i, model=model, opt=opt, loss_fn=loss_fn: one(model, opt, loss_fn, *host[i % len(host)]))
    g_model, g_opt = make(capturable=True)
    sb = bb.StaticBatch(B, C, S, dev)
    s_meg, s_out, s_mask = torch.zeros_like(host[0][0]), torch.zeros_like(host[0][1]), torch.zeros_like(host[0][2])
    dec = bb.FeatureDecodingLoss(builder, scaler)

    def load(i):
        meg, out, mask, batch = host[i % len(host)]
        sb.fill_(batch)
        s_meg.copy_(meg)
        s_out.copy_(out)
        s_mask.copy_(mask)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for i in range(3):
            load(i)
            one(g_model, g_opt, dec, s_meg, s_out, s_mask, sb)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        one(g_model, g_opt, dec, s_meg, s_out, s_mask, sb)

    def replay(i):
        load(i)
        graph.replay()
    variants["captured_drop_in"] = replay
    for fn in variants.values():                   # warm-up
        for i in range(3):
            fn(i)
    times = {name: [] for name in variants}
    for _ in range(rounds):
        for name, fn in variants.items():
            times[name].append(_events_ms(lambda fn=fn: [fn(i) for i in range(steps)], 1) / steps)
    BF.check_tc_status()
    return {name: dict(median_ms=round(statistics.median(t), 3), min_ms=round(min(t), 3), max_ms=round(max(t), 3))
            for name, t in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batches", default="32,64,256")
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profiles/decoding_loss_cost.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    name, limit = card()
    row = dict(card=name, power_limit=limit, kernels={}, decoding_step={})
    for tag in ("decoding", "k1025"):
        row["kernels"][tag] = kernels(tag, args.iters, dev)
    for B in (int(b) for b in args.batches.split(",")):
        row["decoding_step"][f"B{B}"] = decoding_step(B, args.steps, args.rounds, dev)
        torch.cuda.empty_cache()
    line = json.dumps(row)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
