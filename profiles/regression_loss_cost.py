"""What do the drop-in L1Loss / L2Loss cost, and what do they save?

  * kernels: bm_masked_loss_fwd (partials + finalize) and bm_masked_loss_bwd (d_estimate only, the output being a fixed
    target) timed with CUDA events over `--iters` launches, against torch's masked loss of bm/losses.py:11-26
    (estimate[mask], output[mask], then L1Loss / MSELoss; its forward includes the boolean index's host read), at the
    regression baseline's shapes (cfg4: 256 x 120 x 360, ragged [B, 1, T] mask) and the encoding task's (256 x 208 x 324, a
    view of T = 360 cropped by meg_init = 0.3 s at 120 Hz, all-True mask).  Bytes are computed from the shapes: each
    kernel reads the estimate, the output and the [B, 1, T] mask once, the backward also writes d_estimate; achieved
    bytes/s is given over the H100 SXM data sheet's 3.35 TB/s.
  * the encoding training step (SimpleConv meg 208 + features 120, complex_out, L1Loss on estimate[..., limit:], Adam) at
    B = 32, 64 and 256: eager with torch's masked loss, eager with the drop-in, and the drop-in step captured in a CUDA graph
    and replayed, in alternating rounds of `--steps` steps each timed with CUDA events; the median per-step time is reported.
Prints one JSON line; the card's name and power limit are part of it.  Needs cuda:0.
    python profiles/regression_loss_cost.py [--iters 200] [--steps 10] [--rounds 5] [--out FILE]"""
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
from brainmagick_b200 import _lib, functional as BF, synthetic  # noqa: E402
from profiles.graph_cost import card  # noqa: E402

HBM = 3.35e12
LIMIT = int(0.3 * 120)


def _events_ms(fn, n):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    start.record()
    for _ in range(n):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / n


def kernels(tag, kind, iters, dev):
    g = torch.Generator(device=dev).manual_seed(11)
    if tag == "cfg4_regression":
        B, C, T = 256, 120, 360
        est, out = (torch.randn(B, C, T, generator=g, device=dev) for _ in range(2))
        mask = torch.arange(T, device=dev) < (T - torch.randint(0, 90, (B, 1, 1), generator=g, device=dev))
    else:
        B, C, T = 256, 208, 360 - LIMIT
        est, out = (torch.randn(B, C, T + LIMIT, generator=g, device=dev)[..., LIMIT:] for _ in range(2))
        mask = torch.ones(B, 1, T + LIMIT, dtype=torch.bool, device=dev)[..., LIMIT:]
    m = mask.expand_as(est)
    st = _lib.c_void_p(torch.cuda.current_stream().cuda_stream)
    loss, inv_n, gout = (torch.ones(1, device=dev) for _ in range(3))
    ws = torch.empty(max(int(_lib.load().bm_masked_loss_workspace(B, C, T)), 2), device=dev)
    d_est = torch.empty(B, C, T, device=dev)
    ops = [BF._view_ptr(est), est.stride(0), est.stride(1), BF._view_ptr(out), out.stride(0), out.stride(1),
           BF._view_ptr(m), m.stride(0), m.stride(1), m.stride(2)]
    fwd_ms = _events_ms(lambda: _lib.call("bm_masked_loss_fwd", kind, *ops, B, C, T, _lib.ptr(ws), ws.numel(),
                                          _lib.ptr(loss), _lib.ptr(inv_n), st), iters)
    bwd_ms = _events_ms(lambda: _lib.call("bm_masked_loss_bwd", kind, _lib.ptr(gout), _lib.ptr(inv_n), *ops, B, C, T,
                                          _lib.ptr(d_est), None, st), iters)
    ref = torch.nn.L1Loss() if kind == BF.MASKED_L1 else torch.nn.MSELoss()
    e_req = est.detach().requires_grad_(True)
    torch_fwd_ms = _events_ms(lambda: ref(est[m], out[m]), iters)

    def torch_step():
        e_req.grad = None
        ref(e_req[m], out[m]).backward()
    torch_fwd_bwd_ms = _events_ms(torch_step, iters)
    elems = B * C * T
    read = 8 * elems + B * T                       # estimate, output, the [B, 1, T] mask
    return dict(shape=[B, C, T], fwd_ms=round(fwd_ms, 4), bwd_ms=round(bwd_ms, 4),
                fwd_tbps=round(read / fwd_ms / 1e9, 3), bwd_tbps=round((read + 4 * elems) / bwd_ms / 1e9, 3),
                fwd_share_of_hbm=round(read / fwd_ms * 1e3 / HBM, 3),
                bwd_share_of_hbm=round((read + 4 * elems) / bwd_ms * 1e3 / HBM, 3),
                torch_fwd_ms=round(torch_fwd_ms, 4), torch_fwd_bwd_ms=round(torch_fwd_bwd_ms, 4))


def encode_step(B, steps, rounds, dev):
    cfg = dict(bench.CONFIGS["cfg2"], F=120, S=4)
    C, T, F, S = cfg["C"], cfg["T"], cfg["F"], cfg["S"]
    positions = synthetic.normalised_positions(S, C, seed=7)
    recs = [synthetic.SyntheticRecording(s, positions[s]) for s in range(S)]
    host = []
    for seed in range(4):
        meg, feats, subj = bench.make_host_batch(cfg, B, seed)
        meg = meg.to(dev)
        host.append((meg, feats.to(dev), synthetic.SyntheticBatch(meg, subj, [recs[s] for s in subj.tolist()])))
    mask = torch.ones(B, 1, T, dtype=torch.bool, device=dev)
    in_mask = torch.zeros(T, device=dev)
    in_mask[:LIMIT] = 1
    torch_l1 = torch.nn.L1Loss()

    def torch_loss(e, o, m):
        m = m.expand_as(e)
        return torch_l1(e[m], o[m])

    def make(capturable=False):
        torch.manual_seed(2036)
        kw = {k: (dict(v) if isinstance(v, dict) else v) for k, v in bench.CLIP_CONV.items()}
        kw["hidden"] = dict(meg=320, features=320)
        model = bb.SimpleConv(in_channels=dict(meg=C, features=F), out_channels=C, n_subjects=S, **kw).to(dev).train()
        return model, torch.optim.Adam(model.parameters(), lr=3e-4, fused=True, capturable=capturable)

    def one(model, opt, loss_fn, meg, feats, batch):
        opt.zero_grad(set_to_none=True)
        est = model(dict(meg=in_mask * meg, features=feats), batch)
        loss_fn(est[..., LIMIT:], meg[..., LIMIT:], mask[..., LIMIT:]).backward()
        opt.step()

    variants = {}
    for name, loss_fn in (("eager_torch_loss", torch_loss), ("eager_drop_in", bb.L1Loss())):
        model, opt = make()
        variants[name] = (lambda i, model=model, opt=opt, loss_fn=loss_fn: one(model, opt, loss_fn, *host[i % len(host)]))
    g_model, g_opt = make(capturable=True)
    sb = bb.StaticBatch(B, C, S, dev)
    s_meg, s_feats = torch.zeros_like(host[0][0]), torch.zeros_like(host[0][1])
    l1 = bb.L1Loss()

    def load(i):
        meg, feats, batch = host[i % len(host)]
        sb.fill_(batch)
        s_meg.copy_(meg)
        s_feats.copy_(feats)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for i in range(3):
            load(i)
            one(g_model, g_opt, l1, s_meg, s_feats, sb)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        one(g_model, g_opt, l1, s_meg, s_feats, sb)

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
        raise SystemExit("profiles/regression_loss_cost.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    name, limit = card()
    row = dict(card=name, power_limit=limit, kernels={}, encode_step={})
    for tag in ("cfg4_regression", "encode_cropped"):
        for kind, kname in ((BF.MASKED_L1, "l1"), (BF.MASKED_L2, "l2")):
            row["kernels"][f"{tag}.{kname}"] = kernels(tag, kind, args.iters, dev)
    for B in (int(b) for b in args.batches.split(",")):
        row["encode_step"][f"B{B}"] = encode_step(B, args.steps, args.rounds, dev)
        torch.cuda.empty_cache()
    line = json.dumps(row)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
