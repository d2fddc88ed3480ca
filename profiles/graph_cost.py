"""What does capturing the training step in a CUDA graph save?  For bench.py's cfg2 and cfg4 at B = 32, 64 and 256: the eager
step (reference batch, layout built and copied by the model) against the replayed step (StaticBatch.fill_ with the same
host layout, static inputs refilled, graph.replay()), timed in alternating rounds with CUDA events around `--steps` steps
each, the host enqueue time of one eager step (host clock, the queue empty before it), and the size of the captured graph's
private memory pool (reserved memory after the capture minus before it).  Prints one JSON line per (config, B) and the card
name and power limit read in the same run.
    python profiles/graph_cost.py [--steps 10] [--rounds 5] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import brainmagick_b200 as bb  # noqa: E402
from brainmagick_b200 import functional as BF, synthetic  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def make(cfg, B, dev, capturable=False):
    C, T, F, S = cfg["C"], cfg["T"], cfg["F"], cfg["S"]
    torch.manual_seed(2036)
    model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, n_subjects=S,
                          **{k: (dict(v) if isinstance(v, dict) else v) for k, v in bench.CLIP_CONV.items()}).to(dev).train()
    opt = torch.optim.Adam(model.parameters(), lr=3e-4, fused=True, capturable=capturable)    # bench.py's optimizer
    return model, bb.ClipLoss(uniform_batches=True).to(dev).train(), opt


def measure(tag, B, steps, rounds, dev):
    cfg = bench.CONFIGS[tag]
    C, T, S = cfg["C"], cfg["T"], cfg["S"]
    positions = synthetic.normalised_positions(S, C, n_valid=cfg["n_valid"], seed=7)
    recs = [synthetic.SyntheticRecording(s, positions[s]) for s in range(S)]
    host = []
    for seed in range(4):
        meg, feats, subj = bench.make_host_batch(cfg, B, seed)
        meg = meg.to(dev)
        host.append((meg, feats.to(dev), synthetic.SyntheticBatch(meg, subj, [recs[s] for s in subj.tolist()])))
    mask = torch.ones(B, 1, T, dtype=torch.bool, device=dev)

    e_model, e_clip, e_opt = make(cfg, B, dev)

    def eager(i):
        meg, feats, batch = host[i % len(host)]
        e_opt.zero_grad(set_to_none=True)
        e_clip(e_model(dict(meg=meg), batch), feats, mask).backward()
        e_opt.step()

    g_model, g_clip, g_opt = make(cfg, B, dev, capturable=True)
    sb = bb.StaticBatch(B, C, S, dev)
    s_meg, s_feats = torch.zeros_like(host[0][0]), torch.zeros_like(host[0][1])

    def load(i):
        meg, feats, batch = host[i % len(host)]
        sb.fill_(batch)
        s_meg.copy_(meg)
        s_feats.copy_(feats)

    def g_step():
        g_opt.zero_grad(set_to_none=True)
        g_clip(g_model(dict(meg=s_meg), sb), s_feats, mask).backward()
        g_opt.step()

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for i in range(3):
            load(i)
            g_step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()               # what torch.cuda.graph does on entry: cached blocks must not count as freed pool
    reserved = torch.cuda.memory_reserved(dev)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_step()
    torch.cuda.synchronize()
    pool = torch.cuda.memory_reserved(dev) - reserved      # the segments the capture added: the graph's private pool

    def replay(i):
        load(i)
        graph.replay()

    for i in range(3):
        eager(i)
        replay(i)
    torch.cuda.synchronize()

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for i in range(steps):
            fn(i)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    t_eager, t_graph, enqueue = [], [], []
    for _ in range(rounds):
        t_eager.append(timed(eager))
        t_graph.append(timed(replay))
        for i in range(steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eager(i)
            enqueue.append((time.perf_counter() - t0) * 1e3)
    torch.cuda.synchronize()
    BF.check_tc_status()
    out = dict(config=tag, B=B, eager_ms=round(statistics.median(t_eager), 3), replay_ms=round(statistics.median(t_graph), 3),
               eager_spread_ms=[round(min(t_eager), 3), round(max(t_eager), 3)],
               replay_spread_ms=[round(min(t_graph), 3), round(max(t_graph), 3)],
               eager_host_enqueue_ms=round(statistics.median(enqueue), 3),
               graph_pool_gb=round(pool / 2 ** 30, 2))
    del graph, e_model, g_model, e_opt, g_opt
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "graph_cost.py measures on the GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, limit = card()
    rows = [dict(card=name, power_limit=limit)]
    print(json.dumps(rows[0]), flush=True)
    for tag in ("cfg2", "cfg4"):
        for B in (32, 64, 256):
            rows.append(measure(tag, B, args.steps, args.rounds, dev))
            print(json.dumps(rows[-1]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
