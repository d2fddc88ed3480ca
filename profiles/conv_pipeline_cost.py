"""The tensor-core conv launches of the cfg2 training step (B = 256, T = 360; hc_conv_kernel) and the three conv weight
gradients (hw_wgrad_kernel), timed as bench._time_kernel does (CUDA events around back-to-back launches over rotating
operand sets larger than L2) in `--rounds` rounds, both pass counts.  The conv shapes are those of
profiles/conv_phase_probe.py.  `--lib PATH` loads that build of libbm_b200.so instead of the in-tree one, so that one GPU
command can alternate two builds in separate processes.

`--dump DIR` also writes what two builds must agree on, as DIR/digests.json (sha256 of each output's bytes) and
DIR/stats.npz (the fused BatchNorm statistics, which fp64 atomics sum in a run-dependent order):
  * the conv outputs (y, aux, glu_out, channel-major y) of seeded operands at every conv shape of the step, both pass counts,
    every epilogue mode, the three weight formats (raw fp32, tf32 pieces, fp16 pieces), per-sample weight sets
    (bm_tc_pointwise_sel, bm_tc_sensor_mix_bwd_data) and NaN-filled output buffers;
  * dW of the three weight gradients, both pass counts;
  * under torch.use_deterministic_algorithms(True), 3 cfg2 training steps (bench.py's model and optimizer): each step's loss,
    the last estimate and gradients, and the parameters and BatchNorm running statistics after the 3 steps.
`--compare DIR_A DIR_B` reports every digest that differs and the largest relative difference of the statistics.

    python profiles/conv_pipeline_cost.py [--lib PATH] [--rounds 3] [--dump DIR] [--no-kernels] [--out result.json]
    python profiles/conv_pipeline_cost.py --compare DIR_A DIR_B

Prints one JSON line; the card's name and power limit are part of it.  Needs cuda:0 (not --compare).
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from brainmagick_b200 import _lib  # noqa: E402
from profiles.conv_phase_probe import B, CONVS, NSETS, T  # noqa: E402

NROT = 3


def _conv_launches(name, suffix, dev, nrot, seed=5, fmt="raw", nan=False):
    """nrot launches of conv `name` over separate seeded operand sets, and the outputs of the first"""
    from brainmagick_b200._lib import call, ptr, stream
    entry, Cin, N, Kw, dil, sign, mode = CONVS[name]
    g = torch.Generator(device=dev).manual_seed(seed)
    status = torch.zeros(1, dtype=torch.int32, device=dev)

    def out(*shape, dtype=torch.float32):
        return torch.full(shape, float("nan"), device=dev, dtype=dtype) if nan else torch.zeros(*shape, device=dev,
                                                                                                 dtype=dtype)
    fns, outs = [], None
    if entry == "sel":
        w = torch.randn(NSETS, N, Cin, device=dev, generator=g) * 0.05
        hi, lo = torch.empty_like(w), torch.empty_like(w)
        call("bm_tc_weight_split", ptr(w), NSETS * N, Cin, 1, ptr(hi), ptr(lo), None, None, stream())
        wsel = (torch.arange(B, device=dev, dtype=torch.int32) * 7) % NSETS
        for _ in range(nrot):
            x, y = torch.randn(B, T, Cin, device=dev, generator=g), out(B, T, N)
            fns.append(lambda x=x, y=y: call("bm_tc_pointwise_sel" + suffix, ptr(x), ptr(hi), ptr(lo), ptr(wsel), NSETS,
                                             B, T, Cin, N, ptr(y), ptr(status), stream()))
            outs = outs or dict(y=y)
        return fns, outs, status
    w = torch.randn(Kw, N, Cin, device=dev, generator=g) * 0.05
    bias = torch.randn(N, device=dev, generator=g)
    hi, lo = torch.empty_like(w), torch.empty_like(w)
    w_nc = w.permute(1, 2, 0).contiguous()                                          # nn.Conv1d layout [N][Cin][Kw]
    if fmt == "split":
        call("bm_tc_weight_split", ptr(w_nc), N, Cin, Kw, ptr(hi), ptr(lo), None, None, stream())
    elif fmt == "f16":
        amax, xa = torch.empty(1, device=dev), torch.empty(1, device=dev)
        h16, l16 = torch.empty(w.shape, device=dev, dtype=torch.float16), torch.empty(w.shape, device=dev,
                                                                                      dtype=torch.float16)
        call("bm_amax", ptr(w), w.numel(), ptr(amax), stream())
        call("bm_f16_split", ptr(w), w.numel(), ptr(amax), ptr(h16), ptr(l16), stream())
    glu, act, tmaj, acc = int(mode == "glu"), int(mode == "gelu"), int(mode == "tmajor"), int(mode == "accumulate")
    for _ in range(nrot):
        x = torch.randn(B, T, Cin, device=dev, generator=g)
        y = torch.randn(B, T, N, device=dev, generator=g) if acc else out(*((B, N, T) if tmaj else (B, T, N)))
        aux = out(B, T, N) if act else None
        glu_out = out(B, T, N // 2) if glu else None
        stats = out(2 * N, dtype=torch.float64) if mode == "stats" else None
        b = None if acc else bias
        if fmt == "raw":
            fn = (lambda x=x, y=y, aux=aux, glu_out=glu_out, stats=stats, b=b:
                  call("bm_tc_conv1d_persistent" + suffix, ptr(x), ptr(w), ptr(b), acc, B, T, Cin, N, Kw, dil, sign, glu,
                       act, tmaj, ptr(y), ptr(aux), ptr(glu_out), ptr(stats), ptr(status), stream()))
        elif fmt == "split":
            fn = (lambda x=x, y=y, aux=aux, glu_out=glu_out, b=b:
                  call("bm_tc_conv1d" + suffix, ptr(x), ptr(hi), ptr(lo), ptr(b), ptr(y) if acc else None, B, T, Cin, N, Kw,
                       dil, sign, glu, act, tmaj, ptr(y), ptr(aux), ptr(glu_out), None, ptr(status), stream()))
        else:
            fn = (lambda x=x, y=y, aux=aux, glu_out=glu_out, stats=stats, b=b: (
                call("bm_amax", ptr(x), x.numel(), ptr(xa), stream()),
                call("bm_tc_conv1d_f16", ptr(x), ptr(xa), ptr(h16), ptr(l16), ptr(amax), ptr(b), acc, B, T, Cin, N, Kw,
                     dil, sign, glu, act, tmaj, ptr(y), ptr(aux), ptr(glu_out), ptr(stats), None, ptr(status), stream())))
        fns.append(fn)
        if outs is None:
            outs = {k: v for k, v in dict(y=y, aux=aux, glu_out=glu_out, stats=stats).items() if v is not None}
    return fns, outs, status


def kernels(args, dev):
    import bench
    from profiles import wgrad_pipeline_cost
    res = {}
    for name in CONVS:
        times = {"3xtf32": [], "tf32": []}
        for _ in range(args.rounds):
            for form, suffix in (("3xtf32", ""), ("tf32", "_tf32")):
                fns, _, status = _conv_launches(name, suffix, dev, NROT)
                times[form].append(round(bench._time_kernel(fns, iters=args.iters), 4))
                torch.cuda.synchronize()
                assert int(status.item()) == 0, f"{name}{suffix}: status {int(status.item())}"
                del fns
        res[name] = dict(ms=times)
        torch.cuda.empty_cache()
    wa = argparse.Namespace(batch=B, rounds=args.rounds, iters=args.iters, dump="")
    for name, r in wgrad_pipeline_cost.kernels(wa, dev).items():
        res["wg_" + name] = r
    return res


def _digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def dump(args, dev):
    from brainmagick_b200._lib import call, ptr, stream
    digests, stats = {}, {}
    # every conv shape of the step, both pass counts (the fp16 pieces: 3xTF32 only), NaN-filled outputs
    cases = [(n, "raw") for n in CONVS if CONVS[n][0] == "persistent"] + [("subj", "raw")]
    cases += [("k3_fwd", "split"), ("k3_bwd", "split"), ("head0", "split"), ("k4_glu", "f16"), ("k3_fwd", "f16")]
    for name, fmt in cases:
        for suffix in ("", "_tf32"):
            if fmt == "f16" and suffix:
                continue
            if fmt == "split" and CONVS[name][6] == "stats":
                continue                                  # the pre-split entry point has no fused statistics
            fns, outs, status = _conv_launches(name, suffix, dev, 1, seed=11, fmt=fmt, nan=True)
            fns[0]()
            torch.cuda.synchronize()
            assert int(status.item()) == 0, f"{name}{suffix}: status {int(status.item())}"
            for k, v in outs.items():
                key = f"{name}_{fmt}{suffix}_{k}"
                if k == "stats":
                    stats[key] = v.cpu().numpy()
                else:
                    digests[key] = _digest(v)
            del fns, outs
    # the sensor-mix data gradient: per-recording weight sets, a partial last column tile
    g = torch.Generator(device=dev).manual_seed(13)
    Op, Cp, C, R = 320, 288, 273, 5
    w = torch.randn(R, Cp, Op, device=dev, generator=g) * 0.05
    hi, lo = torch.empty_like(w), torch.empty_like(w)
    call("bm_tc_weight_split", ptr(w), R * Cp, Op, 1, ptr(hi), ptr(lo), None, None, stream())
    du = torch.randn(B, T, Op, device=dev, generator=g)
    wsel = (torch.arange(B, device=dev, dtype=torch.int32) * 3) % R
    mask = (torch.rand(C, device=dev, generator=g) > 0.2).float()
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    for suffix in ("", "_tf32"):
        dmeg = torch.full((B, C, T), float("nan"), device=dev)
        call("bm_tc_sensor_mix_bwd_data" + suffix, ptr(du), ptr(hi), ptr(lo), ptr(wsel), R, ptr(mask), B, T, Op, Cp, C,
             ptr(dmeg), ptr(status), stream())
        torch.cuda.synchronize()
        assert int(status.item()) == 0
        digests["sensor_mix_bwd" + suffix] = _digest(dmeg)
    # the weight gradients
    from profiles import wgrad_pipeline_cost
    wdir = os.path.join(args.dump, "wgrad")
    wgrad_pipeline_cost.kernels(argparse.Namespace(batch=B, rounds=0, iters=1, dump=wdir), dev)
    for f in sorted(os.listdir(wdir)):
        digests["wgrad_" + f] = hashlib.sha256(np.load(os.path.join(wdir, f)).tobytes()).hexdigest()
    digests.update(det_steps(dev))
    with open(os.path.join(args.dump, "digests.json"), "w") as f:
        json.dump(digests, f, indent=0, sort_keys=True)
    np.savez(os.path.join(args.dump, "stats.npz"), **stats)
    return len(digests)


def det_steps(dev, steps=3):
    import bench
    import brainmagick_b200 as bb
    from brainmagick_b200 import functional as BF, synthetic
    cfg = bench.CONFIGS["cfg2"]
    C, Tc, F, S = cfg["C"], cfg["T"], cfg["F"], cfg["S"]
    torch.use_deterministic_algorithms(True)
    torch.manual_seed(2036)
    model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, n_subjects=S,
                          **{k: (dict(v) if isinstance(v, dict) else v) for k, v in bench.CLIP_CONV.items()}).to(dev)
    clip = bb.ClipLoss().to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=3e-4, betas=(0.9, 0.999), fused=True)
    positions = synthetic.normalised_positions(S, C, seed=7)
    recs = [synthetic.SyntheticRecording(s, positions[s]) for s in range(S)]
    meg, feats, subj = (t.to(dev) for t in bench.make_host_batch(cfg, B, 2036))
    batch = synthetic.SyntheticBatch(meg, subj, [recs[s] for s in subj.tolist()])
    mask = torch.ones(B, 1, Tc, dtype=torch.bool, device=dev)
    model.train()
    clip.train()
    out = {}
    for i in range(steps):
        opt.zero_grad(set_to_none=True)
        est = model(dict(meg=meg), batch)
        loss = clip(est, feats, mask)
        loss.backward()
        out[f"step{i}_loss"] = _digest(loss)
        if i == steps - 1:
            out["step_estimate"] = _digest(est)
            for n, p in model.named_parameters():
                if p.grad is not None:
                    out["step_grad_" + n] = _digest(p.grad)
        opt.step()
    for n, p in model.named_parameters():
        out["step_param_" + n] = _digest(p)
    for n, b in model.named_buffers():
        out["step_buffer_" + n] = _digest(b)
    BF.check_tc_status()
    torch.use_deterministic_algorithms(False)
    return out


def compare(a, b):
    da, db = (json.load(open(os.path.join(d, "digests.json"))) for d in (a, b))
    diff = sorted(k for k in set(da) | set(db) if da.get(k) != db.get(k))
    sa, sb = np.load(os.path.join(a, "stats.npz")), np.load(os.path.join(b, "stats.npz"))
    rel = {k: float(np.max(np.abs(sa[k] - sb[k]) / np.maximum(np.abs(sa[k]), 1e-300))) for k in sa.files}
    return dict(outputs=len(da), differing=diff, bitwise_equal=not diff, stats_max_rel_diff=rel)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default="", help="path of the libbm_b200.so to load (default: the in-tree build)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=24)
    ap.add_argument("--no-kernels", action="store_true", help="skip the timings")
    ap.add_argument("--dump", default="")
    ap.add_argument("--compare", nargs=2, metavar="DIR")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if args.compare:
        res = compare(*args.compare)
    else:
        if args.lib:
            _lib.LIB_PATH = os.path.abspath(args.lib)
        assert torch.cuda.is_available(), "profiles/conv_pipeline_cost.py measures on cuda:0"
        dev = torch.device("cuda:0")
        torch.cuda.set_device(dev)
        from profiles.input_grad_cost import card
        res = dict(card=card(), lib=_lib.LIB_PATH, batch=B)
        if not args.no_kernels:
            res["kernels"] = kernels(args, dev)
        if args.dump:
            os.makedirs(args.dump, exist_ok=True)
            res["dumped"] = dump(args, dev)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
