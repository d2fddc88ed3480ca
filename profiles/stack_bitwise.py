"""Bitwise fingerprint of deterministic training steps, for comparing two builds of the library's host code.

Under torch.use_deterministic_algorithms(True), from fixed seeds:
  * 3 SimpleConv training steps at bench.py's cfg2 (forward, ClipLoss, backward, Adam), and the same for the front's ablation
    rows merger=False, initial_linear=0 and subject_layers=False with subject_dim=64, and for the head's rows gelu=False
    and complex_out=False;
  * 3 cfg4 training steps (120 output channels: the FP32-FMA head behind tensor-core layers);
  * 3 cfg2 head-only steps: every parameter but `final.*` frozen, Adam on `final.*`;
  * a cfg2 attribution step: eval mode, every parameter frozen, meg requiring grad;
  * 3 stand-alone ChannelMerger -> SubjectLayers steps at clip_conv's widths (270 merger channels, pos_dim 2048), with the
    gradient reaching meg;
  * 3 DeepMel training steps at conf/feature_model/deep_mel.yaml's widths (ClipLoss against a trainable estimate, Adam on
    both).
Every loss, output, gradient, parameter and BatchNorm running statistic after each step is hashed (sha256 of its bytes), so
two host-code versions that issue the same kernels must give identical fingerprints.

    python profiles/stack_bitwise.py --dump a.json [--root TREE]    # TREE: the checkout whose brainmagick_b200 is imported
    python profiles/stack_bitwise.py --compare a.json b.json

Needs cuda:0 for --dump.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


ROWS = {"simpleconv": {}, "no_merger": dict(merger=False), "no_initial_linear": dict(initial_linear=0),
        "no_subject_layers": dict(subject_layers=False, subject_dim=64), "no_gelu": dict(gelu=False),
        "no_complex_out": dict(complex_out=False)}                       # SimpleConv training steps: tag -> overrides


def _digest(t) -> str:
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def _record(out, tag, loss, est, modules):
    out[f"{tag}.loss"] = _digest(loss)
    out[f"{tag}.estimate"] = _digest(est)
    for m_name, m in modules.items():
        for name, p in m.named_parameters():
            out[f"{tag}.{m_name}.grad.{name}"] = None if p.grad is None else _digest(p.grad)
        for name, v in m.state_dict().items():
            out[f"{tag}.{m_name}.state.{name}"] = _digest(v)


def dump(steps, batch, deepmel_batch):
    import torch
    import brainmagick_b200 as bb                  # first: from --root, before bench.py puts this tree on the path
    from brainmagick_b200 import functional as BF, synthetic
    sys.path.append(ROOT)
    import bench

    torch.use_deterministic_algorithms(True)
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    out = {"library": os.path.abspath(bb.__file__)}

    def data(name):
        cfg = bench.CONFIGS[name]
        C, T, S = cfg["C"], cfg["T"], cfg["S"]
        positions = synthetic.normalised_positions(S, C, seed=7)
        recs = [synthetic.SyntheticRecording(s, positions[s]) for s in range(S)]
        meg, feats, subj = (t.to(dev) for t in bench.make_host_batch(cfg, batch, 2036))
        return cfg, meg, feats, subj, synthetic.SyntheticBatch(meg, subj, [recs[s] for s in subj.tolist()])

    cfg, meg, feats, subj, sbatch = data("cfg2")
    T, S = cfg["T"], cfg["S"]
    mask = torch.ones(batch, 1, T, dtype=torch.bool, device=dev)
    clip = bb.ClipLoss().to(dev).train()

    def simpleconv(cfg=cfg, **overrides):
        kw = {k: (dict(v) if isinstance(v, dict) else v) for k, v in bench.CLIP_CONV.items()}
        kw.update(overrides)
        torch.manual_seed(2036)
        model = bb.SimpleConv(in_channels=dict(meg=cfg["C"]), out_channels=cfg["F"], n_subjects=cfg["S"], **kw)
        return model.to(dev).train()

    def train(tag, model, params, meg, feats, sbatch):
        opt = torch.optim.Adam(params, lr=3e-4)
        for step in range(steps):
            opt.zero_grad(set_to_none=True)
            est = model(dict(meg=meg), sbatch)
            loss = clip(est, feats, mask)
            loss.backward()
            _record(out, f"{tag}.{step}", loss, est, {"model": model})
            opt.step()
        BF.check_tc_status()

    for tag, overrides in ROWS.items():
        model = simpleconv(**overrides)
        train(tag, model, model.parameters(), meg, feats, sbatch)
    model = simpleconv()
    model.requires_grad_(False)
    model.final.requires_grad_(True)
    train("head_only", model, model.final.parameters(), meg, feats, sbatch)
    cfg4, meg4, feats4, _, sbatch4 = data("cfg4")
    model = simpleconv(cfg4)
    train("cfg4", model, model.parameters(), meg4, feats4, sbatch4)

    model = simpleconv().eval().requires_grad_(False)
    meg_in = meg.clone().requires_grad_(True)
    est = model(dict(meg=meg_in), sbatch)
    loss = clip(est, feats, mask)
    loss.backward()
    _record(out, "attribution", loss, est, {"model": model})
    out["attribution.grad.meg"] = _digest(meg_in.grad)
    BF.check_tc_status()

    torch.manual_seed(2038)
    merger = bb.ChannelMerger(270, pos_dim=2048, dropout=0.2, n_subjects=S).to(dev).train()
    layer = bb.SubjectLayers(270, 270, S).to(dev)
    gout = torch.randn(batch, 270, T, device=dev)
    opt = torch.optim.Adam(list(merger.parameters()) + list(layer.parameters()), lr=3e-4)
    for step in range(steps):
        opt.zero_grad(set_to_none=True)
        meg_in = meg.clone().requires_grad_(True)
        y = layer(merger(meg_in, sbatch), subj)
        y.backward(gout)
        _record(out, f"merger_subject_layers.{step}", (y * gout).sum(), y, {"merger": merger, "subject_layers": layer})
        out[f"merger_subject_layers.{step}.grad.meg"] = _digest(meg_in.grad)
        opt.step()
    BF.check_tc_status()

    torch.manual_seed(2037)
    dm = bb.DeepMel(n_in_channels=120, n_hidden_channels=320, n_hidden_layers=10, n_out_channels=768, kernel=3, stride=1,
                    dilation_growth=2, dilation_period=5, batch_norm=True, activation_on_last=False, skip=True,
                    glu_context=1, glu=2).to(dev).train()
    mel = torch.randn(deepmel_batch, 120, T, device=dev)
    brain = torch.randn(deepmel_batch, 768, T, device=dev).requires_grad_(True)
    opt = torch.optim.Adam(list(dm.parameters()) + [brain], lr=3e-4)
    mask = torch.ones(deepmel_batch, 1, T, dtype=torch.bool, device=dev)
    for step in range(steps):
        opt.zero_grad(set_to_none=True)
        cand = dm(mel)
        loss = clip(brain, cand, mask)
        loss.backward()
        _record(out, f"deepmel.{step}", loss, cand, {"deepmel": dm})
        out[f"deepmel.{step}.grad.brain"] = _digest(brain.grad)
        opt.step()
    BF.check_tc_status()
    return out


def compare(a, b):
    keys = sorted((set(a) | set(b)) - {"library"})
    diff = [k for k in keys if a.get(k) != b.get(k)]
    print(json.dumps(dict(compared=len(keys), differ=len(diff), first=diff[:20])))
    return not diff


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dump", default="")
    ap.add_argument("--root", default=ROOT, help="tree whose brainmagick_b200 package is imported")
    ap.add_argument("--compare", nargs=2, default=None)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--deepmel-batch", type=int, default=64)
    args = ap.parse_args()
    if args.compare:
        a, b = (json.load(open(p)) for p in args.compare)
        sys.exit(0 if compare(a, b) else 1)
    sys.path.insert(0, os.path.abspath(args.root))
    res = dump(args.steps, args.batch, args.deepmel_batch)
    with open(args.dump, "w") as f:
        json.dump(res, f, indent=0)
    print(f"{len(res)} fingerprints from {res['library']} -> {args.dump}")


if __name__ == "__main__":
    main()
