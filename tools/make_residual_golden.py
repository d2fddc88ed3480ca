"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/residual_*.npz, the fixtures of ConvSequence's residual-branch options
(`scale` = LayerScale, `rewrite`, `post_skip`; bm/models/common.py:65-76,123-130), by running the VERBATIM reference
classes (loaded by `oracle/ref_loader.py`) on small seeded inputs.  The reference tree does not travel with the
repository; the fixtures do.

    python tools/make_residual_golden.py            # (re)writes the residual_*.npz fixtures
    python tools/make_residual_golden.py --check    # regenerates in memory and compares with tests/golden/

ConvSequence fixtures (`SEQ_CASES`): the state_dict after a seeded construction (`p.<key>`, BatchNorm affine / running
statistics and LayerScale perturbed so that every channel differs), the input `x` [B, C0, T], the output weights `w_out`,
then a training step -- `out`, the gradients of loss = sum(out * w_out) (`g.<key>`, `g.x`) and the running statistics after
it (`bn.<key>`) -- and an eval forward / backward with those statistics (`out_eval`, `ge.<key>`, `ge.x`).  `init.<key>`:
the state_dict of the seeded construction before any perturbation.

SimpleConv fixture (`residual_simpleconv`): clip_conv with scale=0.1, rewrite=True, post_skip=True; a ClipLoss training
step laid out like the train_* fixtures of oracle/make_golden.py, plus the gradient to `meg` (`g.meg`).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

# name: ConvSequence keyword arguments (stride=1, odd kernel) + input sizes
SEQ_CASES = {
    "residual_scale": dict(channels=[6, 8, 8, 8], kernel=3, dilation_growth=2, batch_norm=True, skip=True, scale=0.1,
                           activation="gelu", B=3, T=19, seed=11),
    "residual_rewrite": dict(channels=[6, 8, 8, 8], kernel=3, dilation_growth=2, batch_norm=True, skip=True, rewrite=True,
                             leakiness=0.1, activation="gelu", B=3, T=19, seed=12),
    "residual_post_skip": dict(channels=[6, 8, 8, 8], kernel=3, dilation_growth=2, batch_norm=True, skip=True,
                               post_skip=True, activation="gelu", B=3, T=19, seed=13),
    "residual_all": dict(channels=[6, 8, 8, 8, 8], kernel=3, dilation_growth=2, batch_norm=True, skip=True, scale=0.1,
                         rewrite=True, post_skip=True, leakiness=0.05, glu=2, activation="gelu", B=3, T=21, seed=14),
    "residual_nobn_leaky": dict(channels=[5, 7, 7, 7], kernel=3, batch_norm=False, skip=True, scale=0.3, rewrite=True,
                                post_skip=True, leakiness=0.2, activation=None, B=2, T=23, seed=15),
    "residual_bare_last": dict(channels=[6, 6, 6], kernel=3, batch_norm=True, skip=True, scale=0.1, rewrite=True,
                               post_skip=True, activation_on_last=False, activation="relu", B=3, T=17, seed=16),
}

SIMPLECONV_CASE = dict(B=5, Bc=5, C=10, T=24, F=8, S=3, hidden=16, depth=4, MC=12, IL=12, P=32, seed=21,
                       extra=dict(scale=0.1, rewrite=True, post_skip=True))


def seq_kwargs(c):
    """ConvSequence keyword arguments of a SEQ_CASES entry (activation: "gelu" / "relu" / None = LeakyReLU(leakiness))."""
    act = {"gelu": torch.nn.GELU, "relu": torch.nn.ReLU, None: None}[c["activation"]]
    kw = {k: v for k, v in c.items() if k not in ("B", "T", "seed", "activation", "channels")}
    return dict(kw, stride=1, activation=act)


def _perturb(model):
    with torch.no_grad():
        for name, m in model.named_modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.add_(0.1 * torch.randn_like(m.weight))
                m.bias.add_(0.1 * torch.randn_like(m.bias))
                m.running_mean.add_(0.1 * torch.randn_like(m.running_mean))
                m.running_var.mul_(1 + 0.2 * torch.rand_like(m.running_var))
            if type(m).__name__ == "LayerScale":
                m.scale.mul_(1 + 0.5 * torch.randn_like(m.scale))


def make_seq_case(c) -> dict:
    common, _, _ = ref_loader.load_reference()
    torch.manual_seed(c["seed"])
    model = common.ConvSequence(c["channels"], **seq_kwargs(c))
    init = {k: v.detach().clone() for k, v in model.state_dict().items()}
    torch.manual_seed(1000 + c["seed"])
    _perturb(model)
    state = {k: v.detach().clone() for k, v in model.state_dict().items()}
    x = torch.randn(c["B"], c["channels"][0], c["T"])
    out = dict(x=x.numpy())
    w_out = None
    for mode in ("train", "eval"):
        model.train(mode == "train")
        model.zero_grad()
        xi = x.clone().requires_grad_(True)
        y = model(xi)
        if w_out is None:
            w_out = torch.randn_like(y)
            out["w_out"] = w_out.numpy()
        (y * w_out).sum().backward()
        tag = "g." if mode == "train" else "ge."
        out["out" if mode == "train" else "out_eval"] = y.detach().numpy()
        out[tag + "x"] = xi.grad.numpy()
        for k, v in model.named_parameters():
            out[tag + k] = v.grad.numpy()
        if mode == "train":
            for k, v in model.state_dict().items():
                if "running" in k or "num_batches" in k:
                    out["bn." + k] = v.numpy()
    for k, v in state.items():
        out["p." + k] = v.numpy()
    for k, v in init.items():
        out["init." + k] = v.numpy()
    return out


def make_simpleconv_case(c) -> dict:
    common, simpleconv, losses = ref_loader.load_reference()
    torch.manual_seed(100 + c["seed"])
    kw = ref_loader.clip_conv_kwargs(hidden=c["hidden"], depth=c["depth"], merger_channels=c["MC"],
                                     initial_linear=c["IL"], merger_pos_dim=c["P"])
    kw.update(c["extra"])
    model = simpleconv.SimpleConv(in_channels=dict(meg=c["C"]), out_channels=c["F"], n_subjects=c["S"], **kw)
    torch.manual_seed(1000 + c["seed"])
    _perturb(model)
    state = {k: v.detach().clone() for k, v in model.state_dict().items()}
    B, Bc, C, T, F, S = c["B"], c["Bc"], c["C"], c["T"], c["F"], c["S"]
    meg = torch.randn(B, C, T)
    cand = torch.randn(Bc, F, T)
    subj = torch.randint(0, S, (B,))
    recs = [ref_loader.FakeRecording(s, C, C, seed=c["seed"]) for s in range(S)]
    batch = ref_loader.FakeBatch(meg, subj, [recs[int(s)] for s in subj])
    pos_rec = torch.stack([model.merger.position_getter.get_recording_layout(r).clone() for r in recs])
    full = torch.full((S, C, 2), common.PositionGetter.INVALID)
    full[:, :pos_rec.shape[1]] = pos_rec
    model.train()
    clip = losses.ClipLoss()
    torch.manual_seed(9000 + c["seed"])
    ban = torch.rand(2)                       # the one rand(2) the training forward draws (common.py:343)
    torch.manual_seed(9000 + c["seed"])
    meg_in = meg.clone().requires_grad_(True)
    est = model(dict(meg=meg_in), batch)
    mask = torch.ones(B, 1, T, dtype=torch.bool)
    loss = clip(est, cand, mask)
    loss.backward()
    out = dict(meg=meg.numpy(), candidates=cand.numpy(), subject_index=subj.numpy(), rec_positions=full.numpy(),
               ban_centre=ban.numpy(), estimate=est.detach().numpy(), loss=loss.detach().numpy(),
               **{"g.meg": meg_in.grad.numpy()})
    for k, v in state.items():
        out["p." + k] = v.numpy()
    for k, v in model.named_parameters():
        out["g." + k] = v.grad.numpy()
    for k, v in model.state_dict().items():
        if "running" in k or "num_batches" in k:
            out["bn." + k] = v.numpy()
    return out


def all_cases():
    cases = {name: (lambda c=c: make_seq_case(c)) for name, c in SEQ_CASES.items()}
    cases["residual_simpleconv"] = lambda: make_simpleconv_case(SIMPLECONV_CASE)
    return cases


def main(check: bool) -> int:
    bad = 0
    for name, make in all_cases().items():
        arrays = make()
        path = os.path.join(OUT, name + ".npz")
        if check:
            old = np.load(path)
            same = set(old.files) == set(arrays) and all(np.array_equal(old[k], arrays[k]) for k in arrays)
            print(f"{name}: {'same' if same else 'DIFFERS'}")
            bad += not same
        else:
            np.savez_compressed(path, **arrays)
            print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB")
    return bad


if __name__ == "__main__":
    sys.exit(main("--check" in sys.argv))
