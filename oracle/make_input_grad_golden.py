"""TEST INFRASTRUCTURE ONLY -- stores the input gradients the verbatim reference computes (plain PyTorch autograd), so that
tests/test_input_grad_cpu.py can hold the drop-in's backward to `meg` and through ClipLoss.get_scores / get_probabilities to
them wherever the tests run (the reference tree is needed only to regenerate them).

    python oracle/make_input_grad_golden.py       # writes tests/golden/live_input_grad_*.npz

  live_input_grad_clip_conv   clip_conv at a small width, ragged valid sensors: meg.grad of the ClipLoss in train mode (one
                              injected spatial-dropout centre) and in eval mode, from the same parameters
  live_input_grad_ablations   meg.grad of the merger=False and subsample_meg_channels rows (oracle/make_golden.py's
                              ablation case)
  live_input_grad_clip_scores est.grad / cand.grad through get_scores and get_probabilities under a seeded upstream
                              gradient; candidate 3 is all zeros (the norm's backward at 0)
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_loader  # noqa: E402
from oracle.make_golden import ABLATION_BASE  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def _np(t):
    return t.detach().cpu().numpy()


def clip_conv(seed=611):
    common, simpleconv, losses = ref_loader.load_reference()
    torch.manual_seed(seed)
    B, C, T, F, S, hidden, MC, IL, P = 5, 13, 41, 9, 4, 24, 16, 20, 72
    kw = ref_loader.clip_conv_kwargs(hidden=hidden, depth=10, merger_channels=MC, initial_linear=IL, merger_pos_dim=P)
    model = simpleconv.SimpleConv(in_channels=dict(meg=C), out_channels=F, n_subjects=S, **kw)
    state = {k: v.detach().clone() for k, v in model.state_dict().items()}
    meg = torch.randn(B, C, T).clamp_(-20, 20)
    cand = torch.randn(B + 2, F, T)
    subj = torch.tensor([0, 1, 3, 1, 2])
    n_valid = [13, 9, 13, 6]
    recs = [ref_loader.FakeRecording(s, C, n_valid[s], seed=seed) for s in range(S)]
    batch = ref_loader.FakeBatch(meg, subj, [recs[int(s)] for s in subj])
    pos = torch.full((S, C, 2), common.PositionGetter.INVALID)
    for s in range(S):
        lay = model.merger.position_getter.get_recording_layout(recs[s])
        pos[s, :len(lay)] = lay
    out = {"p." + k: _np(v) for k, v in state.items()}
    out.update(meg=_np(meg), cand=_np(cand), subj=_np(subj), pos=_np(pos))
    for mode in ("train", "eval"):
        model.load_state_dict(state)
        model.train(mode == "train")
        x = meg.clone().requires_grad_(True)
        torch.manual_seed(seed + 1)
        ban = torch.rand(2)
        torch.manual_seed(seed + 1)                   # the merger's torch.rand(2) draws this centre in train mode
        est = model(dict(meg=x), batch)
        loss = losses.ClipLoss()(est, cand, torch.ones(B, 1, T, dtype=torch.bool))
        loss.backward()
        out.update({f"{mode}.ban": _np(ban), f"{mode}.loss": _np(loss), f"{mode}.meg_grad": _np(x.grad)})
    return out


def ablations():
    """oracle/make_golden.py's ablation case (ABLATION_BASE) with meg.requires_grad, for the rows that change what lies
    between `meg` and the encoder: merger=False and subsample_meg_channels."""
    common, simpleconv, losses = ref_loader.load_reference()
    out = {}
    for tag, change in (("no_merger", dict(merger=False)), ("subsample", dict(subsample_meg_channels=6))):
        c = dict(ABLATION_BASE)
        torch.manual_seed(c["seed"] + 3)
        kw = ref_loader.clip_conv_kwargs(hidden=c["hidden"], depth=c["depth"], merger_channels=c["MC"],
                                         initial_linear=c["IL"], merger_pos_dim=c["P"])
        kw.update(change)
        model = simpleconv.SimpleConv(in_channels=dict(meg=c["C"]), out_channels=c["F"], n_subjects=c["S"], **kw)
        B, C, T, F, S = c["B"], c["C"], c["T"], c["F"], c["S"]
        state = {k: v.detach().clone() for k, v in model.state_dict().items()}
        meg = torch.randn(B, C, T).clamp_(-20, 20)
        cand = torch.randn(B, F, T)
        subj = torch.randint(0, S, (B,))
        recs = [ref_loader.FakeRecording(s, C, C, seed=c["seed"]) for s in range(S)]
        batch = ref_loader.FakeBatch(meg, subj, [recs[int(s)] for s in subj])
        pos = torch.stack([common.PositionGetter().get_recording_layout(r).clone() for r in recs])
        model.train()
        torch.manual_seed(9200 + c["seed"])
        ban = torch.rand(2)
        torch.manual_seed(9200 + c["seed"])
        x = meg.clone().requires_grad_(True)
        est = model(dict(meg=x), batch)
        loss = losses.ClipLoss()(est, cand, torch.ones(B, 1, T, dtype=torch.bool))
        loss.backward()
        out.update({f"{tag}.p." + k: _np(v) for k, v in state.items()})
        out.update({f"{tag}.meg": _np(meg), f"{tag}.cand": _np(cand), f"{tag}.subj": _np(subj), f"{tag}.pos": _np(pos),
                    f"{tag}.ban": _np(ban), f"{tag}.loss": _np(loss), f"{tag}.meg_grad": _np(x.grad)})
    return out


def clip_scores(seed=612):
    _, _, losses = ref_loader.load_reference()
    torch.manual_seed(seed)
    Bn, Bc, F, T = 6, 7, 8, 20
    est, cand = torch.randn(Bn, F, T), torch.randn(Bc, F, T)
    cand[3] = 0
    up = torch.randn(Bn, Bc)
    out = dict(est=_np(est), cand=_np(cand), up=_np(up))
    clip = losses.ClipLoss()
    for name in ("get_scores", "get_probabilities"):
        e, c = est.clone().requires_grad_(True), cand.clone().requires_grad_(True)
        y = getattr(clip, name)(e, c)
        y.backward(up)
        out.update({f"{name}.out": _np(y), f"{name}.est_grad": _np(e.grad), f"{name}.cand_grad": _np(c.grad)})
    return out


def main():
    torch.set_num_threads(1)
    for name, fn in (("live_input_grad_clip_conv", clip_conv), ("live_input_grad_ablations", ablations),
                     ("live_input_grad_clip_scores", clip_scores)):
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **fn())
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
