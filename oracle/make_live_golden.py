"""TEST INFRASTRUCTURE ONLY -- stores what the verbatim reference computes in the "fresh input" comparisons of
tests/test_oracle.py, tests/test_oracle_vs_reference.py and tests/test_boundary.py, so that those comparisons run
wherever the tests run (the reference tree is needed only to regenerate them).

    python oracle/make_live_golden.py       # writes tests/golden/live_*.npz

Each file holds the inputs the test builds (seeded), the reference's state_dict where the test needs it (`p.<key>`) and
the reference's outputs (estimate, loss, gradients `g.<key>`, prepared batches).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_loader  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def _np(t):
    return t.detach().cpu().numpy()


def oracle_1234():
    """tests/test_oracle.py::test_oracle_matches_live_reference"""
    common, simpleconv, losses = ref_loader.load_reference()
    torch.manual_seed(1234)
    C, F, S, T, B = 9, 6, 3, 31, 5
    kw = ref_loader.clip_conv_kwargs(hidden=20, depth=10, merger_channels=8, initial_linear=12, merger_pos_dim=128)
    model = simpleconv.SimpleConv(in_channels=dict(meg=C), out_channels=F, n_subjects=S, **kw)
    meg, cand = torch.randn(B, C, T), torch.randn(B, F, T)
    subj = torch.randint(0, S, (B,))
    recs = [ref_loader.FakeRecording(s, C, seed=5) for s in range(S)]
    batch = ref_loader.FakeBatch(meg, subj, [recs[int(s)] for s in subj])
    pos = torch.stack([model.merger.position_getter.get_recording_layout(r) for r in recs])
    model.train()
    torch.manual_seed(7)
    ban = torch.rand(2)
    torch.manual_seed(7)
    est = model(dict(meg=meg.clone()), batch)
    loss = losses.ClipLoss()(est, cand, torch.ones(B, 1, T, dtype=torch.bool))
    out = {"p." + k: _np(v) for k, v in model.state_dict().items()}
    out.update(meg=_np(meg), cand=_np(cand), subj=_np(subj), pos=_np(pos), ban=_np(ban), estimate=_np(est), loss=_np(loss))
    return out


def fresh(seed, train):
    """tests/test_oracle_vs_reference.py::test_oracle_equals_live_reference_on_fresh_inputs"""
    common, simpleconv, losses = ref_loader.load_reference()
    torch.manual_seed(seed)
    B, C, T, F, S, hidden, MC, IL, P = 7, 13, 41, 9, 4, 24, 16, 20, 72
    kw = ref_loader.clip_conv_kwargs(hidden=hidden, depth=10, merger_channels=MC, initial_linear=IL, merger_pos_dim=P)
    model = simpleconv.SimpleConv(in_channels=dict(meg=C), out_channels=F, n_subjects=S, **kw)
    state = {k: v.detach().clone() for k, v in model.state_dict().items()}
    meg = torch.randn(B, C, T).clamp_(-20, 20)
    cand = torch.randn(B + 3, F, T)
    subj = torch.randint(0, S, (B,))
    n_valid = [13, 9, 13, 6]
    recs = [ref_loader.FakeRecording(s, C, n_valid[s], seed=seed) for s in range(S)]
    for b in range(B):
        meg[b, n_valid[int(subj[b])]:] = 0
    batch = ref_loader.FakeBatch(meg, subj, [recs[int(s)] for s in subj])
    pos = torch.full((S, C, 2), common.PositionGetter.INVALID)
    for s in range(S):
        lay = model.merger.position_getter.get_recording_layout(recs[s])
        pos[s, :len(lay)] = lay
    model.train(train)
    torch.manual_seed(seed + 1)
    ban = torch.rand(2)
    torch.manual_seed(seed + 1)
    est = model(dict(meg=meg.clone()), batch)
    loss = losses.ClipLoss()(est, cand, torch.ones(B, 1, T, dtype=torch.bool))
    loss.backward()
    out = {"p." + k: _np(v) for k, v in state.items()}
    out.update({"g." + n: _np(p.grad) for n, p in model.named_parameters() if p.grad is not None})
    out.update(meg=_np(meg), cand=_np(cand), subj=_np(subj), pos=_np(pos), ban=_np(ban), estimate=_np(est), loss=_np(loss))
    return out


def prep_77():
    """tests/test_oracle_vs_reference.py::test_prep_oracle_equals_live_reference_on_fresh_inputs"""
    norm = ref_loader.load_reference_norm()
    torch.manual_seed(77)
    B, C, T, off = 9, 8, 25, 2
    fb = ref_loader.FakeFeaturesBuilder({"w": (4, True), "p": (3, False)})
    scaler = norm.BatchScaler(fb, per_channel=True)
    ids = [2, 3, 10]
    for r in ids:
        scaler.meg_scalers[r] = norm.RobustScaler().fit(torch.randn(300, C) * (1 + r))
    feats_fit = torch.randn(40, fb.dimension, T)
    for fname, fs in scaler.feature_scalers.items():
        fs.fit(norm._as_nd(feats_fit[:, fb.get_slice(fname)]), norm._as_nd(torch.ones(40, 1, T, dtype=torch.bool)))
    meg = torch.randn(B, C, T) * 40
    rec = torch.tensor([2, 10, 3, 3, 2, 10, 10, 2, 3])
    feats = torch.randn(B, fb.dimension, T)
    mask = torch.ones(B, 1, T, dtype=torch.bool)
    fc, fs_ = torch.zeros(fb.dimension), torch.ones(fb.dimension)
    for fname, sc in scaler.feature_scalers.items():
        if isinstance(sc, norm.StandardScaler):
            fc[fb.get_slice(fname)], fs_[fb.get_slice(fname)] = sc.center_, sc.scale_
    out = dict(meg=_np(meg), rec=_np(rec), feats=_np(feats), mask=_np(mask), fc=_np(fc), fs=_np(fs_), ids=np.array(ids),
               off=np.array(off))
    for r in ids:
        out[f"center.{r}"] = scaler.meg_scalers[r].center_.numpy()
        out[f"scale.{r}"] = scaler.meg_scalers[r].scale_.numpy()
    for clip in (False, True):
        sr = norm.ScaleReject(scaler, limit=20.0, clip=clip)
        kept, keep = sr(ref_loader.FakeSegmentBatch(meg.clone(), feats.clone(), mask.clone(), rec.clone()))
        out[f"keep.{int(clip)}"] = _np(keep)
        out[f"kept_meg.{int(clip)}"] = _np(kept.meg[..., off:])
        out[f"kept_features.{int(clip)}"] = _np(kept.features[..., :-off])
    return out


def seeded_ctor_77():
    """tests/test_boundary.py::test_seeded_constructor_is_rng_identical_to_reference"""
    _, simpleconv, _ = ref_loader.load_reference()
    kw = dict(hidden=dict(meg=48), batch_norm=True, depth=10, dilation_period=5, kernel_size=3, skip=True,
              subject_layers=True, subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=24,
              gelu=True, merger_pos_dim=128, merger_channels=20)           # the test's constructor arguments
    torch.manual_seed(77)
    ref = simpleconv.SimpleConv(in_channels=dict(meg=30), out_channels=17, n_subjects=5, **kw)
    out = {"p." + k: _np(v) for k, v in ref.state_dict().items()}
    out["keys"] = np.array(list(ref.state_dict()))
    out["subject_layers_repr"] = np.array(repr(ref.subject_layers))
    return out


def main():
    torch.set_num_threads(1)
    for name, fn in (("live_oracle_1234", oracle_1234), ("live_fresh_501", lambda: fresh(501, True)),
                     ("live_fresh_502", lambda: fresh(502, False)), ("live_prep_77", prep_77),
                     ("live_seeded_ctor_77", seeded_ctor_77)):
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **fn())
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
