"""Pin of the oracles against the VERBATIM reference modules on fresh inputs that no other fixture holds: oracle == what
the reference computed (tests/golden/live_*.npz, stored by oracle/make_live_golden.py).  That the committed fixtures are
what the generator produces from the reference today is checked where the reference tree is present, by
`python oracle/make_golden.py --check`."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, rel_err
from oracle import bm_oracle, prep_oracle


@pytest.mark.parametrize("seed,train", [(501, True), (502, False)])
def test_oracle_equals_live_reference_on_fresh_inputs(seed, train):
    g = np.load(os.path.join(GOLDEN_DIR, f"live_fresh_{seed}.npz"))
    B, C, T, F, S, hidden, MC, IL, P = 7, 13, 41, 9, 4, 24, 16, 20, 72
    state = {k[2:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("p.")}
    meg, cand, subj = torch.from_numpy(g["meg"]), torch.from_numpy(g["cand"]), torch.from_numpy(g["subj"])
    cfg = bm_oracle.Config(in_channels=C, out_channels=F, n_subjects=S, hidden=hidden, merger_channels=MC,
                           initial_linear=IL, merger_pos_dim=P)
    ref = bm_oracle.training_step(state, cfg, meg, torch.from_numpy(g["pos"]), subj, subj, cand,
                                  ban_centre=torch.from_numpy(g["ban"]), training=train)
    assert rel_err(ref["estimate"], torch.from_numpy(g["estimate"])) < 2e-6
    assert abs(float(ref["loss"]) - float(g["loss"])) < 1e-6
    for k in g.files:
        if not k.startswith("g."):
            continue
        name, grad = k[2:], torch.from_numpy(g[k])
        if grad.norm() < 1e-6:
            assert ref["grads"][name].abs().max() < 1e-5, name
        else:
            assert rel_err(ref["grads"][name], grad) < 3e-5, name


def test_prep_oracle_equals_live_reference_on_fresh_inputs():
    g = np.load(os.path.join(GOLDEN_DIR, "live_prep_77.npz"))
    ids, off = [int(r) for r in g["ids"]], int(g["off"])
    center = {r: g[f"center.{r}"] for r in ids}
    scale = {r: g[f"scale.{r}"] for r in ids}
    for clip in (False, True):
        got = prep_oracle.prepare(g["meg"], g["rec"], center, scale, g["feats"], g["mask"], g["fc"], g["fs"], limit=20.0,
                                  clip=clip, offset_samples=off)
        assert np.array_equal(got["keep"], g[f"keep.{int(clip)}"])
        assert np.array_equal(got["meg"], g[f"kept_meg.{int(clip)}"])
        assert np.array_equal(got["features"], g[f"kept_features.{int(clip)}"])
