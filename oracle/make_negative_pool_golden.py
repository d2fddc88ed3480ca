"""TEST INFRASTRUCTURE ONLY -- stores what the reference's negative pool (oracle/negative_pool_oracle.py, the restated
bm/solver.py:152-164 and 358-371) feeds the verbatim reference `ClipLoss` (bm/losses.py, loaded by oracle/ref_loader.py),
step by step, so that tests/test_negative_pool_cpu.py can hold the drop-in `NegativePool` + `ClipLoss` to it wherever the
tests run (the reference tree is needed only to regenerate them).

    python oracle/make_negative_pool_golden.py            # writes tests/golden/negative_pool_*.npz
    python oracle/make_negative_pool_golden.py --check    # regenerates in memory and compares with the stored files

Each file holds one run: `meta` = [negatives (-1: None), negative_pool_size as given (-1: None), seed, steps, F, T].  The
CPU default generator is seeded with `seed` before the first step and drawn from only by the pool's `torch.randperm`; the
step data come from a generator of their own.  Per step i:
  `train_{i}` 1 for a training step, `out_{i}` the batch's outputs [B, F, T], `est_{i}` the estimates, `ran_{i}` 1 when
  the pool code ran, `kept_{i}` its randperm draw (int64), `cand_{i}` the candidates the loss received, `loss_{i}`, `gest_{i}`
  the gradient of the loss on the estimates, `gout_{i}` on the outputs (zeros when they do not require grad), `pool_{i}`
  the phase's pool after the step (`pool_train_{i}` and `pool_valid_{i}` both)
and `final_rand` = torch.rand(4) after the last step, which pins the generator's stream.

  negative_pool_fill      B = 3, negatives = 7, default pool (14), 6 steps: the empty start, the filling, a full pool and
                          re-drawn (duplicated) rows
  negative_pool_truncate  negative_pool_size = negatives = 5, B = 3
  negative_pool_phases    interleaved train and valid steps, one pool each
  negative_pool_noop      B = 6 >= negatives = 4, outputs that require grad: the candidates pass through, the gradient flows
  negative_pool_ragged    B varies per step (as after ScaleReject), negatives = 8, pool 12
  negative_pool_odd       F*T = 21 (not a multiple of 4): the drop-in's materialized path
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from oracle.negative_pool_oracle import HostNegativePool  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

# name: (negatives, pool_size, seed, F, T, [(B, training), ...], outputs require grad)
CASES = {
    "negative_pool_fill": (7, None, 11, 4, 10, [(3, True)] * 6, False),
    "negative_pool_truncate": (5, 5, 12, 4, 12, [(3, True)] * 5, False),
    "negative_pool_phases": (6, None, 13, 2, 16, [(3, True), (3, False), (2, True), (3, False), (3, True), (2, False)],
                             False),
    "negative_pool_noop": (4, None, 14, 4, 8, [(6, True), (4, False)], True),
    "negative_pool_ragged": (8, 12, 15, 4, 9, [(4, True), (2, True), (5, True), (3, True), (1, True), (4, True)], False),
    "negative_pool_odd": (6, None, 16, 3, 7, [(3, True)] * 4, False),
}


def run(name):
    negatives, pool_size, seed, F, T, steps, out_grad = CASES[name]
    _, _, losses = ref_loader.load_reference()
    data = torch.Generator().manual_seed(1000 + seed)
    pool = HostNegativePool(negatives, pool_size)
    clip = losses.ClipLoss()
    z = {"meta": np.array([negatives, -1 if pool_size is None else pool_size, seed, len(steps), F, T], dtype=np.int64)}
    torch.manual_seed(seed)
    for i, (B, training) in enumerate(steps):
        out = torch.randn(B, F, T, generator=data).requires_grad_(out_grad)
        est = torch.randn(B, F, T, generator=data).requires_grad_(True)
        clip.train(training)
        cand = pool.complete(out, training)
        loss = clip(est, cand, torch.ones(B, 1, T, dtype=torch.bool))
        loss.backward()
        z[f"train_{i}"] = np.array(int(training))
        z[f"out_{i}"] = out.detach().numpy()
        z[f"est_{i}"] = est.detach().numpy()
        z[f"ran_{i}"] = np.array(int(pool.last_kept is not None))
        z[f"kept_{i}"] = (pool.last_kept if pool.last_kept is not None else torch.empty(0, dtype=torch.long)).numpy()
        z[f"cand_{i}"] = cand.detach().numpy()
        z[f"loss_{i}"] = loss.detach().numpy()
        z[f"gest_{i}"] = est.grad.numpy()
        z[f"gout_{i}"] = out.grad.numpy() if out.grad is not None else np.zeros_like(z[f"out_{i}"])
        for phase in ("train", "valid"):
            z[f"pool_{phase}_{i}"] = pool.negative_pool[phase].numpy()
    z["final_rand"] = torch.rand(4).numpy()
    return z


def main(check=False):
    bad = 0
    for name in CASES:
        z = run(name)
        path = os.path.join(OUT, name + ".npz")
        if check:
            old = np.load(path)
            same = set(old.files) == set(z) and all(np.array_equal(old[k], z[k]) for k in z)
            print(f"{name}: {'ok' if same else 'DIFFERS'}")
            bad += not same
        else:
            np.savez_compressed(path, **z)
            print("wrote", path)
    return bad


if __name__ == "__main__":
    sys.exit(1 if main(check="--check" in sys.argv) else 0)
