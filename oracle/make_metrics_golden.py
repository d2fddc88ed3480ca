"""TEST INFRASTRUCTURE ONLY -- stores what the verbatim reference test metrics (bm/metrics.py: OnlineCorrelation, L2Reg,
L1Reg, ClassificationAcc, plain PyTorch on the CPU) compute, so that tests/test_metrics_cpu.py and
tests/test_gpu_metrics.py can hold the drop-in metrics to them wherever the tests run (the reference tree is needed only
to regenerate them).  bm/metrics.py is loaded by file path; it imports only torch.

    python oracle/make_metrics_golden.py      # writes tests/golden/metrics_*.npz

Each file holds one case, run as play.get_test_metrics runs the metrics: for each recording r, fresh metrics, then
`update(left, right, mask)` per batch, then `get()`.
  metric j:  `kinds` (class name), `names`, slices `l_start`, `l_stop`, `r_start`, `r_stop` (-1: None)
  inputs:    `left_{r}_{u}`, `right_{r}_{u}`, `mask_{r}_{u}` per update u < `updates_{r}`; with `chunk` > 0 instead one
             `left_{r}`, `right_{r}`, `mask_{r}` updated in chunks of `chunk` rows; `crop` > 0: every update takes
             `[..., crop:]` of all three, as the solver's time crop
  results:   `result_{r}_{j}` (get()) and `error_{r}_{j}` (the exception's class name, or ""); `reduced_{j}` the metric
             class's reduce() over the recordings' get().float() when no recording raised (NaN otherwise)

  metrics_encode_corr   corr_meg over 3 fp64 updates [B, 5, 11] with ragged [B, 1, T] masks (B = 4, 4, 3)
  metrics_decode_mix    a regression slice (3 channels: L2Reg and the correlation) and a categorical one (K = 4:
                        ClassificationAcc) with tied logits, -100 and fractional targets, masked positions; 2 recordings
                        of 2 updates, and reduce()
  metrics_fp32_chunks   bm/test_metrics.py's inputs: fp32 [2048, 4], b = sigma * noise + a for sigma = 1e-6 ... 1e4 (one
                        recording each), in chunks of 16
  metrics_mask_shapes   a [1, 1, T] mask (the count adds 1 per update, not N) and a full [N, C, T] mask
  metrics_offset        the decode mix read at an odd element offset (crop 3)
  metrics_reset         a fully masked first update containing an inf, then ordinary updates: the reset drops the NaN
  metrics_errors        a column never counted (AssertionError), an instability from large offsets with tiny noise
                        (ValueError), every mask False (the accumulative metrics' CPU [0.])
"""
from __future__ import annotations

import importlib.util
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_loader  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def _load_metrics():
    spec = importlib.util.spec_from_file_location("ref_bm_metrics", os.path.join(ref_loader.REF, "metrics.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _ragged(gen, B, T, lo=2):
    """[B, 1, T] mask: sample b is True on its first L_b steps, sample 0 on all of them (every column is counted)"""
    lengths = torch.randint(lo, T + 1, (B,), generator=gen)
    lengths[0] = T
    return (torch.arange(T)[None, None, :] < lengths[:, None, None])


def _decode_batch(gen, B, T, masked=True):
    """(estimate [B, 3 + 4, T], ground truth [B, 3 + 1, T], mask [B, 1, T]) of a decoder with a 3-channel regression
    feature and a 4-class categorical one"""
    est = torch.randn(B, 7, T, generator=gen, dtype=torch.float64)
    gt = torch.randn(B, 4, T, generator=gen, dtype=torch.float64)
    gt[:, :3] += 0.5 * est[:, :3]
    est[:, 3:7] = torch.randint(0, 3, (B, 4, T), generator=gen).double()            # many tied logits
    gt[:, 3] = torch.randint(0, 4, (B, T), generator=gen).double()
    gt[0, 3, :3] = -100.0
    gt[-1, 3, 1] = 1.5
    mask = _ragged(gen, B, T) if masked else torch.ones(B, 1, T, dtype=torch.bool)
    return est, gt, mask


DECODE = [("L2Reg", "l2_mel", 0, 3, 0, 3), ("OnlineCorrelation", "corr_mel", 0, 3, 0, 3),
          ("ClassificationAcc", "acc_phoneme", 3, 7, 3, 4)]
REGRESSION = [("OnlineCorrelation", "corr", -1, -1, -1, -1), ("L1Reg", "l1", -1, -1, -1, -1),
              ("L2Reg", "l2", -1, -1, -1, -1)]


def cases():
    gen = torch.Generator().manual_seed(11)
    d = {}

    recs = [[]]
    for B in (4, 4, 3):
        a = torch.randn(B, 5, 11, generator=gen, dtype=torch.float64)
        recs[0].append((a, 0.7 * a + torch.randn(B, 5, 11, generator=gen, dtype=torch.float64), _ragged(gen, B, 11)))
    d["encode_corr"] = ([("OnlineCorrelation", "corr_meg", -1, -1, -1, -1)], recs, {})

    d["decode_mix"] = (DECODE, [[_decode_batch(gen, 5, 9), _decode_batch(gen, 5, 9)] for _ in range(2)], {})

    recs = []
    for sigma in (1e-6, 1e-2, 1, 100, 1e4):
        a = torch.randn(2048, 4, generator=gen)
        b = sigma * torch.randn(2048, 4, generator=gen) + a
        recs.append([(a, b, torch.ones_like(a).bool())])
    d["fp32_chunks"] = ([("OnlineCorrelation", "corr", -1, -1, -1, -1)], recs, dict(chunk=16))

    recs = [[], []]
    for _ in range(3):
        a = torch.randn(6, 3, 8, generator=gen, dtype=torch.float64)
        b = a + torch.randn(6, 3, 8, generator=gen, dtype=torch.float64)
        recs[0].append((a, b, torch.rand(1, 1, 8, generator=gen) > 0.3))
        recs[1].append((a, b, torch.rand(6, 3, 8, generator=gen) > 0.3))
    d["mask_shapes"] = (REGRESSION, recs, {})

    d["offset"] = (DECODE, [[_decode_batch(gen, 4, 12), _decode_batch(gen, 3, 12)]], dict(crop=3))

    est, gt, _ = _decode_batch(gen, 4, 9)
    est[1, 0, 2] = float("inf")
    est[2, 4, 3] = float("inf")
    first = (est, gt, torch.zeros(4, 1, 9, dtype=torch.bool))
    d["reset"] = (DECODE + [("L1Reg", "l1_mel", 0, 3, 0, 3)], [[first, _decode_batch(gen, 4, 9), _decode_batch(gen, 4, 9)]],
                  {})

    a = torch.randn(6, 2, 5, generator=gen, dtype=torch.float64)
    never = torch.rand(6, 2, 5, generator=gen) > 0.2
    never[:, 1, 3] = False
    big = 1e9 + 1e-6 * torch.randn(64, 2, 16, generator=gen, dtype=torch.float64)
    recs = [[(a, a + 0.1, never)],
            [(big, big.flip(0), torch.ones(64, 1, 16, dtype=torch.bool))],
            [(a, a, torch.zeros(6, 1, 5, dtype=torch.bool)), (a, a, torch.zeros(6, 1, 5, dtype=torch.bool))]]
    d["errors"] = ([("OnlineCorrelation", "corr", -1, -1, -1, -1), ("L2Reg", "l2", -1, -1, -1, -1)], recs, {})
    return d


def _slice(start, stop):
    return slice(None if start < 0 else start, None if stop < 0 else stop)


def _updates(rec, chunk, crop):
    for left, right, mask in rec:
        if chunk:
            for k in range(0, left.shape[0], chunk):
                yield left[k:k + chunk], right[k:k + chunk], mask[k:k + chunk]
        elif crop:
            yield left[..., crop:], right[..., crop:], mask[..., crop:]
        else:
            yield left, right, mask


def run(M, specs, recs, chunk=0, crop=0):
    """the reference's metrics over the recordings -> (results[r][j], errors[r][j], reduced[j])"""
    results, errors = [], []
    for rec in recs:
        metrics = [getattr(M, kind)(_slice(ls, le), _slice(rs, re_), name=name) for kind, name, ls, le, rs, re_ in specs]
        for left, right, mask in _updates(rec, chunk, crop):
            for m in metrics:
                m.update(left, right, mask)
        res, err = [], []
        for m in metrics:
            try:
                res.append(m.get())
                err.append("")
            except (ValueError, AssertionError) as e:
                res.append(torch.full((1,), float("nan")))
                err.append(type(e).__name__)
        results.append(res)
        errors.append(err)
    reduced = []
    for j, (kind, *_rest) in enumerate(specs):
        ok = all(not errors[r][j] for r in range(len(recs)))
        reduced.append(getattr(M, kind).reduce([results[r][j].cpu().float() for r in range(len(recs))]) if ok
                       else float("nan"))
    return results, errors, reduced


def main():
    torch.set_num_threads(1)
    M = _load_metrics()
    for case, (specs, recs, opts) in cases().items():
        results, errors, reduced = run(M, specs, recs, **opts)
        arrays = dict(kinds=np.array([s[0] for s in specs]), names=np.array([s[1] for s in specs]),
                      l_start=np.array([s[2] for s in specs]), l_stop=np.array([s[3] for s in specs]),
                      r_start=np.array([s[4] for s in specs]), r_stop=np.array([s[5] for s in specs]),
                      chunk=np.int64(opts.get("chunk", 0)), crop=np.int64(opts.get("crop", 0)),
                      recordings=np.int64(len(recs)), reduced=np.array(reduced, dtype=np.float64))
        for r, rec in enumerate(recs):
            if opts.get("chunk"):
                (left, right, mask), = rec
                arrays.update({f"left_{r}": left.numpy(), f"right_{r}": right.numpy(), f"mask_{r}": mask.numpy()})
            else:
                arrays[f"updates_{r}"] = np.int64(len(rec))
                for u, (left, right, mask) in enumerate(rec):
                    arrays.update({f"left_{r}_{u}": left.numpy(), f"right_{r}_{u}": right.numpy(),
                                   f"mask_{r}_{u}": mask.numpy()})
            for j in range(len(specs)):
                arrays[f"result_{r}_{j}"] = results[r][j].numpy()
                arrays[f"error_{r}_{j}"] = np.array(errors[r][j])
        path = os.path.join(OUT, f"metrics_{case}.npz")
        np.savez_compressed(path, **arrays)
        print(path, os.path.getsize(path), [e for err in errors for e in err if e], reduced)


if __name__ == "__main__":
    main()
