"""Micro-benchmarks of the SURVEY 8(f) rows built after the training step (batch preparation, retrieval evaluation,
DeepMel feature model), each beside a bounded CPU sample of its oracle.  Not the headline metric (that is bench.py);
run on one GPU as a leg of bench.py (the oracle imports below are that leg's `cpu_baseline`):

    python bench.py --next-rows                   # writes gpurun_out/next_rows.json and prints it

Timing: CUDA events on the launching stream after warm-up; inputs larger than L2 (or flushed by the working set).
"""
from __future__ import annotations

import json
import os
import sys
import time
import traceback
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from brainmagick_b200 import functional as BF                      # noqa: E402
from brainmagick_b200 import norm as bnorm                         # noqa: E402
from brainmagick_b200 import retrieval, synthetic                  # noqa: E402
from brainmagick_b200.features import DeepMel                      # noqa: E402
from brainmagick_b200.losses import ClipLoss                       # noqa: E402

DEV = "cuda"


def peaks():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            p = json.load(f)
        return float(p["hbm_gbs"]), float(p["bf16_tflops"])
    except Exception:
        return 6569.6, 1701.0


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


class _Builder(dict):
    def __init__(self, dim):
        super().__init__(wav=types.SimpleNamespace(normalizable=True, categorical=False, cardinality=0))
        self.dimension = dim

    def get_slice(self, name):
        return slice(0, self.dimension)


def bench_prep():
    from oracle import prep_oracle
    B, C, T, F, R, off = 256, 273, 361, 1024, 27, 18
    rng = np.random.RandomState(0)
    sc = bnorm.BatchScaler(_Builder(F))
    center = {r: (rng.randn(C) * 0.1).astype(np.float32) for r in range(R)}
    scale = {r: (0.5 + rng.rand(C)).astype(np.float32) for r in range(R)}
    for r in range(R):
        s = bnorm.Scaler()
        s.center_, s.scale_ = torch.from_numpy(center[r]), torch.from_numpy(scale[r])
        sc.meg_scalers[r] = s
    sc.feature_scalers["wav"].center_, sc.feature_scalers["wav"].scale_ = torch.tensor(0.25), torch.tensor(1.75)
    rec = rng.randint(0, R, size=B)
    batch = synthetic.SyntheticBatch(torch.randn(B, C, T, device=DEV) * 3, torch.zeros(B, dtype=torch.long, device=DEV), [],
                                     features=torch.randn(B, F, T, device=DEV),
                                     features_mask=torch.ones(B, 1, T, dtype=torch.bool, device=DEV),
                                     recording_index=torch.from_numpy(rec).to(DEV))
    sr = bnorm.ScaleReject(sc, limit=20.0, clip=True)
    before = BF._lib.launch_count()
    ms = timed(lambda: sr.prepare(batch, off), 20)
    launches = (BF._lib.launch_count() - before) // 23
    alg = 2 * 4 * B * (C + F) * (T - off)
    hbm, _ = peaks()
    # CPU: the oracle (vectorised numpy; the reference itself loops over the samples in Python) on 32 segments
    n = 32
    meg_h, feat_h = batch.meg[:n].cpu().numpy(), batch.features[:n].cpu().numpy()
    mask_h = np.ones((n, 1, T), dtype=bool)
    t0 = time.perf_counter()
    reps = 3
    for _ in range(reps):
        prep_oracle.prepare(meg_h, rec[:n], center, scale, feat_h, mask_h, np.full(F, 0.25, np.float32),
                            np.full(F, 1.75, np.float32), limit=20.0, clip=True, offset_samples=off)
    cpu_s = (time.perf_counter() - t0) / reps
    return dict(workload=f"scale+clamp+crop B={B} C={C} F={F} T={T}->{T - off}", ms_per_batch=ms,
                segments_per_s=B / ms * 1e3, launches_per_batch=launches,
                roofline=dict(bound="hbm", achieved=alg / ms / 1e6, peak=hbm, unit="GB/s", frac=alg / ms / 1e6 / hbm,
                              algorithmic_bytes=alg),
                cpu_baseline=dict(value=n / cpu_s, unit="segments/s", kind="port", cores=1,
                                  sample=f"{n} segments x {reps}"))


def bench_retrieval():
    from oracle import eval_oracle
    N, M, F, T = 1024, 4096, 1024, 360
    clip = ClipLoss().eval()
    gen = torch.Generator(device=DEV).manual_seed(1)
    trues = torch.randn(M, F, T, device=DEV, generator=gen)
    seg = torch.randint(0, M, (N,), device=DEV, generator=gen)
    preds = 0.02 * trues[seg] + torch.randn(N, F, T, device=DEV, generator=gen)
    labels = torch.arange(M, device=DEV, dtype=torch.int64) * 7 + 3
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    bank = retrieval.CandidateBank(clip, trues)
    torch.cuda.synchronize()
    bank_s = time.perf_counter() - t0
    del trues
    acc = {}

    def run():
        acc.update(retrieval.retrieval_accuracy(clip, preds, None, labels[seg], labels, topk=(1, 5, 10),
                                                batch_size=1024, bank=bank))
    before = BF._lib.launch_count()
    t0 = time.perf_counter()
    run()
    torch.cuda.synchronize()
    first_s = time.perf_counter() - t0
    launches = BF._lib.launch_count() - before
    ms = timed(run, 3, warmup=1)
    BF.check_tc_status()
    flops = 2.0 * N * M * F * T
    _, bf16 = peaks()
    # CPU: the oracle on 16 queries x 256 candidates of the same F*T (work scales with queries x candidates)
    nq, nc = 16, 256
    p_h, t_h = preds[:nq].cpu(), bank.rows[:nc].reshape(nc, F, T).cpu()
    t0 = time.perf_counter()
    probs = eval_oracle.builds_probs(p_h, t_h, batch_size=nq)
    eval_oracle.accuracy_from_probs(probs, torch.zeros(nq, dtype=torch.int64), torch.arange(nc), 10)
    cpu_s = time.perf_counter() - t0
    cpu_pairs = nq * nc / cpu_s
    return dict(workload=f"top-k retrieval N={N} queries x M={M} candidates, F*T={F * T}", ms_per_pass=ms,
                first_pass_s=first_s, bank_build_s=bank_s, launches_per_pass=launches,
                queries_per_s=N / ms * 1e3, query_candidate_pairs_per_s=N * M / ms * 1e3, top10_accuracy=acc.get(10),
                roofline=dict(bound="tensor", achieved=flops / ms / 1e9, peak=bf16 / 6, unit="TFLOP/s",
                              frac=flops / ms / 1e9 / (bf16 / 6), note="3xTF32: peak = measured bf16 / 6"),
                cpu_baseline=dict(value=cpu_pairs, unit="query-candidate pairs/s", kind="port",
                                  cores=torch.get_num_threads(), sample=f"{nq} queries x {nc} candidates"))


def bench_deepmel():
    from oracle import bm_oracle, deepmel_oracle
    B, T = 256, 360
    kw = dict(n_hidden_channels=320, n_hidden_layers=10, n_out_channels=768, kernel=3, stride=1, dilation_growth=2,
              dilation_period=5, batch_norm=True, activation_on_last=False, skip=True, glu_context=1, glu=2)
    torch.manual_seed(0)
    model = DeepMel(n_in_channels=120, **kw).to(DEV).train()
    clip = ClipLoss().to(DEV)
    mel = torch.randn(B, 120, T, device=DEV)
    est = torch.randn(B, 768, T, device=DEV, requires_grad=True)
    mask = torch.ones(B, 1, T, dtype=torch.bool, device=DEV)

    def step():
        model.zero_grad(set_to_none=True)
        est.grad = None
        loss = clip(est, model(mel), mask)
        loss.backward()
    before = BF._lib.launch_count()
    step()
    torch.cuda.synchronize()
    launches = BF._lib.launch_count() - before
    ms = timed(step, 10)
    BF.check_tc_status()
    conv = lambda cin, cout: 2.0 * cin * cout * 3 * T          # noqa: E731
    fwd = conv(120, 320) + 8 * conv(320, 320) + conv(320, 768) + 4 * conv(320, 640) + conv(768, 1536)
    clip_f = 2.0 * B * 768 * T                                   # per segment, scores only
    flops = B * (3 * fwd + 3 * clip_f)
    _, bf16 = peaks()
    # CPU: oracle, 8 segments, one step
    nb = 8
    params = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    okw = {k: v for k, v in kw.items() if k not in ("stride", "n_hidden_channels", "n_hidden_layers", "n_out_channels")}
    spec = deepmel_oracle.deep_mel_spec(120, 320, 10, 768, **okw)
    p = {k: v.clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in params.items()}
    m_h, e_h = mel[:nb].cpu(), est[:nb].detach().cpu().requires_grad_(True)
    t0 = time.perf_counter()
    bm_oracle.clip_loss(e_h, deepmel_oracle.conv_sequence(m_h, p, spec, training=True)).backward()
    cpu_s = time.perf_counter() - t0
    return dict(workload=f"DeepMel 120->9x320->768 + ClipLoss (estimate and candidate gradients), B={B}, T={T}",
                ms_per_step=ms, segments_per_s=B / ms * 1e3, launches_per_step=launches,
                roofline=dict(bound="tensor", achieved=flops / ms / 1e9, peak=bf16 / 6, unit="TFLOP/s",
                              frac=flops / ms / 1e9 / (bf16 / 6), note="algorithmic fwd+bwd FLOPs of the convolutions and "
                              "the three CLIP GEMMs; 3xTF32 peak = measured bf16 / 6"),
                cpu_baseline=dict(value=nb / cpu_s, unit="segments/s", kind="port", cores=torch.get_num_threads(),
                                  sample=f"{nb} segments, 1 step"))


def main(emit=print):
    out = dict(device=torch.cuda.get_device_name(0))
    for name, fn in (("prep", bench_prep), ("deepmel", bench_deepmel), ("retrieval", bench_retrieval)):
        try:
            out[name] = fn()
        except Exception as exc:             # keep the other rows' numbers
            out[name] = dict(error=f"{type(exc).__name__}: {exc}", trace=traceback.format_exc()[-1500:])
        torch.cuda.empty_cache()
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "next_rows.json"), "w") as f:
        json.dump(out, f, indent=1)
    emit(json.dumps(out))


if __name__ == "__main__":
    main()
