"""The sensor-side front's call stream (ChannelMerger attention, sensor mix, initial_linear, SubjectLayers, subject
embedding), without a GPU.

`tests/golden/abi_trace_front.json` holds the full C-ABI call stream (tests/abi_trace.py: entry point, every scalar
argument, NULL-ness of every pointer) of the steps below, stored as a table of the distinct calls ("calls") and, per step,
the indices of its calls in order ("traces").  It was recorded with `python tests/test_front_cpu.py` at the
commit before SimpleConv's encoder, its ablation rows and the stand-alone ChannelMerger / SubjectLayers came to share one
front (`functional.front_forward` / `front_backward`), so the test pins that the shared front issues exactly the calls the
separate front implementations issued.  The cases cover:
  * SimpleConv at the `full` and `mid` widths of abi_trace.CONFIGS (tensor-core chain, mixed tensor-core / FP32-FMA
    chain) for every front row: default, merger=False, initial_linear=0, subject_layers=False (with and without a
    subject embedding), a subject embedding after the full chain, and subsample_meg_channels.  Depth 2 instead of 10:
    the conv stack is pinned by abi_trace_steps.json and abi_trace_convseq.json, and the front does not depend on it;
  * per row: a training step with everything trainable, the same step with meg requiring grad, steps with the merger
    heads, initial_linear and the subject layers frozen one at a time, and an eval-mode `torch.no_grad()` forward;
  * the `small` size (the fused FP32-FMA `bm_sensor_chain_fwd` / `bm_sensor_chain_bwd`) under the same steps, whose
    frozen and meg-gradient cases set NULL pointers in the fused backward;
  * the stand-alone ChannelMerger and SubjectLayers: trainable, weights frozen with the input requiring grad, and
    everything requiring grad, each followed by a `torch.no_grad()` forward;
  * the default flags for all of these, and torch.use_deterministic_algorithms(True) and TF32 matmul precision for the
    trainable and input-gradient steps.
"""
import json
import os

import torch

import abi_trace
from test_conv_stack_cpu import _mode

FIXTURE = os.path.join(abi_trace.ROOT, "tests", "golden", "abi_trace_front.json")

ROWS = {"default": {}, "no_merger": dict(merger=False), "no_initial_linear": dict(initial_linear=0),
        "no_subject_layers": dict(subject_layers=False), "no_subject_layers_emb": dict(subject_layers=False, subject_dim=64),
        "sub_emb": dict(subject_dim=5), "subsample": dict(subsample_meg_channels=5)}
STEPS = ("train", "meg_grad", "frozen_merger", "frozen_initial_linear", "frozen_subject_layers", "eval")
MODES = ("default", "deterministic", "tf32")
MODE_STEPS = ("train", "meg_grad", "input_grad")   # the steps also recorded under the deterministic and TF32 modes
DEPTH = 2


def _simpleconv(cfg, row, step):
    """-> the step's run function, or None when the row has no module for the step to freeze."""
    import brainmagick_b200 as bb
    import brainmagick_b200.functional as BF
    from brainmagick_b200 import synthetic
    B, C, T, F, S, hidden, MC, IL, P = abi_trace.CONFIGS[cfg]
    kw = dict(hidden=dict(meg=hidden), depth=DEPTH, dilation_period=5, kernel_size=3, skip=True, subject_layers=True,
              subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=IL, merger_channels=MC,
              gelu=True, batch_norm=True, merger_pos_dim=P, merger_dropout=0.2, n_subjects=S)
    kw.update(ROWS[row])
    frozen = step[len("frozen_"):] if step.startswith("frozen_") else None
    if frozen and not kw[frozen]:
        return None

    def run():
        torch.manual_seed(0)
        model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, **kw).train(step != "eval")
        if frozen:
            getattr(model, frozen).requires_grad_(False)
        subj = torch.randint(0, S, (B,))
        meg, cand = torch.randn(B, C, T), torch.randn(B, F, T)
        batch = synthetic.make_batch(meg, subj, synthetic.normalised_positions(S, C), subj)
        if step == "eval":
            with torch.no_grad():
                model(dict(meg=meg), batch)
            return
        meg.requires_grad_(step == "meg_grad")
        BF.clip_loss(model(dict(meg=meg), batch), cand, 0).backward()
    return run


def _standalone(module, step):
    """ChannelMerger (merger_channels 12 of 19 sensors) or SubjectLayers (12 -> 10 channels, 3 subjects) on its own."""
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    B, C, T, O, P, S, D = 6, 19, 40, 12, 32, 3, 10

    def run():
        torch.manual_seed(1)
        subj = torch.tensor([0, 2, 1, 2, 0, 1])
        if module == "merger":
            mod = bb.ChannelMerger(O, pos_dim=P, dropout=0.2).train()
            mod.ban_centre_override = torch.tensor([0.4, 0.6])
            x = torch.randn(B, C, T)
            batch = synthetic.make_batch(x, subj, synthetic.normalised_positions(2, C, n_valid=(C, C - 3), seed=3),
                                         torch.tensor([1, 0, 1, 1, 0, 0]))
            fwd = lambda inp: mod(inp, batch)                             # noqa: E731
        else:
            mod = bb.SubjectLayers(O, D, S)
            x = torch.randn(B, O, T)
            fwd = lambda inp: mod(inp, subj)                              # noqa: E731
        mod.requires_grad_(step != "frozen")
        x.requires_grad_(step != "train")
        out = fwd(x)
        out.backward(torch.randn(out.shape))
        with torch.no_grad():
            fwd(x)
    return run


def _record(run, mode):
    import brainmagick_b200.common as CM
    saved, CM._require_cuda_fp32 = CM._require_cuda_fp32, lambda x, who: None   # the recorder's tensors live on the CPU
    try:
        with _mode(mode):
            return abi_trace.record(run)
    finally:
        CM._require_cuda_fp32 = saved


def cases():
    """tag -> run function"""
    out = {}
    for cfg in ("full", "mid", "small"):
        for row in (ROWS if cfg != "small" else ("default",)):
            for step in STEPS:
                run = _simpleconv(cfg, row, step)
                if run is not None:
                    out[f"simpleconv.{cfg}.{row}.{step}"] = run
    for module in ("merger", "subject_layers"):
        for step in ("train", "frozen", "input_grad"):
            out[f"{module}.{step}"] = _standalone(module, step)
    return out


def all_traces():
    traces = {}
    for tag, run in cases().items():
        step = tag.rsplit(".", 1)[1]
        for mode in (MODES if step in MODE_STEPS else MODES[:1]):
            traces[f"{tag}.{mode}"] = _record(run, mode)
    return json.loads(json.dumps(traces))


def test_front_keeps_its_call_stream():
    fixture = json.load(open(FIXTURE))
    want = {tag: [fixture["calls"][i] for i in idx] for tag, idx in fixture["traces"].items()}
    got = all_traces()
    assert set(got) == set(want)
    for tag in want:
        assert got[tag] == want[tag], tag


if __name__ == "__main__":
    calls, traces = {}, {}
    for tag, trace in all_traces().items():
        traces[tag] = [calls.setdefault(json.dumps(c), len(calls)) for c in trace]
    with open(FIXTURE, "w") as f:
        json.dump(dict(calls=[json.loads(c) for c in calls], traces=traces), f, separators=(",", ":"))
        f.write("\n")
