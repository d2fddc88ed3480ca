"""The stand-alone ConvSequence (and DeepMel) call stream, without a GPU.

`tests/golden/abi_trace_convseq.json` holds the full C-ABI call stream (tests/abi_trace.py: entry point, every scalar
argument, NULL-ness of every pointer) of ConvSequence / DeepMel steps.  It was recorded with `python
tests/test_conv_stack_cpu.py` at the commit before ConvSequence and SimpleConv came to share one conv stack
(`functional.conv_stack_forward` / `conv_stack_backward`), so the test pins that the shared stack issues exactly the calls
the stand-alone ConvSequence loop issued.  The cases cover:
  * the DEEPMEL_CASES fixture sizes (FP32-FMA kernels), two DeepMel widths that pass the tensor-core gates (LeakyReLU and
    GELU) and a ConvSequence with a residual on its first layer, BatchNorm + ReLU on every layer and no GLU;
  * a training and an evaluation step, each a ClipLoss forward / backward followed by a `torch.no_grad()` forward;
  * everything trainable (the input too), a frozen first layer, and frozen GLU blocks;
  * the default flags, torch.use_deterministic_algorithms(True), and TF32 matmul precision.
"""
import contextlib
import json
import os

import torch

import abi_trace

FIXTURE = os.path.join(abi_trace.ROOT, "tests", "golden", "abi_trace_convseq.json")

_LAYER = dict(kernel=3, stride=1, dilation_growth=2, dilation_period=5, batch_norm=True, activation_on_last=False, skip=True,
              glu_context=1, glu=2)
MODELS = {   # name -> (constructor kwargs, B, T); "deepmel_*" come from oracle.make_golden.DEEPMEL_CASES
    "tc_lrelu": (dict(n_in_channels=40, n_hidden_channels=160, n_hidden_layers=4, n_out_channels=320, **_LAYER), 2, 72),
    "tc_gelu": (dict(n_in_channels=64, n_hidden_channels=256, n_hidden_layers=3, n_out_channels=256, activation="gelu",
                     **_LAYER), 2, 130),
    "convseq_relu": (dict(channels=[16, 16, 24], kernel=3, stride=1, batch_norm=True, skip=True, activation="relu"), 3, 20),
}
MODES = ("default", "deterministic", "tf32")
FREEZE = ("all", "first", "glu")


def _models():
    from oracle.make_golden import DEEPMEL_CASES
    out = {name: (dict(n_in_channels=c["n_in"], **c["params"]), c["B"], c["T"]) for name, c in DEEPMEL_CASES.items()}
    out.update(MODELS)
    return out


def _build(kw):
    import brainmagick_b200 as bb
    kw = dict(kw)
    act = kw.pop("activation", None)
    if act is not None:
        kw["activation"] = {"gelu": torch.nn.GELU, "relu": torch.nn.ReLU}[act]
    if "channels" in kw:
        return bb.ConvSequence(kw.pop("channels"), **kw)
    return bb.DeepMel(**kw)


@contextlib.contextmanager
def _mode(mode):
    det, det_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    prec = torch.get_float32_matmul_precision()
    try:
        torch.use_deterministic_algorithms(mode == "deterministic")
        torch.set_float32_matmul_precision("high" if mode == "tf32" else "highest")
        yield
    finally:
        torch.use_deterministic_algorithms(det, warn_only=det_warn)
        torch.set_float32_matmul_precision(prec)


def _step(kw, B, T, train, freeze, mode):
    import brainmagick_b200 as bb
    import brainmagick_b200.convseq as CS

    def run():
        torch.manual_seed(0)
        model = _build(kw).train(train)
        if freeze == "first":
            model.sequence[0].requires_grad_(False)
        elif freeze == "glu":
            model.glus.requires_grad_(False)
        c_in = model.sequence[0][0].in_channels
        mel = torch.randn(B, c_in, T).requires_grad_(freeze == "all")
        out = model(mel)
        est = torch.randn(out.shape).requires_grad_(True)
        bb.ClipLoss()(est, out, torch.ones(B, 1, T, dtype=torch.bool)).backward()
        with torch.no_grad():
            model(mel)

    saved, CS._require_cuda = CS._require_cuda, lambda x: None      # the recorder's tensors live on the CPU
    try:
        with _mode(mode):
            return abi_trace.record(run)
    finally:
        CS._require_cuda = saved


def all_traces():
    traces = {}
    for name, (kw, B, T) in _models().items():
        has_glu = kw.get("glu", 0) > 0
        for mode in MODES:
            for train in (True, False):
                for freeze in FREEZE:
                    if freeze == "glu" and not has_glu:
                        continue
                    tag = f"{name}.{mode}.{'train' if train else 'eval'}.{freeze}"
                    traces[tag] = _step(kw, B, T, train, freeze, mode)
    return json.loads(json.dumps(traces))


def test_conv_sequence_steps_keep_their_call_stream():
    want = json.load(open(FIXTURE))
    got = all_traces()
    assert set(got) == set(want)
    for tag in want:
        assert got[tag] == want[tag], tag


if __name__ == "__main__":
    with open(FIXTURE, "w") as f:
        json.dump(all_traces(), f, separators=(",", ":"))
        f.write("\n")
