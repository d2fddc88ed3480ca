"""SimpleConv's output head (`final`: 1x1 conv -> activation -> 1x1 ConvTranspose, or the bare transpose when
complex_out=False), without a GPU.

`tests/golden/abi_trace_head.json` holds the full C-ABI call stream (tests/abi_trace.py: entry point, every scalar
argument, NULL-ness of every pointer) of the steps below, stored like abi_trace_front.json as a table of the distinct calls
("calls") and, per step, the indices of its calls in order ("traces").  It was recorded with `python tests/test_head_cpu.py`
at the commit before the head's forms came to be written once (`functional.head_forward` / `head_backward`), so the test
pins that the shared head issues exactly the calls the inline head issued.  The cases cover:
  * the `full`, `mid` and `small` sizes of abi_trace.CONFIGS (tensor-core convs with tensor-core weight gradients,
    tensor-core convs with `bm_head_bwd_params`, the FP32-FMA `bm_head_fwd` / `bm_head_bwd`), and `full` with 120 output
    channels (bench.py's cfg4: the FP32-FMA head at the tensor-core hidden width).  Depth 2 instead of 10: the conv stack
    and the front are pinned by their own fixtures;
  * the rows default, gelu=False (conv -> activation kernel -> conv -> transpose) and complex_out=False (no head);
  * a training step with everything trainable, with only `final` trainable, with `final` frozen, with each of `final`'s
    four tensors frozen alone, an attribution step (eval mode, every parameter frozen, meg requiring grad), and an
    eval-mode `torch.no_grad()` forward;
  * the default flags for all of these, and torch.use_deterministic_algorithms(True) and TF32 matmul precision for the
    trainable, head-only and attribution steps.

The recorder runs the weight gradients inline.  `test_side_stream_is_joined_before_the_backward_returns` runs the `full`
steps with the side stream on, against fake streams, and checks that every weight-gradient kernel queued there is joined
back into the main stream before the encoder's backward returns.
"""
import contextlib
import json
import os

import pytest
import torch

import abi_trace
from test_front_cpu import _record
from test_frozen_cpu import PATTERNS, _trainable

FIXTURE = os.path.join(abi_trace.ROOT, "tests", "golden", "abi_trace_head.json")

SIZES = {"full": abi_trace.CONFIGS["full"], "mid": abi_trace.CONFIGS["mid"], "small": abi_trace.CONFIGS["small"],
         "full_f120": abi_trace.CONFIGS["full"][:3] + (120,) + abi_trace.CONFIGS["full"][4:]}
ROWS = {"default": {}, "no_gelu": dict(gelu=False), "bare_last": dict(complex_out=False)}
HEAD = ("final.0.weight", "final.0.bias", "final.2.weight", "final.2.bias")
STEPS = ("train", "head_only", "frozen_final") + tuple(f"frozen_{n}" for n in HEAD) + ("attribution", "eval")
MODES = ("default", "deterministic", "tf32")
MODE_STEPS = ("train", "head_only", "attribution")   # the steps also recorded under the deterministic and TF32 modes
DEPTH = 2


def _build(size, row, train):
    import brainmagick_b200 as bb
    B, C, T, F, S, hidden, MC, IL, P = SIZES[size]
    kw = dict(hidden=dict(meg=hidden), depth=DEPTH, dilation_period=5, kernel_size=3, skip=True, subject_layers=True,
              subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=IL, merger_channels=MC,
              gelu=True, batch_norm=True, merger_pos_dim=P, merger_dropout=0.2, n_subjects=S)
    kw.update(ROWS[row])
    torch.manual_seed(0)
    return bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, **kw).train(train)


def _run(size, row, trainable):
    """-> the run function of one step: `trainable(model) -> {name: requires_grad}`, meg requiring grad when every
    parameter is frozen (attribution, in eval mode); trainable None: an eval-mode `torch.no_grad()` forward."""
    import brainmagick_b200.functional as BF
    from brainmagick_b200 import synthetic
    B, C, T, F, S = SIZES[size][:5]

    def run():
        model = _build(size, row, trainable is not None and trainable != "attribution")
        if trainable == "attribution":
            model.requires_grad_(False)
        elif trainable is not None:
            want = trainable(model)
            for name, p in model.named_parameters():
                p.requires_grad_(want[name])
        subj = torch.randint(0, S, (B,))
        meg, cand = torch.randn(B, C, T), torch.randn(B, F, T)
        batch = synthetic.make_batch(meg, subj, synthetic.normalised_positions(S, C), subj)
        if trainable is None:
            with torch.no_grad():
                model(dict(meg=meg), batch)
            return
        meg.requires_grad_(trainable == "attribution")
        BF.clip_loss(model(dict(meg=meg), batch), cand, 0).backward()
    return run


def _step(size, row, step):
    """-> the step's run function, or None when the row has no head for the step to freeze."""
    if step == "eval":
        return _run(size, row, None)
    if step == "attribution":
        return _run(size, row, "attribution")
    if row == "bare_last" and step != "train":
        return None
    if step == "train":
        return _run(size, row, lambda model: {n: True for n, _ in model.named_parameters()})
    if step == "head_only":
        return _run(size, row, lambda model: {n: n.startswith("final.") for n, _ in model.named_parameters()})
    if step == "frozen_final":
        return _run(size, row, lambda model: {n: not n.startswith("final.") for n, _ in model.named_parameters()})
    frozen = step[len("frozen_"):]
    return _run(size, row, lambda model: {n: n != frozen for n, _ in model.named_parameters()})


def all_traces():
    traces = {}
    for size in SIZES:
        for row in ROWS:
            for step in STEPS:
                run = _step(size, row, step)
                if run is None:
                    continue
                for mode in (MODES if step in MODE_STEPS else MODES[:1]):
                    traces[f"{size}.{row}.{step}.{mode}"] = _record(run, mode)
    return json.loads(json.dumps(traces))


def test_head_keeps_its_call_stream():
    fixture = json.load(open(FIXTURE))
    want = {tag: [fixture["calls"][i] for i in idx] for tag, idx in fixture["traces"].items()}
    got = all_traces()
    assert set(got) == set(want)
    for tag in want:
        assert got[tag] == want[tag], tag


class _FakeStream:
    def __init__(self, name, events):
        self.name, self.events = name, events

    def wait_stream(self, other):
        self.events.append(("wait", self.name, other.name))


@pytest.mark.parametrize("pattern", ["all"] + PATTERNS)
def test_side_stream_is_joined_before_the_backward_returns(pattern, monkeypatch):
    """With the weight gradients on the side stream: every run of side-stream calls waits on the main stream's work
    queued before it, and when anything ran there, the main stream waits on the side stream once, after its last call and
    before the encoder's backward returns (so the gradients and the operands the side kernels read are safe to use and to
    free when `backward()` returns)."""
    import brainmagick_b200.functional as BF
    events, current = [], ["main"]
    streams = {name: _FakeStream(name, events) for name in ("main", "side")}

    @contextlib.contextmanager
    def on_stream(s):
        current.append(s.name)
        try:
            yield
        finally:
            current.pop()

    backward = BF._EncoderFn.backward

    def logged_backward(ctx, *grads):
        out = backward(ctx, *grads)
        events.append(("return",))
        return out

    monkeypatch.setattr(torch.cuda, "stream", on_stream)
    monkeypatch.setattr(torch.Tensor, "record_stream", lambda self, s: None)
    monkeypatch.setattr(BF, "_side_stream", lambda device: streams["side"])
    monkeypatch.setattr(BF._EncoderFn, "backward", staticmethod(logged_backward))
    trainable = "attribution" if pattern == "attribution" else \
        (lambda model: _trainable(model, pattern) if pattern != "all" else {n: True for n, _ in model.named_parameters()})
    run = _run("full", "default", trainable)

    def with_side_stream():
        # abi_trace.record restores these three after the run
        BF.OVERLAP_WGRAD = True
        torch.cuda.current_stream = lambda *a, **k: streams[current[-1]]
        call = BF.call
        BF.call = lambda name, *args: (events.append(("call", name, current[-1])), call(name, *args))[1]
        run()

    _record(with_side_stream, "default")
    side_calls = [i for i, e in enumerate(events) if e[0] == "call" and e[2] == "side"]
    joins = [i for i, e in enumerate(events) if e == ("wait", "main", "side")]
    returned = events.index(("return",))
    if pattern in ("all", "head", "bn", "glu"):            # a tensor-core weight gradient to overlap
        assert side_calls
    for i in side_calls:
        last_main = max(j for j in range(i) if events[j][0] == "call" and events[j][2] == "main")
        assert ("wait", "side", "main") in events[last_main:i], events[i]
    if side_calls:
        assert len(joins) == 1 and side_calls[-1] < joins[0] < returned, (side_calls[-1], joins, returned)
    else:
        assert not joins


if __name__ == "__main__":
    calls, traces = {}, {}
    for tag, trace in all_traces().items():
        traces[tag] = [calls.setdefault(json.dumps(c), len(calls)) for c in trace]
    with open(FIXTURE, "w") as f:
        json.dump(dict(calls=[json.loads(c) for c in calls], traces=traces), f, separators=(",", ":"))
        f.write("\n")
