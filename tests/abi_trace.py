"""Records the stream of C-ABI calls (entry point, every scalar argument, NULL-ness of every pointer) that one training /
evaluation step of the drop-in modules issues, WITHOUT a GPU: the ctypes layer is replaced by a recorder and the tensors live
on the CPU (their contents are garbage; only the host-side control flow runs).

Why: which kernels are launched, in which order and with which shapes is decided by host code; the recorder lets CPU tests
assert on that control flow (tests/test_abi_trace.py).
"""
from __future__ import annotations

import json
import os
import sys
from ctypes import c_void_p

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


CONFIGS = {   # B, C, T, F, S, hidden, merger_channels, initial_linear, pos_dim
    "full": (4, 208, 360, 1024, 27, 320, 270, 270, 2048),       # BASELINE widths: every contraction on the tensor cores
    "mid": (8, 40, 130, 128, 3, 160, 48, 24, 128),              # mixed tensor-core / FP32-FMA kernels
    "small": (6, 10, 24, 8, 3, 16, 12, 12, 32),                 # the fixtures' size: FP32-FMA kernels only
}


class _Stream:
    def wait_stream(self, other):
        pass


def record(fn):
    """Runs fn() with the C ABI replaced by a recorder; returns the list of calls."""
    from brainmagick_b200 import _lib
    import brainmagick_b200.convseq as CS
    import brainmagick_b200.functional as BF
    import brainmagick_b200.simpleconv as SC
    trace = []

    def fake_ptr(t):
        if t is None:
            return None
        assert t.is_contiguous(), "non-contiguous tensor handed to the C ABI"
        return c_void_p(t.data_ptr())

    def fake_call(name, *args):
        sig = _lib.SIGNATURES[name]
        assert len(args) == len(sig), f"{name}: {len(args)} arguments for a signature of {len(sig)}"
        for i, (a, kind) in enumerate(zip(args, sig)):
            if kind is _lib.P:
                assert a is None or isinstance(a, c_void_p), f"{name} argument {i}: {type(a)} is not a pointer"
            elif kind is _lib.F:
                assert isinstance(a, float), f"{name} argument {i}: {type(a)} is not a float"
            else:
                assert isinstance(a, int), f"{name} argument {i}: {type(a)} is not an int"
        trace.append([name] + [a if isinstance(a, (int, float)) else (a is not None) for a in args])

    saved = {}
    patches = [(BF, "call", fake_call), (BF, "ptr", fake_ptr), (BF, "stream", lambda: c_void_p(0)),
               (CS, "call", fake_call), (CS, "ptr", fake_ptr), (CS, "stream", lambda: c_void_p(0)),
               (BF, "OVERLAP_WGRAD", False), (SC, "_require_cuda", lambda meg: None),
               (torch.cuda, "current_stream", lambda *a, **k: _Stream())]
    for mod, name, val in patches:
        saved[(mod, name)] = getattr(mod, name)
        setattr(mod, name, val)
    BF._status.setdefault(torch.device("cpu"), torch.zeros(1, dtype=torch.int32))
    BF._clip_ws.clear()                       # the workspace cache only ever grows: start every recording from empty
    try:
        fn()
    finally:
        BF._clip_ws.clear()
        for (mod, name), val in saved.items():
            setattr(mod, name, val)
        BF._status.pop(torch.device("cpu"), None)
    return trace


def simpleconv_step(cfg, train: bool, **overrides):
    import brainmagick_b200 as bb
    import brainmagick_b200.functional as BF
    from brainmagick_b200 import synthetic
    B, C, T, F, S, hidden, MC, IL, P = cfg
    kw = dict(hidden=dict(meg=hidden), depth=10, dilation_period=5, kernel_size=3, skip=True, subject_layers=True,
              subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=IL, merger_channels=MC,
              gelu=True, batch_norm=True, merger_pos_dim=P, merger_dropout=0.2, n_subjects=S)
    kw.update(overrides)

    def run():
        torch.manual_seed(0)
        model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, **kw).train(train)
        subj = torch.randint(0, S, (B,))
        meg, cand = torch.randn(B, C, T), torch.randn(B, F, T)
        batch = synthetic.make_batch(meg, subj, synthetic.normalised_positions(S, C), subj)
        if train:
            BF.clip_loss(model(dict(meg=meg), batch), cand, 0).backward()
        else:
            with torch.no_grad():
                model(dict(meg=meg), batch)
    return record(run)


def all_traces():
    return {f"{tag}.{'train' if train else 'eval'}": simpleconv_step(cfg, train)
            for tag, cfg in CONFIGS.items() for train in (True, False)}


