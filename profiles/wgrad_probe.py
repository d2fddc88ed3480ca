"""How does the all-taps weight-gradient kernel behave?  Three launch patterns at the K3 shape (B=256, T=360, 320x320, k3 d4):
isolated launches after an L2 flush, back-to-back launches on the same operands, back-to-back over rotating operand sets
(> L2), each with the kernel's cycle counters (bm_set_debug_buffer).   python profiles/wgrad_probe.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from brainmagick_b200 import _lib  # noqa: E402
from brainmagick_b200._lib import call, ptr, stream  # noqa: E402

dev = "cuda"
B, T, Kw = 256, 360, 3
lib = _lib.load()
status = torch.zeros(1, dtype=torch.int32, device=dev)
flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
for M, N, dil in ((320, 320, 4), (640, 320, 1)):
    xs = [torch.randn(B, T, N, device=dev) for _ in range(3)]
    dys = [torch.randn(B, T, M, device=dev) for _ in range(3)]
    dw = torch.empty(M, N, Kw, device=dev)
    ws = torch.empty(int(lib.bm_tc_wgrad_conv_workspace(B, T, M, N, Kw)), device=dev)
    dbg = torch.zeros(8 * 148, device=dev, dtype=torch.int64)

    def launch(i):
        call("bm_tc_wgrad_conv", ptr(dys[i]), ptr(xs[i]), B, T, M, N, N, Kw, dil, ptr(ws), ptr(dw), ptr(status), stream())

    def counters():
        d = dbg.reshape(148, 8).double()
        lead = d[0::2]
        return "MMA waits %.0f of %.0f cycles; A conv: split(+wait X) %.0f, wait slot %.0f, st %.0f; B conv: wait TMA %.0f" % (
            lead[:, 0].mean(), lead[:, 1].mean(), lead[:, 2].mean(), lead[:, 3].mean(), lead[:, 4].mean(), lead[:, 5].mean())

    for mode in ("isolated+flush", "back-to-back same", "back-to-back rotating"):
        for use_dbg in (False, True):
            call("bm_set_debug_buffer", ptr(dbg) if use_dbg else None)
            for i in range(3):
                launch(i % 3)
            torch.cuda.synchronize()
            if mode == "isolated+flush":
                ts = []
                for i in range(10):
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(); launch(0); e1.record()
                    torch.cuda.synchronize()
                    ts.append(e0.elapsed_time(e1))
                ms = sum(ts) / len(ts)
            else:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(24):
                    launch(i % 3 if mode.endswith("rotating") else 0)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / 24
            tf = 2.0 * M * N * Kw * T * B / (ms * 1e-3) / 1e12
            print(f"[wgrad_pp {M}x{N} d{dil}] {mode:24s} dbg={int(use_dbg)} {ms:.4f} ms = {tf:.1f} TF" +
                  ("   " + counters() if use_dbg else ""))
    call("bm_set_debug_buffer", None)
assert int(status.item()) == 0
