"""TEST INFRASTRUCTURE ONLY -- the torch-CPU emulation of the channel join / split entry points of include/bm_b200.h
(`bm_channel_join`, `bm_channel_split`) as an extension of `tests/input_grad_emulator.py`, with the conventions of
`tests/abi_emulator.py`: each entry point's documented contract restated with torch ops on the buffers the host code
passes, interpreted through the integer arguments only.

A channel-major stream that is a view cropped in time reaches the C ABI through `functional._view_ptr`; `emulated()` and
`record()` replace it too (by the smallest flat view that spans the stream's elements, or a recorded pointer).
"""
from __future__ import annotations

import contextlib
from ctypes import c_void_p

import torch

import abi_trace
import input_grad_emulator
from abi_emulator import _v
from input_grad_emulator import InputGradEmulator


def _cm(p, B, C, T, ld):
    return p.as_strided((B, C, T), (C * ld, ld, 1))


class EncodeEmulator(InputGradEmulator):
    def bm_channel_join(self, B, T, Cp, n, *rest):
        dst = rest[20]
        out = torch.zeros(B, T, Cp)
        for i in range(n):
            p, C, ld, cm, col = rest[5 * i:5 * i + 5]
            out[:, :, col:col + C] = _cm(p, B, C, T, ld).transpose(1, 2) if cm else _v(p, B * T, ld)[:, :C].reshape(B, T, C)
        _v(dst, B, T, Cp).copy_(out)

    def bm_channel_split(self, src, B, T, Cp, n, *rest):
        g = _v(src, B, T, Cp)
        for i in range(n):
            p, C, ld, cm, col = rest[5 * i:5 * i + 5]
            if p is None:
                continue
            part = g[:, :, col:col + C]
            if cm:
                _cm(p, B, C, T, ld).copy_(part.transpose(1, 2))
            else:
                _v(p, B * T, ld)[:, :C].copy_(part.reshape(B * T, C))


def _span(t):
    """the smallest flat view of t's storage from its first element to its last"""
    n = 1 + sum((s - 1) * st for s, st in zip(t.shape, t.stride()))
    return t.as_strided((n,), (1,))


@contextlib.contextmanager
def _patched_view_ptr(fn):
    import brainmagick_b200.functional as BF
    saved = BF._view_ptr
    BF._view_ptr = fn
    try:
        yield
    finally:
        BF._view_ptr = saved


@contextlib.contextmanager
def emulated():
    """input_grad_emulator.emulated() with the channel join / split entry points."""
    with input_grad_emulator.emulated(EncodeEmulator) as emu, _patched_view_ptr(_span):
        yield emu


def record(fn):
    """abi_trace.record(fn) with the view pointer of a cropped stream recorded like any other pointer."""
    with _patched_view_ptr(lambda t: c_void_p(t.data_ptr())):
        return abi_trace.record(fn)
