"""TEST INFRASTRUCTURE ONLY -- the torch-CPU emulation of `bm_check_all_true` (include/bm_b200.h), ClipLoss's mask check
on the device while a step is captured in a CUDA graph, with the conventions of `tests/abi_emulator.py`.  `CheckAllTrue` is
a mixin: put it first in the bases of the emulator class a test runs on.
"""
from __future__ import annotations

from abi_emulator import _v


class CheckAllTrue:
    def bm_check_all_true(self, mask, n, code, status, stream):
        assert code != 0
        if n and not bool(_v(mask, n).all()) and int(_v(status, 1)[0]) == 0:
            _v(status, 1)[0] = code
