"""TEST INFRASTRUCTURE ONLY -- the torch-CPU emulation of the deterministic (`_det`) entry points of include/bm_b200.h, as an
extension of `tests/input_grad_emulator.py` with the same conventions.

Each `_det` entry point's documented contract is its default form's (only the order of its floating-point reductions
differs, which the CPU restatement does not model), so every method here forwards to the default form's emulation after
dropping the workspace arguments.  The emulator also records the names of the entry points it ran (`calls`), so that a test
can assert which form the host code chose.
"""
from __future__ import annotations

import contextlib

import input_grad_emulator
from input_grad_emulator import InputGradEmulator

# _det entry point -> (default form, True when the det form appends (workspace, workspace_floats) before the stream)
DET_FORMS = {
    "bm_bn_gelu_skip_bwd_det": ("bm_bn_gelu_skip_bwd", True),
    "bm_bn_act_skip_bwd_det": ("bm_bn_act_skip_bwd", True),
    "bm_glu_bwd_det": ("bm_glu_bwd", True),
    "bm_conv1d_bwd_weight_det": ("bm_conv1d_bwd_weight", True),
    "bm_initial_linear_bwd_det": ("bm_initial_linear_bwd", True),
    "bm_sensor_chain_bwd_det": ("bm_sensor_chain_bwd", True),
    "bm_head_bwd_params_det": ("bm_head_bwd_params", True),
    "bm_head_bwd_det": ("bm_head_bwd", True),
    "bm_attention_weights_bwd_det": ("bm_attention_weights_bwd", False),
    "bm_candidate_inv_norms_det": ("bm_candidate_inv_norms", False),
    "bm_clip_scores_det": ("bm_clip_scores", False),
    "bm_clip_loss_fwd_det": ("bm_clip_loss_fwd", False),
}


def _forward(base: str, drops_workspace: bool):
    def fn(self, *args):
        if drops_workspace:
            args = args[:-3] + args[-1:]
        self._inner(base, *args)
    return fn


class DeterministicEmulator(InputGradEmulator):
    def __init__(self):
        super().__init__()
        self.calls = []
        self._depth = 0

    def __getattribute__(self, name):
        if name.startswith("bm_") and object.__getattribute__(self, "_depth") == 0:
            object.__getattribute__(self, "calls").append(name)       # entry points the host code called, not their parts
        return object.__getattribute__(self, name)

    def _inner(self, name, *args):
        self._depth += 1
        try:
            getattr(self, name)(*args)
        finally:
            self._depth -= 1

    # the two column reductions take the workspace in the middle of their arguments
    def bm_col_stats_det(self, y, rows, C, ws, ws_floats, stats, stream):
        self._inner("bm_col_stats", y, rows, C, stats, stream)

    def bm_col_sum_det(self, x, rows, C, ws, ws_floats, out, stream):
        self._inner("bm_col_sum", x, rows, C, out, stream)


for _name, (_base, _drops) in DET_FORMS.items():
    setattr(DeterministicEmulator, _name, _forward(_base, _drops))


@contextlib.contextmanager
def emulated(emulator_class=DeterministicEmulator):
    with input_grad_emulator.emulated(emulator_class) as emu:
        yield emu
