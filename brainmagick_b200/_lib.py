"""ctypes binding of libbm_b200.so (include/bm_b200.h).  There is no fallback: if the CUDA library is missing
or a call fails, this raises."""
from __future__ import annotations

import contextlib
import ctypes
import os
import threading
from ctypes import c_double, c_float, c_int, c_longlong, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbm_b200.so")

P, I, L, F, D = c_void_p, c_int, c_longlong, c_float, c_double

# name -> argtypes, in the order of include/bm_b200.h
SIGNATURES = {
    "bm_attention_weights_fwd": [P, P, P, P, F, I, I, I, I, P, P, P],
    "bm_attention_weights_bwd": [P, P, P, I, I, I, I, P, P, P],
    "bm_fourier_emb": [P, P, I, I, I, P, P],
    "bm_masked_softmax": [P, P, P, F, I, I, I, P],
    "bm_softmax_bwd": [P, P, L, I, P, P],
    "bm_sensor_chain_fwd": [P, P, P, P, P, P, P, I, I, I, I, I, I, I, P, P, P, P],
    "bm_sensor_chain_bwd": [P, P, P, P, P, P, P, P, P, P, P, I, I, I, I, I, I, I, I, I, P, P, P, P, P, P, P],
    "bm_sensor_mix_fwd": [P, P, P, I, I, I, I, I, P, P],
    "bm_initial_linear_fwd": [P, I, P, P, I, I, I, I, I, P, P],
    "bm_subject_layers_fwd": [P, I, P, P, I, I, I, I, I, P, P],
    "bm_subject_layers_bwd": [P, I, P, I, P, P, P, P, I, I, I, I, I, I, P, P, P],
    "bm_initial_linear_bwd": [P, I, P, I, P, I, I, I, I, I, P, P, P, P],
    "bm_sensor_mix_bwd": [P, I, P, P, P, I, I, I, I, I, P, P],
    "bm_sensor_mix_bwd_data": [P, I, P, P, P, I, I, I, I, P, P],
    "bm_conv_weight_prep": [P, I, I, I, P, P, P],
    "bm_conv1d_fwd": [P, P, P, I, I, I, I, I, I, P, P, P],
    "bm_bn_stats_finalize": [P, L, F, F, P, P, P, P, I, P],
    "bm_bn_stats_finalize_counted": [P, F, F, P, P, P, P, I, P],
    "bm_bn_stats_finalize_cumulative": [P, L, F, P, P, P, P, P, I, P],
    "bm_bn_stats_finalize_counted_cumulative": [P, F, P, P, P, P, P, I, P],
    "bm_bn_eval_stats": [P, P, F, P, P, I, P],
    "bm_bn_gelu_skip_fwd": [P, P, P, P, P, P, P, L, I, P, P],
    "bm_bn_gelu_skip_bwd": [P, P, P, P, P, P, I, L, I, P, P, P, P, P, P],
    "bm_bn_gelu_skip_bwd_reduce": [P, P, P, P, P, P, L, I, P, P, P, P],
    "bm_bn_gelu_skip_bwd_apply": [P, P, P, P, P, P, L, I, P, P, P],
    "bm_conv1d_bwd_data": [P, P, P, I, I, I, I, I, I, P, P],
    "bm_conv1d_bwd_weight": [P, P, I, I, I, I, I, I, P, P, P],
    "bm_conv1d_glu_fwd": [P, P, P, I, I, I, I, I, P, P, P],
    "bm_glu_bwd": [P, P, L, I, P, P, P, P],
    "bm_head_fwd": [P, P, P, P, P, I, I, I, I, P, P, P, P],
    "bm_head_bwd": [P, P, P, P, P, P, I, I, I, I, P, P, P, P, P, P, P],
    "bm_head_bwd_params": [P, P, P, P, I, I, I, I, P, P, P, P, P, P],
    "bm_clip_scores": [P, P, I, I, L, I, P, P, P, P, L, P, P],
    "bm_clip_loss_fwd": [P, P, I, I, L, I, P, P, P, P, P, P, L, P, P],
    "bm_clip_loss_bwd": [P, P, P, P, I, I, L, I, P, P, P, P],
    "bm_clip_loss_fwd_pooled": [P, P, I, P, P, I, I, L, I, P, P, P, P, P, P, L, P, P],
    "bm_clip_loss_bwd_pooled": [P, P, P, I, P, P, P, I, I, L, I, P, P, P, P],
    "bm_set_debug_flags": [I],
    "bm_set_debug_buffer": [P],
    "bm_tc_conv_supported": [I, I, I, I, I],
    "bm_tc_weight_split": [P, I, I, I, P, P, P, P, P],
    "bm_tc_conv1d": [P, P, P, P, P, I, I, I, I, I, I, I, I, I, I, P, P, P, P, P, P],
    "bm_tc_conv1d_persistent_supported": [I, I, I, I, I],
    "bm_tc_conv1d_persistent": [P, P, P, I, I, I, I, I, I, I, I, I, I, I, P, P, P, P, P, P],
    "bm_amax": [P, L, P, P],
    "bm_f16_split": [P, L, P, P, P, P],
    "bm_tc_weight_split_f16": [P, P, I, I, I, P, P, P, P, P],
    "bm_tc_conv1d_f16": [P, P, P, P, P, P, I, I, I, I, I, I, I, I, I, I, I, P, P, P, P, P, P, P],
    "bm_col_stats": [P, L, I, P, P],
    "bm_channel_mask": [P, P, I, I, I, P, P],
    "bm_transpose_nt": [P, I, I, I, P, P],
    "bm_transpose_nt_ld": [P, I, I, I, I, P, P],
    "bm_channel_join": [I, I, I, I] + [P, I, I, I, I] * 4 + [P, P],
    "bm_channel_split": [P, I, I, I, I] + [P, I, I, I, I] * 4 + [P],
    "bm_check_all_true": [P, L, I, P, P],
    "bm_masked_loss_workspace": [I, I, I],         # returns long long floats, like the `_det_workspace` queries
    "bm_masked_loss_fwd": [I, P, L, L, P, L, L, P, L, L, L, I, I, I, P, L, P, P, P],
    "bm_masked_loss_bwd": [I, P, P, P, L, L, P, L, L, P, L, L, L, I, I, I, P, P, P],
    "bm_decoding_loss_workspace": [I, I, I],
    "bm_decoding_loss_fwd": [P, L, L, P, L, L, P, L, L, L, I, I, P, I, P, P, P, L, P, P, P, P, P],
    "bm_decoding_loss_bwd": [P, P, P, P, L, L, P, L, L, P, L, L, L, I, I, I, I, P, I, P, P, P, P],
    "bm_metric_workspace": [I, I, I],
    "bm_metric_update": [I, I, P, L, L, L, P, L, L, L, P, L, L, L, I, I, I, I, I, P, P, I, P, L, P],
    "bm_metric_finalize": [I, P, I, I, D, P, I, P, P],
    "bm_svd_table": [I, P, P, P, P, I, I, P, P],
    "bm_svd_penalty_fwd": [P, I, I, I, L, L, P, P, P, D, P, P],
    "bm_svd_penalty_bwd": [P, I, I, I, L, L, L, P, P, P, P, D, P, P],
    "bm_tc_wgrad_supported": [I, I],
    "bm_tc_wgrad": [P, P, I, I, I, I, I, I, I, P, P, P, P, P],
    "bm_tc_wgrad_conv_supported": [I, I, I, I],
    "bm_tc_wgrad_conv": [P, P, I, I, I, I, I, I, I, P, P, P, P],
    "bm_tc_wgrad_conv_f16": [P, P, P, P, I, I, I, I, I, I, I, P, P, P, P],
    "bm_col_sum": [P, L, I, P, P],
    "bm_tc_pointwise_sel": [P, P, P, P, I, I, I, I, I, P, P, P],
    "bm_tc_wgrad_grouped": [P, P, P, P, I, I, I, I, I, P, P, P],
    "bm_tc_sensor_mix_bwd_data": [P, P, P, P, I, P, I, I, I, I, I, P, P, P],
    "bm_gelu_bwd": [P, P, L, P, P],
    "bm_candidate_inv_norms": [P, I, L, P, P, P],
    "bm_retrieval_topk": [P, L, I, I, P, I, I, I, P, P, P, P, P, P, P, P, P, P],
    "bm_retrieval_probs": [P, L, I, I, P, P],
    "bm_retrieval_vocab_probs": [P, L, I, P, P, P, P, P, I, P, P, P],
    "bm_rowdot_scaled": [P, P, I, L, P, P],
    "bm_scale_clamp_crop": [P, P, P, P, I, I, I, I, I, F, I, I, P, P, P],
    "bm_reject_compact": [P, P, L, F, I, P, P, P, P],
    "bm_gather_rows": [P, P, I, L, P, P],
    "bm_scatter_rows": [P, P, I, L, P, P],
    "bm_bn_act_skip_fwd": [P, P, P, P, P, P, P, L, I, I, F, P],
    "bm_bn_act_skip_bwd": [P, P, P, P, P, P, I, L, I, I, F, P, P, P, P, P],
    "bm_bn_act_skip_bwd_reduce": [P, P, P, P, P, P, L, I, I, F, P, P, P, P],
    "bm_bn_act_skip_bwd_apply": [P, P, P, P, P, P, L, I, I, F, P, P, P],
    "bm_bn_act_gain_skip_fwd": [P, P, P, P, P, P, P, L, I, I, F, P, F, P, P],
    "bm_bn_act_gain_skip_bwd": [P, P, P, P, P, P, I, L, I, I, F, P, F, P, P, P, P, P, P, P, P],
    "bm_clip_loss_bwd_cand": [P, P, P, P, P, P, I, I, L, I, P, P, P, P, P],
    "bm_clip_scores_bwd": [P, P, P, P, P, I, I, L, P, P, P, P, P, P],
    # deterministic forms (deterministic() below) and their workspace size queries (which return long long floats)
    "bm_col_stats_det_workspace": [L, I],
    "bm_col_stats_det": [P, L, I, P, L, P, P],
    "bm_col_sum_det_workspace": [L, I],
    "bm_col_sum_det": [P, L, I, P, L, P, P],
    "bm_bn_gelu_skip_bwd_det_workspace": [L, I],
    "bm_bn_gelu_skip_bwd_det": [P, P, P, P, P, P, I, L, I, P, P, P, P, P, P, L, P],
    "bm_bn_act_skip_bwd_det_workspace": [L, I],
    "bm_bn_act_skip_bwd_det": [P, P, P, P, P, P, I, L, I, I, F, P, P, P, P, P, L, P],
    "bm_bn_gelu_skip_bwd_reduce_det_workspace": [L, I],
    "bm_bn_gelu_skip_bwd_reduce_det": [P, P, P, P, P, P, L, I, P, P, P, P, L, P],
    "bm_bn_act_skip_bwd_reduce_det_workspace": [L, I],
    "bm_bn_act_skip_bwd_reduce_det": [P, P, P, P, P, P, L, I, I, F, P, P, P, P, L, P],
    "bm_bn_act_gain_skip_bwd_det_workspace": [L, I],
    "bm_bn_act_gain_skip_bwd_det": [P, P, P, P, P, P, I, L, I, I, F, P, F, P, P, P, P, P, P, P, P, L, P],
    "bm_glu_bwd_det_workspace": [L, I],
    "bm_glu_bwd_det": [P, P, L, I, P, P, P, P, L, P],
    "bm_conv1d_bwd_weight_det_workspace": [I, I, I, I, I],
    "bm_conv1d_bwd_weight_det": [P, P, I, I, I, I, I, I, P, P, P, L, P],
    "bm_initial_linear_bwd_det_workspace": [I, I, I, I],
    "bm_initial_linear_bwd_det": [P, I, P, I, P, I, I, I, I, I, P, P, P, P, L, P],
    "bm_sensor_chain_bwd_det_workspace": [I, I, I, I],
    "bm_sensor_chain_bwd_det": [P, P, P, P, P, P, P, P, P, P, P, I, I, I, I, I, I, I, I, I, P, P, P, P, P, P, P, L, P],
    "bm_attention_weights_bwd_det": [P, P, P, I, I, I, I, P, P, P],
    "bm_head_bwd_params_det_workspace": [I, I, I, I],
    "bm_head_bwd_params_det": [P, P, P, P, I, I, I, I, P, P, P, P, P, P, L, P],
    "bm_head_bwd_det_workspace": [I, I, I, I],
    "bm_head_bwd_det": [P, P, P, P, P, P, I, I, I, I, P, P, P, P, P, P, P, L, P],
    "bm_candidate_inv_norms_det": [P, I, L, P, P, P],
    "bm_clip_scores_det": [P, P, I, I, L, I, P, P, P, P, L, P, P],
    "bm_clip_loss_fwd_det": [P, P, I, I, L, I, P, P, P, P, P, P, L, P, P],
    "bm_clip_loss_fwd_pooled_det": [P, P, I, P, P, I, I, L, I, P, P, P, P, P, P, L, P, P],
}
# single-pass TF32 forms (tf32() below): the default form's arguments
TF32_FORMS = ("bm_tc_conv1d", "bm_tc_conv1d_persistent", "bm_tc_pointwise_sel", "bm_tc_sensor_mix_bwd_data", "bm_tc_wgrad",
              "bm_tc_wgrad_conv", "bm_tc_wgrad_grouped", "bm_clip_scores", "bm_clip_scores_det", "bm_clip_loss_fwd",
              "bm_clip_loss_fwd_det", "bm_clip_loss_bwd", "bm_clip_loss_bwd_cand", "bm_clip_scores_bwd",
              "bm_clip_loss_fwd_pooled", "bm_clip_loss_fwd_pooled_det", "bm_clip_loss_bwd_pooled")
SIGNATURES.update({name + "_tf32": SIGNATURES[name] for name in TF32_FORMS})
# bf16 forms (bf16() below): the same entry points, the default form's arguments
SIGNATURES.update({name + "_bf16": SIGNATURES[name] for name in TF32_FORMS})


_lib = None


class BmB200Error(RuntimeError):
    pass


def load():
    """Loads the shared library (once).  Raises if it has not been built: there is no CPU path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise BmB200Error(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). brainmagick_b200 has no CPU or PyTorch fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    lib.bm_last_error.restype = ctypes.c_char_p
    lib.bm_last_error.argtypes = []
    lib.bm_abi_version.restype = c_int
    lib.bm_abi_version.argtypes = []
    lib.bm_launch_count.restype = ctypes.c_ulonglong
    lib.bm_launch_count.argtypes = []
    lib.bm_tc_wgrad_workspace.restype = c_longlong
    lib.bm_tc_wgrad_workspace.argtypes = [I, I, I, I]
    lib.bm_tc_wgrad_conv_workspace.restype = c_longlong
    lib.bm_tc_wgrad_conv_workspace.argtypes = [I, I, I, I, I]
    lib.bm_clip_workspace.restype = c_longlong
    lib.bm_clip_workspace.argtypes = [I, I, L]
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = c_longlong if name.endswith("_workspace") else c_int
        fn.argtypes = argtypes
    _lib = lib
    return lib


def ptr(t):
    """Device pointer of a contiguous CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    assert t.is_cuda, "brainmagick_b200 kernels need CUDA tensors (no CPU fallback)"
    assert t.is_contiguous(), "non-contiguous tensor handed to the C ABI"
    return c_void_p(t.data_ptr())


def stream():
    """The current CUDA stream's handle (raw C accessors: torch.cuda.current_stream() builds a Stream object and resolves the
    device through several Python layers, 1.9 ms per step over the ~1 400 calls of one)."""
    return c_void_p(torch._C._cuda_getCurrentRawStream(torch._C._cuda_getDevice()))


def deterministic() -> bool:
    """True when every call should take its deterministic (`_det`) form: exactly when PyTorch's
    torch.use_deterministic_algorithms(True) is in effect.  Read per call; the one place the host code asks."""
    return torch.are_deterministic_algorithms_enabled()


def tf32() -> bool:
    """True when every tensor-core contraction should take its single-pass TF32 (`_tf32`) form: exactly when PyTorch's float32
    matmul precision allows TF32 (torch.backends.cuda.matmul.fp32_precision == "tf32", which torch sets whichever of
    set_float32_matmul_precision("high" / "medium"), matmul.allow_tf32 = True or fp32_precision = "tf32" the caller used).
    cuDNN's conv flag is deliberately not read: it defaults to TF32, and the library's default stays 3xTF32.  Read per call;
    the one place the host code asks."""
    return torch.backends.cuda.matmul.fp32_precision == "tf32"


_recorded = threading.local()          # .bf16: the mode an autograd node's backward replays (recorded_bf16), or None


def bf16() -> bool:
    """True when every tensor-core contraction should take its bf16 (`_bf16`) form: exactly when torch.autocast is enabled
    for CUDA with dtype torch.bfloat16 (an fp16 autocast, or a nested `autocast(enabled=False)`, leaves it False).  Inside
    `recorded_bf16(mode)` it is `mode` instead.  Read per call; the one place the host code asks."""
    mode = getattr(_recorded, "bf16", None)
    if mode is not None:
        return mode
    return torch.is_autocast_enabled("cuda") and torch.get_autocast_dtype("cuda") == torch.bfloat16


@contextlib.contextmanager
def recorded_bf16(mode: bool):
    """Runs the body with bf16() == `mode`.  Autocast is thread-local and torch runs the backward outside it, so each
    autograd node records bf16() in its forward and runs its backward (side-stream weight gradients included) inside
    recorded_bf16 of that record."""
    saved = getattr(_recorded, "bf16", None)
    _recorded.bf16 = bool(mode)
    try:
        yield
    finally:
        _recorded.bf16 = saved


def launch_count() -> int:
    return int(load().bm_launch_count())


def call(name, *args):
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise BmB200Error(f"{name} failed (code {rc}): {lib.bm_last_error().decode()}")
