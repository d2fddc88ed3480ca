"""Runs each hot kernel a few times at the BASELINE shape (B=256, T=360, H=320) so that one `ncu --set full`
capture per kernel is short (which = convh | convh_glu | convh_acc | wgradh | conv | conv_glu | conv_acc | wgrad | prep | topk | scores | scores_train | bn_bwd | bn_fwd):   ncu --set full --clock-control none --import-source on -k regex:<name> -s 3 -c 2 \
                               -o gpurun_out/prof_<name> python profiles/profile_kernels.py <which>"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from brainmagick_b200 import _lib  # noqa: E402
from brainmagick_b200._lib import call, ptr, stream  # noqa: E402

which = sys.argv[1] if len(sys.argv) > 1 else "conv"
dev = "cuda"
B, T, H, Kw = 256, 360, 320, 3
status = torch.zeros(1, dtype=torch.int32, device=dev)
if which in ("convh", "convh_glu", "convh_acc", "wgradh"):
    # -k regex:conv_hp_kernel / wgrad_hp_kernel: the F16-pipe kernels the training step runs (K3 forward with BatchNorm
    # statistics | K4 GLU forward (h saved, amax reported) | K3 data gradient, y += tile | K3 weight gradient)
    lib = _lib.load()
    x = torch.randn(B, T, H, device=dev)
    N = 2 * H if which == "convh_glu" else H
    w = torch.randn(N, H, Kw, device=dev) * 0.03
    f, g = torch.empty(Kw, N, H, device=dev), torch.empty(Kw, H, N, device=dev)
    call("bm_tc_weight_split", ptr(w), N, H, Kw, ptr(f), None, ptr(g), None, stream())
    op = g if which == "convh_acc" else f
    amax = torch.empty(4, device=dev)
    call("bm_amax", ptr(x), x.numel(), ptr(amax[0:1]), stream())
    call("bm_amax", ptr(op), op.numel(), ptr(amax[1:2]), stream())
    hi, lo = torch.empty(op.shape, device=dev, dtype=torch.float16), torch.empty(op.shape, device=dev, dtype=torch.float16)
    call("bm_f16_split", ptr(op), op.numel(), ptr(amax[1:2]), ptr(hi), ptr(lo), stream())
    y = torch.zeros(B, T, H, device=dev)
    h = torch.empty(B, T, 2 * H, device=dev) if which == "convh_glu" else None
    stats = torch.empty(2 * H, device=dev, dtype=torch.float64)
    dy = torch.randn(B, T, H, device=dev) * 1e-3
    call("bm_amax", ptr(dy), dy.numel(), ptr(amax[2:3]), stream())
    ws = torch.empty(int(lib.bm_tc_wgrad_conv_workspace(B, T, H, H, Kw)), device=dev)
    dw = torch.empty(H, H, Kw, device=dev)
    for _ in range(6):
        if which == "convh":
            call("bm_tc_conv1d_f16", ptr(x), ptr(amax[0:1]), ptr(hi), ptr(lo), ptr(amax[1:2]), None, 0, B, T, H, H, Kw, 4, 1, 0, 0,
                 0, ptr(y), None, None, ptr(stats), None, ptr(status), stream())
        elif which == "convh_glu":
            call("bm_tc_conv1d_f16", ptr(x), ptr(amax[0:1]), ptr(hi), ptr(lo), ptr(amax[1:2]), None, 0, B, T, H, 2 * H, Kw, 1, 1,
                 1, 0, 0, ptr(h), None, ptr(y), None, ptr(amax[3:4]), ptr(status), stream())
        elif which == "convh_acc":
            call("bm_tc_conv1d_f16", ptr(x), ptr(amax[0:1]), ptr(hi), ptr(lo), ptr(amax[1:2]), None, 1, B, T, H, H, Kw, 4, -1, 0,
                 0, 0, ptr(y), None, None, None, None, ptr(status), stream())
        else:
            call("bm_tc_wgrad_conv_f16", ptr(dy), ptr(amax[2:3]), ptr(x), ptr(amax[0:1]), B, T, H, H, H, Kw, 4, ptr(ws), ptr(dw),
                 ptr(status), stream())
elif which in ("conv", "conv_glu", "conv_acc"):
    # -k regex:conv_pp_kernel: K3 forward with BatchNorm statistics | K4 GLU forward (h saved) | K3 data gradient, y += tile
    x = torch.randn(B, T, H, device=dev)
    N = 2 * H if which == "conv_glu" else H
    w = torch.randn(N, H, Kw, device=dev) * 0.03
    f, g = torch.empty(Kw, N, H, device=dev), torch.empty(Kw, H, N, device=dev)
    call("bm_tc_weight_split", ptr(w), N, H, Kw, ptr(f), None, ptr(g), None, stream())
    y = torch.zeros(B, T, H, device=dev)
    h = torch.empty(B, T, 2 * H, device=dev) if which == "conv_glu" else None
    stats = torch.empty(2 * H, device=dev, dtype=torch.float64)
    for _ in range(6):
        if which == "conv":
            call("bm_tc_conv1d_persistent", ptr(x), ptr(f), None, 0, B, T, H, H, Kw, 4, 1, 0, 0, 0, ptr(y), None, None,
                 ptr(stats), ptr(status), stream())
        elif which == "conv_glu":
            call("bm_tc_conv1d_persistent", ptr(x), ptr(f), None, 0, B, T, H, 2 * H, Kw, 1, 1, 1, 0, 0, ptr(h), None, ptr(y),
                 None, ptr(status), stream())
        else:
            call("bm_tc_conv1d_persistent", ptr(x), ptr(g), None, 1, B, T, H, H, Kw, 4, -1, 0, 0, 0, ptr(y), None, None,
                 None, ptr(status), stream())
elif which == "wgrad":
    dy = torch.randn(B, T, H, device=dev)
    x = torch.randn(B, T, H, device=dev)
    ws = torch.empty(_lib.load().bm_tc_wgrad_conv_workspace(B, T, H, H, Kw), device=dev)      # -k regex:wgrad_pp_kernel
    dw = torch.empty(H, H, Kw, device=dev)
    for _ in range(6):
        call("bm_tc_wgrad_conv", ptr(dy), ptr(x), B, T, H, H, H, Kw, 4, ptr(ws), ptr(dw), ptr(status), stream())
elif which == "prep":          # -k regex:scale_clamp_crop_kernel   (batch preparation, HBM-bound)
    C, Tm, off, R = 273, 361, 18, 27
    x = torch.randn(B, C, Tm, device=dev)
    slot = torch.randint(0, R, (B,), device=dev, dtype=torch.int32)
    center, scale = torch.randn(R, C, device=dev) * 0.1, torch.rand(R, C, device=dev) + 0.5
    y = torch.empty(B, C, Tm - off, device=dev)
    for _ in range(6):
        call("bm_scale_clamp_crop", ptr(x), ptr(slot), ptr(center), ptr(scale), B, C, Tm, off, Tm - off, 20.0, 1, 0, ptr(y),
             None, stream())
elif which == "topk":          # -k regex:retrieval_topk_kernel     (fused softmax + top-k over an L2-resident score row)
    Bn, M = 1024, 4096
    scores = torch.randn(Bn, M, device=dev)
    labels = torch.arange(M, device=dev, dtype=torch.int64)
    targets = torch.randint(0, M, (Bn,), device=dev, dtype=torch.int64)
    top_idx = torch.empty(Bn, 10, device=dev, dtype=torch.int64)
    top_p = torch.empty(Bn, 10, device=dev)
    hit = torch.empty(Bn, device=dev, dtype=torch.int32)
    for _ in range(6):
        call("bm_retrieval_topk", ptr(scores), M, Bn, M, None, 0, 0, 10, ptr(labels), None, ptr(targets), ptr(top_idx),
             ptr(top_p), ptr(hit), None, None, None, stream())
elif which == "scores_train":  # -k regex:clip_scores_kernel          (training shape: 256 x 256 x 368 640, norms + CE fused)
    Bn, M, KT = 256, 256, 1024 * 360
    est = torch.randn(Bn, KT, device=dev) * 0.01
    cand = torch.randn(M, KT, device=dev)
    inv, sc, pr = torch.empty(M, device=dev), torch.empty(Bn, M, device=dev), torch.empty(Bn, M, device=dev)
    rl, loss = torch.empty(Bn, device=dev), torch.empty(1, device=dev)
    ws = torch.empty(max(int(_lib.load().bm_clip_workspace(Bn, M, KT)), 2), device=dev)
    for _ in range(4):
        call("bm_clip_loss_fwd", ptr(est), ptr(cand), Bn, M, KT, 0, ptr(inv), ptr(sc), ptr(pr), ptr(rl), ptr(loss), ptr(ws),
             ws.numel(), ptr(status), stream())
elif which == "scores":        # -k regex:clip_scores_kernel           (retrieval / CLIP score GEMM, K = F*T = 368 640)
    Bn, M, KT = 1024, 2048, 1024 * 360
    est = torch.randn(Bn, KT, device=dev)
    cand = torch.randn(M, KT, device=dev)
    inv = torch.ones(M, device=dev)
    out = torch.empty(Bn, M, device=dev)
    need = int(_lib.load().bm_clip_workspace(Bn, M, KT))
    ws = torch.empty(max(need, 2), device=dev)
    for _ in range(3):
        call("bm_clip_scores", ptr(est), ptr(cand), Bn, M, KT, 1, ptr(inv), ptr(out), None, ptr(ws), ws.numel(), ptr(status),
             stream())
elif which in ("bn_bwd", "bn_fwd"):   # -k regex:epi_bwd_(reduce|apply)_cs_kernel | -k regex:epi_fwd_cs_kernel
    rows = B * T
    dy, x, gy = (torch.randn(B, T, H, device=dev) for _ in range(3))
    gam, bet = torch.ones(H, device=dev), torch.zeros(H, device=dev)
    mean, invstd = torch.zeros(H, device=dev), torch.ones(H, device=dev)
    sums = torch.empty(2 * H, device=dev, dtype=torch.float64)
    dgam, dbet = torch.empty(H, device=dev), torch.empty(H, device=dev)
    amax = torch.empty(1, device=dev)
    for _ in range(6):
        if which == "bn_bwd":
            call("bm_bn_gelu_skip_bwd", ptr(dy), ptr(x), ptr(mean), ptr(invstd), ptr(gam), ptr(bet), 1, rows, H, ptr(sums),
                 ptr(gy), ptr(dgam), ptr(dbet), ptr(amax), stream())
        else:
            call("bm_bn_gelu_skip_fwd", ptr(dy), ptr(mean), ptr(invstd), ptr(gam), ptr(bet), ptr(x), ptr(gy), rows, H, ptr(amax),
                 stream())
torch.cuda.synchronize()
assert int(status.item()) == 0
print("done", which)
