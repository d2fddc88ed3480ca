"""Where the clocks of the warp-specialised tensor-core loops go, phase by phase: compiles its own copy of libbm_b200.so with
-DBM_HC_PHASES (tc_common.cuh HcProbe: per-CTA %clock sums, never in the shipped library) into --outdir, then runs the conv
shapes of the cfg2 training step (B = 256, T = 360) and the three conv weight gradients, in both pass counts:

  k3_fwd      320 -> 320, k = 3, dilation 2, BatchNorm statistics        (bm_tc_conv1d_persistent)
  k3_bwd      its data gradient (sign -1), accumulated in place
  k4_glu      320 -> 640, k = 3, GLU
  k4_bwd      the GLU conv's data gradient 640 -> 320
  head0       1x1 320 -> 640, GELU (pre-activation copy)
  head1       1x1 640 -> 1024, channel-major output
  head_bwd    1x1 1024 -> 640
  subj        subject layers 288 -> 320 with 4 per-sample weight sets    (bm_tc_pointwise_sel)
  wg_k3, wg_k4, wg_head   bm_tc_wgrad_conv at 320 x 320 x 3, 640 x 320 x 3, 640 x 1024 x 1

Per shape and pass count it prints, in SM clocks: the consumer warpgroup's full-barrier wait, A split + release + adds and MMA issue-to-drain per K block, and its epilogue per tile in three phases (load: the bias / addend / mask loads until issued; store: the math and the
stores; stats: BatchNorm statistics and max |output| after the last store; the weight gradient's whole epilogue is
`store`); the producer's empty-barrier wait,
B load latency (issue, or the point of use when loaded ahead, to registers; the weight gradient: the wait for its staged
dY slot) and TMA / store / fence / arrive per K block (the weight gradient: dY transpose and producer barrier included),
and its start-to-first-full per CTA; and the launch's wall time (CUDA events, probe build: the clock reads cost a little).

    python profiles/conv_phase_probe.py [--csrc DIR] [--outdir DIR] [--lib PATH] [--out result.json]

--csrc compiles another source tree (a csrc/ directory whose ../../include holds bm_b200.h), e.g. the previous commit's
with the same probe; --lib skips the compile and loads a probe build made before.  Prints one JSON line; the card's name and power limit are part of it.  Needs cuda:0.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from brainmagick_b200 import _lib, build  # noqa: E402

PHASES = ["full_wait", "split_add", "mma", "epi_load", "epi_store", "epi_stats", "c_blocks", "tiles",
          "empty_wait", "b_load", "store", "first_full", "p_blocks", "ctas"]          # tc_common.cuh HcPhase
B, T = 256, 360
# name: (entry, Cin, Ntot, Kw, dilation, sign, mode)
CONVS = {
    "k3_fwd": ("persistent", 320, 320, 3, 2, 1, "stats"),
    "k3_bwd": ("persistent", 320, 320, 3, 2, -1, "accumulate"),
    "k4_glu": ("persistent", 320, 640, 3, 1, 1, "glu"),
    "k4_bwd": ("persistent", 640, 320, 3, 1, -1, "plain"),
    "head0": ("persistent", 320, 640, 1, 1, 1, "gelu"),
    "head1": ("persistent", 640, 1024, 1, 1, 1, "tmajor"),
    "head_bwd": ("persistent", 1024, 640, 1, 1, 1, "plain"),
    "subj": ("sel", 288, 320, 1, 1, 1, "plain"),
}
WGRADS = {"wg_k3": (320, 320, 3, 4), "wg_k4": (640, 320, 3, 1), "wg_head": (640, 1024, 1, 1)}
NSETS = 4


def compile_probe(csrc, outdir):
    return build.compile_library(os.path.join(outdir, "libbm_b200_phases.so"), ["-DBM_HC_PHASES"], csrc=csrc)


def conv_call(name, suffix, dev):
    """the launch of conv `name` (a closure over seeded operands)"""
    from brainmagick_b200._lib import call, ptr, stream
    entry, Cin, N, Kw, dil, sign, mode = CONVS[name]
    g = torch.Generator(device=dev).manual_seed(5)
    x = torch.randn(B, T, Cin, device=dev, generator=g)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    if entry == "sel":
        w = torch.randn(NSETS, N, Cin, device=dev, generator=g) * 0.05
        hi, lo = torch.empty_like(w), torch.empty_like(w)
        call("bm_tc_weight_split", ptr(w), NSETS * N, Cin, 1, ptr(hi), ptr(lo), None, None, stream())
        wsel = torch.arange(B, device=dev, dtype=torch.int32) % NSETS
        y = torch.empty(B, T, N, device=dev)
        return lambda: call("bm_tc_pointwise_sel" + suffix, ptr(x), ptr(hi), ptr(lo), ptr(wsel), NSETS, B, T, Cin, N,
                            ptr(y), ptr(status), stream()), status
    w = torch.randn(Kw, N, Cin, device=dev, generator=g) * 0.05
    bias = torch.randn(N, device=dev, generator=g)
    y = torch.empty((B, N, T) if mode == "tmajor" else (B, T, N), device=dev)
    aux = torch.empty(B, T, N, device=dev) if mode == "gelu" else None
    glu_out = torch.empty(B, T, N // 2, device=dev) if mode == "glu" else None
    stats = torch.empty(2 * N, device=dev, dtype=torch.float64) if mode == "stats" else None
    acc = int(mode == "accumulate")
    return lambda: call("bm_tc_conv1d_persistent" + suffix, ptr(x), ptr(w), None if acc else ptr(bias), acc, B, T, Cin,
                        N, Kw, dil, sign, int(mode == "glu"), int(mode == "gelu"), int(mode == "tmajor"), ptr(y),
                        ptr(aux), ptr(glu_out), ptr(stats), ptr(status), stream()), status


def wgrad_call(name, suffix, dev):
    from brainmagick_b200._lib import call, ptr, stream
    M, N, Kw, dil = WGRADS[name]
    g = torch.Generator(device=dev).manual_seed(17)
    dy, x = torch.randn(B, T, M, device=dev, generator=g), torch.randn(B, T, N, device=dev, generator=g)
    ws = torch.empty(int(_lib.load().bm_tc_wgrad_conv_workspace(B, T, M, N, Kw)), device=dev)
    dw = torch.empty(M, N, Kw, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    return lambda: call("bm_tc_wgrad_conv" + suffix, ptr(dy), ptr(x), B, T, M, N, N, Kw, dil, ptr(ws), ptr(dw),
                        ptr(status), stream()), status


def breakdown(c, kernel, launches):
    v = dict(zip(PHASES, c[kernel * len(PHASES):(kernel + 1) * len(PHASES)]))
    cb, pb = max(v["c_blocks"], 1), max(v["p_blocks"], 1)
    r = dict(k_blocks_per_tile=round(v["c_blocks"] / max(v["tiles"], 1), 2), tiles=v["tiles"] // 2 // launches,
             ctas=v["ctas"] // launches)
    r["consumer_per_kblock"] = {k: round(v[k] / cb, 1) for k in ("full_wait", "split_add", "mma")}
    r["consumer_per_kblock"]["total"] = round(sum(r["consumer_per_kblock"].values()), 1)
    r["consumer_epilogue_per_tile"] = {k[4:]: round(v[k] / max(v["tiles"], 1), 1) for k in ("epi_load", "epi_store",
                                                                                             "epi_stats")}
    r["consumer_epilogue_per_tile"]["total"] = round(sum(r["consumer_epilogue_per_tile"].values()), 1)
    r["producer_per_kblock"] = {k: round(v[k] / pb, 1) for k in ("empty_wait", "b_load", "store")}
    r["producer_first_full_per_cta"] = round(v["first_full"] / max(v["ctas"], 1), 1)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--csrc", default=os.path.join(ROOT, "brainmagick_b200", "csrc"))
    ap.add_argument("--outdir", default="")
    ap.add_argument("--lib", default="", help="a probe build to load instead of compiling one")
    ap.add_argument("--launches", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    else:
        outdir = args.outdir or tempfile.mkdtemp(prefix="conv_phase_probe_")
        os.makedirs(outdir, exist_ok=True)
        _lib.LIB_PATH = compile_probe(os.path.abspath(args.csrc), outdir)
    assert torch.cuda.is_available(), "profiles/conv_phase_probe.py measures on cuda:0"
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    lib = _lib.load()
    fn = lib.bm_hc_phases
    fn.argtypes, fn.restype = [ctypes.c_void_p, ctypes.c_int], ctypes.c_int
    counters = (ctypes.c_ulonglong * (2 * len(PHASES)))()
    from profiles.input_grad_cost import card
    res = dict(card=card(), lib=_lib.LIB_PATH, batch=B, T=T, unit="SM clocks", shapes={})
    jobs = [(n, conv_call, 0) for n in CONVS] + [(n, wgrad_call, 1) for n in WGRADS]
    for name, make, kernel in jobs:
        for form, suffix in (("3xtf32", ""), ("tf32", "_tf32")):
            launch, status = make(name, suffix, dev)
            launch()
            assert fn(counters, 1) == 0
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.launches):
                launch()
            e1.record()
            torch.cuda.synchronize()
            assert fn(counters, 1) == 0
            assert int(status.item()) == 0, f"{name}{suffix}: status {int(status.item())}"
            r = breakdown(list(counters), kernel, args.launches)
            r["ms_per_launch"] = round(e0.elapsed_time(e1) / args.launches, 4)
            res["shapes"].setdefault(name, {})[form] = r
            del launch
            torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
