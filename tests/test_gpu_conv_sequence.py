"""The stand-alone ConvSequence (brainmagick_b200.common.ConvSequence, the layers SimpleConv and DeepMel share) at every
option it accepts and on every kernel path `functional._Conv` can pick, against plain references:

* the verbatim reference class, through the `convseq_*` fixtures (oracle/make_golden.py CONVSEQ_CASES), train and eval;
* the oracle (oracle/deepmel_oracle.py) in float64 on the same inputs and parameters, over a matrix of option x width
  configurations that also asserts which kernel classes ran (so that it cannot drift to FMA-only unnoticed);
* BatchNorm batch statistics under large channel offsets: the kernels that produce them, directly, and a ConvSequence /
  SimpleConv step whose BatchNorm-fed conv biases are all shifted by a constant (which changes nothing in exact arithmetic).

Bars: the output, dL/dx, every gradient and the running statistics within 1e-4 relative Frobenius of the reference AND every
element within 1e-3 * max|reference| of it, so that one wrong tile edge cannot hide in a norm."""
import contextlib

import numpy as np
import pytest
import torch

from conftest import load_arrays, rel_err
from oracle import deepmel_oracle
from oracle.make_golden import CONVSEQ_ACTIVATIONS, CONVSEQ_CASES
from brainmagick_b200 import _lib
from brainmagick_b200 import functional as BF
from brainmagick_b200.common import ConvSequence

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = 1e-4            # relative Frobenius
ELEM = 1e-3           # max |err| / max |ref|, per tensor
TF32_TOL = 1e-2       # single-pass TF32: a guess at a bound only a defect would exceed, not yet a measured one

_ACT_NAME = {None: None, "relu": torch.nn.ReLU, "leaky_relu": torch.nn.LeakyReLU, "gelu": torch.nn.GELU}


# ---- helpers ------------------------------------------------------------------------------------------------------
def _module(channels, activation=None, seed=0, perturb=True, **kw):
    torch.manual_seed(seed)
    m = ConvSequence(channels, stride=1, activation=_ACT_NAME[activation], **kw)
    if perturb:
        with torch.no_grad():
            for mod in m.modules():
                if isinstance(mod, torch.nn.BatchNorm1d):
                    mod.weight.add_(0.1 * torch.randn_like(mod.weight))
                    mod.bias.add_(0.1 * torch.randn_like(mod.bias))
                    mod.running_mean.add_(0.1 * torch.randn_like(mod.running_mean))
                    mod.running_var.mul_(1 + 0.2 * torch.rand_like(mod.running_var))
    return m


def _oracle(spec, params, x, gout, training, frozen=(), x_grad=True, dtype=torch.float64):
    """-> dict(out, dx, grads {name: grad}, stats {buffer: new value}, pre_act [...]) of the oracle in `dtype`."""
    p = {k: v.to(dtype).clone() for k, v in params.items() if v.is_floating_point()}
    for k, v in p.items():
        v.requires_grad_("running" not in k and k not in frozen)
    xx = x.to(dtype).clone().requires_grad_(x_grad)
    stats, pre = {}, []
    out = deepmel_oracle.conv_sequence(xx, p, spec, training=training, new_stats=stats, pre_act=pre)
    out.backward(gout.to(dtype))
    return dict(out=out.detach(), dx=xx.grad, grads={k: v.grad for k, v in p.items() if v.requires_grad},
                stats={k: v.detach() for k, v in stats.items()}, pre_act=pre)


def _err(got, ref):
    """(relative Frobenius, max|err| / max|ref|) of got against the reference ref."""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    den = ref.abs().max().item()
    return rel_err(got, ref), (got - ref).abs().max().item() / (den if den > 0 else 1.0)


def _near_kinks(ref):
    return sum(int((z.abs() < 1e-5).sum()) for z in ref["pre_act"])


def _compare(model, out, dx, ref, tag, tol=TOL, elem=ELEM, check_stats=True):
    """Asserts every tensor of the CUDA step against the reference; returns the worst (relative, element) errors."""
    worst = [0.0, 0.0, ""]

    def check(name, got, want):
        assert got is not None, (tag, name, "no gradient")
        r, e = _err(got, want)
        if r > worst[0]:
            worst[0], worst[2] = r, name
        worst[1] = max(worst[1], e)
        assert r <= tol and e <= elem, (f"{tag} {name}: rel {r:.2e} elem {e:.2e}; "
                                        f"{_near_kinks(ref)} pre-activations within 1e-5 of 0")

    check("out", out, ref["out"])
    if ref["dx"] is not None:
        check("dx", dx, ref["dx"])
    wscale = max(v.norm().item() for k, v in ref["grads"].items() if k.endswith("weight"))
    for name, p in model.named_parameters():
        want = ref["grads"].get(name)
        if want is None:
            assert p.grad is None, (tag, name, "a frozen parameter received a gradient")
            continue
        if want.norm().item() < 1e-9 * wscale:        # a conv bias in front of a training BatchNorm: exactly 0
            assert p.grad is not None and p.grad.abs().max().item() <= 1e-6 * wscale, (tag, name)
            continue
        check(name, p.grad, want)
    if check_stats:
        sd = model.state_dict()
        for k, v in ref["stats"].items():
            check(k, sd[k], v)
    return worst


class _PathRecorder:
    """Records the kernel classes every `_Conv` built inside the context selects (functional.py: _Conv / tc_wgrad)."""

    def __init__(self):
        self.seen = set()

    @contextlib.contextmanager
    def active(self):
        orig = BF._Conv.__init__
        rec = self

        def init(conv, w, T, glu, allow_tc, pad_cin_to=0, want_bwd=True):
            orig(conv, w, T, glu, allow_tc, pad_cin_to=pad_cin_to, want_bwd=want_bwd)
            lib = _lib.load()
            rec.seen.add("fwd_pp" if conv.fwd_pp else "fwd_split" if conv.fwd_tc else "fwd_fma")
            if want_bwd:
                rec.seen.add("bwd_pp" if conv.bwd_pp else "bwd_split" if conv.bwd_tc else "bwd_fma")
            if conv.wgrad_tc:
                rows = conv.kw * conv.cin
                pair = bool(lib.bm_tc_wgrad_conv_supported(T, conv.cout, conv.cin, conv.kw)) and \
                    rows / (-(-rows // 256) * 256) >= 0.9
                rec.seen.add("wgrad_pair" if pair else "wgrad_tc")
            else:
                rec.seen.add("wgrad_fma")
            if not glu and conv.fwd_pp:
                rec.seen.add("bn_fused_ok" if conv.cout <= 320 else "bn_unfused_wide")

        BF._Conv.__init__ = init
        try:
            yield self
        finally:
            BF._Conv.__init__ = orig


# ---- 1. the verbatim reference, through the fixtures ---------------------------------------------------------------
@pytest.mark.parametrize("case", list(CONVSEQ_CASES))
def test_convseq_matches_reference_fixture(case):
    g = load_arrays(case)
    c = CONVSEQ_CASES[case]
    model = ConvSequence(c["channels"], stride=1, activation=CONVSEQ_ACTIVATIONS[c["activation"]], **c["kw"])
    model.load_state_dict({k[2:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("p.")}, strict=True)
    model = model.to(DEV).train()
    wscale = max(float(np.linalg.norm(v)) for k, v in g.items() if k.startswith("g.") and k.endswith("weight"))
    for mode, pre in (("train", "g."), ("eval", "ge.")):
        model.train(mode == "train")
        model.zero_grad(set_to_none=True)
        x = torch.from_numpy(g["x"]).to(DEV).requires_grad_(True)
        out = model(x)
        out.backward(torch.from_numpy(g["gout" if mode == "train" else "gout_eval"]).to(DEV))
        BF.check_tc_status()
        assert rel_err(out.detach().cpu(), torch.from_numpy(g["out" if mode == "train" else "out_eval"])) < TOL, mode
        assert rel_err(x.grad.cpu(), torch.from_numpy(g[pre + "x"])) < TOL, mode
        for name, p in model.named_parameters():
            want = torch.from_numpy(g[pre + name])
            if want.norm().item() < 1e-6 * wscale:
                assert p.grad.abs().max().item() < 1e-5 * wscale, (mode, name)
            else:
                assert rel_err(p.grad.cpu(), want) < TOL, (mode, name, rel_err(p.grad.cpu(), want))
        if mode == "train":
            sd = model.state_dict()
            for k, v in g.items():
                if k.startswith("bn."):
                    if "num_batches" in k:
                        assert int(sd[k[3:]]) == int(v), k
                    else:
                        assert rel_err(sd[k[3:]].cpu(), torch.from_numpy(v)) < TOL, k


# ---- 2. option x width matrix against the fp64 oracle --------------------------------------------------------------
def _cfg(ch, B, T, k=3, act=None, leak=0.0, bn=True, skip=True, aol=True, glu=0, ctx=0, dg=2, dp=None, mode="train"):
    return dict(ch=ch, B=B, T=T, kw=dict(kernel=k, batch_norm=bn, skip=skip, activation_on_last=aol, glu=glu,
                                         glu_context=ctx, dilation_growth=dg, dilation_period=dp, leakiness=leak),
                act=act, mode=mode)


MATRIX = [
    # FMA only, C % 4 != 0 (the scalar epilogue kernels) and C % 4 == 0
    _cfg((6, 10, 10, 7), 3, 37, act="relu", aol=False),
    _cfg((6, 10, 10, 7), 2, 150, k=1, act="gelu", skip=False, glu=1, mode="eval"),
    _cfg((12, 16, 16, 16), 3, 9, act="leaky_relu", bn=False, glu=2, ctx=1, dg=3),          # dilation 9 >= T
    _cfg((12, 16, 16, 16), 2, 130, leak=0.2),
    _cfg((6, 10, 10, 7), 2, 12, act="gelu", dg=5, mode="eval"),                             # dilations 5, 25 >= T
    _cfg((16, 16), 2, 50, act="relu"),
    # all tensor cores
    _cfg((160, 160, 160), 2, 100, act="gelu", aol=False, glu=2, ctx=1),
    _cfg((160, 160, 160), 2, 140, k=1, act="relu", bn=False, skip=False, mode="eval"),
    _cfg((256, 256, 256), 2, 60, act="leaky_relu", glu=1),
    _cfg((256, 256, 256), 1, 200, leak=0.1, skip=False, aol=False, glu=2, ctx=1, mode="eval"),
    _cfg((320, 320, 320), 2, 72, act="gelu"),
    _cfg((320, 320, 320), 2, 150, k=1, act="relu", aol=False, glu=1, ctx=1),
    _cfg((320, 320, 320), 1, 100, act="leaky_relu", bn=False, glu=2),
    _cfg((320, 320, 320, 320), 2, 16, act="relu", dg=4),                                    # dilation 16 >= T
    _cfg((160, 320, 320), 2, 100, leak=0.3, glu=2, ctx=1),
    _cfg((320, 160, 160), 2, 130, k=1, act="gelu", bn=False, glu=1, ctx=1),
    # mixed gates: one layer's forward, data gradient and weight gradient on different kernel classes
    _cfg((128, 80, 128), 2, 100, act="relu"),
    _cfg((128, 80, 128), 2, 160, act="gelu", skip=False, aol=False, glu=1, ctx=1, mode="eval"),
    _cfg((80, 128, 80), 2, 50, k=1, leak=0.05, bn=False),
    _cfg((256, 128, 256), 2, 90, aol=False),
    _cfg((128, 256, 256), 2, 130, act="gelu", glu=1, ctx=1),
    _cfg((64, 64, 64), 2, 150, act="relu", bn=False, skip=False, aol=False),
    _cfg((96, 192, 96), 2, 70, act="gelu", mode="eval"),
    _cfg((128, 128, 128), 2, 100, act="leaky_relu", skip=False, mode="eval"),
    # first-layer padding (C0 = 40), without and with a residual on layer 0
    _cfg((40, 160, 160), 3, 60, act="gelu", aol=False, glu=2, ctx=1),
    _cfg((40, 40, 320), 2, 140, act="relu"),
    _cfg((40, 320, 320), 2, 100, act="leaky_relu", glu=1, mode="eval"),
    # BatchNorm wider than 320 (unfused statistics): hidden, and the last layer under activation_on_last
    _cfg((320, 384, 320), 2, 70, act="gelu", aol=False),
    _cfg((256, 640), 2, 140, act="relu"),
    _cfg((320, 384, 384, 320), 1, 130, k=1, act="leaky_relu", glu=2, mode="eval"),
]


def _cfg_id(c):
    kw = c["kw"]
    return (f"{'-'.join(map(str, c['ch']))}_B{c['B']}T{c['T']}_k{kw['kernel']}_{c['act'] or 'lrelu%g' % kw['leakiness']}"
            f"{'_bn' if kw['batch_norm'] else ''}{'_skip' if kw['skip'] else ''}{'_aol' if kw['activation_on_last'] else ''}"
            f"_glu{kw['glu']}c{kw['glu_context']}_{c['mode']}")


def _spec(c):
    return deepmel_oracle.convseq_spec(c["ch"], c["act"], **c["kw"])


def _run_cfg(c, seed, frozen=(), x_grad=True, det=False, tol=TOL, elem=ELEM):
    """One CUDA step of configuration c against the fp64 oracle; -> (worst errors, the CUDA results)."""
    model = _module(c["ch"], c["act"], seed=seed, **c["kw"])
    params = {k: v.detach().clone() for k, v in model.state_dict().items()}
    for name, p in model.named_parameters():
        p.requires_grad_(name not in frozen)
    torch.manual_seed(seed + 1)
    x = torch.randn(c["B"], c["ch"][0], c["T"])
    gout = torch.randn(c["B"], c["ch"][-1], c["T"])
    training = c["mode"] == "train"
    ref = _oracle(_spec(c), params, x, gout, training, frozen=frozen, x_grad=x_grad)
    model = model.to(DEV).train(training)
    xd = x.to(DEV).requires_grad_(x_grad)
    out = model(xd)
    out.backward(gout.to(DEV))
    torch.cuda.synchronize()
    BF.check_tc_status()
    worst = _compare(model, out, xd.grad, ref, _cfg_id(c), tol=tol, elem=elem)
    if training and c["kw"]["batch_norm"]:
        for k, v in model.state_dict().items():
            if "num_batches" in k:
                assert int(v) == 1, k
    res = [out.detach().clone()] + ([xd.grad.clone()] if x_grad else []) + \
        [p.grad.clone() for p in model.parameters() if p.grad is not None] + \
        [v.clone() for k, v in model.state_dict().items() if "running" in k]
    return worst, res


def test_convseq_option_width_matrix_against_fp64():
    rec = _PathRecorder()
    lines = []
    with rec.active():
        for i, c in enumerate(MATRIX):
            worst, _ = _run_cfg(c, seed=100 + i)
            lines.append(f"  {_cfg_id(c):62s} worst rel {worst[0]:.2e} ({worst[2]}), worst elem {worst[1]:.2e}")
    print("\n[conv_sequence] option x width matrix against fp64:\n" + "\n".join(lines))
    print(f"[conv_sequence] kernel classes covered: {sorted(rec.seen)}")
    want = {"fwd_pp", "fwd_split", "fwd_fma", "bwd_pp", "bwd_split", "bwd_fma", "wgrad_pair", "wgrad_tc", "wgrad_fma",
            "bn_fused_ok", "bn_unfused_wide"}
    assert want <= rec.seen, f"kernel classes the matrix no longer reaches: {sorted(want - rec.seen)}"


FROZEN = [
    ("first_layer", _cfg((40, 160, 160), 2, 60, act="gelu", aol=False, glu=2, ctx=1),
     ("sequence.0.0.weight", "sequence.0.0.bias", "sequence.0.1.weight", "sequence.0.1.bias"), True),
    ("glu_blocks", _cfg((128, 256, 256), 2, 130, act="gelu", glu=1, ctx=1), ("glus.0.0.weight", "glus.0.0.bias",
                                                                               "glus.1.0.weight", "glus.1.0.bias"), True),
    ("eval_bn_affine", _cfg((320, 320, 320), 2, 72, act="relu", mode="eval"),
     ("sequence.0.1.weight", "sequence.0.1.bias", "sequence.1.1.weight", "sequence.1.1.bias"), True),
    ("eval_bn_affine_fma", _cfg((6, 10, 10, 7), 2, 37, act="gelu", mode="eval"),
     ("sequence.0.1.weight", "sequence.0.1.bias", "sequence.1.1.weight", "sequence.1.1.bias",
      "sequence.2.1.weight", "sequence.2.1.bias"), True),
    ("input_without_grad", _cfg((128, 80, 128), 2, 100, act="relu"), (), False),
]


@pytest.mark.parametrize("name,c,frozen,x_grad", FROZEN, ids=[f[0] for f in FROZEN])
def test_convseq_frozen_against_fp64(name, c, frozen, x_grad):
    worst, _ = _run_cfg(c, seed=300, frozen=frozen, x_grad=x_grad)
    print(f"\n[conv_sequence] frozen {name}: worst rel {worst[0]:.2e} ({worst[2]}), worst elem {worst[1]:.2e}")


MODES_SUBSET = [MATRIX[0], MATRIX[6], MATRIX[16], MATRIX[27]]


@pytest.mark.parametrize("c", MODES_SUBSET, ids=[_cfg_id(c) for c in MODES_SUBSET])
def test_convseq_deterministic_against_fp64(c):
    """under torch.use_deterministic_algorithms(True): two steps bitwise equal, and both within the fp64 bars"""
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        _, a = _run_cfg(c, seed=400)
        _, b = _run_cfg(c, seed=400)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert len(a) == len(b)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


@pytest.mark.parametrize("c", MODES_SUBSET, ids=[_cfg_id(c) for c in MODES_SUBSET])
def test_convseq_tf32_against_fp64(c):
    """single-pass TF32 (torch.backends.cuda.matmul.fp32_precision = "tf32") within TF32_TOL of fp64 -- the bound is a
    guess at what only a defect would exceed, not a measured one"""
    prev = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    try:
        worst, _ = _run_cfg(c, seed=500, tol=TF32_TOL, elem=10 * TF32_TOL)
    finally:
        torch.backends.cuda.matmul.fp32_precision = prev
    print(f"\n[conv_sequence] tf32 {_cfg_id(c)}: worst rel {worst[0]:.2e} ({worst[2]}), worst elem {worst[1]:.2e}")


# ---- 3. BatchNorm statistics under large channel offsets -----------------------------------------------------------
OFFSETS = (0.0, 10.0, 1e2, 1e3)        # per-channel mean / std of y, cycled over the channels


def _finalize_check(y, stats, C, tag):
    """bm_bn_stats_finalize of the kernel's stats against an fp64 two-pass over the kernel's own fp32 y"""
    rows = y.numel() // C
    mean, invstd = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
    rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    _lib.call("bm_bn_stats_finalize", _lib.ptr(stats), rows, 1e-5, 0.1, _lib.ptr(rm), _lib.ptr(rv), _lib.ptr(mean),
              _lib.ptr(invstd), C, _lib.stream())
    yd = y.reshape(rows, C).double().cpu()
    m = yd.mean(0)
    var = ((yd - m) ** 2).mean(0)
    e_mean = ((mean.cpu().double() - m).abs() / m.abs().clamp_min(var.sqrt())).max().item()
    e_inv = ((invstd.cpu().double() * (var + 1e-5).sqrt()) - 1).abs().max().item()
    rv_ref = 0.9 + 0.1 * var * rows / (rows - 1)
    e_rv = ((rv.cpu().double() - rv_ref).abs() / rv_ref).max().item()
    print(f"  {tag:42s} mean {e_mean:.1e}  invstd {e_inv:.1e}  running_var {e_rv:.1e}")
    return e_mean, e_inv, e_rv


def _offset_bias(C, std):
    return torch.tensor([OFFSETS[c % len(OFFSETS)] * std for c in range(C)], dtype=torch.float32)


def test_bn_statistics_exact_under_channel_offsets():
    torch.manual_seed(7)
    B, T = 4, 360
    results = []
    print("\n[conv_sequence] BatchNorm statistics, channel mean/std cycling through", OFFSETS)
    # bm_col_stats (+ _det) on a y with the offsets built in
    C = 384
    y = (torch.randn(B * T, C) + _offset_bias(C, 1.0)).to(DEV)
    for det in (False, True):
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(det)
        try:
            stats = torch.empty(2 * C, device=DEV, dtype=torch.float64)
            BF.col_stats(y, B * T, C, stats, _lib.stream())
        finally:
            torch.use_deterministic_algorithms(prev)
        results.append(_finalize_check(y, stats, C, "bm_col_stats" + ("_det" if det else "")))
    # the conv kernels with statistics: bm_conv1d_fwd (FP32 FMA) and the fused epilogue of bm_tc_conv1d_persistent
    # (+ _tf32); the bias provides the offset
    for cin, cout, tc, tf32 in ((24, 36, False, False), (256, 256, True, False), (256, 320, True, True),
                                (256, 320, True, False)):
        w = torch.randn(cout, cin, 3) / (3 * cin) ** 0.5
        x = torch.randn(B, T, cin).to(DEV)
        # y's std per channel is ~ ||w[c]||; the offset in units of it
        std = w.reshape(cout, -1).norm(dim=1)
        bias = (_offset_bias(cout, 1.0) * std).to(DEV)
        prev = torch.backends.cuda.matmul.fp32_precision
        torch.backends.cuda.matmul.fp32_precision = "tf32" if tf32 else "ieee"
        try:
            conv = BF._Conv(w.to(DEV), T, False, tc, want_bwd=False)
            assert conv.fwd_pp == tc
            yb = torch.empty(B, T, cout, device=DEV)
            stats = torch.empty(2 * cout, device=DEV, dtype=torch.float64)
            conv.forward(x, bias, B, T, 2, yb, stats, BF.tc_status_tensor(DEV))
        finally:
            torch.backends.cuda.matmul.fp32_precision = prev
        BF.check_tc_status()
        name = "bm_tc_conv1d_persistent" + ("_tf32" if tf32 else "") if tc else "bm_conv1d_fwd"
        results.append(_finalize_check(yb, stats, cout, f"{name} {cin}->{cout}"))
    for e_mean, e_inv, e_rv in results:
        assert e_mean <= 1e-7 and e_inv <= 1e-6 and e_rv <= 1e-6, (e_mean, e_inv, e_rv)


def _shifted(model, shift):
    """every conv bias that feeds a training-mode BatchNorm + shift (the output does not change in exact arithmetic)"""
    with torch.no_grad():
        for k, blk in enumerate(model.sequence):
            if len(blk) > 1 and isinstance(blk[1], torch.nn.BatchNorm1d):
                blk[0].bias.add_(shift)


@pytest.mark.parametrize("ch,T", [((40, 320, 320, 320), 150), ((20, 24, 24, 24), 100), ((256, 384, 256), 90)])
def test_convseq_bias_offset_invariance(ch, T):
    results = []
    for shift in (0.0, 1e3):
        model = _module(ch, "gelu", seed=11, perturb=True, kernel=3, batch_norm=True, skip=True,
                        activation_on_last=True, glu=2, glu_context=1, dilation_growth=2)
        _shifted(model, shift)
        model = model.to(DEV).train()
        torch.manual_seed(12)
        x = torch.randn(2, ch[0], T, device=DEV).requires_grad_(True)
        out = model(x)
        out.backward(torch.randn(2, ch[-1], T, device=DEV))
        BF.check_tc_status()
        grads = {n: p.grad.clone() for n, p in model.named_parameters() if not n.endswith("0.bias")}
        results.append(dict(out=out.detach(), dx=x.grad, **grads))
    base, shifted = results
    worst = max((rel_err(shifted[k].cpu(), base[k].cpu()), k) for k in base)
    print(f"\n[conv_sequence] {'-'.join(map(str, ch))} conv biases + 1e3: worst rel {worst[0]:.2e} ({worst[1]})")
    assert worst[0] <= 1e-3, worst


def test_simpleconv_bias_offset_invariance():
    """a small SimpleConv step at tensor-core widths: output and gradients unchanged when every conv bias in front of a
    BatchNorm is shifted by 1e3.  Ten layers deep, storing y ~ 1e3 std in fp32 moves the deepest gradients by more than 1e-3
    in any fp32 implementation: the oracle in fp32 (two-pass BatchNorm statistics) moves initial_linear's by 3.5e-3.  So
    each tensor is held to 1e-3 or twice the fp32 oracle's own change, whichever is larger (before the statistics were
    exact, the change was ~1e11)."""
    from oracle import bm_oracle
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    cfg = bm_oracle.Config(in_channels=40, out_channels=128, n_subjects=3, hidden=160, merger_channels=48,
                           initial_linear=24, merger_pos_dim=128)
    params = bm_oracle.init_state_dict(cfg, seed=1)
    d = bm_oracle.synthetic_batch(cfg, batch=8, T=60, seed=2)
    d["rec_positions"] = synthetic.normalised_positions(cfg.n_subjects, cfg.in_channels, seed=3)
    results = []
    for shift in (0.0, 1e3):
        model = bb.SimpleConv(
            in_channels=dict(meg=cfg.in_channels), out_channels=cfg.out_channels, hidden=dict(meg=cfg.hidden),
            depth=cfg.depth, dilation_period=cfg.dilation_period, kernel_size=3, skip=True, subject_layers=True,
            subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=cfg.initial_linear,
            merger_channels=cfg.merger_channels, gelu=True, batch_norm=True, merger_pos_dim=cfg.merger_pos_dim,
            n_subjects=cfg.n_subjects)
        model.load_state_dict(params)
        bn_fed = set()          # their gradients are 0 in exact arithmetic (rounding noise on the reference too)
        with torch.no_grad():
            for name, mod in model.named_modules():
                if isinstance(mod, ConvSequence):
                    for k, blk in enumerate(mod.sequence):
                        if len(blk) > 1 and isinstance(blk[1], torch.nn.BatchNorm1d):
                            blk[0].bias.add_(shift)
                            bn_fed.add(f"{name}.sequence.{k}.0.bias")
        assert bn_fed
        model = model.cuda().train()
        model.merger.ban_centre_override = d["ban_centre"]
        meg = d["meg"].cuda()
        batch = synthetic.make_batch(meg, d["subject_index"].cuda(), d["rec_positions"], d["rec_of_sample"])
        est = model(dict(meg=meg), batch)
        loss = bb.ClipLoss().cuda().train()(est, d["candidates"].cuda(),
                                            torch.ones(8, 1, 60, dtype=torch.bool, device="cuda"))
        loss.backward()
        BF.check_tc_status()
        results.append(dict(est=est.detach(), **{n: p.grad.clone() for n, p in model.named_parameters()
                                                 if p.grad is not None and n not in bn_fed}))
    base, shifted = results
    assert sorted(base) == sorted(shifted)
    floor = []                  # the fp32 oracle's own change under the same shift
    for shift in (0.0, 1e3):
        p = {k: v.clone() for k, v in params.items()}
        for k in p:
            if k.endswith(".0.bias") and k.replace(".0.bias", ".1.running_mean") in p:
                p[k] += shift
        floor.append(bm_oracle.training_step(p, cfg, d["meg"], d["rec_positions"], d["rec_of_sample"], d["subject_index"],
                                             d["candidates"], ban_centre=d["ban_centre"], training=True))
    fa, fb = floor
    ref_change = {k: rel_err(fb["grads"][k], fa["grads"][k]) for k in base if k != "est"}
    ref_change["est"] = rel_err(fb["estimate"], fa["estimate"])
    worst = max((rel_err(shifted[k].cpu(), base[k].cpu()), k) for k in base)
    print(f"\n[conv_sequence] SimpleConv conv biases + 1e3: worst rel {worst[0]:.2e} ({worst[1]}; the fp32 oracle moves it "
          f"by {ref_change[worst[1]]:.2e})")
    for k in base:
        err = rel_err(shifted[k].cpu(), base[k].cpu())
        assert err <= max(1e-3, 2 * ref_change[k]), (k, err, ref_change[k])
