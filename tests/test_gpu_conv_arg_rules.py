"""GPU: which argument combinations the tensor-core conv entry points accept.  Every conv entry point and its `_tf32` form is
called on small real buffers with each combination of its epilogue flags (glu, act, out_tmajor, aux, addend / accumulate,
stats, amax_out), at shapes on both sides of its shape gate.  A call either returns 0 and writes finite outputs, or returns
2 with bm_last_error() naming the entry point; which one is written below as one rule per entry point."""
import itertools

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
B, T, KW, DIL = 2, 40, 3, 2


# ---- the rules --------------------------------------------------------------------------------------------------------
def tc_gate(Cin, Ntot, glu):
    """bm_tc_conv_supported: K chunks of 32 input channels; Ntot with a divisor in [64, 160] that is a multiple of 16
    (GLU: H = Ntot / 2 a multiple of 80)"""
    if Cin % 32:
        return False
    if glu:
        return Ntot % 2 == 0 and (Ntot // 2) % 80 == 0
    return any(Ntot % bn == 0 for bn in range(64, 161, 16))


def half_width(Ntot, glu):
    """bm_tc_conv1d_persistent_supported's column halves: nh = 160 or 128 with Ntot a multiple of 2 nh (GLU: H a multiple
    of nh); 0 if neither"""
    if glu and Ntot % 2:
        return 0
    n = Ntot // 2 if glu else Ntot
    for nh in (160, 128):
        if n % (nh if glu else 2 * nh) == 0:
            return nh
    return 0


def halves_gate(Cin, Ntot, glu):
    return Cin % 32 == 0 and half_width(Ntot, glu) != 0


def conv1d_accepts(f, Cin, Ntot):
    """bm_tc_conv1d[_tf32]: no statistics; GLU excludes act, out_tmajor and aux (an addend is accepted and ignored);
    act and out_tmajor combine with each other and with the addend"""
    if f["stats"]:
        return False
    if f["glu"] and (f["act"] or f["tmajor"] or f["aux"]):
        return False
    return tc_gate(Cin, Ntot, f["glu"])


def persistent_accepts(f, Cin, Ntot):
    """bm_tc_conv1d_persistent[_tf32]: GLU excludes every other epilogue; channel-major output is a plain store;
    accumulate excludes the activation; statistics only of a plain conv of one pair of column halves (Ntot = 2 nh)"""
    glu, act, tm, aux, acc, stats = (f[k] for k in ("glu", "act", "tmajor", "aux", "add", "stats"))
    if not halves_gate(Cin, Ntot, glu):
        return False
    if stats and (glu or tm or act or acc or Ntot != 2 * half_width(Ntot, 0)):
        return False
    if glu and (act or tm or aux or acc):
        return False
    if tm and (act or acc):
        return False
    return not (act and acc)


def f16_accepts(f, Cin, Ntot):
    """bm_tc_conv1d_f16: the persistent rules; amax_out only of a GLU or GELU output stored row-major"""
    if f["amax"] and not ((f["glu"] or f["act"]) and not f["tmajor"]):
        return False
    return persistent_accepts(f, Cin, Ntot)


def pointwise_accepts(Cin, Ntot):
    """bm_tc_pointwise_sel[_tf32]: the shape gate of bm_tc_conv1d at one tap"""
    return tc_gate(Cin, Ntot, 0)


def sensor_mix_accepts(Op, Cp, C):
    """bm_tc_sensor_mix_bwd_data[_tf32]: the shape gate of bm_tc_conv1d at one tap over (Op, Cp), C <= Cp live rows"""
    return tc_gate(Op, Cp, 0) and C <= Cp


# ---- the calls --------------------------------------------------------------------------------------------------------
def _lib():
    from brainmagick_b200 import _lib as L
    return L.load(), L.ptr, L.stream


class _Calls:
    """Runs calls and collects every one whose outcome breaks its rule."""

    def __init__(self, token):
        self.lib, self.ptr, self.stream = _lib()
        self.token = token
        self.status = torch.zeros(1, dtype=torch.int32, device=DEV)
        self.failures = []

    def run(self, entry, args, accepted, outputs, case):
        lib = self.lib
        # a refusal with a known message first: the message checked below must be the one this call wrote
        assert lib.bm_gather_rows(None, None, 0, 0, None, None) == 2
        rc = getattr(lib, entry)(*args)
        msg = lib.bm_last_error().decode()
        if accepted:
            if rc != 0:
                self.failures.append(f"{entry} {case}: refused ({rc}: {msg}), expected accepted")
                return
            torch.cuda.synchronize()
            if int(self.status.item()) != 0:
                self.failures.append(f"{entry} {case}: status {int(self.status.item())}")
                self.status.zero_()
            for name, t in outputs:
                if not bool(torch.isfinite(t).all()):
                    self.failures.append(f"{entry} {case}: {name} not finite")
        elif rc != 2 or msg.startswith("bm_gather_rows") or self.token not in msg:
            self.failures.append(f"{entry} {case}: returned {rc} ({msg}), expected 2 naming {self.token}")

    def check(self):
        assert not self.failures, f"{len(self.failures)} calls broke their rule:\n" + "\n".join(self.failures[:30])


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


# Cin, Ntot, glu: both sides of bm_tc_conv_supported (Ntot 200, H 100, Cin 48 fail it) and of the column-halves gate
# (Ntot 256 / 320 / 640 and H 160 pass it; 256 and 320 are single pairs of halves, 640 is two)
SHAPES = [(32, 160, 0), (32, 200, 0), (32, 256, 0), (32, 320, 0), (32, 640, 0), (48, 320, 0),
          (32, 160, 1), (32, 200, 1), (32, 320, 1)]
FLAGS = ("act", "tmajor", "aux", "add", "stats")


def _operands(Cin, Ntot, Bn=B, Tn=T):
    """x [Bn,Tn,Cin], weights [KW,Ntot,Cin] (also read as per-sample weight sets), their second tf32 piece, bias [Ntot]"""
    g = torch.Generator(device=DEV).manual_seed(Cin * 1000 + Ntot)
    x = torch.randn(Bn, Tn, Cin, device=DEV, generator=g)
    w = torch.randn(KW, Ntot, Cin, device=DEV, generator=g) * 0.05
    return x, w, w * 1e-4, torch.randn(Ntot, device=DEV, generator=g)


def _f16_pieces(w):
    """fp16 pieces of w scaled by 2^14 (= f16_scale_of(1.0)), and 1.0 as their amax"""
    return (w * 2.0 ** 14).half(), torch.zeros_like(w, dtype=torch.float16), torch.ones(1, device=DEV)


@pytest.mark.parametrize("Cin,Ntot,glu", SHAPES)
@pytest.mark.parametrize("entry", ["bm_tc_conv1d", "bm_tc_conv1d_tf32", "bm_tc_conv1d_persistent",
                                   "bm_tc_conv1d_persistent_tf32", "bm_tc_conv1d_f16"])
def test_conv_epilogue_rules(entry, Cin, Ntot, glu):
    c = _Calls("conv")
    lib, ptr, st = c.lib, c.ptr, c.stream
    x, w, w_lo, bias = _operands(Cin, Ntot)
    hi16, lo16, w_amax = _f16_pieces(w)
    x_amax = x.abs().max().reshape(1)
    addend = torch.randn(B, T, Ntot, device=DEV)
    base = entry.removesuffix("_tf32")
    names = FLAGS + (("amax",) if base == "bm_tc_conv1d_f16" else ())
    rule = {"bm_tc_conv1d": conv1d_accepts, "bm_tc_conv1d_persistent": persistent_accepts,
            "bm_tc_conv1d_f16": f16_accepts}[base]
    gate = lib.bm_tc_conv_supported if base == "bm_tc_conv1d" else lib.bm_tc_conv1d_persistent_supported
    assert bool(gate(T, Cin, Ntot, KW, glu)) == (tc_gate if base == "bm_tc_conv1d" else halves_gate)(Cin, Ntot, glu)
    for bits in itertools.product((0, 1), repeat=len(names)):
        f = dict(zip(names, bits), glu=glu)
        # accumulate adds onto y: it then starts finite
        y = torch.zeros(B, T, Ntot, device=DEV) if f["add"] and base != "bm_tc_conv1d" else _nan(B, T, Ntot)
        aux = _nan(B, T, Ntot) if f["aux"] else None
        glu_out = _nan(B, T, Ntot // 2) if glu else None
        stats = torch.full((2 * Ntot,), float("nan"), device=DEV, dtype=torch.float64) if f["stats"] else None
        amax = _nan(1) if f.get("amax") else None
        shape = (B, T, Cin, Ntot, KW, DIL, 1, glu, f["act"], f["tmajor"])
        outs = (ptr(y), ptr(aux), ptr(glu_out), ptr(stats))
        if base == "bm_tc_conv1d":
            args = (ptr(x), ptr(w), ptr(w_lo), ptr(bias), ptr(addend if f["add"] else None)) + shape + outs
        elif base == "bm_tc_conv1d_persistent":
            args = (ptr(x), ptr(w), ptr(bias), f["add"]) + shape + outs
        else:
            args = (ptr(x), ptr(x_amax), ptr(hi16), ptr(lo16), ptr(w_amax), ptr(bias), f["add"]) + shape + outs + \
                (ptr(amax),)
        written = [("glu_out", glu_out)] if glu else [("y", y)]
        written += [("stats", stats)] if stats is not None else []
        written += [("amax_out", amax)] if amax is not None else []
        c.run(entry, args + (ptr(c.status), st()), rule(f, Cin, Ntot), written, f"Cin={Cin} Ntot={Ntot} {f}")
    c.check()


@pytest.mark.parametrize("Cin,Ntot", [(32, 160), (32, 200), (32, 320), (32, 640), (48, 160)])
@pytest.mark.parametrize("entry", ["bm_tc_pointwise_sel", "bm_tc_pointwise_sel_tf32"])
def test_pointwise_sel_rules(entry, Cin, Ntot):
    c = _Calls("pointwise_sel")
    ptr, st = c.ptr, c.stream
    n_sets = 3
    x = torch.randn(B, T, Cin, device=DEV)
    w = torch.randn(n_sets, Ntot, Cin, device=DEV) * 0.05
    w_lo = w * 1e-4
    wsel = torch.tensor([2, 0], device=DEV, dtype=torch.int32)
    assert bool(c.lib.bm_tc_conv_supported(T, Cin, Ntot, 1, 0)) == pointwise_accepts(Cin, Ntot)
    y = _nan(B, T, Ntot)
    c.run(entry, (ptr(x), ptr(w), ptr(w_lo), ptr(wsel), n_sets, B, T, Cin, Ntot, ptr(y), ptr(c.status), st()),
          pointwise_accepts(Cin, Ntot), [("y", y)], f"Cin={Cin} Ntot={Ntot}")
    c.check()


@pytest.mark.parametrize("Op,Cp", [(32, 160), (32, 200), (32, 320), (48, 160)])
@pytest.mark.parametrize("entry", ["bm_tc_sensor_mix_bwd_data", "bm_tc_sensor_mix_bwd_data_tf32"])
def test_sensor_mix_bwd_data_rules(entry, Op, Cp):
    c = _Calls("sensor_mix")
    ptr, st = c.ptr, c.stream
    n_sets = 3
    du = torch.randn(B, T, Op, device=DEV)
    w = torch.randn(n_sets, Cp, Op, device=DEV) * 0.05
    w_lo = w * 1e-4
    wsel = torch.tensor([1, 2], device=DEV, dtype=torch.int32)
    for C, masked in itertools.product((Cp - 7, Cp, Cp + 1), (0, 1)):
        mask = (torch.arange(C, device=DEV) % 3 != 0).float() if masked else None
        dmeg = _nan(B, C, T)
        c.run(entry, (ptr(du), ptr(w), ptr(w_lo), ptr(wsel), n_sets, ptr(mask), B, T, Op, Cp, C, ptr(dmeg),
                      ptr(c.status), st()),
              sensor_mix_accepts(Op, Cp, C), [("dmeg", dmeg)], f"Op={Op} Cp={Cp} C={C} mask={masked}")
    c.check()


@pytest.mark.parametrize("entry", ["bm_tc_conv1d", "bm_tc_conv1d_tf32", "bm_tc_pointwise_sel", "bm_tc_pointwise_sel_tf32",
                                   "bm_tc_sensor_mix_bwd_data", "bm_tc_sensor_mix_bwd_data_tf32"])
def test_second_weight_piece(entry):
    """The 3xTF32 forms need both tf32 pieces of the weights; the `_tf32` forms read the first alone."""
    c = _Calls("sensor_mix" if "sensor" in entry else "pointwise_sel" if "pointwise" in entry else "conv")
    ptr, st = c.ptr, c.stream
    Cin, Ntot = 32, 320
    x, w, _, bias = _operands(Cin, Ntot)
    wsel = torch.tensor([1, 0], device=DEV, dtype=torch.int32)
    out = _nan(B, T, Ntot)
    if entry.startswith("bm_tc_conv1d"):
        args = (ptr(x), ptr(w), None, ptr(bias), None, B, T, Cin, Ntot, KW, DIL, 1, 0, 0, 0, ptr(out), None, None, None)
    elif "pointwise" in entry:
        args = (ptr(x), ptr(w[:2]), None, ptr(wsel), 2, B, T, Cin, Ntot, ptr(out))
    else:
        args = (ptr(x), ptr(w[:2]), None, ptr(wsel), 2, None, B, T, Cin, Ntot, Ntot, ptr(out))
    c.run(entry, args + (ptr(c.status), st()), entry.endswith("_tf32"), [("output", out)], "w_lo = NULL")
    c.check()


@pytest.mark.parametrize("entry,tmajor", [(e, tm) for e in ("bm_tc_conv1d", "bm_tc_conv1d_tf32", "bm_tc_conv1d_persistent",
                                                            "bm_tc_conv1d_persistent_tf32", "bm_tc_conv1d_f16")
                                           for tm in (0, 1)] +
                         [("bm_tc_sensor_mix_bwd_data", 1), ("bm_tc_sensor_mix_bwd_data_tf32", 1)])
def test_output_alignment(entry, tmajor):
    """The conv epilogue stores row-major outputs as float2: such an output 4 bytes off an 8-byte boundary is refused.  The
    channel-major output and the sensor mix's dmeg are stored element by element and accepted there."""
    c = _Calls("sensor_mix" if "sensor" in entry else "conv")
    ptr, st = c.ptr, c.stream
    Cin, Ntot = 32, 320
    x, w, w_lo, bias = _operands(Cin, Ntot)
    buf = _nan(B * T * Ntot + 1)
    out = buf[1:]                                                     # contiguous, 4 bytes past an 8-byte boundary
    if entry.startswith("bm_tc_sensor_mix"):                          # dmeg is channel-major
        wsel = torch.tensor([1, 0], device=DEV, dtype=torch.int32)
        args = (ptr(x), ptr(w[:2]), ptr(w_lo[:2]), ptr(wsel), 2, None, B, T, Cin, Ntot, Ntot, ptr(out))
        accepted = True
    else:
        shape = (B, T, Cin, Ntot, KW, DIL, 1, 0, 0, tmajor, ptr(out), None, None, None)
        if entry.startswith("bm_tc_conv1d_persistent"):
            args = (ptr(x), ptr(w), ptr(bias), 0) + shape
        elif entry == "bm_tc_conv1d_f16":
            hi16, lo16, one = _f16_pieces(w)
            args = (ptr(x), ptr(one), ptr(hi16), ptr(lo16), ptr(one), ptr(bias), 0) + shape + (None,)
        else:
            args = (ptr(x), ptr(w), ptr(w_lo), ptr(bias), None) + shape
        accepted = bool(tmajor)
    c.run(entry, args + (ptr(c.status), st()), accepted, [("output", out)], f"misaligned output, out_tmajor={tmajor}")
    c.check()


@pytest.mark.parametrize("entry", ["bm_tc_conv1d", "bm_tc_conv1d_tf32", "bm_tc_conv1d_persistent",
                                   "bm_tc_conv1d_persistent_tf32", "bm_tc_conv1d_f16", "bm_tc_pointwise_sel",
                                   "bm_tc_pointwise_sel_tf32", "bm_tc_sensor_mix_bwd_data",
                                   "bm_tc_sensor_mix_bwd_data_tf32"])
def test_batch_limit(entry):
    """bm_tc_conv1d and bm_tc_pointwise_sel take at most 65535 samples; the persistent, fp16-piece and sensor-mix entry
    points take more."""
    c = _Calls("sensor_mix" if "sensor" in entry else "pointwise_sel" if "pointwise" in entry else "conv")
    ptr, st = c.ptr, c.stream
    Bn, Tn, Cin, Ntot = 65536, 8, 32, 320
    x, w, w_lo, bias = _operands(Cin, Ntot, Bn, Tn)
    wsel = torch.arange(Bn, device=DEV, dtype=torch.int32) % 2
    out = _nan(Bn, Tn, Ntot)
    if entry.startswith("bm_tc_sensor_mix"):
        args = (ptr(x), ptr(w[:2]), ptr(w_lo[:2]), ptr(wsel), 2, None, Bn, Tn, Cin, Ntot, Ntot, ptr(out))
    elif entry.startswith("bm_tc_pointwise_sel"):
        args = (ptr(x), ptr(w[:2]), ptr(w_lo[:2]), ptr(wsel), 2, Bn, Tn, Cin, Ntot, ptr(out))
    else:
        shape = (Bn, Tn, Cin, Ntot, KW, DIL, 1, 0, 0, 0, ptr(out), None, None, None)
        if entry.startswith("bm_tc_conv1d_persistent"):
            args = (ptr(x), ptr(w), ptr(bias), 0) + shape
        elif entry == "bm_tc_conv1d_f16":
            hi16, lo16, one = _f16_pieces(w)
            args = (ptr(x), ptr(one), ptr(hi16), ptr(lo16), ptr(one), ptr(bias), 0) + shape + (None,)
        else:
            args = (ptr(x), ptr(w), ptr(w_lo), ptr(bias), None) + shape
    accepted = entry.removesuffix("_tf32") not in ("bm_tc_conv1d", "bm_tc_pointwise_sel")
    c.run(entry, args + (ptr(c.status), st()), accepted, [("output", out)], f"B={Bn}")
    c.check()
