"""GPU: every C entry point that is not a contraction -- the ConvSequence layer epilogue (csrc/convseq.cuh), the BatchNorm
finalize, the column reductions, the GLU / GELU backward, the attention pieces, the layouts and the ClipLoss norms
(csrc/elementwise.cuh, front.cuh, prep.cuh, clip.cuh) -- against a plain fp64 reference, element by element, on each of its
kernel forms.

The reference is computed in fp64 from the fp32 operands the kernel read.  Each output is held to a componentwise bound

    |got - ref| <= K * (first-order rounding error of the kernel's arithmetic) + TINY

with one constant K per group (K_EPI, K_BN, K_RED, K_GLU, K_ATT) that covers the second-order terms and the 1 / (1 - n u)
factors.  The first-order error counts u = 2^-24 per fp32 rounding, times the magnitude of the rounded value, and carries
each operand's error through the operations that follow (the error of the batch means into dz - m1 - yhat*m2, of sigma into
1 - sigma).  A sum of n fp32 terms errs by at most gamma_n = n u times the sum of |terms| whatever the order, so the fp32
per-thread sums of the reductions are held to gamma_rows * sum|terms|.  Where a kernel approximates a function, the bound adds
that approximation's documented error:
  - erfcc (Numerical Recipes, GELU's Phi in common.cuh): fractional error below 1.2e-7;
  - __expf: 2 + floor(|1.173 x|) ulp (CUDA C++ Programming Guide, intrinsic functions); expf: 2 ulp;
  - rcp.approx.ftz.f32: 1 ulp (PTX ISA);
  - sincosf: 2 ulp (CUDA C++ Programming Guide, single-precision functions).
One ulp of a value is at most 2 u times its magnitude.  Layout kernels (transposes, the channel mask, the weight re-layout) are
compared bit for bit.

Every output starts as NaN inside a buffer whose guard zones hold a sentinel bit pattern: an element left unwritten stays NaN,
a write outside the output changes the sentinel.  The epilogue, GLU and GELU cases read the names of the kernels that ran from
torch.profiler and assert which form each shape took: column-stationary (`*_cs_kernel`), the generic float4 form (template
argument VEC = 4, `*_v4_kernel`) or the generic scalar form.
"""
import contextlib
import math
import re

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24                # unit roundoff of fp32
UD = 2.0 ** -53               # unit roundoff of fp64
TINY = 2.0 ** -140            # underflow: a few fp32 subnormal steps
GUARD = 64                    # elements of sentinel before and after every output
SENT = {torch.float32: 0x7FA5A5A5, torch.float64: 0x7FF5A5A5A5A5A5A5}   # NaN bit patterns no kernel computes
IVIEW = {torch.float32: torch.int32, torch.float64: torch.int64}
K_EPI = 2.0                   # layer epilogue
K_BN = 2.0                    # BatchNorm finalize
K_RED = 2.0                   # column reductions and the ClipLoss norms
K_GLU = 2.0                   # GLU and GELU backward
K_ATT = 2.0                   # softmax pieces


def _abi():
    from brainmagick_b200 import _lib
    return _lib.call, _lib.ptr, _lib.stream


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _rand(gen, *shape, scale=1.0):
    return torch.randn(*shape, generator=gen, device=DEV) * scale


def _gamma(n):
    return n * U / (1 - n * U)


def _dev(t, off=0):
    """t as a contiguous device tensor starting `off` floats past a 16-byte aligned allocation"""
    buf = torch.empty(t.numel() + off, dtype=t.dtype, device=DEV)
    v = buf[off:].view(t.shape)
    v.copy_(t)
    return v


class Out:
    """A NaN-filled output `shape` (last dimension padded to `ld` columns) starting `off` elements into a flat buffer with
    sentinel guard zones and sentinel padding columns.  .t: the full (padded) tensor the kernel receives; .v: the valid
    columns."""

    def __init__(self, *shape, ld=None, off=0, dtype=torch.float32):
        full = list(shape)
        full[-1] = ld or shape[-1]
        n = math.prod(full)
        self.dtype = dtype
        self.lead = GUARD + off
        self.flat = torch.full((n + self.lead + GUARD,), SENT[dtype], dtype=IVIEW[dtype], device=DEV).view(dtype)
        self.t = self.flat[self.lead:self.lead + n].view(full)
        self.v = self.t[..., :shape[-1]]
        self.v.fill_(float("nan"))
        self.width = shape[-1]

    def untouched(self, what):
        bits = self.flat.view(IVIEW[self.dtype])
        s = SENT[self.dtype]
        assert (bits[:self.lead] == s).all() and (bits[-GUARD:] == s).all(), f"{what}: write outside the output"
        pad = self.t.view(IVIEW[self.dtype])[..., self.width:]
        assert (pad == s).all(), f"{what}: padding columns overwritten"

    def unwritten(self, what):
        assert torch.isnan(self.v).all(), f"{what}: written by a refused call"
        self.untouched(what)


def _p(o):
    """pointer of an Out, a tensor or None"""
    from brainmagick_b200 import _lib
    if o is None:
        return None
    return _lib.ptr(o.t if isinstance(o, Out) else o)


def _bad(what, bad, got, ref, tol):
    i = tuple(bad.nonzero()[0].tolist())
    return (f"{what}: {int(bad.sum())} of {bad.numel()} elements off, first at {list(i)}: got {got[i].item():.9g} "
            f"ref {ref[i].item():.9g} tol {tol[i].item():.3g}")


def _check(what, got, ref, tol):
    got = got.double()
    ref = torch.as_tensor(ref, dtype=torch.float64, device=DEV).expand_as(got)
    nan = torch.isnan(got)
    assert not nan.any(), f"{what}: {int(nan.sum())} of {nan.numel()} elements left unwritten (NaN)"
    tol = torch.as_tensor(tol, dtype=torch.float64, device=DEV).expand_as(ref)
    bad = (got - ref).abs() > tol
    assert not bad.any(), _bad(what, bad, got, ref, tol)


def _same(what, a, b):
    """bitwise equality of two tensors (NaN payloads included)"""
    a, b = (x.contiguous() if not isinstance(x, Out) else x.v.contiguous() for x in (a, b))
    it = IVIEW[a.dtype]
    assert torch.equal(a.view(it), b.view(it)), f"{what}: not bitwise equal"


def _refused(name, *args):
    """a call the host-side argument checks refuse, with a message"""
    from brainmagick_b200 import _lib
    lib = _lib.load()
    rc = getattr(lib, name)(*args)
    assert rc != 0, f"{name}: accepted a workspace one float short"
    assert lib.bm_last_error().decode(), f"{name}: refused without a message"


@contextlib.contextmanager
def _kernels():
    """the names of the CUDA kernels launched inside the block (torch.profiler, CUDA activity)"""
    from torch.profiler import ProfilerActivity, profile
    names = []
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        yield names
        torch.cuda.synchronize()
    names.extend(ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA)


def _profiled(family, run):
    """(run(), the kernel names it launched).  torch.profiler now and then delivers none of a session's kernel records: a
    session that recorded no kernel of `family` is repeated (run() makes fresh outputs, so the result is one whole run)"""
    for _ in range(3):
        with _kernels() as names:
            res = run()
        if _forms(names, family):
            break
    return res, names


def _forms(names, family):
    """the kernel forms among `names` for one kernel family: 'cs' (`<family>_cs_kernel`), 'v4' / 's' (the generic kernels
    with VEC = 4 / 1, or `<family>_v4_kernel` / `<family>_kernel`) and 'reduce' (the generic column reduction, one form for
    both).  `family`: 'epi', 'glu_bwd' or 'gelu_bwd'."""
    forms = set()
    for n in names:
        m = re.search(r"\b(%s\w*?)(_cs|_v4)?_kernel\b(<([^>]*)>)?" % family, n)
        if not m or "epi_param_grad" in n:
            continue
        kind, suffix, args = m.group(1), m.group(2), m.group(4)
        if suffix == "_cs":
            forms.add("cs")
        elif suffix == "_v4":
            forms.add("v4")
        elif kind == "epi_bwd_reduce":
            forms.add("reduce")
        elif family == "epi":
            vec = [a.strip() for a in args.split(",")][3]
            forms.add({"4": "v4", "1": "s"}[vec])
        else:
            forms.add("s")
    return forms


def _assert_form(names, family, want, reduced=False):
    got = _forms(names, family)
    assert got - {"reduce"} == {want}, f"{family}: ran {sorted(got)}, expected the {want} form; kernels: {names}"
    if want != "cs" and reduced:
        assert "reduce" in got, f"{family}: the generic form ran no generic column reduction; kernels: {names}"
    if want == "cs":
        assert "reduce" not in got, f"{family}: the column-stationary form ran the generic reduction; kernels: {names}"


# ---------------------------------------------------------------------------------------------------------------------
# approximated functions (common.cuh), each in fp64 with its first-order error bound
# ---------------------------------------------------------------------------------------------------------------------
# erfcc's coefficients, innermost first: Phi(-|z|) = 0.5 t exp(-ax^2 + P(t)), t = 1 / (1 + ax / 2), ax = |z| / sqrt(2)
NR_ERFCC = (0.17087277, -0.82215223, 1.48851587, -1.13520398, 0.27886807, -0.18628806, 0.09678418, 0.37409196,
            1.00002368, -1.26551223)
ERFCC_REL = 1.2e-7


def _expf_fast_rel(x):
    """relative error of __expf(x): (2 + floor(|1.173 x|)) ulp"""
    return (2 + torch.floor((1.173 * x).abs())) * 2 * U


def _gelu_parts(z):
    """gelu_parts (common.cuh) in fp64: (cdf, pdf) and their error bounds.  ax carries 2 u (the rounded 1/sqrt2 and the
    product); t = rcp.approx(fma(0.5, ax, 1)) 5 u (ax's share, the fma, 1 ulp of rcp); the Horner sum of the 10 fp32
    coefficients 18.5 u sum |c_i| t^i (18 roundings and each coefficient's own rounding) plus |P'(t)| t 5 u; the exponent
    ax^2 4 u and its fma u; __expf its ulp bound; erfcc its fractional error; 0.5 t e one rounding; 1 - Phi(-|z|) one.
    pdf = 0.3989f * __expf(-0.5f z z): u z^2 / 2 in the argument, __expf, the constant and the product."""
    ax = z.abs() / math.sqrt(2.0)
    t = 1.0 / (1.0 + 0.5 * ax)
    p = torch.zeros_like(z)
    dp = torch.zeros_like(z)
    pabs = torch.zeros_like(z)
    for c in NR_ERFCC:
        dp = dp * t + p
        p = p * t + c
        pabs = pabs * t + abs(c)
    arg = p - ax * ax
    e_t = 5 * U
    e_arg = 4 * U * ax * ax + U * arg.abs() + 18.5 * U * pabs + dp.abs() * t * e_t
    he = 0.5 * torch.special.erfc(ax)                           # Phi(-|z|)
    rel_he = e_arg + _expf_fast_rel(arg) + e_t + U + ERFCC_REL
    cdf = torch.where(z >= 0, 1.0 - he, he)
    e_cdf = he * rel_he + torch.where(z >= 0, U * cdf, 0.0)
    pdf = torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)
    e_pdf = pdf * (0.5 * U * z * z + _expf_fast_rel(0.5 * z * z) + 2 * U)
    return cdf, pdf, e_cdf, e_pdf


def _gelu(z):
    """gelu_f: (value, error bound)"""
    cdf, _, e_cdf, _ = _gelu_parts(z)
    a = z * cdf
    return a, z.abs() * e_cdf + U * a.abs()


def _gelu_grad(z):
    """gelu_grad_f = fma(z, pdf, cdf): (value, error bound)"""
    cdf, pdf, e_cdf, e_pdf = _gelu_parts(z)
    d = z * pdf + cdf
    return d, z.abs() * e_pdf + e_cdf + U * d.abs()


def _sigmoid(b, fast):
    """(sigma(b), error bound) of sigmoid_fast = rcp.approx(1 + __expf(-b)) or sigmoid_f = 1 / (1 + expf(-b)): the
    exponential's relative error enters 1 + e scaled by e / (1 + e) = 1 - sigma, then one rounding of 1 + e and the
    reciprocal (1 ulp approximate, or the IEEE division)"""
    s = torch.sigmoid(b)
    e_exp = _expf_fast_rel(b) if fast else 4 * U
    rel = e_exp * (1 - s) + U + (2 * U if fast else U)
    return s, rel * s


# =====================================================================================================================
# 1. The ConvSequence layer epilogue
# =====================================================================================================================
ACT_GELU, ACT_LRELU, ACT_NONE = 0, 1, 2
BOOST = 5.0
# shape -> (C, 1-float offset views, the form it takes)
EPI_SHAPES = {"cs-C4": (4, 0, "cs"), "cs-C320": (320, 0, "cs"), "cs-C1024": (1024, 0, "cs"),
              "v4-C1028": (1028, 0, "v4"), "s-C33": (33, 0, "s"), "s-C320-offset": (320, 1, "s")}
# around CS_ROWS_PER_BLOCK = 96, CS_U * RY (16 at C = 320) and the generic reduction's 128-row blocks
EPI_ROWS = (1, 95, 96, 97, 289, 129, 250, 257, 383)
# name -> (family, act, slope, BatchNorm, gains, x_old, mode); gains: none / scale / post / both (each given and its
# gradient asked for), grads (both NULL, dscale and dpost asked for), frozen (both given, no gradient); mode: train
# (batch_stats 1), eval (batch_stats 0 with dgamma / dbeta), frozen (batch_stats 0, no dgamma / dbeta: one elementwise pass)
EPI_VARIANTS = {
    "gelu-bn-train-xold": ("gelu", ACT_GELU, 0.0, True, "none", True, "train"),
    "gelu-bn-eval": ("gelu", ACT_GELU, 0.0, True, "none", False, "eval"),
    "gelu-bn-frozen-xold": ("gelu", ACT_GELU, 0.0, True, "none", True, "frozen"),
    "act-lrelu.1-bn-train-xold": ("act", ACT_LRELU, 0.1, True, "none", True, "train"),
    "act-relu-bn-eval": ("act", ACT_LRELU, 0.0, True, "none", False, "eval"),
    "act-none-bn-frozen-xold": ("act", ACT_NONE, 0.0, True, "none", True, "frozen"),
    "act-none-bn-train": ("act", ACT_NONE, 0.0, True, "none", False, "train"),
    "act-gelu-nobn-xold": ("act", ACT_GELU, 0.0, False, "none", True, "train"),
    "act-lrelu.1-nobn": ("act", ACT_LRELU, 0.1, False, "none", False, "train"),
    "gain-gelu-bn-scale-train-xold": ("gain", ACT_GELU, 0.0, True, "scale", True, "train"),
    "gain-lrelu.1-bn-post-eval": ("gain", ACT_LRELU, 0.1, True, "post", False, "eval"),
    "gain-none-bn-both-train-xold": ("gain", ACT_NONE, 0.0, True, "both", True, "train"),
    "gain-gelu-nobn-both": ("gain", ACT_GELU, 0.0, False, "both", False, "train"),
    "gain-relu-bn-grads-train-xold": ("gain", ACT_LRELU, 0.0, True, "grads", True, "train"),
    "gain-none-nobn-scale-xold": ("gain", ACT_NONE, 0.0, False, "scale", True, "train"),
    "gain-gelu-bn-frozen-frozen": ("gain", ACT_GELU, 0.0, True, "frozen", False, "frozen"),
    "gain-lrelu.1-nobn-grads": ("gain", ACT_LRELU, 0.1, False, "grads", False, "train"),
    "gain-relu-bn-post-frozen-xold": ("gain", ACT_LRELU, 0.0, True, "post", True, "frozen"),
}
EPI_CASES = {f"{s}-{v}-rows{EPI_ROWS[(i + 5 * j) % len(EPI_ROWS)]}": (s, v, EPI_ROWS[(i + 5 * j) % len(EPI_ROWS)])
             for j, s in enumerate(EPI_SHAPES) for i, v in enumerate(EPI_VARIANTS)}
EPI_CASES["real-cs-C320-gelu-bn-train-xold-rows23040"] = ("cs-C320", "gelu-bn-train-xold", 64 * 360)


class EpiCase:
    """the operands of one epilogue case (fp32, on the device, at the shape's offset) and its fp64 reference"""

    def __init__(self, shape, variant, rows, seed):
        C, off, self.form = EPI_SHAPES[shape]
        (self.family, self.act, self.slope, self.bn, gains, xold, self.mode) = EPI_VARIANTS[variant]
        self.rows, self.C, self.off = rows, C, off
        gen = _gen(seed)
        mu = _rand(gen, C, scale=2.0)
        sd = 0.5 + 1.5 * torch.rand(C, generator=gen, device=DEV)
        d = dict(y=_rand(gen, rows, C) * sd + mu, g=_rand(gen, rows, C))
        if self.bn:
            d.update(mean=mu + _rand(gen, C, scale=0.1), invstd=1.0 / sd, gamma=1.0 + _rand(gen, C, scale=0.3),
                     beta=_rand(gen, C, scale=0.3))
        if gains in ("scale", "both", "frozen"):
            d["scale"] = _rand(gen, C, scale=0.1)
        if gains in ("post", "both", "frozen"):
            d["post"] = _rand(gen, C)
        if xold:
            d["x_old"] = _rand(gen, rows, C)
        self.d = {k: _dev(v, off) for k, v in d.items()}
        self.want_dscale = gains in ("scale", "both", "grads")
        self.want_dpost = gains in ("post", "both", "grads")
        self.gain = gains != "none"
        self.batch_stats = 1 if self.mode == "train" else 0
        self.want_bn_grads = self.bn and self.mode != "frozen"
        self.reduces = self.want_bn_grads or self.want_dscale or self.want_dpost
        self.W = (3 if self.gain else 2) * C
        self._reference()

    def get(self, k):
        return self.d.get(k)

    def _reference(self):
        """fp64 forward, sums, parameter gradients and dy with their first-order error bounds (module docstring)"""
        d = {k: v.double() for k, v in self.d.items()}
        y, g = d["y"], d["g"]
        n = self.rows
        if self.bn:
            yh = (y - d["mean"]) * d["invstd"]
            z = yh * d["gamma"] + d["beta"]
            e_yh = 2 * U * yh.abs()                                  # y - mean, * invstd
            e_z = d["gamma"].abs() * e_yh + U * ((yh * d["gamma"]).abs() + z.abs())
        else:
            yh, e_yh = None, None
            z, e_z = y, torch.zeros_like(y)
        if self.act == ACT_GELU:
            a, e_a = _gelu(z)
            e_a = e_a + 1.13 * e_z                                   # |GELU'| <= 1.13
            da, e_da = _gelu_grad(z)
            e_da = e_da + 0.8 * e_z                                  # |GELU''| <= 2 phi(0) < 0.8
        elif self.act == ACT_LRELU:
            s = self.slope
            a = torch.where(z > 0, z, z * s)
            e_a = max(1.0, abs(s)) * e_z + U * a.abs()
            da = torch.where(z > 0, 1.0, s)
            e_da = torch.where(z.abs() <= e_z, abs(1.0 - s), 0.0)    # z's rounding may cross the kink
        else:
            a, e_a = z, e_z
            da, e_da = torch.ones_like(z), torch.zeros_like(z)
        ks = BOOST * d["scale"] if "scale" in d else torch.ones(self.C, dtype=torch.float64, device=DEV)
        kp = d["post"] if "post" in d else torch.ones(self.C, dtype=torch.float64, device=DEV)
        ng = 2 * ("scale" in d) + ("post" in d)                      # boost * scale, * branch, post * (...)
        k = ks * kp
        branch = k * a
        x = branch + d["x_old"] if "x_old" in d else branch
        self.x_ref = x
        self.x_tol = K_EPI * (k.abs() * e_a + ng * U * branch.abs() + ("x_old" in d) * U * x.abs()) + TINY
        gb = k * g
        e_gb = ng * U * gb.abs()
        dz = gb * da
        e_dz = gb.abs() * e_da + da.abs() * e_gb + U * dz.abs()
        self.S = [dz.sum(0), (dz * yh).sum(0) if self.bn else None, (g * a).sum(0)]
        eS1 = e_dz.sum(0) + _gamma(n) * dz.abs().sum(0)
        eS2 = ((e_dz * yh.abs() + dz.abs() * e_yh).sum(0) + _gamma(n + 1) * (dz * yh).abs().sum(0)) if self.bn else None
        eS3 = (g.abs() * e_a).sum(0) + _gamma(n + 1) * (g * a).abs().sum(0)
        self.eS = [eS1, eS2, eS3]
        if self.want_dscale or self.want_dpost:
            pst = d["post"] if "post" in d else 1.0
            self.dscale = BOOST * pst * self.S[2]
            self.e_dscale = K_EPI * (BOOST * abs(pst) * eS3 + U * self.dscale.abs()) + TINY
            self.dpost = ks * self.S[2]
            self.e_dpost = K_EPI * (ks.abs() * eS3 + 2 * U * self.dpost.abs()) + TINY
        if not self.bn:
            self.dy, self.e_dy = dz, K_EPI * e_dz + TINY
            return
        kk = d["gamma"] * d["invstd"]
        if self.batch_stats:
            m1, m2 = self.S[0] / n, self.S[1] / n
            e_m1 = eS1 / n + 3 * U * m1.abs()                        # (float) sum, (float)(1 / n) or / n, the product
            e_m2 = eS2 / n + 3 * U * m2.abs()
            v = dz - m1 - yh * m2
            e_v = (e_dz + e_m1 + yh.abs() * e_m2 + m2.abs() * e_yh
                   + 3 * U * (dz.abs() + m1.abs() + (yh * m2).abs()))
        else:
            v, e_v = dz, e_dz
        self.dy = kk * v
        self.e_dy = K_EPI * (kk.abs() * e_v + 2 * U * self.dy.abs()) + TINY

    def check_sums(self, what, sums):
        """the kernel's fp64 sums [W]: (sum dz, sum dz*yhat) with a BatchNorm (0 without), S with the gains"""
        C = self.C
        s = sums.v if isinstance(sums, Out) else sums
        if self.bn:   # the reduction computes them whenever it runs with a BatchNorm
            _check(what + " sum dz", s[:C], self.S[0], K_EPI * self.eS[0] + TINY)
            _check(what + " sum dz*yhat", s[C:2 * C], self.S[1], K_EPI * self.eS[1] + TINY)
        elif not self.bn:
            assert (s[:2 * C] == 0).all(), f"{what}: BatchNorm sums without a BatchNorm"
        if self.gain and (self.want_dscale or self.want_dpost):
            _check(what + " S", s[2 * C:3 * C], self.S[2], K_EPI * self.eS[2] + TINY)

    def check_param_grads(self, what, dgamma, dbeta, dscale=None, dpost=None):
        if dbeta is not None:
            _check(what + " dbeta", dbeta.v, self.S[0], K_EPI * (self.eS[0] + U * self.S[0].abs()) + TINY)
            _check(what + " dgamma", dgamma.v, self.S[1], K_EPI * (self.eS[1] + U * self.S[1].abs()) + TINY)
            dgamma.untouched(what + " dgamma")
            dbeta.untouched(what + " dbeta")
        if dscale is not None:
            _check(what + " dscale", dscale.v, self.dscale, self.e_dscale)
            dscale.untouched(what + " dscale")
        if dpost is not None:
            _check(what + " dpost", dpost.v, self.dpost, self.e_dpost)
            dpost.untouched(what + " dpost")


def _epi_fwd(c, x_new, amax):
    call, _, stream = _abi()
    g = c.get
    common = (_p(g("y")), _p(g("mean")), _p(g("invstd")), _p(g("gamma")), _p(g("beta")), _p(g("x_old")), _p(x_new),
              c.rows, c.C)
    if c.family == "gelu":
        call("bm_bn_gelu_skip_fwd", *common, _p(amax), stream())
    elif c.family == "act":
        call("bm_bn_act_skip_fwd", *common, c.act, c.slope, stream())
    else:
        call("bm_bn_act_gain_skip_fwd", *common, c.act, c.slope, _p(g("scale")), BOOST, _p(g("post")), stream())


def _epi_bwd_args(c, o, det, ws=None, ws_floats=0):
    """(entry point, arguments) of the fused backward into the outputs `o` (dict of Out / None)"""
    _, _, stream = _abi()
    g = c.get
    head = (_p(g("g")), _p(g("y")), _p(g("mean")), _p(g("invstd")), _p(g("gamma")), _p(g("beta")), c.batch_stats,
            c.rows, c.C)
    tail = ((_p(ws), ws_floats) if det else ()) + (stream(),)
    if c.family == "gelu":
        name = "bm_bn_gelu_skip_bwd"
        args = head + (_p(o["sums"]), _p(o["dy"]), _p(o["dgamma"]), _p(o["dbeta"]), _p(o["amax"])) + tail
    elif c.family == "act":
        name = "bm_bn_act_skip_bwd"
        args = head + (c.act, c.slope, _p(o["sums"]), _p(o["dy"]), _p(o["dgamma"]), _p(o["dbeta"])) + tail
    else:
        name = "bm_bn_act_gain_skip_bwd"
        args = head + (c.act, c.slope, _p(g("scale")), BOOST, _p(g("post")), _p(o["sums"]), _p(o["dy"]),
                       _p(o["dgamma"]), _p(o["dbeta"]), _p(o["dscale"]), _p(o["dpost"])) + tail
    return name + ("_det" if det else ""), args


def _epi_outputs(c):
    o = dict(dy=Out(c.rows, c.C, off=c.off),
             dgamma=Out(c.C, off=c.off) if c.want_bn_grads else None,
             dbeta=Out(c.C, off=c.off) if c.want_bn_grads else None,
             dscale=Out(c.C) if c.want_dscale else None, dpost=Out(c.C) if c.want_dpost else None,
             sums=Out(c.W + 1, dtype=torch.float64) if c.reduces else None,
             amax=Out(1) if c.family == "gelu" else None)
    return o


def _check_bwd(c, what, o):
    _check(what + " dy", o["dy"].v, c.dy, c.e_dy)
    o["dy"].untouched(what + " dy")
    if c.reduces:
        c.check_sums(what, o["sums"].v[:c.W])
        o["sums"].untouched(what + " sums")
    c.check_param_grads(what, o["dgamma"], o["dbeta"], o["dscale"], o["dpost"])
    if o["amax"] is not None:
        _same(what + " amax", o["amax"].v[0], o["dy"].v.abs().max())
        o["amax"].untouched(what + " amax")


def _ws_query(c, name):
    from brainmagick_b200 import _lib
    return int(getattr(_lib.load(), name + "_workspace")(c.rows, c.C))


@pytest.mark.parametrize("case", list(EPI_CASES))
def test_layer_epilogue(case):
    shape, variant, rows = EPI_CASES[case]
    c = EpiCase(shape, variant, rows, seed=1000 + len(case) * 7 + rows)
    call, _, stream = _abi()
    train_pair = c.bn and c.mode == "train" and not c.gain       # the _reduce / _apply halves exist for this contract
    def run():
        # forward
        x_new, amax = Out(rows, c.C, off=c.off), (Out(1) if c.family == "gelu" else None)
        _epi_fwd(c, x_new, amax)
        # fused backward, atomic form
        o = _epi_outputs(c)
        name, args = _epi_bwd_args(c, o, det=False)
        call(name, *args)
        # deterministic form: a NaN workspace and a random one (nothing reduced: no workspace at all)
        det = []
        need = _ws_query(c, name + "_det") if c.reduces else 0
        for fill in ("nan", "rand"):
            od = _epi_outputs(c)
            ws = None
            if c.reduces:
                ws = torch.full((need,), float("nan"), device=DEV) if fill == "nan" else torch.randn(need, device=DEV)
            dname, dargs = _epi_bwd_args(c, od, det=True, ws=ws, ws_floats=need)
            call(dname, *dargs)
            det.append(od)
        if c.reduces:   # one float short: refused, nothing written
            orf = _epi_outputs(c)
            ws = torch.zeros(need, device=DEV)
            rname, rargs = _epi_bwd_args(c, orf, det=True, ws=ws, ws_floats=need - 1)
            _refused(rname, *rargs)
        # the SyncBatchNorm halves: _reduce(_det), then _apply on sums [2C + 1] with sums[2C] = n
        if train_pair:
            fam = "bm_bn_gelu_skip" if c.family == "gelu" else "bm_bn_act_skip"
            actargs = () if c.family == "gelu" else (c.act, c.slope)
            g = c.get
            ops = (_p(g("g")), _p(g("y")), _p(g("mean")), _p(g("invstd")), _p(g("gamma")), _p(g("beta")), c.rows, c.C)
            halves = []
            rneed = _ws_query(c, fam + "_bwd_reduce_det")
            for det_form in (False, True, True):
                h = dict(sums=Out(2 * c.C + 1, dtype=torch.float64), dgamma=Out(c.C, off=c.off),
                         dbeta=Out(c.C, off=c.off), dy=Out(rows, c.C, off=c.off))
                rargs = ops + actargs + (_p(h["sums"]), _p(h["dgamma"]), _p(h["dbeta"]))
                if det_form:
                    fill = "nan" if len(halves) == 1 else "rand"
                    ws = torch.full((rneed,), float("nan"), device=DEV) if fill == "nan" else torch.randn(rneed, device=DEV)
                    call(fam + "_bwd_reduce_det", *rargs, _p(ws), rneed, stream())
                else:
                    call(fam + "_bwd_reduce", *rargs, stream())
                h["sums"].v[2 * c.C] = float(rows)
                call(fam + "_bwd_apply", *ops, *actargs, _p(h["sums"]), _p(h["dy"]), stream())
                halves.append(h)
            hr = dict(sums=Out(2 * c.C + 1, dtype=torch.float64), dgamma=Out(c.C, off=c.off), dbeta=Out(c.C, off=c.off))
            _refused(fam + "_bwd_reduce_det", *ops, *actargs, _p(hr["sums"]), _p(hr["dgamma"]), _p(hr["dbeta"]),
                     _p(torch.zeros(rneed, device=DEV)), rneed - 1, stream())
        return (x_new, amax, o, det, orf if c.reduces else None, halves if train_pair else None,
                hr if train_pair else None)

    (x_new, amax, o, det, orf, halves, hr), names = _profiled("epi", run)
    torch.cuda.synchronize()
    _assert_form(names, "epi", c.form, reduced=c.reduces)

    _check("x_new", x_new.v, c.x_ref, c.x_tol)
    x_new.untouched("x_new")
    if amax is not None:
        _same("forward amax", amax.v[0], x_new.v.abs().max())
        amax.untouched("forward amax")
    _check_bwd(c, "bwd", o)
    _check_bwd(c, "bwd_det", det[0])
    for k in det[0]:
        if det[0][k] is not None:
            _same(f"bwd_det {k}: NaN workspace vs random workspace", det[0][k].v, det[1][k].v)
    if c.reduces:
        for k, v in orf.items():
            if v is not None:
                v.unwritten(f"refused bwd_det {k}")
    if train_pair:
        for i, h in enumerate(halves):
            what = ("_bwd_reduce", "_bwd_reduce_det", "_bwd_reduce_det (random workspace)")[i]
            c.check_sums(what, h["sums"].v[:2 * c.C])
            c.check_param_grads(what, h["dgamma"], h["dbeta"])
            _check(what + " + _bwd_apply dy", h["dy"].v, c.dy, c.e_dy)
            h["dy"].untouched(what + " + _bwd_apply dy")
        # the deterministic halves give the fused deterministic backward's bits
        for h in halves[1:]:
            _same("_bwd_reduce_det sums vs bwd_det", h["sums"].v[:2 * c.C], det[0]["sums"].v[:2 * c.C])
            _same("_bwd_reduce_det dgamma vs bwd_det", h["dgamma"], det[0]["dgamma"])
            _same("_bwd_reduce_det dbeta vs bwd_det", h["dbeta"], det[0]["dbeta"])
            _same("_bwd_reduce_det + _bwd_apply dy vs bwd_det", h["dy"], det[0]["dy"])
        for k in ("sums", "dgamma", "dbeta"):
            hr[k].unwritten(f"refused _bwd_reduce_det {k}")
        # _apply on the fused call's own sums gives its bits (whichever order the atomics took)
        h = dict(dy=Out(rows, c.C, off=c.off))
        s = o["sums"].v.clone()
        s[2 * c.C] = float(rows)
        g = c.get
        call(("bm_bn_gelu_skip" if c.family == "gelu" else "bm_bn_act_skip") + "_bwd_apply", _p(g("g")), _p(g("y")),
             _p(g("mean")), _p(g("invstd")), _p(g("gamma")), _p(g("beta")), c.rows, c.C,
             *(() if c.family == "gelu" else (c.act, c.slope)), _p(s), _p(h["dy"]), stream())
        torch.cuda.synchronize()
        _same("_bwd_apply on bwd's sums vs bwd dy", h["dy"], o["dy"])


def test_layer_epilogue_forms_all_occur():
    """every epilogue family runs on each of the three forms in the cases above"""
    seen = {}
    for shape, variant, _ in EPI_CASES.values():
        seen.setdefault(EPI_VARIANTS[variant][0], set()).add(EPI_SHAPES[shape][2])
    assert seen == {f: {"cs", "v4", "s"} for f in ("gelu", "act", "gain")}, seen


# =====================================================================================================================
# 2. BatchNorm finalize
# =====================================================================================================================
BN_EPS = 1e-5


def _bn_stats(gen, n, C):
    """y [n, C] and its fp64 sums; column 0's sums are replaced by ones whose variance rounds below zero (the clamp)"""
    mu = _rand(gen, C)
    sd = 0.5 + 1.5 * torch.rand(C, generator=gen, device=DEV)
    y = _rand(gen, n, C) * sd + mu
    S, Q = y.double().sum(0), (y.double() ** 2).sum(0)
    S[0] = 3.0 * n
    Q[0] = 9.0 * n * (1 - 2.0 ** -40)
    return y, S, Q


@pytest.mark.parametrize("C", [1, 127, 128, 129])
@pytest.mark.parametrize("entry", ["bm_bn_stats_finalize", "bm_bn_stats_finalize_counted",
                                   "bm_bn_stats_finalize_cumulative", "bm_bn_stats_finalize_counted_cumulative"])
def test_bn_finalize(entry, C):
    """mean = S / n, var = max(Q / n - mean^2, 0), invstd = 1 / sqrt(var + eps) in fp64, each rounded once; the running
    statistics (1 - m) r + m x in fp32 with the unbiased variance var n / (n - 1) (var itself at n = 1), against the formulas
    and against torch.nn.BatchNorm1d's update in fp64 on the CPU"""
    call, ptr, stream = _abi()
    counted = "counted" in entry
    cumulative = entry.endswith("cumulative")
    gen = _gen(20 + C)
    settings = [(1, None), (7, None)] if cumulative else [(m, nul) for m in (0.0, 0.1, 1.0) for nul in (False, True)]
    for n in (1, 7, 360):
        y, S, Q = _bn_stats(gen, n, C)
        stats = torch.cat([S, Q, torch.tensor([float(n)], dtype=torch.float64, device=DEV)])
        m = S / n
        var_raw = Q / n - m * m
        var = var_raw.clamp_min(0)
        assert var_raw[0] < 0
        e_var = 4 * UD * (Q / n + m * m)
        inv = 1 / torch.sqrt(var + float(torch.tensor(BN_EPS, dtype=torch.float32)))
        for setting, null in settings:
            rm0 = _rand(gen, C)
            rv0 = 0.5 + torch.rand(C, generator=gen, device=DEV)
            rm, rv = Out(C), Out(C)
            rm.v.copy_(rm0)
            rv.v.copy_(rv0)
            mean, invstd = Out(C), Out(C)
            nbt = torch.tensor([setting], dtype=torch.int64, device=DEV) if cumulative else None
            run = (None, None) if null else (ptr(rm.t), ptr(rv.t))
            eps = BN_EPS
            if entry == "bm_bn_stats_finalize":
                call(entry, ptr(stats), n, eps, setting, *run, ptr(mean.t), ptr(invstd.t), C, stream())
            elif entry == "bm_bn_stats_finalize_counted":
                call(entry, ptr(stats), eps, setting, *run, ptr(mean.t), ptr(invstd.t), C, stream())
            elif entry == "bm_bn_stats_finalize_cumulative":
                call(entry, ptr(stats), n, eps, ptr(nbt), *run, ptr(mean.t), ptr(invstd.t), C, stream())
            else:
                call(entry, ptr(stats), eps, ptr(nbt), *run, ptr(mean.t), ptr(invstd.t), C, stream())
            torch.cuda.synchronize()
            what = f"{entry} C={C} n={n} setting={setting} null={null}"
            _check(what + " mean", mean.v, m, K_BN * (U * m.abs() + 2 * UD * m.abs()) + TINY)
            _check(what + " invstd", invstd.v, inv, K_BN * (U * inv + 0.5 * inv ** 3 * e_var) + TINY)
            mean.untouched(what + " mean")
            invstd.untouched(what + " invstd")
            if null:
                _same(what + " running_mean untouched", rm.v, rm0)
                continue
            mom = 1.0 / setting if cumulative else setting
            momf = float(torch.tensor(mom, dtype=torch.float32))       # the kernel's float momentum
            unb = var * n / (n - 1) if n > 1 else var
            e_unb = U * unb + e_var * (n / (n - 1) if n > 1 else 1.0)
            rm0d, rv0d = rm0.double(), rv0.double()
            ref_m = (1 - mom) * rm0d + mom * m
            ref_v = (1 - mom) * rv0d + mom * unb
            tol_m = K_BN * (3 * U * ((1 - momf) * rm0d.abs() + momf * m.abs()) + abs(momf - mom) * (rm0d.abs() + m.abs())
                            + U * ref_m.abs()) + TINY
            tol_v = K_BN * (3 * U * ((1 - momf) * rv0d.abs() + momf * unb) + momf * e_unb
                            + abs(momf - mom) * (rv0d.abs() + unb) + U * ref_v.abs()) + TINY
            _check(what + " running_mean", rm.v, ref_m, tol_m)
            _check(what + " running_var", rv.v, ref_v, tol_v)
            rm.untouched(what + " running_mean")
            rv.untouched(what + " running_var")
            if n > 1 and C > 1:    # torch.nn.BatchNorm1d's own update (column 0's sums are synthetic: not comparable)
                bn = torch.nn.BatchNorm1d(C, eps=BN_EPS, momentum=None if cumulative else mom).double()
                bn.running_mean.copy_(rm0d.cpu())
                bn.running_var.copy_(rv0d.cpu())
                if cumulative:
                    bn.num_batches_tracked.fill_(setting - 1)
                bn.train()
                with torch.no_grad():
                    bn(y.double().cpu())
                tm = bn.running_mean.to(DEV)
                tv = bn.running_var.to(DEV)
                # torch takes the variance in two passes: the two fp64 variances differ by a few n 2^-53 (Q / n + m^2)
                e64 = 4 * n * UD * (Q / n + m * m)
                _check(what + " running_mean vs BatchNorm1d", rm.v[1:], tm[1:], tol_m[1:] + e64[1:])
                _check(what + " running_var vs BatchNorm1d", rv.v[1:], tv[1:], tol_v[1:] + e64[1:])


@pytest.mark.parametrize("C", [1, 127, 128, 129])
def test_bn_eval_stats(C):
    """mean = running_mean bit for bit, invstd = 1 / sqrtf(running_var + eps): three roundings"""
    call, ptr, stream = _abi()
    gen = _gen(30 + C)
    rm = _rand(gen, C)
    rv = torch.rand(C, generator=gen, device=DEV) * 4
    rv[0] = 0.0
    mean, invstd = Out(C), Out(C)
    call("bm_bn_eval_stats", ptr(rm), ptr(rv), BN_EPS, ptr(mean.t), ptr(invstd.t), C, stream())
    torch.cuda.synchronize()
    _same("mean", mean.v, rm)
    ref = 1 / torch.sqrt(rv.double() + float(torch.tensor(BN_EPS, dtype=torch.float32)))
    _check("invstd", invstd.v, ref, K_BN * 3 * U * ref + TINY)
    mean.untouched("mean")
    invstd.untouched("invstd")


# =====================================================================================================================
# 3. Column reductions
# =====================================================================================================================
@pytest.mark.parametrize("rows", [1, 127, 128, 129, 255, 256, 257])
@pytest.mark.parametrize("entry", ["bm_col_stats", "bm_col_stats_det", "bm_col_sum", "bm_col_sum_det"])
def test_col_reductions(entry, rows):
    """bm_col_stats(_det): fp64 sums of y and y^2 (fp64 per thread), gamma_n sum|.| in fp64 units; bm_col_sum(_det): fp32
    sums, gamma_n sum|y| in fp32 units"""
    from brainmagick_b200 import _lib
    call, ptr, stream = _abi()
    stats_form = entry.startswith("bm_col_stats")
    det = entry.endswith("_det")
    for C in (1, 127, 128, 129):
        y = _rand(_gen(40 + rows + C), rows, C) + 3.0
        yd = y.double()
        width = 2 * C if stats_form else C
        dtype = torch.float64 if stats_form else torch.float32
        outs = []
        need = int(getattr(_lib.load(), entry + "_workspace")(rows, C)) if det else 0
        for fill in (("nan", "rand") if det else ("",)):
            out = Out(width, dtype=dtype)
            if det:
                ws = torch.full((need,), float("nan"), device=DEV) if fill == "nan" else torch.randn(need, device=DEV)
                call(entry, ptr(y), rows, C, ptr(ws), need, ptr(out.t), stream())
            else:
                call(entry, ptr(y), rows, C, ptr(out.t), stream())
            outs.append(out)
        torch.cuda.synchronize()
        what = f"{entry} rows={rows} C={C}"
        out = outs[0]
        if stats_form:
            eps = K_RED * (rows + 2) * UD
            q = (yd * yd).sum(0)
            _check(what + " sum", out.v[:C], yd.sum(0), eps * yd.abs().sum(0) + TINY)
            _check(what + " sumsq", out.v[C:], q, eps * q + TINY)
        else:
            _check(what, out.v, yd.sum(0), K_RED * _gamma(rows) * yd.abs().sum(0) + TINY)
        out.untouched(what)
        if det:
            _same(what + ": NaN workspace vs random workspace", outs[0], outs[1])
            refused = Out(width, dtype=dtype)
            _refused(entry, ptr(y), rows, C, ptr(torch.zeros(need, device=DEV)), need - 1, ptr(refused.t), stream())
            torch.cuda.synchronize()
            refused.unwritten(what + " refused")


# =====================================================================================================================
# 4. GLU and GELU backward
# =====================================================================================================================
# name -> (H, 1-float offset views, form); the column-stationary form uses sigmoid_fast, the generic ones sigmoid_f
GLU_SHAPES = {"cs-H4": (4, 0, "cs"), "cs-H80": (80, 0, "cs"), "cs-H160": (160, 0, "cs"), "v4-H1028": (1028, 0, "v4"),
              "s-H7": (7, 0, "s"), "s-H80-offset": (80, 1, "s")}
GLU_CASES = {f"{s}-rows{r}": (s, r) for s in GLU_SHAPES for r in (1, 95, 97, 289)}
GLU_CASES["real-cs-H160-rows23040"] = ("cs-H160", 64 * 360)


@pytest.mark.parametrize("case", list(GLU_CASES))
def test_glu_bwd(case):
    """dh_a = g sigma(b), dh_b = g a sigma(b) (1 - sigma(b)) against fp64 sigma, with sigma's bound (_sigmoid): the gate
    inputs reach |b| = 30, where 1 - sigma rounds to 0 in fp32.  dbias against the fp64 column sums of the REFERENCE dh;
    amax_out = max |dh| bit for bit"""
    from brainmagick_b200 import _lib
    call, ptr, stream = _abi()
    shape, rows = GLU_CASES[case]
    H, off, form = GLU_SHAPES[shape]
    gen = _gen(50 + H + rows)
    h = _rand(gen, rows, 2 * H)
    b = h[:, H:]
    b.mul_(4.0)
    for i, v in enumerate((30.0, -30.0, 20.0, -20.0, 0.0, 12.0, -12.0)):
        b[i % rows, (3 * i) % H] = v
    g = _rand(gen, rows, H)
    hd, gd = _dev(h, off), _dev(g, off)
    a64, b64, g64 = h[:, :H].double(), h[:, H:].double(), g.double()
    s, e_s = _sigmoid(b64, fast=form == "cs")
    da = g64 * s
    db = g64 * a64 * s * (1 - s)
    ref = torch.cat([da, db], 1)
    tol = torch.cat([g64.abs() * e_s + U * da.abs(), (g64 * a64).abs() * e_s + 4 * U * db.abs()], 1)
    need = int(_lib.load().bm_glu_bwd_det_workspace(rows, H))
    def run():
        runs = []
        for det, fill in ((False, ""), (True, "nan"), (True, "rand")):
            dh, dbias, amax = Out(rows, 2 * H, off=off), Out(2 * H), Out(1)
            if det:
                ws = torch.full((need,), float("nan"), device=DEV) if fill == "nan" else torch.randn(need, device=DEV)
                call("bm_glu_bwd_det", ptr(gd), ptr(hd), rows, H, ptr(dh.t), ptr(dbias.t), ptr(amax.t), ptr(ws), need,
                     stream())
            else:
                call("bm_glu_bwd", ptr(gd), ptr(hd), rows, H, ptr(dh.t), ptr(dbias.t), ptr(amax.t), stream())
            runs.append((dh, dbias, amax))
        nob = Out(rows, 2 * H, off=off)          # no bias gradient: no workspace
        call("bm_glu_bwd_det", ptr(gd), ptr(hd), rows, H, ptr(nob.t), None, None, None, 0, stream())
        rdh, rdb = Out(rows, 2 * H, off=off), Out(2 * H)
        _refused("bm_glu_bwd_det", ptr(gd), ptr(hd), rows, H, ptr(rdh.t), ptr(rdb.t), None,
                 ptr(torch.zeros(need, device=DEV)), need - 1, stream())
        return runs, nob, rdh, rdb

    (runs, nob, rdh, rdb), names = _profiled("glu_bwd", run)
    torch.cuda.synchronize()
    _assert_form(names, "glu_bwd", form)
    for i, (dh, dbias, amax) in enumerate(runs):
        what = ("bm_glu_bwd", "bm_glu_bwd_det", "bm_glu_bwd_det (random workspace)")[i]
        _check(what + " dh", dh.v, ref, K_GLU * tol + TINY)
        _check(what + " dbias", dbias.v, ref.sum(0), K_GLU * (tol.sum(0) + _gamma(rows) * ref.abs().sum(0)) + TINY)
        _same(what + " amax", amax.v[0], dh.v.abs().max())
        for o, nm in ((dh, "dh"), (dbias, "dbias"), (amax, "amax")):
            o.untouched(f"{what} {nm}")
    for k in range(3):
        _same("bm_glu_bwd_det NaN vs random workspace", runs[1][k], runs[2][k])
    _same("bm_glu_bwd_det without dbias: dh", nob, runs[1][0])
    rdh.unwritten("refused bm_glu_bwd_det dh")
    rdb.unwritten("refused bm_glu_bwd_det dbias")


def test_glu_forms_all_occur():
    assert {GLU_SHAPES[s][2] for s, _ in GLU_CASES.values()} == {"cs", "v4", "s"}


GELU_SPECIALS = (0.0, 1e-30, -1e-30, 5.0, -5.0, -12.0, 12.0, 1.0, -1.0, 0.5)
# name -> (n, offset, form)
GELU_CASES = {"v4-n4096": (4096, 0, "v4"), "s-n4099": (4099, 0, "s"), "s-n4096-offset": (4096, 1, "s"),
              "s-n10": (10, 0, "s"), "v4-n12": (12, 0, "v4")}


@pytest.mark.parametrize("case", list(GELU_CASES))
def test_gelu_bwd(case):
    """dh = dq GELU'(h) against fp64 Phi and phi with GELU's bound (_gelu_parts); h includes 0, +-1e-30, +-5 and -12"""
    call, ptr, stream = _abi()
    n, off, form = GELU_CASES[case]
    gen = _gen(60 + n + off)
    h = _rand(gen, n, scale=3.0)
    sp = torch.tensor(GELU_SPECIALS, device=DEV)
    h[:min(n, sp.numel())] = sp[:min(n, sp.numel())]
    dq = _rand(gen, n)
    hd, dqd = _dev(h, off), _dev(dq, off)
    def run():
        dh = Out(n, off=off)
        call("bm_gelu_bwd", ptr(dqd), ptr(hd), n, ptr(dh.t), stream())
        return dh

    dh, names = _profiled("gelu_bwd", run)
    _assert_form(names, "gelu_bwd", form)
    d, e_d = _gelu_grad(h.double())
    ref = dq.double() * d
    _check("dh", dh.v, ref, K_GLU * (dq.double().abs() * e_d + U * ref.abs()) + TINY)
    dh.untouched("dh")


# =====================================================================================================================
# 5. Attention pieces
# =====================================================================================================================
def _ulp(x):
    """one ulp of the fp32 value nearest each fp64 x"""
    _, e = torch.frexp(x)
    return torch.where(x == 0, 2.0 ** -149, torch.ldexp(torch.ones_like(x), (e - 24).clamp_min(-149)))


@pytest.mark.parametrize("P", [2, 8, 2048])
def test_fourier_emb(P):
    """loc = (x + 0.2) f[k] + (y + 0.2) f[l] bit for bit torch's fp32 result in that operation order; cos / sin within
    sincosf's 2 ulp of fp64 cos / sin of that loc"""
    call, ptr, stream = _abi()
    n = int(round(math.sqrt(P // 2)))
    R, C = 2, (273 if P == 2048 else 33)
    gen = _gen(70 + P)
    pos = torch.rand(R, C, 2, generator=gen, device=DEV)
    pos[0, 0] = -0.1
    freq = 2 * math.pi * torch.arange(n, device=DEV, dtype=torch.float32) / 1.4
    emb = Out(R, C, P)
    call("bm_fourier_emb", ptr(pos), ptr(freq), R, C, P, ptr(emb.t), stream())
    torch.cuda.synchronize()
    margin = torch.tensor(0.2, dtype=torch.float32, device=DEV)
    x, y = pos[..., 0] + margin, pos[..., 1] + margin
    loc = ((x[..., None] * freq)[..., :, None] + (y[..., None] * freq)[..., None, :]).reshape(R, C, n * n).double()
    half = n * n
    for what, got, ref in (("cos", emb.v[..., :half], torch.cos(loc)), ("sin", emb.v[..., half:], torch.sin(loc))):
        _check(what, got, ref, 2 * _ulp(ref))
    emb.untouched("emb")


@pytest.mark.parametrize("C", [1, 31, 32, 33, 273])
@pytest.mark.parametrize("ban", [False, True], ids=["eval", "train-ban"])
def test_masked_softmax(C, ban):
    """softmax over c of scores with -inf on invalid sensors (-0.1, -0.1) and, in training, on sensors within `radius` of
    the ban centre (<=, bm_oracle.attention_weights): sensor 1 sits exactly at the radius (offset (3/16, 4/16), radius 5/16,
    all exact in fp32).  R * O = 15 rows: not a multiple of the 8 warps per block"""
    call, ptr, stream = _abi()
    R, O = 3, 5
    gen = _gen(80 + C)
    pos = torch.rand(R, C, 2, generator=gen, device=DEV)
    centre = torch.tensor([0.5, 0.5], device=DEV)
    radius = 5.0 / 16
    if C > 1:
        pos[:, 1] = centre + torch.tensor([3.0 / 16, 4.0 / 16], device=DEV)
        pos[:, 0] = -0.1
    if C > 2:
        pos[1, 2] = centre + torch.tensor([-0.1, 0.05], device=DEV)           # inside
        pos[2, 2] = centre + torch.tensor([0.0, 5.0 / 16 + 2.0 ** -20], device=DEV)   # just outside
    pos[:, -1] = torch.tensor([0.95, 0.95], device=DEV)                       # every row keeps a valid sensor
    scores = _rand(gen, R, O, C, scale=3.0)
    w = _dev(scores)
    call("bm_masked_softmax", ptr(w), ptr(pos), ptr(centre) if ban else None, radius, R, O, C, stream())
    torch.cuda.synchronize()
    masked = (pos[..., 0] == -0.1) & (pos[..., 1] == -0.1)
    if ban:   # the kernel's fp32 distance: products and their sum rounded separately, IEEE sqrt
        dxy = pos - centre
        masked = masked | (torch.sqrt(dxy[..., 0] * dxy[..., 0] + dxy[..., 1] * dxy[..., 1]) <= radius)
        if C > 1:
            assert masked[:, 1].all()
        if C > 2:
            assert masked[1, 2] and not masked[2, 2]
    valid = ~masked[:, None, :]
    s = scores.double().masked_fill(~valid, -math.inf)
    ref = torch.softmax(s, -1)
    # each term: u |s - max| in the exponent's argument and 2 ulp (4 u) of expf; their sum: the largest such term error
    # plus (C - 1) u for adding C positive terms; then the reciprocal and the scale, one rounding each
    d = (s - s.max(-1, keepdim=True).values).abs().nan_to_num(0.0, posinf=0.0)
    rel = U * (d + d.amax(-1, keepdim=True)) + (C + 10) * U
    _check("weights", w, ref, K_ATT * rel * ref + TINY)
    assert (w[~valid.expand_as(w)] == 0).all(), "masked entries are not exactly 0"


@pytest.mark.parametrize("C", [1, 31, 32, 33, 273])
def test_softmax_bwd(C):
    """dscores = w (dw - sum_c w dw): the dot errs by (C + 1) u sum |w dw|, then one rounding each for the difference and
    the product"""
    call, ptr, stream = _abi()
    rows = 15
    gen = _gen(90 + C)
    w = torch.softmax(_rand(gen, rows, C), -1)
    dw = _rand(gen, rows, C)
    ds = Out(rows, C)
    call("bm_softmax_bwd", ptr(w), ptr(dw), rows, C, ptr(ds.t), stream())
    torch.cuda.synchronize()
    wd, dwd = w.double(), dw.double()
    dot = (wd * dwd).sum(-1, keepdim=True)
    ref = wd * (dwd - dot)
    err = wd.abs() * ((C + 1) * U * (wd * dwd).abs().sum(-1, keepdim=True) + U * (dwd - dot).abs()) + U * ref.abs()
    _check("dscores", ds.v, ref, K_ATT * err + TINY)
    ds.untouched("dscores")


# =====================================================================================================================
# 6. Layout and norms
# =====================================================================================================================
@pytest.mark.parametrize("N", [1, 31, 32, 33])
@pytest.mark.parametrize("T", [1, 31, 32, 33])
def test_transpose_nt(N, T):
    """[Z, N, T] -> [Z, T, N] bit for bit; the _ld form's pad columns [N, ld_out) are +0 and nothing past them is written"""
    call, ptr, stream = _abi()
    Z = 3
    x = _rand(_gen(100 + N * 40 + T), Z, N, T)
    ref = x.transpose(1, 2)
    out = Out(Z, T, N)
    call("bm_transpose_nt", ptr(x), Z, N, T, ptr(out.t), stream())
    for ld in (N + 1, N + 31, 64 + N):
        o = Out(Z, T, ld)
        call("bm_transpose_nt_ld", ptr(x), Z, N, T, ld, ptr(o.t), stream())
        torch.cuda.synchronize()
        _same(f"bm_transpose_nt_ld ld={ld}", o.v[..., :N], ref)
        pad = o.v[..., N:].contiguous().view(torch.int32)
        assert (pad == 0).all(), f"bm_transpose_nt_ld ld={ld}: pad columns are not +0"
        o.untouched(f"bm_transpose_nt_ld ld={ld}")
    torch.cuda.synchronize()
    _same("bm_transpose_nt", out, ref)
    out.untouched("bm_transpose_nt")


@pytest.mark.parametrize("shape", [(1, 1, 1), (2, 33, 7), (3, 270, 361)])
def test_channel_mask(shape):
    """y = x * mask[c] bit for bit (one IEEE product, as torch's), in place too"""
    call, ptr, stream = _abi()
    B, C, T = shape
    gen = _gen(110 + C)
    x = _rand(gen, B, C, T)
    mask = (torch.rand(C, generator=gen, device=DEV) > 0.3).float()
    mask[:C // 3] *= torch.rand(C // 3, generator=gen, device=DEV) * 3
    y = Out(B, C, T)
    call("bm_channel_mask", ptr(x), ptr(mask), B, C, T, ptr(y.t), stream())
    xi = x.clone()
    call("bm_channel_mask", ptr(xi), ptr(mask), B, C, T, ptr(xi), stream())
    torch.cuda.synchronize()
    ref = x * mask[None, :, None]
    _same("y", y, ref)
    _same("in place", xi, ref)
    y.untouched("y")


@pytest.mark.parametrize("shape", [(1, 1, 1), (3, 5, 3), (33, 17, 5), (320, 320, 3)])
def test_conv_weight_prep(shape):
    """W [O, I, Kw] -> Wf [Kw, I, O] and Wb [Kw, O, I], bit for bit, either output NULL"""
    call, ptr, stream = _abi()
    O, I, Kw = shape
    w = _rand(_gen(120 + O), O, I, Kw)
    for want_f, want_b in ((True, True), (True, False), (False, True)):
        wf = Out(Kw, I, O) if want_f else None
        wb = Out(Kw, O, I) if want_b else None
        call("bm_conv_weight_prep", ptr(w), O, I, Kw, _p(wf), _p(wb), stream())
        torch.cuda.synchronize()
        if wf is not None:
            _same("Wf", wf, w.permute(2, 1, 0))
            wf.untouched("Wf")
        if wb is not None:
            _same("Wb", wb, w.permute(2, 0, 1))
            wb.untouched("Wb")


@pytest.mark.parametrize("off", [0, 1, 2, 3])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 1027, 64 * 360 * 320 + 3])
def test_amax(n, off):
    """bm_amax = max |x| bit for bit, on views starting at every float offset from a 16-byte boundary (the scalar epilogue
    and GLU forms hand it their misaligned outputs); the largest element sits first, last or in the middle"""
    call, ptr, stream = _abi()
    x = _rand(_gen(140 + n + off), n)
    outs = []
    for where in (0, n // 2, n - 1):
        y = x.clone()
        y[where] = -1e3
        xd = _dev(y, off)
        cell = Out(1)
        call("bm_amax", ptr(xd), n, ptr(cell.t), stream())
        outs.append((cell, y))
    torch.cuda.synchronize()
    for cell, y in outs:
        _same("amax", cell.v[0], y.abs().max())
        cell.untouched("amax")


@pytest.mark.parametrize("K", [1, 63, 64, 65, 64 * 256 + 1, 65537, 368640, 368641])
def test_candidate_inv_norms(K):
    """ss = sum_k c^2: fp32 chunks of at most 64 fused terms per thread, each added to an fp64 sum, so the error is below
    gamma_64 sum c^2 whatever K; inv_norm = 1 / (1e-8 + sqrt(ss)): the fp64 sqrt rounded to fp32, the add and the
    division, plus half ss's relative error.  The last term of every row is large, so a dropped tail shows"""
    call, ptr, stream = _abi()
    Bc = 3
    cand = _rand(_gen(130 + K % 1000), Bc, K)
    cand[:, -1] = 10.0
    cand[1] *= 1e-3
    ss = Out(Bc, dtype=torch.float64)
    inv = Out(Bc)
    call("bm_candidate_inv_norms", ptr(cand), Bc, K, ptr(ss.t), ptr(inv.t), stream())
    torch.cuda.synchronize()
    q = (cand.double() ** 2).sum(1)
    e_q = K_RED * _gamma(64) * q
    _check("ss", ss.v, q, e_q + TINY)
    ref = 1 / (1e-8 + torch.sqrt(q))
    _check("inv_norm", inv.v, ref, K_RED * ref * (3 * U + 0.5 * e_q / q) + TINY)
    ss.untouched("ss")
    inv.untouched("inv_norm")
