"""GPU: every C entry point that runs on the FP32-FMA GEMM (csrc/gemm_simt.cuh) against a plain fp64 reference, element by
element, at the kernel's tile (GBM = GBN = 128, GBK = 16, 64-column GLU tiles), K-split, batch-segment and padding edges.

Each contraction is held to the fp32 dot-product bound

    |got - ref| <= C_BOUND * (K_total + 2) * 2^-24 * (|A| |B|)_ij + TINY

with K_total the full reduction length of that element (taps x K x the samples summed into its segment) and |A| |B| the
same contraction over absolute values, both in fp64 from the operands the kernel read.  Chained entry points are checked
stage by stage: each stage's reference is computed from the previous stage's fp32 output as the kernel wrote it, so every
bound stays componentwise.  Every output starts as NaN inside a buffer whose guard zones and padding columns hold a
sentinel bit pattern: an element left unwritten stays NaN, a write outside the output changes the sentinel.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24                # unit roundoff of fp32
# Any fp32 summation order of n terms with one rounding per step (FMA or add, serial, tree or atomic) errs by at most
# gamma_n = n u / (1 - n u) times the sum of the magnitudes; the "+ 2" covers the epilogue's scale / bias / addend roundings.
# C_BOUND = 2 allows for the 1 / (1 - n u) factor and for one more rounding per split partial (the column scale applied to
# each K-split partial before its atomic add, the ordered sum of the `_det` partial planes), both below one n u at the
# reduction lengths here.  It is one constant for every case.
C_BOUND = 2.0
TINY = 2.0 ** -140            # underflow: a few fp32 subnormal steps
GUARD = 64                    # floats of sentinel before and after every output
SENT = 0x7FA5A5A5             # a NaN bit pattern no kernel computes


def _abi():
    from brainmagick_b200 import _lib
    return _lib.call, _lib.ptr, _lib.stream


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _split(B, tiles):
    """(nseg, zchunk) of the split-batch weight-gradient GEMMs (csrc/api.cuh pick_chunks)"""
    want = min(max(1, -(-2 * _sms() // tiles)), B)
    zchunk = -(-B // want)
    return -(-B // zchunk), zchunk


def _tiles(M, N):
    return -(-M // 128) * -(-N // 128)


class Out:
    """A NaN-filled output `shape` (last dimension padded to `ld` columns) in a flat buffer with sentinel guard zones and
    sentinel padding columns.  .t: the full (padded) tensor the kernel receives; .v: the valid columns."""

    def __init__(self, *shape, ld=None):
        full = list(shape)
        full[-1] = ld or shape[-1]
        n = math.prod(full)
        self.flat = torch.full((n + 2 * GUARD,), SENT, dtype=torch.int32, device=DEV).view(torch.float32)
        self.t = self.flat[GUARD:GUARD + n].view(full)
        self.v = self.t[..., :shape[-1]]
        self.v.fill_(float("nan"))
        self.width = shape[-1]

    def untouched(self, what):
        bits = self.flat.view(torch.int32)
        assert (bits[:GUARD] == SENT).all() and (bits[-GUARD:] == SENT).all(), f"{what}: write outside the output"
        pad = self.t.view(torch.int32)[..., self.width:]
        assert (pad == SENT).all(), f"{what}: padding columns overwritten"


def _padded_in(t, ld):
    """input t in a row of ld >= width floats whose padding holds NaN (a read of it would poison the result)"""
    out = torch.full(t.shape[:-1] + (ld,), float("nan"), device=DEV)
    out[..., :t.shape[-1]] = t
    return out


def _bad(what, bad, got, ref, tol):
    i = tuple(bad.nonzero()[0].tolist())
    return (f"{what}: {int(bad.sum())} of {bad.numel()} elements off, first at {list(i)}: got {got[i].item():.9g} "
            f"ref {ref[i].item():.9g} tol {tol[i].item():.3g}")


def _check(what, got, ref, tol):
    got = got.double()
    nan = torch.isnan(got)
    assert not nan.any(), f"{what}: {int(nan.sum())} of {nan.numel()} elements left unwritten (NaN)"
    tol = torch.as_tensor(tol, dtype=torch.float64, device=DEV).expand_as(ref)
    bad = (got - ref).abs() > tol
    assert not bad.any(), _bad(what, bad, got, ref, tol)


def _check_dot(what, got, ref, mag, k_total):
    """the fp32 dot-product bound (module docstring); k_total: a number or a tensor broadcastable to ref"""
    _check(what, got, ref, C_BOUND * (torch.as_tensor(k_total, dtype=torch.float64, device=DEV) + 2) * U * mag + TINY)


def _check_sums(what, got, vals, dim):
    """fp64 column sums and sums of squares of the kernel's own fp32 values: n fp64 additions of exact fp32 squares err by
    at most n 2^-53 times the sum of magnitudes, so anything above that is a missing or double-counted row"""
    v = vals.double()
    n = v.numel() // v.shape[-1]
    eps = C_BOUND * (n + 2) * 2.0 ** -53
    s, q = v.sum(dim), (v * v).sum(dim)
    _check(what + " sum", got[0], s, eps * v.abs().sum(dim) + TINY)
    _check(what + " sumsq", got[1], q, eps * q + TINY)


def _rand(gen, *shape, scale=1.0):
    return torch.randn(*shape, generator=gen, device=DEV) * scale


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _groups(gen, B, G):
    """sample -> group (G >= 3: group 0 empty, group 1 one sample in the middle of the batch, the rest repeated)
    and its CSR (order, off) with each group's samples in shuffled, not sample, order"""
    if G == 1:
        a = torch.zeros(B, dtype=torch.int64, device=DEV)
    else:
        a = torch.randint(2, G, (B,), generator=gen, device=DEV) if G > 2 else torch.full((B,), 1, device=DEV)
        a[B // 2] = 1
    order = []
    for g in range(G):
        idx = (a == g).nonzero().flatten()
        order.append(idx[torch.randperm(idx.numel(), generator=gen, device=DEV)])
    order = torch.cat(order).int()
    off = torch.zeros(G + 1, dtype=torch.int32, device=DEV)
    off[1:] = torch.bincount(a, minlength=G).cumsum(0)
    return a, order, off


def _by_group(per_sample, a, G):
    """sum over the samples of each group of per_sample [B, ...] (fp64)"""
    out = torch.zeros((G,) + per_sample.shape[1:], dtype=torch.float64, device=DEV)
    return out.index_add_(0, a, per_sample)


def _refuse(name, args, ws_index):
    """a `_det` call with one float less workspace than required is refused with a message"""
    from brainmagick_b200 import _lib
    lib = _lib.load()
    args = list(args)
    args[ws_index] = args[ws_index] - 1
    rc = getattr(lib, name)(*args)
    assert rc != 0, f"{name}: accepted a workspace one float short"
    assert lib.bm_last_error().decode(), f"{name}: refused without a message"


def _gelu64(z):
    return z * 0.5 * torch.special.erfc(-z / math.sqrt(2.0))


# gelu_f / gelu_grad_f (common.cuh) take Phi(-|z|) from Numerical Recipes' erfc series (fractional error < 1.2e-7, 2 u)
# through an approximate reciprocal (1 ulp) and __expf of -z^2/2 + poly, whose error is (2 + 1.16 |arg|) ulp plus the
# 2 u z^2 / 2 of rounding z^2: Phi(-|z|) is good to (16 + 3 z^2) u relative, phi(z) to (6 + 2 z^2) u.
def _gelu_err(z):
    he = 0.5 * torch.special.erfc(z.abs() / math.sqrt(2.0))
    return C_BOUND * (z.abs() * (he * (16 + 3 * z * z) * U + U) + U * _gelu64(z).abs()) + TINY


def _gelu_grad64(z):
    return 0.5 * torch.special.erfc(-z / math.sqrt(2.0)) + z * torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)


def _gelu_grad_err(z):
    he = 0.5 * torch.special.erfc(z.abs() / math.sqrt(2.0))
    pdf = torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)
    return (z.abs() * pdf * (6 + 2 * z * z) + he * (16 + 3 * z * z) + 1 + _gelu_grad64(z).abs()) * U


def _check_softmax(what, got, s, delta, valid):
    """got = softmax over the last axis of scores s (fp64, -inf where not valid) whose fp32 values may be off by delta.
    A score error moves log(w) by at most 2 max|delta|; the kernel adds u |s - max| in the exponent's argument, 2 ulp of
    expf, (C - 1) u in the sum of C positive terms and two roundings in the scale."""
    C = s.shape[-1]
    w = torch.softmax(s, -1)
    d = (s - s.max(-1, keepdim=True).values).abs().nan_to_num(0.0, posinf=0.0)
    dmax = torch.where(valid, delta, 0).amax(-1, keepdim=True)
    rel = 2 * dmax + U * (d + d.amax(-1, keepdim=True)) + (C + 6) * U
    _check(what, got, w, C_BOUND * rel * w + TINY)
    assert (got[~valid.expand_as(got)] == 0).all(), f"{what}: masked entries are not exactly 0"


# =====================================================================================================================
# K1: spatial attention
# =====================================================================================================================
ATT = {"R1-C1-O1-P2": (1, 1, 1, 1), "R2-C127-O129-P18": (2, 127, 129, 3), "R3-C129-O128-P128": (3, 129, 128, 8),
       "R2-C16-O127-P32": (2, 16, 127, 4), "R5-C15-O64-P162": (5, 15, 64, 9), "real-R4-C273-O270-P2048": (4, 273, 270, 32)}


def _attention_inputs(R, C, O, n, gen):
    P = 2 * n * n
    pos = torch.rand(R, C, 2, generator=gen, device=DEV)
    if C > 2:          # padded sensors (INVALID = -0.1) at both ends of the first and the last recording
        pos[0, 0] = -0.1
        pos[-1, -1] = -0.1
    freq = 2 * math.pi * torch.arange(n, device=DEV, dtype=torch.float32) / 1.4
    heads = _rand(gen, O, P, scale=P ** -0.5)
    return pos, freq, heads, P


@pytest.mark.parametrize("case", list(ATT), ids=[f"bm_attention_weights_fwd-{k}" for k in ATT])
def test_attention_weights_fwd(case):
    call, ptr, stream = _abi()
    R, C, O, n = ATT[case]
    pos, freq, heads, P = _attention_inputs(R, C, O, n, _gen(11))
    emb, w = Out(R, C, P), Out(R, O, C)
    call("bm_attention_weights_fwd", ptr(pos), ptr(freq), ptr(heads), None, 0.0, R, C, O, P, ptr(emb.t), ptr(w.t), stream())
    torch.cuda.synchronize()
    assert torch.isfinite(emb.v).all(), "emb: elements left unwritten"
    e, h = emb.v.double(), heads.double()
    s = torch.einsum("rcp,op->roc", e, h)
    delta = C_BOUND * (P + 2) * U * torch.einsum("rcp,op->roc", e.abs(), h.abs())
    valid = ~((pos[..., 0] == -0.1) & (pos[..., 1] == -0.1))[:, None, :]
    _check_softmax("weights", w.v, s.masked_fill(~valid, -math.inf), delta, valid)
    emb.untouched("emb")
    w.untouched("weights")


@pytest.mark.parametrize("det", [False, True], ids=["bm_attention_weights_bwd", "bm_attention_weights_bwd_det"])
@pytest.mark.parametrize("case", list(ATT))
def test_attention_weights_bwd(case, det):
    call, ptr, stream = _abi()
    R, C, O, n = ATT[case]
    gen = _gen(12)
    pos, freq, heads, P = _attention_inputs(R, C, O, n, gen)
    emb, w = torch.empty(R, C, P, device=DEV), torch.empty(R, O, C, device=DEV)
    call("bm_attention_weights_fwd", ptr(pos), ptr(freq), ptr(heads), None, 0.0, R, C, O, P, ptr(emb), ptr(w), stream())
    dw = _rand(gen, R, O, C)
    name = "bm_attention_weights_bwd" + ("_det" if det else "")
    ds, dh = Out(R, O, C), Out(O, P)
    call(name, ptr(dw), ptr(w), ptr(emb), R, C, O, P, ptr(ds.t), ptr(dh.t), stream())
    torch.cuda.synchronize()
    # dscores = w (dw - sum_c w dw): the dot errs by (C + 1) u sum|w dw|, then one rounding each for the difference and product
    wd, dwd = w.double(), dw.double()
    dot = (wd * dwd).sum(-1, keepdim=True)
    ref = wd * (dwd - dot)
    err = wd.abs() * ((C + 1) * U * (wd * dwd).abs().sum(-1, keepdim=True) + U * (dwd - dot).abs()) + U * ref.abs()
    _check("dscores", ds.v, ref, C_BOUND * err + TINY)
    dsd, e = ds.v.double(), emb.double()
    _check_dot("dheads", dh.v, torch.einsum("roc,rcp->op", dsd, e), torch.einsum("roc,rcp->op", dsd.abs(), e.abs()), R * C)
    ds.untouched("dscores")
    dh.untouched("dheads")
    if det:   # a repeated call onto different scratch / output contents gives the same bits
        ds2, dh2 = torch.randn(R, O, C, device=DEV), torch.randn(O, P, device=DEV)
        call(name, ptr(dw), ptr(w), ptr(emb), R, C, O, P, ptr(ds2), ptr(dh2), stream())
        torch.cuda.synchronize()
        assert torch.equal(dh2, dh.v) and torch.equal(ds2, ds.v), "det: repeated call differs"


# =====================================================================================================================
# K2: sensor chain
# =====================================================================================================================
# (B, C, T, O, IL, D, S, R, pad): pad = extra columns of every leading dimension that may exceed its width
CHAIN = {"B3-C15-T1-O129-IL127-D128-S3-R4": (3, 15, 1, 129, 127, 128, 3, 4, 3),
         "B4-C17-T127-O128-IL129-D1-S1-R1": (4, 17, 127, 128, 129, 1, 1, 1, 5),
         "B5-C1-T129-O127-IL1-D129-S4-R3": (5, 1, 129, 127, 1, 129, 4, 3, 1),
         "B2-C16-T128-O1-IL128-D127-S3-R3": (2, 16, 128, 1, 128, 127, 3, 3, 2),
         "real-B8-C273-T360-O270-IL270-D320-S4-R5": (8, 273, 360, 270, 270, 320, 4, 5, 32)}


def _chain_inputs(case, seed):
    B, C, T, O, IL, D, S, R, pad = CHAIN[case]
    gen = _gen(seed)
    subj, subj_order, subj_off = _groups(gen, B, S)
    rec, rec_order, rec_off = _groups(gen, B, R)
    return dict(B=B, C=C, T=T, O=O, IL=IL, D=D, S=S, R=R, pad=pad, gen=gen, meg=_rand(gen, B, C, T),
                weights=torch.softmax(_rand(gen, R, O, C), -1), il_w=_rand(gen, IL, O, scale=O ** -0.5),
                il_b=_rand(gen, IL), subj_w=_rand(gen, S, IL, D, scale=IL ** -0.5), subj=subj, subj_order=subj_order,
                subj_off=subj_off, rec=rec, rec_order=rec_order, rec_off=rec_off, subj32=subj.int(), rec32=rec.int())


def _mix_ref(meg, weights, rec):
    m, w = meg.double(), weights.double()[rec]
    return torch.einsum("bct,boc->bto", m, w), torch.einsum("bct,boc->bto", m.abs(), w.abs())


def _il_ref(u, il_w, il_b):
    u, w, b = u.double(), il_w.double(), il_b.double()
    return u @ w.T + b, u.abs() @ w.abs().T + b.abs()


def _subj_ref(v, subj_w, subj):
    v, m = v.double(), subj_w.double()[subj]
    return torch.einsum("btp,bpd->btd", v, m), torch.einsum("btp,bpd->btd", v.abs(), m.abs())


@pytest.mark.parametrize("case", list(CHAIN), ids=[f"bm_sensor_mix_fwd+bm_initial_linear_fwd+bm_subject_layers_fwd-{k}"
                                                   for k in CHAIN])
def test_sensor_pieces_fwd(case):
    """the three stages with leading dimensions wider than their widths (inputs padded with NaN, outputs with sentinels);
    the weight sets are picked per sample (bsel) with repeated and unused sets"""
    call, ptr, stream = _abi()
    d = _chain_inputs(case, 21)
    B, C, T, O, IL, D, pad = d["B"], d["C"], d["T"], d["O"], d["IL"], d["D"], d["pad"]
    rec, subj = d["rec32"], d["subj32"]
    u = Out(B, T, O, ld=O + pad)
    call("bm_sensor_mix_fwd", ptr(d["meg"]), ptr(d["weights"]), ptr(rec), B, C, T, O, O + pad, ptr(u.t), stream())
    torch.cuda.synchronize()
    _check_dot("u", u.v, *_mix_ref(d["meg"], d["weights"], d["rec"]), C)
    u.untouched("u")
    u_in = _padded_in(u.v, O + 2 * pad)
    v = Out(B * T, IL, ld=IL + pad)
    call("bm_initial_linear_fwd", ptr(u_in), O + 2 * pad, ptr(d["il_w"]), ptr(d["il_b"]), B, T, O, IL, IL + pad, ptr(v.t),
         stream())
    torch.cuda.synchronize()
    _check_dot("v", v.v, *_il_ref(u.v.reshape(B * T, O), d["il_w"], d["il_b"]), O)
    v.untouched("v")
    v_in = _padded_in(v.v.reshape(B, T, IL), IL + 2 * pad)
    x0 = Out(B, T, D, ld=D + pad)
    call("bm_subject_layers_fwd", ptr(v_in), IL + 2 * pad, ptr(d["subj_w"]), ptr(subj), B, T, IL, D, D + pad, ptr(x0.t),
         stream())
    torch.cuda.synchronize()
    _check_dot("x0", x0.v, *_subj_ref(v.v.reshape(B, T, IL), d["subj_w"], d["subj"]), IL)
    x0.untouched("x0")


@pytest.mark.parametrize("case", list(CHAIN), ids=[f"bm_sensor_chain_fwd-{k}" for k in CHAIN])
def test_sensor_chain_fwd(case):
    call, ptr, stream = _abi()
    d = _chain_inputs(case, 22)
    B, C, T, O, IL, D, pad = d["B"], d["C"], d["T"], d["O"], d["IL"], d["D"], d["pad"]
    u, v, x0 = Out(B, T, O), Out(B, T, IL), Out(B, T, D, ld=D + pad)
    call("bm_sensor_chain_fwd", ptr(d["meg"]), ptr(d["weights"]), ptr(d["rec32"]), ptr(d["il_w"]), ptr(d["il_b"]),
         ptr(d["subj_w"]), ptr(d["subj32"]), B, C, T, O, IL, D, D + pad, ptr(u.t), ptr(v.t), ptr(x0.t), stream())
    torch.cuda.synchronize()
    _check_dot("u", u.v, *_mix_ref(d["meg"], d["weights"], d["rec"]), C)
    _check_dot("v", v.v, *_il_ref(u.v, d["il_w"], d["il_b"]), O)
    _check_dot("x0", x0.v, *_subj_ref(v.v, d["subj_w"], d["subj"]), IL)
    for o, name in ((u, "u"), (v, "v"), (x0, "x0")):
        o.untouched(name)


def _check_subj_bwd(d, dx0, v, dv, dsw):
    B, T, S, subj = d["B"], d["T"], d["S"], d["subj"]
    g, m = dx0.double(), d["subj_w"].double()[subj]
    if dv is not None:
        _check_dot("dv", dv, torch.einsum("btd,bpd->btp", g, m), torch.einsum("btd,bpd->btp", g.abs(), m.abs()), d["D"])
    if dsw is not None:
        vd = v.double()
        k = T * torch.bincount(subj, minlength=S).view(S, 1, 1)
        _check_dot("d_subj_w", dsw, _by_group(torch.einsum("btp,btd->bpd", vd, g), subj, S),
                   _by_group(torch.einsum("btp,btd->bpd", vd.abs(), g.abs()), subj, S), k)


def _check_il_bwd(d, dv, u, du, dilw, dilb):
    BT, IL, O = d["B"] * d["T"], d["IL"], d["O"]
    g = dv.reshape(BT, IL).double()
    if du is not None:
        w = d["il_w"].double()
        _check_dot("du", du.reshape(BT, O), g @ w, g.abs() @ w.abs(), IL)
    if dilw is not None:
        ud = u.reshape(BT, O).double()
        _check_dot("d_il_w", dilw, g.T @ ud, g.abs().T @ ud.abs(), BT)
    if dilb is not None:
        _check_dot("d_il_b", dilb, g.sum(0), g.abs().sum(0), BT)


def _check_mix_bwd(d, du, dwt):
    T, R, rec = d["T"], d["R"], d["rec"]
    g, m = du.double(), d["meg"].double()
    k = T * torch.bincount(rec, minlength=R).view(R, 1, 1)
    _check_dot("d_weights", dwt, _by_group(torch.einsum("bto,bct->boc", g, m), rec, R),
               _by_group(torch.einsum("bto,bct->boc", g.abs(), m.abs()), rec, R), k)


@pytest.mark.parametrize("case", list(CHAIN), ids=[f"bm_subject_layers_bwd+bm_sensor_mix_bwd+bm_sensor_mix_bwd_data-{k}"
                                                   for k in CHAIN])
def test_sensor_pieces_bwd(case):
    """subject-layer and mix gradients over CSR segments (an empty one, a single sample, shuffled order, S = 1), data
    gradients with padded leading dimensions, and the sensor mask as the column scale (masked sensors exactly 0)"""
    call, ptr, stream = _abi()
    d = _chain_inputs(case, 23)
    B, C, T, O, IL, D, S, R, pad, gen = (d[k] for k in ("B", "C", "T", "O", "IL", "D", "S", "R", "pad", "gen"))
    dx0 = _rand(gen, B, T, D)
    v = _rand(gen, B, T, IL)
    dv, dsw = Out(B, T, IL, ld=IL + pad), Out(S, IL, D)
    dx0_in, v_in = _padded_in(dx0, D + pad), _padded_in(v, IL + 2 * pad)      # (held: ptr() keeps no reference)
    call("bm_subject_layers_bwd", ptr(dx0_in), D + pad, ptr(v_in), IL + 2 * pad,
         ptr(d["subj_w"]), ptr(d["subj32"]), ptr(d["subj_order"]), ptr(d["subj_off"]), B, T, IL, D, S, IL + pad,
         ptr(dv.t), ptr(dsw.t), stream())
    torch.cuda.synchronize()
    _check_subj_bwd(d, dx0, v, dv.v, dsw.v)
    dv.untouched("dv")
    dsw.untouched("d_subj_w")

    du = _rand(gen, B, T, O)
    du_in = _padded_in(du, O + pad)
    dwt = Out(R, O, C)
    call("bm_sensor_mix_bwd", ptr(du_in), O + pad, ptr(d["meg"]), ptr(d["rec_order"]), ptr(d["rec_off"]),
         B, C, T, O, R, ptr(dwt.t), stream())
    torch.cuda.synchronize()
    _check_mix_bwd(d, du, dwt.v)
    dwt.untouched("d_weights")

    for mask in (None, (torch.rand(C, generator=gen, device=DEV) < 0.7).float()):
        if mask is not None:
            mask[0] = 0.0
        dmeg = Out(B, C, T)
        call("bm_sensor_mix_bwd_data", ptr(du_in), O + pad, ptr(d["weights"]), ptr(d["rec32"]),
             ptr(mask), B, C, T, O, ptr(dmeg.t), stream())
        torch.cuda.synchronize()
        g, w = du.double(), d["weights"].double()[d["rec"]]
        scale = torch.ones(C, dtype=torch.float64, device=DEV) if mask is None else mask.double()
        ref = torch.einsum("bto,boc->bct", g, w) * scale[:, None]
        mag = torch.einsum("bto,boc->bct", g.abs(), w.abs()) * scale[:, None]
        _check_dot("dmeg", dmeg.v, ref, mag, O)
        if mask is not None:
            assert (dmeg.v[:, mask == 0] == 0).all(), "dmeg: masked sensors are not exactly 0"
        dmeg.untouched("dmeg")


# initial_linear_bwd cases: the chain cases plus one whose d_il_w GEMM splits the batch into segments with a ragged last one
IL_BWD = dict(CHAIN)
IL_SPLIT = "split-B2SMs+1-T2-O9-IL6"


def _il_case(case):
    if case != IL_SPLIT:
        return _chain_inputs(case, 24)
    B = 2 * _sms() + 1
    nseg, zchunk = _split(B, _tiles(6, 9))
    assert nseg > 1 and B % zchunk != 0, "the split case must split the batch with a ragged last segment"
    gen = _gen(24)
    return dict(B=B, T=2, O=9, IL=6, pad=3, gen=gen, il_w=_rand(gen, 6, 9, scale=1 / 3), nseg=nseg)


def _ws(name, *dims):
    from brainmagick_b200 import _lib
    return int(getattr(_lib.load(), name)(*dims))


@pytest.mark.parametrize("det", [False, True], ids=["bm_initial_linear_bwd", "bm_initial_linear_bwd_det"])
@pytest.mark.parametrize("case", list(IL_BWD) + [IL_SPLIT])
def test_initial_linear_bwd(case, det):
    call, ptr, stream = _abi()
    d = _il_case(case)
    B, T, O, IL, pad, gen = d["B"], d["T"], d["O"], d["IL"], d["pad"], d["gen"]
    dv, u = _rand(gen, B * T, IL), _rand(gen, B * T, O)
    dv_in, u_in = _padded_in(dv, IL + pad), _padded_in(u, O + 2 * pad)

    def run(ws, du=None, dilw=None, dilb=None, name="bm_initial_linear_bwd_det"):
        args = [ptr(dv_in), IL + pad, ptr(u_in), O + 2 * pad, ptr(d["il_w"]), B, T, O, IL, O + pad,
                du and ptr(du.t), dilw and ptr(dilw.t), dilb and ptr(dilb.t)]
        if det:
            args += [ptr(ws), 0 if ws is None else ws.numel()]
        call(name if det else "bm_initial_linear_bwd", *args, stream())
        torch.cuda.synchronize()
        return args

    outs = lambda: (Out(B * T, O, ld=O + pad), Out(IL, O), Out(IL))  # noqa: E731
    du, dilw, dilb = outs()
    nws = _ws("bm_initial_linear_bwd_det_workspace", B, T, O, IL)
    if "nseg" in d:   # the library sized the deterministic planes for the split the test claims
        assert nws >= d["nseg"] * IL * O
    ws = torch.full((nws,), float("nan"), device=DEV)
    args = run(ws, du, dilw, dilb)
    _check_il_bwd(d, dv, u, du.v, dilw.v, dilb.v)
    for o, n in ((du, "du"), (dilw, "d_il_w"), (dilb, "d_il_b")):
        o.untouched(n)
    if not det:
        return
    _refuse("bm_initial_linear_bwd_det", args + [stream()], 14)
    full = [o.v.clone() for o in (du, dilw, dilb)]
    ws.copy_(torch.randn(nws, generator=gen, device=DEV))
    for keep in ((0, 1, 2), (0,), (1,), (2,), (0, 2)):       # frozen parameters / no data gradient
        o = [x if i in keep else None for i, x in enumerate(outs())]
        run(ws if keep != (0,) else None, *o)
        for i in keep:
            assert torch.equal(o[i].v, full[i]), f"outputs {keep}: output {i} differs from the full call's bits"
            o[i].untouched(f"outputs {keep}: output {i}")


@pytest.mark.parametrize("det", [False, True], ids=["bm_sensor_chain_bwd", "bm_sensor_chain_bwd_det"])
@pytest.mark.parametrize("case", list(CHAIN))
def test_sensor_chain_bwd(case, det):
    call, ptr, stream = _abi()
    d = _chain_inputs(case, 25)
    B, C, T, O, IL, D, S, R, pad, gen = (d[k] for k in ("B", "C", "T", "O", "IL", "D", "S", "R", "pad", "gen"))
    dx0, u, v = _rand(gen, B, T, D), _rand(gen, B, T, O), _rand(gen, B, T, IL)
    nws = _ws("bm_sensor_chain_bwd_det_workspace", B, T, O, IL)
    name = "bm_sensor_chain_bwd" + ("_det" if det else "")

    dx0_in = _padded_in(dx0, D + pad)

    def argv(outs, ws):
        args = [ptr(dx0_in), ptr(d["meg"]), ptr(d["il_w"]), ptr(d["subj_w"]), ptr(d["subj32"]),
                ptr(u), ptr(v), ptr(d["subj_order"]), ptr(d["subj_off"]), ptr(d["rec_order"]), ptr(d["rec_off"]),
                B, C, T, O, IL, D, D + pad, S, R] + [o and ptr(o.t) for o in outs]
        return args + ([ptr(ws), 0 if ws is None else ws.numel()] if det else []) + [stream()]

    def run(outs, ws):
        call(name, *argv(outs, ws))
        torch.cuda.synchronize()

    mk = lambda: [Out(B, T, IL), Out(B, T, O), Out(S, IL, D), Out(IL, O), Out(IL), Out(R, O, C)]  # noqa: E731
    outs = mk()
    ws = torch.full((nws,), float("nan"), device=DEV)
    run(outs, ws)
    dv, du, dsw, dilw, dilb, dwt = (o.v for o in outs)
    _check_subj_bwd(d, dx0, v, dv, dsw)
    _check_il_bwd(d, dv, u, du, dilw, dilb)
    _check_mix_bwd(d, du, dwt)
    for i, o in enumerate(outs):
        o.untouched(f"output {i}")
    if not det:
        return
    fresh = mk()           # a refused call does nothing: no stage runs before the workspace is checked
    _refuse(name, argv(fresh, ws), 27)
    torch.cuda.synchronize()
    for i, o in enumerate(fresh):
        assert torch.isnan(o.v).all(), f"refused call wrote output {i}"
        o.untouched(f"refused call: output {i}")
    full = [o.v.clone() for o in outs]
    ws.copy_(torch.randn(nws, generator=gen, device=DEV))
    # (dv, du, d_subj_w, d_il_w, d_il_b, d_weights): frozen parameters and stages with nothing left to compute
    for keep in ((0, 1, 2, 3, 4, 5), (2,), (0, 3), (0, 1, 5), (0, 1, 2, 4), (0, 1)):
        o = [x if i in keep else None for i, x in enumerate(mk())]
        run(o, ws if (3 in keep or 4 in keep) else None)
        for i in keep:
            assert torch.equal(o[i].v, full[i]), f"outputs {keep}: output {i} differs from the full call's bits"
            o[i].untouched(f"outputs {keep}: output {i}")


# =====================================================================================================================
# K3 / K4: dilated conv, its gradients and the GLU conv
# =====================================================================================================================
def _conv_ref(x, wop, dil, sign):
    """y[b,t,n] = sum_tap x[b, t + sign*(tap - Kw//2)*dil, :] . wop[tap][n, :] (zero outside [0, T)), and over |x| |w|"""
    B, T, _ = x.shape
    Kw, N, _ = wop.shape
    xd, wd = x.double(), wop.double()
    y = torch.zeros(B, T, N, dtype=torch.float64, device=DEV)
    a = torch.zeros_like(y)
    for tap in range(Kw):
        s = sign * (tap - Kw // 2) * dil
        lo, hi = max(0, -s), min(T, T - s)
        if lo < hi:
            y[:, lo:hi] += xd[:, lo + s:hi + s] @ wd[tap].T
            a[:, lo:hi] += xd[:, lo + s:hi + s].abs() @ wd[tap].abs().T
    return y, a


# (B, T, Cin, Cout, Kw, dilation)
CONV = {"B2-T129-Cin17-Cout127-Kw3-d1": (2, 129, 17, 127, 3, 1), "B3-T128-Cin15-Cout129-Kw3-d2": (3, 128, 15, 129, 3, 2),
        "B2-T127-Cin16-Cout128-Kw1-d1": (2, 127, 16, 128, 1, 1), "B2-T5-Cin1-Cout1-Kw3-d7": (2, 5, 1, 1, 3, 7),
        "B1-T1-Cin129-Cout3-Kw3-d1": (1, 1, 129, 3, 3, 1), "B3-T16-Cin128-Cout1-Kw3-d16": (3, 16, 128, 1, 3, 16),
        "real-B8-T360-Cin320-Cout320-Kw3-d2": (8, 360, 320, 320, 3, 2)}


def _conv_inputs(case, seed):
    B, T, Cin, Cout, Kw, dil = CONV[case]
    gen = _gen(seed)
    return (B, T, Cin, Cout, Kw, dil, gen, _rand(gen, B, T, Cin), _rand(gen, Cout, Cin, Kw, scale=(Cin * Kw) ** -0.5),
            _rand(gen, Cout))


@pytest.mark.parametrize("case", list(CONV), ids=[f"bm_conv1d_fwd-{k}" for k in CONV])
def test_conv1d_fwd(case):
    call, ptr, stream = _abi()
    B, T, Cin, Cout, Kw, dil, gen, x, w, bias = _conv_inputs(case, 31)
    y = Out(B, T, Cout)
    stats = torch.full((2 * Cout,), float("nan"), dtype=torch.float64, device=DEV)
    wf = w.permute(2, 1, 0).contiguous()
    call("bm_conv1d_fwd", ptr(x), ptr(wf), ptr(bias), B, T, Cin, Cout, Kw, dil, ptr(y.t),
         ptr(stats), stream())
    torch.cuda.synchronize()
    ref, mag = _conv_ref(x, w.permute(2, 0, 1), dil, +1)
    _check_dot("y", y.v, ref + bias.double(), mag + bias.double().abs(), Kw * Cin)
    _check_sums("stats", stats.view(2, Cout), y.v.reshape(B * T, Cout), 0)
    y.untouched("y")


@pytest.mark.parametrize("case", list(CONV), ids=[f"bm_conv1d_bwd_data-{k}" for k in CONV])
def test_conv1d_bwd_data(case):
    call, ptr, stream = _abi()
    B, T, Cin, Cout, Kw, dil, gen, _, w, _ = _conv_inputs(case, 32)
    dy, addend = _rand(gen, B, T, Cout), _rand(gen, B, T, Cin)
    ref, mag = _conv_ref(dy, w.permute(2, 1, 0), dil, -1)
    wb = w.permute(2, 0, 1).contiguous()
    for add in (None, addend):
        dx = Out(B, T, Cin)
        call("bm_conv1d_bwd_data", ptr(dy), ptr(wb), ptr(add), B, T, Cin, Cout, Kw, dil,
             ptr(dx.t), stream())
        torch.cuda.synchronize()
        a = 0 if add is None else add.double()
        _check_dot("dx" + ("" if add is None else " + addend"), dx.v, ref + a, mag + abs(a), Kw * Cout)
        dx.untouched("dx")


WGRAD = dict(CONV)
WGRAD_SPLIT = "split-B2SMs+1-T5-Cin5-Cout7-Kw3-d1"


@pytest.mark.parametrize("det", [False, True], ids=["bm_conv1d_bwd_weight", "bm_conv1d_bwd_weight_det"])
@pytest.mark.parametrize("case", list(WGRAD) + [WGRAD_SPLIT])
def test_conv1d_bwd_weight(case, det):
    call, ptr, stream = _abi()
    if case == WGRAD_SPLIT:
        B, T, Cin, Cout, Kw, dil, gen = 2 * _sms() + 1, 5, 5, 7, 3, 1, _gen(33)
        nseg, zchunk = _split(B, _tiles(Cout, Cin) * Kw)
        assert nseg > 1 and B % zchunk != 0, "the split case must split the batch with a ragged last segment"
        x = _rand(gen, B, T, Cin)
    else:
        B, T, Cin, Cout, Kw, dil, gen, x, _, _ = _conv_inputs(case, 33)
        nseg = _split(B, _tiles(Cout, Cin) * Kw)[0]
    dy = _rand(gen, B, T, Cout)
    nws = _ws("bm_conv1d_bwd_weight_det_workspace", B, T, Cin, Cout, Kw)
    assert nws >= nseg * Cout * Cin * Kw
    name = "bm_conv1d_bwd_weight" + ("_det" if det else "")

    def run(ws):
        dw, db = Out(Cout, Cin, Kw), Out(Cout)
        args = [ptr(dy), ptr(x), B, T, Cin, Cout, Kw, dil, ptr(dw.t), ptr(db.t)] + ([ptr(ws), nws] if det else [])
        call(name, *args, stream())
        torch.cuda.synchronize()
        return dw, db, args

    ws = torch.full((nws,), float("nan"), device=DEV)
    dw, db, args = run(ws)
    g, xd = dy.double(), x.double()
    ref = torch.zeros(Cout, Cin, Kw, dtype=torch.float64, device=DEV)
    mag = torch.zeros_like(ref)
    for tap in range(Kw):
        s = (tap - Kw // 2) * dil
        lo, hi = max(0, -s), min(T, T - s)
        if lo < hi:
            ref[:, :, tap] = torch.einsum("bto,bti->oi", g[:, lo:hi], xd[:, lo + s:hi + s])
            mag[:, :, tap] = torch.einsum("bto,bti->oi", g[:, lo:hi].abs(), xd[:, lo + s:hi + s].abs())
    _check_dot("dw", dw.v, ref, mag, B * T)
    _check_dot("dbias", db.v, g.sum((0, 1)), g.abs().sum((0, 1)), B * T)
    dw.untouched("dw")
    db.untouched("dbias")
    if det:
        _refuse(name, args + [stream()], 11)
        ws.copy_(torch.randn(nws, generator=gen, device=DEV))
        dw2, db2, _ = run(ws)
        assert torch.equal(dw2.v, dw.v) and torch.equal(db2.v, db.v), "det: result depends on the workspace contents"


# (B, T, Cin, H, Kw): GLU tiles hold 64 `a` columns and their 64 gates
GLU = {"B2-T129-Cin17-H63-Kw3": (2, 129, 17, 63, 3), "B3-T127-Cin16-H64-Kw1": (3, 127, 16, 64, 1),
       "B2-T128-Cin15-H65-Kw3": (2, 128, 15, 65, 3), "B2-T1-Cin1-H130-Kw3": (2, 1, 1, 130, 3),
       "real-B4-T360-Cin320-H320-Kw3": (4, 360, 320, 320, 3)}


@pytest.mark.parametrize("case", list(GLU), ids=[f"bm_conv1d_glu_fwd-{k}" for k in GLU])
def test_conv1d_glu_fwd(case):
    call, ptr, stream = _abi()
    B, T, Cin, H, Kw = GLU[case]
    gen = _gen(34)
    x, w, bias = _rand(gen, B, T, Cin), _rand(gen, 2 * H, Cin, Kw, scale=(Cin * Kw) ** -0.5), _rand(gen, 2 * H)
    h, out = Out(B, T, 2 * H), Out(B, T, H)
    wf = w.permute(2, 1, 0).contiguous()
    call("bm_conv1d_glu_fwd", ptr(x), ptr(wf), ptr(bias), B, T, Cin, H, Kw, ptr(h.t),
         ptr(out.t), stream())
    torch.cuda.synchronize()
    ref, mag = _conv_ref(x, w.permute(2, 0, 1), 1, +1)
    _check_dot("h", h.v, ref + bias.double(), mag + bias.double().abs(), Kw * Cin)
    # out = a * sigmoid(g) from the kernel's own h: expf (2 ulp), 1 + e, the IEEE division and the product: <= 7 u relative
    a, gt = h.v[..., :H].double(), h.v[..., H:].double()
    glu = a * torch.sigmoid(gt)
    _check("glu out", out.v, glu, C_BOUND * 7 * U * glu.abs() + TINY)
    h.untouched("h")
    out.untouched("out")
    out2 = Out(B, T, H)        # without the saved pre-activation: the same bits
    call("bm_conv1d_glu_fwd", ptr(x), ptr(wf), ptr(bias), B, T, Cin, H, Kw, None, ptr(out2.t),
         stream())
    torch.cuda.synchronize()
    assert torch.equal(out2.v, out.v), "glu out differs without h"
    out2.untouched("out (h NULL)")


# =====================================================================================================================
# K5: output head  x [B,T,H] -> h1 = x w0^T + b0 -> q = GELU(h1) -> est [B,F,T] = q w2 + b2
# =====================================================================================================================
HEAD = {"B1-T1-H1-F1": (1, 1, 1, 1), "B2-T127-H64-F129": (2, 127, 64, 129), "B2-T129-H65-F127": (2, 129, 65, 127),
        "B3-T128-H8-F128": (3, 128, 8, 128), "B2-T17-H15-F16": (2, 17, 15, 16),
        "real-B32-T360-H640-F208": (32, 360, 640, 208)}
HEAD_SPLIT = "split-B2SMs+1-T2-H3-F5"


def _head_case(case, seed):
    if case == HEAD_SPLIT:
        B, T, H, F = 2 * _sms() + 1, 2, 3, 5
        nseg, zchunk = _split(B, _tiles(2 * H, F))
        assert nseg > 1 and B % zchunk != 0, "the split case must split the batch with a ragged last segment"
    else:
        B, T, H, F = HEAD[case]
    gen = _gen(seed)
    return (B, T, H, F, gen, _rand(gen, B, T, H), _rand(gen, 2 * H, H, scale=H ** -0.5), _rand(gen, 2 * H),
            _rand(gen, 2 * H, F, scale=(2 * H) ** -0.5), _rand(gen, F))


@pytest.mark.parametrize("case", list(HEAD), ids=[f"bm_head_fwd-{k}" for k in HEAD])
def test_head_fwd(case):
    call, ptr, stream = _abi()
    B, T, H, F, gen, x, w0, b0, w2, b2 = _head_case(case, 41)
    h1, q, est = Out(B, T, 2 * H), Out(B, T, 2 * H), Out(B, F, T)
    call("bm_head_fwd", ptr(x), ptr(w0), ptr(b0), ptr(w2), ptr(b2), B, T, H, F, ptr(h1.t), ptr(q.t), ptr(est.t), stream())
    torch.cuda.synchronize()
    xd, w0d, b0d = x.double(), w0.double(), b0.double()
    _check_dot("h1", h1.v, xd @ w0d.T + b0d, xd.abs() @ w0d.abs().T + b0d.abs(), H)
    z = h1.v.double()
    _check("q = GELU(h1)", q.v, _gelu64(z), _gelu_err(z))
    qd, w2d, b2d = q.v.double(), w2.double(), b2.double()
    _check_dot("est", est.v, (qd @ w2d + b2d).transpose(1, 2), (qd.abs() @ w2d.abs() + b2d.abs()).transpose(1, 2), 2 * H)
    for o, n in ((h1, "h1"), (q, "q"), (est, "est")):
        o.untouched(n)


def _head_state(case, seed):
    """inputs and the forward's saved h1, q (computed by bm_head_fwd) and an upstream dest"""
    call, ptr, stream = _abi()
    B, T, H, F, gen, x, w0, b0, w2, b2 = _head_case(case, seed)
    h1, q, est = (torch.empty(B, T, 2 * H, device=DEV), torch.empty(B, T, 2 * H, device=DEV),
                  torch.empty(B, F, T, device=DEV))
    call("bm_head_fwd", ptr(x), ptr(w0), ptr(b0), ptr(w2), ptr(b2), B, T, H, F, ptr(h1), ptr(q), ptr(est), stream())
    return B, T, H, F, gen, x, w0, w2, h1, q, _rand(gen, B, F, T)


def _check_head_params(B, T, H, F, x, q, dest, dh1, dw0, db0, dw2, db2):
    g, qd = dest.double(), q.double()
    if dw2 is not None:
        _check_dot("dw2", dw2, torch.einsum("bti,bft->if", qd, g), torch.einsum("bti,bft->if", qd.abs(), g.abs()), B * T)
    if db2 is not None:
        _check_dot("db2", db2, g.sum((0, 2)), g.abs().sum((0, 2)), B * T)
    d1, xd = dh1.double().reshape(B * T, 2 * H), x.double().reshape(B * T, H)
    if dw0 is not None:
        _check_dot("dw0", dw0, d1.T @ xd, d1.abs().T @ xd.abs(), B * T)
    if db0 is not None:
        _check_dot("db0", db0, d1.sum(0), d1.abs().sum(0), B * T)


HEAD_BWD = list(HEAD) + [HEAD_SPLIT]


@pytest.mark.parametrize("det", [False, True], ids=["bm_head_bwd", "bm_head_bwd_det"])
@pytest.mark.parametrize("case", HEAD_BWD)
def test_head_bwd(case, det):
    call, ptr, stream = _abi()
    B, T, H, F, gen, x, w0, w2, h1, q, dest = _head_state(case, 42)
    nws = _ws("bm_head_bwd_det_workspace", B, T, H, F)
    name = "bm_head_bwd" + ("_det" if det else "")
    mk = lambda: [Out(B, T, 2 * H), Out(B, T, H), Out(2 * H, H), Out(2 * H), Out(2 * H, F), Out(F)]  # noqa: E731

    def run(outs, ws, w2_=w2, h1_=h1):
        args = [ptr(dest), ptr(x), ptr(w0), ptr(w2_), ptr(h1_), ptr(q), B, T, H, F] + [o and ptr(o.t) for o in outs]
        if det:
            args += [ptr(ws), 0 if ws is None else ws.numel()]
        call(name, *args, stream())
        torch.cuda.synchronize()
        return args

    outs = mk()
    ws = torch.full((nws,), float("nan"), device=DEV)
    args = run(outs, ws)
    dq, dx, dw0, db0, dw2, db2 = (o.v for o in outs)
    # dq (after the call: dh1 = (dest w2^T) * GELU'(h1)): the F-term dot's bound through GELU', GELU''s own error, one product
    g, w2d, z = dest.double(), w2.double(), h1.double()
    dq64 = torch.einsum("bft,if->bti", g, w2d)
    mag = torch.einsum("bft,if->bti", g.abs(), w2d.abs())
    gg = _gelu_grad64(z)
    dh1 = dq64 * gg
    tol = C_BOUND * (gg.abs() * (F + 2) * U * mag + dq64.abs() * _gelu_grad_err(z) + U * dh1.abs()) + TINY
    _check("dh1", dq, dh1, tol)
    _check_head_params(B, T, H, F, x, q, dest, dq, dw0, db0, dw2, db2)
    d1, w0d = dq.double(), w0.double()
    _check_dot("dx", dx, d1 @ w0d, d1.abs() @ w0d.abs(), 2 * H)
    for i, o in enumerate(outs):
        o.untouched(f"output {i}")
    if not det:
        return
    _refuse(name, args + [stream()], 17)
    full = [o.v.clone() for o in outs]
    ws.copy_(torch.randn(nws, generator=gen, device=DEV))
    # (dq, dx, dw0, db0, dw2, db2); with dx, dw0, db0 all NULL, dq, h1 and w2 may be NULL too
    for keep in ((0, 1, 2, 3, 4, 5), (0, 1), (0, 2, 3), (4, 5), (4,), (0, 1, 5)):
        o = [x_ if i in keep else None for i, x_ in enumerate(mk())]
        no_dh1 = not ({1, 2, 3} & set(keep))
        run(o, ws if ({2, 3, 4, 5} & set(keep)) else None, None if no_dh1 else w2, None if no_dh1 else h1)
        for i in keep:
            if i == 0 and no_dh1:
                continue
            assert torch.equal(o[i].v, full[i]), f"outputs {keep}: output {i} differs from the full call's bits"
            o[i].untouched(f"outputs {keep}: output {i}")


@pytest.mark.parametrize("det", [False, True], ids=["bm_head_bwd_params", "bm_head_bwd_params_det"])
@pytest.mark.parametrize("case", HEAD_BWD)
def test_head_bwd_params(case, det):
    call, ptr, stream = _abi()
    B, T, H, F, gen, x, w0, w2, h1, q, dest = _head_state(case, 43)
    dq_in = _rand(gen, B, T, 2 * H)
    nws = _ws("bm_head_bwd_params_det_workspace", B, T, H, F)
    name = "bm_head_bwd_params" + ("_det" if det else "")

    def run(ws):
        dq = Out(B, T, 2 * H)
        dq.v.copy_(dq_in)
        outs = [Out(2 * H, H), Out(2 * H), Out(2 * H, F), Out(F)]
        args = [ptr(dest), ptr(x), ptr(h1), ptr(q), B, T, H, F, ptr(dq.t)] + [ptr(o.t) for o in outs]
        if det:
            args += [ptr(ws), nws]
        call(name, *args, stream())
        torch.cuda.synchronize()
        return dq, outs, args

    ws = torch.full((nws,), float("nan"), device=DEV)
    dq, outs, args = run(ws)
    z = h1.double()
    dh1 = dq_in.double() * _gelu_grad64(z)
    _check("dh1", dq.v, dh1, C_BOUND * (dq_in.double().abs() * _gelu_grad_err(z) + U * dh1.abs()) + TINY)
    _check_head_params(B, T, H, F, x, q, dest, dq.v, *(o.v for o in outs))
    dq.untouched("dq")
    for i, o in enumerate(outs):
        o.untouched(f"output {i}")
    if det:
        _refuse(name, args + [stream()], 14)
        ws.copy_(torch.randn(nws, generator=gen, device=DEV))
        dq2, outs2, _ = run(ws)
        assert torch.equal(dq2.v, dq.v) and all(torch.equal(a.v, b.v) for a, b in zip(outs2, outs)), \
            "det: result depends on the workspace contents"


# =====================================================================================================================
# CLIP on the FP32-FMA GEMM: feature sizes that are not a multiple of 4 (no tensor-core row pitch)
# =====================================================================================================================
def _clip_cases():
    k = 2 * _sms() * 16        # one 16-deep K block per split at the default split count on one tile
    return {"Bn1-Bc1-KT1": (1, 1, 1), "Bn127-Bc129-KT15": (127, 129, 15), "Bn129-Bc129-KT17": (129, 129, 17),
            "Bn128-Bc128-KT2SMs*16+1": (128, 128, k + 1), "Bn2-Bc3-KT2SMs*16-1": (2, 3, k - 1),
            "real-Bn256-Bc256-KT75001": (256, 256, 75001)}


CLIP_IDS = ["Bn1-Bc1-KT1", "Bn127-Bc129-KT15", "Bn129-Bc129-KT17", "Bn128-Bc128-KT2SMs*16+1", "Bn2-Bc3-KT2SMs*16-1",
            "real-Bn256-Bc256-KT75001"]


def _clip_inputs(case, seed):
    Bn, Bc, KT = _clip_cases()[case]
    assert KT % 4 != 0
    gen = _gen(seed)
    return Bn, Bc, KT, gen, _rand(gen, Bn, KT), _rand(gen, Bc, KT)


def _check_inv_norm(inv, cand):
    """1 / (1e-8 + ||c||): fp32 chunk sums of <= 64 squares (64 u relative), halved by the sqrt, then the float conversion,
    the add and the division"""
    ref = 1.0 / (1e-8 + cand.double().pow(2).sum(1).sqrt())
    _check("inv_norm", inv, ref, C_BOUND * 35 * U * ref)


def _check_scores(scores, est, cand, inv):
    e, c, i = est.double(), cand.double(), inv.double()
    _check_dot("scores", scores, (e @ c.T) * i, (e.abs() @ c.abs().T) * i, est.shape[1])


@pytest.mark.parametrize("det", [False, True], ids=["bm_clip_scores", "bm_clip_scores_det"])
@pytest.mark.parametrize("norms_given", [0, 1], ids=["norms", "norms_given"])
@pytest.mark.parametrize("case", CLIP_IDS)
def test_clip_scores_fma(case, norms_given, det):
    call, ptr, stream = _abi()
    Bn, Bc, KT, gen, est, cand = _clip_inputs(case, 51)
    from brainmagick_b200 import _lib
    nws = int(_lib.load().bm_clip_workspace(Bn, Bc, KT))
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    given = 1.0 / (1e-8 + cand.double().norm(dim=1)).float()
    name = "bm_clip_scores" + ("_det" if det else "")

    def run(ws):
        inv, scores, probs = Out(Bc), Out(Bn, Bc), Out(Bn, Bc)
        if norms_given:
            inv.v.copy_(given)
        call(name, ptr(est), ptr(cand), Bn, Bc, KT, norms_given, ptr(inv.t), ptr(scores.t), ptr(probs.t), ptr(ws), nws,
             ptr(status), stream())
        torch.cuda.synchronize()
        return inv, scores, probs

    ws = torch.full((nws,), float("nan"), device=DEV)
    inv, scores, probs = run(ws)
    if norms_given:
        assert torch.equal(inv.v, given), "inv_norm (an input) was changed"
    else:
        _check_inv_norm(inv.v, cand)
    _check_scores(scores.v, est, cand, inv.v)
    s = scores.v.double()
    _check_softmax("probs", probs.v, s, torch.zeros_like(s), torch.ones_like(s, dtype=torch.bool))
    assert status.item() == 0
    for o, n in ((inv, "inv_norm"), (scores, "scores"), (probs, "probs")):
        o.untouched(n)
    if det:
        ws.copy_(torch.randn(nws, generator=gen, device=DEV))
        inv2, scores2, probs2 = run(ws)
        assert torch.equal(inv2.v, inv.v) and torch.equal(scores2.v, scores.v) and torch.equal(probs2.v, probs.v), \
            "det: result depends on the workspace contents"
        _refuse(name, [ptr(est), ptr(cand), Bn, Bc, KT, norms_given, ptr(inv2.t), ptr(scores2.t), ptr(probs2.t), ptr(ws),
                       nws, ptr(status), stream()], 10)


@pytest.mark.parametrize("det", [False, True], ids=["bm_clip_loss_fwd", "bm_clip_loss_fwd_det"])
@pytest.mark.parametrize("case", CLIP_IDS)
def test_clip_loss_fwd_fma(case, det):
    call, ptr, stream = _abi()
    Bn, Bc, KT, gen, est, cand = _clip_inputs(case, 52)
    from brainmagick_b200 import _lib
    nws = int(_lib.load().bm_clip_workspace(Bn, Bc, KT))
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    off = Bc - Bn
    name = "bm_clip_loss_fwd" + ("_det" if det else "")

    def run(ws):
        outs = [Out(Bc), Out(Bn, Bc), Out(Bn, Bc), Out(Bn), Out(1)]
        call(name, ptr(est), ptr(cand), Bn, Bc, KT, off, *(ptr(o.t) for o in outs), ptr(ws), nws, ptr(status), stream())
        torch.cuda.synchronize()
        return outs

    ws = torch.full((nws,), float("nan"), device=DEV)
    outs = run(ws)
    inv, scores, probs, row_loss, loss = (o.v for o in outs)
    _check_inv_norm(inv, cand)
    _check_scores(scores, est, cand, inv)
    s = scores.double()
    _check_softmax("probs", probs, s, torch.zeros_like(s), torch.ones_like(s, dtype=torch.bool))
    # row loss = log sum exp(s - m) + m - s[target] from the kernel's scores: (Bc + 4) u in the sum's log, 2 ulp of logf,
    # and one rounding each of the two additions
    m = s.max(1).values
    lse = torch.logsumexp(s, 1)
    tgt = s[torch.arange(Bn, device=DEV), off + torch.arange(Bn, device=DEV)]
    rl = lse - tgt
    _check("row_loss", row_loss, rl, C_BOUND * U * ((Bc + 4) + 2 * (lse - m).abs() + lse.abs() + rl.abs()) + TINY)
    mean = row_loss.double().mean()        # fp64 sum, one rounding to fp32
    _check("loss", loss, mean.view(1), C_BOUND * U * mean.abs().view(1) + TINY)
    assert status.item() == 0
    for i, o in enumerate(outs):
        o.untouched(f"output {i}")
    if det:
        ws.copy_(torch.randn(nws, generator=gen, device=DEV))
        outs2 = run(ws)
        assert all(torch.equal(a.v, b.v) for a, b in zip(outs2, outs)), "det: result depends on the workspace contents"
        _refuse(name, [ptr(est), ptr(cand), Bn, Bc, KT, off] + [ptr(o.t) for o in outs2] + [ptr(ws), nws, ptr(status),
                                                                                           stream()], 12)
