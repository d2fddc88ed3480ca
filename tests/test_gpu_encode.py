"""SimpleConv over several input streams on the H100 at the widths of an encoding model (bm/train.py:61-67): `meg` 208
sensors (and 273 padded, with ragged valid sensors), `features` 120 (mel) or 1024 (wav2vec), hidden 320 per stream, depth
10, the clip_conv options, T = 360, B = 64.

  * output, every parameter gradient and the input streams' gradients within 1e-4 of the fp64 restatement
    (oracle/encode_oracle.py) for each head form and `concatenate`, in train and eval mode;
  * under torch.use_deterministic_algorithms(True): repeated steps bitwise equal, and the frozen variants (features
    encoder frozen, head only, features.grad only) bitwise equal to the full backward;
  * under TF32: within the tolerance of tests/test_gpu_tf32.py;
  * bm_channel_join / bm_channel_split bitwise equal to torch.cat / slicing plus a transpose.
"""
import contextlib

import pytest
import torch

from conftest import rel_err
from oracle import encode_oracle

pytestmark = pytest.mark.gpu
DEV = "cuda"

# name: (meg sensors, valid sensors per recording, features, head, concatenate)
CASES = {
    "complex_208_mel": (208, (), 120, "complex", False),
    "linear_273_wav2vec": (273, (273, 250, 208), 1024, "linear", False),
    "concat_bare_208_mel": (208, (), 120, "bare", True),
    "concat_linear_273_mel": (273, (273, 230), 120, "linear", True),
}


def _variant(C, Fin, head, concatenate, S=4):
    return encode_oracle.EncodeVariant(in_channels=dict(meg=C, features=Fin), hidden=dict(meg=320, features=320),
                                       out_channels=C, n_subjects=S, concatenate=concatenate,
                                       linear_out=head == "linear", complex_out=head == "complex")


def _setup(case, B=64, T=360, seed=0):
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    C, n_valid, Fin, head, concatenate = CASES[case]
    v = _variant(C, Fin, head, concatenate)
    torch.manual_seed(seed)
    model = bb.SimpleConv(**v.kwargs())
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.add_(0.1 * torch.randn_like(m.weight))
                m.bias.add_(0.1 * torch.randn_like(m.bias))
                m.running_mean.add_(0.1 * torch.randn_like(m.running_mean))
                m.running_var.mul_(1 + 0.2 * torch.rand_like(m.running_var))
    model = model.to(DEV)
    S = v.n_subjects
    g = torch.Generator().manual_seed(seed + 1)
    subj = torch.randint(0, S, (B,), generator=g)
    pos = synthetic.normalised_positions(S, C, n_valid=n_valid, seed=seed)
    meg = torch.randn(B, C, T, generator=g)
    feats_full = torch.randn(B, Fin, T + 24, generator=g)
    w_out = torch.randn(B, C, T, generator=g)
    ban = torch.rand(2, generator=g)
    d = dict(subj=subj, pos=pos, meg=meg, feats_full=feats_full, w_out=w_out, ban=ban, T=T)
    return v, model, d


def _inputs(d, grad=True):
    meg = d["meg"].to(DEV).requires_grad_(grad)
    feats = d["feats_full"].to(DEV)[:, :, 7:7 + d["T"]].requires_grad_(grad)    # the solver's offset crop: a view
    return dict(meg=meg, features=feats)


def _batch(d):
    from brainmagick_b200 import synthetic
    return synthetic.make_batch(d["meg"].to(DEV), d["subj"].to(DEV), d["pos"], d["subj"])


def _run(model, d, train: bool, grad_inputs=True):
    """one forward / backward of loss = sum(out * w_out) -> {name: tensor} (output, every gradient)"""
    model.train(train)
    model.merger.ban_centre_override = d["ban"].to(DEV)
    model.zero_grad(set_to_none=True)
    inputs = _inputs(d, grad_inputs)
    out = model(dict(inputs), _batch(d))
    (out * d["w_out"].to(DEV)).sum().backward()
    torch.cuda.synchronize()
    from brainmagick_b200 import functional as BF
    BF.check_tc_status()
    res = {"out": out.detach().clone()}
    res.update({"g.in." + n: t.grad.clone() for n, t in inputs.items() if t.grad is not None})
    res.update({"g." + k: t.grad.clone() for k, t in model.named_parameters() if t.grad is not None})
    if train:
        res.update({"bn." + k: t.clone() for k, t in model.state_dict().items() if "running" in k})
    return res


def _oracle(v, state, d, train: bool, dtype=torch.float64):
    p = {k: t.detach().to(DEV, dtype).requires_grad_("running" not in k and "num_batches" not in k)
         for k, t in state.items() if t.is_floating_point()}
    inputs = {"meg": d["meg"].to(DEV, dtype).requires_grad_(True),
              "features": d["feats_full"][:, :, 7:7 + d["T"]].to(DEV, dtype).requires_grad_(True)}
    subj = d["subj"].to(DEV)
    stats = {} if train else None
    out = encode_oracle.forward(p, v, inputs, d["pos"].to(DEV, dtype), subj, subj, train, d["ban"].to(DEV, dtype), stats)
    (out * d["w_out"].to(DEV, dtype)).sum().backward()
    res = {"out": out.detach()}
    res.update({"g.in." + n: t.grad for n, t in inputs.items()})
    res.update({"g." + k: t.grad for k, t in p.items() if t.requires_grad})
    if train:
        res.update({"bn." + k: t for k, t in stats.items()})
    return res


def _errors(got, want):
    out = {}
    scale = max(want[k].abs().max().item() for k in want if k.startswith("g."))
    for k, w in want.items():
        g = got[k].double()
        if ".sequence." in k and k.endswith(".0.bias") and w.abs().max() < 1e-6 * scale:
            out[k] = g.abs().max().item() / scale            # exactly zero in truth (a training-mode BatchNorm follows)
        else:
            out[k] = rel_err(g, w)
    return out


@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("case", list(CASES))
def test_matches_fp64_oracle(case, train):
    v, model, d = _setup(case)
    state = {k: t.clone() for k, t in model.state_dict().items()}
    got = _run(model, d, train)
    want = _oracle(v, state, d, train)
    assert set(want) <= set(got), set(want) - set(got)
    err = _errors(got, want)
    worst = max(err.items(), key=lambda kv: kv[1])
    print(f"\n[{case} {'train' if train else 'eval'}] worst {worst[0]} {worst[1]:.2e}; out {err['out']:.2e} "
          f"meg.grad {err['g.in.meg']:.2e} features.grad {err['g.in.features']:.2e}")
    bad = {k: e for k, e in err.items() if e > 1e-4}
    assert not bad, bad


@contextlib.contextmanager
def _deterministic():
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was)


def _assert_bitwise(a, b, keys=None):
    for k in keys if keys is not None else a:
        assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("case", ["complex_208_mel", "concat_linear_273_mel"])
def test_repeated_steps_are_bitwise_equal_with_determinism(case):
    v, model, d = _setup(case, B=32)
    state = {k: t.clone() for k, t in model.state_dict().items()}
    with _deterministic():
        first = _run(model, d, True)
        model.load_state_dict(state)
        second = _run(model, d, True)
    _assert_bitwise(first, second)


def test_frozen_variants_match_the_full_backward_bitwise():
    v, model, d = _setup("complex_208_mel", B=32)
    state = {k: t.clone() for k, t in model.state_dict().items()}
    with _deterministic():
        full = _run(model, d, True)
        # the features encoder frozen
        model.load_state_dict(state)
        model.encoders["features"].requires_grad_(False)
        part = _run(model, d, True)
        assert not any(k.startswith("g.encoders.features.") for k in part)
        _assert_bitwise(full, part, [k for k in part])
        # the head alone
        model.load_state_dict(state)
        model.requires_grad_(False)
        model.final.requires_grad_(True)
        part = _run(model, d, True, grad_inputs=False)
        assert sorted(k for k in part if k.startswith("g.")) == sorted(k for k in full if k.startswith("g.final."))
        _assert_bitwise(full, part, [k for k in part])
        # features.grad alone
        model.load_state_dict(state)
        model.requires_grad_(False)
        model.train()
        model.merger.ban_centre_override = d["ban"].to(DEV)
        inputs = _inputs(d, False)
        inputs["features"].requires_grad_(True)
        out = model(dict(inputs), _batch(d))
        (out * d["w_out"].to(DEV)).sum().backward()
        assert torch.equal(inputs["features"].grad, full["g.in.features"])


def test_tf32_within_the_tf32_tolerance():
    import test_gpu_tf32 as t32
    v, model, d = _setup("complex_208_mel", B=32)
    state = {k: t.clone() for k, t in model.state_dict().items()}
    want = _oracle(v, state, d, True)
    with t32.precision(True):
        got = _run(model, d, True)
        torch_tf32 = _oracle(v, state, d, True, dtype=torch.float32)     # torch's own ops with TF32 allowed
    err, err_t = _errors(got, want), _errors(torch_tf32, want)
    bad = {k: (e, err_t[k]) for k, e in err.items() if e > max(2 * err_t[k], 2e-3)}
    assert not bad, bad


# ---- the join / split kernels --------------------------------------------------------------------------------------
def _call(name, *args):
    from brainmagick_b200._lib import call, stream
    call(name, *args, stream())


def _p(t):
    from ctypes import c_void_p
    return None if t is None else c_void_p(t.data_ptr())


@pytest.mark.parametrize("B,T", [(3, 37), (2, 360), (5, 1)])
@pytest.mark.parametrize("layout", ["odd", "aligned", "mixed"])
def test_join_and_split_are_exact_copies(B, T, layout):
    g = torch.Generator(device=DEV).manual_seed(B * 1000 + T)
    # (width, channel-major, gap before it)
    spec = {"odd": [(7, True, 0), (13, False, 3), (1, True, 0), (5, False, 2)],
            "aligned": [(64, False, 0), (120, True, 0), (320, False, 0)],
            "mixed": [(320, False, 0), (208, True, 4), (9, False, 0)]}[layout]
    off, pad = (0, 4) if layout == "aligned" else (1, 5)     # aligned: the float4 path; else the scalar one
    parts, cols, at = [], [], 0
    for C, cm, gap in spec:
        at += gap
        cols.append(at)
        if cm:      # a channel-major view cropped in time, with an odd offset
            full = torch.randn(B, C, T + 11, device=DEV, generator=g)
            parts.append(full[:, :, 3:3 + T])
        else:       # channels-last rows of stride ld >= C, at an odd element offset
            full = torch.randn(B * T * (C + pad) + off, device=DEV, generator=g)
            parts.append(full[off:].view(B, T, C + pad)[:, :, :C])
        at += C
    Cp = at + (8 if layout == "aligned" else 6)
    want = torch.zeros(B, T, Cp, device=DEV)
    for (C, cm, _), t, col in zip(spec, parts, cols):
        want[:, :, col:col + C] = t.transpose(1, 2) if cm else t
    dst_buf = torch.full((B * T * Cp + 64,), float("nan"), device=DEV)      # with a guard past the last row
    dst = dst_buf[:B * T * Cp].view(B, T, Cp)
    args = []
    for (C, cm, _), t, col in zip(spec, parts, cols):
        args += [_p(t), C, t.stride(1), int(cm), col]
    args += [None, 0, 0, 0, 0] * (4 - len(spec))            # unused slots
    _call("bm_channel_join", B, T, Cp, len(spec), *args, _p(dst))
    torch.cuda.synchronize()
    assert torch.equal(dst, want)
    assert torch.isnan(dst_buf[B * T * Cp:]).all()
    # the reverse into NaN-filled buffers of the same layouts, each with a guard of 64 elements past its last row; the
    # second range NULL (not wanted).  Every element outside a destination view must stay NaN, and src unchanged.
    src = torch.randn(B, T, Cp, device=DEV, generator=g)
    src_before = src.clone()

    def view_of(buf, C, cm):
        if cm:
            return buf[:B * C * (T + 11)].view(B, C, T + 11)[:, :, 3:3 + T]
        return buf[off:off + B * T * (C + pad)].view(B, T, C + pad)[:, :, :C]
    bufs, outs, args = [], [], []
    for i, ((C, cm, _), col) in enumerate(zip(spec, cols)):
        buf = o = None
        if i != 1:
            n = (B * C * (T + 11) if cm else B * T * (C + pad) + off) + 64
            buf = torch.full((n,), float("nan"), device=DEV)
            o = view_of(buf, C, cm)
        bufs.append(buf)
        outs.append(o)
        args += [_p(o), C, (o.stride(1) if o is not None else 0), int(cm), col]
    args += [None, 0, 0, 0, 0] * (4 - len(spec))
    _call("bm_channel_split", _p(src), B, T, Cp, len(spec), *args)
    torch.cuda.synchronize()
    assert torch.equal(src, src_before)
    for (C, cm, _), buf, o, col in zip(spec, bufs, outs, cols):
        if o is None:
            continue
        ref = src[:, :, col:col + C]
        assert torch.equal(o, ref.transpose(1, 2) if cm else ref)
        covered = torch.zeros(buf.shape, dtype=torch.bool, device=DEV)
        view_of(covered, C, cm).fill_(True)
        assert torch.isnan(buf[~covered]).all(), "the split wrote outside its destination view"
