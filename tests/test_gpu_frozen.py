"""Backpropagating only what requires grad, on the H100.

  * Under torch.use_deterministic_algorithms(True), every gradient a freezing pattern asks for -- and the BatchNorm running
    statistics -- are bitwise those of the full backward from the same state and seed: SimpleConv at the BASELINE widths
    (C = 208 at T = 360, and padded mixed 273/208/128/60 at T = 343; B = 64; train and eval), on the tensor-core and the
    FP32-FMA model, and DeepMel with its first half frozen.
  * With the flag off, the trainable gradients are within 1e-4 of fp64 autograd of the oracle.
  * The eval-mode BatchNorm backward without parameter gradients (one elementwise pass) gives the reducing form's dy bitwise.
  * A head-only step holds less memory than a full step by at least the per-layer conv outputs it no longer keeps."""
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

PATTERNS = ["attribution", "head", "subject", "merger", "bn", "glu"]


@pytest.fixture
def deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def _trainable(name, pattern, final):
    if pattern == "attribution":
        return False
    if pattern == "head":
        return name.startswith("final.") if final else name.startswith("encoders.meg.sequence.9.0.")
    if pattern == "subject":
        return name == "subject_layers.weights"
    if pattern == "merger":
        return name == "merger.heads"
    if pattern == "bn":
        return not any(name.startswith(f"encoders.meg.sequence.{k}.1.") for k in range(10))
    return ".glus." not in name


def _model(C, tc, seed=3):
    import brainmagick_b200 as bb
    torch.manual_seed(seed)
    model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=1024, hidden=dict(meg=320), depth=10, dilation_period=5,
                          kernel_size=3, skip=True, subject_layers=True, subject_dim=0, complex_out=True, glu=2,
                          glu_context=1, merger=True, initial_linear=270, merger_channels=270, gelu=True, batch_norm=True,
                          merger_pos_dim=2048, merger_dropout=0.2, n_subjects=4).cuda()
    model.use_tensor_cores = tc
    with torch.no_grad():
        for name, buf in model.named_buffers():
            if "running_mean" in name:
                buf.normal_(0, 0.1)
            elif "running_var" in name:
                buf.uniform_(0.5, 2.0)
    return model


def _run(model, state, pattern, train, C, T, n_valid, B=64):
    """one ClipLoss step from `state` -> ({name: grad}, meg.grad, {buffer: value})"""
    import brainmagick_b200 as bb
    from brainmagick_b200 import functional as BF, synthetic
    model.load_state_dict(state)
    model.train(train)
    for n, p in model.named_parameters():
        p.requires_grad_(pattern is None or _trainable(n, pattern, True))
        p.grad = None
    g = torch.Generator().manual_seed(11)
    meg = torch.randn(B, C, T, generator=g)
    subj = torch.randint(0, 4, (B,), generator=g)
    for b in range(B):
        meg[b, n_valid[int(subj[b])]:] = 0
    cand = torch.randn(B, 1024, T, generator=g).cuda()
    pos = synthetic.normalised_positions(4, C, n_valid, seed=4)
    model.merger.ban_centre_override = torch.tensor([0.31, 0.64])
    x = meg.cuda().requires_grad_(pattern in (None, "attribution"))
    est = model(dict(meg=x), synthetic.make_batch(x.detach(), subj.cuda(), pos, subj))
    bb.ClipLoss().cuda()(est, cand, torch.ones(B, 1, T, dtype=torch.bool, device="cuda")).backward()
    torch.cuda.synchronize()
    BF.check_tc_status()
    return ({n: None if p.grad is None else p.grad.clone() for n, p in model.named_parameters()}, x.grad,
            {n: b.clone() for n, b in model.named_buffers()})


SHAPES = {"c208": (208, 360, (208, 208, 208, 208)), "mixed": (273, 343, (273, 208, 128, 60))}


@pytest.mark.parametrize("tc", [True, False], ids=["tensor_cores", "fp32_fma"])
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
def test_frozen_gradients_bitwise_equal_full_backward(tc, shape, train, deterministic):
    C, T, n_valid = SHAPES[shape]
    model = _model(C, tc)
    state = {k: v.clone() for k, v in model.state_dict().items()}
    full, full_meg, full_bufs = _run(model, state, None, train, C, T, n_valid)
    for pattern in PATTERNS:
        if pattern == "attribution" and train:
            continue
        grads, meg_grad, bufs = _run(model, state, pattern, train, C, T, n_valid)
        for n, gr in grads.items():
            if _trainable(n, pattern, True):
                assert gr is not None and torch.equal(gr, full[n]), (pattern, n)
            else:
                assert gr is None, (pattern, n)
        if pattern == "attribution":
            assert torch.equal(meg_grad, full_meg)
        for n, b in bufs.items():
            assert torch.equal(b, full_bufs[n]), (pattern, n)


@pytest.mark.parametrize("pattern", ["head", "subject", "merger", "bn", "glu"])
def test_frozen_gradients_match_fp64_autograd(pattern):
    import brainmagick_b200 as bb
    from brainmagick_b200 import functional as BF, synthetic
    from oracle import ablation_oracle, bm_oracle
    C, T, B = 208, 360, 2
    model = _model(C, True, seed=23).train()
    v = ablation_oracle.Variant(in_channels=C, out_channels=1024, n_subjects=4)
    p = {k: t.detach().cpu().double().requires_grad_(t.is_floating_point() and "running" not in k and
                                                      _trainable(k, pattern, True))
         for k, t in model.state_dict().items()}
    g = torch.Generator().manual_seed(23)
    meg, cand = torch.randn(B, C, T, generator=g), torch.randn(B + 1, 1024, T, generator=g)
    subj = torch.tensor([3, 1])
    pos = synthetic.normalised_positions(4, C, (208, 150, 208, 97), seed=4)
    for b in range(B):
        meg[b, (208, 150, 208, 97)[int(subj[b])]:] = 0
    ban = torch.tensor([0.31, 0.64])
    est_ref = ablation_oracle.forward(p, v, meg.double(), pos.double(), subj, subj, training=True, ban_centre=ban.double())
    bm_oracle.clip_loss(est_ref, cand.double()).backward()
    for n, q in model.named_parameters():
        q.requires_grad_(_trainable(n, pattern, True))
    model.merger.ban_centre_override = ban
    x = meg.cuda()
    est = model(dict(meg=x), synthetic.make_batch(x, subj.cuda(), pos, subj))
    bb.ClipLoss().cuda()(est, cand.cuda(), torch.ones(B, 1, T, dtype=torch.bool, device="cuda")).backward()
    torch.cuda.synchronize()
    BF.check_tc_status()
    for n, q in model.named_parameters():
        if not _trainable(n, pattern, True):
            assert q.grad is None, n
            continue
        want = p[n].grad
        if want.norm() < 1e-6 * max(1.0, p[n].detach().norm().item()):
            assert q.grad.abs().max().item() < 1e-5, n        # a conv bias in front of a training BatchNorm
        else:
            assert rel_err(q.grad.cpu(), want) < 1e-4, (n, rel_err(q.grad.cpu(), want))


@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
def test_deepmel_first_half_frozen_bitwise(train, deterministic):
    import brainmagick_b200 as bb
    torch.manual_seed(5)
    model = bb.DeepMel(n_in_channels=120, n_hidden_channels=320, n_hidden_layers=10, n_out_channels=768, kernel=3, stride=1,
                       dilation_growth=2, dilation_period=5, batch_norm=True, activation_on_last=False, skip=True,
                       glu_context=1, glu=2).cuda()
    state = {k: v.clone() for k, v in model.state_dict().items()}
    g = torch.Generator().manual_seed(6)
    mel, est = torch.randn(64, 120, 360, generator=g).cuda(), torch.randn(64, 768, 360, generator=g).cuda()
    out = {}
    for frozen in (0, 5):
        model.load_state_dict(state)
        model.train(train)
        model.requires_grad_(True)
        model.zero_grad(set_to_none=True)
        for k in range(frozen):
            model.sequence[k].requires_grad_(False)
            if model.glus[k] is not None:
                model.glus[k].requires_grad_(False)
        e = est.clone().requires_grad_(True)
        bb.ClipLoss().cuda()(e, model(mel), torch.ones(64, 1, 360, dtype=torch.bool, device="cuda")).backward()
        torch.cuda.synchronize()
        out[frozen] = ({n: p.grad for n, p in model.named_parameters()}, e.grad,
                       {n: b.clone() for n, b in model.named_buffers()})
    full, half = out[0], out[5]
    assert torch.equal(half[1], full[1])
    for n, gr in half[0].items():
        if any(n.startswith(f"{m}.{k}.") for m in ("sequence", "glus") for k in range(5)):
            assert gr is None, n
        else:
            assert torch.equal(gr, full[0][n]), n
    for n, b in half[2].items():
        assert torch.equal(b, full[2][n]), n


@pytest.mark.parametrize("name,act", [("bm_bn_gelu_skip_bwd", None), ("bm_bn_act_skip_bwd", 0), ("bm_bn_act_skip_bwd", 1)])
@pytest.mark.parametrize("rows,C", [(64 * 360, 320), (1000, 37), (997, 320), (333, 1028), (96 * 7 + 5, 64)])
@pytest.mark.parametrize("det", [False, True])
def test_eval_bn_backward_without_parameter_gradients(name, act, rows, C, det):
    """batch_stats = 0 with sums / dgamma / dbeta NULL (one elementwise pass; the _det form without a workspace) against the
    reducing form: dy bitwise, at odd C, partial row blocks, and C on the column-stationary and the generic paths."""
    from brainmagick_b200 import _lib
    from brainmagick_b200._lib import call, ptr, stream
    gen = torch.Generator().manual_seed(rows + C)
    g, y = (torch.randn(rows, C, generator=gen).cuda() for _ in range(2))
    mean, beta = (0.3 * torch.randn(C, generator=gen).cuda() for _ in range(2))
    invstd, gamma = (torch.rand(C, generator=gen).cuda() + 0.5 for _ in range(2))
    sums = torch.empty(2 * C, dtype=torch.float64, device="cuda")
    dg, db = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    dy_ref, dy = torch.empty_like(g), torch.full_like(g, float("nan"))
    extra = () if act is None else (act, 0.1)
    head = (ptr(g), ptr(y), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), 0, rows, C) + extra
    tail = (None,) if act is None else ()                            # amax_out
    ws = torch.empty(max(int(getattr(_lib.load(), name + "_det_workspace")(rows, C)), 2), device="cuda")
    if det:
        call(name + "_det", *head, ptr(sums), ptr(dy_ref), ptr(dg), ptr(db), *tail, ptr(ws), ws.numel(), stream())
        call(name + "_det", *head, None, ptr(dy), None, None, *tail, None, 0, stream())
    else:
        call(name, *head, ptr(sums), ptr(dy_ref), ptr(dg), ptr(db), *tail, stream())
        call(name, *head, None, ptr(dy), None, None, *tail, stream())
    torch.cuda.synchronize()
    assert torch.equal(dy, dy_ref)


def test_head_only_step_holds_less_memory():
    """B = 64, T = 360, H = 320: a head-only step keeps none of the per-layer conv outputs (depth*B*T*H*4 bytes = 295 MB)"""
    C, T, B, H, depth = 208, 360, 64, 320, 10
    model = _model(C, True)
    state = {k: v.clone() for k, v in model.state_dict().items()}
    peak = {}
    for pattern in (None, "head", None, "head"):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        _run(model, state, pattern, True, C, T, (208,) * 4, B=B)
        peak[pattern] = torch.cuda.max_memory_allocated() - base
    assert peak[None] - peak["head"] >= depth * B * T * H * 4, peak
