"""FeatureDecodingLoss on the H100:

  * the loss, the saved log-sum-exp and every element of both gradients against fp64, through the C entry points, for
    [regression 3, categorical K, regression 1, categorical 7] with class weights (zero weights included), -100 and
    fractional targets and a ragged mask, at K in {1, 2, 3, 41, 1025}, T in {1, 3, 4, 33, 342, 343}, B in {1, 256}, on the
    float4 and the scalar paths (outputs 16-byte aligned or not, operands read at an odd element offset), with every output
    between NaN-filled guard zones;
  * bitwise equal results across repeated calls, with and without torch.use_deterministic_algorithms, and under bf16
    autocast;
  * the data errors 904 (empty mask), 905 (a class target >= K) and 906 (a masked negative target) raised by
    functional.check_tc_status() after a captured step is replayed on such data, without a fault;
  * a clip_conv SimpleConv decoding step (B 64, C 208, T 342, 120 mel + 41 + 2 classes, weighted) against the fp64 oracle
    (oracle/bm_oracle.py with the loss restated in fp64): estimate, loss and every parameter gradient within 1e-4;
  * the same step captured on a StaticBatch and replayed on fresh batches, bitwise equal to eager under the determinism flag.
"""
from ctypes import c_void_p

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from test_decoding_loss_cpu import Builder, Feature, Scaler
from test_gpu_cuda_graph import CLIP_DIMS, _assert_bitwise, _capture, _clip_conv, _items, deterministic  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 2.0 ** -24          # fp32 unit roundoff
GUARD = 64                # floats of NaN before and after every output (256 bytes: the interior stays 16-byte aligned)


def _class_weights(K, gen):
    """norm.py:289-308 over random counts with one empty class: 1 / sqrt(p), 0 where p = 0, normalised"""
    counts = torch.randint(1, 50, (K,), generator=gen).double()
    if K > 1:
        counts[K // 2] = 0
    p = counts / counts.sum()
    w = 1 / torch.sqrt(p)
    w[p == 0] = 0
    return (w / torch.sqrt(p).sum()).float(), counts.float()


def _mixed(K, B, T, seed=0, weighted=True):
    gen = torch.Generator().manual_seed(seed)
    builder = Builder([("mel", Feature("mel", 3)), ("cls", Feature("cls", 1, K)), ("env", Feature("env", 1)),
                       ("pos", Feature("pos", 1, 7))])
    est = torch.randn(B, builder.output_dimension, T + 1, generator=gen) * 3
    out = torch.randn(B, builder.dimension, T + 1, generator=gen)
    out[:, 3] = torch.randint(0, K, (B, T + 1), generator=gen) + 0.9 * torch.rand(B, T + 1, generator=gen)
    out[:, 3] = out[:, 3].clamp(max=K - 0.01)
    out[:, 5] = torch.randint(0, 7, (B, T + 1), generator=gen).float()
    out[:, 3][torch.rand(B, T + 1, generator=gen) < 0.1] = -100.0
    mask = torch.rand(B, 1, T + 1, generator=gen) > 0.3
    mask[:, :, :2] = True                   # one masked entry at least, in either crop, with class 0 (a nonzero weight):
    out[:, 3, :2] = 0.0                     # no term is 0 / 0
    out[:, 5, :2] = 0.0
    scaler = None
    if weighted:
        (wc, cc), (wp, cp) = _class_weights(K, gen), _class_weights(7, gen)
        scaler = Scaler({"cls": wc, "pos": wp}, {"cls": cc, "pos": cp})
    return builder, scaler, est.to(DEV), out.to(DEV), mask.to(DEV)


def _fp64(builder, scaler, est, out, mask, g=1.0):
    """(loss, per-feature lse, d_est, d_out) in fp64 from the reference's definition, on the fp32 operands"""
    e = est.double().detach().requires_grad_(True)
    o = out.double().detach().requires_grad_(True)
    loss, lse = 0, []
    for f in builder.values():
        es, os_ = builder.get_slice(f.name, model_output=True), builder.get_slice(f.name)
        if f.categorical:
            m = mask[:, 0]
            logits = e[:, es].transpose(1, 2)
            lse.append(torch.logsumexp(logits.detach(), dim=2))
            w = None if scaler is None else scaler.weights[f.name].double().to(DEV)
            loss = loss + F.cross_entropy(logits[m], out[:, os_.start][m].long(), w)
        else:
            mm = mask.expand_as(e[:, es])
            loss = loss + F.mse_loss(e[:, es][mm], o[:, os_][mm])
    d_e, d_o = torch.autograd.grad(loss * g, [e, o])
    return loss.detach(), lse, d_e, d_o


def _lse_bound(K, lse):
    return 4 * (K + 2) * EPS * lse.abs().clamp(min=1)


def _bounds(builder, scaler, est, out, mask, lse, d_est, d_out, loss, g):
    """componentwise error bounds from fp32 rounding.  Regression: (e - o), the scale 2/N and two products: 6 eps |ref|.
    Categorical: the online log-sum-exp takes K steps of expf (2 ulp), a product and a sum in fp32, so lse is off by up
    to eps_K = 4 (K + 2) eps max(1, |lse|); a gradient element g w_y / W (p_k - [k = y]) is then off by up to
    |g w_y / W| (p_k eps_K 2 + 6 eps) + 6 eps |ref|.  The loss: each term's own error, 4 eps |term| plus eps_K."""
    b_est = 6 * EPS * d_est.abs()
    b_out = 6 * EPS * d_out.abs() + 1e-30
    b_loss = 8 * EPS * abs(float(loss))
    i = 0
    for f in builder.values():
        es, os_ = builder.get_slice(f.name, model_output=True), builder.get_slice(f.name)
        if not f.categorical:
            continue
        K = f.cardinality
        eps_k = _lse_bound(K, lse[i])                                             # [B, T]
        v = out[:, os_.start]
        y = torch.where((v < K) & (v > -1), v, torch.zeros_like(v)).long()
        ok = mask[:, 0] & (v < K) & (v > -1)
        w = torch.ones(K, device=DEV) if scaler is None else scaler.weights[f.name].to(DEV)
        wy = torch.where(ok, w[y], torch.zeros_like(v)).double()
        W = wy.sum()
        coef = (g * wy / W)[:, None]                                              # [B, 1, T]
        p = torch.exp(est[:, es].double() - lse[i][:, None])
        b_est[:, es] += coef.abs() * (2 * p * eps_k[:, None] + 6 * EPS)
        b_loss += float((wy * eps_k).sum() / W) * 2
        i += 1
    return b_loss, b_est, b_out


def _guarded(n):
    buf = torch.full((GUARD + n + GUARD + 4,), float("nan"), device=DEV)
    return buf


def _check_guards(buf, at, n, what):
    assert torch.isnan(buf[:at]).all() and torch.isnan(buf[at + n:]).all(), f"{what}: a guard zone was written"


CASES = [(1, 1, 1), (256, 3, 1), (1, 4, 2), (256, 33, 2), (256, 343, 2), (1, 342, 3), (256, 4, 3), (256, 342, 41),
         (1, 343, 41), (256, 33, 41), (1, 1, 1025), (256, 4, 1025), (1, 342, 1025), (256, 343, 1025)]


@pytest.mark.parametrize("path", ["float4", "scalar"])
@pytest.mark.parametrize("B,T,K", CASES)
def test_every_element_against_fp64(B, T, K, path):
    import brainmagick_b200 as bb
    from brainmagick_b200 import functional as BF
    from brainmagick_b200._lib import stream
    builder, scaler, est_full, out_full, mask_full = _mixed(K, B, T, seed=K + T)
    # float4: the operands and outputs start on 16-byte boundaries; scalar: the operands are the solver's crop [..., 1:] at
    # an odd element offset and the outputs start one float past a boundary
    est, out, mask = ((est_full[..., :T].contiguous(), out_full[..., :T].contiguous(), mask_full[..., :T])
                      if path == "float4" else
                      (est_full[..., 1:], out_full[..., 1:], mask_full[..., 1:]))
    loss_fn = bb.FeatureDecodingLoss(builder, scaler)
    table, weights = loss_fn._table(torch.device(DEV)), loss_fn._class_weights(torch.device(DEV))
    Fn, Ce, Co = table.shape[0], est.shape[1], out.shape[1]
    shift = 0 if path == "float4" else 1
    at = GUARD + shift
    lse_b, loss_b, scale_b = _guarded(2 * B * T), _guarded(1), _guarded(Fn)
    de_b, do_b = _guarded(B * Ce * T), _guarded(B * Co * T)
    flag = torch.full((1,), -7, dtype=torch.int32, device=DEV)
    ws = torch.full((max(int(bb._lib.load().bm_decoding_loss_workspace(B, T, Fn)), 2),), float("nan"), device=DEV)
    g = torch.tensor([0.75], device=DEV)

    def p(buf):
        return c_void_p(buf[at:].data_ptr())
    ms = BF._mask_strides(mask)
    BF.call("bm_decoding_loss_fwd", c_void_p(est.data_ptr()), est.stride(0), est.stride(1), c_void_p(out.data_ptr()),
            out.stride(0), out.stride(1), c_void_p(mask.data_ptr()), *ms, B, T, BF.ptr(table), Fn, BF.ptr(weights),
            p(lse_b), BF.ptr(ws), ws.numel(), p(loss_b), p(scale_b), BF.ptr(flag), None, stream())
    BF.call("bm_decoding_loss_bwd", BF.ptr(g), p(scale_b), p(lse_b), c_void_p(est.data_ptr()), est.stride(0),
            est.stride(1), c_void_p(out.data_ptr()), out.stride(0), out.stride(1), c_void_p(mask.data_ptr()), *ms, B, T, Ce,
            Co, BF.ptr(table), Fn, BF.ptr(weights), p(de_b), p(do_b), stream())
    torch.cuda.synchronize()
    assert int(flag.item()) == 0
    for buf, n, what in ((lse_b, 2 * B * T, "lse"), (loss_b, 1, "loss"), (scale_b, Fn, "scale"),
                         (de_b, B * Ce * T, "d_est"), (do_b, B * Co * T, "d_out")):
        _check_guards(buf, at, n, what)
    loss64, lse64, de64, do64 = _fp64(builder, scaler, est, out, mask, g=0.75)
    b_loss, b_est, b_out = _bounds(builder, scaler, est, out, mask, lse64, de64, do64, loss64, 0.75)
    got_loss = loss_b[at].double()
    assert abs(got_loss - loss64) <= b_loss, (float(got_loss), float(loss64), b_loss)
    got_lse = lse_b[at:at + 2 * B * T].view(2, B, T).double()
    for i, K_ in enumerate((K, 7)):
        assert ((got_lse[i] - lse64[i]).abs() <= _lse_bound(K_, lse64[i])).all(), "lse"
    d_est = de_b[at:at + B * Ce * T].view(B, Ce, T).double()
    d_out = do_b[at:at + B * Co * T].view(B, Co, T).double()
    err_e, err_o = (d_est - de64).abs(), (d_out - do64).abs()
    assert (err_e <= b_est).all(), (err_e - b_est).max().item()
    assert (err_o <= b_out).all(), (err_o - b_out).max().item()


def _run(loss_fn, est, out, mask):
    e = est.clone().requires_grad_(True)
    o = out.clone().requires_grad_(True)
    loss = loss_fn(e, o, mask)
    loss.backward()
    return loss.detach(), e.grad, o.grad


def test_bitwise_repeatable_with_and_without_the_determinism_flag_and_under_bf16_autocast():
    import brainmagick_b200 as bb
    builder, scaler, est, out, mask = _mixed(41, 64, 342, seed=3)
    est, out, mask = est[..., 1:], out[..., 1:], mask[..., 1:]
    loss_fn = bb.FeatureDecodingLoss(builder, scaler)
    first = _run(loss_fn, est, out, mask)
    was = torch.are_deterministic_algorithms_enabled()
    try:
        for flag in (False, True):
            torch.use_deterministic_algorithms(flag)
            for _ in range(2):
                for a, b in zip(first, _run(loss_fn, est, out, mask)):
                    assert torch.equal(a, b)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                under = _run(loss_fn, est, out, mask)
            for a, b in zip(first, under):
                assert a.dtype == torch.float32 and torch.equal(a, b)
    finally:
        torch.use_deterministic_algorithms(was)


@pytest.mark.parametrize("code,exc", [(904, AssertionError), (905, AssertionError), (906, IndexError)])
def test_data_errors_of_a_captured_step_raise_at_the_status_check(code, exc):
    import brainmagick_b200 as bb
    from brainmagick_b200 import functional as BF
    builder, scaler, est, out, mask = _mixed(41, 16, 33, seed=1)
    loss_fn = bb.FeatureDecodingLoss(builder, scaler)
    est = est.clone().requires_grad_(True)
    good_out, good_mask = out.clone(), mask.clone()

    def step():
        est.grad = None
        loss = loss_fn(est, out, mask)
        loss.backward()
        return loss
    graph, _ = _capture(step, [lambda: None])
    if code == 904:
        mask.zero_()
    else:
        out[3, 3, 5] = 41.0 if code == 905 else -3.0
        mask[3, 0, 5] = True
    graph.replay()
    torch.cuda.synchronize()
    with pytest.raises(exc):
        BF.check_tc_status()
    out.copy_(good_out)
    mask.copy_(good_mask)
    graph.replay()
    torch.cuda.synchronize()
    BF.check_tc_status()


# ---- the decoding training step -----------------------------------------------------------------------------------------
DEC_DIMS = dict(CLIP_DIMS, T=342, F=122)       # 120 mel + WordHash-like 41 classes + WordSegment's 2: 122 targets, 163 outputs


def _decoding_features(seed=9):
    gen = torch.Generator().manual_seed(seed)
    builder = Builder([("mel", Feature("mel", 120)), ("hash", Feature("hash", 1, 41)), ("seg", Feature("seg", 1, 2))])
    (wh, ch), (ws, cs) = _class_weights(41, gen), _class_weights(2, gen)
    return builder, Scaler({"hash": wh, "seg": ws}, {"hash": ch, "seg": cs})


def _targets(item, T):
    """the decoding targets of a batch: 120 regression channels and two class channels drawn from the batch's data"""
    feat = item.cand.clone()
    feat[:, 120] = ((item.meg[:, 0] * 1e3).abs().long() % 41).float()
    feat[:, 121] = ((item.meg[:, 1] * 1e3).abs().long() % 2).float()
    mask = (torch.arange(T, device=DEV) < (T - (item.meg[:, :1, :1].abs() * 100).long() % 90))
    return feat, mask


class _DecodingStep:
    """clip_conv SimpleConv -> 163 outputs, FeatureDecodingLoss (weighted), Adam(capturable=True), on static inputs"""

    def __init__(self, dims):
        import brainmagick_b200 as bb
        B, C, T, S = (dims[k] for k in "BCTS")
        torch.manual_seed(0)
        builder, scaler = _decoding_features()
        self.model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=builder.output_dimension, n_subjects=S,
                                   **_clip_conv()).cuda().train()
        self.loss = bb.FeatureDecodingLoss(builder, scaler)
        self.opt = torch.optim.Adam(self.model.parameters(), lr=1e-3, capturable=True)
        self.sb = bb.StaticBatch(B, C, 2 * S, "cuda")
        self.meg = torch.zeros(B, C, T, device=DEV)
        self.feat = torch.zeros(B, builder.dimension, T, device=DEV)
        self.mask = torch.ones(B, 1, T, dtype=torch.bool, device=DEV)
        self.ban = torch.zeros(2, device=DEV)
        self.model.merger.ban_centre_override = self.ban

    def load(self, item):
        self.sb.fill_(item.batch)
        self.meg.copy_(item.meg)
        self.ban.copy_(item.ban)
        feat, mask = _targets(item, self.meg.shape[-1])
        self.feat.copy_(feat)
        self.mask.copy_(mask)

    def step(self):
        self.opt.zero_grad(set_to_none=True)
        est = self.model(dict(meg=self.meg), self.sb)
        loss = self.loss(est, self.feat, self.mask)
        loss.backward()
        self.opt.step()
        return est, loss

    def state(self, est, loss):
        out = dict(est=est.detach().clone(), loss=loss.detach().clone())
        out.update({"model." + k: v.detach().clone() for k, v in self.model.state_dict().items()})
        return out


def test_decoding_step_against_the_fp64_oracle():
    import brainmagick_b200 as bb
    from brainmagick_b200 import functional as BF
    from brainmagick_b200 import synthetic
    from oracle import bm_oracle
    from test_gpu_parity import _build_model, _check_grads
    builder, scaler = _decoding_features()
    B, C, T, S = (DEC_DIMS[k] for k in "BCTS")
    cfg = bm_oracle.Config(in_channels=C, out_channels=builder.output_dimension, n_subjects=S)
    params = bm_oracle.init_state_dict(cfg, seed=11)
    d = bm_oracle.synthetic_batch(cfg, batch=B, T=T, seed=5, n_valid=DEC_DIMS["n_valid"])
    d["rec_positions"] = synthetic.normalised_positions(cfg.n_subjects, C, DEC_DIMS["n_valid"], seed=3)
    gen = torch.Generator().manual_seed(6)
    feat = torch.randn(B, builder.dimension, T, generator=gen)
    feat[:, 120] = torch.randint(0, 41, (B, T), generator=gen).float()
    feat[:, 121] = torch.randint(0, 2, (B, T), generator=gen).float()
    mask = torch.arange(T) < torch.randint(T // 2, T + 1, (B, 1, 1), generator=gen)
    feat, mask = feat.to(DEV), mask.to(DEV)

    # fp64: the oracle's SimpleConv and the reference loss restated in fp64, on the GPU
    p64 = {k: (v.double().to(DEV).requires_grad_(True) if v.is_floating_point() and
               not k.endswith(("running_mean", "running_var")) else v.to(DEV)) for k, v in params.items()}
    est64 = bm_oracle.simpleconv_forward(p64, cfg, d["meg"].double().to(DEV), d["rec_positions"].double().to(DEV),
                                         d["rec_of_sample"].to(DEV), d["subject_index"].to(DEV), True,
                                         d["ban_centre"].double().to(DEV), {})
    loss64 = 0
    for f in builder.values():
        es, os_ = builder.get_slice(f.name, model_output=True), builder.get_slice(f.name)
        if f.categorical:
            loss64 = loss64 + F.cross_entropy(est64[:, es].transpose(1, 2)[mask[:, 0]],
                                              feat[:, os_.start][mask[:, 0]].long(),
                                              scaler.weights[f.name].double().to(DEV))
        else:
            mm = mask.expand_as(est64[:, es])
            loss64 = loss64 + F.mse_loss(est64[:, es][mm], feat[:, os_].double()[mm])
    names = [k for k, v in p64.items() if v.requires_grad]
    grads64 = dict(zip(names, (g.cpu() for g in torch.autograd.grad(loss64, [p64[k] for k in names]))))

    model = _build_model(cfg, params).train()
    meg = d["meg"].to(DEV)
    batch = synthetic.make_batch(meg, d["subject_index"].to(DEV), d["rec_positions"], d["rec_of_sample"])
    model.merger.ban_centre_override = d["ban_centre"]
    est = model(dict(meg=meg), batch)
    loss = bb.FeatureDecodingLoss(builder, scaler)(est, feat, mask)
    loss.backward()
    torch.cuda.synchronize()
    BF.check_tc_status()
    assert rel_err(est.detach(), est64.detach()) < 1e-4
    assert abs(loss.item() - loss64.item()) < 1e-4 * max(1.0, abs(loss64.item()))
    _check_grads(model, grads64, True, 1e-4)


def test_captured_decoding_step_is_bitwise_equal_to_eager(deterministic):
    from brainmagick_b200 import functional as BF
    warm, fresh = _items(DEC_DIMS, 3, 1), _items(DEC_DIMS, 3, 2)
    g, e = _DecodingStep(DEC_DIMS), _DecodingStep(DEC_DIMS)
    graph, (g_est, g_loss) = _capture(g.step, [lambda it=it: g.load(it) for it in warm])
    for it in warm:
        e.load(it)
        e.step()
    for i, it in enumerate(fresh):
        g.load(it)
        graph.replay()
        e.load(it)
        e_est, e_loss = e.step()
        torch.cuda.synchronize()
        _assert_bitwise(g.state(g_est, g_loss), e.state(e_est, e_loss), f"step {i}")
    BF.check_tc_status()
