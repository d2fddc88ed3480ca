"""L1Loss / L2Loss on the H100:

  * the loss and both gradients against fp64 per element, at T not a multiple of 4, odd element offsets, every broadcast of
    the mask, the regression baseline's shapes (cfg4: 256 x 120 x 360) and the encoding task's (256 x 208 x 324, a view of
    T = 360 cropped by meg_init = 0.3 s at 120 Hz), exact ties, NaN inputs and an empty mask (against torch's masked loss);
  * bitwise equal results across repeated calls, with and without torch.use_deterministic_algorithms, and under bf16
    autocast;
  * captured training steps (forward, loss, backward, Adam(capturable=True)) replayed on fresh batches, bitwise equal to the
    same steps run eagerly under the determinism flag: the regression baseline (clip_conv SimpleConv with 120 outputs, L2Loss,
    a ragged mask) and an encoding model (meg 208 + features 120, complex_out, L1Loss on estimate[..., limit:]);
  * one eager training step with the drop-in loss: every parameter gradient within 1e-5 of the step with torch's loss over
    estimate[mask] (bm/losses.py:11-26).
"""
import pytest
import torch

from conftest import rel_err
from test_gpu_cuda_graph import CLIP_DIMS, _assert_bitwise, _capture, _clip_conv, _items, deterministic  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _losses(kind):
    import brainmagick_b200 as bb
    return (bb.L1Loss(), torch.nn.L1Loss()) if kind == "l1" else (bb.L2Loss(), torch.nn.MSELoss())


def _fp64(kind, est, out, mask, g=1.0):
    """(loss, d_est, d_out) in fp64 from the definition"""
    m = mask.expand_as(est)
    d = est.double() - out.double()
    n = int(m.sum())
    loss = (d.abs() if kind == "l1" else d * d)[m].sum() / n
    grad = torch.where(m, (torch.sign(d) if kind == "l1" else 2 * d) * g / n, torch.zeros((), dtype=torch.float64,
                                                                                           device=est.device))
    return loss, grad, -grad


def _run(kind, est, out, mask, g=1.0):
    e, o = est.detach().requires_grad_(True), out.detach().requires_grad_(True)
    loss = _losses(kind)[0](e, o, mask)
    loss.backward(torch.tensor(g, device=DEV))
    return loss.detach(), e.grad, o.grad


def _check_fp64(kind, est, out, mask, g=0.75):
    loss, d_est, d_out = _run(kind, est, out, mask, g)
    w_loss, w_est, w_out = _fp64(kind, est, out, mask, g)
    assert abs(loss.item() - w_loss.item()) <= 2 ** -22 * abs(w_loss.item())
    for got, want in ((d_est, w_est), (d_out, w_out)):
        assert got.shape == want.shape and got.is_contiguous()
        err = (got.double() - want).abs()
        assert (err <= 8 * 2 ** -24 * want.abs() + 1e-30).all(), err.max().item()
        assert torch.equal(got == 0, want == 0)         # masked-out entries and ties exactly zero


def _data(shape, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, generator=g, device=DEV), torch.randn(shape, generator=g, device=DEV)


@pytest.mark.parametrize("kind", ["l1", "l2"])
@pytest.mark.parametrize("T", [1, 3, 45, 360])
def test_against_fp64_at_t_not_a_multiple_of_4(kind, T):
    est, out = _data((5, 7, T), 1)
    mask = torch.rand(5, 1, T, device=DEV) > 0.3
    mask[0, 0, 0] = True
    _check_fp64(kind, est, out, mask)


@pytest.mark.parametrize("kind", ["l1", "l2"])
@pytest.mark.parametrize("offset", [0, 1, 2, 3, 5])
def test_views_at_odd_element_offsets_are_read_in_place(kind, offset):
    est_full, out_full = _data((6, 9, 64), 2)
    est = est_full[1:, 2:, offset:offset + 49]
    out = out_full[:5, 1:8, 64 - 49 - offset:64 - offset]
    mask = (torch.rand(6, 1, 64, device=DEV) > 0.25)[1:, :, offset:offset + 49]
    _check_fp64(kind, est, out, mask)


@pytest.mark.parametrize("kind", ["l1", "l2"])
@pytest.mark.parametrize("shape", [(4, 6, 23), (4, 1, 23), (1, 1, 23), (4, 6, 1), (1, 6, 1), (23,), (6, 23)])
def test_every_mask_broadcast(kind, shape):
    est, out = _data((4, 6, 23), 3)
    mask = torch.rand(shape, device=DEV) > 0.4
    mask.view(-1)[0] = True
    _check_fp64(kind, est, out, mask)


def _crop(t, limit):
    return t[..., limit:]


@pytest.mark.parametrize("kind", ["l1", "l2"])
@pytest.mark.parametrize("case", ["cfg4_regression", "encode_cropped"])
def test_full_size_shapes(kind, case):
    if case == "cfg4_regression":
        est, out = _data((256, 120, 360), 4)
        mask = torch.ones(256, 1, 360, dtype=torch.bool, device=DEV)
        mask[::3, :, 300:] = False                      # ragged, as with task.mask_loss
    else:
        limit = int(0.3 * 120)
        est_full, out_full = _data((256, 208, 360), 5)
        est, out = _crop(est_full, limit), _crop(out_full, limit)
        mask = _crop(torch.ones(256, 1, 360, dtype=torch.bool, device=DEV), limit)
        assert est.shape == (256, 208, 324)
    _check_fp64(kind, est, out, mask)


@pytest.mark.parametrize("kind", ["l1", "l2"])
def test_ties_nan_and_empty_mask_as_torch(kind):
    ref = _losses(kind)[1]
    est, out = _data((3, 4, 17), 6)
    out = torch.where(torch.rand(3, 4, 17, device=DEV) < 0.4, est, out)          # exact ties
    _check_fp64(kind, est, out, torch.ones(3, 1, 17, dtype=torch.bool, device=DEV))
    nan_est = est.clone()
    nan_est[1, 2, 5] = float("nan")
    nan_est[2, 0, 3] = float("inf")
    masks = {"all": torch.ones(3, 1, 17, dtype=torch.bool, device=DEV),
             "nan_out": torch.ones(3, 1, 17, dtype=torch.bool, device=DEV),
             "empty": torch.zeros(3, 1, 17, dtype=torch.bool, device=DEV)}
    masks["nan_out"][1, 0, 5] = masks["nan_out"][2, 0, 3] = False       # the non-finite entries masked out
    for name, mask in masks.items():
        got = _run(kind, nan_est, out, mask)
        e, o = nan_est.clone().requires_grad_(True), out.clone().requires_grad_(True)
        m = mask.expand_as(e)
        want_loss = ref(e[m], o[m])
        want_loss.backward()
        for a, b in zip(got, (want_loss.detach(), e.grad, o.grad)):
            torch.testing.assert_close(a, b, rtol=1e-6, atol=0, equal_nan=True, msg=name)
        if name == "empty":
            assert torch.isnan(got[0]) and not got[1].any() and not got[2].any()
        if name == "nan_out":
            assert torch.isfinite(got[0]) and torch.isfinite(got[1]).all()


@pytest.mark.parametrize("kind", ["l1", "l2"])
def test_bitwise_repeatable_with_and_without_the_determinism_flag_and_under_bf16_autocast(kind):
    est_full, out_full = _data((256, 208, 360), 7)
    est, out = est_full[..., 36:], out_full[..., 36:]
    mask = torch.rand(256, 1, 360, device=DEV)[..., 36:] > 0.1
    first = _run(kind, est, out, mask)
    was = torch.are_deterministic_algorithms_enabled()
    try:
        for flag in (False, True):
            torch.use_deterministic_algorithms(flag)
            for _ in range(3):
                for a, b in zip(first, _run(kind, est, out, mask)):
                    assert torch.equal(a, b)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                under = _run(kind, est, out, mask)
            for a, b in zip(first, under):
                assert a.dtype == torch.float32 and torch.equal(a, b)
    finally:
        torch.use_deterministic_algorithms(was)


# ---- training steps ---------------------------------------------------------------------------------------------------
ENC_DIMS = dict(CLIP_DIMS, F=120)             # B 64, meg 208, T 360; F: the regression targets / the encoding features
LIMIT = int(0.3 * 120)                        # the encode task's meg_init = 0.3 s at 120 Hz (bm/solver.py:287-293)


class _Step:
    """A regression ("regression": clip_conv SimpleConv -> 120 mel, L2Loss, ragged mask) or encoding ("encode": meg 208 +
    features 120, complex_out, L1Loss on estimate[..., limit:] against the MEG) training step reading static inputs."""

    def __init__(self, task, dims, loss=None):
        import brainmagick_b200 as bb
        B, C, T, F, S = (dims[k] for k in "BCTFS")
        self.task = task
        torch.manual_seed(0)
        if task == "regression":
            self.model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, n_subjects=S, **_clip_conv())
            self.loss = loss or bb.L2Loss()
        else:
            kw = _clip_conv()
            kw["hidden"] = dict(meg=320, features=320)
            self.model = bb.SimpleConv(in_channels=dict(meg=C, features=F), out_channels=C, n_subjects=S, **kw)
            self.loss = loss or bb.L1Loss()
        self.model = self.model.cuda().train()
        self.opt = torch.optim.Adam(self.model.parameters(), lr=1e-3, capturable=True)
        self.sb = bb.StaticBatch(B, C, 2 * S, "cuda")
        self.meg = torch.zeros(B, C, T, device=DEV)
        self.feat = torch.zeros(B, F, T, device=DEV)
        self.mask = torch.ones(B, 1, T, dtype=torch.bool, device=DEV)
        self.ban = torch.zeros(2, device=DEV)
        self.model.merger.ban_centre_override = self.ban
        self.in_mask = torch.zeros(T, device=DEV)
        self.in_mask[:LIMIT] = 1

    def load(self, item):
        self.sb.fill_(item.batch)
        self.meg.copy_(item.meg)
        self.feat.copy_(item.cand)
        self.ban.copy_(item.ban)
        T = self.mask.shape[-1]
        ragged = torch.arange(T, device=DEV) < (T - (item.meg[:, :1, :1].abs() * 100).long() % 90)   # per-sample ends
        self.mask.copy_(ragged if self.task == "regression" else torch.ones_like(self.mask))

    def forward(self):
        if self.task == "regression":
            return self.model(dict(meg=self.meg), self.sb), self.feat, self.mask
        est = self.model(dict(meg=self.in_mask * self.meg, features=self.feat), self.sb)      # bm/solver.py:291
        return est[..., LIMIT:], self.meg[..., LIMIT:], self.mask[..., LIMIT:]

    def step(self):
        self.opt.zero_grad(set_to_none=True)
        est, out, mask = self.forward()
        loss = self.loss(est, out, mask)
        loss.backward()
        self.opt.step()
        return est, loss

    def state(self, est, loss):
        out = dict(est=est.detach().clone(), loss=loss.detach().clone())
        out.update({"model." + k: v.detach().clone() for k, v in self.model.state_dict().items()})
        return out


@pytest.mark.parametrize("task", ["regression", "encode"])
def test_captured_step_is_bitwise_equal_to_eager(task, deterministic):
    from brainmagick_b200 import functional as BF
    warm, fresh = _items(ENC_DIMS, 3, 1), _items(ENC_DIMS, 3, 2)
    g, e = _Step(task, ENC_DIMS), _Step(task, ENC_DIMS)
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


class _TorchMaskedLoss(torch.nn.Module):
    """bm/losses.py:11-14 with torch's loss: boolean-mask indexing, then L1Loss / MSELoss"""

    def __init__(self, loss):
        super().__init__()
        self._loss = loss

    def forward(self, estimate, output, mask):
        m = mask.expand_as(estimate)
        return self._loss(estimate[m], output[m])


@pytest.mark.parametrize("task", ["regression", "encode"])
def test_eager_step_gradients_match_torchs_masked_loss(task):
    dims = dict(ENC_DIMS, B=16)
    item = _items(dims, 1, 5)[0]
    grads = []
    for torch_loss in (False, True):
        ref = _TorchMaskedLoss(torch.nn.MSELoss() if task == "regression" else torch.nn.L1Loss())
        s = _Step(task, dims, loss=ref if torch_loss else None)
        s.load(item)
        s.opt.zero_grad(set_to_none=True)
        s.loss(*s.forward()).backward()
        grads.append({k: p.grad.double() for k, p in s.model.named_parameters()})
    drop, want = grads
    scale = max(v.norm().item() for k, v in want.items() if k.endswith("weight"))
    for k in want:
        if want[k].norm() < 1e-5 * scale:     # rounding noise around zero (a conv bias in front of a BatchNorm)
            assert (drop[k] - want[k]).abs().max().item() < 1e-5 * scale, k
        else:
            assert rel_err(drop[k], want[k]) < 1e-5, (k, rel_err(drop[k], want[k]))
