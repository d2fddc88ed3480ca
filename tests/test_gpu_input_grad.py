"""Input gradients on the H100: meg.grad of SimpleConv at the clip_conv widths (tensor-core sensor-mix data gradient) and
of the ablation rows that change the sensor chain, the stand-alone ChannelMerger, and the est / cand gradients of
ClipLoss.get_scores / get_probabilities at the cfg2 size, each against fp64 autograd of the oracle."""
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

TOL = 1e-4


@pytest.fixture
def abi_calls(monkeypatch):
    """Names of the C-ABI entry points called while the test runs (the calls still go to the library)."""
    from brainmagick_b200 import functional as BF
    names, real = [], BF.call

    def spy(name, *args):
        names.append(name)
        return real(name, *args)
    monkeypatch.setattr(BF, "call", spy)
    return names


def _meg_grad_vs_oracle(C, n_valid, change, train, B=2, T=360, seed=23):
    import brainmagick_b200 as bb
    from brainmagick_b200 import functional as BF, synthetic
    from oracle import ablation_oracle, bm_oracle
    Fo, S = 1024, 4
    torch.manual_seed(seed)
    kw = dict(hidden=dict(meg=320), depth=10, dilation_period=5, kernel_size=3, skip=True, subject_layers=True,
              subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=270, merger_channels=270,
              gelu=True, batch_norm=True, merger_pos_dim=2048, merger_dropout=0.2, n_subjects=S)
    kw.update(change)
    model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=Fo, **kw).train(train)
    with torch.no_grad():                            # eval mode reads running statistics that are not the init's 0 / 1
        for name, buf in model.named_buffers():
            if "running_mean" in name:
                buf.normal_(0, 0.1)
            elif "running_var" in name:
                buf.uniform_(0.5, 2.0)
    v = ablation_oracle.Variant(in_channels=C, out_channels=Fo, n_subjects=S)._replace(**change)
    p = {k: t.detach().double() for k, t in model.state_dict().items()}
    g = torch.Generator().manual_seed(seed)
    meg = torch.randn(B, C, T, generator=g)
    cand = torch.randn(B + 1, Fo, T, generator=g)
    subj = torch.tensor([3, 1])[:B]
    pos = synthetic.normalised_positions(S, C, n_valid, seed=4)
    for b in range(B):
        meg[b, n_valid[int(subj[b])]:] = 0
    ban = torch.tensor([0.31, 0.64])
    x = meg.double().requires_grad_(True)
    est_ref = ablation_oracle.forward(p, v, x, pos.double(), subj, subj, training=train, ban_centre=ban.double())
    bm_oracle.clip_loss(est_ref, cand.double()).backward()
    model = model.cuda()
    if model.merger is not None:
        model.merger.ban_centre_override = ban
    xg = meg.cuda().requires_grad_(True)
    est = model(dict(meg=xg), synthetic.make_batch(xg.detach(), subj.cuda(), pos, subj))
    bb.ClipLoss().cuda()(est, cand.cuda(), torch.ones(B, 1, T, dtype=torch.bool, device="cuda")).backward()
    torch.cuda.synchronize()
    BF.check_tc_status()
    grad = xg.grad.cpu()
    assert rel_err(grad, x.grad) < TOL, rel_err(grad, x.grad)
    dead = (pos == -0.1).all(-1)
    if train and model.merger is not None:
        dead = dead | ((pos - ban).norm(dim=-1) <= 0.2)
    if model.merger is not None:
        assert (grad[dead[subj]] == 0).all()
    if "subsample_meg_channels" in change:
        dropped = torch.ones(C, dtype=torch.bool)
        dropped[model.subsampled_meg_channels] = False
        assert (grad[:, dropped] == 0).all()
    return grad


@pytest.mark.parametrize("C,n_valid", [(208, (208, 208, 208, 208)), (273, (273, 200, 150, 273))], ids=["C208", "C273"])
@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
def test_clip_conv_meg_grad_on_tensor_cores(C, n_valid, train, abi_calls):
    _meg_grad_vs_oracle(C, n_valid, {}, train)
    assert "bm_tc_sensor_mix_bwd_data" in abi_calls and "bm_sensor_mix_bwd_data" not in abi_calls


@pytest.mark.parametrize("change", [dict(merger=False), dict(initial_linear=0), dict(subject_layers=False),
                                    dict(subject_layers=False, subject_dim=64), dict(subsample_meg_channels=150)],
                         ids=lambda c: ",".join(f"{k}={v}" for k, v in c.items()))
def test_ablation_rows_meg_grad(change):
    _meg_grad_vs_oracle(208, (208, 150, 208, 97), change, True)


def test_frozen_model_attribution_pass():
    """Eval mode, every parameter frozen: only meg receives a gradient."""
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    torch.manual_seed(3)
    model = bb.SimpleConv(in_channels=dict(meg=208), out_channels=1024, hidden=dict(meg=320), depth=10, dilation_period=5,
                          kernel_size=3, skip=True, subject_layers=True, subject_dim=0, complex_out=True, glu=2,
                          glu_context=1, merger=True, initial_linear=270, merger_channels=270, gelu=True, batch_norm=True,
                          merger_pos_dim=2048, n_subjects=4).cuda().eval().requires_grad_(False)
    meg = torch.randn(3, 208, 200, device="cuda", requires_grad=True)
    subj = torch.tensor([0, 2, 3])
    est = model(dict(meg=meg), synthetic.make_batch(meg.detach(), subj.cuda(), synthetic.normalised_positions(4, 208), subj))
    est.square().sum().backward()
    assert meg.grad is not None and torch.isfinite(meg.grad).all() and meg.grad.abs().sum() > 0
    assert all(p.grad is None for p in model.parameters())


def test_standalone_channel_merger_meg_grad():
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    from oracle import bm_oracle
    g = torch.Generator().manual_seed(9)
    B, C, T, O = 4, 273, 360, 270
    meg = torch.randn(B, C, T, generator=g)
    rec_of_sample = torch.tensor([1, 0, 2, 1])
    pos = synthetic.normalised_positions(3, C, n_valid=(273, 208, 150), seed=5)
    merger = bb.ChannelMerger(O, pos_dim=2048, dropout=0.2).train()
    ban = torch.tensor([0.45, 0.5])
    merger.ban_centre_override = ban
    gout = torch.randn(B, O, T, generator=g)
    x = meg.double().requires_grad_(True)
    att = bm_oracle.attention_weights(pos.double(), merger.heads.detach().double(), ban.double(), 0.2)
    torch.einsum("bct,boc->bot", x, att[rec_of_sample]).backward(gout.double())
    merger = merger.cuda()
    m = meg.cuda().requires_grad_(True)
    merger(m, synthetic.make_batch(m.detach(), rec_of_sample.cuda(), pos, rec_of_sample)).backward(gout.cuda())
    grad = m.grad.cpu()
    assert rel_err(grad, x.grad) < TOL, rel_err(grad, x.grad)
    dead = ((pos == -0.1).all(-1) | ((pos - ban).norm(dim=-1) <= 0.2))[rec_of_sample]
    assert dead.any() and (grad[dead] == 0).all()


@pytest.mark.parametrize("name", ["get_scores", "get_probabilities"])
def test_clip_scores_grads_at_cfg2_size(name):
    """Bn = Bc = 256, K = F*T = 368 640; candidate 5 is all zeros (its gradient is the 1e8-scaled sum of estimates)."""
    import brainmagick_b200 as bb
    from brainmagick_b200 import functional as BF
    g = torch.Generator(device="cuda").manual_seed(31)
    Bn, Bc, F, T = 256, 256, 1024, 360
    est = torch.randn(Bn, F, T, device="cuda", generator=g)
    cand = torch.randn(Bc, F, T, device="cuda", generator=g)
    cand[5] = 0
    up = torch.randn(Bn, Bc, device="cuda", generator=g)
    e, c = est.double().requires_grad_(True), cand.double().requires_grad_(True)
    inv = 1 / (1e-8 + c.norm(dim=(1, 2), p=2))
    ref = torch.einsum("bct,oct,o->bo", e, c, inv)
    if name == "get_probabilities":
        ref = torch.softmax(ref, dim=1)
    ref.backward(up.double())
    e32, c32 = est.clone().requires_grad_(True), cand.clone().requires_grad_(True)
    out = getattr(bb.ClipLoss(), name)(e32, c32)
    out.backward(up)
    torch.cuda.synchronize()
    BF.check_tc_status()
    with torch.no_grad():
        assert torch.equal(out.detach(), getattr(bb.ClipLoss(), name)(est, cand))       # same forward call, same values
    assert rel_err(e32.grad, e.grad) < TOL, rel_err(e32.grad, e.grad)
    live = torch.ones(Bc, dtype=torch.bool, device="cuda")
    live[5] = False
    assert rel_err(c32.grad[live], c.grad[live]) < TOL, rel_err(c32.grad[live], c.grad[live])
    assert rel_err(c32.grad[5], c.grad[5]) < TOL
