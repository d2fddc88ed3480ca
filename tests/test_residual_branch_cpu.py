"""CPU checks of ConvSequence's residual-branch options (`scale` = LayerScale, `rewrite`, `post_skip`;
bm/models/common.py:65-76,123-130) against fixtures written by tools/make_residual_golden.py from the verbatim reference
classes: a functional restatement of the layers, seeded construction parity, and the drop-in ConvSequence / DeepMel /
SimpleConv host paths on the ABI emulator with the residual-gain entry points emulated."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import abi_emulator
from abi_emulator import _act, _act_grad, _v
from conftest import load_arrays, rel_err
from input_grad_emulator import InputGradEmulator
from tools.make_residual_golden import SEQ_CASES, SIMPLECONV_CASE, seq_kwargs

TOL = 2e-5


class ResidualEmulator(InputGradEmulator):
    """The emulator (with the input-gradient entry points) plus the residual-gain entry points (include/bm_b200.h), restated
    with torch CPU ops."""

    def bm_bn_act_gain_skip_fwd(self, y, mean, invstd, gamma, beta, x_old, x_new, rows, C, act, slope, scale, boost, post,
                                stream):
        z = _v(y, rows, C)
        if mean is not None:
            z = (z - _v(mean, C)) * _v(invstd, C) * _v(gamma, C) + _v(beta, C)
        a = _act(act, z, slope)
        if scale is not None:
            a = (boost * _v(scale, C)) * a
        if post is not None:
            a = _v(post, C) * a
        if x_old is not None:
            a = a + _v(x_old, rows, C)
        _v(x_new, rows, C).copy_(a)

    def bm_bn_act_gain_skip_bwd(self, g, y, mean, invstd, gamma, beta, batch_stats, rows, C, act, slope, scale, boost, post,
                                sums, dy, dgamma, dbeta, dscale, dpost, stream):
        gg, yy = _v(g, rows, C).clone(), _v(y, rows, C)
        yh = z = yy
        if mean is not None:
            yh = (yy - _v(mean, C)) * _v(invstd, C)
            z = yh * _v(gamma, C) + _v(beta, C)
        S = (gg.double() * _act(act, z, slope).double()).sum(0)
        ls = boost * _v(scale, C) if scale is not None else None
        if dscale is not None:
            _v(dscale, C).copy_((boost * (_v(post, C).double() if post is not None else 1.0) * S).float())
        if dpost is not None:
            _v(dpost, C).copy_(((ls.double() if ls is not None else 1.0) * S).float())
        gb = gg if ls is None else ls * gg
        gb = gb if post is None else _v(post, C) * gb
        dz = gb * _act_grad(act, z, slope)
        if mean is None:
            _v(dy, rows, C).copy_(dz)
            return
        s1, s2 = dz.double().sum(0), (dz * yh).double().sum(0)
        if dbeta is not None:
            _v(dbeta, C).copy_(s1.float())
            _v(dgamma, C).copy_(s2.float())
        v = dz - (s1 / rows).float() - yh * (s2 / rows).float() if batch_stats else dz
        _v(dy, rows, C).copy_(_v(gamma, C) * _v(invstd, C) * v)


@pytest.fixture
def emulated(monkeypatch):
    monkeypatch.setattr(abi_emulator, "Emulator", ResidualEmulator)
    return abi_emulator.emulated


# ---- functional restatement of the reference layers (common.py:98-151) -------------------------------------------------
def seq_oracle(x, p, c, training, new_stats=None):
    """ConvSequence.forward of a SEQ_CASES configuration with the state `p` (key -> tensor); `new_stats` receives the
    running statistics a training forward leaves behind."""
    chans, kernel, growth = c["channels"], c["kernel"], c.get("dilation_growth", 1)
    leak = c.get("leakiness", 0.0)
    act = {"gelu": F.gelu, "relu": F.relu, None: lambda z: F.leaky_relu(z, leak)}[c["activation"]]
    dilation = 1
    for k, (chin, chout) in enumerate(zip(chans[:-1], chans[1:])):
        pre = f"sequence.{k}."
        old = x
        x = F.conv1d(x, p[pre + "0.weight"], p[pre + "0.bias"], padding=(kernel // 2) * dilation, dilation=dilation)
        dilation *= growth
        i = 1
        if c.get("activation_on_last", True) or k < len(chans) - 2:
            if c["batch_norm"]:
                rm, rv = p[pre + f"{i}.running_mean"].clone(), p[pre + f"{i}.running_var"].clone()
                x = F.batch_norm(x, rm, rv, p[pre + f"{i}.weight"], p[pre + f"{i}.bias"], training=training)
                if new_stats is not None:
                    new_stats[pre + f"{i}.running_mean"], new_stats[pre + f"{i}.running_var"] = rm, rv
                i += 1
            x = act(x)
            i += 1
            if c.get("rewrite"):
                x = F.leaky_relu(F.conv1d(x, p[pre + f"{i}.weight"], p[pre + f"{i}.bias"]), leak)
                i += 2
        if chin == chout and c["skip"]:
            if c.get("scale") is not None:
                x = (5 * p[pre + f"{i}.scale"])[:, None] * x
                i += 1
            if c.get("post_skip"):
                x = p[pre + f"{i}.weight"][:, 0, 0][:, None] * x
        if c["skip"] and x.shape == old.shape:
            x = x + old
        if c.get("glu") and (k + 1) % c["glu"] == 0:
            x = F.glu(F.conv1d(x, p[f"glus.{k}.0.weight"], p[f"glus.{k}.0.bias"]), dim=1)
    return x


def _params(g, dtype=torch.float64):
    return {k[2:]: torch.from_numpy(v).to(dtype if v.dtype == np.float32 else torch.from_numpy(v).dtype).clone()
            .requires_grad_(v.dtype == np.float32 and "running" not in k) for k, v in g.items() if k.startswith("p.")}


@pytest.mark.parametrize("case", list(SEQ_CASES))
def test_oracle_matches_reference_fixture(case):
    g, c = load_arrays(case), SEQ_CASES[case]
    for train, tag, out in ((True, "g.", "out"), (False, "ge.", "out_eval")):
        p = _params(g)
        if not train:                                   # the eval pass runs with the statistics of the training step
            for k, v in g.items():
                if k.startswith("bn.") and "running" in k:
                    p[k[3:]] = torch.from_numpy(v).double()
        x = torch.from_numpy(g["x"]).double().requires_grad_(True)
        stats = {}
        y = seq_oracle(x, p, c, train, stats)
        assert rel_err(y.detach(), torch.from_numpy(g[out])) < 1e-5
        (y * torch.from_numpy(g["w_out"]).double()).sum().backward()
        assert rel_err(x.grad, torch.from_numpy(g[tag + "x"])) < 1e-5
        for k, v in p.items():
            ref = torch.from_numpy(g[tag + k]) if v.requires_grad else None
            if ref is not None and ref.norm() < 1e-5:   # conv biases in front of a training BatchNorm: 0 up to rounding
                assert v.grad.abs().max() < 1e-5, (k, tag)
            elif ref is not None:
                assert rel_err(v.grad, ref) < 1e-4, (k, tag)
        for k, v in stats.items():
            assert rel_err(v, torch.from_numpy(g["bn." + k])) < 1e-6, k


@pytest.mark.parametrize("case", list(SEQ_CASES))
def test_seeded_construction_matches_reference(case):
    from brainmagick_b200.common import ConvSequence
    g, c = load_arrays(case), SEQ_CASES[case]
    torch.manual_seed(c["seed"])
    model = ConvSequence(c["channels"], **seq_kwargs(c))          # the options no longer raise
    ref_keys = [k[5:] for k in g if k.startswith("init.")]
    assert list(model.state_dict().keys()) == ref_keys             # same keys, same order
    for k, v in model.state_dict().items():
        assert np.array_equal(v.numpy(), g["init." + k]), k


def test_simpleconv_accepts_the_options():
    import brainmagick_b200 as bb
    from oracle.ref_loader import clip_conv_kwargs
    c = SIMPLECONV_CASE
    kw = clip_conv_kwargs(hidden=c["hidden"], depth=c["depth"], merger_channels=c["MC"], initial_linear=c["IL"],
                          merger_pos_dim=c["P"])
    kw.update(c["extra"])
    model = bb.SimpleConv(in_channels=dict(meg=c["C"]), out_channels=c["F"], n_subjects=c["S"], **kw)
    g = load_arrays("residual_simpleconv")
    assert sorted(model.state_dict().keys()) == sorted(k[2:] for k in g if k.startswith("p."))
    seq = model.encoders["meg"]
    assert seq.has_rewrite == [True] * c["depth"] and seq.has_scale[1:] == [True] * (c["depth"] - 1)


def _seq_step(model, g, emulated):
    """Training step then eval forward / backward of a stand-alone ConvSequence on the emulator -> {name: tensor}."""
    out = {}
    w_out = torch.from_numpy(g["w_out"])
    with emulated():
        for train, tag in ((True, "g."), (False, "ge.")):
            model.train(train)
            model.zero_grad()
            x = torch.from_numpy(g["x"]).clone().requires_grad_(True)
            y = model(x)
            (y * w_out).sum().backward()
            out["out" if train else "out_eval"] = y.detach()
            out[tag + "x"] = x.grad
            for k, v in model.named_parameters():
                out[tag + k] = v.grad.clone()
            if train:
                out.update({"bn." + k: v.clone() for k, v in model.state_dict().items() if "running" in k})
    return out


def _compare(got, g):
    for k, v in got.items():
        ref = torch.from_numpy(g[k])
        if ref.norm() < 1e-5:             # conv biases in front of a training BatchNorm: 0 up to rounding
            assert v.abs().max() < 1e-5, k
        else:
            assert rel_err(v, ref) < 5e-5, (k, rel_err(v, ref))


@pytest.mark.parametrize("case", list(SEQ_CASES))
def test_convsequence_on_the_emulator(case, emulated):
    from brainmagick_b200.common import ConvSequence
    g, c = load_arrays(case), SEQ_CASES[case]
    model = ConvSequence(c["channels"], **seq_kwargs(c))
    model.load_state_dict({k[2:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("p.")}, strict=True)
    _compare(_seq_step(model, g, emulated), g)


def test_deepmel_on_the_emulator(emulated):
    from brainmagick_b200.features import DeepMel
    g, c = load_arrays("residual_all"), SEQ_CASES["residual_all"]
    ch = c["channels"]
    model = DeepMel(ch[0], ch[1], len(ch) - 1, ch[-1], **seq_kwargs(c))
    model.load_state_dict({k[2:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("p.")}, strict=True)
    _compare(_seq_step(model, g, emulated), g)


def test_simpleconv_on_the_emulator(emulated):
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    from oracle.ref_loader import clip_conv_kwargs
    c = SIMPLECONV_CASE
    g = load_arrays("residual_simpleconv")
    kw = clip_conv_kwargs(hidden=c["hidden"], depth=c["depth"], merger_channels=c["MC"], initial_linear=c["IL"],
                          merger_pos_dim=c["P"])
    kw.update(c["extra"])
    model = bb.SimpleConv(in_channels=dict(meg=c["C"]), out_channels=c["F"], n_subjects=c["S"], **kw)
    model.load_state_dict({k[2:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("p.")}, strict=True)
    model.train()
    model.merger.ban_centre_override = torch.from_numpy(g["ban_centre"])
    subj = torch.from_numpy(g["subject_index"])
    meg = torch.from_numpy(g["meg"]).clone().requires_grad_(True)
    batch = synthetic.make_batch(meg.detach(), subj, torch.from_numpy(g["rec_positions"]), subj)
    with emulated():
        est = model(dict(meg=meg), batch)
        loss = bb.ClipLoss()(est, torch.from_numpy(g["candidates"]), torch.ones(len(meg), 1, meg.shape[2], dtype=torch.bool))
        loss.backward()
    assert rel_err(est.detach(), torch.from_numpy(g["estimate"])) < TOL
    assert abs(loss.item() - float(g["loss"])) < 1e-5
    got = {"g." + k: v.grad for k, v in model.named_parameters()}
    got["g.meg"] = meg.grad
    got.update({"bn." + k: v for k, v in model.state_dict().items() if "running" in k})
    _compare(got, g)
