"""CPU checks of SimpleConv over several input streams (the encoding configuration of bm/train.py:61-67: `features` next
to `meg`, `concatenate`, `linear_out`; bm/models/simpleconv.py:150-249) against the fixtures tools/make_encode_golden.py
writes from the verbatim reference: seeded construction and state_dict, the fp64 restatement (oracle/encode_oracle.py),
the drop-in end to end on the ABI emulator, and the host call streams (tests/golden/abi_trace_encode.json) of full and
frozen steps at the widths an encoding model runs."""
import json
import os

import numpy as np
import pytest
import torch

import encode_emulator
from conftest import GOLDEN_DIR, load_arrays, rel_err
from oracle import encode_oracle
from tools.make_encode_golden import CASES

TRACE = os.path.join(GOLDEN_DIR, "abi_trace_encode.json")


def _model(v):
    import brainmagick_b200 as bb
    return bb.SimpleConv(**v.kwargs())


def _state(g, prefix="p."):
    return {k[len(prefix):]: torch.from_numpy(t) for k, t in g.items() if k.startswith(prefix)}


@pytest.mark.parametrize("case", list(CASES))
def test_seeded_construction_matches_reference(case):
    v, _, _, seed = CASES[case]
    g = load_arrays(case)
    torch.manual_seed(seed)
    model = _model(v)
    ref_keys = [k[5:] for k in g if k.startswith("init.")]
    assert list(model.state_dict().keys()) == ref_keys                # same keys, same order
    for k, t in model.state_dict().items():
        assert np.array_equal(t.numpy(), g["init." + k]), k
    model.load_state_dict(_state(g), strict=True)                     # a reference checkpoint loads


def _compare(got: dict, g, tol):
    for k, t in got.items():
        ref = torch.from_numpy(g[k])
        if ref.abs().max() < 1e-4:        # conv biases in front of a training BatchNorm: 0 up to rounding
            assert t.abs().max() < 1e-4, k
        else:
            assert rel_err(t, ref) < tol, (k, rel_err(t, ref))


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_reference_fixture(case):
    v = CASES[case][0]
    g = load_arrays(case)
    p = {k: t.double().requires_grad_(t.dtype == torch.float32 and "running" not in k) for k, t in _state(g).items()}
    inputs = {name: torch.from_numpy(g["in." + name]).double().requires_grad_(True) for name in v.in_channels}
    subj = torch.from_numpy(g["subject_index"]).long()
    pos = torch.from_numpy(g["rec_positions"]).double()
    stats = {}
    out = encode_oracle.forward(p, v, inputs, pos, subj, subj, True, torch.from_numpy(g["ban_centre"]).double(), stats)
    (out * torch.from_numpy(g["w_out"]).double()).sum().backward()
    got = {"out": out.detach()}
    got.update({"g.in." + n: t.grad for n, t in inputs.items()})
    got.update({"g." + k: t.grad for k, t in p.items() if t.requires_grad})
    got.update({"bn." + k: t for k, t in stats.items()})
    _compare(got, g, 1e-5)
    p_eval = {k: t.detach() for k, t in p.items()}
    p_eval.update({k[3:]: torch.from_numpy(t).double() for k, t in g.items() if k.startswith("bn.") and "running" in k})
    with torch.no_grad():
        out_eval = encode_oracle.forward(p_eval, v, {n: t.detach() for n, t in inputs.items()}, pos, subj, subj, False)
    assert rel_err(out_eval, torch.from_numpy(g["out_eval"])) < 1e-5


def _batch(g):
    from brainmagick_b200 import synthetic
    subj = torch.from_numpy(g["subject_index"])
    return synthetic.make_batch(torch.from_numpy(g["in.meg"]), subj, torch.from_numpy(g["rec_positions"]), subj)


def _cropped(t, offset=3):
    """t as the solver's offset crop hands it over: a view into a longer window"""
    B, C, T = t.shape
    full = torch.randn(B, C, T + 2 * offset)
    full[:, :, offset:offset + T] = t
    return full[:, :, offset:offset + T]


@pytest.mark.parametrize("case", list(CASES))
def test_drop_in_on_the_emulator(case):
    v = CASES[case][0]
    g = load_arrays(case)
    model = _model(v)
    model.load_state_dict(_state(g), strict=True)
    model.train()
    model.merger.ban_centre_override = torch.from_numpy(g["ban_centre"])
    leaves = {n: _cropped(torch.from_numpy(g["in." + n])).requires_grad_(True) if n != "meg" else
              torch.from_numpy(g["in.meg"]).clone().requires_grad_(True) for n in v.in_channels}
    with encode_emulator.emulated():
        out = model(dict(leaves), _batch(g))
        (out * torch.from_numpy(g["w_out"])).sum().backward()
        model.eval()
        with torch.no_grad():
            out_eval = model({n: torch.from_numpy(g["in." + n]) for n in v.in_channels}, _batch(g))
    got = {"out": out.detach(), "out_eval": out_eval}
    got.update({"g.in." + n: t.grad for n, t in leaves.items()})
    got.update({"g." + k: t.grad for k, t in model.named_parameters()})
    got.update({"bn." + k: t for k, t in model.state_dict().items() if "running" in k or "num_batches" in k})
    _compare(got, g, 5e-5)


def test_constructor_rejections():
    import brainmagick_b200 as bb
    v = CASES["encode_two_complex"][0]
    with pytest.raises(NotImplementedError, match="growth"):
        bb.SimpleConv(**dict(v.kwargs(), growth=1.5))
    with pytest.raises(AssertionError):
        _model(v._replace(linear_out=True, complex_out=True))
    with pytest.raises(AssertionError):                  # two encoders need a head (simpleconv.py:190-191)
        _model(v._replace(complex_out=False))
    with pytest.raises(NotImplementedError, match="meg"):
        bb.SimpleConv(**dict(v.kwargs(), in_channels=dict(features=7), hidden=dict(features=12)))
    five = dict(meg=10, a=3, b=3, c=3, d=3)                 # the channel join takes at most 4 sources
    for concatenate, head in ((True, dict(complex_out=False)), (False, dict(complex_out=True))):
        with pytest.raises(NotImplementedError, match="at most 4"):
            bb.SimpleConv(**dict(v.kwargs(), in_channels=dict(five), hidden={k: 8 for k in five}, concatenate=concatenate,
                                 **head))


@pytest.mark.parametrize("case", ["encode_two_complex", "encode_concat_bare"])
@pytest.mark.parametrize("width", [5, 9])
def test_a_stream_of_another_width_is_rejected(case, width):
    """a features tensor whose channel count differs from in_channels["features"] raises, as the reference's conv does"""
    v = CASES[case][0]
    g = load_arrays(case)
    model = _model(v)
    model.load_state_dict(_state(g), strict=True)
    inputs = {"meg": torch.from_numpy(g["in.meg"]), "features": torch.randn(4, width, 22)}
    with encode_emulator.emulated(), pytest.raises(ValueError, match="channels"):
        model(inputs, _batch(g))


# ---- host call streams ------------------------------------------------------------------------------------------------
def _encode_step(head: str, freeze: str = "", concatenate=False, B=4, C=208, T=360, Fin=120, hidden=320, S=4):
    """One training step of an encoding model (L1 to the MEG itself) at real widths, with some tensors frozen:
    freeze "features": the features encoder; "head": everything but the head; "input": every parameter (features.grad)."""
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic

    def run():
        torch.manual_seed(0)
        v = encode_oracle.EncodeVariant(in_channels=dict(meg=C, features=Fin), hidden=dict(meg=hidden, features=hidden),
                                        out_channels=C, n_subjects=S, concatenate=concatenate,
                                        linear_out=head == "linear", complex_out=head == "complex")
        model = bb.SimpleConv(**v.kwargs()).train()
        if freeze == "features":
            model.encoders["features"].requires_grad_(False)
        elif freeze in ("head", "input"):
            model.requires_grad_(False)
            if freeze == "head":
                model.final.requires_grad_(True)
        subj = torch.randint(0, S, (B,))
        meg = torch.randn(B, C, T)
        feats = torch.randn(B, Fin, T + 10)[:, :, 5:5 + T].requires_grad_(freeze == "input")
        batch = synthetic.make_batch(meg, subj, synthetic.normalised_positions(S, C), subj)
        out = model(dict(meg=meg, features=feats), batch)
        out.abs().sum().backward()
    return encode_emulator.record(run)


def all_traces():
    return {
        "complex": _encode_step("complex"),
        "linear": _encode_step("linear"),
        "concat_linear": _encode_step("linear", concatenate=True),
        "concat_bare": _encode_step("bare", concatenate=True),
        "complex.features_frozen": _encode_step("complex", "features"),
        "complex.head_only": _encode_step("complex", "head"),
        "complex.input_grad_only": _encode_step("complex", "input"),
    }


def test_call_streams_match_the_fixture():
    with open(TRACE) as f:
        want = json.load(f)
    got = all_traces()
    assert list(got) == list(want)
    for name in want:
        assert got[name] == want[name], name


def test_frozen_call_streams_skip_the_frozen_work():
    with open(TRACE) as f:
        t = json.load(f)

    def names(trace):
        return [c[0] for c in trace]
    full = names(t["complex"])
    wgrad = ("bm_tc_wgrad", "bm_tc_wgrad_conv", "bm_conv1d_bwd_weight", "bm_head_bwd_params")
    assert len(names(t["complex.features_frozen"])) < len(full)
    head_only = names(t["complex.head_only"])
    assert "bm_channel_split" not in head_only and "bm_conv1d_bwd_data" not in head_only
    inp = names(t["complex.input_grad_only"])
    assert "bm_channel_split" in inp and not any(n.startswith(wgrad) for n in inp)
    assert "bm_attention_weights_bwd" not in inp                # the sensor front is not backpropagated


if __name__ == "__main__":                      # (re)writes the call-stream fixture
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    with open(TRACE, "w") as f:
        json.dump(all_traces(), f)
