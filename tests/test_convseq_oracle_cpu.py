"""CPU checks that pin the ConvSequence oracle (oracle/deepmel_oracle.py) to the verbatim reference class at the options
DeepMel's own settings leave out (oracle/make_golden.py CONVSEQ_CASES): kernel 1, BatchNorm + activation on the last layer,
ReLU / LeakyReLU / GELU / LeakyReLU(leakiness), no skip, skips across width changes, GLU contexts 0 and 1, dilations
reaching past T, no BatchNorm -- a training step and an eval-mode forward and backward each."""
import numpy as np
import pytest
import torch

from conftest import load_arrays, rel_err
from oracle import deepmel_oracle
from oracle.make_golden import CONVSEQ_CASES


def convseq_spec(case):
    c = CONVSEQ_CASES[case]
    return deepmel_oracle.convseq_spec(c["channels"], c["activation"], **c["kw"])


def oracle_run(spec, params, x, gout, training, dtype=torch.float64):
    """One forward/backward of the oracle in `dtype` -> (out, dL/dx, {param: grad}, new running statistics)."""
    p = {k: v.to(dtype).clone().requires_grad_("running" not in k and "num_batches" not in k)
         for k, v in params.items() if v.is_floating_point()}
    xx = x.to(dtype).clone().requires_grad_(True)
    stats = {}
    out = deepmel_oracle.conv_sequence(xx, p, spec, training=training, new_stats=stats)
    out.backward(gout.to(dtype))
    grads = {k: v.grad for k, v in p.items() if v.requires_grad}
    return out.detach(), xx.grad, grads, {k: v.detach() for k, v in stats.items()}


@pytest.mark.parametrize("case", list(CONVSEQ_CASES))
def test_convseq_oracle_matches_reference(case):
    g = load_arrays(case)
    spec = convseq_spec(case)
    params = {k[2:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("p.")}
    x = torch.from_numpy(g["x"])
    wscale = max(float(np.linalg.norm(v)) for k, v in g.items() if k.startswith("g.") and k.endswith("weight"))
    for mode, pre in (("train", "g."), ("eval", "ge.")):
        p = dict(params)
        if mode == "eval":      # eval mode on the running statistics the training step left behind
            p.update({k[3:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("bn.")})
        out, dx, grads, stats = oracle_run(spec, p, x, torch.from_numpy(g["gout" if mode == "train" else "gout_eval"]),
                                           training=mode == "train", dtype=torch.float32)
        assert rel_err(out, torch.from_numpy(g["out" if mode == "train" else "out_eval"])) < 2e-6, mode
        assert rel_err(dx, torch.from_numpy(g[pre + "x"])) < 1e-5, mode
        names = sorted(k[len(pre):] for k in g if k.startswith(pre) and k != pre + "x")
        assert sorted(grads) == names, mode
        for k in names:
            ref = torch.from_numpy(g[pre + k])
            if ref.norm() < 1e-6 * wscale:      # a conv bias in front of a training BatchNorm: 0 up to rounding
                assert grads[k].abs().max() < 1e-5 * wscale, (mode, k)
            else:
                assert rel_err(grads[k], ref) < 2e-5, (mode, k)
        if mode == "train":
            assert sorted(stats) == sorted(k[3:] for k in g if k.startswith("bn.") and "running" in k)
            for k, v in stats.items():
                assert rel_err(v, torch.from_numpy(g["bn." + k])) < 1e-6, k


def test_convseq_cases_cover_the_options():
    """the fixture table keeps covering every option it was written for"""
    specs = [convseq_spec(c) for c in CONVSEQ_CASES]
    acts = {CONVSEQ_CASES[c]["activation"] for c in CONVSEQ_CASES}
    assert acts == {None, "relu", "leaky_relu", "gelu"}
    assert any(s.kernel == 1 for s in specs)
    assert any(s.activation_on_last and s.batch_norm for s in specs)
    assert any(not s.skip for s in specs) and any(not s.batch_norm for s in specs)
    assert {s.glu_context for s in specs if s.glu} == {0, 1}
    assert any(s.skip and len(set(s.channels[1:])) > 1 for s in specs)           # a skip where the width changes
    assert any(max(s.dilations()) >= CONVSEQ_CASES[c]["T"] for c, s in zip(CONVSEQ_CASES, specs))
