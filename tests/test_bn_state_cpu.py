"""CPU checks of BatchNorm layers that follow their own module (per-layer train / eval, eps, momentum, and the cumulative
average of momentum=None) in SimpleConv, ConvSequence and DeepMel: the per-layer oracle (tests/bn_state_oracle.py) and the
drop-ins on the ABI emulator against fixtures written by tools/make_bn_state_golden.py from the verbatim reference, the
plan and call stream of uniform models, the rejection of track_running_stats=False, and two gloo ranks of a converted
DeepMel with one eval-mode layer against one process on the concatenated batch."""
import contextlib
import os
import sys
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import bn_state_oracle as O
import encode_emulator
import frozen_emulator
from bn_state_emulator import CumulativeFinalize
from conftest import load_arrays, rel_err
from oracle import deepmel_oracle
from tools.make_bn_state_golden import CASES, DEEPMEL, SETUPS, streams

HERE = os.path.dirname(os.path.abspath(__file__))


class _Emulator(CumulativeFinalize, frozen_emulator.FrozenEmulator, encode_emulator.EncodeEmulator):
    """the cumulative-average finalize, frozen BatchNorm parameters (no dgamma / dbeta reduction) and the channel join of
    several input streams"""


@contextlib.contextmanager
def emulated():
    with frozen_emulator.emulated(_Emulator) as emu, encode_emulator._patched_view_ptr(encode_emulator._span):
        yield emu


def make_model(c, sd=None):
    """The drop-in module of a case, with the state `sd` (a state_dict) and the case's layer modes and settings."""
    import brainmagick_b200 as bb
    model = bb.DeepMel(**c.get("deepmel", DEEPMEL)) if c["model"] == "deepmel" else bb.SimpleConv(**c["model"].kwargs())
    if sd is not None:
        model.load_state_dict(sd, strict=True)
    SETUPS[c["setup"]](model)
    return model


def _batch(meg, subj, pos):
    from brainmagick_b200 import synthetic
    return synthetic.make_batch(meg.detach(), subj, pos, subj)


def dropin_steps(model, c, steps, subj=None, pos=None):
    """steps: [(inputs, w, ban)] -> {"s{i}.out", "s{i}.g.<param>", "s{i}.g.in.<stream>", "bn.<buffer>"} of the training
    steps on the drop-in module (whatever device its tensors are on), then "out_eval" on the first step's inputs."""
    got = {}
    mode = {m: m.training for m in model.modules()}
    for i, (inputs, w, ban) in enumerate(steps):
        model.zero_grad(set_to_none=True)
        leaves = {s: t.clone().requires_grad_(True) for s, t in inputs.items()}
        if c["model"] == "deepmel":
            out = model(leaves["x"])
        else:
            model.merger.ban_centre_override = ban
            out = model(dict(leaves), _batch(leaves["meg"], subj, pos))
        (out * w).sum().backward()
        got[f"s{i}.out"] = out.detach().clone()
        got.update({f"s{i}.g.in.{s}": t.grad for s, t in leaves.items()})
        got.update({f"s{i}.g.{k}": t.grad.clone() for k, t in model.named_parameters() if t.grad is not None})
    got.update({"bn." + k: t.clone() for k, t in model.state_dict().items() if "running" in k or "num_batches" in k})
    model.eval()
    with torch.no_grad():
        inputs = steps[0][0]
        got["out_eval"] = model(inputs["x"]) if c["model"] == "deepmel" else model(dict(inputs), _batch(inputs["meg"], subj, pos))
    for m, training in mode.items():
        m.train(training)
    return got


def deepmel_spec(kw):
    """the oracle's SequenceSpec of DeepMel(**kw); activation nn.GELU or the default LeakyReLU(leakiness)"""
    kw = dict(kw)
    kw["activation"] = "gelu" if kw.get("activation") is torch.nn.GELU else "lrelu"
    return deepmel_oracle.deep_mel_spec(**kw)


def oracle_steps(c, model, steps, subj=None, pos=None, trainable=None):
    """dropin_steps on the fp64 oracle, from the state and layer settings of the (set-up) drop-in `model`; `trainable`:
    the parameters whose gradients are reported (default: those that require grad in `model`).  `c["deepmel"]`: the
    DeepMel keyword arguments of a case at other widths than the fixtures'."""
    device = next(iter(steps[0][0].values())).device
    p, state = O.split_state(model.state_dict())
    p = {k: t.detach().to(device).requires_grad_(True) for k, t in p.items()}
    state = {k: t.to(device) for k, t in state.items()}
    if subj is not None:
        subj, pos = subj.to(device).long(), pos.to(device).double()
    bn = O.layers_of(model)
    trainable = trainable or {k for k, t in model.named_parameters() if t.requires_grad}
    got = {}

    def run(inputs, bn, training, ban=None):
        if c["model"] == "deepmel":
            return O.conv_sequence(inputs["x"], p, deepmel_spec(c.get("deepmel", DEEPMEL)), bn, state)
        return O.simpleconv(p, c["model"], inputs, pos, subj, subj, training, bn, state,
                            None if ban is None else ban.double())

    for i, (inputs, w, ban) in enumerate(steps):
        for t in p.values():
            t.grad = None
        leaves = {s: t.double().requires_grad_(True) for s, t in inputs.items()}
        out = run(leaves, bn, True, ban)
        (out * w.double()).sum().backward()
        got[f"s{i}.out"] = out.detach()
        got.update({f"s{i}.g.in.{s}": t.grad for s, t in leaves.items()})
        got.update({f"s{i}.g.{k}": t.grad for k, t in p.items() if k in trainable})
    got.update({"bn." + k: t for k, t in state.items()})
    frozen = {k: O.Layer(False, layer.eps, layer.momentum) for k, layer in bn.items()}
    with torch.no_grad():
        got["out_eval"] = run({s: t.double() for s, t in steps[0][0].items()}, frozen, False)
    return got


def compare(got, want, tol, what=""):
    assert set(got) == set(want), (what, set(got) ^ set(want))
    for k, ref in want.items():
        t = got[k]
        if not t.is_floating_point():
            assert torch.equal(t.cpu(), ref.cpu()), (what, k)
        elif ref.abs().max() < 1e-4:         # conv biases in front of a training BatchNorm: 0 up to rounding
            assert t.abs().max() < 1e-4, (what, k)
        else:
            assert rel_err(t.cpu(), ref.cpu()) < tol, (what, k, rel_err(t.cpu(), ref.cpu()))


def _fixture(case):
    c, g = CASES[case], load_arrays(case)
    sd = {k[2:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("p.")}
    steps = [({s: torch.from_numpy(g[f"in{i}.{s}"]) for s in streams(c)}, torch.from_numpy(g[f"w{i}"]),
              torch.from_numpy(g[f"ban{i}"])) for i in range(c["steps"])]
    extra = {} if c["model"] == "deepmel" else dict(subj=torch.from_numpy(g["subject_index"]),
                                                   pos=torch.from_numpy(g["rec_positions"]))
    want = {k: torch.from_numpy(v) for k, v in g.items() if k[:2] == "s0" or k[:2] == "s1" or k[:2] == "s2"
            or k.startswith("bn.") or k == "out_eval"}
    return c, sd, steps, extra, want


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_reference_fixture(case):
    c, sd, steps, extra, want = _fixture(case)
    compare(oracle_steps(c, make_model(c, sd), steps, **extra), want, 1e-5, case)


@pytest.mark.parametrize("case", list(CASES))
def test_drop_in_on_the_emulator(case):
    c, sd, steps, extra, want = _fixture(case)
    model = make_model(c, sd)
    with emulated():
        got = dropin_steps(model, c, steps, **extra)
    compare(got, want, 5e-5, case)


def test_uniform_models_build_the_uniform_plan():
    """a model whose layers share its mode and settings leaves bn_layers None; one differing layer sets it"""
    import brainmagick_b200.functional as BF
    from tools.make_bn_state_golden import CLIP_CONV
    import brainmagick_b200 as bb
    for training in (True, False):
        model = bb.DeepMel(**DEEPMEL).train(training)
        bns = [blk[1] if model.has_act[k] else None for k, blk in enumerate(model.sequence)]
        fields = BF.bn_plan_fields(bns, training)
        assert fields["bn_layers"] is None and fields["training"] == training
        assert (fields["bn_eps"], fields["bn_momentum"]) == (1e-5, 0.1)
        bns[1].eval() if training else bns[1].train()
        assert BF.bn_plan_fields(bns, training)["bn_layers"][1].training == (not training)
    model = bb.SimpleConv(**CLIP_CONV.kwargs())
    bns = [blk[1] for blk in model.encoders["meg"].sequence]
    bns[3].momentum = None
    layers = BF.bn_plan_fields(bns, True)["bn_layers"]
    assert layers[3].momentum is None and layers[3].num_batches_tracked is bns[3].num_batches_tracked
    assert all(layer.momentum == 0.1 and layer.num_batches_tracked is None for k, layer in enumerate(layers) if k != 3)


@pytest.mark.parametrize("how", ["constructor", "flipped"])
def test_track_running_stats_false_raises(how):
    import brainmagick_b200 as bb
    from tools.make_bn_state_golden import CLIP_CONV
    c, sd, steps, extra, _ = _fixture("bn_state_eval_layers")
    for model in (bb.SimpleConv(**CLIP_CONV.kwargs()), bb.DeepMel(**DEEPMEL)):
        seq = model.encoders["meg"] if isinstance(model, bb.SimpleConv) else model
        bn = seq.sequence[1][1]
        if how == "constructor":                 # the module built without buffers
            seq.sequence[1][1] = torch.nn.BatchNorm1d(bn.num_features, track_running_stats=False)
        else:                                    # buffers kept, the flag flipped after construction
            bn.track_running_stats = False
        model.train()
        with emulated(), pytest.raises(NotImplementedError, match="track_running_stats"):
            if isinstance(model, bb.SimpleConv):
                model.merger.ban_centre_override = steps[0][2]
                model(dict(steps[0][0]), _batch(steps[0][0]["meg"], extra["subj"], extra["pos"]))
            else:
                model(torch.randn(2, DEEPMEL["n_in_channels"], 12))


# ---- two gloo ranks: a converted DeepMel with one eval-mode layer -------------------------------------------------------
COUNTS = (3, 2)


def _deepmel_step(rank=None):
    """one training step of a SyncBatchNorm-converted DeepMel whose layer 1 is in eval mode and layer 2 averages
    cumulatively; rank None: the whole batch in one process"""
    import brainmagick_b200 as bb
    import brainmagick_b200.functional as BF
    import syncbn_emulator
    torch.manual_seed(5)
    model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(bb.DeepMel(**DEEPMEL))
    model.train()
    model.sequence[1][1].eval()
    model.sequence[2][1].momentum = None
    gen = torch.Generator().manual_seed(6)
    N, T = sum(COUNTS), 20
    x_all = torch.randn(N, DEEPMEL["n_in_channels"], T, generator=gen)
    w_all = torch.randn(N, DEEPMEL["n_out_channels"], T, generator=gen)
    rows = slice(None) if rank is None else slice(sum(COUNTS[:rank]), sum(COUNTS[:rank + 1]))
    x = x_all[rows].clone().requires_grad_(True)
    class Emulator(CumulativeFinalize, syncbn_emulator.SyncBNEmulator):
        pass
    with syncbn_emulator.emulated(Emulator):
        out = model(x)
        (out * w_all[rows]).sum().backward()
    return dict(out=out.detach(), x=x.grad, grads={k: t.grad.clone() for k, t in model.named_parameters()},
                buffers={k: t.clone() for k, t in model.named_buffers()},
                groups=[g is not None for g in BF.bn_sync_groups(
                    [blk[1] if model.has_act[k] else None for k, blk in enumerate(model.sequence)]) or []])


def _worker(rank, world, init, ret):
    sys.path.insert(0, HERE)
    dist.init_process_group("gloo", init_method=init, rank=rank, world_size=world)
    try:
        ret[rank] = _deepmel_step(rank)
    finally:
        dist.destroy_process_group()


def test_two_ranks_with_an_eval_layer_match_the_concatenated_batch():
    with tempfile.TemporaryDirectory() as tmp, mp.Manager() as mgr:
        ret = mgr.dict()
        mp.spawn(_worker, args=(len(COUNTS), f"file://{os.path.join(tmp, 'store')}", ret), nprocs=len(COUNTS), join=True)
        per_rank = [ret[r] for r in range(len(COUNTS))]
    whole = _deepmel_step()
    for r, st in enumerate(per_rank):
        assert st["groups"] == [True, False, True, False]       # the eval-mode layer neither syncs nor takes statistics
        rows = slice(sum(COUNTS[:r]), sum(COUNTS[:r + 1]))
        assert rel_err(st["out"], whole["out"][rows]) < 1e-5
        assert rel_err(st["x"], whole["x"][rows]) < 1e-5
        for k, b in whole["buffers"].items():
            assert (torch.equal(st["buffers"][k], b) if not b.is_floating_point() else rel_err(st["buffers"][k], b) < 1e-5), k
    for k, g in whole["grads"].items():
        total = sum(st["grads"][k] for st in per_rank)
        if g.abs().max() < 1e-4:
            assert total.abs().max() < 1e-4, k
        else:
            assert rel_err(total, g) < 1e-5, k
