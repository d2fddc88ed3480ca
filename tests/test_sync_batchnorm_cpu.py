"""nn.SyncBatchNorm without a GPU: SimpleConv, ConvSequence and DeepMel converted with
`torch.nn.SyncBatchNorm.convert_sync_batchnorm`, on the CPU emulator (tests/syncbn_emulator.py) and gloo ranks.

  * Where no layer syncs (world size 1, eval mode) the converted model issues exactly the C-ABI calls of the unconverted one
    (tests/golden/abi_trace_steps.json).
  * Two ranks with ragged batches (5 and 3 samples) and a loss that sums over samples match one unconverted process on the
    concatenated batch: each rank's rows of the output (and of meg.grad), the running statistics, and the sum over ranks of
    every parameter gradient.  Nothing in the package reads a tensor back on the host during those steps.
  * A syncing layer with a LayerScale or post_skip gain raises NotImplementedError; a rewrite layer is supported.
"""
import json
import os
import sys
import tempfile
from unittest import mock

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import abi_trace
from conftest import GOLDEN_DIR, rel_err

HERE = os.path.dirname(os.path.abspath(__file__))
COUNTS = [5, 3]                                       # rows per rank
STARTS = [sum(COUNTS[:r]) for r in range(len(COUNTS))]
TOL = 1e-5
SMALL = abi_trace.CONFIGS["small"]                     # B, C, T, F, S, hidden, merger_channels, initial_linear, pos_dim
SIMPLECONV_ROWS = {"gelu": {}, "relu": dict(gelu=False), "bare_last": dict(complex_out=False), "frozen_bn": {},
                   "meg_grad": {}, "bn_only": {}}


def _simpleconv(cfg, depth=10, **change):
    import brainmagick_b200 as bb
    B, C, T, F, S, hidden, MC, IL, P = cfg
    kw = dict(hidden=dict(meg=hidden), depth=depth, dilation_period=5, kernel_size=3, skip=True, subject_layers=True,
              subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=IL, merger_channels=MC,
              gelu=True, batch_norm=True, merger_pos_dim=P, merger_dropout=0.2, n_subjects=S)
    kw.update(change)
    return bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, **kw)


def _trace(cfg, train, convert):
    """abi_trace.simpleconv_step with the model optionally converted to SyncBatchNorm."""
    from brainmagick_b200 import synthetic
    import brainmagick_b200.functional as BF
    B, C, T, F, S = cfg[:5]

    def run():
        torch.manual_seed(0)
        model = _simpleconv(cfg)
        if convert:
            model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
        model.train(train)
        subj = torch.randint(0, S, (B,))
        meg, cand = torch.randn(B, C, T), torch.randn(B, F, T)
        batch = synthetic.make_batch(meg, subj, synthetic.normalised_positions(S, C), subj)
        if train:
            BF.clip_loss(model(dict(meg=meg), batch), cand, 0).backward()
        else:
            with torch.no_grad():
                model(dict(meg=meg), batch)
    return json.loads(json.dumps(abi_trace.record(run)))


def _golden_traces():
    return json.load(open(os.path.join(GOLDEN_DIR, "abi_trace_steps.json")))


@pytest.mark.parametrize("cfg", list(abi_trace.CONFIGS))
@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
def test_converted_model_without_distributed_keeps_its_call_stream(cfg, train):
    assert not dist.is_initialized()
    want = _golden_traces()[f"{cfg}.{'train' if train else 'eval'}"]
    assert _trace(abi_trace.CONFIGS[cfg], train, convert=True) == want


# ---- gloo ranks ---------------------------------------------------------------------------------------------------------
class _Counter:
    """dist.all_reduce as functional.py calls it, counted."""

    def __init__(self):
        self.n = 0
        self.inner = dist.all_reduce

    def __call__(self, *a, **k):
        self.n += 1
        return self.inner(*a, **k)


def _no_host_reads():
    """Tensor.item / Tensor.tolist raise when the package calls them (the emulator itself may)."""
    def guard(name):
        orig = getattr(torch.Tensor, name)

        def fn(self, *a, **k):
            caller = sys._getframe(1).f_globals.get("__name__", "")
            if caller.startswith("brainmagick_b200"):
                raise AssertionError(f"Tensor.{name} called by {caller} during a SyncBatchNorm step")
            return orig(self, *a, **k)
        return mock.patch.object(torch.Tensor, name, fn)
    return guard("item"), guard("tolist")


def _state(model, out, x):
    return dict(out=out.detach().clone(), meg=None if x.grad is None else x.grad.clone(),
                grads={n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None},
                buffers={n: b.clone() for n, b in model.named_buffers()})


def _simpleconv_step(row, rank=None, convert=False):
    """One training step of SimpleConv on the emulator; rank None: the whole batch in one process -> _state + all-reduces."""
    import brainmagick_b200.functional as BF
    import syncbn_emulator
    from brainmagick_b200 import synthetic
    _, C, T, F, S = SMALL[:5]
    N = sum(COUNTS)
    torch.manual_seed(0)
    model = _simpleconv(SMALL, **SIMPLECONV_ROWS[row])
    if convert:
        model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
    model.train()
    model.merger.ban_centre_override = torch.tensor([0.35, 0.6])
    if row in ("frozen_bn", "bn_only"):
        for name, p in model.named_parameters():
            is_bn = any(name.startswith(f"encoders.meg.sequence.{k}.1.") for k in range(len(model.encoders["meg"].sequence)))
            p.requires_grad_(not is_bn if row == "frozen_bn" else is_bn)
    gen = torch.Generator().manual_seed(1)
    meg, subj = torch.randn(N, C, T, generator=gen), torch.randint(0, S, (N,), generator=gen)
    Fo = model.out_channels
    w = torch.randn(N, Fo, T, generator=gen)
    rows = slice(None) if rank is None else slice(STARTS[rank], STARTS[rank] + COUNTS[rank])
    x = meg[rows].clone().requires_grad_(row == "meg_grad")
    batch = synthetic.make_batch(x.detach(), subj[rows], synthetic.normalised_positions(S, C), subj[rows])
    counter = _Counter()
    item, tolist = _no_host_reads()
    with syncbn_emulator.emulated(), mock.patch.object(BF.dist, "all_reduce", counter), item, tolist:
        out = model(dict(meg=x), batch)
        (out * w[rows]).sum().backward()
    return _state(model, out, x), counter.n


def _sequence_step(kind, rank=None, convert=False, train=True):
    """One training step of a stand-alone DeepMel / ConvSequence with a rewrite conv on the emulator."""
    import brainmagick_b200 as bb
    import syncbn_emulator
    N, T = sum(COUNTS), 20
    torch.manual_seed(3)
    if kind == "deepmel":
        model = bb.DeepMel(10, 16, 4, 24, kernel=3, stride=1, dilation_growth=2, dilation_period=5, batch_norm=True,
                           activation_on_last=False, skip=True, glu_context=1, glu=2)
    else:
        model = bb.ConvSequence([10, 16, 16, 16], kernel=3, stride=1, dilation_growth=2, batch_norm=True, skip=True,
                                **{kind: {"scale": 0.1, "post_skip": True, "rewrite": True}[kind]})
    if convert:
        model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
    model.train(train)
    gen = torch.Generator().manual_seed(4)
    mel = torch.randn(N, 10, T, generator=gen)
    w = torch.randn(N, model.sequence[-1][0].out_channels, T, generator=gen)
    rows = slice(None) if rank is None else slice(STARTS[rank], STARTS[rank] + COUNTS[rank])
    x = mel[rows].clone()
    item, tolist = _no_host_reads()
    from test_residual_branch_cpu import ResidualEmulator            # the LayerScale / post_skip gain entry points

    class Emulator(syncbn_emulator.SyncBNEmulator, ResidualEmulator):
        pass
    with syncbn_emulator.emulated(Emulator), item, tolist:
        out = model(x)
        (out * w[rows]).sum().backward()
    return _state(model, out, x)


def _worker(rank, world, init, ret):
    sys.path.insert(0, HERE)
    dist.init_process_group("gloo", init_method=init, rank=rank, world_size=world)
    try:
        out = {}
        for row in SIMPLECONV_ROWS:
            out[row] = _simpleconv_step(row, rank, convert=True)
        for kind in ("deepmel", "rewrite"):
            out[kind] = _sequence_step(kind, rank, convert=True)
        for kind in ("scale", "post_skip"):
            with pytest.raises(NotImplementedError, match="SyncBatchNorm"):
                _sequence_step(kind, rank, convert=True)
            _sequence_step(kind, rank, convert=False)                  # unconverted: per-rank statistics, runs
            _sequence_step(kind, rank, convert=True, train=False)      # eval mode: nothing syncs, runs
        out["eval_trace"] = _trace(SMALL, False, convert=True)
        ret[rank] = out
    finally:
        dist.destroy_process_group()


def _world1_worker(rank, init, ret):
    sys.path.insert(0, HERE)
    dist.init_process_group("gloo", init_method=init, rank=0, world_size=1)
    try:
        ret[0] = {f"{cfg}.{mode}": _trace(abi_trace.CONFIGS[cfg], mode == "train", convert=True)
                  for cfg in ("small", "mid") for mode in ("train", "eval")}
    finally:
        dist.destroy_process_group()


def _spawn(fn, nprocs, *args):
    with tempfile.TemporaryDirectory() as tmp, mp.Manager() as mgr:
        ret = mgr.dict()
        mp.spawn(fn, args=args + (f"file://{os.path.join(tmp, 'store')}", ret), nprocs=nprocs, join=True)
        return dict(ret)


def test_world_size_one_keeps_its_call_stream():
    got = _spawn(_world1_worker, 1)[0]
    want = _golden_traces()
    for tag, trace in got.items():
        assert trace == want[tag], tag


def _check(per_rank, oracle, what):
    for r, st in enumerate(per_rank):
        rows = slice(STARTS[r], STARTS[r] + COUNTS[r])
        assert rel_err(st["out"], oracle["out"][rows]) < TOL, (what, r)
        if oracle["meg"] is not None:
            assert rel_err(st["meg"], oracle["meg"][rows]) < TOL, (what, r)
        for name, b in oracle["buffers"].items():
            if b.is_floating_point():
                assert rel_err(st["buffers"][name], b) < TOL, (what, r, name)
            else:
                assert torch.equal(st["buffers"][name], b), (what, r, name)
    assert set(oracle["grads"]) == set(per_rank[0]["grads"]), what
    for name, g in oracle["grads"].items():
        total = sum(st["grads"][name] for st in per_rank)
        if g.norm() < 1e-4:        # conv biases in front of a training BatchNorm: exactly 0 up to rounding
            assert total.abs().max() < 1e-4, (what, name)
        else:
            assert rel_err(total, g) < TOL, (what, name)


@pytest.fixture(scope="module")
def two_ranks():
    world = len(COUNTS)
    got = _spawn(_worker, world, world)
    return [got[r] for r in range(world)]


@pytest.mark.parametrize("row", list(SIMPLECONV_ROWS))
def test_simpleconv_two_ranks_match_the_concatenated_batch(two_ranks, row):
    oracle, _ = _simpleconv_step(row)
    _check([r[row][0] for r in two_ranks], oracle, row)
    depth = 10
    n_bn = depth - (1 if row == "bare_last" else 0)
    # one all-reduce per BatchNorm layer in the forward, one in the backward where the layer's input needs a gradient:
    # with only gamma / beta trainable the first layer's does not
    want = 2 * n_bn - (1 if row == "bn_only" else 0)
    assert all(r[row][1] == want for r in two_ranks), [r[row][1] for r in two_ranks]


@pytest.mark.parametrize("kind", ["deepmel", "rewrite"])
def test_sequences_two_ranks_match_the_concatenated_batch(two_ranks, kind):
    _check([r[kind] for r in two_ranks], _sequence_step(kind), kind)


def test_eval_mode_on_two_ranks_keeps_its_call_stream(two_ranks):
    want = _golden_traces()["small.eval"]
    assert all(r["eval_trace"] == want for r in two_ranks)
