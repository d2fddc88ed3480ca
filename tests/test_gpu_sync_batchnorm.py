"""nn.SyncBatchNorm on the H100.

  * The SyncBatchNorm entry points against fp64, and bitwise against the fused ones they split: with the local sums and the
    local count, bm_bn_stats_finalize_counted == bm_bn_stats_finalize and `_bwd_reduce` -> `_bwd_apply` ==
    bm_bn_gelu_skip_bwd / bm_bn_act_skip_bwd, in the default and the `_det` forms, at C = 320 (column-stationary kernels),
    1040 (float4 kernels) and 10 (generic kernels), with row counts off the block sizes.
  * Two ranks on one GPU over gloo (mp.spawn, join=True: no process outlives the test), ragged batches of 24 and 17 at the
    clip_conv widths (C = 208, hidden 320, F = 1024, T = 360) and a per-sample loss: each rank's estimate rows and meg.grad
    rows, the sum over ranks of every parameter gradient, and the running statistics are within 1e-4 of fp64 autograd of
    the oracle on the concatenated batch, with and without the determinism flag; the same for a DeepMel candidate branch
    (with GELU: LeakyReLU(0)'s derivative jumps at 0, which moves fp32 gradients ~1e-3 from fp64, see test_gpu_deepmel.py).
    Under the flag, two repeats of a 3-step two-rank run are bitwise equal.  Over NCCL where two GPUs are visible.
"""
import os
import sys
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import rel_err

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
COUNTS = [24, 17]
STARTS = [0, 24]
C_MEG, T, F, S = 208, 360, 1024, 4
BAN = (0.31, 0.64)
DEEPMEL = dict(n_hidden_channels=320, n_hidden_layers=4, n_out_channels=768, kernel=3, stride=1, dilation_growth=2,
               dilation_period=5, batch_norm=True, activation_on_last=False, skip=True, glu_context=1, glu=2)
MEL_IN = 120
TOL = 1e-4


# ---- entry points -------------------------------------------------------------------------------------------------------
def _det_ws(lib, name, rows, C):
    return torch.empty(max(int(getattr(lib, name + "_workspace")(rows, C)), 2), device="cuda")


@pytest.mark.parametrize("C", [320, 1040, 10])
@pytest.mark.parametrize("act", ["gelu", "relu"])
@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
def test_split_entry_points_equal_the_fused_ones(C, act, det):
    from brainmagick_b200 import _lib
    from brainmagick_b200._lib import call, ptr, stream
    lib = _lib.load()
    rows = 1000 + 37                                    # off the 96- and 128-row blocks
    g = torch.Generator().manual_seed(C)
    y = (torch.randn(rows, C, generator=g) * 2 + 0.5).cuda()
    dz = torch.randn(rows, C, generator=g).cuda()
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).cuda()
    beta = (0.1 * torch.randn(C, generator=g)).cuda()
    st = stream()
    # forward statistics: fused and counted finalize from the same sums
    stats = torch.empty(2 * C + 1, dtype=torch.float64, device="cuda")
    call("bm_col_stats", ptr(y), rows, C, ptr(stats), st)
    stats[2 * C] = float(rows)
    outs = []
    for counted in (False, True):
        mean, invstd = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
        rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
        if counted:
            call("bm_bn_stats_finalize_counted", ptr(stats), 1e-5, 0.1, ptr(rm), ptr(rv), ptr(mean), ptr(invstd), C, st)
        else:
            call("bm_bn_stats_finalize", ptr(stats), rows, 1e-5, 0.1, ptr(rm), ptr(rv), ptr(mean), ptr(invstd), C, st)
        outs.append((mean, invstd, rm, rv))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    mean, invstd, rm, rv = outs[0]
    y64 = y.double()
    assert rel_err(mean.cpu(), y64.mean(0).cpu()) < 1e-6
    assert rel_err(invstd.cpu(), (1 / torch.sqrt(y64.var(0, unbiased=False) + 1e-5)).cpu()) < 1e-6
    assert rel_err(rv.cpu(), (0.9 + 0.1 * y64.var(0, unbiased=True)).cpu()) < 1e-6
    # backward: fused vs reduce -> apply with the local sums and count
    name = "bm_bn_gelu_skip_bwd" if act == "gelu" else "bm_bn_act_skip_bwd"
    act_args = () if act == "gelu" else (1, 0.0)
    head = (ptr(dz), ptr(y), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta))
    fused = [torch.empty(rows, C, device="cuda"), torch.empty(C, device="cuda"), torch.empty(C, device="cuda")]
    sums = torch.empty(2 * C + 1, dtype=torch.float64, device="cuda")
    tail = (None,) if act == "gelu" else ()             # amax_out
    args = head + (1, rows, C) + act_args + (ptr(sums), ptr(fused[0]), ptr(fused[1]), ptr(fused[2])) + tail
    if det:
        ws = _det_ws(lib, name + "_det", rows, C)
        call(name + "_det", *args, ptr(ws), ws.numel(), st)
    else:
        call(name, *args, st)
    split = [torch.empty(rows, C, device="cuda"), torch.empty(C, device="cuda"), torch.empty(C, device="cuda")]
    sums2 = torch.empty(2 * C + 1, dtype=torch.float64, device="cuda")
    rargs = head + (rows, C) + act_args + (ptr(sums2), ptr(split[1]), ptr(split[2]))
    if det:
        ws = _det_ws(lib, name + "_reduce_det", rows, C)
        call(name + "_reduce_det", *rargs, ptr(ws), ws.numel(), st)
    else:
        call(name + "_reduce", *rargs, st)
    sums2[2 * C] = float(rows)
    call(name + "_apply", *head, rows, C, *act_args, ptr(sums2), ptr(split[0]), st)
    torch.cuda.synchronize()
    for a, b in zip(fused, split):
        assert torch.equal(a, b)
    # fp64 reference of the apply: dy = gamma*invstd*(dz' - mean(dz') - yhat*mean(dz'*yhat))
    yh = (y64 - mean.double()) * invstd.double()
    z = yh * gamma.double() + beta.double()
    if act == "gelu":
        grad = 0.5 * (1 + torch.erf(z / 2 ** 0.5)) + z * torch.exp(-0.5 * z * z) / (2 * torch.pi) ** 0.5
    else:
        grad = (z > 0).double()
    d = dz.double() * grad
    want = gamma.double() * invstd.double() * (d - d.mean(0) - yh * (d * yh).mean(0))
    assert rel_err(split[0].cpu(), want.cpu()) < 1e-5
    assert rel_err(split[1].cpu(), (d * yh).sum(0).cpu()) < 1e-5
    assert rel_err(split[2].cpu(), d.sum(0).cpu()) < 1e-5


# ---- two ranks --------------------------------------------------------------------------------------------------------
def _simpleconv():
    import brainmagick_b200 as bb
    torch.manual_seed(3)
    model = bb.SimpleConv(in_channels=dict(meg=C_MEG), out_channels=F, hidden=dict(meg=320), depth=10, dilation_period=5,
                          kernel_size=3, skip=True, subject_layers=True, subject_dim=0, complex_out=True, glu=2,
                          glu_context=1, merger=True, initial_linear=270, merger_channels=270, gelu=True, batch_norm=True,
                          merger_pos_dim=2048, merger_dropout=0.2, n_subjects=S)
    with torch.no_grad():
        for name, buf in model.named_buffers():
            if "running_mean" in name:
                buf.normal_(0, 0.1)
            elif "running_var" in name:
                buf.uniform_(0.5, 2.0)
    return model


def _deepmel():
    import brainmagick_b200 as bb
    torch.manual_seed(5)
    return bb.DeepMel(MEL_IN, activation=torch.nn.GELU, **DEEPMEL)


def _data():
    g = torch.Generator().manual_seed(11)
    N = sum(COUNTS)
    meg = torch.randn(N, C_MEG, T, generator=g)
    subj = torch.randint(0, S, (N,), generator=g)
    w = torch.randn(N, F, T, generator=g)
    mel = torch.randn(N, MEL_IN, T, generator=g)
    wm = torch.randn(N, DEEPMEL["n_out_channels"], T, generator=g)
    return meg, subj, w, mel, wm


def _state(model, out, x):
    return dict(out=out.detach().cpu(), meg=None if x.grad is None else x.grad.cpu(),
                grads={n: p.grad.cpu() for n, p in model.named_parameters() if p.grad is not None},
                buffers={n: b.cpu() for n, b in model.named_buffers()})


def _worker(rank, world, backend, det, steps, init, ret):
    sys.path.insert(0, HERE)
    device = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(device)
    dist.init_process_group(backend, init_method=init, rank=rank, world_size=world)
    try:
        import brainmagick_b200.functional as BF
        from brainmagick_b200 import distrib, synthetic
        torch.use_deterministic_algorithms(det)
        meg, subj, w, mel, wm = _data()
        rows = slice(STARTS[rank], STARTS[rank] + COUNTS[rank])
        pos = synthetic.normalised_positions(S, C_MEG)
        out = {}
        model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(_simpleconv()).to(device).train()
        model.merger.ban_centre_override = torch.tensor(BAN)
        for step in range(steps):
            model.zero_grad(set_to_none=True)
            x = meg[rows].to(device).requires_grad_(True)
            est = model(dict(meg=x), synthetic.make_batch(x.detach(), subj[rows].to(device), pos, subj[rows]))
            (est * w[rows].to(device)).sum().backward()
            torch.cuda.synchronize()
            BF.check_tc_status()
            if step == 0:
                out["simpleconv"] = _state(model, est, x)
            if steps > 1:
                distrib.sync_gradients(model.parameters())
                with torch.no_grad():
                    for p in model.parameters():
                        p -= 1e-4 * p.grad
        if steps > 1:
            out["final"] = {k: v.cpu() for k, v in model.state_dict().items()}
        dm = torch.nn.SyncBatchNorm.convert_sync_batchnorm(_deepmel()).to(device).train()
        x = mel[rows].to(device)
        cand = dm(x)
        (cand * wm[rows].to(device)).sum().backward()
        torch.cuda.synchronize()
        out["deepmel"] = _state(dm, cand, x)
        ret[rank] = out
    finally:
        dist.destroy_process_group()


def _spawn(backend, det, steps):
    world = len(COUNTS)
    with tempfile.TemporaryDirectory() as tmp, mp.Manager() as mgr:
        ret = mgr.dict()
        mp.spawn(_worker, args=(world, backend, det, steps, f"file://{os.path.join(tmp, 'store')}", ret), nprocs=world,
                 join=True)
        return [ret[r] for r in range(world)]


@pytest.fixture(scope="module")
def oracle():
    """fp64 autograd of the oracle on the concatenated batch: {"simpleconv": ..., "deepmel": ...} like `_state`."""
    from oracle import ablation_oracle, deepmel_oracle
    from brainmagick_b200 import synthetic
    meg, subj, w, mel, wm = _data()
    model = _simpleconv()
    v = ablation_oracle.Variant(in_channels=C_MEG, out_channels=F, n_subjects=S)
    p = {k: t.detach().double().requires_grad_(t.is_floating_point() and "running" not in k)
         for k, t in model.state_dict().items()}
    x = meg.double().requires_grad_(True)
    stats = {}
    est = ablation_oracle.forward(p, v, x, synthetic.normalised_positions(S, C_MEG).double(), subj, subj, training=True,
                                  ban_centre=torch.tensor(BAN).double(), new_stats=stats)
    (est * w.double()).sum().backward()
    buffers = {k: t for k, t in model.state_dict().items() if "running" in k or "num_batches" in k}
    buffers.update(stats)
    out = {"simpleconv": dict(out=est.detach(), meg=x.grad, grads={k: t.grad for k, t in p.items() if t.grad is not None},
                              buffers=buffers)}
    dm = _deepmel()
    spec = deepmel_oracle.deep_mel_spec(MEL_IN, **DEEPMEL, activation="gelu")
    q = {k: t.detach().double().requires_grad_(t.is_floating_point() and "running" not in k)
         for k, t in dm.state_dict().items()}
    stats = {}
    cand = deepmel_oracle.conv_sequence(mel.double(), q, spec, training=True, new_stats=stats)
    (cand * wm.double()).sum().backward()
    buffers = {k: t for k, t in dm.state_dict().items() if "running" in k or "num_batches" in k}
    buffers.update(stats)
    out["deepmel"] = dict(out=cand.detach(), meg=None, grads={k: t.grad for k, t in q.items() if t.grad is not None},
                          buffers=buffers)
    return out


def _check(per_rank, ref, what):
    for r, st in enumerate(per_rank):
        rows = slice(STARTS[r], STARTS[r] + COUNTS[r])
        assert rel_err(st["out"], ref["out"][rows]) < TOL, (what, r)
        if ref["meg"] is not None:
            assert rel_err(st["meg"], ref["meg"][rows]) < TOL, (what, r)
        for name, b in st["buffers"].items():
            if "num_batches" in name:
                assert int(b) == int(ref["buffers"][name]) + 1, (what, name)
            else:
                assert rel_err(b, ref["buffers"][name]) < TOL, (what, r, name)
    for name, g in ref["grads"].items():
        total = sum(st["grads"][name].double() for st in per_rank)
        scale = max(st["grads"][name].abs().max().item() for st in per_rank)
        if g.abs().max() < 1e-6 * scale:
            # a conv bias in front of a training BatchNorm: each rank's is its local sum, the sum over ranks is 0 up to rounding
            assert total.abs().max() < 1e-4 * scale, (what, name)
        else:
            assert rel_err(total, g) < TOL, (what, name, rel_err(total, g))


_runs = {}


def _gloo(det):
    if det not in _runs:
        _runs[det] = _spawn("gloo", det, 3 if det else 1)
    return _runs[det]


@pytest.mark.parametrize("det", [False, True], ids=["default", "deterministic"])
def test_two_ranks_on_gloo_match_fp64(oracle, det):
    got = _gloo(det)
    for what in ("simpleconv", "deepmel"):
        _check([r[what] for r in got], oracle[what], what)


def test_deterministic_two_rank_runs_repeat_bitwise():
    first = _gloo(True)
    again = _spawn("gloo", True, 3)
    for a, b in zip(first, again):
        for k in a["final"]:
            assert torch.equal(a["final"][k], b["final"][k]), k


def test_two_ranks_on_nccl_match_fp64(oracle):
    if torch.cuda.device_count() < 2:
        pytest.skip("NCCL needs one GPU per rank; one GPU is visible")
    got = _spawn("nccl", False, 1)
    for what in ("simpleconv", "deepmel"):
        _check([r[what] for r in got], oracle[what], what)
