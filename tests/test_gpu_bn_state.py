"""GPU: BatchNorm layers that follow their own module (per-layer train / eval, eps, momentum, and the cumulative average
of momentum=None) at clip_conv widths -- C = 208 and a ragged 273, hidden 320, depth 10, T = 360, B = 64 -- against the
fp64 per-layer oracle (tests/bn_state_oracle.py): every setup of tools/make_bn_state_golden.py, the two cumulative-average
finalize entry points at their edges, bitwise repeats under torch.use_deterministic_algorithms, no host read of the
count, and torch.optim.swa_utils.update_bn on a DeepMel."""
import pytest
import torch

import bn_state_oracle as O
from conftest import rel_err
from oracle.encode_oracle import EncodeVariant
from test_bn_state_cpu import compare, deepmel_spec, dropin_steps, oracle_steps
from tools.make_bn_state_golden import CASES, SETUPS

pytestmark = pytest.mark.gpu

B, T, HIDDEN, DEPTH, S = 64, 360, 320, 10, 4
_FULL = dict(n_subjects=S, depth=DEPTH, merger_channels=270, initial_linear=270, merger_pos_dim=2048)
# GELU: with ReLU, the units whose input lies within rounding of 0 take different branches in fp32 and fp64, and at these
# sizes that alone moves the gradients by ~1e-3 whatever the BatchNorm modes (the fp32 FMA path included)
DEEPMEL = dict(n_in_channels=273, n_hidden_channels=HIDDEN, n_hidden_layers=DEPTH, n_out_channels=HIDDEN, kernel=3,
               stride=1, dilation_growth=2, dilation_period=5, batch_norm=True, activation_on_last=False, skip=True,
               glu_context=1, glu=2, activation=torch.nn.GELU)
# the fixtures' setups at full width, the meg channel count alternating between 208 and 273
WIDE = {
    name: dict(c, deepmel=DEEPMEL) if c["model"] == "deepmel" else dict(c, model=EncodeVariant(
        in_channels=dict(c["model"].in_channels, meg=208 if i % 2 == 0 else 273),
        hidden={s: HIDDEN for s in c["model"].in_channels}, out_channels=512, **_FULL), B=B, T=T)
    for i, (name, c) in enumerate(CASES.items())}


def _model(c, seed=0):
    import brainmagick_b200 as bb
    torch.manual_seed(seed)
    model = bb.DeepMel(**DEEPMEL) if c["model"] == "deepmel" else bb.SimpleConv(**c["model"].kwargs())
    with torch.no_grad():                 # every channel's affine parameters and running statistics differ
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.add_(0.1 * torch.randn_like(m.weight))
                m.bias.add_(0.1 * torch.randn_like(m.bias))
                m.running_mean.add_(0.1 * torch.randn_like(m.running_mean))
                m.running_var.mul_(1 + 0.2 * torch.rand_like(m.running_var))
    SETUPS[c["setup"]](model)
    return model.cuda()


def _inputs(c, seed=1):
    """[(inputs, w, ban)] per step, subject index, recording positions"""
    from brainmagick_b200 import synthetic
    gen = torch.Generator().manual_seed(seed)
    chans = dict(x=DEEPMEL["n_in_channels"]) if c["model"] == "deepmel" else c["model"].in_channels
    n_out = DEEPMEL["n_out_channels"] if c["model"] == "deepmel" else c["model"].out_channels
    steps = [({s: torch.randn(B, ch, T, generator=gen).cuda() for s, ch in chans.items()},
              torch.randn(B, n_out, T, generator=gen).cuda(), torch.rand(2, generator=gen)) for _ in range(c["steps"])]
    if c["model"] == "deepmel":
        return steps, {}
    subj = torch.randint(0, S, (B,), generator=gen)
    pos = synthetic.normalised_positions(S, chans["meg"], seed=seed)       # read on the host by the batch layout
    return steps, dict(subj=subj.cuda(), pos=pos)


@pytest.mark.parametrize("case", list(WIDE))
def test_setup_matches_the_fp64_oracle(case):
    c = WIDE[case]
    model = _model(c)
    steps, extra = _inputs(c)
    want = oracle_steps(c, model, steps, **extra)           # from the state before the drop-in's steps
    got = dropin_steps(model, c, steps, **extra)
    torch.cuda.synchronize()
    compare(got, want, 1e-4, case)


def _finalize(stats, n, eps, count, rm, rv, C, counted):
    from brainmagick_b200._lib import call, ptr, stream
    mean, invstd = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    st = stream()
    if counted:
        call("bm_bn_stats_finalize_counted_cumulative", ptr(stats), eps, ptr(count), ptr(rm), ptr(rv), ptr(mean),
             ptr(invstd), C, st)
    else:
        call("bm_bn_stats_finalize_cumulative", ptr(stats), n, eps, ptr(count), ptr(rm), ptr(rv), ptr(mean), ptr(invstd),
             C, st)
    return mean, invstd


@pytest.mark.parametrize("counted", [False, True])
@pytest.mark.parametrize("C,n,count", [(1, 1, 1), (129, 2, 1), (320, 23040, 2), (273, 7, 3), (64, 5, 2 ** 31 + 5)])
def test_cumulative_finalize_against_fp64(counted, C, n, count):
    """factor 1 / num_batches_tracked read on the device: count 1 takes the batch statistics as they are, a count past
    2^31 needs the int64 counter; one row keeps the biased variance; C = 1 and 129 end inside a block"""
    from brainmagick_b200 import _lib
    _lib.load()
    gen = torch.Generator().manual_seed(C + n)
    y = (3.0 + torch.randn(n, C, generator=gen, dtype=torch.float64)).cuda()
    stats = torch.cat([y.sum(0), (y * y).sum(0), torch.tensor([float(n)], device="cuda", dtype=torch.float64)])
    rm0 = torch.randn(C, generator=gen).cuda()
    rv0 = (1 + torch.rand(C, generator=gen)).cuda()
    rm, rv = rm0.clone(), rv0.clone()
    counter = torch.tensor(count, dtype=torch.int64, device="cuda")
    eps = 1e-3
    mean, invstd = _finalize(stats, n, eps, counter, rm, rv, C, counted)
    torch.cuda.synchronize()
    m, var = y.mean(0), y.var(0, unbiased=False)
    unb = y.var(0, unbiased=True) if n > 1 else var
    f = 1.0 / count
    assert rel_err(mean, m) < 1e-6 and rel_err(invstd, 1 / torch.sqrt(var + eps)) < 1e-6
    assert rel_err(rm, (1 - f) * rm0.double() + f * m) < 1e-6
    assert rel_err(rv, (1 - f) * rv0.double() + f * unb) < 1e-6
    assert int(counter) == count                              # read, never written


def _bitwise_step(c, seed):
    model = _model(c, seed)
    steps, extra = _inputs(c, seed)
    return dropin_steps(model, c, steps[:1], **extra)


@pytest.mark.parametrize("case", ["bn_state_eval_layers", "bn_state_cumulative"])
def test_deterministic_repeats_are_bitwise(case):
    c = WIDE[case]
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    try:
        a, b = _bitwise_step(c, 3), _bitwise_step(c, 3)
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def _runs_without_host_sync(momentum):
    """a DeepMel training step (forward, a torch loss, backward) under sync debug mode "error" -> "ran" or the error"""
    c = dict(WIDE["bn_state_deepmel"], setup="deepmel_mixed")
    model = _model(c)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm1d):
            m.momentum = momentum
    steps, _ = _inputs(c)
    x, w = steps[0][0]["x"], steps[0][1]

    def step():
        (model(x) * w).sum().backward()
    step()                                                    # warm-up: library load, workspaces, status word
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
        return "ran"
    except RuntimeError as e:
        return str(e).splitlines()[0]
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_cumulative_average_never_reads_the_count_on_the_host():
    """under sync debug mode "error", a momentum=None step runs exactly when the same step at momentum=0.1 runs"""
    cumulative, fixed = _runs_without_host_sync(None), _runs_without_host_sync(0.1)
    assert cumulative == fixed, (cumulative, fixed)


def test_swa_update_bn_on_deepmel():
    """torch.optim.swa_utils.update_bn (reset, momentum=None, a pass over the batches) against the oracle's cumulative
    average over the same batches"""
    c = dict(WIDE["bn_state_deepmel"], setup="deepmel_mixed", steps=3)
    model = _model(c)
    model.eval()
    steps, _ = _inputs(c)
    loader = [inputs["x"] for inputs, _, _ in steps]
    torch.optim.swa_utils.update_bn(loader, model)
    torch.cuda.synchronize()
    ref = _model(c)
    ref.train()
    p, state = O.split_state(ref.state_dict())
    for bn in (m for m in ref.modules() if isinstance(m, torch.nn.BatchNorm1d)):
        bn.momentum = None
    for k in state:
        if "running_mean" in k:
            state[k].zero_()
        elif "running_var" in k:
            state[k].fill_(1)
        else:
            state[k].zero_()
    bn = O.layers_of(ref)
    spec = deepmel_spec(DEEPMEL)
    with torch.no_grad():
        for x in loader:
            O.conv_sequence(x.double(), p, spec, bn, state)
    got = {k: t for k, t in model.state_dict().items() if "running" in k or "num_batches" in k}
    assert set(got) == set(state)
    for k, t in state.items():
        if t.is_floating_point():
            assert rel_err(got[k], t) < 1e-4, k
        else:
            assert int(got[k]) == int(t) == len(loader), k
    assert all(m.momentum is not None for m in model.modules() if isinstance(m, torch.nn.BatchNorm1d))
