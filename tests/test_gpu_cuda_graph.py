"""Steps captured in CUDA graphs (torch.cuda.graph) with a StaticBatch, on the GPU: a captured training step (forward,
ClipLoss, backward, Adam(capturable=True)) replayed on fresh batches is bitwise equal to the same steps run eagerly under the
determinism flag, at clip_conv widths, on the FP32-FMA model, under TF32, for the ablation rows and with a trainable DeepMel;
a captured eval forward likewise; the padded recording slots of a StaticBatch change nothing; spatial dropout draws a new
centre on every replay; a mask with a False entry raises at the next status read; and bm_check_all_true at its edges."""
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture
def deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def _clip_conv(hidden=320, MC=270, IL=270, P=2048, **change):
    kw = dict(hidden=dict(meg=hidden), depth=10, dilation_period=5, kernel_size=3, skip=True, subject_layers=True,
              subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=IL, merger_channels=MC,
              gelu=True, batch_norm=True, merger_pos_dim=P, merger_dropout=0.2)
    kw.update(change)
    return kw


SMALL = dict(hidden=16, MC=12, IL=12, P=32)                  # the FP32-FMA kernels
CLIP_DIMS = dict(C=208, T=360, B=64, F=1024, S=4, n_valid=(208, 190, 160, 131))     # 2 recordings per subject
CASES = {
    "clip_conv": (_clip_conv(), CLIP_DIMS),
    "small_fp32_fma": (_clip_conv(**SMALL), dict(C=10, T=24, B=6, F=8, S=3, n_valid=(10, 7))),
    "no_merger": (_clip_conv(merger=False), CLIP_DIMS),
    "subject_embedding": (_clip_conv(subject_layers=False, subject_dim=16), CLIP_DIMS),
    "subsample_channels": (_clip_conv(subsample_meg_channels=150), CLIP_DIMS),
}


class _Item:
    """One fresh batch: a reference batch (host subject_index and recordings) and its device tensors"""

    def __init__(self, dims, gen, deepmel):
        from brainmagick_b200 import synthetic
        B, C, T, F, S = (dims[k] for k in "BCTFS")
        self.meg = torch.randn(B, C, T, generator=gen).cuda()
        self.subj = torch.randint(0, S, (B,), generator=gen)
        rec = 2 * self.subj + torch.randint(0, 2, (B,), generator=gen)          # 2 recordings per subject
        pos = synthetic.normalised_positions(2 * S, C, dims.get("n_valid", ()), seed=4)
        self.batch = synthetic.make_batch(self.meg, self.subj, pos, rec)
        self.R = len(set(rec.tolist()))
        n_in = F if deepmel is None else deepmel["n_in"]
        self.cand = torch.randn(B, n_in, T, generator=gen).cuda()              # the candidates, or DeepMel's input
        self.ban = torch.rand(2, generator=gen).cuda()


def _items(dims, n, seed, deepmel=None):
    gen = torch.Generator().manual_seed(seed)
    return [_Item(dims, gen, deepmel) for _ in range(n)]


class _Trainer:
    """SimpleConv (+ DeepMel) + ClipLoss + Adam(capturable=True) reading static inputs: a StaticBatch, meg, the candidates
    (or DeepMel's input), the mask and the dropout centre"""

    def __init__(self, kw, dims, deepmel=None, train=True):
        import brainmagick_b200 as bb
        B, C, T, F, S = (dims[k] for k in "BCTFS")
        torch.manual_seed(0)
        kw = {k: (dict(v) if isinstance(v, dict) else v) for k, v in kw.items()}
        self.model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, n_subjects=S, **kw).cuda().train(train)
        params = list(self.model.parameters())
        self.feat = None
        if deepmel is not None:
            self.feat = bb.DeepMel(n_in_channels=deepmel["n_in"], **dict(deepmel["params"], n_out_channels=F)).cuda().train()
            params += list(self.feat.parameters())
        self.opt = torch.optim.Adam(params, lr=1e-3, capturable=True)
        self.clip = bb.ClipLoss().cuda().train(train)
        self.sb = bb.StaticBatch(B, C, 2 * S, "cuda")
        self.meg = torch.zeros(B, C, T, device="cuda")
        self.cand = torch.zeros(B, F if deepmel is None else deepmel["n_in"], T, device="cuda")
        self.mask = torch.ones(B, 1, T, dtype=torch.bool, device="cuda")
        self.ban = torch.zeros(2, device="cuda")
        if self.model.merger is not None:
            self.model.merger.ban_centre_override = self.ban

    def load(self, item):
        self.sb.fill_(item.batch)
        self.meg.copy_(item.meg)
        self.cand.copy_(item.cand)
        self.ban.copy_(item.ban)

    def step(self):
        self.opt.zero_grad(set_to_none=True)
        cand = self.cand if self.feat is None else self.feat(self.cand)
        est = self.model(dict(meg=self.meg), self.sb)
        loss = self.clip(est, cand, self.mask)
        loss.backward()
        self.opt.step()
        return est, loss

    def state(self, est, loss):
        out = dict(est=est.detach().clone(), loss=loss.detach().clone())
        out.update({"model." + k: v.detach().clone() for k, v in self.model.state_dict().items()})
        if self.feat is not None:
            out.update({"feat." + k: v.detach().clone() for k, v in self.feat.state_dict().items()})
        return out


def _assert_bitwise(a, b, where):
    assert a.keys() == b.keys()
    for k in a:
        if a[k].is_floating_point():
            assert torch.isfinite(a[k]).all(), (where, k)
        assert torch.equal(a[k], b[k]), (where, k, (a[k].double() - b[k].double()).abs().max().item())


def _capture(run, warm):
    """Warm-up steps on a side stream (lazy set-up), then one capture of run() -> (graph, run()'s outputs)"""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for prepare in warm:
            prepare()
            run()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):          # capture_error_mode="global": any host sync or host copy fails the capture
        out = run()
    return graph, out


def _graph_vs_eager(kw, dims, deepmel=None, steps=4):
    from brainmagick_b200 import functional as BF
    warm, fresh = _items(dims, 3, 1, deepmel), _items(dims, steps, 2, deepmel)
    g, e = _Trainer(kw, dims, deepmel), _Trainer(kw, dims, deepmel)
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
    counts = [int(v) for k, v in g.model.state_dict().items() if k.endswith("num_batches_tracked")]
    assert counts and set(counts) == {len(warm) + steps}        # the capture itself counts nothing


@pytest.mark.parametrize("case", list(CASES))
def test_captured_training_step_is_bitwise_equal_to_eager(case, deterministic):
    kw, dims = CASES[case]
    _graph_vs_eager(kw, dims)


def test_captured_training_step_under_tf32(deterministic):
    m = torch.backends.cuda.matmul
    saved_new, saved_legacy = m.fp32_precision, torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision("high")
    try:
        _graph_vs_eager(*CASES["clip_conv"])
    finally:
        torch.set_float32_matmul_precision(saved_legacy)
        m.fp32_precision = saved_new


def test_captured_training_step_with_a_trainable_deepmel(deterministic):
    from oracle.make_golden import DEEPMEL_CASES
    kw, dims = CASES["clip_conv"]
    _graph_vs_eager(kw, dict(dims, F=120), deepmel=DEEPMEL_CASES["deepmel_small"])


@pytest.mark.parametrize("case", ["clip_conv", "small_fp32_fma"])
def test_captured_eval_forward_is_bitwise_equal_to_eager(case):
    kw, dims = CASES[case]
    g, e = _Trainer(kw, dims, train=False), _Trainer(kw, dims, train=False)

    def run(t):
        with torch.no_grad():
            est = t.model(dict(meg=t.meg), t.sb)
            return est, t.clip.get_probabilities(est, t.cand)
    graph, (g_est, g_probs) = _capture(lambda: run(g), [lambda it=it: g.load(it) for it in _items(dims, 2, 1)])
    for i, it in enumerate(_items(dims, 3, 2)):
        g.load(it)
        graph.replay()
        e.load(it)
        e_est, e_probs = run(e)
        torch.cuda.synchronize()
        _assert_bitwise(dict(est=g_est, probs=g_probs), dict(est=e_est, probs=e_probs), f"batch {i}")


def _oracle_heads_grad(model, item, dims):
    """d loss / d merger.heads in fp64 (oracle/bm_oracle.training_step) for the model's parameters before its step"""
    from oracle import bm_oracle
    cfg = bm_oracle.Config(in_channels=dims["C"], out_channels=dims["F"], n_subjects=dims["S"])
    params = {k: v.detach().cpu().double() if v.is_floating_point() else v.cpu() for k, v in model.state_dict().items()}
    from brainmagick_b200 import synthetic
    rec = torch.tensor([r.recording_index for r in item.batch._recordings])
    pos = synthetic.normalised_positions(2 * dims["S"], dims["C"], dims.get("n_valid", ()), seed=4).double()
    ref = bm_oracle.training_step(params, cfg, item.meg.cpu().double(), pos, rec, item.subj, item.cand.cpu().double(),
                                  ban_centre=item.ban.cpu().double(), training=True)
    return ref["grads"]["merger.heads"]


def test_captured_standalone_merger_is_bitwise_equal_to_eager(deterministic):
    """The stand-alone ChannelMerger on a StaticBatch: forward and backward to its heads and to meg, captured (nothing copied
    from the host: the frequency table is the merger's device copy), replayed on fresh batches, bitwise equal to eager."""
    import brainmagick_b200 as bb
    dims = dict(CLIP_DIMS, B=16)
    B, C, T, S, O = dims["B"], dims["C"], dims["T"], dims["S"], 270

    class Merger:
        def __init__(self):
            torch.manual_seed(0)
            self.m = bb.ChannelMerger(O, pos_dim=2048, dropout=0.2).cuda().train()
            self.ban = torch.zeros(2, device="cuda")
            self.m.ban_centre_override = self.ban
            self.sb = bb.StaticBatch(B, C, 2 * S, "cuda")
            self.meg = torch.zeros(B, C, T, device="cuda", requires_grad=True)
            self.w = torch.zeros(B, O, T, device="cuda")

        def load(self, item):
            self.sb.fill_(item.batch)
            with torch.no_grad():
                self.meg.copy_(item.meg)
            self.w.copy_(item.cand[:, :O])
            self.ban.copy_(item.ban)

        def run(self):
            self.m.heads.grad = self.meg.grad = None
            out = self.m(self.meg, self.sb)
            (out * self.w).sum().backward()
            return dict(out=out.detach(), dheads=self.m.heads.grad, dmeg=self.meg.grad)

    g, e = Merger(), Merger()
    graph, g_out = _capture(g.run, [lambda it=it: g.load(it) for it in _items(dims, 2, 1)])
    for i, it in enumerate(_items(dims, 3, 2)):
        g.load(it)
        graph.replay()
        e.load(it)
        e_out = e.run()
        torch.cuda.synchronize()
        _assert_bitwise({k: v.clone() for k, v in g_out.items()}, e_out, f"batch {i}")


@pytest.mark.parametrize("case", ["clip_conv", "small_fp32_fma"])
def test_padded_slots_change_nothing(case, deterministic):
    """Eager with a StaticBatch of R + 5 slots against eager with the reference batch: the estimate and the loss bitwise, and
    every gradient bitwise except, on the tensor-core path, merger.heads: its contraction over the R x C attention rows
    (tc_wgrad with B = R) splits its rows by R, so it is held to 1e-4 against fp64 instead."""
    import brainmagick_b200 as bb
    kw, dims = CASES[case]
    item = _items(dims, 1, 3)[0]
    runs = []
    for static in (False, True):
        t = _Trainer(kw, dims)
        t.model.merger.ban_centre_override = item.ban
        batch = bb.StaticBatch(dims["B"], dims["C"], item.R + 5, "cuda").fill_(item.batch) if static else item.batch
        est = t.model(dict(meg=item.meg), batch)
        loss = t.clip(est, item.cand, t.mask)
        loss.backward()
        runs.append(dict(est=est.detach(), loss=loss.detach(),
                         **{"g." + k: p.grad for k, p in t.model.named_parameters()}))
    torch.cuda.synchronize()
    ref, got = runs
    if case == "clip_conv":
        want = _oracle_heads_grad(t.model, item, dims)
        assert rel_err(got.pop("g.merger.heads").cpu(), want) < 1e-4
        assert rel_err(ref.pop("g.merger.heads").cpu(), want) < 1e-4
    _assert_bitwise(got, ref, case)


@pytest.mark.parametrize("R,R_max", [(1, 4), (3, 8), (5, 6)])
def test_empty_trailing_segments_write_exact_zeros(R, R_max):
    """The per-recording weight gradients of the sensor mix, on FP32-FMA (bm_sensor_mix_bwd) and on the tensor cores
    (bm_tc_wgrad_grouped), write exact zeros for segments without samples, over outputs filled with NaN."""
    from brainmagick_b200 import functional as BF
    from brainmagick_b200._lib import ptr, stream
    B, C, T, O = 16, 256, 64, 320                  # the clip_conv mix: 320 outputs, 208 sensors padded to 256
    gen = torch.Generator().manual_seed(R)
    rec = torch.sort(torch.randint(0, R, (B,), generator=gen)).values
    rec[:R] = torch.arange(R)
    order = torch.argsort(rec, stable=True).to(torch.int32).cuda()
    off = torch.full((R_max + 1,), B, dtype=torch.int32)
    off[:R + 1] = torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(torch.bincount(rec, minlength=R), 0)]).int()
    off = off.cuda()
    du, meg = torch.randn(B, T, O, device="cuda"), torch.randn(B, C, T, device="cuda")
    d_att = torch.full((R_max, O, C), float("nan"), device="cuda")
    BF.call("bm_sensor_mix_bwd", ptr(du), O, ptr(meg), ptr(order), ptr(off), B, C, T, O, R_max, ptr(d_att), stream())
    megT = meg.transpose(1, 2).contiguous()
    dwp = torch.full((R_max, BF._round_up(O, 128), C), float("nan"), device="cuda")
    BF._tc_call("bm_tc_wgrad_grouped", ptr(du), ptr(megT), ptr(order), ptr(off), R_max, B, T, O, C, ptr(dwp),
                ptr(BF.tc_status_tensor("cuda")), stream())
    torch.cuda.synchronize()
    BF.check_tc_status()
    want = torch.zeros(R_max, O, C, dtype=torch.float64, device="cuda")
    want.index_add_(0, rec.cuda(), torch.einsum("bto,bct->boc", du.double(), meg.double()))
    for got in (d_att, dwp[:, :O]):
        assert torch.equal(got[R:], torch.zeros_like(got[R:]))
        assert rel_err(got[:R], want[:R]) < 1e-5


@pytest.mark.parametrize("dropout", [0.2, 0.0])
def test_dropout_draws_a_new_centre_on_every_replay(dropout):
    kw, dims = _clip_conv(merger_dropout=dropout), dict(CLIP_DIMS, B=16)
    t = _Trainer(kw, dims)
    t.model.merger.ban_centre_override = None

    def run():
        with torch.no_grad():
            return t.model(dict(meg=t.meg), t.sb)
    item = _items(dims, 1, 5)[0]
    graph, est = _capture(run, [lambda: t.load(item)] * 2)
    t.load(item)
    outs = []
    for _ in range(2):
        graph.replay()
        outs.append(est.clone())
    torch.cuda.synchronize()
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0], outs[1]) == (dropout == 0.0)


def test_mask_with_a_false_entry_raises_after_the_replay():
    from brainmagick_b200 import functional as BF
    kw, dims = CASES["small_fp32_fma"]
    t = _Trainer(kw, dims)
    item = _items(dims, 1, 6)[0]
    graph, _ = _capture(t.step, [lambda: t.load(item)] * 2)
    t.load(item)
    graph.replay()
    torch.cuda.synchronize()
    BF.check_tc_status()
    t.mask.view(-1)[dims["B"] * dims["T"] // 2] = False
    graph.replay()
    torch.cuda.synchronize()
    with pytest.raises(AssertionError, match="mask is not supported"):
        BF.check_tc_status()
    t.mask.fill_(True)
    graph.replay()
    torch.cuda.synchronize()
    BF.check_tc_status()


@pytest.mark.parametrize("n", [1, 15, 16, 17, 4096 + 5, (1 << 20) + 3])
@pytest.mark.parametrize("offset", [0, 1])
def test_check_all_true_entry_point_edges(n, offset):
    """bm_check_all_true on all-true masks, and with a single False at the first, a middle and the last element; 16-byte
    aligned (uint4 reads) and not (offset 1); the status word keeps an earlier code."""
    from brainmagick_b200 import functional as BF
    from brainmagick_b200._lib import ptr, stream
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    base = torch.ones(n + offset + 16, dtype=torch.bool, device="cuda")
    base[:offset] = False
    base[n + offset:] = False                          # outside the range: never read as part of it
    mask = base[offset:offset + n]

    def check():
        status.zero_()
        BF.call("bm_check_all_true", ptr(mask), n, 903, ptr(status), stream())
        return int(status.item())
    assert check() == 0
    for where in sorted({0, n // 2, n - 1}):
        mask[where] = False
        assert check() == 903, where
        mask[where] = True
    assert check() == 0
    status.fill_(900)
    mask[n - 1] = False
    BF.call("bm_check_all_true", ptr(mask), n, 903, ptr(status), stream())
    assert int(status.item()) == 900
    status.zero_()
    BF.call("bm_check_all_true", ptr(mask), 0, 903, ptr(status), stream())
    assert int(status.item()) == 0
