"""GPU: the drop-in test metrics (bm/metrics.py; DESIGN §4.9) against fp64 definitions, element by element -- every update
form (correlation, L1Reg, L2Reg, ClassificationAcc) in fp32 and fp64, on both sides of the row-split choice, at the
encode and decode shapes, under every mask broadcast and with masked inf and NaN; the finalize of each kind; bitwise
repeatability; no synchronisation during updates; the fixed launch count of an update; the reference's fixtures; and the
test-stage loop over an encoding SimpleConv.  Tolerances: 1e-10 with fp64 operands, 1e-5 with fp32 (bm/test_metrics.py's);
ClassificationAcc exactly."""
import pytest
import torch

import test_metrics_cpu
from test_gpu_regression_loss import ENC_DIMS, LIMIT, _Step
from test_gpu_cuda_graph import _items

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _bm():
    import brainmagick_b200.metrics as BM
    return BM


def _metric(name, ls=slice(None), rs=slice(None)):
    BM = _bm()
    return dict(corr=BM.OnlineCorrelation, l1=BM.L1Reg, l2=BM.L2Reg, acc=BM.ClassificationAcc)[name](ls, rs)


def ref_sums(name, left, right, mask):
    """the fp64 definition of one update's accumulator planes [NP, cols] (bm/metrics.py with the sums in fp64)"""
    if left.dim() == 2:
        left, right, mask = left[..., None], right[..., None], mask[..., None]
    m = mask.double()
    if name == "acc":
        hit = mask & (left.argmax(1, keepdim=True).double() == right.double())
        sums = [hit.double().sum(0)]
    else:
        l, r = left.double(), right.double()
        mm = m.expand_as(l)
        if name == "corr":
            sums = [(l * r * mm).sum(0), (l * mm).sum(0), (r * mm).sum(0), ((l * mm) ** 2).sum(0), ((r * mm) ** 2).sum(0)]
        else:
            d = (left - right).double() * mm
            sums = [d.abs().sum(0) if name == "l1" else (d * d).sum(0)]
    count = m.sum(0).expand_as(sums[0])
    return torch.stack([s.reshape(-1) for s in sums] + [count.reshape(-1)])


def _assert_close(got, want, tol):
    assert torch.equal(got.isnan(), want.isnan())
    ok = ~want.isnan()
    err = (got[ok] - want[ok]).abs()
    assert err.max().item() <= tol * max(1.0, want[ok].abs().max().item()), err.max().item()


def _operands(name, N, C, T, dtype, K=5, full_T=None, seed=0):
    """(left, right) with left a view cropped in time at an odd offset when full_T is given"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    Tf = full_T or T
    if name == "acc":
        left = torch.randint(0, 3, (N, K, Tf), generator=g, device=DEV).to(dtype)      # ties
        right = torch.randint(0, K, (N, 1, Tf), generator=g, device=DEV).to(dtype)
        right[0, 0, :2] = -100
    else:
        left = torch.randn(N, C, Tf, generator=g, device=DEV, dtype=dtype)
        right = 0.5 * left + torch.randn(N, C, Tf, generator=g, device=DEV, dtype=dtype)
    return left[..., Tf - T:], right[..., Tf - T:]


SHAPES = [(2048, 4, 1), (64, 3, 7), (8, 600, 400), (1, 5, 3)]          # split rows / split / no split / one row


@pytest.mark.parametrize("name", ["corr", "l1", "l2", "acc"])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("shape", SHAPES)
def test_update_forms_match_fp64(name, dtype, shape):
    from brainmagick_b200 import _lib
    N, C, T = shape
    left, right = _operands(name, N, C, T, dtype, full_T=T + 3)
    mask = torch.rand(N, 1, T, device=DEV) > 0.3
    mask[0] = True
    metric = _metric(name)
    lib = _lib.load()
    before = lib.bm_launch_count()
    metric.update(left, right, mask)
    cols = T if name == "acc" else C * T
    launches = lib.bm_launch_count() - before
    assert launches == (1 if lib.bm_metric_workspace(N, 1 if name == "acc" else C, T) == 0 else 2)
    metric.update(left, right, mask)                      # the second update adds into the first
    assert lib.bm_launch_count() - before == 2 * launches
    want = 2 * ref_sums(name, left, right, mask)
    got = metric._sums.acc
    assert got.shape == (want.shape[0], cols)
    if name == "acc":
        assert torch.equal(got, want)
    else:
        # both sides sum the same fp64 values (fp32 operands widened exactly, l - r formed in fp32) in different orders:
        # a difference formed in another dtype would show far above this
        _assert_close(got, want, 1e-12)


def _get_ref(name, sums, tol=1e-8):
    """the reference's get() on fp64 sums"""
    cnt = sums[-1]
    if name != "corr":
        return sums[0] / cnt
    sd, sl, sr, sll, srr = sums[:5]
    nl = (sll - sl.abs().pow(2) / cnt).clamp(0, float("inf")).sqrt()
    nr = (srr - sr.abs().pow(2) / cnt).clamp(0, float("inf")).sqrt()
    return (sd - sl * sr / cnt) / (nl * nr).clamp(tol, float("inf"))


NO_SPLIT = (4, 600, 400)                     # 938 column blocks: one launch, the sums go straight into the accumulators


@pytest.mark.parametrize("name", ["corr", "l1", "l2"])
def test_single_launch_reset_and_broadcast_count(name):
    """on the single-launch path: a fully masked first update containing an inf is overwritten by the next (the reset
    rule), and a [1, 1, T] mask counts once per update"""
    from brainmagick_b200 import _lib
    N, C, T = NO_SPLIT
    assert _lib.load().bm_metric_workspace(N, C, T) == 0
    left, right = _operands(name, N, C, T, torch.float64, seed=23)
    bad = left.clone()
    bad[1, 7, 9], bad[2, 8, 10] = float("inf"), float("nan")
    mask = torch.rand(N, 1, T, device=DEV) > 0.3
    mask[0] = True
    metric = _metric(name).update(bad, right, torch.zeros_like(mask))
    assert metric._sums.acc.view(-1, C, T)[0, 7, 9].isnan()          # the masked inf gave NaN, as in the reference
    metric.update(left, right, mask)
    _assert_close(metric._sums.acc, ref_sums(name, left, right, mask), 1e-12)
    one = torch.rand(1, 1, T, device=DEV) > 0.5
    metric = _metric(name)
    for _ in range(3):
        metric.update(left, right, one)
    want = 3 * ref_sums(name, left, right, one)
    assert torch.equal(metric._sums.acc[-1], want[-1]) and metric._sums.acc[-1].max().item() == 3.0
    _assert_close(metric._sums.acc, want, 1e-12)


def test_empty_slices_and_crops():
    """no columns: the accumulative metrics give the reference's CPU [0.], the correlation raises RuntimeError"""
    BM = _bm()
    a = torch.randn(4, 3, 5, dtype=torch.float64, device=DEV)
    m = torch.ones(4, 1, 5, dtype=torch.bool, device=DEV)
    for metric, args in ((BM.L2Reg(slice(0, 0), slice(0, 0)), (a, a, m)),
                         (BM.L1Reg(slice(None), slice(None)), (a[..., 5:], a[..., 5:], m[..., 5:])),
                         (BM.ClassificationAcc(slice(0, 2), slice(2, 3)), (a[..., 5:], a[..., 5:], m[..., 5:]))):
        got = metric.update(*args).update(*args).get()
        assert torch.equal(got, torch.Tensor([0.])) and got.device.type == "cpu"
    with pytest.raises(RuntimeError):
        BM.OnlineCorrelation(slice(0, 0), slice(0, 0)).update(a, a, m).get()


MASKS = [(1, 1, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 0, 0), (0, 0, 1), (0, 1, 0), (0, 0, 0)]   # 1: full size


@pytest.mark.parametrize("name", ["corr", "l1", "l2"])
@pytest.mark.parametrize("bcast", MASKS)
def test_mask_broadcasts_and_masked_inf_nan(name, bcast):
    N, C, T = 33, 6, 70
    left, right = _operands(name, N, C, T, torch.float64, seed=3)
    mshape = tuple(s if b else 1 for s, b in zip((N, C, T), bcast))
    g = torch.Generator(device=DEV).manual_seed(5)
    mask = (torch.rand(mshape, generator=g, device=DEV) > 0.2).expand(mshape)
    metric = _metric(name)
    for k in range(3):
        metric.update(left, right, mask)
    want = 3 * ref_sums(name, left, right, mask)
    _assert_close(metric._sums.acc, want, 1e-10)
    # an inf and a NaN where the mask is False still give NaN sums: the reference multiplies by the mask
    m = torch.ones(N, 1, T, dtype=torch.bool, device=DEV)
    m[:, :, 4] = False
    l2 = left.clone()
    l2[2, 1, 4], l2[3, 2, 4] = float("inf"), float("nan")
    metric = _metric(name).update(left, right, m).update(l2, right, m)
    got = metric._sums.acc.view(-1, C, T)
    assert got[0, 1, 4].isnan() and got[0, 2, 4].isnan() and not got[0, 0, 4].isnan()
    assert not got[:, :, :4].isnan().any()


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_finalize_matches_fp64_and_the_output_dtype(dtype):
    for name in ("corr", "l1", "l2", "acc"):
        N, C, T = 50, 4, 30
        left, right = _operands(name, N, C, T, dtype, seed=7)
        mask = torch.ones(N, 1, T, dtype=torch.bool, device=DEV)
        metric = _metric(name).update(left, right, mask)
        out = metric.get()
        want = _get_ref(name, metric._sums.acc).view(out.shape)
        assert out.dtype == dtype and out.device.type == "cuda"
        _assert_close(out.double(), want if dtype == torch.float64 else want.float().double(),
                      1e-12 if dtype == torch.float64 else 1e-6)


def test_encode_shape_fp64():
    """corr_meg at 256 x 208 x 324, a crop of T = 360, fp64 as the solver passes it"""
    left, right = _operands("corr", 256, 208, 324, torch.float64, full_T=360, seed=11)
    mask = torch.arange(324, device=DEV)[None, None] < torch.randint(200, 325, (256, 1, 1), device=DEV)
    mask[0] = True
    metric = _bm().OnlineCorrelation(slice(None), slice(None), "corr_meg").update(left, right, mask)
    _assert_close(metric._sums.acc, ref_sums("corr", left, right, mask), 1e-10)
    _assert_close(metric.get(), _get_ref("corr", ref_sums("corr", left, right, mask)).view(208, 324), 1e-10)


def test_decode_shape():
    """the decoding metric list at 256 x (120 mel + 41 classes) x 342: L2Reg and the correlation on the mel slice,
    ClassificationAcc on the classes"""
    BM = _bm()
    g = torch.Generator(device=DEV).manual_seed(13)
    est = torch.randn(256, 161, 342, generator=g, device=DEV, dtype=torch.float64)
    gt = torch.randn(256, 121, 342, generator=g, device=DEV, dtype=torch.float64)
    gt[:, 120] = torch.randint(0, 41, (256, 342), generator=g, device=DEV).double()
    est[:, 120:] = est[:, 120:].round()                  # ties
    mask = torch.arange(342, device=DEV)[None, None] < torch.randint(100, 343, (256, 1, 1), generator=g, device=DEV)
    mask[0] = True
    mel, cls = slice(0, 120), slice(120, 161)
    metrics = [BM.L2Reg(mel, mel), BM.OnlineCorrelation(mel, mel), BM.ClassificationAcc(cls, slice(120, 121))]
    for m in metrics:
        m.update(est, gt, mask)
    _assert_close(metrics[0]._sums.acc, ref_sums("l2", est[:, mel], gt[:, mel], mask), 1e-10)
    _assert_close(metrics[1]._sums.acc, ref_sums("corr", est[:, mel], gt[:, mel], mask), 1e-10)
    assert torch.equal(metrics[2]._sums.acc, ref_sums("acc", est[:, cls], gt[:, 120:121], mask))


def test_nan_logits_count_as_maximal():
    N, K, T = 6, 4, 40
    left, right = _operands("acc", N, 1, T, torch.float64, K=K, seed=17)
    left[1, 2, :10] = float("nan")
    left[2, 0, 5:] = float("nan")
    right[1, 0, :10] = 2
    mask = torch.ones(N, 1, T, dtype=torch.bool, device=DEV)
    metric = _metric("acc").update(left, right, mask)
    assert torch.equal(metric._sums.acc, ref_sums("acc", left, right, mask))


def test_bitwise_repeatable_and_no_sync():
    shapes = [("corr", (256, 40, 100)), ("l2", (2048, 4, 1)), ("acc", (128, 1, 90))]
    runs = []
    was = torch.are_deterministic_algorithms_enabled()
    try:
        for det in (False, True, False):
            torch.use_deterministic_algorithms(det)
            accs = []
            for name, (N, C, T) in shapes:
                left, right = _operands(name, N, C, T, torch.float64, seed=19)
                mask = torch.rand(N, 1, T, device=DEV, generator=torch.Generator(device=DEV).manual_seed(2)) > 0.5
                metric = _metric(name)
                metric.update(left, right, mask)          # allocates the accumulators
                torch.cuda.synchronize()
                torch.cuda.set_sync_debug_mode("error")
                try:
                    for _ in range(3):
                        metric.update(left, right, mask)
                finally:
                    torch.cuda.set_sync_debug_mode(0)
                accs.append(metric._sums.acc.clone())
            runs.append(accs)
    finally:
        torch.use_deterministic_algorithms(was)
    for other in runs[1:]:
        for a, b in zip(runs[0], other):
            assert torch.equal(a, b)


@pytest.mark.parametrize("name", test_metrics_cpu.CASES)
def test_reference_fixtures(name):
    specs, recs, f = test_metrics_cpu.load_case(name)
    test_metrics_cpu.check_case(f, *test_metrics_cpu.run_case(_bm(), specs, recs, to=lambda t: t.to(DEV)))


def test_test_stage_loop_over_an_encoding_simpleconv():
    """play.get_test_metrics over an encoding SimpleConv in eval mode: estimate and MEG cropped by the encode task's
    offset, cast to fp64, corr_meg updated per batch -- against an fp64 restatement of the reference"""
    dims = dict(ENC_DIMS, B=16)
    step = _Step("encode", dims)
    step.model.eval()
    metric = _bm().OnlineCorrelation(slice(None), slice(None), "corr_meg")
    sums = None
    for item in _items(dims, 4, 5):
        step.load(item)
        with torch.no_grad():
            est, gt, mask = step.forward()
        mask = mask.clone()
        mask[1:, :, -7:] = False
        metric.update(est.double(), gt.double(), mask)
        s = ref_sums("corr", est.double(), gt.double(), mask)
        sums = s if sums is None else sums + s
    C, T = dims["C"], dims["T"] - LIMIT
    _assert_close(metric._sums.acc, sums, 1e-10)
    _assert_close(metric.get(), _get_ref("corr", sums).view(C, T), 1e-10)
