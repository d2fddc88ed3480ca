"""CPU checks of the drop-in test metrics (bm/metrics.py): on the ABI emulator (tests/metrics_emulator.py) they match the
verbatim reference's fixtures (oracle/make_metrics_golden.py) for every case, results, errors and reduce() alike; the
module surface and the errors of the port; and the C-ABI call stream -- one update call per update and nothing read on
the host, one finalize call and one flag read per get(), and the single read of the "seen" word when an update's column
shape changes."""
import os

import numpy as np
import pytest
import torch

import metrics_emulator
from conftest import GOLDEN_DIR
from test_regression_loss_cpu import _host_reads_forbidden

CASES = ["encode_corr", "decode_mix", "fp32_chunks", "mask_shapes", "offset", "reset", "errors"]


def _bm():
    import brainmagick_b200.metrics as BM
    return BM


def _slice(start, stop):
    return slice(None if start < 0 else start, None if stop < 0 else stop)


def load_case(name):
    """(metric constructors, recordings: lists of (left, right, mask) updates, fixture dict) of metrics_<name>.npz"""
    z = np.load(os.path.join(GOLDEN_DIR, f"metrics_{name}.npz"))
    f = {k: z[k] for k in z.files}
    specs = [(str(k), str(n), _slice(ls, le), _slice(rs, re_))
             for k, n, ls, le, rs, re_ in zip(f["kinds"], f["names"], f["l_start"], f["l_stop"], f["r_start"], f["r_stop"])]
    chunk, crop = int(f["chunk"]), int(f["crop"])
    recs = []
    for r in range(int(f["recordings"])):
        if chunk:
            left, right, mask = (torch.from_numpy(f[f"{k}_{r}"]) for k in ("left", "right", "mask"))
            recs.append([(left[k:k + chunk], right[k:k + chunk], mask[k:k + chunk]) for k in range(0, left.shape[0], chunk)])
        else:
            ups = [tuple(torch.from_numpy(f[f"{k}_{r}_{u}"]) for k in ("left", "right", "mask"))
                   for u in range(int(f[f"updates_{r}"]))]
            recs.append([(a[..., crop:], b[..., crop:], m[..., crop:]) if crop else (a, b, m) for a, b, m in ups])
    return specs, recs, f


def run_case(BM, specs, recs, to=lambda t: t):
    """play.get_test_metrics' loop: fresh metrics per recording, update per batch, get() -> (results, errors, reduced)"""
    results, errors = [], []
    for rec in recs:
        metrics = [getattr(BM, kind).get_constructor(ls, rs, name=name)() for kind, name, ls, rs in specs]
        for left, right, mask in rec:
            for m in metrics:
                m.update(to(left), to(right), to(mask))
        res, err = [], []
        for m in metrics:
            try:
                res.append(m.get())
                err.append("")
            except (ValueError, AssertionError) as e:
                res.append(None)
                err.append(type(e).__name__)
        results.append(res)
        errors.append(err)
    reduced = []
    for j, (kind, *_r) in enumerate(specs):
        ok = all(not errors[r][j] for r in range(len(recs)))
        reduced.append(getattr(BM, kind).reduce([results[r][j].cpu().float() for r in range(len(recs))]) if ok
                       else float("nan"))
    return results, errors, reduced


def check_case(f, results, errors, reduced):
    for r in range(len(results)):
        for j, got in enumerate(results[r]):
            assert errors[r][j] == str(f[f"error_{r}_{j}"]), (r, j)
            if errors[r][j]:
                continue
            want = torch.from_numpy(f[f"result_{r}_{j}"])
            got = got.cpu()
            assert got.dtype == want.dtype and got.shape == want.shape, (r, j, got.dtype, want.dtype)
            tol = 1e-10 if want.dtype == torch.float64 else 1e-5
            assert torch.equal(got.isnan(), want.isnan())
            assert (got.double() - want.double()).abs().max().item() <= tol * max(1.0, want.abs().max().item())
    np.testing.assert_allclose(np.array(reduced), f["reduced"], rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("name", CASES)
def test_drop_in_matches_the_reference_fixture(name):
    specs, recs, f = load_case(name)
    with metrics_emulator.emulated():
        check_case(f, *run_case(_bm(), specs, recs))


def test_surface():
    import brainmagick_b200 as bb
    BM = _bm()
    assert bb.metrics is BM and not {"TestMetric", "OnlineCorrelation", "L2Reg", "ClassificationAcc"} & set(bb.__all__)
    c = BM.OnlineCorrelation.get_constructor(slice(None), slice(2, 5), "corr_meg")()
    assert (c.name, c.left_slice, c.right_slice, c.dim, c.tol) == ("corr_meg", slice(None), slice(2, 5), 0, 1e-8)
    a = BM.ClassificationAcc.get_constructor(slice(3, 7), slice(3, 4), name="acc_ph")()
    assert (a.name, a.left_slice, a.right_slice, a.dim) == ("acc_ph", slice(3, 7), slice(3, 4), 0)
    assert BM.AccumulativeMetric(slice(None), slice(None)).name == "N/A"
    for cls in (BM.OnlineCorrelation, BM.L1Reg, BM.L2Reg, BM.ClassificationAcc):
        assert issubclass(cls, BM.TestMetric)
    for cls in (BM.L1Reg, BM.L2Reg, BM.ClassificationAcc):
        assert issubclass(cls, BM.AccumulativeMetric)
    stats = [torch.tensor([1.0, 3.0]), torch.tensor([5.0, 7.0])]
    assert BM.L1Reg.reduce(stats) == 4.0 and BM.L2Reg.reduce(stats) == 2.0
    with pytest.raises(AssertionError):
        BM.OnlineCorrelation(slice(None), slice(None), tol=-1.0)
    empty = BM.L2Reg(slice(None), slice(None)).get()                 # never updated: the reference's CPU [0.]
    assert torch.equal(empty, torch.Tensor([0.])) and empty.device.type == "cpu"
    with pytest.raises(AttributeError):
        BM.OnlineCorrelation(slice(None), slice(None)).get()


def test_errors():
    BM = _bm()
    a, m = torch.randn(4, 3, 5, dtype=torch.float64), torch.ones(4, 1, 5, dtype=torch.bool)
    with pytest.raises(RuntimeError, match="CUDA"):                      # no CPU fallback
        BM.OnlineCorrelation(slice(None), slice(None)).update(a, a, m)
    with pytest.raises(NotImplementedError):
        BM.OnlineCorrelation(slice(None), slice(None), dim=1).update(a, a, m)
    with pytest.raises(NotImplementedError):
        BM.L2Reg(slice(None), slice(None)).update(a.to(torch.complex128), a.to(torch.complex128), m)
    with pytest.raises(TypeError, match="bool"):
        BM.L2Reg(slice(None), slice(None)).update(a, a, m.double())
    with pytest.raises(NotImplementedError):
        BM.AccumulativeMetric(slice(None), slice(None)).update(a, a, m)
    with metrics_emulator.emulated():
        with pytest.raises(TypeError, match="fp32 or fp64"):
            BM.L1Reg(slice(None), slice(None)).update(a.half(), a.half(), m)
        with pytest.raises(RuntimeError):
            BM.L1Reg(slice(None), slice(None)).update(a, a[:, :2], m)
        with pytest.raises(RuntimeError):
            BM.L1Reg(slice(None), slice(None)).update(a, a, torch.ones(4, 2, 5, dtype=torch.bool))
        acc = BM.ClassificationAcc(slice(0, 2), slice(2, 3))
        with pytest.raises(IndexError):                                  # preds[~mask] in the reference
            acc.update(a, a, torch.ones(1, 1, 5, dtype=torch.bool))
        with pytest.raises(IndexError):
            BM.ClassificationAcc(slice(0, 2), slice(1, 3)).update(a, a, m)
        # another column shape: re-initialised while no mask entry was True, an error afterwards
        c = BM.OnlineCorrelation(slice(None), slice(None))
        c.update(a, a, torch.zeros_like(m)).update(a[:, :2], a[:, :2], m)
        assert c.get().shape == (2, 5)
        with pytest.raises(RuntimeError, match="columns"):
            c.update(a, a, m)


def test_empty_slices_and_crops_follow_the_reference():
    """no columns (an empty slice, or a time crop that leaves T = 0): the accumulative metrics give the reference's CPU
    [0.], the correlation raises as the reference's min() of an empty tensor, an empty class slice as its argmax"""
    from brainmagick_b200 import _lib
    BM = _bm()
    a, m = torch.randn(4, 3, 5, dtype=torch.float64), torch.ones(4, 1, 5, dtype=torch.bool)
    assert _lib.load().bm_metric_workspace(4, 0, 5) == 0 and _lib.load().bm_metric_workspace(4, 3, 0) == 0
    with metrics_emulator.emulated():
        for cls in (BM.L1Reg, BM.L2Reg):
            for metric, args in ((cls(slice(0, 0), slice(0, 0)), (a, a, m)),
                                 (cls(slice(None), slice(None)), (a[..., 5:], a[..., 5:], m[..., 5:]))):
                got = metric.update(*args).update(*args).get()
                assert torch.equal(got, torch.Tensor([0.])) and got.device.type == "cpu"
        got = BM.ClassificationAcc(slice(0, 2), slice(2, 3)).update(a[..., 5:], a[..., 5:], m[..., 5:]).get()
        assert torch.equal(got, torch.Tensor([0.]))
        with pytest.raises(IndexError):
            BM.ClassificationAcc(slice(0, 0), slice(2, 3)).update(a, a, m)
        for args in ((a[:, :0], a[:, :0], m), (a[..., 5:], a[..., 5:], m[..., 5:])):
            with pytest.raises(RuntimeError):
                BM.OnlineCorrelation(slice(None), slice(None)).update(*args).get()


def test_reset_and_dtype_follow_the_reference():
    """while no mask entry has been True every update starts the sums over, in its own dtype; afterwards the first
    counted update's dtype is kept"""
    BM = _bm()
    a = torch.randn(4, 3, 5, dtype=torch.float64)
    b = a + torch.randn(4, 3, 5, dtype=torch.float64)
    inf = a.clone()
    inf[0, 0, 0] = float("inf")
    m, off = torch.ones(4, 1, 5, dtype=torch.bool), torch.zeros(4, 1, 5, dtype=torch.bool)
    with metrics_emulator.emulated():
        r = BM.L2Reg(slice(None), slice(None)).update(inf.float(), b.float(), off).update(a, b, m)
        assert r.get().dtype == torch.float64 and not r.get().isnan().any()
        r = BM.L2Reg(slice(None), slice(None)).update(a.float(), b.float(), m).update(a, b, m)
        assert r.get().dtype == torch.float32
        want = (((a - b) ** 2).sum(0) + ((a.float() - b.float()).double() ** 2).sum(0)) / 8
        assert torch.allclose(r.get().double(), want, rtol=1e-6)


def _traced(monkeypatch):
    """inside emulated(): records the entry points called; every host read outside them raises"""
    import brainmagick_b200.functional as BF
    calls = []
    emulated_call = BF.call

    def recording(name, *args):
        calls.append(name)
        return emulated_call(name, *args)
    monkeypatch.setattr(BF, "call", recording)
    _host_reads_forbidden(monkeypatch)
    return calls


def test_each_update_is_one_call_and_reads_nothing_on_the_host(monkeypatch):
    BM = _bm()
    specs, recs, f = load_case("decode_mix")
    with metrics_emulator.emulated():
        metrics = [getattr(BM, kind)(ls, rs, name=name) for kind, name, ls, rs in specs]
        with monkeypatch.context() as mp:
            calls = _traced(mp)
            for left, right, mask in recs[0]:
                for m in metrics:
                    m.update(left, right, mask)
        assert calls == ["bm_metric_update"] * (len(metrics) * len(recs[0]))
        reads = [0]
        item = torch.Tensor.item

        def counted(self):
            reads[0] += 1
            return item(self)
        with monkeypatch.context() as mp:
            calls = _traced(mp)
            mp.setattr(torch.Tensor, "item", counted)
            results = [m.get() for m in metrics]
        assert calls == ["bm_metric_finalize"] * len(metrics) and reads[0] == len(metrics)
        for j, got in enumerate(results):
            assert torch.allclose(got, torch.from_numpy(f[f"result_0_{j}"]), rtol=1e-10, atol=1e-12)


def test_a_new_column_shape_reads_the_seen_word_once(monkeypatch):
    BM = _bm()
    a = torch.randn(4, 3, 5, dtype=torch.float64)
    m = torch.ones(4, 1, 5, dtype=torch.bool)
    with metrics_emulator.emulated():
        c = BM.OnlineCorrelation(slice(None), slice(None)).update(a, a, torch.zeros_like(m))
        reads = []
        original = torch.Tensor.__int__

        def counted(self):
            reads.append(self.numel())
            return original(self)
        monkeypatch.setattr(torch.Tensor, "__int__", counted)
        c.update(a, a, m)
        assert reads == []                                              # the same columns: nothing read
        c2 = BM.OnlineCorrelation(slice(None), slice(None)).update(a, a, torch.zeros_like(m))
        c2.update(a[:, :2], a[:, :2], m)
        assert reads == [1]                                             # new columns: the word is read once
