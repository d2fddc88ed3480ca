"""GPU parity for the SURVEY 8(f) rows built after the training step: batch preparation (bit-exact against the verbatim
reference fixture and the oracle) and retrieval evaluation (fixture, oracle, and self-consistency of the fused top-k)."""
import types

import numpy as np
import pytest
import torch

from conftest import load_arrays
from oracle import bm_oracle, eval_oracle, prep_oracle
from brainmagick_b200 import functional as BF
from brainmagick_b200 import norm as bnorm
from brainmagick_b200 import retrieval, synthetic
from brainmagick_b200.losses import ClipLoss

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ------------------------------------------------------------------------------------------------------------------
# batch preparation
# ------------------------------------------------------------------------------------------------------------------
class _Builder(dict):
    def __init__(self, dims):
        super().__init__()
        self._slices, start = {}, 0
        for name, (dim, normalizable) in dims.items():
            self[name] = types.SimpleNamespace(normalizable=normalizable, categorical=False, cardinality=0)
            self._slices[name] = slice(start, start + dim)
            start += dim
        self.dimension = start

    def get_slice(self, name):
        return self._slices[name]


def _fixture_scaler(g, tag):
    sc = bnorm.BatchScaler(_Builder({"a": (3, True), "b": (2, False)}), per_channel=(tag == "pc1."))
    for i, r in enumerate(g["rec_ids"]):
        s = bnorm.Scaler()
        s.center_, s.scale_ = torch.from_numpy(g[tag + "meg_center"][i]), torch.from_numpy(g[tag + "meg_scale"][i])
        sc.meg_scalers[int(r)] = s
    sc.feature_scalers["a"].center_ = torch.from_numpy(g[tag + "feat_center"][:3])
    sc.feature_scalers["a"].scale_ = torch.from_numpy(g[tag + "feat_scale"][:3])
    return sc


def _fixture_batch(g, meg=None, features=None):
    meg = g["meg"] if meg is None else meg
    features = g["features"] if features is None else features
    B = len(meg)
    return synthetic.SyntheticBatch(torch.from_numpy(meg).to(DEV), torch.zeros(B, dtype=torch.long, device=DEV), [],
                                    features=torch.from_numpy(features).to(DEV),
                                    features_mask=torch.from_numpy(g["features_mask"]).to(DEV),
                                    recording_index=torch.from_numpy(g["recording_index"]).to(DEV))


@pytest.mark.parametrize("tag", ["pc0.", "pc1."])
def test_prep_transform_bit_exact(tag):
    g = load_arrays("prep_small")
    sc = _fixture_scaler(g, tag)
    out = sc.transform(_fixture_batch(g))
    assert np.array_equal(out.meg.cpu().numpy(), g[tag + "transform.meg"])
    assert np.array_equal(out.features.cpu().numpy(), g[tag + "transform.features"])
    back = sc.inverse_transform(out)
    assert np.array_equal(back.meg.cpu().numpy(), g[tag + "inverse.meg"])
    assert np.array_equal(back.features.cpu().numpy(), g[tag + "inverse.features"])


@pytest.mark.parametrize("clip", [0, 1])
@pytest.mark.parametrize("excl", [0, 1])
def test_prep_scale_reject_bit_exact(clip, excl):
    g = load_arrays("prep_small")
    off = int(g["offset"])
    for tag in ("pc0.", "pc1."):
        k = f"{tag}clip{clip}.excl{excl}."
        sr = bnorm.ScaleReject(_fixture_scaler(g, tag), limit=float(g["limit"]), exclude_empty_features=bool(excl),
                               clip=bool(clip))
        kept, keep = sr(_fixture_batch(g))
        assert np.array_equal(keep.cpu().numpy(), g[k + "keep"])
        assert len(kept) == int(g[k + "keep"].sum())
        assert np.array_equal(kept.meg[..., off:].cpu().numpy(), g[k + "meg"])
        assert np.array_equal(kept.features[..., :-off].cpu().numpy(), g[k + "features"])
        assert np.array_equal(kept.recording_index.cpu().numpy(), g["recording_index"][g[k + "keep"]])
        assert sr.rejection_rate == pytest.approx(float(g[k + "rejection_rate"]))
        # the fused form: scale + clamp + reject + offset crop in one pass
        meg, feats, mask, keep2 = sr.prepare(_fixture_batch(g), off)
        assert np.array_equal(keep2.cpu().numpy(), g[k + "keep"])
        assert np.array_equal(meg.cpu().numpy(), g[k + "meg"])
        assert np.array_equal(feats.cpu().numpy(), g[k + "features"])
        assert np.array_equal(mask.cpu().numpy(), g[k + "features_mask"])


def _big_prep(B=256, C=273, T=361, F=1024, R=27, seed=3):
    rng = np.random.RandomState(seed)
    center = {r: rng.randn(C).astype(np.float32) * 0.1 for r in range(R)}
    scale = {r: (0.5 + rng.rand(C)).astype(np.float32) for r in range(R)}
    for r in range(R):
        scale[r][C - 5:] = 1.0                                   # padded channels
    meg = (rng.randn(B, C, T) * 3).astype(np.float32)
    meg[7, 3, 100] = 1000.0
    rec = rng.randint(0, R, size=B)
    feats = rng.randn(B, F, T).astype(np.float32)
    fc = np.full(F, 0.25, np.float32)
    fs = np.full(F, 1.75, np.float32)
    return center, scale, meg, rec, feats, fc, fs


def test_prep_full_size_bit_exact_and_rate():
    """BASELINE shape (B=256, C=273, T=361 -> 343 after the 150 ms offset, F=1024): bit-exact against the oracle, and
    the one-pass kernel's HBM rate (algorithmic bytes = read + write of the kept window)."""
    center, scale, meg, rec, feats, fc, fs = _big_prep()
    B, C, T = meg.shape
    F = feats.shape[1]
    sc = bnorm.BatchScaler(_Builder({"wav": (F, True)}))
    for r in center:
        s = bnorm.Scaler()
        s.center_, s.scale_ = torch.from_numpy(center[r]), torch.from_numpy(scale[r])
        sc.meg_scalers[r] = s
    sc.feature_scalers["wav"].center_ = torch.tensor(0.25)
    sc.feature_scalers["wav"].scale_ = torch.tensor(1.75)
    mask = np.ones((B, 1, T), dtype=bool)
    batch = synthetic.SyntheticBatch(torch.from_numpy(meg).to(DEV), torch.zeros(B, dtype=torch.long, device=DEV), [],
                                     features=torch.from_numpy(feats).to(DEV),
                                     features_mask=torch.from_numpy(mask).to(DEV),
                                     recording_index=torch.from_numpy(rec).to(DEV))
    off = 18
    for clip in (True, False):
        sr = bnorm.ScaleReject(sc, limit=20.0, clip=clip)
        m, f, msk, keep = sr.prepare(batch, off)
        want = prep_oracle.prepare(meg, rec, center, scale, feats, mask, fc, fs, limit=20.0, clip=clip,
                                   offset_samples=off)
        assert np.array_equal(keep.cpu().numpy(), want["keep"])
        assert (not clip) == (not want["keep"].all())
        assert np.array_equal(m.cpu().numpy(), want["meg"])
        assert np.array_equal(f.cpu().numpy(), want["features"])
        assert msk.shape == want["features_mask"].shape
    # round trip
    out = sc.transform(batch)
    back = sc.inverse_transform(out)
    assert (back.meg - batch.meg).abs().max().item() < 5e-3
    # rate of the fused pass (clip=True: the training configuration)
    sr = bnorm.ScaleReject(sc, limit=20.0, clip=True)
    for _ in range(3):
        sr.prepare(batch, off)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        sr.prepare(batch, off)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    gbytes = 2 * 4 * B * (C + F) * (T - off) / 1e9
    print(f"\n[prep] B={B} C={C} F={F} T={T}->{T - off}: {ms:.3f} ms/batch (2 launches, no host sync), "
          f"{gbytes / ms * 1e3:.0f} GB/s algorithmic, {B / ms * 1e3:.0f} seg/s")


# ------------------------------------------------------------------------------------------------------------------
# retrieval evaluation
# ------------------------------------------------------------------------------------------------------------------
def test_topk_kernel_against_torch():
    torch.manual_seed(0)
    Bn, n, ld, k = 37, 1000, 1024, 10
    scores = torch.randn(Bn, ld, device=DEV)
    labels = torch.randint(-5, 60, (n,), device=DEV, dtype=torch.int64) * 1_000_003
    targets = labels[torch.randint(0, n, (Bn,), device=DEV)]
    r = retrieval._topk(scores, n, k, labels, targets, want_soft=True, want_stats=True)
    p = torch.softmax(scores[:, :n], dim=1)
    tv, ti = p.topk(k, dim=1)
    assert torch.equal(r["top_idx"], ti)
    assert torch.allclose(r["top_prob"], tv, rtol=1e-5, atol=1e-9)
    match = labels[ti] == targets[:, None]
    first = torch.where(match.any(1), match.float().argmax(1), torch.full((Bn,), -1, device=DEV)).int()
    assert torch.equal(r["hit"], first)
    soft = (p * (labels[None] == targets[:, None])).sum(1)
    assert torch.allclose(r["soft"], soft, rtol=1e-5, atol=1e-8)
    assert torch.allclose(r["row_max"], scores[:, :n].max(1).values)
    # own column: per-row override of one column's value and label
    own = torch.randn(Bn, device=DEV) + 3
    own_l = targets.clone()
    r2 = retrieval._topk(scores, n, k, labels, targets, own_values=own, own_col=n - 1, own_labels=own_l, want_soft=True)
    s2 = scores[:, :n].clone()
    s2[:, n - 1] = own
    p2 = torch.softmax(s2, dim=1)
    assert torch.equal(r2["top_idx"], p2.topk(k, dim=1).indices)
    lab2 = labels[None].repeat(Bn, 1)
    lab2[:, n - 1] = own_l
    assert torch.allclose(r2["soft"], (p2 * (lab2 == targets[:, None])).sum(1), rtol=1e-5, atol=1e-8)
    # probabilities with holes, fewer columns than k, ties -> lower column first
    pv = torch.tensor([[0.5, -1.0, 0.25, 0.25, -1.0]], device=DEV)
    r3 = retrieval._topk(pv, 5, 4, torch.arange(5, device=DEV), torch.tensor([3], device=DEV), is_prob=True)
    assert r3["top_idx"].tolist() == [[0, 2, 3, -1]] and r3["hit"].tolist() == [2]
    assert r3["top_prob"].tolist() == [[0.5, 0.25, 0.25, 0.0]]


def test_retrieval_fixture():
    g = load_arrays("retrieval_small")
    clip = ClipLoss().eval()
    preds, trues = torch.from_numpy(g["preds"]), torch.from_numpy(g["trues"])
    labels, targets = torch.from_numpy(g["vocab_labels"]), torch.from_numpy(g["target_labels"])
    args = types.SimpleNamespace(tmin=-0.5, sample_rate=120.0)
    probs = retrieval.builds_probs(clip, preds, trues, args, batch_size=10)
    assert not probs.is_cuda and probs.shape == (24, 17)
    assert np.abs(probs.numpy() - g["probs"]).max() < 2e-6
    pw = retrieval.builds_probs(clip, preds, trues, args, batch_size=7, tmin=-0.45, tmax=-0.4)
    assert np.abs(pw.numpy() - g["probs_window"]).max() < 2e-6
    for k, want in zip((1, 5, 10), g["acc"]):
        assert retrieval._get_accuracy_from_probs(torch.from_numpy(g["probs"]), targets, labels, topk=k) == \
            pytest.approx(float(want))
    acc = retrieval.retrieval_accuracy(clip, preds, trues, targets, labels, topk=(1, 5, 10), batch_size=9)
    assert [acc[1], acc[5], acc[10]] == pytest.approx([float(a) for a in g["acc"]])


def test_wer_fixture():
    g = load_arrays("retrieval_small")
    t = lambda k: torch.from_numpy(g[k])     # noqa: E731
    clip = ClipLoss().eval()
    for bs in (5, 64):
        res = retrieval.wer_ranking(clip, t("wer_estimates"), t("wer_word_hashes"), t("wer_outputs"),
                                    t("wer_negatives"), t("wer_negative_hashes"), int(g["wer_topx"]), batch_size=bs)
        assert res["wer"] == pytest.approx(float(g["wer"]))
        assert res["wer_vocab"] == pytest.approx(float(g["wer_vocab"]))
        assert res["soft_correct"] == pytest.approx(float(g["wer_soft"]), rel=1e-4)


def _retrieval_task(n, m, F, T, n_words, signal, seed):
    gen = torch.Generator().manual_seed(seed)
    trues = torch.randn(m, F, T, generator=gen)
    seg = torch.randint(0, m, (n,), generator=gen)
    preds = signal * trues[seg] + torch.randn(n, F, T, generator=gen)
    labels = torch.randperm(1 << 20, generator=gen)[:m].to(torch.int64) - (1 << 19)
    words = torch.randint(1, n_words + 1, (m,), generator=gen, dtype=torch.int32)
    return trues, seg, preds, labels, words


def test_retrieval_tensor_core_path():
    """Candidate axis padded to the tensor-core tile (1000 -> 1024), K = F*T = 2048: scores against the oracle, the fused
    top-k against torch.topk on the very same scores, accuracies against the oracle's."""
    trues, seg, preds, labels, _ = _retrieval_task(n=300, m=1000, F=16, T=128, n_words=0 + 1, signal=0.06, seed=11)
    clip = ClipLoss().eval()
    bank = retrieval.CandidateBank(clip, trues)
    assert bank.n_pad == 1024 and bank.rows.shape == (1024, 2048)
    before = BF._lib.launch_count()
    scores = bank.scores(clip, preds)
    assert BF._lib.launch_count() - before == 2, "expected the tensor-core score GEMM + its split-K reduction"
    BF.check_tc_status()
    want = bm_oracle.clip_scores(preds, trues)
    got = scores[:, :1000].cpu()
    assert (got - want).norm() / want.norm() < 3e-5
    assert scores[:, 1000:].abs().max().item() == 0.0            # zero padding rows score exactly 0
    r = retrieval._topk(scores, 1000, 10, labels.to(DEV), labels[seg].to(DEV))
    assert torch.equal(r["top_idx"], torch.softmax(scores[:, :1000], 1).topk(10, dim=1).indices)
    acc = retrieval.retrieval_accuracy(clip, preds, trues, labels[seg], labels, topk=(1, 5, 10), batch_size=128)
    probs = eval_oracle.builds_probs(preds, trues, batch_size=100)
    for k in (1, 5, 10):
        ref = eval_oracle.accuracy_from_probs(probs, labels[seg], labels, k)
        assert abs(acc[k] - ref) <= 2 / 300 + 1e-9, (k, acc[k], ref)
    assert 0.05 < acc[10] < 0.95


def test_wer_tensor_core_path():
    trues, seg, _, _, words = _retrieval_task(n=10, m=700, F=16, T=128, n_words=60, signal=0.0, seed=12)
    gen = torch.Generator().manual_seed(13)
    n, n_neg, topx = 160, 513, 10
    outputs = trues[:n]
    word_hashes = words[:n]
    estimates = 0.035 * outputs + torch.randn(n, 16, 128, generator=gen)
    kept = torch.randperm(700, generator=gen)[:n_neg]
    negatives, negative_hashes = trues[kept], words[kept]
    clip = ClipLoss().eval()
    res = retrieval.wer_ranking(clip, estimates, word_hashes, outputs, negatives, negative_hashes, topx, batch_size=100)
    BF.check_tc_status()
    ref = eval_oracle.wer_ranking(estimates, word_hashes, outputs, negatives, negative_hashes, topx)
    assert abs(res["wer"] - ref["wer"]) <= 2 / n + 1e-9, (res, ref)
    assert abs(res["wer_vocab"] - ref["wer_vocab"]) <= 2 / n + 1e-9, (res, ref)
    assert res["soft_correct"] == pytest.approx(ref["soft_correct"], rel=2e-4)
    assert 0.05 < ref["wer"] < 0.95 and 0.02 < ref["wer_vocab"] < 0.98
    rnd = retrieval.wer_ranking(clip, estimates, word_hashes, outputs, negatives, negative_hashes, topx, wer_random=True)
    assert rnd["wer"] > ref["wer"]
