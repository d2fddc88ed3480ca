"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/bn_state_*.npz, the fixtures of BatchNorm layers that follow their own
module (torch.nn.BatchNorm1d): per-layer train / eval mode inside a training step, per-layer eps and momentum, and the
cumulative moving average of momentum=None, by running the VERBATIM reference SimpleConv and DeepMel (loaded by
`oracle/ref_loader.py`) on small seeded inputs.  The reference tree does not travel with the repository; the fixtures do.

    python tools/make_bn_state_golden.py            # (re)writes the bn_state_*.npz fixtures
    python tools/make_bn_state_golden.py --check    # regenerates in memory and compares with tests/golden/

Each case is a seeded construction whose BatchNorm affine parameters and running statistics are perturbed (`p.<key>`),
then `SETUPS[case["setup"]]` -- the same function the tests apply to the drop-in modules -- sets the layers' modes and
settings.  Then `steps` training steps of loss = sum(out * w{i}) on the inputs `in{i}.<stream>` (the merger's dropout
centre `ban{i}`), each recording `s{i}.out`, every parameter gradient `s{i}.g.<key>` and the input gradients
`s{i}.g.in.<stream>`; after them the running buffers and counters `bn.<key>`, and an eval forward on the first step's
inputs (`out_eval`).
"""
from __future__ import annotations

import os
import sys

if __name__ == "__main__" and "--compute" in sys.argv:
    # pinned arithmetic in the child process, as in tools/make_encode_golden.py: --check compares bitwise on any x86 host
    os.environ["ATEN_CPU_CAPABILITY"] = "default"
    os.environ["MKL_CBWR"] = "COMPATIBLE"
    os.environ["OMP_NUM_THREADS"] = "1"

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from oracle.encode_oracle import EncodeVariant  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

_SMALL = dict(n_subjects=3, merger_channels=12, initial_linear=12, merger_pos_dim=32)
CLIP_CONV = EncodeVariant(in_channels=dict(meg=10), hidden=dict(meg=16), out_channels=8, depth=6, **_SMALL)
TWO_STREAM = EncodeVariant(in_channels=dict(meg=10, features=7), hidden=dict(meg=16, features=12), out_channels=10, depth=4,
                           **_SMALL)
DEEPMEL = dict(n_in_channels=10, n_hidden_channels=16, n_hidden_layers=4, n_out_channels=24, kernel=3, stride=1,
               dilation_growth=2, dilation_period=5, batch_norm=True, activation_on_last=False, skip=True, glu_context=1,
               glu=2)

# per-layer eps and momentum of the `eps_momentum` setup, layer k of the 6-layer encoder
EPS = (1e-5, 1e-3, 1e-1, 1e-4, 3e-2, 1e-2)
MOMENTUM = (0.1, 0.01, 0.5, 0.3, 0.9, 0.05)


def _bns(seq):
    return [m for m in seq.modules() if isinstance(m, torch.nn.BatchNorm1d)]


def eval_layers(model):
    """clip_conv with BatchNorm layers 2 and 5 in eval mode inside a training step"""
    model.train()
    for k in (2, 5):
        model.encoders["meg"].sequence[k][1].eval()


def frozen_encoders(model):
    """head-only fine-tuning / subject adaptation: model.train(); model.encoders.eval(), the encoders frozen"""
    model.train()
    model.encoders.eval()
    for t in model.encoders.parameters():
        t.requires_grad_(False)


def eps_momentum(model):
    model.train()
    for bn, eps, momentum in zip(_bns(model.encoders["meg"]), EPS, MOMENTUM):
        bn.eps, bn.momentum = eps, momentum


def cumulative(model):
    """what torch.optim.swa_utils.update_bn does: fresh buffers, momentum=None on every layer"""
    model.train()
    for bn in _bns(model):
        bn.reset_running_stats()
        bn.momentum = None


def two_stream(model):
    model.train()
    model.encoders["features"].eval()


def deepmel_mixed(model):
    model.train()
    model.sequence[1][1].eval()
    model.sequence[0][1].eps = 1e-3
    model.sequence[2][1].momentum = 0.3


SETUPS = dict(eval_layers=eval_layers, frozen_encoders=frozen_encoders, eps_momentum=eps_momentum, cumulative=cumulative,
              two_stream=two_stream, deepmel_mixed=deepmel_mixed)

# name: model (an EncodeVariant of SimpleConv, or "deepmel"), setup, training steps, B, T, seed
CASES = {
    "bn_state_eval_layers": dict(model=CLIP_CONV, setup="eval_layers", steps=2, B=4, T=22, seed=41),
    "bn_state_frozen_encoders": dict(model=CLIP_CONV, setup="frozen_encoders", steps=2, B=4, T=22, seed=42),
    "bn_state_eps_momentum": dict(model=CLIP_CONV, setup="eps_momentum", steps=2, B=4, T=22, seed=43),
    "bn_state_cumulative": dict(model=CLIP_CONV, setup="cumulative", steps=3, B=4, T=22, seed=44),
    "bn_state_deepmel": dict(model="deepmel", setup="deepmel_mixed", steps=2, B=5, T=20, seed=45),
    "bn_state_two_stream": dict(model=TWO_STREAM, setup="two_stream", steps=2, B=4, T=22, seed=46),
}


def streams(c) -> dict:
    """input stream -> channels of a case"""
    return dict(x=DEEPMEL["n_in_channels"]) if c["model"] == "deepmel" else dict(c["model"].in_channels)


def out_channels(c) -> int:
    return DEEPMEL["n_out_channels"] if c["model"] == "deepmel" else c["model"].out_channels


def _reference_model(c):
    if c["model"] == "deepmel":
        import importlib.util
        ref_loader.load_reference()
        spec = importlib.util.spec_from_file_location("bm.models.features", ref_loader.REF + "/models/features.py")
        feats = importlib.util.module_from_spec(spec)
        sys.modules["bm.models.features"] = feats
        spec.loader.exec_module(feats)
        return feats.DeepMel(**DEEPMEL)
    _, simpleconv, _ = ref_loader.load_reference()
    return simpleconv.SimpleConv(**c["model"].kwargs())


def _perturb(model):
    with torch.no_grad():
        for m in _bns(model):
            m.weight.add_(0.1 * torch.randn_like(m.weight))
            m.bias.add_(0.1 * torch.randn_like(m.bias))
            m.running_mean.add_(0.1 * torch.randn_like(m.running_mean))
            m.running_var.mul_(1 + 0.2 * torch.rand_like(m.running_var))


def make_case(name: str) -> dict:
    """the seeded construction and the random draws here, the reference's steps in a pinned child process"""
    import subprocess
    import tempfile
    c = CASES[name]
    seed = c["seed"]
    torch.manual_seed(seed)
    model = _reference_model(c)
    torch.manual_seed(1000 + seed)
    _perturb(model)
    res = {"p." + k: t.detach().clone().numpy() for k, t in model.state_dict().items()}
    gen = torch.Generator().manual_seed(seed)
    for i in range(c["steps"]):
        for s, ch in streams(c).items():
            res[f"in{i}.{s}"] = torch.randn((c["B"], ch, c["T"]), generator=gen).numpy()
        res[f"w{i}"] = torch.randn((c["B"], out_channels(c), c["T"]), generator=gen).numpy()
    if c["model"] != "deepmel":
        res["subject_index"] = torch.randint(0, c["model"].n_subjects, (c["B"],), generator=gen).numpy()
    with tempfile.TemporaryDirectory() as tmp:
        src, dst = os.path.join(tmp, "in.npz"), os.path.join(tmp, "out.npz")
        np.savez(src, **res)
        subprocess.run([sys.executable, os.path.abspath(__file__), "--compute", name, src, dst], check=True)
        with np.load(dst) as z:
            res.update({k: z[k] for k in z.files})
    return res


def compute(name: str, src: str, dst: str) -> None:
    """the reference's training steps and eval forward on the parameters and inputs of `src` (see make_case)"""
    torch.set_num_threads(1)
    torch.backends.mkldnn.enabled = False
    c = CASES[name]
    g = np.load(src)
    model = _reference_model(c)
    model.load_state_dict({k[2:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("p.")}, strict=True)
    SETUPS[c["setup"]](model)
    res = {}
    batch = None
    if c["model"] != "deepmel":
        common, _, _ = ref_loader.load_reference()
        C, S = c["model"].in_channels["meg"], c["model"].n_subjects
        subj = torch.from_numpy(g["subject_index"])
        recs = [ref_loader.FakeRecording(s, C, C, seed=c["seed"]) for s in range(S)]
        batch = ref_loader.FakeBatch(torch.from_numpy(g["in0.meg"]), subj, [recs[int(s)] for s in subj])
        pos_rec = torch.stack([model.merger.position_getter.get_recording_layout(r).clone() for r in recs])
        full = torch.full((S, C, 2), common.PositionGetter.INVALID)
        full[:, :pos_rec.shape[1]] = pos_rec
        res["rec_positions"] = full.numpy()

    def run(inputs):
        return model(inputs["x"]) if batch is None else model(dict(inputs), batch)

    for i in range(c["steps"]):
        model.zero_grad(set_to_none=True)
        torch.manual_seed(9000 + c["seed"] + i)
        res[f"ban{i}"] = torch.rand(2).numpy()      # the one rand(2) the training forward draws (common.py:343)
        torch.manual_seed(9000 + c["seed"] + i)
        leaves = {s: torch.from_numpy(g[f"in{i}.{s}"]).clone().requires_grad_(True) for s in streams(c)}
        out = run(leaves)
        (out * torch.from_numpy(g[f"w{i}"])).sum().backward()
        res[f"s{i}.out"] = out.detach().numpy()
        res.update({f"s{i}.g.in.{s}": t.grad.numpy() for s, t in leaves.items()})
        res.update({f"s{i}.g.{k}": t.grad.numpy() for k, t in model.named_parameters() if t.grad is not None})
    res.update({"bn." + k: t.numpy() for k, t in model.state_dict().items() if "running" in k or "num_batches" in k})
    model.eval()
    with torch.no_grad():
        res["out_eval"] = run({s: torch.from_numpy(g[f"in0.{s}"]) for s in streams(c)}).numpy()
    np.savez(dst, **res)


def main(check: bool) -> int:
    bad = 0
    for name in CASES:
        arrays = make_case(name)
        path = os.path.join(OUT, name + ".npz")
        if check:
            old = np.load(path)
            same = set(old.files) == set(arrays) and all(np.array_equal(old[k], arrays[k]) for k in arrays)
            print(f"{name}: {'same' if same else 'DIFFERS'}")
            bad += not same
        else:
            np.savez_compressed(path, **arrays)
            print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB")
    return bad


if __name__ == "__main__":
    if "--compute" in sys.argv:
        compute(*sys.argv[sys.argv.index("--compute") + 1:][:3])
        sys.exit(0)
    sys.exit(main("--check" in sys.argv))
