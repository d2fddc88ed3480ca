"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/encode_*.npz, the fixtures of SimpleConv over several input streams
(the encoding configuration, bm/train.py:61-67 and bm/solver.py:283-294; `concatenate`, `linear_out`, the join of the
encoder outputs; bm/models/simpleconv.py:150-249), by running the VERBATIM reference SimpleConv (loaded by
`oracle/ref_loader.py`) on small seeded inputs.  The reference tree does not travel with the repository; the fixtures do.

    python tools/make_encode_golden.py            # (re)writes the encode_*.npz fixtures
    python tools/make_encode_golden.py --check    # regenerates in memory and compares with tests/golden/

Each fixture: `init.<key>` the state_dict of the seeded construction, `p.<key>` the state after perturbing the BatchNorm
affine parameters and running statistics, the inputs `in.<stream>` [B, C_s, T] with `subject_index`, `rec_positions`,
`ban_centre`, the output weights `w_out`, then a training step of loss = sum(out * w_out): `out`, the gradient of every
parameter (`g.<key>`) and of every input stream (`g.in.<stream>`), the running statistics after it (`bn.<key>`), and an
eval forward with those statistics (`out_eval`).
"""
from __future__ import annotations

import os
import sys

if __name__ == "__main__" and "--compute" in sys.argv:
    # The reference's arithmetic runs in a child process pinned to one path on every x86 host, so that --check compares
    # bitwise wherever it runs: ATen's portable (non-AVX) kernels, MKL's conditional-numerical-reproducibility mode, one
    # thread, no oneDNN.  Without them the fp32 results move by a rounding step between CPUs that dispatch to different
    # vector widths.  The seeded construction and every random draw stay in the parent, on the default kernels: they are
    # what a user's seeded constructor reproduces.
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

_SMALL = dict(n_subjects=3, depth=4, merger_channels=12, initial_linear=12, merger_pos_dim=32)
# name: (variant, B, T, seed)
CASES = {
    # two streams, complex_out, the full clip_conv front on meg
    "encode_two_complex": (EncodeVariant(in_channels=dict(meg=10, features=7), hidden=dict(meg=16, features=12),
                                         out_channels=10, **_SMALL), 4, 22, 31),
    "encode_two_linear": (EncodeVariant(in_channels=dict(meg=10, features=7), hidden=dict(meg=16, features=12),
                                        out_channels=10, linear_out=True, complex_out=False, **_SMALL), 4, 22, 32),
    "encode_concat_bare": (EncodeVariant(in_channels=dict(meg=10, features=7), hidden=dict(meg=16, features=12),
                                         out_channels=10, concatenate=True, complex_out=False, **_SMALL), 4, 22, 33),
    "encode_concat_linear_emb": (EncodeVariant(in_channels=dict(meg=10, features=7), hidden=dict(meg=16, features=12),
                                               out_channels=10, concatenate=True, linear_out=True, complex_out=False,
                                               subject_layers=False, subject_dim=4, **_SMALL), 4, 22, 34),
    # three streams whose sorted order (audio, meg, wav) is not their insertion order
    "encode_three": (EncodeVariant(in_channels=dict(wav=6, meg=10, audio=5), hidden=dict(wav=8, meg=16, audio=12),
                                   out_channels=10, **_SMALL), 3, 20, 35),
}


def _perturb(model):
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.add_(0.1 * torch.randn_like(m.weight))
                m.bias.add_(0.1 * torch.randn_like(m.bias))
                m.running_mean.add_(0.1 * torch.randn_like(m.running_mean))
                m.running_var.mul_(1 + 0.2 * torch.rand_like(m.running_var))


def make_case(name: str) -> dict:
    """the seeded construction and the random draws here, the reference's forward / backward in a pinned child process"""
    import subprocess
    import tempfile
    v, B, T, seed = CASES[name]
    _, simpleconv, _ = ref_loader.load_reference()
    torch.manual_seed(seed)
    model = simpleconv.SimpleConv(**v.kwargs())
    init = {k: t.detach().clone() for k, t in model.state_dict().items()}
    torch.manual_seed(1000 + seed)
    _perturb(model)
    state = {k: t.detach().clone() for k, t in model.state_dict().items()}
    inputs = {name: torch.randn(B, c, T) for name, c in v.in_channels.items()}
    subj = torch.randint(0, v.n_subjects, (B,))
    w_out = torch.randn((B, v.out_channels, T), generator=torch.Generator().manual_seed(seed))
    res = dict(subject_index=subj.numpy(), w_out=w_out.numpy())
    res.update({"in." + n: t.numpy() for n, t in inputs.items()})
    res.update({"p." + k: t.numpy() for k, t in state.items()})
    with tempfile.TemporaryDirectory() as tmp:
        src, dst = os.path.join(tmp, "in.npz"), os.path.join(tmp, "out.npz")
        np.savez(src, **res)
        subprocess.run([sys.executable, os.path.abspath(__file__), "--compute", name, src, dst], check=True)
        with np.load(dst) as z:
            res.update({k: z[k] for k in z.files})
    res.update({"init." + k: t.numpy() for k, t in init.items()})
    return res


def compute(name: str, src: str, dst: str) -> None:
    """the reference's training step and eval forward on the parameters and inputs of `src` (see make_case)"""
    torch.set_num_threads(1)
    torch.backends.mkldnn.enabled = False
    v, B, T, seed = CASES[name]
    g = np.load(src)
    common, simpleconv, _ = ref_loader.load_reference()
    model = simpleconv.SimpleConv(**v.kwargs())
    model.load_state_dict({k[2:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("p.")}, strict=True)
    inputs = {n: torch.from_numpy(g["in." + n]) for n in v.in_channels}
    subj = torch.from_numpy(g["subject_index"])
    C, S = v.in_channels["meg"], v.n_subjects
    recs = [ref_loader.FakeRecording(s, C, C, seed=seed) for s in range(S)]
    batch = ref_loader.FakeBatch(inputs["meg"], subj, [recs[int(s)] for s in subj])
    pos_rec = torch.stack([model.merger.position_getter.get_recording_layout(r).clone() for r in recs])
    full = torch.full((S, C, 2), common.PositionGetter.INVALID)
    full[:, :pos_rec.shape[1]] = pos_rec
    model.train()
    torch.manual_seed(9000 + seed)
    ban = torch.rand(2)                       # the one rand(2) the training forward draws (common.py:343)
    torch.manual_seed(9000 + seed)
    leaves = {n: t.clone().requires_grad_(True) for n, t in inputs.items()}
    out = model(dict(leaves), batch)
    (out * torch.from_numpy(g["w_out"])).sum().backward()
    res = dict(rec_positions=full.numpy(), ban_centre=ban.numpy(), out=out.detach().numpy())
    res.update({"g.in." + n: t.grad.numpy() for n, t in leaves.items()})
    res.update({"g." + k: t.grad.numpy() for k, t in model.named_parameters()})
    res.update({"bn." + k: t.numpy() for k, t in model.state_dict().items() if "running" in k or "num_batches" in k})
    model.eval()
    with torch.no_grad():
        res["out_eval"] = model(dict(inputs), batch).numpy()
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
