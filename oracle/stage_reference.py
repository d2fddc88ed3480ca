"""TEST / BENCH INFRASTRUCTURE ONLY -- stages the UNMODIFIED reference under `oracle/_ref/` (git-ignored; it is made by
`__graft_entry__.build()` where the reference source tree is present and travels with the built tree to machines where it is
not) so that `bench.py --impl reference` and the `cpu_baseline` leg time the reference's own modules, not a port.

    python oracle/stage_reference.py          # where the reference source tree is present; build() calls it

Step 1 is an offline install:  pip install --no-index --no-build-isolation --no-deps --target oracle/_ref <copy>
(from a copy under /tmp: /root/reference is read-only and setup.py writes an egg-info beside itself; --no-deps because the
reference's requirements -- mne, flashy, dora-search, hydra, julius ... -- are not in the wheelhouse).  It succeeds, but
the reference's setup.py lists `packages=['bm']` only, so the wheel has bm/losses.py and NOT the sub-package bm/models/.
Step 2 therefore copies bm/models/{__init__,common,simpleconv,features}.py verbatim beside it (byte-identical; checked).
Nothing under oracle/_ref/ is ever committed or edited; oracle/ref_loader.py loads it with the same two stub modules
(`mne.find_layout`, `bm.studies.api.Recording`) it uses for /root/reference.
"""
from __future__ import annotations

import filecmp
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.environ.get("BM_REFERENCE_SRC", "/root/reference")
DST = os.path.join(ROOT, "oracle", "_ref")
MODEL_FILES = ["__init__.py", "common.py", "simpleconv.py", "features.py"]


def staged() -> bool:
    return all(os.path.isfile(os.path.join(DST, "bm", "models", f)) for f in MODEL_FILES) and \
        os.path.isfile(os.path.join(DST, "bm", "losses.py"))


def stage(force: bool = False) -> str:
    """Returns a one-line outcome (also what DESIGN.md records)."""
    if not os.path.isdir(os.path.join(SRC, "bm")):
        return "reference source tree absent: using the staged oracle/_ref" if staged() else \
            "reference source tree absent and oracle/_ref not staged"
    if staged() and not force:
        same = all(filecmp.cmp(os.path.join(SRC, "bm", "models", f), os.path.join(DST, "bm", "models", f), shallow=False)
                   for f in MODEL_FILES)
        if same:
            return "oracle/_ref already staged (bm/models byte-identical to the reference)"
    os.makedirs(DST, exist_ok=True)
    pip_outcome = "skipped"
    with tempfile.TemporaryDirectory() as tmp:
        copy = os.path.join(tmp, "reference")
        shutil.copytree(SRC, copy, ignore=shutil.ignore_patterns(".git", "*.png", "doc", "notebook_templates"))
        res = subprocess.run([sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps",
                              "--find-links", "/opt/wheelhouse", "--upgrade", "--target", DST, copy],
                             capture_output=True, text=True)
        pip_outcome = "ok" if res.returncode == 0 else f"failed rc={res.returncode}: {res.stderr.strip().splitlines()[-1:]}"
    if not os.path.isfile(os.path.join(DST, "bm", "losses.py")):      # pip failed altogether: take the flat package files too
        os.makedirs(os.path.join(DST, "bm"), exist_ok=True)
        for f in ("__init__.py", "losses.py", "norm.py"):
            shutil.copyfile(os.path.join(SRC, "bm", f), os.path.join(DST, "bm", f))
    os.makedirs(os.path.join(DST, "bm", "models"), exist_ok=True)
    for f in MODEL_FILES:                                                # the sub-package setup.py forgets
        shutil.copyfile(os.path.join(SRC, "bm", "models", f), os.path.join(DST, "bm", "models", f))
    assert staged()
    return f"pip install --no-deps --target oracle/_ref: {pip_outcome}; bm/models/ (absent from the wheel) copied verbatim"


if __name__ == "__main__":
    print(stage(force="--force" in sys.argv))
