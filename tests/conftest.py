import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
GOLDEN_CASES = ["train_small", "eval_small", "train_padded_negs", "train_depth4"]


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    """Returns (cfg: oracle.Config, train: bool, tensors: dict) for one fixture made by oracle/make_golden.py."""
    from oracle import bm_oracle
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    B, Bc, C, T, F, S, hidden, depth, MC, IL, P, train = [int(v) for v in z["cfg"]]
    cfg = bm_oracle.Config(in_channels=C, out_channels=F, n_subjects=S, hidden=hidden, depth=depth,
                           merger_channels=MC, initial_linear=IL, merger_pos_dim=P)
    t = {k: torch.from_numpy(z[k]) for k in z.files if k != "cfg"}
    return cfg, bool(train), t


def load_arrays(name):
    """Plain dict of numpy arrays of a fixture without a model configuration (prep_small, retrieval_small)."""
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    return {k: z[k] for k in z.files}


def rel_err(a, b):
    """Relative Frobenius error ||a-b|| / ||b|| (b = reference)."""
    a, b = a.double(), b.double()
    den = b.norm().item()
    return (a - b).norm().item() / (den if den > 0 else 1.0)


@pytest.fixture(params=GOLDEN_CASES)
def golden(request):
    return (request.param,) + load_golden(request.param)
