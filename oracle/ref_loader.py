"""TEST INFRASTRUCTURE ONLY -- loads the *verbatim* brainmagick hot-path modules from /root/reference (build container) or
from the unmodified copy build() stages under oracle/_ref/ (oracle/stage_reference.py; `bench.py --impl reference`).

Used by the fixture generators (`oracle/make_golden.py`, incl. its `--check`, and `oracle/make_live_golden.py`); the
tests read what they stored and use only `clip_conv_kwargs`; they never load the reference.  `load_reference_norm()` adds the verbatim
`bm/norm.py`; `bm/models/features.py` (DeepMel) is loaded by the generator the same way.  Nothing in the product package
(`brainmagick_b200/`) imports this file.

The three hot-path files import cleanly once two stub modules exist (SURVEY.md appendix B):
  * `mne`             -- only `mne.find_layout(info)` is touched (bm/models/common.py:196)
  * `bm.studies.api`  -- only the name `Recording` is needed (bm/models/common.py:16)
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

import numpy as np

_STAGED = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


def _find_root() -> str:
    """The reference source tree where present, else the copy build() staged under oracle/_ref (oracle/stage_reference.py)."""
    env = os.environ.get("BM_REFERENCE_ROOT")
    if env:
        return env
    if os.path.isfile("/root/reference/bm/models/simpleconv.py"):
        return "/root/reference"
    return _STAGED


REF_ROOT = _find_root()
REF = os.path.join(REF_ROOT, "bm")
REF_KIND = "source tree" if REF_ROOT == "/root/reference" else "staged copy (oracle/_ref)"


def reference_available() -> bool:
    return os.path.isfile(os.path.join(REF, "models", "simpleconv.py"))


_loaded = None


def load_reference():
    """Returns (common, simpleconv, losses) modules loaded verbatim from the reference tree."""
    global _loaded
    if _loaded is not None:
        return _loaded
    if not reference_available():
        raise RuntimeError(f"reference tree not found under {REF_ROOT}")

    def _pkg(name, path):
        m = types.ModuleType(name)
        m.__path__ = [path]
        sys.modules[name] = m
        return m

    _pkg("bm", REF)
    _pkg("bm.models", REF + "/models")
    _pkg("bm.studies", REF + "/studies")
    if "mne" not in sys.modules:
        sys.modules["mne"] = types.ModuleType("mne")
    mne = sys.modules["mne"]
    mne.find_layout = fake_find_layout
    api = types.ModuleType("bm.studies.api")
    api.Recording = object
    sys.modules["bm.studies.api"] = api

    def _load(name, path):
        spec = importlib.util.spec_from_file_location(name, path)
        m = importlib.util.module_from_spec(spec)
        sys.modules[name] = m
        spec.loader.exec_module(m)
        return m

    common = _load("bm.models.common", REF + "/models/common.py")
    simpleconv = _load("bm.models.simpleconv", REF + "/models/simpleconv.py")
    losses = _load("bm.losses", REF + "/losses.py")
    _loaded = (common, simpleconv, losses)
    return _loaded


# ----------------------------------------------------------------------------------------------
# Fake recordings / layouts / batches (stand-ins for bm.studies.api.Recording + mne layouts)
# ----------------------------------------------------------------------------------------------
class FakeInfo:
    def __init__(self, ch_names, layout_names, layout_pos):
        self.ch_names = list(ch_names)
        self._layout_names = list(layout_names)
        self._layout_pos = np.asarray(layout_pos, dtype=np.float64)


def fake_find_layout(info):
    """Stand-in for mne.find_layout: an object with .names and .pos[n,4] (common.py:196,215)."""
    return types.SimpleNamespace(names=list(info._layout_names), pos=info._layout_pos)


class FakeRecording:
    """Has exactly what PositionGetter touches (common.py:190-209)."""

    def __init__(self, recording_index: int, n_channels: int, n_valid: int | None = None, seed: int = 0):
        n_valid = n_channels if n_valid is None else n_valid
        rng = np.random.RandomState(1000 + seed + 7919 * recording_index)
        names = [f"CH{recording_index}_{i}" for i in range(n_channels)]
        pos = rng.uniform(-3.0, 5.0, size=(n_valid, 4))
        self.recording_index = recording_index
        self.recording_uid = f"fake_rec_{recording_index}"
        # channels >= n_valid are absent from the layout -> INVALID positions (common.py:203-214)
        self.mne_info = FakeInfo(names, names[:n_valid], pos)

    def study_name(self):
        return "fake"


class FakeBatch:
    """Has exactly what SimpleConv.forward touches (simpleconv.py:199, common.py:225-233)."""

    def __init__(self, meg, subject_index, recordings):
        self.meg = meg
        self.subject_index = subject_index
        self._recordings = list(recordings)

    def __len__(self):
        return len(self._recordings)


CLIP_CONV = dict(hidden=dict(meg=320), batch_norm=True, depth=10, dilation_period=5, kernel_size=3,
                 skip=True, subject_layers=True, subject_dim=0, complex_out=True, glu=2, glu_context=1,
                 merger=True, initial_linear=270, gelu=True, merger_pos_dim=2048)   # conf/model/clip_conv.yaml:6-22


def clip_conv_kwargs(hidden=320, depth=10, merger_channels=270, initial_linear=270, merger_pos_dim=2048,
                     merger_dropout=0.2):
    kw = dict(CLIP_CONV)
    kw.update(hidden=dict(meg=hidden), depth=depth, merger_channels=merger_channels,
              initial_linear=initial_linear, merger_pos_dim=merger_pos_dim, merger_dropout=merger_dropout)
    return kw


# ----------------------------------------------------------------------------------------------
# bm/norm.py (SURVEY.md 8(f) row 2: BatchScaler._transform + ScaleReject), loaded verbatim
# ----------------------------------------------------------------------------------------------
_norm = None


def load_reference_norm():
    """Returns the verbatim `bm.norm` module.  It imports `dora.log.LogProgress`, `bm.features.{FeaturesBuilder,
    Feature}` and `bm.dataset.SegmentBatch` for type annotations and the (unused here) `fit` loop only; empty
    stand-ins are enough for `RobustScaler` / `StandardScaler` / `BatchScaler._transform` / `ScaleReject`."""
    global _norm
    if _norm is not None:
        return _norm
    load_reference()
    if "dora" not in sys.modules:
        dora = types.ModuleType("dora")
        dora.__path__ = []
        sys.modules["dora"] = dora
    log = types.ModuleType("dora.log")
    log.LogProgress = lambda logger, it, **kw: it
    sys.modules["dora.log"] = log
    feats = types.ModuleType("bm.features")
    feats.FeaturesBuilder = object
    feats.Feature = object
    sys.modules["bm.features"] = feats
    dset = types.ModuleType("bm.dataset")
    dset.SegmentBatch = FakeSegmentBatch
    sys.modules["bm.dataset"] = dset
    spec = importlib.util.spec_from_file_location("bm.norm", REF + "/norm.py")
    m = importlib.util.module_from_spec(spec)
    sys.modules["bm.norm"] = m
    spec.loader.exec_module(m)
    _norm = m
    return m


class FakeSegmentBatch:
    """What BatchScaler._transform / ScaleReject.__call__ touch on a SegmentBatch (norm.py:248-275, 325-341):
    `.meg`, `.features`, `.features_mask`, `.recording_index`, `.replace(**kw)`, boolean-mask `__getitem__`."""

    def __init__(self, meg, features, features_mask, recording_index):
        self.meg, self.features, self.features_mask = meg, features, features_mask
        self.recording_index = recording_index

    def replace(self, **kw):
        d = dict(meg=self.meg, features=self.features, features_mask=self.features_mask,
                 recording_index=self.recording_index)
        d.update(kw)
        return FakeSegmentBatch(**d)

    def __getitem__(self, keep):
        return FakeSegmentBatch(self.meg[keep], self.features[keep], self.features_mask[keep],
                                self.recording_index[keep])

    def __len__(self):
        return len(self.meg)


class FakeFeaturesBuilder(dict):
    """name -> (slice, normalizable) ; stands in for bm.features.FeaturesBuilder (norm.py:160-162, 232, 264)."""

    def __init__(self, spec):
        super().__init__()
        start = 0
        self._slices = {}
        for name, (dim, normalizable) in spec.items():
            self[name] = types.SimpleNamespace(normalizable=normalizable, categorical=False, cardinality=0)
            self._slices[name] = slice(start, start + dim)
            start += dim
        self.dimension = start

    def get_slice(self, name):
        return self._slices[name]
