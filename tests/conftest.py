"""pytest configuration: the `gpu` marker, import path and shared fixtures."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
GOLDEN_NAMES = ["simplevit_tiny", "vit_tiny_cls", "vit_tiny_mean_nonsquare", "vit_tiny_tokens"]
# The unmodified reference package (lucidrains/vit-pytorch 1.23.6).  Only the CPU tests that run the reference's own
# wrapper code need it: they import it from oracle/_ref/, which build() installs (oracle/reference_install.py), or from
# a checkout named by VIT_REFERENCE.  Everything else compares with data stored under tests/golden/.
REFERENCE_DIR = os.environ.get("VIT_REFERENCE", "")
BUILT_REFERENCE_DIR = os.path.join(ROOT, "oracle", "_ref")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90); run with -m gpu")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    return torch.load(os.path.join(GOLDEN_DIR, name + ".pt"), weights_only=False)


@pytest.fixture(params=GOLDEN_NAMES)
def golden(request):
    return load_golden(request.param)


def _reference_dir() -> str:
    for d in (REFERENCE_DIR, BUILT_REFERENCE_DIR):
        if d and os.path.isdir(os.path.join(d, "vit_pytorch")):
            return d
    return ""


def reference_available() -> bool:
    return bool(_reference_dir())


def reference_live():
    """What the reference computed for the seeded cases of tests/golden/make_golden.py (make_reference_live)."""
    return load_golden("reference_live")


def state_digest(sd) -> dict:
    """Per tensor (shape, dtype, sha256 of the bytes), as make_golden.state_digest."""
    import hashlib
    return {k: (tuple(v.shape), str(v.dtype), hashlib.sha256(v.detach().contiguous().cpu().numpy().tobytes()).hexdigest())
            for k, v in sd.items()}


def signature(cls) -> list:
    import inspect
    return [(k, repr(v.default)) for k, v in inspect.signature(cls.__init__).parameters.items() if k != "self"]


def import_reference():
    """Import the unmodified reference package (VIT_REFERENCE, else oracle/_ref)."""
    import importlib
    sys.dont_write_bytecode = True
    d = _reference_dir()
    if d not in sys.path:
        sys.path.insert(0, d)
    return importlib.import_module("vit_pytorch")
