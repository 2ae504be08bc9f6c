"""Every drop-in family against the UNMODIFIED reference, without a GPU: the constructor signatures, the seeded-init
state_dict digests and the eager graph's outputs on the seeded cases, all against the fixtures
tests/golden/<family>.pt (made by tests/golden/make_family_golden.py; the recipe is tests/golden/parity.py)."""
import functools
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, load_golden, state_digest

sys.path.insert(0, GOLDEN_DIR)
from parity import DROPIN, families, input_digest, weights_digest  # noqa: E402

FAMILIES = families()
golden = functools.lru_cache(maxsize=None)(load_golden)


@pytest.mark.parametrize("family", list(FAMILIES))
def test_signatures_match_reference(family):
    got = FAMILIES[family].signature_fields(DROPIN)
    assert got == {k: golden(family)[k] for k in got}


@pytest.mark.parametrize("family,variant", [
    pytest.param(f, v, id=f if v is None else f"{f}-{v}") for f in FAMILIES for v in FAMILIES[f].init])
def test_seeded_init_matches_reference(family, variant):
    init = golden(family)["init"]
    want = init if variant is None else init[variant]
    sd = FAMILIES[family].init_state(DROPIN, variant)
    assert list(sd) == list(want)                          # names and registration order
    assert state_digest(sd) == want                        # shapes, dtypes and the bytes of every tensor


def _assert_close(got, want, where):
    if isinstance(want, dict):
        assert list(got) == list(want), where
        for k in want:
            _assert_close(got[k], want[k], f"{where}[{k}]")
    elif isinstance(want, torch.Tensor):
        torch.testing.assert_close(got, want, rtol=0, atol=1e-5, msg=lambda m: f"{where}: {m}")
    else:
        assert got == want, where


@pytest.mark.parametrize("family,name", [(f, c) for f in FAMILIES for c in sorted(FAMILIES[f].cases)])
def test_eager_forward_matches_reference(family, name):
    """Weights and input rebuilt from the seeds are the ones the reference ran (their digests match); the drop-in's
    PyTorch graph reproduces every output the reference stored for the case."""
    f = FAMILIES[family]
    case, spec = golden(family)["cases"][name], f.cases[name]
    assert case["spec"] == spec
    m = f.build(spec)
    x = f.input(spec)
    assert weights_digest(m) == case["weights"] and input_digest(x) == case["input"]
    with torch.inference_mode():
        assert m.fused_reason(x.float()) == "input is not on a CUDA device"
        got = f.outputs(m, x, spec)
    for k in got:
        _assert_close(got[k], case[k], k)
