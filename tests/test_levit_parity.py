"""LeViT against the UNMODIFIED reference, without a GPU: the checks of test_family_parity.py (constructor signature,
seeded-init state_dict digest, the eager graph's outputs on the seeded cases) on the family record of
tests/golden/levit_spec.py and the fixture tests/golden/levit.pt (made by make_levit_golden.py), plus the distill-head
case, whose (out, distill) tuple the fixture stores under "distill"."""
import sys

import pytest
import torch

import test_family_parity as T
from conftest import GOLDEN_DIR, load_golden

sys.path.insert(0, GOLDEN_DIR)
from levit_spec import DISTILL, FAMILY  # noqa: E402
from parity import input_digest, weights_digest  # noqa: E402


@pytest.fixture(autouse=True)
def family(monkeypatch):
    monkeypatch.setitem(T.FAMILIES, FAMILY.name, FAMILY)


def test_signatures_match_reference():
    T.test_signatures_match_reference(FAMILY.name)


def test_seeded_init_matches_reference():
    T.test_seeded_init_matches_reference(FAMILY.name, None)


@pytest.mark.parametrize("name", sorted(FAMILY.cases))
def test_eager_forward_matches_reference(name):
    T.test_eager_forward_matches_reference(FAMILY.name, name)


def test_distill_head_returns_the_reference_tuple():
    case = load_golden("levit")["distill"]
    assert case["spec"] == DISTILL
    model, x = FAMILY.build(DISTILL), FAMILY.input(DISTILL)
    assert weights_digest(model) == case["weights"] and input_digest(x) == case["input"]
    with torch.inference_mode():
        got = model(x.float())
    assert isinstance(got, tuple) and len(got) == 2
    for g, want in zip(got, (case["out_fp32"], case["distill_fp32"])):
        assert g.shape == want.shape
        assert torch.allclose(g, want, atol=1e-4, rtol=1e-4), (g - want).abs().max()
