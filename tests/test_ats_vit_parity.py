"""Adaptive Token Sampling ViT against the UNMODIFIED reference, without a GPU: the checks of test_family_parity.py
(constructor signature, seeded-init state_dict digest, the eager graph's outputs on the seeded cases: logits, the
token ids, every sampling layer's uniforms and padded lengths) on the family record of tests/golden/ats_vit_spec.py and
the fixture tests/golden/ats_vit.pt (made by make_ats_vit_golden.py)."""
import sys

import pytest

import test_family_parity as T
from conftest import GOLDEN_DIR

sys.path.insert(0, GOLDEN_DIR)
from ats_vit_spec import FAMILY  # noqa: E402


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
