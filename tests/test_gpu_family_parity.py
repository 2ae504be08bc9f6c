"""-m gpu: every drop-in family's fused forward on the H100 against the reference's stored fp32 logits
(tests/golden/<family>.pt) and a second expectation computed here, on the seeded cases of tests/golden/<family>_spec.py.
What differs between families is stated in GPU below."""
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, load_golden
from vit_pytorch_b200 import _lib

sys.path.insert(0, GOLDEN_DIR)
from parity import families, weights_digest  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
FAMILIES = families()
BOTH = ("fold", "exact")                                   # B200VIT_LN_MODE values; None leaves the default

# per family: the bound on max |fused - expected| for both expectations; the LayerNorm modes it runs; the second
# expectation ("eager bf16": the module's own graph in bf16 on the GPU, "own fp32": its own graph in fp32 on the CPU,
# None: the reference's logits only).  Every case of every family runs.
GPU = {
    "pit": dict(tol=3e-2, ln_modes=BOTH, second="eager bf16"),
    "cct": dict(tol=3e-2, ln_modes=BOTH, second="eager bf16"),
    "cait": dict(tol=3e-2, ln_modes=BOTH, second="eager bf16"),
    "deepvit": dict(tol=3e-2, ln_modes=BOTH, second="eager bf16"),
    "xcit": dict(tol=3e-2, ln_modes=BOTH, second="eager bf16"),
    "cross_vit": dict(tol=2e-2, ln_modes=(None,), second="eager bf16"),
    "vit_small": dict(tol=2e-2, ln_modes=(None,), second="eager bf16"),
    "vivit": dict(tol=2e-2, ln_modes=(None,), second="own fp32"),
    "vit_nd": dict(tol=2e-2, ln_modes=(None,), second=None),
}


def stats(got, ref, rtol=1e-2, atol=1e-3):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    return d.max().item(), (d <= atol + rtol * ref.float().cpu().abs()).float().mean().item()


def _run(f, m, x, kwargs, spec):
    with torch.inference_mode():
        if f.before_forward is not None:
            f.before_forward(spec)
        return m(x, **kwargs)


@pytest.mark.parametrize("family,name,ln_mode", [
    pytest.param(family, name, ln_mode, id=f"{family}-{name}-{ln_mode or 'default'}")
    for family, s in GPU.items() for name in sorted(FAMILIES[family].cases) for ln_mode in s["ln_modes"]])
def test_fused_against_reference_goldens(family, name, ln_mode, monkeypatch):
    """Weights rebuilt from the seeds (their digest checked first) and the case's input, for every forward the
    fixture stores (ViViT: every frame-mask kind)."""
    f, s = FAMILIES[family], GPU[family]
    if ln_mode is not None:
        monkeypatch.setenv("B200VIT_LN_MODE", ln_mode)
    case, spec = load_golden(family)["cases"][name], f.cases[name]
    ref = f.build(spec)
    assert weights_digest(ref) == case["weights"]
    x = f.input(spec)
    m = f.build(spec).to(DEV, torch.bfloat16)
    for key, kwargs in f.forwards(spec):
        stored = case["logits_fp32"] if key is None else case["logits_fp32"][key]
        dev_kwargs = {k: v.to(DEV) if isinstance(v, torch.Tensor) else v for k, v in kwargs.items()}
        with torch.inference_mode():
            assert m.fused_reason(x.to(DEV), **dev_kwargs) is None
        _lib.reset_launch_count()
        out = _run(f, m, x.to(DEV), dev_kwargs, spec)
        torch.cuda.synchronize()
        assert _lib.launch_count() > 0 and out.shape == stored.shape
        wants = [("reference fp32", stored)]
        if s["second"] == "eager bf16":
            with monkeypatch.context() as mp:
                mp.setenv("B200VIT_DISABLE_FUSED", "1")
                wants.append(("eager bf16", _run(f, m, x.to(DEV), dev_kwargs, spec)))
        elif s["second"] == "own fp32":
            wants.append(("own fp32", _run(f, ref, x.float(), kwargs, spec)))
        for what, want in wants:
            mx, frac = stats(out, want)
            print(f"{family} {name} {key or ''} {ln_mode or 'default'} vs {what}: max {mx:.5f} within {frac:.4f}")
            assert mx < s["tol"], (key, what, mx, frac)
