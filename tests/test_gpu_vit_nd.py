"""-m gpu: the N-d patch gather, the rotary q/k kernel and both fused ViTNDs (vit_nd, vit_nd_rotary) on the H100.
Kernels are checked bit for bit against torch; the models against their own fp32 PyTorch graph on the same
bf16-representable weights and inputs, and the rotary model's return_embed output against the reference's
(tests/golden/vit_nd.pt; the logits are checked in test_gpu_family_parity.py)."""
import math
import os
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, load_golden
from oracle.layer_trace import rope_reference
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.vit_nd import PatchifyND, ViTND, ensure_tuple
from vit_pytorch_b200.vit_nd_rotary import ViTND as RotaryViTND
from vit_pytorch_b200.vit_nd_rotary import rope_table

sys.path.insert(0, GOLDEN_DIR)
from parity import weights_digest  # noqa: E402
from vit_nd_spec import FAMILY, VIT_ND_CASES  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
RTOL, ATOL = 1e-2, 1e-3
CLASSES = {"vit_nd": ViTND, "vit_nd_rotary": RotaryViTND}


def stats(got, ref):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    return d.max().item(), (d <= ATOL + RTOL * ref.float().cpu().abs()).float().mean().item()


# ------------------------------------------------------------------------------------------------------ patchify_nd
def nd_shapes():
    for r in range(1, 8):
        for C in (1, 3, 5):
            for pl in (1, 2, 16):
                # leading axes alternate patch 2 / 1 with 2 patches each; the last axis holds 3 patches
                patch = [2 if i % 2 == 0 else 1 for i in range(r - 1)] + [pl]
                shape = [2 * p for p in patch[:-1]] + [3 * pl]
                yield r, C, tuple(shape), tuple(patch)


@pytest.mark.parametrize("r,C,shape,patch", list(nd_shapes()))
def test_patchify_nd_equals_rearrange_bitwise(r, C, shape, patch):
    torch.manual_seed(r * 100 + C * 10 + patch[-1])
    B = 2
    img = torch.randn(B, C, *shape, device=DEV).bfloat16()
    ref = PatchifyND(patch)(img).reshape(-1, C * math.prod(patch))
    K = ref.shape[1]
    ldo = (K + 63) // 64 * 64 + 8                          # K padding, and a stride beyond it
    out = torch.full((ref.shape[0], ldo), float("nan"), device=DEV, dtype=torch.bfloat16)
    _lib.patchify_nd(img, out, patch)
    assert torch.equal(out[:, :K], ref)
    assert torch.equal(out[:, K:], torch.zeros_like(out[:, K:]))


def test_patchify_nd_large_rows_vector_path():
    """224 x 224 x 3, patch 16: 16-byte loads, several patches per CTA."""
    img = torch.randn(3, 3, 224, 224, device=DEV).bfloat16()
    ref = PatchifyND((16, 16))(img).reshape(-1, 768)
    out = torch.empty(ref.shape[0], 768, device=DEV, dtype=torch.bfloat16)
    _lib.patchify_nd(img, out, (16, 16))
    assert torch.equal(out, ref)


# ------------------------------------------------------------------------------------------------------ rope_qk
@pytest.mark.parametrize("dh", [32, 64, 80, 128])
@pytest.mark.parametrize("per_token", [False, True])
def test_rope_qk_bitwise(dh, per_token):
    torch.manual_seed(dh + per_token)
    B, N, H = 3, 77, 3
    T = B * N
    R = T if per_token else N
    qkv = (3 * torch.randn(T, 3 * H * dh, device=DEV)).bfloat16()
    theta = 50 * torch.randn(R, H, dh // 2, device=DEV)
    cs = torch.stack((theta.cos(), theta.sin()), dim=-1).contiguous()
    ref = rope_reference(qkv, cs, R, H, dh)
    v0 = qkv[:, 2 * H * dh:].clone()
    _lib.rope_qk(qkv, cs, R, H, dh)
    assert torch.equal(qkv, ref)
    assert torch.equal(qkv[:, 2 * H * dh:], v0)


def test_rope_table_matches_module_expression():
    """The fused table holds the values GoldenGateRoPENd.forward computes (same expression, same device)."""
    m = RotaryViTND(ndim=2, input_shape=(16, 24), patch_size=(4, 8), num_classes=3, dim=64, depth=1, heads=2,
                    dim_head=32, mlp_dim=64).to(DEV, torch.bfloat16)
    grid = (4, 3)
    cs = m.grid_table(grid, torch.device(DEV))
    q = torch.randn(1, 2, 12, 32, device=DEV).bfloat16()
    pos = torch.stack(torch.meshgrid(torch.arange(4., device=DEV), torch.arange(3., device=DEV), indexing="ij"),
                      -1).reshape(1, 12, 2)
    want = m.rotary_emb(q, pos)                                      # the module's own rotation
    qkv = torch.zeros(12, 3 * 64, device=DEV, dtype=torch.bfloat16)
    qkv[:, :64] = q[0].transpose(0, 1).reshape(12, 64)
    _lib.rope_qk(qkv, cs, 12, 2, 32)
    assert torch.equal(qkv[:, :64], want[0].transpose(0, 1).reshape(12, 64))
    assert torch.equal(cs, rope_table(m.rotary_emb.freqs, pos))


# ------------------------------------------------------------------------------------------------------ models
def rounded_pair(cls, kwargs, seed):
    """(bf16 model on the GPU, fp32 model on the GPU) holding the same bf16-representable weights and buffers."""
    torch.manual_seed(seed)
    m = cls(**kwargs).eval()
    with torch.no_grad():
        for t in list(m.parameters()) + list(m.buffers()):
            t.copy_(t.bfloat16().float())
    ref = cls(**kwargs).eval()
    ref.load_state_dict(m.state_dict())
    return m.to(DEV, torch.bfloat16), ref.to(DEV)


MODEL_CASES = [
    ("vit_nd", dict(ndim=1, input_shape=256, patch_size=8, channels=3), "cls", 2e-2, 0.85),
    ("vit_nd", dict(ndim=2, input_shape=(32, 48), patch_size=(4, 8), channels=3), "mean", 2e-2, 0.85),
    ("vit_nd", dict(ndim=3, input_shape=(4, 16, 16), patch_size=(2, 4, 4), channels=2), "cls", 2e-2, 0.85),
    ("vit_nd", dict(ndim=2, input_shape=(96, 96), patch_size=4, channels=3), "mean", 2e-2, 0.85),  # N = 577
    ("vit_nd_rotary", dict(ndim=1, input_shape=256, patch_size=8, channels=3), None, 2e-2, 0.85),
    ("vit_nd_rotary", dict(ndim=2, input_shape=(32, 48), patch_size=(4, 8), channels=3), None, 2e-2, 0.85),
    ("vit_nd_rotary", dict(ndim=3, input_shape=(4, 16, 16), patch_size=(2, 4, 4), channels=2), None, 2e-2, 0.85),
    ("vit_nd_rotary", dict(ndim=3, input_shape=(8, 48, 32), patch_size=(1, 4, 4), channels=1), None, 2e-2,
     0.85),                                                                                     # N = 768
]
BASE = dict(num_classes=10, dim=128, depth=2, heads=2, dim_head=64, mlp_dim=256)


@pytest.mark.parametrize("kind,geo,pool,max_tol,frac_tol", MODEL_CASES)
def test_fused_model_against_own_fp32_graph(kind, geo, pool, max_tol, frac_tol):
    kwargs = dict(BASE, **geo)
    if pool is not None:
        kwargs["pool"] = pool
    m, ref = rounded_pair(CLASSES[kind], kwargs, seed=7)
    torch.manual_seed(8)
    x = torch.randn(3, geo["channels"], *ensure_tuple(geo["input_shape"], geo["ndim"]), device=DEV).bfloat16()
    _lib.reset_launch_count()
    with torch.inference_mode():
        assert m.fused_reason(x) is None
        out = m(x)
        torch.cuda.synchronize()
        launches = _lib.launch_count()
        want = ref(x.float())
    mx, frac = stats(out, want)
    print(f"{kind} {geo} pool={pool}: max {mx:.5f} within {frac:.4f}, {launches} launches")
    assert launches >= 3 + 5 * kwargs["depth"]
    assert mx < max_tol and frac > frac_tol, (mx, frac)


@pytest.mark.parametrize("name", ["rot_r1", "rot_r2", "rot_r3"])
def test_fused_return_embed_against_reference_goldens(name):
    """The rotary model's return_embed output for the first sample, weights and input rebuilt from the seeds, against
    the reference's (the logits are checked in test_gpu_family_parity.py)."""
    case, spec = load_golden("vit_nd")["cases"][name], VIT_ND_CASES[name]
    m = FAMILY.build(spec)
    assert weights_digest(m) == case["weights"]
    m = m.to(DEV, torch.bfloat16)
    x = FAMILY.input(spec).to(DEV)
    with torch.inference_mode():
        assert m.fused_reason(x) is None
        e = m(x, return_embed=True)[:1]
    assert e.shape == case["embed0_fp32"].shape
    mx, frac = stats(e, case["embed0_fp32"])
    print(f"{name}: max {mx:.5f} within {frac:.4f}")
    assert mx < 6e-2, (mx, frac)


@pytest.mark.parametrize("geo", [dict(ndim=2, input_shape=(32, 48), patch_size=(4, 8)),
                                 dict(ndim=3, input_shape=(8, 48, 32), patch_size=(1, 4, 4))])   # N = 384, 768
def test_one_call_encoder_with_rope_equals_python_loop(geo, monkeypatch):
    m, _ = rounded_pair(RotaryViTND, dict(BASE, channels=3, **geo), seed=9)
    torch.manual_seed(10)
    x = torch.randn(2, 3, *geo["input_shape"], device=DEV).bfloat16()
    outs, counts = {}, {}
    for loop in ("c", "python"):
        monkeypatch.setenv("B200VIT_HOST_LOOP", loop)
        _lib.reset_launch_count()
        with torch.inference_mode():
            outs[loop] = m(x).clone()
        torch.cuda.synchronize()
        counts[loop] = _lib.launch_count()
    assert torch.equal(outs["c"], outs["python"])
    assert counts["c"] == counts["python"]


def test_transformer_called_on_tokens_with_per_token_positions():
    m, ref = rounded_pair(RotaryViTND, dict(BASE, ndim=2, input_shape=(16, 16), patch_size=4, channels=3), seed=11)
    torch.manual_seed(12)
    tok = torch.randn(3, 21, 128, device=DEV).bfloat16()
    pos = 4 * torch.rand(3, 21, 2, device=DEV)                        # arbitrary, different per sequence
    with torch.inference_mode():
        assert m.transformer.fused_reason(tok, pos) is None
        _lib.reset_launch_count()
        out = m.transformer(tok, pos)
        torch.cuda.synchronize()
        assert _lib.launch_count() > 0
        want = ref.transformer(tok.float(), pos)
    mx, frac = stats(out, want)
    assert mx < 6e-2 and frac > 0.85, (mx, frac)


def test_table_follows_the_freqs_buffer():
    """An in-place change of the shared freqs buffer rebuilds the cached table."""
    m, _ = rounded_pair(RotaryViTND, dict(BASE, ndim=2, input_shape=(16, 16), patch_size=4, channels=3), seed=13)
    x = torch.randn(2, 3, 16, 16, device=DEV).bfloat16()
    with torch.inference_mode():
        a = m(x).clone()
    with torch.no_grad():
        m.rotary_emb.freqs.mul_(0.5)
    with torch.inference_mode():
        b = m(x)
        os.environ["B200VIT_DISABLE_FUSED"] = "1"
        try:
            want = m(x)
        finally:
            del os.environ["B200VIT_DISABLE_FUSED"]
    assert not torch.equal(a, b)
    assert stats(b, want)[0] < 3e-2


def test_unsupported_head_width_runs_eager():
    m = RotaryViTND(ndim=2, input_shape=16, patch_size=4, num_classes=3, dim=192, depth=1, heads=2, dim_head=96,
                    mlp_dim=64).eval().to(DEV, torch.bfloat16)
    x = torch.randn(2, 3, 16, 16, device=DEV).bfloat16()
    with torch.inference_mode():
        assert "dim_head=96" in m.fused_reason(x)
        _lib.reset_launch_count()
        out = m(x)
        torch.cuda.synchronize()
    assert _lib.launch_count() == 0 and out.shape == (2, 3)
