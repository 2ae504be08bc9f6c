"""-m gpu: the talking-heads attention kernels (b200vit_attention_headmix_ex with a pre-softmax mix,
b200vit_attention_cls_headmix) and the fused CaiT on the H100.  Every element of the kernels' outputs is checked against
the fp64 references and bounds of oracle/headmix_bounds.py and oracle/attention_fp32_bounds.py; the model's CUDA-graph
replay and fallback rules (its reference parity is in test_gpu_family_parity.py)."""
import sys

import pytest
import torch

from conftest import GOLDEN_DIR
from oracle import attention_fp32_bounds as FB
from oracle import bounds as Bd
from oracle import headmix_bounds as HB
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.cait import CaiT, Transformer

sys.path.insert(0, GOLDEN_DIR)
from cait_spec import CAIT_CASES, FAMILY  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def stats(got, ref, rtol=1e-2, atol=1e-3):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    return d.max().item(), (d <= atol + rtol * ref.float().cpu().abs()).float().mean().item()


# ------------------------------------------------------------------------------------------------ attention_headmix_ex
def headmix_inputs(B, N, H, dh, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkv = torch.randn(B * N, 3 * H * dh, device=DEV, generator=g).bfloat16()
    pre = torch.randn(H, H, device=DEV, generator=g)
    post = torch.randn(H, H, device=DEV, generator=g)
    ln = (1 + 0.2 * torch.randn(H, device=DEV, generator=g), 0.1 * torch.randn(H, device=DEV, generator=g), 1e-5)
    return qkv, pre, post, ln


@pytest.mark.parametrize("mode", ["pre_post", "pre_post_ln"])
@pytest.mark.parametrize("N", [1, 2, 63, 64, 65, 196, 197, 577, 1025])
@pytest.mark.parametrize("dh", [32, 48, 64, 80, 128])
@pytest.mark.parametrize("H", [1, 2, 3, 8, 16])
def test_attention_headmix_pre_against_fp32(H, dh, N, mode):
    if H * dh > 1024:
        pytest.skip("H * dim_head > 1024 is rejected (test_deepvit.py checks the message)")
    B = 2
    qkv, pre, post, ln = headmix_inputs(B, N, H, dh, H * 100000 + dh * 1000 + N + 7)
    ln = ln if mode == "pre_post_ln" else None
    scale = dh ** -0.5
    out = torch.empty(B * N, H * dh, device=DEV, dtype=torch.bfloat16)
    _lib.attention_headmix(qkv, out, B, N, H, dh, scale, post, ln, pre=pre)
    Bd.check(out, *HB.headmix_reference(qkv, B, N, H, dh, scale, pre, post, ln), f"headmix H{H} dh{dh} N{N} {mode}")


def test_one_head_negative_pre_turns_the_softmax_around():
    """heads = 1, pre = -1: softmax(-s), so the output differs from plain attention and matches the reference."""
    B, N, H, dh = 2, 70, 1, 64
    qkv, _, _, _ = headmix_inputs(B, N, H, dh, 13)
    pre, post = torch.full((1, 1), -1.0, device=DEV), torch.ones(1, 1, device=DEV)
    out = torch.empty(B * N, dh, device=DEV, dtype=torch.bfloat16)
    _lib.attention_headmix(qkv, out, B, N, H, dh, 0.125, post, None, pre=pre)
    Bd.check(out, *HB.headmix_reference(qkv, B, N, H, dh, 0.125, pre, post), "pre = -1")
    plain, _ = HB.headmix_reference(qkv, B, N, H, dh, 0.125, -pre, post)
    assert (out.double() - plain).abs().max().item() > 0.1


# ------------------------------------------------------------------------------------------------ attention_cls_headmix
@pytest.mark.parametrize("first", [0, 1])
@pytest.mark.parametrize("n", [0, 1, 15, 16, 196, 576, 4096])
@pytest.mark.parametrize("H,dh", [(1, 64), (3, 48), (4, 32), (8, 48), (16, 64), (6, 80), (8, 128)])
def test_attention_cls_headmix_against_fp32(H, dh, n, first):
    B, I = 3, H * dh
    g = torch.Generator(device=DEV).manual_seed(H * 1000 + dh + n)
    qkv_self = torch.randn(B, 3 * I, device=DEV, generator=g).bfloat16()
    rows = n + first + 2
    ld = 2 * I + 24                                   # strided context rows with unused columns
    ctx = torch.randn(B * rows, ld, device=DEV, generator=g).bfloat16()
    pre, post = torch.randn(H, H, device=DEV, generator=g), torch.randn(H, H, device=DEV, generator=g)
    buf = torch.full((B, I + 16), 3.0, device=DEV, dtype=torch.bfloat16)
    buf[:, :I] = float("nan")
    out = buf[:, :I]
    _lib.attention_cls_headmix(qkv_self, ctx, out, rows, first, n, H, dh, dh ** -0.5, pre, post)
    first_out = out.clone()
    _lib.attention_cls_headmix(qkv_self, ctx, out, rows, first, n, H, dh, dh ** -0.5, pre, post)
    torch.cuda.synchronize()
    assert torch.equal(out, first_out)                # repeat calls are bit-identical
    assert (buf[:, I:] == 3.0).all()                  # columns outside out untouched
    ref, bound = FB.cls_headmix_reference(qkv_self, ctx, rows, first, n, H, dh, dh ** -0.5, pre, post)
    Bd.check(out, ref, bound, f"attention_cls_headmix H{H} dh{dh} n{n} first{first}")


# ------------------------------------------------------------------------------------------------ model
def test_cuda_graph_replay_is_bit_identical():
    from vit_pytorch_b200.graph import GraphedForward
    spec = CAIT_CASES["n576_h8"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    a = FAMILY.input(spec).to(DEV)
    b = torch.randn_like(a.float()).bfloat16()
    with torch.inference_mode():
        ya, yb = m(a).clone(), m(b).clone()
        g = GraphedForward(m, a)
        assert torch.equal(g(b), yb)
        assert torch.equal(g(a), ya)


def test_cuda_graph_refused_with_layer_dropout():
    from vit_pytorch_b200.graph import GraphedForward
    spec = CAIT_CASES["dh32_n64"]
    m = FAMILY.build({**spec, "layer_dropout": 0.1}).to(DEV, torch.bfloat16)
    with pytest.raises(RuntimeError, match="layer_dropout"):
        GraphedForward(m, FAMILY.input(spec).to(DEV))


def test_direct_patch_transformer_call():
    torch.manual_seed(3)
    t = Transformer(128, 2, 4, 48, 256).eval()
    with torch.no_grad():
        for p in t.parameters():
            p.copy_(p.bfloat16().float())
    ref = Transformer(128, 2, 4, 48, 256).eval()
    ref.load_state_dict(t.state_dict())
    t = t.to(DEV, torch.bfloat16)
    x = torch.randn(5, 33, 128, device=DEV).bfloat16()
    with torch.inference_mode():
        assert t.fused_reason(x) is None
        _lib.reset_launch_count()
        out = t(x)
        torch.cuda.synchronize()
        assert _lib.launch_count() > 0
        want = ref(x.float().cpu())
    scale = want.abs().max().item()
    mx, frac = stats(out, want, rtol=1e-2, atol=1e-2 * scale)
    assert mx < 1e-2 * scale and frac > 0.99, (mx, frac, scale)


FALLBACK_KW = dict(image_size=32, patch_size=4, num_classes=3, dim=64, depth=1, cls_depth=1, mlp_dim=64)


def _model(**kw):
    return CaiT(**{**FALLBACK_KW, "heads": 4, "dim_head": 32, **kw}).eval().to(DEV, torch.bfloat16)


def test_fallback_unsupported_head_width():
    m, x = _model(heads=2, dim_head=96), torch.randn(2, 3, 32, 32, device=DEV).bfloat16()
    with torch.inference_mode():
        assert "dim_head=96" in m.fused_reason(x)
        assert m(x).shape == (2, 3)                        # eager, like the reference


def test_fallback_too_many_heads():
    m, x = _model(heads=17, dim_head=32), torch.randn(2, 3, 32, 32, device=DEV).bfloat16()
    with torch.inference_mode():
        assert "heads=17" in m.fused_reason(x)
        assert m(x).shape == (2, 3)


def test_fallback_positional_table_and_divisibility():
    m = _model()
    with torch.inference_mode():
        assert "positional table" in m.fused_reason(torch.randn(2, 3, 36, 36, device=DEV).bfloat16())
        assert "divisible" in m.fused_reason(torch.randn(2, 3, 30, 30, device=DEV).bfloat16())
        assert "channel count" in m.fused_reason(torch.randn(2, 1, 32, 32, device=DEV).bfloat16())
