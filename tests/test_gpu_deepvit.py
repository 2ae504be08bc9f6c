"""-m gpu: the head-mixing attention kernel (b200vit_attention_headmix) and the fused DeepViT on the H100.  Every
element of the kernel's output is checked against the fp64 reference and bound of oracle/headmix_bounds.py; the model at batch one, its CUDA-graph replay
and fallback rules (its reference parity is in test_gpu_family_parity.py)."""
import sys

import pytest
import torch

from conftest import GOLDEN_DIR
from oracle import bounds as Bd
from oracle import headmix_bounds as HB
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.deepvit import DeepViT, Transformer

sys.path.insert(0, GOLDEN_DIR)
from deepvit_spec import DEEPVIT_CASES, FAMILY  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def stats(got, ref, rtol=1e-2, atol=1e-3):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    return d.max().item(), (d <= atol + rtol * ref.float().cpu().abs()).float().mean().item()


# ------------------------------------------------------------------------------------------------ attention_headmix
def headmix_inputs(B, N, H, dh, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkv = torch.randn(B * N, 3 * H * dh, device=DEV, generator=g).bfloat16()
    post = torch.randn(H, H, device=DEV, generator=g)
    ln = (1 + 0.2 * torch.randn(H, device=DEV, generator=g), 0.1 * torch.randn(H, device=DEV, generator=g), 1e-5)
    return qkv, post, ln


@pytest.mark.parametrize("mode", ["post", "post_ln"])
@pytest.mark.parametrize("N", [1, 2, 63, 64, 65, 196, 197, 577, 1025])
@pytest.mark.parametrize("dh", [32, 48, 64, 80, 128])
@pytest.mark.parametrize("H", [1, 2, 3, 8, 16])
def test_attention_headmix_against_fp32(H, dh, N, mode):
    if H * dh > 1024:
        pytest.skip("H * dim_head > 1024 is rejected (test_deepvit.py checks the message)")
    B = 2
    qkv, post, ln = headmix_inputs(B, N, H, dh, H * 100000 + dh * 1000 + N)
    ln = ln if mode == "post_ln" else None
    scale = dh ** -0.5
    out = torch.empty(B * N, H * dh, device=DEV, dtype=torch.bfloat16)
    _lib.attention_headmix(qkv, out, B, N, H, dh, scale, post, ln)
    Bd.check(out, *HB.headmix_reference(qkv, B, N, H, dh, scale, None, post, ln), f"headmix H{H} dh{dh} N{N} {mode}")


@pytest.mark.parametrize("H,dh,N", [(16, 64, 197), (3, 48, 65), (8, 128, 577)])
def test_attention_headmix_leaves_other_rows_and_repeats_bit_identically(H, dh, N):
    B = 3
    qkv, post, ln = headmix_inputs(B, N, H, dh, 7)
    buf = torch.full((B * N + 64, H * dh), 3.0, device=DEV, dtype=torch.bfloat16)
    out = buf[:B * N]
    _lib.attention_headmix(qkv, out, B, N, H, dh, dh ** -0.5, post, ln)
    first = out.clone()
    _lib.attention_headmix(qkv, out, B, N, H, dh, dh ** -0.5, post, ln)
    torch.cuda.synchronize()
    assert torch.equal(out, first)
    assert (buf[B * N:] == 3.0).all()


def test_one_head_layernorm_gives_beta():
    """heads = 1: the LayerNorm over one head leaves beta at every (i, j), so each query's output is beta * sum_j v_j."""
    B, N, H, dh = 2, 70, 1, 64
    qkv, post, _ = headmix_inputs(B, N, H, dh, 11)
    ln = (torch.tensor([1.3], device=DEV), torch.tensor([0.25], device=DEV), 1e-5)
    out = torch.empty(B * N, dh, device=DEV, dtype=torch.bfloat16)
    _lib.attention_headmix(qkv, out, B, N, H, dh, 0.125, post, ln)
    v = qkv.double().view(B, N, 3, dh)[:, :, 2]
    want = (0.25 * v.sum(1, keepdim=True)).expand(B, N, dh).reshape(B * N, dh)
    ref, bound = HB.headmix_reference(qkv, B, N, H, dh, 0.125, None, post, ln)
    assert torch.allclose(ref, want, rtol=1e-12, atol=1e-12)
    Bd.check(out, ref, bound, "one head")


# ------------------------------------------------------------------------------------------------ model
def _eager_bf16(m, x, monkeypatch):
    """The module's own PyTorch graph in bf16 (every submodule, the Transformer included)."""
    with monkeypatch.context() as mp:
        mp.setenv("B200VIT_DISABLE_FUSED", "1")
        with torch.inference_mode():
            return m(x)


def test_batch_one(monkeypatch):
    spec = DEEPVIT_CASES["dh48_n197"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    x = FAMILY.input(spec).to(DEV)
    with torch.inference_mode():
        both = m(x)
        one = m(x[1:2])
    eager = _eager_bf16(m, x[1:2], monkeypatch)
    assert stats(one, both[1:2])[0] < 1e-2
    assert stats(one, eager)[0] < 3e-2


def test_cuda_graph_replay_is_bit_identical():
    from vit_pytorch_b200.graph import GraphedForward
    spec = DEEPVIT_CASES["n577_h8"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    a = FAMILY.input(spec).to(DEV)
    b = torch.randn_like(a.float()).bfloat16()
    with torch.inference_mode():
        ya, yb = m(a).clone(), m(b).clone()
        g = GraphedForward(m, a)
        assert torch.equal(g(b), yb)
        assert torch.equal(g(a), ya)


def test_transformer_hook_keeps_the_fused_path():
    """A hook on .transformer (the Extractor pattern) sees the encoder output while the blocks still run fused."""
    spec = DEEPVIT_CASES["dh32_n65"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    x = FAMILY.input(spec).to(DEV)
    seen = []
    h = m.transformer.register_forward_hook(lambda mod, i, o: seen.append(o.shape))
    with torch.inference_mode():
        assert m.fused_reason(x) is None
        _lib.reset_launch_count()
        out = m(x)
        torch.cuda.synchronize()
        assert _lib.launch_count() > 0
        h.remove()
        plain = m(x)
    assert seen == [(2, 65, 64)]
    assert stats(out, plain)[0] < 1e-2


def test_direct_transformer_call():
    torch.manual_seed(3)
    t = Transformer(128, 2, 4, 32, 256).eval()
    with torch.no_grad():
        for p in t.parameters():
            p.copy_(p.bfloat16().float())
    ref = Transformer(128, 2, 4, 32, 256).eval()
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
    # re-attention weights are O(1) for every key after the LayerNorm over heads, so the stream grows to tens: judge
    # the bf16 output (one ulp at 16..32 is 0.125) against the largest value
    scale = want.abs().max().item()
    mx, frac = stats(out, want, rtol=1e-2, atol=1e-2 * scale)
    assert mx < 1e-2 * scale and frac > 0.99, (mx, frac, scale)


FALLBACK_KW = dict(image_size=32, patch_size=4, num_classes=3, dim=64, depth=1, mlp_dim=64)


def _img(channels=3, side=32):
    return torch.randn(2, channels, side, side, device=DEV).bfloat16()


def _model(**kw):
    return DeepViT(**{**FALLBACK_KW, "heads": 4, "dim_head": 32, **kw}).eval().to(DEV, torch.bfloat16)


def test_fallback_unsupported_head_width():
    m, x = _model(heads=2, dim_head=96), _img()
    with torch.inference_mode():
        assert "dim_head=96" in m.fused_reason(x)
        assert m(x).shape == (2, 3)                        # eager, like the reference


def test_fallback_too_many_heads():
    m, x = _model(heads=17, dim_head=32), _img()
    with torch.inference_mode():
        assert "heads=17" in m.fused_reason(x)
        assert m(x).shape == (2, 3)


def test_fallback_heads_times_width_over_limit():
    m, x = _model(heads=16, dim_head=80), _img()
    with torch.inference_mode():
        assert "heads * dim_head <= 1024" in m.fused_reason(x)


def test_fallback_dropout_in_training():
    m, x = _model(dropout=0.1), _img()
    with torch.inference_mode():
        assert m.train().fused_reason(x) == "dropout is active"
        assert m.eval().fused_reason(x) is None


def test_fallback_channel_count():
    m = _model()
    with torch.inference_mode():
        assert "channel count" in m.fused_reason(_img(channels=1))


def test_fallback_positional_table_overflow():
    m = _model()
    with torch.inference_mode():
        assert "positional table" in m.fused_reason(_img(side=36))


def test_fallback_inner_hooks():
    m, x = _model(), _img()
    h = m.transformer.layers[0][0].reattn_norm.register_forward_hook(lambda *a: None)
    with torch.inference_mode():
        assert "hooks" in m.fused_reason(x)
    h.remove()
    with torch.inference_mode():
        assert m.fused_reason(x) is None


def test_fallback_autograd():
    m, x = _model(), _img()
    assert "autograd" in m.fused_reason(x)
    with torch.inference_mode():
        assert m.fused_reason(x) is None
