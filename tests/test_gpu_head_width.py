"""-m gpu: head widths 32, 80 and 128 through every layer that knows the head width -- the attention kernels (single
pass and key-block, and the tiled kernel test hook 15 forces), the per-head norms, the NaViT attention pooling and whole
models -- against the fp32 oracle or the module's own fp32 graph."""
import pytest
import torch

from oracle import attention_bounds as AB
from oracle import attention_fp32_bounds as FB
from oracle import bounds as Bd
from oracle import row_bounds as RB
from vit_pytorch_b200 import NaViT, SimpleViT, ViT, _lib
from vit_pytorch_b200.na_vit_nested_tensor import NaViT as NestedNaViT
from vit_pytorch_b200.simple_vit_with_qk_norm import SimpleViT as QKNormViT

pytestmark = pytest.mark.gpu
DEV = "cuda"


def run_attention(qkv, B, N, H, dh, hooks):
    """b200vit_attention with test hooks {key: value} set for this call only."""
    L = _lib.lib()
    out = torch.full((B * N, H * dh), float("nan"), device=DEV, dtype=torch.bfloat16)
    try:
        for key, value in hooks.items():
            L.b200vit_debug_set(key, value)
        _lib.attention(qkv, out, B, N, H, dh, dh ** -0.5)
        torch.cuda.synchronize()
    finally:
        L.b200vit_debug_set(15, 0)
    return out


# the kernel each length runs by default, and the tiled kernel at 128 < N <= 256 as well (hook 15)
HOOKS = [{}, {15: 1}]
GRID = [(4, 197, 12), (3, 64, 3), (2, 257, 16), (5, 50, 4), (2, 16, 2), (2, 129, 2), (1, 512, 1), (2, 1, 2),
        # more CTAs than SMs, key counts on and just past a key-block boundary
        (40, 197, 12), (70, 196, 16), (200, 128, 3), (37, 224, 5), (3, 225, 2), (9, 33, 7)]


@pytest.mark.parametrize("dh", [32, 128])
@pytest.mark.parametrize("B,N,H", GRID)
def test_attention_new_widths(B, N, H, dh):
    torch.manual_seed(N + dh)
    qkv = torch.randn(B * N, 3 * H * dh, device=DEV).bfloat16()
    for hooks in HOOKS:
        out = run_attention(qkv, B, N, H, dh, hooks)
        Bd.check(out, *AB.qkv_attention_reference(qkv, [N] * B, H, dh, dh ** -0.5), f"hooks {hooks}")


@pytest.mark.parametrize("dh", [32, 128])
@pytest.mark.parametrize("B,N,H", [(3, 257, 4), (2, 258, 2), (2, 260, 3), (40, 257, 16), (1, 261, 2), (300, 257, 2)])
def test_attention_key_tail_new_widths(B, N, H, dh):
    """N = 256 + (1..5) with the tail keys made the dominant ones."""
    torch.manual_seed(N + dh)
    I = H * dh
    qkv = torch.randn(B * N, 3 * I, device=DEV)
    qkv.view(B, N, 3, I)[:, N - 2:, 1] *= 2.5            # the last keys attract most of the attention
    qkv = qkv.bfloat16()
    out = run_attention(qkv, B, N, H, dh, {})
    Bd.check(out, *AB.qkv_attention_reference(qkv, [N] * B, H, dh, dh ** -0.5), f"key tail N{N} dh{dh}")


@pytest.mark.parametrize("dh", [32, 80, 128])
def test_varlen_attention_new_widths(dh):
    """Packed sequences of mixed lengths (1 token to 1024)."""
    lengths = [197, 1, 130, 577, 64, 1024, 129, 65, 63, 128, 300, 1]
    H = 3
    T = sum(lengths)
    torch.manual_seed(dh)
    qkv = torch.randn(T, 3 * H * dh, device=DEV).bfloat16()
    cu, tp, tiles = _lib.varlen_index(lengths, DEV)
    out = torch.full((T, H * dh), float("nan"), device=DEV, dtype=torch.bfloat16)
    _lib.attention_varlen(qkv, out, cu, tp, tiles, H, dh, dh ** -0.5)
    torch.cuda.synchronize()
    Bd.check(out, *AB.qkv_attention_reference(qkv, lengths, H, dh, dh ** -0.5), f"varlen dh{dh}")


def test_attention_dh128_is_deterministic_and_batch_invariant():
    torch.manual_seed(11)
    B, N, H, dh = 64, 197, 8, 128
    qkv = torch.randn(B * N, 3 * H * dh, device=DEV).bfloat16()
    out = run_attention(qkv, B, N, H, dh, {})
    out2 = run_attention(qkv, B, N, H, dh, {})
    assert torch.equal(out, out2)
    out3 = run_attention(qkv[5 * N: 9 * N].contiguous(), 4, N, H, dh, {})
    assert torch.equal(out3, out[5 * N: 9 * N])


def _layernorm_heads(buf, gamma, nheads, dh, eps):
    rc = _lib.lib().b200vit_layernorm_heads(buf.data_ptr(), buf.stride(0), gamma.data_ptr(), buf.shape[0], nheads, dh,
                                            float(eps), _lib._stream())
    assert rc == 0, _lib.lib().b200vit_last_error()


@pytest.mark.parametrize("dh", [32, 80, 128])
@pytest.mark.parametrize("H", [3, 5, 16])
def test_head_norms_new_widths(dh, H):
    """rmsnorm_heads / layernorm_heads on the k half of a kv buffer and qk_rmsnorm on a packed qkv buffer (head counts
    on both sides of the kernels' unroll switch, not multiples of the heads per step)."""
    torch.manual_seed(dh + H)
    T, I = 301, H * dh
    kv = torch.randn(T, 2 * I, device=DEV).bfloat16()
    g = torch.randn(H, dh, device=DEV)
    k = kv[:, :I].view(T, H, dh)
    buf = kv.clone()
    _lib.rmsnorm_heads(buf, g.reshape(-1).contiguous(), H, dh)
    RB.check(buf[:, :I].view(T, H, dh), *RB.rmsnorm_heads_reference(k, g), "rmsnorm_heads")
    assert torch.equal(buf[:, I:], kv[:, I:])                             # v untouched
    buf = kv.clone()
    _layernorm_heads(buf, g.reshape(-1).contiguous(), H, dh, 1e-5)
    RB.check(buf[:, :I].view(T, H, dh), *RB.layernorm_heads_reference(k, g, 1e-5), "layernorm_heads")
    assert torch.equal(buf[:, I:], kv[:, I:])
    # q / k RMSNorm in place on qkv[T, 3 H dh]
    qkv = torch.randn(T, 3 * I, device=DEV).bfloat16()
    gqk = torch.randn(2, H, dh, device=DEV)
    got = qkv.clone()
    _lib.qk_rmsnorm(got, gqk.reshape(-1).contiguous(), H, dh)
    for s in (0, 1):
        RB.check(got.view(T, 3, H, dh)[:, s], *RB.rmsnorm_heads_reference(qkv.view(T, 3, H, dh)[:, s], gqk[s]), "qk")
    assert torch.equal(got[:, 2 * I:], qkv[:, 2 * I:])


@pytest.mark.parametrize("dh", [32, 80, 128])
@pytest.mark.parametrize("headln", [False, True])
def test_gemm_headnorm_new_widths(dh, headln):
    """QKV GEMM + per-head RMSNorm / LayerNorm (EPI_HEADLN) of the q and k heads, against the norm applied to the
    bf16-rounded GEMM output."""
    torch.manual_seed(dh)
    M, H, K = 700, 3, 256
    I = H * dh
    a = torch.randn(M, K, device=DEV).bfloat16()
    w = (torch.randn(3 * I, K, device=DEV) / K ** 0.5).bfloat16()
    g = torch.randn(2 * H, dh, device=DEV)
    plain = torch.empty(M, 3 * I, device=DEV, dtype=torch.bfloat16)
    _lib.gemm(a, w, out_bf16=plain)
    got = torch.empty_like(plain)
    _lib.gemm_headnorm(a, w, out_bf16=got, head_gamma=g.reshape(-1).contiguous(), norm_heads=2 * H, dh=dh,
                       head_layernorm_eps=1e-5 if headln else None)
    torch.cuda.synchronize()
    x = plain[:, :2 * I].view(M, 2 * H, dh)
    ref, bound = RB.layernorm_heads_reference(x, g, 1e-5) if headln else RB.rmsnorm_heads_reference(x, g)
    RB.check(got[:, :2 * I].view(M, 2 * H, dh), ref, bound, "gemm_headnorm")
    assert torch.equal(got[:, 2 * I:], plain[:, 2 * I:])                  # v columns untouched


@pytest.mark.parametrize("dh", [32, 80, 128])
@pytest.mark.parametrize("H", [1, 3, 16])
def test_attn_pool_new_widths(dh, H):
    torch.manual_seed(dh + H)
    lengths = [100, 1, 199, 1030, 33]
    T, I = sum(lengths), H * dh
    kv = torch.randn(T, 2 * I, device=DEV).bfloat16()
    qn = torch.randn(I, device=DEV) * dh ** -0.5
    cu, _, _ = _lib.varlen_index(lengths, DEV)
    out = torch.full((len(lengths), I), float("nan"), device=DEV, dtype=torch.bfloat16)
    _lib.attn_pool(kv, qn, cu, out, H, dh)
    torch.cuda.synchronize()
    ref, bound = FB.navit_pool_reference(kv, qn, lengths, H, dh)
    Bd.check(out, ref, bound, f"attn_pool H{H} dh{dh}")


# ---------------------------------------------------------------------------------------------------- whole models
def _check_floor(m, fp32_call, bf16_call):
    """Fused bf16 forward no worse than the module's own bf16 eager graph, both against its fp32 eager graph."""
    m = m.eval().to(DEV)
    with torch.inference_mode():
        ref = fp32_call(m).float().cpu()
    mb = m.bfloat16()           # outside inference mode: buffers stay ordinary tensors with version counters
    with torch.inference_mode():
        floor = bf16_call(mb, eager=True).float().cpu()
        _lib.reset_launch_count()
        out = bf16_call(mb, eager=False).float().cpu()
        torch.cuda.synchronize()
    assert _lib.launch_count() > 0
    d, f = (out - ref).abs(), (floor - ref).abs()
    print(f"fused max {d.max():.4f} mean {d.mean():.5f}; bf16 graph max {f.max():.4f} mean {f.mean():.5f}")
    assert torch.isfinite(out).all()
    assert d.mean() <= f.mean() * 1.05 + 1e-4 and d.max() <= f.max() * 1.5 + 1e-3


def _image_model_calls(img):
    def fp32(m):
        return m.forward_eager(img.to(DEV, torch.float32))

    def bf16(m, eager):
        x = img.to(DEV, torch.bfloat16)
        if eager:
            return m.forward_eager(x)
        assert m.fused_reason(x) is None, m.fused_reason(x)
        return m(x)
    return fp32, bf16


IMAGE_MODELS = {
    "vit_cls": lambda dh: ViT(image_size=64, patch_size=8, num_classes=10, dim=2 * dh, depth=2, heads=3, mlp_dim=256,
                              dim_head=dh),
    "vit_mean": lambda dh: ViT(image_size=64, patch_size=8, num_classes=10, dim=128, depth=2, heads=2, mlp_dim=256,
                               dim_head=dh, pool="mean"),
    "simple_vit": lambda dh: SimpleViT(image_size=64, patch_size=8, num_classes=10, dim=128, depth=2, heads=3,
                                       mlp_dim=256, dim_head=dh),
    "qk_norm": lambda dh: QKNormViT(image_size=64, patch_size=8, num_classes=10, dim=128, depth=2, heads=2, mlp_dim=256,
                                    dim_head=dh),
    # N = 1025 > 512: key-block attention inside the encoder
    "vit_448_p14": lambda dh: ViT(image_size=448, patch_size=14, num_classes=10, dim=256, depth=2, heads=2, mlp_dim=512,
                                  dim_head=dh),
}


@pytest.mark.parametrize("name,dh", [(n, dh) for n in IMAGE_MODELS for dh in (32, 80, 128)
                                     if not (n == "vit_448_p14" and dh == 32)])
def test_image_models_new_widths(name, dh):
    torch.manual_seed(dh)
    m = IMAGE_MODELS[name](dh)
    size = 448 if name == "vit_448_p14" else 64
    img = torch.randn(2 if size == 448 else 4, 3, size, size, generator=torch.Generator().manual_seed(1))
    _check_floor(m, *_image_model_calls(img))


def test_identity_out_projection_dh128():
    """heads = 1 and dim_head == dim: to_out is nn.Identity (reference vit.py:34,46-49)."""
    torch.manual_seed(3)
    m = ViT(image_size=64, patch_size=8, num_classes=10, dim=128, depth=2, heads=1, mlp_dim=256, dim_head=128)
    assert isinstance(m.transformer.layers[0][0].to_out, torch.nn.Identity)
    img = torch.randn(4, 3, 64, 64, generator=torch.Generator().manual_seed(2))
    _check_floor(m, *_image_model_calls(img))


NAVIT_SIZES = [(384, 384), (16, 16), (64, 128), (224, 160), (32, 32)]      # 576 tokens down to 1


def _navit_calls(imgs):
    def fp32(m):
        return m.forward_eager([im.to(DEV, torch.float32) for im in imgs])

    def bf16(m, eager):
        xs = [im.to(DEV, torch.bfloat16) for im in imgs]
        if eager:
            return m.forward_eager(xs)
        assert m.fused_reason(xs) is None, m.fused_reason(xs)
        return m(xs)
    return fp32, bf16


@pytest.mark.parametrize("dh", [32, 80, 128])
def test_navit_new_widths(dh):
    torch.manual_seed(dh)
    m = NaViT(image_size=384, patch_size=16, num_classes=10, dim=192, depth=2, heads=3, mlp_dim=384, dim_head=dh)
    g = torch.Generator().manual_seed(4)
    imgs = [torch.randn(3, h, w, generator=g) for h, w in NAVIT_SIZES]
    _check_floor(m, *_navit_calls(imgs))


@pytest.mark.parametrize("dh", [32, 80, 128])
@pytest.mark.parametrize("qk", [False, True])
def test_nested_navit_new_widths(dh, qk):
    torch.manual_seed(dh + qk)
    m = NestedNaViT(image_size=384, patch_size=16, num_classes=10, dim=192, depth=2, heads=3, mlp_dim=384,
                    dim_head=dh, qk_rmsnorm=qk)
    g = torch.Generator().manual_seed(5)
    imgs = [torch.randn(3, h, w, generator=g) for h, w in NAVIT_SIZES]
    _check_floor(m, *_navit_calls(imgs))


# ---------------------------------------------------------------------------------- one-call C encoder vs Python loop
ENCODER_CASES = {
    "dh32": (lambda: ViT(image_size=64, patch_size=8, num_classes=5, dim=128, depth=2, heads=4, mlp_dim=256,
                         dim_head=32), 64),
    "dh128": (lambda: ViT(image_size=64, patch_size=8, num_classes=5, dim=256, depth=2, heads=2, mlp_dim=512,
                          dim_head=128), 64),
    "dh80_qk_norm": (lambda: QKNormViT(image_size=64, patch_size=8, num_classes=7, dim=160, depth=2, heads=2,
                                       mlp_dim=320, dim_head=80), 64),
    "dh80_long": (lambda: ViT(image_size=448, patch_size=14, num_classes=5, dim=160, depth=2, heads=2, mlp_dim=320,
                              dim_head=80), 448),
}


@pytest.mark.parametrize("case", list(ENCODER_CASES))
def test_one_call_encoder_equals_the_per_kernel_host_loop_new_widths(case, monkeypatch):
    torch.manual_seed(0)
    make, size = ENCODER_CASES[case]
    m = make().eval().to(DEV, torch.bfloat16)
    x = torch.randn(2 if size == 448 else 3, 3, size, size, device=DEV).bfloat16()
    outs, counts = {}, {}
    for loop in ("c", "python"):
        monkeypatch.setenv("B200VIT_HOST_LOOP", loop)
        _lib.reset_launch_count()
        with torch.inference_mode():
            assert m.fused_reason(x) is None, m.fused_reason(x)
            outs[loop] = m(x).clone()
        torch.cuda.synchronize()
        counts[loop] = _lib.launch_count()
    assert torch.equal(outs["c"], outs["python"])
    assert counts["c"] == counts["python"] > 0
