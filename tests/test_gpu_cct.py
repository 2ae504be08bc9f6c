"""-m gpu: the convolutional tokenizer's kernels (b200vit_conv_im2col_nchw / _nhwc, b200vit_relu_maxpool), the
sequence-pooling kernel (b200vit_seq_pool), the post-norm encoder layer and the fused CCT on the H100.  The im2col
and the pool are checked bit for bit against F.unfold and F.max_pool2d; the sequence pooling and the post-norm layer
against fp64 references; the model's CUDA-graph replay and weight updates (its reference parity is in
test_gpu_family_parity.py)."""
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN_DIR
from vit_pytorch_b200 import _lib, cct as cct_mod
from vit_pytorch_b200.cct import CCT, TransformerClassifier

sys.path.insert(0, GOLDEN_DIR)
from cct_spec import CCT_CASES, FAMILY  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
U32 = 2.0 ** -24


def stats(got, ref, rtol=1e-2, atol=1e-3):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    return d.max().item(), (d <= atol + rtol * ref.float().cpu().abs()).float().mean().item()


def out_size(n, k, s, p):
    return (n + 2 * p - k) // s + 1


def poisoned(rows, ld, extra=4096, dtype=torch.bfloat16):
    """A [rows, ld] view at the head of a NaN-filled flat buffer `extra` elements longer."""
    big = torch.full((rows * ld + extra,), float("nan"), device=DEV, dtype=dtype)
    return big, big[:rows * ld].view(rows, ld)


# ------------------------------------------------------------------------------------------------ im2col
IM2COL = [(k, s, p) for k in (1, 3, 7) for s in (1, 2, 3) for p in (0, 1, 3) if p < k]


@pytest.mark.parametrize("k,s,p", IM2COL)
@pytest.mark.parametrize("C", [3, 64])
@pytest.mark.parametrize("hw", [(17, 17), (16, 22)])
def test_conv_im2col_nchw_is_bit_exact(hw, C, k, s, p):
    H, W = hw
    torch.manual_seed(k * 100 + s * 10 + p + C)
    img = torch.randn(2, C, H, W, device=DEV).bfloat16()
    K = C * k * k
    ldo = (K + 7) // 8 * 8 + (8 if C == 3 else 0)                      # K padding of a few columns, or none
    rows = 2 * out_size(H, k, s, p) * out_size(W, k, s, p)
    big, out = poisoned(rows, ldo)
    _lib.conv_im2col_nchw(img, out, k, s, p)
    want = F.unfold(img.float(), k, padding=p, stride=s).transpose(1, 2).reshape(-1, K).bfloat16()
    assert torch.equal(out[:, :K], want)
    assert (out[:, K:] == 0).all()                                        # the K padding is zeros, not NaN
    assert torch.isnan(big[out.numel():].float()).all()                  # nothing past the output is written


@pytest.mark.parametrize("k,s,p", IM2COL)
@pytest.mark.parametrize("C", [8, 64])
@pytest.mark.parametrize("hw", [(17, 17), (16, 22)])
def test_conv_im2col_nhwc_is_bit_exact(hw, C, k, s, p):
    H, W = hw
    B = 2
    torch.manual_seed(k * 100 + s * 10 + p + C + 1)
    img = torch.randn(B, C, H, W, device=DEV).bfloat16()
    x = img.permute(0, 2, 3, 1).reshape(B * H * W, C).contiguous()
    K = C * k * k
    ldo = K + 16
    oh, ow = out_size(H, k, s, p), out_size(W, k, s, p)
    big, out = poisoned(B * oh * ow, ldo)
    _lib.conv_im2col_nhwc(x, out, B, H, W, k, s, p)
    # (ky, kx, c) order: F.unfold's (c, ky, kx) columns with the channel moved last
    want = F.unfold(img.float(), k, padding=p, stride=s).reshape(B, C, k * k, oh * ow).permute(0, 3, 2, 1)
    assert torch.equal(out[:, :K], want.reshape(-1, K).bfloat16())
    assert (out[:, K:] == 0).all()
    assert torch.isnan(big[out.numel():].float()).all()


def test_conv_im2col_readme_shapes_and_repeat_calls():
    """The README's first (3 -> 64 at 224 x 448, k7 s2 p3) and second (64 -> 384 at 56 x 112) gathers."""
    torch.manual_seed(0)
    img = torch.randn(2, 3, 224, 448, device=DEV).bfloat16()
    out = torch.empty(2 * 112 * 224, 152, device=DEV, dtype=torch.bfloat16)
    _lib.conv_im2col_nchw(img, out, 7, 2, 3)
    want = F.unfold(img.float(), 7, padding=3, stride=2).transpose(1, 2).reshape(-1, 147).bfloat16()
    assert torch.equal(out[:, :147], want) and (out[:, 147:] == 0).all()
    first = out.clone()
    _lib.conv_im2col_nchw(img, out, 7, 2, 3)
    assert torch.equal(out, first)
    x = torch.randn(2 * 56 * 112, 64, device=DEV).bfloat16()
    out2 = torch.empty(2 * 28 * 56, 3136, device=DEV, dtype=torch.bfloat16)
    _lib.conv_im2col_nhwc(x, out2, 2, 56, 112, 7, 2, 3)
    im = x.view(2, 56, 112, 64).permute(0, 3, 1, 2).float()
    want2 = F.unfold(im, 7, padding=3, stride=2).reshape(2, 64, 49, -1).permute(0, 3, 2, 1).reshape(-1, 3136)
    assert torch.equal(out2, want2.bfloat16())


# ------------------------------------------------------------------------------------------------ relu_maxpool
def _special(y):
    """NaN, +-Inf and an all-negative region planted into channels-last y [B*H*W, C]."""
    y = y.clone()
    y[3, 0] = float("nan")
    y[10, 5] = float("inf")
    y[11, 6] = float("-inf")
    y[20:40, 8:16] = -y[20:40, 8:16].abs() - 0.5                          # every window there: all negative
    y[50, 9] = float("nan")
    y[50, 10] = float("-inf")
    return y


def _pool_ref(y, B, H, W, pk, ps, pp):
    C = y.shape[1]
    img = y.view(B, H, W, C).permute(0, 3, 1, 2)
    ref = F.max_pool2d(F.relu(img), pk, ps, pp)                           # on bf16, as the reference's tokenizer
    return ref.permute(0, 2, 3, 1).reshape(-1, C)


def _same(got, want):
    nan = torch.isnan(want.float())
    return torch.equal(torch.isnan(got.float()), nan) and torch.equal(got.float()[~nan], want.float()[~nan])


@pytest.mark.parametrize("pool", [(3, 2, 1), (2, 2, 0), (3, 1, 1), (1, 1, 0), (5, 3, 2), (4, 2, 1)])
@pytest.mark.parametrize("hw", [(16, 16), (15, 21)])
@pytest.mark.parametrize("f32", [False, True])
def test_relu_maxpool_is_bit_exact(f32, hw, pool):
    H, W = hw
    pk, ps, pp = pool
    B, C = 2, 64
    torch.manual_seed(H + pk * 7 + ps)
    y = _special(torch.randn(B * H * W, C, device=DEV).bfloat16())
    oh, ow = out_size(H, pk, ps, pp), out_size(W, pk, ps, pp)
    ld = C + 8
    big, out = poisoned(B * oh * ow, ld, dtype=torch.float32 if f32 else torch.bfloat16)
    view = out[:, :C]
    _lib.relu_maxpool(y, B, H, W, pk, ps, pp, **({"out_f32": view} if f32 else {"out_bf16": view}))
    want = _pool_ref(y, B, H, W, pk, ps, pp)
    assert _same(view, want.float() if f32 else want)
    assert torch.isnan(out[:, C:].float()).all() and torch.isnan(big[out.numel():].float()).all()
    assert torch.isnan(want.float()).any() and torch.isinf(want.float()).any()   # the special values reach the output


# ------------------------------------------------------------------------------------------------ seq_pool
def seq_pool_reference(x, B, n, g, be, w, bias, eps):
    """fp64 (ref, bound).  The kernel's fp32 error: the LayerNorm'd tokens within e_y = (D/4 + 40) u (|xhat g| +
    |beta| + |g| |mean| rstd) (the tree sums of mean and variance, rsqrt, two fmas); each logit within
    sum_c |w_c| e_y + (D/4 + 8) u sum_c |y_c w_c| + u |z|; so every probability within a relative 2 max_t e_z plus
    the exponentials and the running sum, (n + 64) u; the weighted sum adds (n + 32) u per term; then the bf16
    rounding of the result, 2^-8 (|ref| + E)."""
    D = x.shape[1]
    xd = x.double().view(B, n, D)
    mean = xd.mean(-1, keepdim=True)
    var = ((xd - mean) ** 2).mean(-1, keepdim=True)
    rstd = (var + eps).rsqrt()
    xhat = (xd - mean) * rstd
    gd, bd, wd = g.double(), be.double(), w.double()
    y = xhat * gd + bd
    z = y @ wd + bias.double()
    p = z.softmax(-1)
    ref = torch.einsum('bn,bnd->bd', p, y)
    u = U32
    ey = (D / 4 + 40) * u * ((xhat * gd).abs() + bd.abs() + gd.abs() * mean.abs() * rstd)
    ez = ey @ wd.abs() + (D / 4 + 8) * u * ((y * wd).abs().sum(-1)) + u * z.abs()
    rel_p = 2 * ez.amax(-1, keepdim=True) + (n + 64) * u
    E = torch.einsum('bn,bnd->bd', p, (rel_p[..., None] + (n + 32) * u) * y.abs() + ey)
    return ref, 2.0 ** -8 * (ref.abs() + E) + E + 1e-30


def _seq_inputs(B, n, D, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B * n, D, device=DEV, generator=g) * 2 + 0.5
    gamma = 1 + 0.2 * torch.randn(D, device=DEV, generator=g)
    beta = 0.1 * torch.randn(D, device=DEV, generator=g)
    w = 0.3 * torch.randn(D, device=DEV, generator=g)
    bias = 0.1 * torch.randn(1, device=DEV, generator=g)
    return x, gamma, beta, w, bias


@pytest.mark.parametrize("n", [1, 7, 256, 3136, 12544])
@pytest.mark.parametrize("B", [1, 64])
@pytest.mark.parametrize("D", [256, 384])
def test_seq_pool_against_fp64(D, B, n):
    x, g, be, w, bias = _seq_inputs(B, n, D, n * 10 + B + D)
    big, out = poisoned(B, D + 8)
    view = out[:, :D]
    _lib.seq_pool(x, B, n, g, be, w, bias, view)
    ref, bound = seq_pool_reference(x, B, n, g, be, w, bias, 1e-5)
    err = (view.double() - ref).abs()
    assert (err <= bound).all(), (err / bound).max().item()
    assert torch.isnan(out[:, D:].float()).all() and torch.isnan(big[out.numel():].float()).all()


def test_seq_pool_keeps_each_image_to_itself_and_repeats_bits():
    B, n, D = 3, 3136, 384                                  # several CTAs per image
    x, g, be, w, bias = _seq_inputs(B, n, D, 7)
    out = torch.empty(B, D, device=DEV, dtype=torch.bfloat16)
    _lib.seq_pool(x, B, n, g, be, w, bias, out)
    first = out.clone()
    for _ in range(2):
        _lib.seq_pool(x, B, n, g, be, w, bias, out)
        assert torch.equal(out, first)
    x[n + 1000, 17] = float("nan")                          # one element of image 1
    x[n + 2000, 3] = float("inf")
    _lib.seq_pool(x, B, n, g, be, w, bias, out)
    assert torch.equal(out[0], first[0]) and torch.equal(out[2], first[2])
    assert torch.isnan(out[1].float()).all()


# ------------------------------------------------------------------------------------------------ post-norm layer
@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
def test_post_norm_layer_against_fp64(ln_mode, monkeypatch):
    monkeypatch.setenv("B200VIT_LN_MODE", ln_mode)
    torch.manual_seed(11)
    cl = TransformerClassifier(embedding_dim=256, num_layers=1, num_heads=4, mlp_ratio=2, num_classes=3,
                               positional_embedding="none").eval()
    with torch.no_grad():
        for name, p in cl.named_parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
            p.copy_(p.bfloat16().float())
    ref_blk = cl.blocks[0].double()
    B, N = 4, 197
    x = torch.randn(B, N, 256)
    with torch.no_grad():
        want = ref_blk(x.bfloat16().double())
    cl = cl.float().to(DEV, torch.bfloat16)
    xs = x.bfloat16().float().reshape(B * N, 256).to(DEV).contiguous()
    with torch.inference_mode():
        cl.engine().run_blocks(xs, B, N)
    got = xs.view(B, N, 256).double().cpu()
    scale = want.abs().max().item()
    mx, frac = stats(got, want, rtol=1e-2, atol=1e-2 * scale)
    print(f"post-norm {ln_mode}: max {mx:.4f} (scale {scale:.2f}) within {frac:.4f}")
    assert mx < 2e-2 * scale and frac > 0.99, (mx, frac, scale)


# ------------------------------------------------------------------------------------------------ model
README_CCT = dict(img_size=(224, 448), embedding_dim=384, n_conv_layers=2, kernel_size=7, stride=2, padding=3,
                  pooling_kernel_size=3, pooling_stride=2, pooling_padding=1, num_layers=14, num_heads=6, mlp_ratio=3.,
                  num_classes=1000, positional_embedding='learnable')
README_CCT14 = dict(img_size=224, n_conv_layers=1, kernel_size=7, stride=2, padding=3, pooling_kernel_size=3,
                    pooling_stride=2, pooling_padding=1, num_classes=1000, positional_embedding='learnable')


def test_readme_configs_take_the_fused_path():
    for make, kw, shape in ((CCT, README_CCT, (224, 448)), (cct_mod.cct_14, README_CCT14, (224, 224))):
        m = make(**kw).eval().to(DEV, torch.bfloat16)
        x = torch.randn(2, 3, *shape, device=DEV).bfloat16()
        with torch.inference_mode():
            assert m.fused_reason(x) is None
            out = m(x)
            assert out.shape == (2, 1000) and torch.isfinite(out.float()).all()
        del m


def test_cuda_graph_replay_is_bit_identical():
    from vit_pytorch_b200.graph import GraphedForward
    spec = CCT_CASES["two_layers_k7_nonsquare"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    a = FAMILY.input(spec).to(DEV)
    b = torch.randn_like(a.float()).bfloat16()
    with torch.inference_mode():
        ya, yb = m(a).clone(), m(b).clone()
        g = GraphedForward(m, a)
        assert torch.equal(g(b), yb)
        assert torch.equal(g(a), ya)


def test_weight_updates_reach_the_fused_output():
    """load_state_dict and in-place updates of a conv weight, the pooling Linear and the positional table all rebuild
    the prepared weights: afterwards the fused output equals, bit for bit, that of a fresh model with the same state."""
    spec = CCT_CASES["learnable"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    x = FAMILY.input(spec).to(DEV)
    with torch.inference_mode():
        before = m(x).clone()
    with torch.no_grad():
        m.tokenizer.conv_layers[0][0].weight.mul_(-1.0)
        m.classifier.attention_pool.weight.mul_(3.0)
        m.classifier.positional_emb.add_(0.25)
    fresh = FAMILY.build(spec).to(DEV, torch.bfloat16)
    with torch.inference_mode():
        fresh(x)                                          # prepares fresh's weights from the old state first
    fresh.load_state_dict(m.state_dict())
    with torch.inference_mode():
        assert m.fused_reason(x) is None
        after = m(x)
        assert not torch.equal(after, before)
        assert torch.equal(after, fresh(x))


def test_fallback_rules_on_the_gpu():
    kw = dict(img_size=32, embedding_dim=64, kernel_size=3, stride=1, padding=1, num_layers=1, num_heads=1,
              num_classes=3)
    m = CCT(**kw).eval().to(DEV, torch.bfloat16)
    x = torch.randn(2, 3, 32, 32, device=DEV).bfloat16()
    assert "autograd" in m.fused_reason(x)
    with torch.inference_mode():
        assert m.fused_reason(x) is None
        assert m.fused_reason(x.float()) is not None
        assert "dropout" in m.train().fused_reason(x)
        m.eval()
        h = m.classifier.blocks[0].norm1.register_forward_hook(lambda *a: None)
        assert "hooks" in m.fused_reason(x)
        h.remove()
        bad = torch.randn(2, 3, 36, 32, device=DEV).bfloat16()
        assert "positional table" in m.fused_reason(bad)
        with pytest.raises(RuntimeError):
            m(bad)
