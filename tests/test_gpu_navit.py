"""-m gpu: NaViT through the fused padding-free sm_90a path against the reference golden and the per-image oracle."""
import random

import pytest
import torch

from conftest import load_golden
from oracle import attention_bounds as AB
from oracle import attention_fp32_bounds as FB
from oracle import bounds as Bd
from oracle import navit_oracle as NO
from oracle import vit_oracle as O
from vit_pytorch_b200 import NaViT, _lib

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _stats(got, ref, rtol=1e-2, atol=1e-3):
    d = (got.float().cpu() - ref).abs()
    return d.max().item(), d.mean().item(), (d <= atol + rtol * ref.abs()).float().mean().item()


def test_navit_golden_fused():
    g = load_golden("navit_tiny")
    m = NaViT(**g["kwargs"]).eval()
    m.load_state_dict(g["state_dict"])
    m = m.to(DEV, torch.bfloat16)
    imgs = [im.to(DEV) for im in g["images"]]
    rows = [[imgs[i] for i in r] for r in g["rows"]]
    _lib.reset_launch_count()
    with torch.inference_mode():
        assert m.fused_reason(rows) is None
        out = m(rows)
        out_grouped = m(imgs, group_images=True, group_max_seq_len=g["group_max_seq_len"])
    assert _lib.launch_count() > 0
    mx, mean, frac = _stats(out, g["logits_fp32"])
    print(f"navit_tiny fused vs reference fp32: max {mx:.5f} mean {mean:.5f} within {frac:.4f}")
    assert out.shape == g["logits_fp32"].shape and mx < 1.5e-2 and frac > 0.85
    assert torch.equal(out, out_grouped)          # packing does not exist on the fused path: identical bits


def test_navit_varied_resolutions_against_oracle():
    """BASELINE.json configs[4] style batch (variable resolutions up to 32x32 patches => up to 1024 tokens per image,
    multi key-block attention), small width/depth so the per-image oracle finishes in seconds."""
    kwargs = dict(image_size=512, patch_size=16, num_classes=100, dim=256, depth=2, heads=4, mlp_dim=512)
    torch.manual_seed(3)
    m = NaViT(**kwargs).eval().bfloat16()
    random.seed(1)
    sizes = [(16 * random.randrange(1, 33), 16 * random.randrange(1, 33)) for _ in range(12)] + [(512, 512), (16, 16)]
    torch.manual_seed(4)
    imgs = [torch.randn(3, h, w).bfloat16() for h, w in sizes]
    ref = NO.navit_forward(O.upcast(m.state_dict()), kwargs, [[im.float() for im in imgs]])
    m = m.to(DEV)
    with torch.inference_mode():
        assert m.fused_reason([im.to(DEV) for im in imgs]) is None
        out = m([im.to(DEV) for im in imgs])
    mx, mean, frac = _stats(out, ref)
    print(f"navit 14 images (1..1024 tokens) fused vs fp32 oracle: max {mx:.5f} mean {mean:.5f} within {frac:.4f}")
    assert out.shape == (14, 100) and torch.isfinite(out.float()).all()
    assert mx < 3e-2 and frac > 0.80


def test_navit_config5_geometry_against_reference_golden():
    """BASELINE.json configs[4] GEOMETRY: dim 1024, depth 6, heads 16, mlp 4096 (K = 1024 / N = 3072 head-norm QKV
    epilogue, K = 4096 FC2), 10 images from 1 token to 32 x 32 patches = 1024 tokens.  Weights and images are rebuilt
    from the seeds (tests/golden/navit_c5_spec.py); the expectation is the UNMODIFIED reference's fp32 forward and the
    pass criterion its own bf16 error on the same inputs (both stored by make_golden.py in navit_config5.pt)."""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from navit_c5_spec import NAVIT_C5, navit_config5_images, navit_config5_model
    g = load_golden("navit_config5")
    assert g["spec"] == NAVIT_C5
    m = navit_config5_model(NaViT).to(DEV, torch.bfloat16)
    imgs = [im.to(DEV) for im in navit_config5_images()]
    _lib.reset_launch_count()
    with torch.inference_mode():
        assert m.fused_reason(imgs) is None
        out = m(imgs)
        out_rows = m([imgs[:3], imgs[3:]])              # pre-packed rows: same images, same order
    assert _lib.launch_count() > 0
    ref, floor = g["logits_fp32"], g["ref_bf16_floor"]
    mx, mean, frac = _stats(out, ref)
    print(f"navit config-5 geometry fused vs reference fp32: max {mx:.5f} mean {mean:.5f} within {frac:.4f}; "
          f"reference-bf16 floor max {floor['max']:.5f} mean {floor['mean']:.5f} within {floor['frac_within_tol']:.4f}")
    assert out.shape == ref.shape and torch.isfinite(out.float()).all()
    assert mx <= floor["max"] and mean <= floor["mean"] and frac >= floor["frac_within_tol"]
    assert torch.equal(out, out_rows)


def test_varlen_attention_kernel_against_oracle():
    lengths = [197, 1, 130, 577, 64, 1024, 129, 65, 63, 128, 300]
    H, dh = 3, 64
    T = sum(lengths)
    torch.manual_seed(0)
    qkv = torch.randn(T, 3 * H * dh, device=DEV).bfloat16()
    out = torch.full((T, H * dh), float("nan"), device=DEV, dtype=torch.bfloat16)
    cu, tp, tiles = _lib.varlen_index(lengths, DEV)
    _lib.attention_varlen(qkv, out, cu, tp, tiles, H, dh, dh ** -0.5)
    torch.cuda.synchronize()
    ref, bound = AB.qkv_attention_reference(qkv, lengths, H, dh, dh ** -0.5)
    Bd.check(out, ref, bound, "varlen attention")


@pytest.mark.parametrize("pattern", ["rising", "falling", "spike_late", "mixed_rows"])
def test_varlen_attention_one_pass_moves_its_reference_max(pattern):
    """The online softmax rescales O whenever a later key block raises the running max.  Scores built to rise by ~2^40
    per 64-key block (every block triggers the rescale), to fall, to spike in the last block only, and to do so for
    some rows of a warp only; same expectation as the ordinary test."""
    lengths = [700, 130, 64, 321]
    H, dh = 2, 64
    T = sum(lengths)
    g = torch.Generator().manual_seed(3)
    u = torch.randn(dh, generator=g)
    u = u / u.norm()
    q = torch.randn(T, H, dh, generator=g) * 0.05
    k = torch.randn(T, H, dh, generator=g) * 0.05
    v = torch.randn(T, H, dh, generator=g)
    o = 0
    for n in lengths:
        pos = torch.arange(n, dtype=torch.float32)
        blk = (pos // 64)
        if pattern == "rising":
            amp = blk + 1.0
        elif pattern == "falling":
            amp = (n // 64 + 1) - blk
        elif pattern == "spike_late":
            amp = torch.where(blk == (n - 1) // 64, torch.tensor(6.0), torch.tensor(0.1))
        else:
            amp = blk + 1.0
        # score(i, j) = 240 * amp_j * (+-1)  (scale 1/8 -> 30 * amp_j in softmax units, x 1.44 in log2 units)
        sign = torch.ones(n)
        if pattern == "mixed_rows":
            sign = torch.where(torch.arange(n) % 3 == 0, torch.tensor(-1.0), torch.tensor(1.0))
        q[o:o + n] += (sign[:, None, None] * 15.5) * u
        k[o:o + n] += (amp[:, None, None] * 15.5) * u
        o += n
    qkv = torch.stack([q, k, v], dim=1).reshape(T, 3 * H * dh).bfloat16().to(DEV)
    cu, tp, tiles = _lib.varlen_index(lengths, DEV)
    out = torch.full((T, H * dh), float("nan"), device=DEV, dtype=torch.bfloat16)
    _lib.attention_varlen(qkv, out, cu, tp, tiles, H, dh, dh ** -0.5)
    torch.cuda.synchronize()
    ref, bound = AB.qkv_attention_reference(qkv, lengths, H, dh, dh ** -0.5)
    Bd.check(out, ref, bound, pattern)


@pytest.mark.parametrize("H", [3, 4, 16])
def test_qk_rmsnorm_and_attn_pool_kernels(H):
    torch.manual_seed(1)
    T, dh = 300, 64
    I = H * dh
    qkv = torch.randn(T, 3 * I, device=DEV).bfloat16()
    g = torch.randn(2, H, dh, device=DEV)
    ref = qkv.float().clone().view(T, 3, H, dh)
    for s in (0, 1):
        ref[:, s] = NO.rms_norm_heads(ref[:, s].permute(1, 0, 2).cpu(), g[s].cpu()[:, None, :]).permute(1, 0, 2).to(DEV)
    _lib.qk_rmsnorm(qkv, g.reshape(-1).contiguous(), H, dh)
    assert torch.allclose(qkv.float().view(T, 3, H, dh), ref, rtol=1e-2, atol=1e-2)
    lengths = [100, 1, 199]
    cu, _, _ = _lib.varlen_index(lengths, DEV)
    kv = qkv[:, I:].contiguous()
    qn = torch.randn(I, device=DEV)
    out = torch.full((3, I), float("nan"), device=DEV, dtype=torch.bfloat16)
    _lib.attn_pool(kv, qn, cu, out, H, dh)
    ref, bound = FB.navit_pool_reference(kv, qn, lengths, H, dh)
    Bd.check(out, ref, bound, f"attn_pool H{H}")


def test_rmsnorm_heads_on_the_k_half_of_a_kv_buffer():
    torch.manual_seed(2)
    T, H, dh = 77, 5, 64
    I = H * dh
    kv = torch.randn(T, 2 * I, device=DEV).bfloat16()
    g = torch.randn(H, dh, device=DEV)
    before = kv.clone()
    _lib.rmsnorm_heads(kv, g.reshape(-1).contiguous(), H, dh)
    want = NO.rms_norm_heads(before[:, :I].float().view(T, H, dh).permute(1, 0, 2).cpu(), g.cpu()[:, None, :])
    assert torch.allclose(kv[:, :I].float().view(T, H, dh).permute(1, 0, 2).cpu(), want, rtol=1e-2, atol=1e-2)
    assert torch.equal(kv[:, I:], before[:, I:])                      # v untouched


def test_embed_varlen_matches_torch():
    torch.manual_seed(5)
    p, D = 16, 192
    sizes = [(48, 32), (16, 16), (64, 80), (32, 128)]
    imgs = [torch.empty(3, h, w, device=DEV, dtype=torch.bfloat16) for h, w in sizes]
    ix = _lib.VarlenIndex(imgs, p, DEV)
    T = ix.T
    y = torch.randn(T, D, device=DEV)
    gamma = torch.randn(D, device=DEV)
    pos_h, pos_w = torch.randn(9, D, device=DEV), torch.randn(9, D, device=DEV)
    x = torch.empty(T, D, device=DEV)
    xb = torch.empty(T, D, device=DEV, dtype=torch.bfloat16)
    st = torch.empty(T, 1, 2, device=DEV)
    _lib.embed_varlen(y, gamma, pos_h, pos_w, ix, x, p, xb=xb, stats=st)
    hi = torch.cat([torch.arange(h // p).repeat_interleave(w // p) for h, w in sizes]).to(DEV)
    wi = torch.cat([torch.arange(w // p).repeat(h // p) for h, w in sizes]).to(DEV)
    want = torch.nn.functional.layer_norm(y, (D,), gamma, None) + pos_h[hi] + pos_w[wi]
    assert torch.allclose(x, want, rtol=1e-5, atol=1e-5)
    assert torch.equal(xb, x.bfloat16())
    xf = xb.float()
    assert torch.allclose(st[:, 0, 0], xf.sum(1), rtol=1e-4, atol=1e-3)
    assert torch.allclose(st[:, 0, 1], (xf * xf).sum(1), rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("misalign", [False, True])
def test_patchify_varlen_ln_fast_path(misalign):
    """p = 16 kernel: 16-byte staged images and element-wise staged (2-byte aligned) images give the reference
    'c (h p1) (w p2) -> (h w) (c p1 p2)' + LayerNorm(no bias)."""
    torch.manual_seed(6)
    p, C = 16, 3
    sizes = [(32, 48), (16, 16), (80, 512), (48, 16)]
    imgs = []
    for h, w in sizes:
        flat = torch.randn(C * h * w + 8, device=DEV).bfloat16()
        off = 1 if misalign else 0
        imgs.append(flat[off:off + C * h * w].view(C, h, w))
        assert imgs[-1].is_contiguous() and (imgs[-1].data_ptr() % 16 == 0) == (not misalign)
    ix = _lib.VarlenIndex(imgs, p, DEV)
    gamma = torch.randn(C * p * p, device=DEV)
    out = torch.empty(ix.T, C * p * p, device=DEV, dtype=torch.bfloat16)
    _lib.patchify_varlen_ln(imgs, gamma, out, ix.cu, p, index=ix)
    want = torch.cat([torch.nn.functional.layer_norm(NO.patchify_cpp(im.float().cpu(), p), (C * p * p,), gamma.cpu(), None)
                      for im in imgs])
    assert torch.allclose(out.float().cpu(), want, rtol=1e-2, atol=1e-2)


@pytest.mark.parametrize("mode", ["exact", "fold"])
def test_navit_ln_modes_agree_with_golden(mode, monkeypatch):
    monkeypatch.setenv("B200VIT_LN_MODE", mode)
    g = load_golden("navit_tiny")
    m = NaViT(**g["kwargs"]).eval()
    m.load_state_dict(g["state_dict"])
    m = m.to(DEV, torch.bfloat16)
    rows = [[g["images"][i].to(DEV) for i in r] for r in g["rows"]]
    with torch.inference_mode():
        out = m(rows)
    mx, mean, frac = _stats(out, g["logits_fp32"])
    print(f"navit_tiny {mode}: max {mx:.5f} mean {mean:.5f} within {frac:.4f}")
    assert mx < 1.5e-2 and frac > 0.85


@pytest.mark.parametrize("M", [300, 5000])
@pytest.mark.parametrize("fold", [False, True])
def test_gemm_headnorm_matches_gemm_then_rmsnorm(M, fold):
    torch.manual_seed(8)
    H, dh, K = 4, 64, 256
    I = H * dh
    a = torch.randn(M, K, device=DEV).bfloat16()
    w = (torch.randn(3 * I, K, device=DEV) / K ** 0.5).bfloat16()
    g = torch.randn(2 * I, device=DEV)
    kw = {}
    if fold:
        af = a.float()
        kw = dict(bias=torch.randn(3 * I, device=DEV), col_s=w.float().sum(1).contiguous(),
                  ln_sums=torch.stack([af.sum(1), (af * af).sum(1)], 1).contiguous())
    want = torch.empty(M, 3 * I, device=DEV, dtype=torch.bfloat16)
    _lib.gemm(a, w, out_bf16=want, **kw)
    v_part = want[:, 2 * I:].clone()
    _lib.qk_rmsnorm(want, g, H, dh)
    got = torch.empty_like(want)
    _lib.gemm_headnorm(a, w, out_bf16=got, head_gamma=g, norm_heads=2 * H, **kw)
    assert torch.equal(got[:, 2 * I:], v_part)                          # v columns untouched
    d = (got.float() - want.float()).abs()
    assert (d <= 1e-3 + 1e-2 * want.float().abs()).float().mean() > 0.999, d.max()
