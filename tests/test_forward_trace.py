"""Whole fused forwards traced from the pixels to the logits without a GPU
(oracle/layer_trace.check_forward_provenance).

The encoder-layer traces (tests/test_layer_trace.py and its siblings) start after the embedding.  Here each model's
forward_fused runs on CPU with every library launch traced and emulated (oracle/layer_trace.emulate_impl: each output
gets the fp64 reference of its kernel on the operands the launch received, rounded to its dtype), and the walk
attributes every launch -- the patch embedding in both patch modes, the token assembly, the encoder layers, the final
LayerNorm, the pooling, NaViT's attention pooling and the head -- to the reference module's attributes.  Every case
consumes every launch, and its emulated logits must match the module's own fp32 PyTorch forward.

Then defects in the embedding and the head bookkeeping are planted with monkeypatch; the walk must name the launch and
the operand each one corrupts."""
import copy

import pytest
import torch
from torch import nn

from oracle import layer_trace as LT
from test_layer_trace import lib  # noqa: F401  (the module fixture that builds the library)
from vit_pytorch_b200 import (deepvit, engine, na_vit, simple_flash_attn_vit, simple_vit, simple_vit_1d, simple_vit_3d,
                              simple_vit_with_patch_dropout, simple_vit_with_qk_norm, simple_vit_with_register_tokens,
                              vit, vit_for_small_dataset, vit_nd, vit_nd_rotary, vivit)

EPS = (1e-5, 1e-6, 1e-3)
D, HEADS, DH, MLP = 64, 2, 32, 128
B = 2


def set_eps(model):
    """The nn.LayerNorms take eps 1e-5, 1e-6, 1e-3 in module order, the head's LayerNorm 1e-3: a LayerNorm run at
    another one's eps, or at the default, is a wrong argument."""
    norms = [m for m in model.modules() if isinstance(m, nn.LayerNorm)]
    for j, m in enumerate(norms):
        m.eps = EPS[j % len(EPS)]
    head = getattr(model, "mlp_head", None)
    if isinstance(head, nn.Sequential) and isinstance(head[0], nn.LayerNorm):
        head[0].eps = EPS[2]


def perturbed(build, seed=0, device="cpu"):
    """build() in eval mode with every parameter moved by noise, so that LayerNorm gains and shifts are not their
    constants, and with set_eps."""
    torch.manual_seed(seed)
    model = build().eval()
    with torch.no_grad():
        for p in model.parameters():
            p.add_(0.05 * torch.randn_like(p))
    set_eps(model)
    return model.to(device)


def _kw(**extra):
    return dict(num_classes=10, dim=D, depth=2, heads=HEADS, dim_head=DH, mlp_dim=MLP, **extra)


def _video_kw(temporal_depth=1, **extra):
    kw = _kw(**extra)
    kw.pop("depth")
    return dict(kw, spatial_depth=2, temporal_depth=temporal_depth)


# name: (model, input shape after (batch, channels) -- NaViT: the list of image sizes)
CASES = {
    "vit cls": (lambda: vit.ViT(image_size=(32, 48), patch_size=16, pool="cls", **_kw()), (32, 48)),
    "vit mean": (lambda: vit.ViT(image_size=(48, 32), patch_size=16, pool="mean", **_kw()), (48, 32)),
    "vit patch 8": (lambda: vit.ViT(image_size=32, patch_size=8, pool="cls", **_kw()), (32, 32)),
    "simple_vit": (lambda: simple_vit.SimpleViT(image_size=(32, 48), patch_size=16, **_kw()), (32, 48)),
    "simple_vit register tokens": (lambda: simple_vit_with_register_tokens.SimpleViT(
        image_size=32, patch_size=8, num_register_tokens=3, **_kw()), (32, 32)),
    "simple_vit qk norm": (lambda: simple_vit_with_qk_norm.SimpleViT(image_size=32, patch_size=16, **_kw()), (32, 32)),
    "simple_vit patch dropout (eval)": (lambda: simple_vit_with_patch_dropout.SimpleViT(
        image_size=32, patch_size=8, patch_dropout=0.5, **_kw()), (32, 32)),
    "simple_flash_attn_vit": (lambda: simple_flash_attn_vit.SimpleViT(image_size=32, patch_size=16, **_kw()),
                              (32, 48)),
    "vit small dataset (SPT)": (lambda: vit_for_small_dataset.ViT(image_size=32, patch_size=8, pool="cls", **_kw()),
                                (32, 32)),
    "vit small dataset mean": (lambda: vit_for_small_dataset.ViT(image_size=32, patch_size=8, pool="mean", **_kw()),
                               (32, 32)),
    "deepvit": (lambda: deepvit.DeepViT(image_size=32, patch_size=16, pool="cls", **_kw()), (32, 32)),
    # non-square images of a square table: pos_embed_height and pos_embed_width have one shape, not one content
    "navit": (lambda: na_vit.NaViT(image_size=64, patch_size=16, **_kw()), [(32, 64), (48, 16), (16, 16), (64, 48)]),
    "vit_nd 3-d cls": (lambda: vit_nd.ViTND(ndim=3, input_shape=(8, 16, 24), patch_size=(2, 8, 8), pool="cls",
                                            **_kw()), (8, 16, 24)),
    "vit_nd 2-d mean": (lambda: vit_nd.ViTND(ndim=2, input_shape=(32, 48), patch_size=16, pool="mean", **_kw()),
                        (32, 48)),
    "vit_nd_rotary 3-d": (lambda: vit_nd_rotary.ViTND(ndim=3, input_shape=(4, 16, 24), patch_size=(2, 8, 8), **_kw()),
                          (4, 16, 24)),
    "simple_vit_1d": (lambda: simple_vit_1d.SimpleViT(seq_len=128, patch_size=16, **_kw()), (128,)),
    "simple_vit_3d": (lambda: simple_vit_3d.SimpleViT(image_size=(32, 48), image_patch_size=16, frames=3,
                                                      frame_patch_size=1, **_kw()), (3, 32, 48)),
    "simple_vit_3d frame patch 2": (lambda: simple_vit_3d.SimpleViT(image_size=32, image_patch_size=8, frames=4,
                                                                    frame_patch_size=2, **_kw()), (4, 32, 32)),
    "vivit factorized encoder cls": (lambda: vivit.ViViT(image_size=(32, 48), image_patch_size=16, frames=4,
                                                         frame_patch_size=2, pool="cls", **_video_kw()),
                                     (4, 32, 48)),
    "vivit factorized encoder mean": (lambda: vivit.ViViT(image_size=32, image_patch_size=16, frames=3,
                                                          frame_patch_size=1, pool="mean", **_video_kw()),
                                      (3, 32, 32)),
    "vivit factorized self-attention cls": (lambda: vivit.ViViT(
        image_size=32, image_patch_size=16, frames=3, frame_patch_size=1, pool="cls",
        variant="factorized_self_attention", **_video_kw(temporal_depth=2)), (3, 32, 32)),
    "vivit factorized self-attention mean": (lambda: vivit.ViViT(
        image_size=32, image_patch_size=8, frames=4, frame_patch_size=2, pool="mean",
        variant="factorized_self_attention", **_video_kw(temporal_depth=2)), (4, 32, 32)),
}


def tma_eligible(model) -> bool:
    """The patch embedding runs the 16 x 16 TMA kernel unless B200VIT_PATCH_MODE=gather: patches of one 16 x 16 box
    (engine.PatchEmbedEngine: fused_patch_box or patch_size) of whole channels, not shifted patches, not NaViT's
    varlen or the N-d gather."""
    if isinstance(model, (na_vit.NaViT, vit_nd.ViTND, vit_nd_rotary.ViTND)):
        return False
    pe = model.to_patch_embedding
    if hasattr(pe, "to_patch_tokens"):
        return False
    box = getattr(model, "fused_patch_box", None) or model.patch_size
    return tuple(box) == (16, 16) and pe[2].in_features % 256 == 0


def patch_modes(cases):
    """(name, patch mode) pairs: both modes where the TMA patch embedding applies."""
    out = []
    for name, (build, _) in cases.items():
        torch.manual_seed(0)
        out += [(name, m) for m in (("tma", "gather") if tma_eligible(build()) else ("gather",))]
    return out


def inputs(name, device="cpu", batch=B):
    """Seeded bf16 input of the case: [batch, 3, *shape], or NaViT's list of [3, h, w] images."""
    size = CASES[name][1]
    g = torch.Generator(device=device).manual_seed(len(name))
    if isinstance(size, list):
        return [torch.randn(3, h, w, device=device, generator=g).bfloat16() for h, w in size]
    return torch.randn(batch, 3, *size, device=device, generator=g).bfloat16()


def rows(model, img):
    """The rows of the encoder's residual stream."""
    if isinstance(model, na_vit.NaViT):
        p = model.patch_size
        return sum((im.shape[-2] // p) * (im.shape[-1] // p) for im in img)
    if isinstance(model, (vit_nd.ViTND, vit_nd_rotary.ViTND)):
        return img.shape[0] * model._nd_engine.tokens(img)[1]
    if isinstance(model, simple_vit_1d.SimpleViT):
        return img.shape[0] * (img.shape[2] // model.fused_patch_box[1])
    if isinstance(model, (simple_vit_3d.SimpleViT, vivit.ViViT)):
        pf = getattr(model, "frame_patch_size", None) or model._pf
        f, h, w = img.shape[2] // pf, img.shape[3] // model.patch_size[0], img.shape[4] // model.patch_size[1]
        ncls = 1 if isinstance(model, vivit.ViViT) and not model.global_average_pool else 0
        return img.shape[0] * f * (h * w + ncls)
    b, n = engine.patch_engine(model).geometry(img)
    return b * n


def trace(model, img, ln_mode, impl=LT.emulate_impl):
    """(launches, logits) of model.forward_fused(img) with every launch traced; every workspace buffer starts as NaN."""
    outs = []

    def setup():
        dev = img[0].device if isinstance(img, list) else img.device
        enc = model.transformer if hasattr(model, "transformer") else (
            model.spatial_transformer if model.variant == "factorized_encoder" else model.factorized_transformer)
        for buf in enc.engine().workspace(rows(model, img), dev).values():
            buf.fill_(float("nan"))
    with torch.inference_mode():
        launches = LT.trace_call(lambda: outs.append(model.forward_fused(img)), ln_mode, impl, setup=setup)
    return launches, outs[0]


def eager(model, img):
    with torch.inference_mode():
        if isinstance(img, list):
            return model.forward_eager([im.float() for im in img])
        return model.forward_eager(img.float())


def run(name, ln_mode, patch_mode, mp):
    mp.setenv("B200VIT_PATCH_MODE", patch_mode)
    model = perturbed(CASES[name][0])
    img = inputs(name)
    launches, logits = trace(model, img, ln_mode)
    return model, img, launches, logits


PARAMS = patch_modes(CASES)


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("name,patch_mode", PARAMS, ids=[f"{n} | {m}" for n, m in PARAMS])
def test_forward_traces_from_the_pixels_to_the_logits(name, patch_mode, ln_mode, monkeypatch):
    model, img, launches, logits = run(name, ln_mode, patch_mode, monkeypatch)
    case = f"{name} | {patch_mode} | {ln_mode}"
    assert LT.check_forward_provenance(model, img, launches, ln_mode, case) == len(launches) > 0
    kinds = {c.name for c in launches}
    assert ("patch_embed_tma" in kinds) == (patch_mode == "tma"), kinds
    LT.check_accuracy(launches, case)
    want = eager(model, img)
    d = (logits.float() - want).abs().max().item()
    assert d < 5e-2, (case, d)


# ------------------------------------------------------------------------------------------------------ planted defects
def _tma_w_unpermuted(mp):
    orig = engine.PatchEmbedEngine._build

    def bad(self, device):
        t = orig(self, device)
        pe = self.owner.to_patch_embedding
        w = (pe[2].weight.detach().float() * pe[1].weight.detach().float()[None, :]).bfloat16().contiguous()
        t["tma.w"], t["tma.s"] = w, w.float().sum(1).contiguous()
        return t
    mp.setattr(engine.PatchEmbedEngine, "_build", bad)


def _tma_s_unrounded(mp):
    orig = engine.PatchEmbedEngine._build

    def bad(self, device):
        t = orig(self, device)
        pe = self.owner.to_patch_embedding
        wg = pe[2].weight.detach().float() * pe[1].weight.detach().float()[None, :]
        C = wg.shape[1] // 256
        t["tma.s"] = wg.view(-1, 256, C).permute(0, 2, 1).reshape(wg.shape).sum(1).contiguous()
        return t
    mp.setattr(engine.PatchEmbedEngine, "_build", bad)


def _pool_over_registers(mp):
    orig = simple_vit_with_register_tokens.fused_mean_pooled_features
    mp.setattr(simple_vit_with_register_tokens, "fused_mean_pooled_features",
               lambda owner, img, pool_tokens=None, **kw: orig(owner, img, **kw))


def _navit_pos_swapped(mp):
    orig = na_vit.NaViT._build

    def bad(self):
        t = orig(self)
        t["pos_h"], t["pos_w"] = t["pos_w"], t["pos_h"]
        return t
    mp.setattr(na_vit.NaViT, "_build", bad)


def _head_ln_default_eps(mp):
    orig = vit_for_small_dataset.head_ln_pool

    def bad(owner, ln, x, B, N, *, mean):
        ln = copy.copy(ln)
        ln.eps = 1e-5
        return orig(owner, ln, x, B, N, mean=mean)
    mp.setattr(vit_for_small_dataset, "head_ln_pool", bad)


# name: (case, LayerNorm mode, plant(monkeypatch), what the failure must name)
DEFECTS = {
    "tma.w columns left in the (p1 p2 c) order": ("vit cls", "fold", _tma_w_unpermuted,
                                                  ("patch embedding", "patch_embed_tma", "operand w_perm")),
    "tma.s from the unrounded gamma W": ("vit mean", "exact", _tma_s_unrounded,
                                         ("patch embedding", "patch_embed_tma", "operand col_s")),
    "mean pool over the register tokens": ("simple_vit register tokens", "fold", _pool_over_registers,
                                           ("head", "mean_pool", "operand n_pool")),
    "NaViT pos_h and pos_w swapped": ("navit", "fold", _navit_pos_swapped,
                                      ("token assembly", "embed_varlen", "operand pos_h")),
    "head LayerNorm at the default eps": ("vit small dataset (SPT)", "exact", _head_ln_default_eps,
                                          ("head", "layernorm", "operand eps")),
}


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_planted_defect_is_named(defect, monkeypatch):
    name, ln_mode, plant, want = DEFECTS[defect]
    model, img, launches, _ = run(name, ln_mode, "tma", monkeypatch)
    assert LT.check_forward_provenance(model, img, launches, ln_mode, name) == len(launches)
    plant(monkeypatch)
    model, img, launches, _ = run(name, ln_mode, "tma", monkeypatch)
    with pytest.raises(LT.ProvenanceError) as e:
        LT.check_forward_provenance(model, img, launches, ln_mode, name)
    assert all(w in str(e.value) for w in want), str(e.value)


def test_an_untraced_launch_fails_the_walk(monkeypatch):
    """A launch the reference forward does not define -- here a cast after the head GEMM -- is named by _end."""
    orig = simple_vit.classify

    def extra(owner, linear, pooled):
        out = orig(owner, linear, pooled)
        engine._lib.cast_f32_bf16(pooled.float(), torch.empty_like(pooled))
        return out
    monkeypatch.setattr(simple_vit, "classify", extra)
    model, img, launches, _ = run("simple_vit", "fold", "tma", monkeypatch)
    with pytest.raises(LT.ProvenanceError, match="after the last layer.*cast_f32_bf16"):
        LT.check_forward_provenance(model, img, launches, "fold", "simple_vit")
