"""Host-side drop-in contract of vit_pytorch_b200.ViT / SimpleViT: constructor signature, state_dict
layout, attribute surface, eager-graph values against the reference goldens, dispatch rules.  CPU only."""
import inspect

import pytest
import torch
from torch import nn

from conftest import import_reference, load_golden, reference_available, reference_live, state_digest
from vit_pytorch_b200 import SimpleViT, ViT
from vit_pytorch_b200 import simple_vit as sv_mod
from vit_pytorch_b200 import vit as vit_mod


def _build(g):
    cls = ViT if g["kind"] == "vit" else SimpleViT
    m = cls(**g["kwargs"]).eval()
    m.load_state_dict(g["state_dict"])      # strict: key set and shapes must equal the reference's
    return m


def test_state_dict_layout_equals_reference(golden):
    cls = ViT if golden["kind"] == "vit" else SimpleViT
    m = cls(**golden["kwargs"])
    ours, ref = m.state_dict(), golden["state_dict"]
    assert list(ours.keys()) == list(ref.keys())          # same names AND same registration order
    for k in ref:
        assert ours[k].shape == ref[k].shape, k


def test_eager_forward_equals_reference_golden(golden):
    m = _build(golden).float()
    with torch.inference_mode():
        out = m(golden["input"].float())
    assert torch.allclose(out, golden["logits_fp32"], rtol=1e-5, atol=5e-6)


def test_constructor_signatures():
    sig = inspect.signature(ViT.__init__)
    names = [p for p in sig.parameters if p != "self"]
    assert names == ["image_size", "patch_size", "num_classes", "dim", "depth", "heads", "mlp_dim", "pool", "channels",
                     "dim_head", "dropout", "emb_dropout"]
    assert all(sig.parameters[n].kind is inspect.Parameter.KEYWORD_ONLY for n in names)
    assert sig.parameters["pool"].default == "cls" and sig.parameters["dim_head"].default == 64
    sig = inspect.signature(SimpleViT.__init__)
    names = [p for p in sig.parameters if p != "self"]
    assert names == ["image_size", "patch_size", "num_classes", "dim", "depth", "heads", "mlp_dim", "channels",
                     "dim_head"]


def test_assertion_messages():
    with pytest.raises(AssertionError, match="Image dimensions must be divisible by the patch size."):
        ViT(image_size=30, patch_size=4, num_classes=2, dim=8, depth=1, heads=1, mlp_dim=8)
    with pytest.raises(AssertionError, match="pool type must be either cls"):
        ViT(image_size=32, patch_size=4, num_classes=2, dim=8, depth=1, heads=1, mlp_dim=8, pool="max")
    with pytest.raises(AssertionError, match="multiple of 4"):
        SimpleViT(image_size=32, patch_size=4, num_classes=2, dim=6, depth=1, heads=1, mlp_dim=8)


def test_attribute_surface():
    v = ViT(image_size=32, patch_size=(8, 4), num_classes=5, dim=64, depth=2, heads=2, mlp_dim=96, dim_head=16)
    assert v.patch_size == (8, 4) and v.pool == "cls"
    assert isinstance(v.to_latent, nn.Identity) and isinstance(v.dropout, nn.Dropout)
    assert isinstance(v.to_patch_embedding[1], nn.LayerNorm) and isinstance(v.to_patch_embedding[2], nn.Linear)
    assert v.to_patch_embedding[2].weight.shape == (64, 3 * 8 * 4)
    assert v.cls_token.shape == (1, 64) and v.pos_embedding.shape == (4 * 8 + 1, 64)
    attn, ff = v.transformer.layers[1]
    assert isinstance(attn, vit_mod.Attention) and isinstance(attn.attend, nn.Softmax)
    assert attn.heads == 2 and attn.scale == 16 ** -0.5
    assert isinstance(attn.to_out, nn.Sequential) and isinstance(ff.net, nn.Sequential) and len(ff.net) == 6
    # to_patch_embedding[0] alone is the patchify op (MAE uses it separately, reference mae.py:28-31)
    img = torch.randn(2, 3, 32, 32)
    assert v.to_patch_embedding[0](img).shape == (2, 32, 96)
    s = SimpleViT(image_size=32, patch_size=8, num_classes=5, dim=64, depth=1, heads=2, mlp_dim=96, dim_head=16)
    assert "pos_embedding" not in s.state_dict() and s.pos_embedding.shape == (16, 64)
    assert isinstance(s.transformer.layers[0][0].to_out, nn.Linear) and s.transformer.layers[0][0].to_out.bias is None
    assert len(s.transformer.layers[0][1].net) == 4 and hasattr(s, "linear_head")


def test_edge_cases_shapes():
    # pool='mean' -> no cls token; num_classes=0 -> tokens; heads=1 & dim_head=dim -> Identity projection
    v = ViT(image_size=32, patch_size=8, num_classes=0, dim=32, depth=1, heads=1, mlp_dim=48, dim_head=32,
            pool="mean").eval()
    assert v.cls_token.shape == (0, 32) and v.mlp_head is None
    assert isinstance(v.transformer.layers[0][0].to_out, nn.Identity)
    assert v(torch.randn(2, 3, 32, 32)).shape == (2, 16, 32)
    # smaller, non-square input than image_size (reference README.md:1720-1745)
    v = ViT(image_size=64, patch_size=16, num_classes=7, dim=32, depth=1, heads=2, mlp_dim=48, dim_head=16).eval()
    assert v(torch.randn(2, 3, 64, 32)).shape == (2, 7)
    # the reference's own shape test (tests/test_vit.py:4-20), in train mode with dropout
    v = ViT(image_size=256, patch_size=32, num_classes=1000, dim=64, depth=2, heads=4, mlp_dim=96, dropout=0.1,
            emb_dropout=0.1)
    assert v(torch.randn(1, 3, 256, 256)).shape == (1, 1000)


def test_transformer_callable_on_arbitrary_tokens():
    v = ViT(image_size=32, patch_size=8, num_classes=3, dim=32, depth=2, heads=2, mlp_dim=48, dim_head=16).eval()
    assert v.transformer(torch.randn(2, 5, 32)).shape == (2, 5, 32)     # MAE-style subset of tokens


def test_dispatch_reasons_on_cpu():
    v = ViT(image_size=32, patch_size=8, num_classes=3, dim=128, depth=1, heads=2, mlp_dim=128).eval()
    img = torch.randn(1, 3, 32, 32)
    assert v.fused_reason(img) == "input is not on a CUDA device"
    assert v.transformer.fused_reason(torch.randn(1, 4, 128)) == "input is not on a CUDA device"
    s = SimpleViT(image_size=32, patch_size=8, num_classes=3, dim=128, depth=1, heads=2, mlp_dim=128).eval()
    assert s.fused_reason(img) is not None


def test_hooks_force_the_observable_graph():
    from vit_pytorch_b200.engine import hooks_inside
    v = ViT(image_size=32, patch_size=8, num_classes=3, dim=32, depth=1, heads=2, mlp_dim=48, dim_head=16).eval()
    assert not hooks_inside(v, skip=(v.to_latent,))
    v.to_latent.register_forward_hook(lambda m, i, o: None)       # Dino-style hook on to_latent is allowed
    assert not hooks_inside(v, skip=(v.to_latent,))
    seen = []
    h = v.transformer.layers[0][0].attend.register_forward_hook(lambda m, i, o: seen.append(o.shape))
    assert hooks_inside(v, skip=(v.to_latent,)) and hooks_inside(v.transformer)
    v(torch.randn(2, 3, 32, 32))
    assert seen == [torch.Size([2, 2, 17, 17])]                    # Recorder-style attention maps (B,H,N,N)
    h.remove()


@pytest.mark.parametrize("kind", ["vit", "simple"])
def test_same_seed_gives_bit_identical_init(kind):
    """The reference's initialisation under the same seed, stored as per-tensor digests of its state_dict."""
    want = reference_live()["init"][f"dropin_{kind}"]
    kwargs = dict(image_size=32, patch_size=8, num_classes=5, dim=64, depth=2, heads=2, mlp_dim=96, dim_head=32)
    torch.manual_seed(123)
    b = (ViT if kind == "vit" else SimpleViT)(**kwargs)
    got = state_digest(b.state_dict())
    assert list(got) == list(want)
    for k in want:
        assert got[k] == want[k], k
    if kind == "simple":
        assert state_digest({"pos_embedding": b.pos_embedding}) == reference_live()["init"]["dropin_simple_pos"]


@pytest.mark.skipif(not reference_available(), reason="runs the reference's own code: no reference package (oracle/_ref or VIT_REFERENCE)")
def test_reference_wrappers_accept_the_dropin():
    """Recorder / Extractor from the reference operate on our module tree."""
    import importlib
    import_reference()
    Extractor = importlib.import_module("vit_pytorch.extractor").Extractor
    v = ViT(image_size=32, patch_size=8, num_classes=3, dim=32, depth=2, heads=2, mlp_dim=48, dim_head=16).eval()
    logits, emb = Extractor(v)(torch.randn(2, 3, 32, 32))
    assert logits.shape == (2, 3) and emb.shape == (2, 17, 32)


def _pair_with_reference(**kwargs):
    """Our ViT and the reference's with the same weights (fp32, eval)."""
    import importlib
    import_reference()
    RefViT = importlib.import_module("vit_pytorch.vit").ViT
    torch.manual_seed(0)
    ours = ViT(**kwargs).eval()
    ref = RefViT(**kwargs).eval()
    ref.load_state_dict(ours.state_dict())
    return ours, ref


@pytest.mark.skipif(not reference_available(), reason="runs the reference's own code: no reference package (oracle/_ref or VIT_REFERENCE)")
def test_reference_mae_wrapper_runs_on_the_dropin():
    """MAE (reference mae.py:28-31,50-55,74) reads `to_patch_embedding[0]`, `[1:]`, `[2].weight`, `pos_embedding`,
    `pool` and calls `encoder.transformer(tokens)` on the unmasked quarter of the tokens: same loss as on the
    reference's own ViT.  (pool='mean': with the 2-D `pos_embedding` of vit.py:107 the wrapper's `[:, 1:n+1]` slice for
    pool='cls' -- and SimMIM's, simmim.py:45 -- fails on the reference's own ViT too, so there is nothing to match.)"""
    import importlib
    ours, ref = _pair_with_reference(image_size=32, patch_size=8, num_classes=5, dim=64, depth=2, heads=2, mlp_dim=96,
                                     pool="mean")
    MAE = importlib.import_module("vit_pytorch.mae").MAE
    make = lambda enc: MAE(encoder=enc, decoder_dim=32, masking_ratio=0.75, decoder_depth=1, decoder_heads=2,  # noqa
                           decoder_dim_head=16)
    torch.manual_seed(1)
    a = make(ours).eval()
    b = make(ref).eval()
    b.load_state_dict(a.state_dict())
    img = torch.randn(3, 3, 32, 32)
    with torch.no_grad():
        torch.manual_seed(2)
        la = a(img)
        torch.manual_seed(2)
        lb = b(img)
    assert torch.allclose(la, lb, rtol=1e-5, atol=1e-6), (la, lb)
    a(img).backward()                                # and it trains: gradients reach the encoder through the wrapper
    assert ours.transformer.layers[0][0].to_qkv.weight.grad is not None


@pytest.mark.skipif(not reference_available(), reason="runs the reference's own code: no reference package (oracle/_ref or VIT_REFERENCE)")
def test_reference_distill_wrapper_accepts_the_dropin_as_teacher():
    """DistillWrapper (reference distill.py:104-152) calls `teacher(img)` under no_grad."""
    import importlib
    import_reference()
    distill = importlib.import_module("vit_pytorch.distill")
    kw = dict(image_size=32, patch_size=8, num_classes=5, dim=64, depth=1, heads=2, mlp_dim=96)
    torch.manual_seed(0)
    teacher = ViT(**kw).eval()
    student = distill.DistillableViT(**kw)
    loss = distill.DistillWrapper(student=student, teacher=teacher, temperature=3, alpha=0.5)(
        torch.randn(2, 3, 32, 32), torch.tensor([1, 3]))
    assert loss.dim() == 0 and torch.isfinite(loss)


def test_recorder_and_extractor_twins():
    """vit_pytorch_b200.recorder / .extractor mirror reference recorder.py:10-59 / extractor.py:18-92."""
    from vit_pytorch_b200.extractor import Extractor
    from vit_pytorch_b200.recorder import Recorder
    torch.manual_seed(0)
    v = ViT(image_size=32, patch_size=8, num_classes=3, dim=32, depth=2, heads=2, mlp_dim=48, dim_head=16).eval()
    img = torch.randn(2, 3, 32, 32)
    with torch.no_grad():
        plain = v(img)
        rec = Recorder(v)
        pred, attns = rec(img)
        assert attns.shape == (2, 2, 2, 17, 17) and torch.allclose(attns.sum(-1), torch.ones(2, 2, 2, 17), atol=1e-5)
        assert torch.equal(pred, plain)
        assert rec.eject() is v and not any(l[0].attend._forward_hooks for l in v.transformer.layers)
        ext = Extractor(v)
        pred, emb = ext(img)
        assert torch.equal(pred, plain) and emb.shape == (2, 17, 32)
        assert ext(img, return_embeddings_only=True).shape == (2, 17, 32)
        first = Extractor(v, layer=v.transformer.layers[0][1], layer_save_input=True)
        _, inp = first(img)
        assert isinstance(inp, tuple) and inp[0].shape == (2, 17, 32)
    # the reference's Recorder on the reference ViT with the same seed and input
    live = reference_live()
    assert state_digest(v.state_dict()) == live["init"]["recorder_vit"]
    assert torch.allclose(live["logits"]["recorder"]["attns"], attns, atol=1e-6)


@pytest.mark.skipif(not reference_available(), reason="runs the reference's own code: no reference package (oracle/_ref or VIT_REFERENCE)")
def test_reference_accept_video_wrapper_runs_on_the_dropin():
    """AcceptVideoWrapper (reference accept_video_wrapper.py:26-150) reads `image_net.patch_size` and feeds the frames
    of a clip through `image_net.forward` as one batch: same output as on the reference's own ViT."""
    import importlib
    ours, ref = _pair_with_reference(image_size=32, patch_size=8, num_classes=7, dim=32, depth=1, heads=2, mlp_dim=48,
                                     dim_head=16)
    Wrapper = importlib.import_module("vit_pytorch.accept_video_wrapper").AcceptVideoWrapper
    a = Wrapper(ours, add_time_pos_emb=True, time_seq_len=4, dim_emb=7)
    b = Wrapper(ref, add_time_pos_emb=True, time_seq_len=4, dim_emb=7)
    b.load_state_dict(a.state_dict())
    assert a.patch_size == b.patch_size == (8, 8)
    video = torch.randn(2, 3, 4, 32, 32)
    with torch.no_grad():
        assert torch.allclose(a(video), b(video), rtol=1e-5, atol=1e-6)
