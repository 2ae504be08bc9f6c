"""Generate golden fixtures from the UNMODIFIED reference (lucidrains/vit-pytorch 1.23.6, a checkout of which
VIT_REFERENCE points at):

    VIT_REFERENCE=<checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden.py [reference_live]

For each case: build the reference model under torch.manual_seed(seed), round its parameters to bf16-representable
values (so the same numbers can be fed to the bf16 CUDA path), run the reference forward in fp32 on CPU on a
bf16-representable input, and additionally run the reference's own bf16 forward (its noise floor).  Saved per case
(tests/golden/<name>.pt): kind, ctor kwargs, state_dict (bf16), input (bf16), logits_fp32, logits_ref_bf16,
tokens_fp32 (transformer output for the first sample) and the library versions.
"""
from __future__ import annotations

import os
import sys

import torch

REF = os.environ["VIT_REFERENCE"]
sys.path.insert(0, REF)
sys.dont_write_bytecode = True

from vit_pytorch import ViT, SimpleViT  # noqa: E402  (the reference)

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

CASES = {
    # BASELINE.json configs[0]: SimpleViT tiny
    "simplevit_tiny": dict(kind="simple", seed=0, batch=4, img=(32, 32),
                           kwargs=dict(image_size=32, patch_size=4, num_classes=10, dim=192, depth=2, heads=3,
                                       mlp_dim=768)),
    # ViT, cls pooling, with biases everywhere, same tiny geometry
    "vit_tiny_cls": dict(kind="vit", seed=1, batch=3, img=(32, 32),
                         kwargs=dict(image_size=32, patch_size=4, num_classes=10, dim=192, depth=2, heads=3,
                                     mlp_dim=768)),
    # ViT, mean pooling, tuple sizes, smaller non-square input than image_size (README.md:1720-1766), N = 8 tokens
    "vit_tiny_mean_nonsquare": dict(kind="vit", seed=2, batch=2, img=(32, 16),
                                    kwargs=dict(image_size=(32, 32), patch_size=(8, 4), num_classes=24, dim=128,
                                                depth=3, heads=2, mlp_dim=256, pool="mean")),
    # ViT without head: returns tokens (vit.py:132-133)
    "vit_tiny_tokens": dict(kind="vit", seed=3, batch=2, img=(32, 32),
                            kwargs=dict(image_size=32, patch_size=8, num_classes=0, dim=128, depth=1, heads=2,
                                        mlp_dim=256)),
}

# Round 2: attention without output projection (vit.py:34,46-49) and the SimpleViT-family variants.
# `kind` = module name inside the reference package for the variants.
CASES2 = {
    "vit_tiny_noproj": dict(kind="vit", seed=4, batch=3, img=(32, 32),
                            kwargs=dict(image_size=32, patch_size=8, num_classes=7, dim=64, depth=2, heads=1,
                                        dim_head=64, mlp_dim=128)),
    "simplevit_registers": dict(kind="simple_vit_with_register_tokens", seed=6, batch=3, img=(32, 32),
                                kwargs=dict(image_size=32, patch_size=4, num_classes=10, dim=128, depth=2, heads=2,
                                            mlp_dim=256, num_register_tokens=4)),
    "simplevit_qknorm": dict(kind="simple_vit_with_qk_norm", seed=7, batch=3, img=(32, 32),
                             kwargs=dict(image_size=32, patch_size=4, num_classes=10, dim=128, depth=2, heads=2,
                                         mlp_dim=256)),
    "simplevit_patchdrop": dict(kind="simple_vit_with_patch_dropout", seed=8, batch=3, img=(32, 48),
                                kwargs=dict(image_size=64, patch_size=8, num_classes=10, dim=128, depth=2, heads=2,
                                            mlp_dim=256, patch_dropout=0.5)),
    "simplevit_flash": dict(kind="simple_flash_attn_vit", seed=9, batch=3, img=(48, 32),
                            kwargs=dict(image_size=64, patch_size=8, num_classes=10, dim=128, depth=2, heads=2,
                                        mlp_dim=256, use_flash=True)),
}


# Round 2, later: the 1-D / 3-D front-ends (series and video inputs; `img` = the non-channel dims)
CASES3 = {
    "simplevit_1d": dict(kind="simple_vit_1d", seed=12, batch=3, img=(256,),
                         kwargs=dict(seq_len=256, patch_size=16, num_classes=10, dim=128, depth=2, heads=2,
                                     mlp_dim=256)),
    "simplevit_3d": dict(kind="simple_vit_3d", seed=13, batch=2, img=(4, 32, 24),
                         kwargs=dict(image_size=(32, 24), image_patch_size=8, frames=4, frame_patch_size=2,
                                     num_classes=10, dim=128, depth=2, heads=2, mlp_dim=256)),
    "simplevit_3d_pf1": dict(kind="simple_vit_3d", seed=14, batch=2, img=(3, 32, 48),
                             kwargs=dict(image_size=(32, 48), image_patch_size=16, frames=3, frame_patch_size=1,
                                         num_classes=10, dim=192, depth=2, heads=3, mlp_dim=384)),
}


def reference_class(kind: str):
    """kind -> class of the UNMODIFIED reference."""
    import importlib
    if kind in ("vit", "simple"):
        return ViT if kind == "vit" else SimpleViT
    return importlib.import_module("vit_pytorch." + kind).SimpleViT


def make(name: str, spec: dict) -> None:
    torch.manual_seed(spec["seed"])
    cls = reference_class(spec["kind"])
    model = cls(**spec["kwargs"]).eval()
    # bf16-representable parameters; perturb LayerNorm affine params so gamma/beta are actually exercised
    g = torch.Generator().manual_seed(1000 + spec["seed"])
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.dim() == 1 and ("norm" in n or n.split(".")[-2] in ("0", "1", "3")) and n.endswith("weight"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1 and n.endswith("bias"):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
            elif n.endswith("gamma"):                       # per-head q / k RMSNorm scales
                p.mul_(1.0 + 0.2 * torch.randn(p.shape, generator=g))
            p.copy_(p.bfloat16().float())
    torch.manual_seed(100 + spec["seed"])
    img = torch.randn(spec["batch"], 3, *spec["img"]).bfloat16()
    with torch.inference_mode():
        logits = model(img.float())
        tokens = None
        if spec["kind"] == "vit":
            x = model.to_patch_embedding(img.float()[:1])
            x = torch.cat((model.cls_token[None], x), dim=1)
            x = x + model.pos_embedding[: x.shape[1]]
            tokens = model.transformer(x)
        model_bf16 = cls(**spec["kwargs"]).eval()
        model_bf16.load_state_dict(model.state_dict())
        model_bf16 = model_bf16.bfloat16()
        logits_bf16 = model_bf16(img)
    blob = {
        "name": name,
        "kind": spec["kind"],
        "kwargs": spec["kwargs"],
        "state_dict": {k: v.bfloat16() for k, v in model.state_dict().items()},
        "input": img,
        "logits_fp32": logits.clone(),
        "logits_ref_bf16": logits_bf16.float().clone(),
        "tokens_fp32": None if tokens is None else tokens.clone(),
        "versions": {"torch": str(torch.__version__), "reference": "vit-pytorch 1.23.6"},
    }
    path = os.path.join(HERE, name + ".pt")
    torch.save(blob, path)
    print(f"{name}: logits {tuple(logits.shape)} |max| {logits.abs().max():.4f}; "
          f"ref-bf16 max err {(logits_bf16.float() - logits).abs().max():.5f}; {os.path.getsize(path) / 1e6:.2f} MB")


def make_navit() -> None:
    """NaViT (reference na_vit.py): 7 images of 5 different resolutions, given as two pre-packed rows AND re-packed by
    the reference's own greedy grouping; fp32 logits of both calls are stored."""
    from vit_pytorch.na_vit import NaViT
    kwargs = dict(image_size=64, patch_size=8, num_classes=11, dim=128, depth=2, heads=2, mlp_dim=192, dim_head=64)
    torch.manual_seed(5)
    model = NaViT(**kwargs).eval()
    g = torch.Generator().manual_seed(1005)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if n.endswith("gamma"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            p.copy_(p.bfloat16().float())
    torch.manual_seed(105)
    sizes = [(64, 64), (32, 48), (16, 16), (64, 32), (24, 40), (8, 64), (48, 48)]
    imgs = [torch.randn(3, h, w).bfloat16() for h, w in sizes]
    rows = [[0, 1, 2], [3, 4, 5, 6]]
    with torch.inference_mode():
        packed = model([[imgs[i].float() for i in r] for r in rows])
        grouped = model([im.float() for im in imgs], group_images=True, group_max_seq_len=80)
    blob = {"name": "navit_tiny", "kind": "navit", "kwargs": kwargs,
            "state_dict": {k: v.bfloat16() for k, v in model.state_dict().items()},
            "images": imgs, "rows": rows, "group_max_seq_len": 80,
            "logits_fp32": packed.clone(), "logits_grouped_fp32": grouped.clone(),
            "versions": {"torch": str(torch.__version__), "reference": "vit-pytorch 1.23.6"}}
    path = os.path.join(HERE, "navit_tiny.pt")
    torch.save(blob, path)
    print(f"navit_tiny: logits {tuple(packed.shape)} |max| {packed.abs().max():.4f}; packed vs grouped "
          f"{(packed - grouped).abs().max():.2e}; {os.path.getsize(path) / 1e6:.2f} MB")


from navit_c5_spec import NAVIT_C5, navit_config5_images, navit_config5_model  # noqa: E402  (tests/golden/)


def make_navit_config5() -> None:
    from vit_pytorch.na_vit import NaViT
    model = navit_config5_model(NaViT)
    imgs = navit_config5_images()
    with torch.inference_mode():
        fp32 = model([im.float() for im in imgs], group_images=True, group_max_seq_len=4096)
        bf16 = model.bfloat16()([im for im in imgs], group_images=True, group_max_seq_len=4096)
    d = (bf16.float() - fp32).abs()
    floor = {"max": d.max().item(), "mean": d.mean().item(),
             "frac_within_tol": (d <= 1e-3 + 1e-2 * fp32.abs()).float().mean().item()}
    blob = {"name": "navit_config5", "kind": "navit", "spec": NAVIT_C5, "logits_fp32": fp32.clone(),
            "logits_ref_bf16": bf16.clone(), "ref_bf16_floor": floor,
            "versions": {"torch": str(torch.__version__), "reference": "vit-pytorch 1.23.6"}}
    path = os.path.join(HERE, "navit_config5.pt")
    torch.save(blob, path)
    print(f"navit_config5: logits {tuple(fp32.shape)} |max| {fp32.abs().max():.4f}; reference-bf16 floor {floor}; "
          f"{os.path.getsize(path) / 1e6:.2f} MB")


def make_navit_nested() -> None:
    """Nested-tensor NaViT (reference na_vit_nested_tensor.py): 6 images of 5 resolutions, with and without the q / k
    LayerNorm.  The reference runs its jagged-batch forward (torch.nested + SDPA) on CPU."""
    from vit_pytorch.na_vit_nested_tensor import NaViT
    for name, qk in (("navit_nested_tiny", True), ("navit_nested_noqknorm", False)):
        kwargs = dict(image_size=64, patch_size=8, num_classes=11, dim=128, depth=2, heads=2, mlp_dim=192, dim_head=64,
                      qk_rmsnorm=qk)
        torch.manual_seed(11)
        model = NaViT(**kwargs).eval()
        g = torch.Generator().manual_seed(1011)
        with torch.no_grad():
            for n, p in model.named_parameters():
                if p.dim() == 1 and n.endswith("weight"):               # every LayerNorm scale (incl. the per-head ones)
                    p.add_(0.1 * torch.randn(p.shape, generator=g))
                elif p.dim() == 1 and n.endswith("bias"):
                    p.add_(0.05 * torch.randn(p.shape, generator=g))
                p.copy_(p.bfloat16().float())
        torch.manual_seed(111)
        sizes = [(64, 64), (32, 48), (8, 8), (64, 16), (24, 40), (48, 48)]
        imgs = [torch.randn(3, h, w).bfloat16() for h, w in sizes]
        with torch.inference_mode():
            fp32 = model([im.float() for im in imgs])
            bf16 = model.bfloat16()([im for im in imgs])
        blob = {"name": name, "kind": "navit_nested", "kwargs": kwargs,
                "state_dict": {k: v.bfloat16() for k, v in model.state_dict().items()}, "images": imgs,
                "logits_fp32": fp32.clone(), "logits_ref_bf16": bf16.float().clone(),
                "versions": {"torch": str(torch.__version__), "reference": "vit-pytorch 1.23.6"}}
        path = os.path.join(HERE, name + ".pt")
        torch.save(blob, path)
        print(f"{name}: logits {tuple(fp32.shape)} |max| {fp32.abs().max():.4f}; ref-bf16 max err "
              f"{(bf16.float() - fp32).abs().max():.5f}; {os.path.getsize(path) / 1e6:.2f} MB")


def state_digest(sd) -> dict:
    """sha256 of every tensor's bytes: bit-identical initialisation is checked without storing the weights."""
    import hashlib
    return {k: (tuple(v.shape), str(v.dtype), hashlib.sha256(v.detach().contiguous().cpu().numpy().tobytes()).hexdigest())
            for k, v in sd.items()}


def signature(cls) -> list:
    import inspect
    return [(k, repr(v.default)) for k, v in inspect.signature(cls.__init__).parameters.items() if k != "self"]


def make_reference_live():
    """tests/golden/reference_live.pt: what the tests used to read off a live reference checkout -- same-seed
    initialisations (as digests), constructor signatures, reference logits of seeded models and inputs, and the
    reference Recorder's attention maps."""
    import importlib
    ref = importlib.import_module("vit_pytorch")
    out = {"init": {}, "signature": {}, "logits": {}, "versions": {"torch": str(torch.__version__),
                                                                    "reference": "vit-pytorch 1.23.6"}}
    kw = dict(image_size=32, patch_size=8, num_classes=5, dim=64, depth=2, heads=2, mlp_dim=96, dim_head=32)
    for kind, cls in (("vit", ref.ViT), ("simple", ref.SimpleViT)):
        torch.manual_seed(123)
        m = cls(**kw)
        out["init"][f"dropin_{kind}"] = state_digest(m.state_dict())
        if kind == "simple":
            out["init"]["dropin_simple_pos"] = state_digest({"pos_embedding": m.pos_embedding})
    # SimpleViT-family variants and the nested-tensor NaViT (tests/test_variants.py)
    for name, spec in {**CASES2, **CASES3}.items():
        if spec["kind"] == "vit":
            continue
        cls = importlib.import_module("vit_pytorch." + spec["kind"]).SimpleViT
        out["signature"][name] = signature(cls)
        torch.manual_seed(123)
        out["init"][name] = state_digest(cls(**spec["kwargs"]).state_dict())
    nested = importlib.import_module("vit_pytorch.na_vit_nested_tensor").NaViT
    out["signature"]["navit_nested"] = signature(nested)
    torch.manual_seed(5)
    out["init"]["navit_nested"] = state_digest(nested(image_size=32, patch_size=8, num_classes=5, dim=64, depth=1,
                                                      heads=1, mlp_dim=64).state_dict())
    # NaViT: init and forward on three images in two groups (tests/test_navit.py)
    navit = importlib.import_module("vit_pytorch.na_vit").NaViT
    nkw = dict(image_size=32, patch_size=8, num_classes=5, dim=64, depth=1, heads=2, mlp_dim=96, dim_head=32)
    torch.manual_seed(9)
    a = navit(**nkw).eval()
    out["init"]["navit"] = state_digest(a.state_dict())
    imgs = [torch.randn(3, 32, 16), torch.randn(3, 8, 8), torch.randn(3, 24, 32)]
    with torch.inference_mode():
        out["logits"]["navit"] = {"logits": a([imgs[:2], imgs[2:]])}
    # seeded reference forwards (tests/test_oracle.py): model under seed, then the input from the global generator
    for kind, seed in (("vit", 11), ("simple", 12), ("vit", 13)):
        torch.manual_seed(seed)
        okw = dict(image_size=64, patch_size=16, num_classes=17, dim=128, depth=2, heads=2, mlp_dim=192)
        if kind == "vit" and seed == 13:
            okw["pool"] = "mean"
        model = (ref.ViT if kind == "vit" else ref.SimpleViT)(**okw).eval()
        out["init"][f"oracle_{kind}_{seed}"] = state_digest(model.state_dict())
        img = torch.randn(3, 3, 64, 64)
        with torch.inference_mode():
            out["logits"][f"oracle_{kind}_{seed}"] = {"logits": model(img)}
    torch.manual_seed(0)
    bkw = dict(image_size=224, patch_size=16, num_classes=1000, dim=768, depth=12, heads=12, mlp_dim=3072)
    model = ref.ViT(**bkw).eval()
    out["init"]["oracle_vit_b16"] = state_digest(model.state_dict())
    torch.manual_seed(1)
    img = torch.randn(1, 3, 224, 224)
    with torch.inference_mode():
        out["logits"]["oracle_vit_b16"] = {"logits": model(img)}
    # the reference Recorder's attention maps (tests/test_dropin.py::test_recorder_and_extractor_twins)
    Recorder = importlib.import_module("vit_pytorch.recorder").Recorder
    torch.manual_seed(0)
    r = ref.ViT(image_size=32, patch_size=8, num_classes=3, dim=32, depth=2, heads=2, mlp_dim=48, dim_head=16).eval()
    out["init"]["recorder_vit"] = state_digest(r.state_dict())
    img = torch.randn(2, 3, 32, 32)
    with torch.no_grad():
        out["logits"]["recorder"] = {"attns": Recorder(r)(img)[1]}
    path = os.path.join(HERE, "reference_live.pt")
    torch.save(out, path)
    print(f"reference_live: {os.path.getsize(path) / 1e3:.1f} kB")


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "reference_live":
        make_reference_live()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "navit_nested":
        make_navit_nested()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "navit_config5":
        make_navit_config5()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "frontends":
        for n, s in CASES3.items():
            make(n, s)
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "round2":
        for n, s in CASES2.items():
            make(n, s)
        sys.exit(0)
    for n, s in {**CASES, **CASES2, **CASES3}.items():
        make(n, s)
    make_navit()
    make_navit_config5()
    make_navit_nested()
