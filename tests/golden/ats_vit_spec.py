"""Adaptive Token Sampling ViT parity cases (reference ats_vit.py), on the shared recipe of parity.py.

Besides the logits, a case stores what its seeded forward drew and kept, recorded by a pass-through wrapper of the
module's `sample_gumbel` (`recorded_forward`): the uniforms of every sampling layer, the returned token ids, every
layer's padded length, and the smallest Gumbel-max margin (winner minus runner-up, in the graph's fp32) over all
draws.  Every case's noise seed was chosen so that this margin is at least MARGIN, so a bf16 forward whose
pseudo-logits stay within MARGIN / 2 of the fp32 graph's draws the same tokens; the GPU tests hold the fused path to
that."""
import sys

import torch

from parity import Family

BASE = dict(num_classes=7, dim=64, depth=6, max_tokens_per_depth=(256, 128, 64, 32, 16, 8), heads=2, mlp_dim=128,
            dim_head=32, channels=3, dropout=0., emb_dropout=0.)
BATCH = 2
MARGIN = 0.05
# constructor keywords on top of BASE; `input` = (height, width) of the image, `batch` its batch size (default BATCH);
# `noise_seed` seeds torch's generator right before every forward.  The comments give the token counts per layer.
ATS_CASES = {
    # the README's max_tokens_per_depth at a smaller width: 64 patches, layers 3, 4 and 5 sample (K = 32, 16, 8)
    "readme": dict(seed=501, noise_seed=326, image_size=64, patch_size=8, input=(64, 64)),
    # layer 0 keeps at most 9 of 65 rows; layer 1 (K = 7) could sample but every image kept <= 8 rows: it stays off
    "stays_off": dict(seed=502, noise_seed=13, image_size=64, patch_size=8, depth=3, max_tokens_per_depth=(8, 7, 3),
                      input=(64, 64)),
    # three images ending with different counts: padding rows and -1 ids
    "ragged": dict(seed=503, noise_seed=13, image_size=32, patch_size=8, depth=2, max_tokens_per_depth=(12, 10),
                   batch=3, input=(32, 32)),
    # no layer samples: every K is at least the 16 patches
    "no_sampling": dict(seed=504, noise_seed=14, image_size=32, patch_size=8, depth=2, max_tokens_per_depth=(64, 16),
                        input=(32, 32)),
    # heads 80 wide
    "dh80": dict(seed=505, noise_seed=16, image_size=32, patch_size=8, dim=160, heads=2, dim_head=80, mlp_dim=160,
                 depth=2, max_tokens_per_depth=(8, 4), input=(32, 32)),
    # an input smaller than image_size: the first n + 1 rows of the positional table (16 patches of 64)
    "smaller_input": dict(seed=506, noise_seed=16, image_size=64, patch_size=8, depth=2, max_tokens_per_depth=(10, 5),
                          input=(32, 32)),
    # heads 16 wide: no attention kernel is built for them, the PyTorch graph runs
    "fallback_dh16": dict(seed=507, noise_seed=24, image_size=32, patch_size=8, heads=4, dim_head=16, depth=2,
                          max_tokens_per_depth=(8, 4), input=(32, 32)),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 521
INIT_KWARGS = dict(BASE, image_size=32, patch_size=8)

_SPEC_KEYS = ("seed", "noise_seed", "input", "batch")


def case_kwargs(spec: dict) -> dict:
    kw = dict(BASE)
    kw.update({k: v for k, v in spec.items() if k not in _SPEC_KEYS})
    return kw


def before_forward(spec: dict) -> None:
    torch.manual_seed(spec["noise_seed"])


def recorded_forward(model, x: torch.Tensor, spec: dict) -> dict:
    """A seeded forward with return_sampled_token_ids=True, through a pass-through wrapper of the model module's
    sample_gumbel that draws exactly as it does and returns the same value: the fields the fixture stores."""
    mod = sys.modules[type(model).__module__]
    original = mod.sample_gumbel
    rec = {"uniforms": {}, "padded_lengths": [], "margin": float("inf")}
    state = {}

    def pre_attention(i):
        def hook(m, args, kwargs):
            rec["padded_lengths"].append(args[0].shape[1])
            state["layer"] = i
        return hook

    def pre_ats(m, args, kwargs):
        attn, value = args[0], args[1]
        mask = kwargs["mask"]
        scores = torch.einsum('b h n, b h n -> b n', attn[..., 0, 1:], value[..., 1:, :].norm(dim=-1))
        logits = torch.log(scores / (scores.sum(dim=-1, keepdim=True) + m.eps) + m.eps)
        state["logits"] = logits.masked_fill(~mask[:, 1:], -float("inf"))

    def recorder(shape, device, dtype, eps=1e-6):
        u = torch.empty(shape, device=device, dtype=dtype).uniform_(0, 1)
        g = -torch.log(-torch.log(u + eps) + eps)
        rec["uniforms"][f"layer{state['layer']}"] = u.clone()
        v = (state["logits"].unsqueeze(1) + g).float()
        top = v.topk(2, dim=-1).values if v.shape[-1] > 1 else None
        if top is not None:
            rec["margin"] = min(rec["margin"], float((top[..., 0] - top[..., 1]).min()))
        return g

    handles = []
    for i, (attn, _) in enumerate(model.transformer.layers):
        handles.append(attn.register_forward_pre_hook(pre_attention(i), with_kwargs=True))
        if attn.ats is not None:
            handles.append(attn.ats.register_forward_pre_hook(pre_ats, with_kwargs=True))
    mod.sample_gumbel = recorder
    try:
        before_forward(spec)
        logits, ids = model(x.float(), return_sampled_token_ids=True)
    finally:
        mod.sample_gumbel = original
        for h in handles:
            h.remove()
    return {"logits_sampled": logits.clone(), "token_ids": ids.clone(), "uniforms": rec["uniforms"],
            "padded_lengths": rec["padded_lengths"], "margin": rec["margin"]}


FAMILY = Family(
    name="ats_vit", model="ats_vit.ViT", cases=ATS_CASES, case_kwargs=case_kwargs,
    input_shape=lambda spec: (spec.get("batch", BATCH), case_kwargs(spec)["channels"], *spec["input"]),
    init_seed=INIT_SEED, init={None: INIT_KWARGS}, before_forward=before_forward,
    embed=recorded_forward)
