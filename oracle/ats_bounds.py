"""fp64 references of Adaptive Token Sampling's kernels (b200vit_ats_select, b200vit_ats_gather,
b200vit_attention_kv_lens)  --  TEST INFRASTRUCTURE.

select_reference: per image, in fp64 on the kernel's own bf16 qkv and uniforms, the pseudo-logits of the reference
(ats_vit.py:51-75) plus the Gumbel noise, the argmax of every draw, its top-2 gap, and a per-candidate bound on how far
the kernel's fp32 arithmetic can move a candidate's value.  A draw whose gap exceeds twice the bound must be the fp64
argmax; inside it, any candidate within twice the bound of the maximum is a valid outcome.

select_outputs: the row map, lengths and ids as an exact function of the draws (torch.unique + pad_sequence + F.pad,
ats_vit.py:91-103), so the kernel's outputs can be checked bit for bit against its own draws.

kv_lens_reference: the attention of each image's queries over its first nk[b] keys, with the per-element bounds of
oracle/attention_bounds.py (the keys past nk[b] masked, as the kernel's 64-key blocks see them)."""
from __future__ import annotations

import math
from typing import List, Sequence, Tuple

import torch

from oracle import attention_bounds as AB

Tensor = torch.Tensor
EPS = 1e-6
U32 = 2.0 ** -24


def _f32(v: float) -> float:
    return torch.tensor(v, dtype=torch.float32).item()


def select_reference(qkv: Tensor, lens: Sequence[int], u: Tensor, B: int, S: int, K: int, H: int, dh: int,
                     scale: float) -> dict:
    """fp64 values of every draw of a sampling layer: 'logit' [B, S - 1] the pseudo-logits alone, 'value' [B, K, S - 1]
    (-inf past each image's candidates),
    'bound' [B, K, S - 1], 'argmax' [B, K], 'gap' [B, K] (the winner minus the runner-up, inf with one candidate)."""
    q = qkv.double().view(B, S, 3, H, dh)
    value = torch.full((B, K, S - 1), -math.inf, dtype=torch.float64)
    logits = torch.full((B, S - 1), -math.inf, dtype=torch.float64)
    bound = torch.zeros(B, K, S - 1, dtype=torch.float64)
    sc = _f32(scale)
    for b in range(B):
        L = int(lens[b])
        qc, k, v = q[b, 0, 0], q[b, :L, 1], q[b, :L, 2]                  # [H, dh], [L, H, dh] x 2
        dots = torch.einsum('hd,jhd->hj', qc, k) * sc
        p = torch.softmax(dots, dim=-1)
        vn = v.norm(dim=-1).t()                                          # [H, L]
        s = (p[:, 1:] * vn[:, 1:]).sum(0)                                # [L - 1]
        logit = torch.log(s / (s.sum() + EPS) + EPS)
        # fp32 arithmetic of the kernel: the dot products (dh terms), exp, the head sum and the normalisation
        # move s by a relative error of a few hundred U32 at most; log turns that into an absolute error
        dabs = torch.einsum('hd,jhd->hj', qc.abs(), k.abs()) * sc
        rel = (2 * dh + 64 + 4 * H) * U32 + (dabs.amax() * (dh + 8) * U32) * 4
        lb = (rel * s / (s + (s.sum() + EPS) * EPS)) + 8 * U32 * (1 + logit.abs())
        ub = u[b, :, :L - 1].double()
        inner = -torch.log(ub + EPS) + EPS
        g = -torch.log(inner)
        # u + eps, the inner log and the outer log each round once in fp32
        gb = (4 * U32 * (1 + ub) / (ub + EPS) / inner.clamp_min(1e-30)) + 4 * U32 * (1 + g.abs())
        value[b, :, :L - 1] = logit[None] + g
        logits[b, :L - 1] = logit
        bound[b, :, :L - 1] = lb[None] + gb
    top = value.topk(min(2, S - 1), dim=-1)
    gap = top.values[..., 0] - top.values[..., 1] if S > 2 else torch.full((B, K), math.inf, dtype=torch.float64)
    gap = torch.where(torch.isnan(gap), torch.full_like(gap, math.inf), gap)
    return {"value": value, "bound": bound, "argmax": value.argmax(-1), "gap": gap, "logit": logits}


def allowed_draws(ref: dict) -> Tensor:
    """bool [B, K, S - 1]: the candidates a draw may land on -- the fp64 argmax where its gap exceeds twice the
    bound, else every candidate within twice the bound of the maximum."""
    v, bd = ref["value"], ref["bound"]
    m = v.amax(-1, keepdim=True)
    slack = 2 * bd.amax(-1, keepdim=True)
    return v >= m - slack


def select_outputs(draws: Tensor, lens: Sequence[int], ids: Tensor, B: int, S_in: int, K: int
                   ) -> Tuple[Tensor, Tensor, Tensor, bool]:
    """(src int32 [B*S_out], lens_out int32 [B], ids_out int32 [B*S_out], sampled) of draws [B, K] (candidate c is row
    c + 1), as b200vit_ats_select defines them; without sampling the identity map, whatever draws holds."""
    S_out = min(S_in, K + 1)
    ids = ids.view(B, S_in)
    sampled = max(int(v) for v in lens) - 1 > K
    src = torch.empty(B, S_out, dtype=torch.int32)
    lo = torch.empty(B, dtype=torch.int32)
    io = torch.empty(B, S_out, dtype=torch.int32)
    for b in range(B):
        L = int(lens[b])
        if sampled:
            pos = [0] + sorted(set(int(c) + 1 for c in draws[b]))
        else:
            pos = list(range(L))
        pos = pos + [0] * (S_out - len(pos))
        src[b] = torch.tensor(pos, dtype=torch.int32) + b * S_in
        io[b] = ids[b, torch.tensor(pos)]
        lo[b] = L if not sampled else len(set(int(c) for c in draws[b])) + 1
    return src.view(-1), lo, io.view(-1), sampled


def kv_lens_reference(q: Tensor, kv: Tensor, nk: Sequence[int], B: int, Nq: int, Nk: int, H: int, dh: int,
                      scale: float) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [B*Nq, H*dh] of b200vit_attention_kv_lens: q [B*Nq, H*dh], kv [B*Nk, 2*H*dh] (bf16)."""
    I = H * dh
    ref = torch.empty(B * Nq, I, dtype=torch.float64)
    bound = torch.empty_like(ref)
    n = max(Nq, Nk)
    for b in range(B):
        c = min(max(int(nk[b]), 1), Nk)
        qb = torch.zeros(n, H, dh, dtype=q.dtype)
        qb[:Nq] = q[b * Nq:(b + 1) * Nq].view(Nq, H, dh)
        kb = torch.zeros(n, H, dh, dtype=kv.dtype)
        vb = torch.zeros(n, H, dh, dtype=kv.dtype)
        kb[:c] = kv[b * Nk:b * Nk + c, :I].view(c, H, dh)
        vb[:c] = kv[b * Nk:b * Nk + c, I:].view(c, H, dh)
        mask = torch.zeros(H, n, dtype=torch.bool)
        mask[:, :c] = True
        r, e = AB.attention_reference(qb.transpose(0, 1), kb.transpose(0, 1), vb.transpose(0, 1), scale, key_mask=mask)
        ref[b * Nq:(b + 1) * Nq] = r[:, :Nq].transpose(0, 1).reshape(Nq, I)
        bound[b * Nq:(b + 1) * Nq] = e[:, :Nq].transpose(0, 1).reshape(Nq, I)
    return ref, bound


def emulate_select(qkv: Tensor, lens: Tensor, ids: Tensor, u: Tensor, B: int, S_in: int, K: int, H: int, dh: int,
                   scale: float) -> Tuple[Tensor, Tensor, Tensor]:
    """b200vit_ats_select emulated on CPU: the fp64 argmax of every draw, then select_outputs."""
    lens_l: List[int] = [int(v) for v in lens.cpu()]
    if max(lens_l) - 1 > K:
        draws = select_reference(qkv.cpu(), lens_l, u.cpu(), B, S_in, K, H, dh, scale)["argmax"]
    else:
        draws = torch.zeros(B, K, dtype=torch.long)
    src, lo, io, _ = select_outputs(draws, lens_l, ids.cpu(), B, S_in, K)
    return src, lo, io
