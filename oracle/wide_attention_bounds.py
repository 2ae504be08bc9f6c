"""fp64 reference with a per-element error bound for b200vit_attention_wide (csrc/t2t.cu): the attention of one head
as wide as the token that materialises its scores  --  TEST INFRASTRUCTURE.

`wide_attention_reference` returns `(ref, bound)`, fp64 tensors of the kernel output's shape on the inputs' device, to
be checked with oracle.bounds.check.  It takes the kernel's own bf16 q, k and v, so the bound counts only the rounding
the kernel does.  Notation as in oracle/bounds.py: u = 2^-24.

The kernel runs three steps per image; the reference replays the one rounding that matters, P to bf16:
  - S.  s_j = fl(acc_j * scale), acc_j the fp32 accumulation of dp bf16 products (wgmma k16 steps):
    |ds_j| <= C_WIDE dp u scale sum|q||k| + u |s_j|.  C_WIDE = 1 is the worst case of a sequential fp32 sum, with no
    measured constant in it.
  - Softmax.  The kernel's max m~ is the max of its own s~, within dm = max_j |ds_j| of m.  e~_j = expf(s~_j - m~):
    the subtraction rounds (u |s_j - m|) and expf has a relative error EXP_REL, so
    e~_j in e_j [exp(-d_j), exp(d_j)],  d_j = |ds_j| + dm + u |s_j - m| + EXP_REL.
    l~ = the fp32 sum of the e~_j (32 lanes of n / 32 adds, then a 5-level shuffle tree):
    l~ in l [exp(-dl), exp(dl)],  dl = max_j d_j + (n / 32 + 6) u.
    P'_j = bf16(fl(e~_j fl(1 / l~))) before its rounding lies in P_j [exp(-t_j), exp(t_j)], t_j = d_j + dl + 2u,
    with P_j = e_j / l exact.  bf16 rounding is monotone, so the kernel's probability lies in [bf16(lo_j), bf16(hi_j)],
    and the reference takes bf16(P_j):  |P'_j - bf16(P_j)| <= A_j = max(bf16(hi_j) - bf16(P_j), bf16(P_j) - bf16(lo_j)).
  - P V.  The bf16 products are exact; the fp32 accumulation over the n keys (padded to a multiple of 32 with zeros)
    adds C_WIDE n u sum_j (bf16(P_j) + A_j) |v_j|.
  - Output.  bf16 rounding of a value within E of ref: bound = E + ulp_bf16(|ref| + E) / 2, E = sum_j A_j |v_j| + the
    accumulation term.
"""
from __future__ import annotations

from typing import Tuple

import torch

from oracle.bounds import U, bf16_ulp

Tensor = torch.Tensor

C_WIDE = 1.0
# expf: CUDA documents a maximum error of 2 ulp (CUDA C++ Programming Guide, mathematical functions); 4 ulp here.
EXP_REL = 2.0 ** -21


def _bf16(x: Tensor) -> Tensor:
    return x.to(torch.bfloat16).double()


def wide_attention_reference(q: Tensor, k: Tensor, v: Tensor, scale: float) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [G, n, dp] of the attention of G images of n tokens, q, k, v: [G, n, dp] bf16, one head."""
    G, n, dp = q.shape
    q64, k64, v64 = q.double(), k.double(), v.double()
    sc = float(torch.tensor(scale, dtype=torch.float32).item())
    s = (q64 @ k64.transpose(1, 2)) * sc
    ds = C_WIDE * dp * U * sc * (q64.abs() @ k64.abs().transpose(1, 2)) + U * s.abs()
    m = s.amax(-1, keepdim=True)
    dm = ds.amax(-1, keepdim=True)
    e = torch.exp(s - m)
    p = e / e.sum(-1, keepdim=True)
    d = ds + dm + U * (s - m).abs() + EXP_REL
    dl = d.amax(-1, keepdim=True) + (n / 32 + 6) * U
    t = d + dl + 2 * U
    pb = _bf16(p)
    amb = torch.maximum(_bf16(p * torch.exp(t)) - pb, pb - _bf16(p * torch.exp(-t)))
    vabs = v64.abs()
    ref = pb @ v64
    err = amb @ vabs + C_WIDE * (-(-n // 32) * 32) * U * ((pb + amb) @ vabs)
    return ref, err + 0.5 * bf16_ulp(ref.abs() + err)


def qkv_wide_reference(qkv: Tensor, B: int, n: int, dp: int, scale: float) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [B n, dp] of b200vit_attention_wide over qkv[B n, 3 dp] (image b at rows b n ..)."""
    x = qkv.view(B, n, 3, dp)
    ref, bound = wide_attention_reference(x[:, :, 0], x[:, :, 1], x[:, :, 2], scale)
    return ref.reshape(B * n, dp), bound.reshape(B * n, dp)


def wide_inputs(B: int, n: int, w: int, dp: int, *, seed: int = 0, qk_std: float = 1.0, device="cpu") -> Tensor:
    """Seeded packed q | k | v [B n, 3 dp] bf16, N(0, 1) on the first w columns of each of q, k, v (q and k times
    qk_std) and zero on the padding to dp, as a soft split's zero-padded projection writes it."""
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.zeros(B * n, 3, dp, device=device)
    x[:, :, :w] = torch.randn(B * n, 3, w, generator=g, device=device)
    x[:, :2, :w] *= qk_std
    return x.view(B * n, 3 * dp).bfloat16()
