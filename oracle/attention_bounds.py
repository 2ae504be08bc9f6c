"""fp64 references with a per-element error bound for the softmax attention kernels of attention.cu
(b200vit_attention / _ex, b200vit_attention_varlen / _ex)  --  TEST INFRASTRUCTURE.

Every function returns `(ref, bound)`: fp64 tensors of the kernel output's shape, on the device of the inputs, to be
checked with oracle.bounds.check.  The reference takes the kernel's own bf16 q, k and v, so the bound counts only the
rounding the kernel does.  Notation as in oracle/bounds.py: u = 2^-24, C_ACC the wgmma accumulation constant.

The kernel rounds the probabilities to bf16 before P V on purpose, and that rounding (up to 2^-8 relative per key) is
far larger than all of its fp32 noise.  A bound that treated it as an independent error per key would be loose enough
to let a 1 % error through, so the reference replays it: per query row i,
  - the keys go in blocks of KB = 64 counted from the sequence start; x_j = s_j c with c = scale log2(e) (log2
    units), masked keys (past the sequence, and the row's own key under MASK_SELF unless the sequence has one token)
    x_j = -inf;
  - m_b = the max of x over blocks 0..b (the running max after block b), e_j = 2^(x_j - m_b(j)), P_j = bf16(e_j);
  - O and l are rescaled by corr = 2^(m_old - m_new) when the max rises.  corr multiplies O and l alike, so its ex2
    error cancels in O / l; relative to the final max M every key weighs W_j = P_j 2^(m_b(j) - M), and
    ref = sum_j W_j v_j / l,  l = sum_j e_j 2^(m_b(j) - M).

What the kernel can do differently from that replay, and the bound of each:
  - Score.  wgmma computes s_j within ds_j = (C_ACC dh + 2) u sum|q||k|; x_j = fl(s_j c) with c rounded twice in fp32
    (scale log2e, the product): dx_j = c ds_j + 4 u |x_j|.
  - Max.  The kernel's m_b is the max of its own x, within dm_b = max dx over the keys of blocks 0..b of m_b.  Scaling
    e's block by f = 2^(m_b - m~_b) changes nothing after corr except where the bf16 grid falls: the kernel weighs key j
    with P'_j / f, P'_j = bf16(e_j f g_j).
  - exp2.  x~_j - m~_b is rounded in fp32 (u |x_j - m_b|), and ex2.approx.ftz.f32 has a relative error EX2_REL.  So
    e_j f g_j lies in [lo_j, hi_j] = e_j [2^-d_j (1 - EX2_REL), 2^d_j (1 + EX2_REL)]
    with d_j = dx_j + dm_b + u |x_j - m_b|; lo_j = 0 where it falls below 2^-126 (ftz).
  - Ambiguous roundings.  bf16 rounding is monotone, so P'_j lies in [bf16(lo_j), bf16(hi_j)], and
    |P'_j / f - P_j| <= A_j = max(bf16(hi_j) - P_j, P_j - bf16(lo_j)) 2^dm_b + P_j (2^dm_b - 1).  A_j is 0 up to the
    fp32 noise for every key whose interval lies within one bf16 rounding interval, and an ulp of P_j for the few
    keys whose interval straddles a rounding boundary.
  - P V.  The bf16 products are exact; the chain of len fp32 accumulations gives (C_ACC len + 2) u sum_j W_j |v_j|,
    and each of the nblocks rescales of O adds u sum_j W_j |v_j|.
  - l.  Each thread adds its keys (a quarter of them, two per add) in fp32, rescales per block and joins a 2-level
    shuffle tree: (len / 4 + 2 nblocks + 4) u l, plus the uncertainty of the unrounded e: sum_j 2^(m_b - M)
    max(hi_j - e_j, e_j - lo_j).  Relative: eta = dl / l.
  - ftz of corr.  A whole earlier block drops out when 2^(m_old - m_new) < 2^-126: at most len 2^-126 max|v| in the
    numerator and len 2^-126 in l (negligible, kept for completeness).
  - Output.  y = fl(O fl(1 / l)) with IEEE division: with E_num the numerator's bound above,
        E32 = (E_num / l + |ref| eta) / (1 - eta) + 3 u (|ref| + E32),
    and the bf16 rounding of a value within E32 of ref is within half an ulp of |ref| + E32:
        bound = E32 + ulp_bf16(|ref| + E32) / 2.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence, Tuple

import torch

from oracle.bounds import C_ACC, U, bf16_ulp

Tensor = torch.Tensor

LOG2E = 1.4426950408889634
# ex2.approx.ftz.f32: NVIDIA documents a maximum error of 2 ulp over the full range (PTX ISA, ex2; CUDA C++
# Programming Guide, exp2f); EX2_REL = 2^-21 is 4 ulp of fp32.  Against the 2^-8 rounding of P the constant is
# irrelevant, so it is generous rather than exact.
EX2_REL = 2.0 ** -21
FTZ = 2.0 ** -126           # smallest normal fp32: ex2.approx.ftz flushes results below it to 0
KB = 64                     # keys per block of attention.cu


def scale_log2e(scale: float) -> float:
    """The kernel's fp32 scale * log2(e): the scale rounded to fp32 (the C ABI takes a float), times fp32 log2(e)."""
    return (torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)).item()


def _bf16(x: Tensor) -> Tensor:
    """fp64 -> the bf16 rounding of its fp32 value (the kernel rounds fp32 e to bf16)."""
    return x.float().bfloat16().double()


def attention_reference(q: Tensor, k: Tensor, v: Tensor, scale: float, *, mask_self: bool = False,
                        key_mask: Optional[Tensor] = None, zero_masked_rows: bool = False,
                        elems: int = 1 << 23) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [G, n, dh] of the attention of G independent sequences of n tokens, q, k, v: [G, n, dh] bf16.

    mask_self: each query's own key is excluded (n > 1); key_mask: None or bool [G, n] (True = keep), the masked keys
    -inf.  A sequence with no kept key gets exactly 0 under zero_masked_rows, else every key at weight 1: the kernel's
    P = 1 and l = n are exact, so its reference is the mean of the values with the P V and O fl(1 / l) terms alone.
    Query rows go in chunks of at most `elems` scores, so 16384-key sequences fit."""
    G, n, dh = q.shape
    dev = q.device
    k64, v64 = k.double(), v.double()
    kabs, vabs = k64.abs(), v64.abs()
    vmax = vabs.amax(dim=(1, 2))[:, None, None]
    nb = -(-n // KB)
    c = float(torch.tensor(scale, dtype=torch.float32).item()) * LOG2E
    key = torch.arange(n, device=dev)
    blk = key // KB
    rel = torch.full((n,), EX2_REL, dtype=torch.float64, device=dev)
    empty = None
    if key_mask is not None:
        km = key_mask.to(device=dev, dtype=torch.bool)
        empty = ~km.any(-1)[:, None, None]                              # [G, 1, 1]: no kept key
        rel = torch.where(empty, torch.zeros_like(rel), rel)             # [G, 1, n]: P = 1 exactly there
    ref = torch.empty(G, n, dh, dtype=torch.float64, device=dev)
    bound = torch.empty_like(ref)
    rows = max(1, min(n, elems // max(1, G * n)))
    for r0 in range(0, n, rows):
        r1 = min(n, r0 + rows)
        q64 = q[:, r0:r1].double()
        x = (q64 @ k64.transpose(1, 2)) * c
        dx = c * (C_ACC * dh + 2) * U * (q64.abs() @ kabs.transpose(1, 2)) + 4 * U * x.abs()
        valid = torch.ones(r1 - r0, n, dtype=torch.bool, device=dev)
        if mask_self and n > 1:
            qi = torch.arange(r0, r1, device=dev)
            valid = qi[:, None] != key[None, :]
        valid = valid.expand(G, -1, -1)
        if key_mask is not None:
            valid = (valid & km[:, None, :]) | empty
            x = torch.where(empty, torch.zeros_like(x), x)
            dx = torch.where(empty, torch.zeros_like(dx), dx)
        x = torch.where(valid, x, torch.full_like(x, -math.inf))
        dx = torch.where(valid, dx, torch.zeros_like(dx))
        pad = nb * KB - n
        xp = torch.nn.functional.pad(x, (0, pad), value=-math.inf).view(G, r1 - r0, nb, KB)
        dxp = torch.nn.functional.pad(dx, (0, pad)).view(G, r1 - r0, nb, KB)
        mb = xp.amax(-1).cummax(-1).values           # running max after each block
        dmb = dxp.amax(-1).cummax(-1).values
        m, dm = mb[..., blk], dmb[..., blk]
        t = torch.where(valid, x - m, torch.zeros_like(x))
        e = torch.where(valid, torch.exp2(t), torch.zeros_like(x))
        d = torch.where(valid, dx + dm + U * t.abs(), torch.zeros_like(x))
        hi = e * torch.exp2(d) * (1 + rel)
        lo = e * torch.exp2(-d) * (1 - rel)
        lo = torch.where(lo < FTZ, torch.zeros_like(lo), lo)
        p = _bf16(e)
        fm = torch.exp2(dm)
        amb = torch.maximum(_bf16(hi) - p, p - _bf16(lo)) * fm + p * (fm - 1)
        sc = torch.exp2(m - mb[..., -1:])          # 2^(m_b - M); masked keys have e = p = 0
        w = p * sc
        l = (e * sc).sum(-1, keepdim=True)
        out = (w @ v64) / l
        e_num = (amb * sc) @ vabs + (C_ACC * n + 2 + nb) * U * (w @ vabs) + n * FTZ * vmax
        dl = (torch.maximum(hi - e, e - lo) * sc).sum(-1, keepdim=True) + (n / 4 + 2 * nb + 4) * U * l + n * FTZ
        eta = dl / l
        e32 = (e_num / l + out.abs() * eta) / (1 - eta)
        e32 = e32 + 3 * U * (out.abs() + e32)
        if key_mask is not None and zero_masked_rows:
            out = torch.where(empty, torch.zeros_like(out), out)
            e32 = torch.where(empty, torch.zeros_like(e32), e32)
        ref[:, r0:r1] = out
        bound[:, r0:r1] = e32 + 0.5 * bf16_ulp(out.abs() + e32)
    return ref, bound


def qkv_attention_reference(qkv: Tensor, lengths: Sequence[int], H: int, dh: int, scale: float, *,
                            mask_self: bool = False) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [T, H dh] of the attention of the packed q | k | v buffer qkv[T, 3 H dh] (bf16) over consecutive
    sequences of `lengths` tokens (T = sum(lengths)), as b200vit_attention (equal lengths) or _varlen lays it out."""
    T, I = qkv.shape[0], H * dh
    assert qkv.shape[1] == 3 * I and sum(lengths) == T
    dev = qkv.device
    ref = torch.empty(T, I, dtype=torch.float64, device=dev)
    bound = torch.empty_like(ref)
    by_len, s0 = {}, 0
    for n in lengths:
        by_len.setdefault(int(n), []).append(s0)
        s0 += int(n)
    for n, st in by_len.items():
        idx = (torch.tensor(st, device=dev)[:, None] + torch.arange(n, device=dev)[None]).reshape(-1)
        x = qkv[idx].view(len(st), n, 3, H, dh).permute(2, 0, 3, 1, 4).reshape(3, len(st) * H, n, dh)
        r, b = attention_reference(x[0], x[1], x[2], scale, mask_self=mask_self)
        ref[idx] = r.view(len(st), H, n, dh).permute(0, 2, 1, 3).reshape(-1, I)
        bound[idx] = b.view(len(st), H, n, dh).permute(0, 2, 1, 3).reshape(-1, I)
    return ref, bound


def axial_reference(qkv: Tensor, key_mask: Optional[Tensor], B: int, L: int, G: int, H: int, dh: int, scale: float,
                    zero_masked_rows: bool) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [B L G, H dh] of the B*G*H sequences (token j of b*G + p at row b*L*G + j*G + p) from
    attention_reference with the key mask of each sequence's batch element: one 64-key block, a row
    without a kept key 0 (zero_masked_rows) or the mean of its sequence's values."""
    t = qkv.view(B, L, G, 3, H, dh).permute(3, 0, 2, 4, 1, 5).reshape(3, B * G * H, L, dh)
    km = None if key_mask is None else key_mask.bool()[:, None, None, :].expand(B, G, H, L).reshape(B * G * H, L)
    ref, bound = attention_reference(t[0], t[1], t[2], scale, key_mask=km, zero_masked_rows=zero_masked_rows)
    back = lambda x: x.view(B, G, H, L, dh).permute(0, 3, 1, 2, 4).reshape(B * L * G, H * dh)   # noqa: E731
    return back(ref), back(bound)


def qkv_inputs(kind: str, lengths: Sequence[int], H: int, dh: int, *, seed: int = 0, device="cpu") -> Tensor:
    """Seeded packed q | k | v [sum(lengths), 3 H dh] bf16 in one of four distributions:
      normal    N(0, 1);
      peaked    q, k of std 2: logits scale * q.k of std about 4 at scale dh^-0.5, a few keys take most of each row;
      late_max  q of mean 1 and the last key of every sequence (in its last key block for any KB) near all ones, so the
                row max rises in the last block by several units and corr there is far from 1 (about e^-4 at dh 64)
                while the earlier keys still carry weight;
      vmean     v of mean 3 and std 1: |v_j - out| cancels, so an error in l shows against a large |out|."""
    g = torch.Generator(device=device).manual_seed(seed)
    T, I = sum(int(n) for n in lengths), H * dh
    x = torch.randn(T, 3, I, generator=g, device=device)
    if kind == "peaked":
        x[:, :2] *= 2
    elif kind == "late_max":
        x[:, 0] += 1
        last = torch.tensor(lengths, device=device).cumsum(0) - 1
        x[last, 1] = 1 + 0.5 * torch.randn(len(lengths), I, generator=g, device=device)
    elif kind == "vmean":
        x[:, 2] += 3
    else:
        assert kind == "normal", kind
    return x.view(T, 3 * I).bfloat16()


KINDS = ("normal", "peaked", "late_max", "vmean")
