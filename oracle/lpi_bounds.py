"""fp64 reference with a per-element error bound for the local patch interaction kernel (lpi.cu)  --  TEST
INFRASTRUCTURE.

The conventions are those of oracle/bounds.py: `(ref, bound)` fp64 on the inputs' device, the reference takes the
kernel's own inputs (the fp32 stream x, the LayerNorm's gamma / beta / eps and the folded fp32 weights w1, b1, w2, b2),
and the bound counts only the rounding the kernel does, in its order.  u = 2^-24.

The kernel, per channel c of every token of an h x w grid:
  - z = fmaf((x - mean) rstd, gamma, beta) with (mean, rstd) from ln_row_stats: the LayerNorm of row_bounds, whose
    fp32 error E_z is bounds.layernorm_e32 at depth row_bounds.ln_depth(D).  Outside the grid z is an exact 0.
  - a1 = b1 + sum over the k x k taps of w1 z: a chain of k^2 fmas starting at the bias, each rounding once, so
    E_1 = k^2 u (|b1| + sum |w1| |z|) + sum |w1| E_z.
  - g = GELU(a1) = 0.5 a1 (1 + erff(a1 fl32(1 / sqrt 2))).  The argument is off by 2 u relative, which moves erf by at
    most (2 / sqrt pi) max(t e^-t^2) 2 u < u; erff is within 2 ulp (4 u); 1 + e rounds (u |1 + e| <= 2 u); 0.5 a1 is
    exact; the product rounds (u |g|).  So the evaluation adds 3.5 u |a1| + u |g|, and the propagated E_1 is scaled by
    at most GELU's largest slope, 1.13: E_g = 1.13 E_1 + 3.5 u (|a1| + E_1) + u |g|.  Outside the grid g is 0.
  - a2 = b2 + sum of w2 g over the taps: E_2 = k^2 u (|b2| + sum |w2| (|g| + E_g)) + sum |w2| E_g.
  - y = x + a2: E_y = E_2 + u (|y| + E_2).
The bf16 copy and row statistics the kernel writes with y are those of rowstats_cast of its own y
(row_bounds.row_stats_reference)."""
from __future__ import annotations

import math
from typing import Tuple

import torch
import torch.nn.functional as F

from oracle.bounds import GELU_SLOPE, U, layernorm_e32
from oracle.row_bounds import ln_depth

Tensor = torch.Tensor


def _eps32(eps: float) -> float:
    return torch.tensor(eps, dtype=torch.float32).item()


def lpi_reference(x: Tensor, ln: tuple, w1: Tensor, b1: Tensor, w2: Tensor, b2: Tensor, B: int, gh: int, gw: int,
                  k: int) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [B gh gw, D] of y = x + conv2'(GELU(conv1'(LN(x)))) as b200vit_local_patch_interaction computes
    it: x fp32 [B gh gw, D], ln = (gamma, beta, eps), w1 / w2 fp32 [k k, D] tap-major depthwise weights, b1 / b2 [D]."""
    D = x.shape[1]
    gamma, beta, eps = ln
    z, ez = layernorm_e32(x, gamma, beta, _eps32(eps), ln_depth(D))

    def grid(t):                                       # [B gh gw, D] -> [B, D, gh, gw]
        return t.view(B, gh, gw, D).permute(0, 3, 1, 2)

    def conv(t, w):                                    # depthwise k x k, zero padding k // 2, no bias
        return F.conv2d(t, w.double().t().reshape(D, 1, k, k), padding=k // 2, groups=D)

    z, ez = grid(z), grid(ez)
    bb1, bb2 = b1.double()[None, :, None, None], b2.double()[None, :, None, None]
    a1 = conv(z, w1) + bb1
    e1 = k * k * U * (conv(z.abs(), w1.abs()) + bb1.abs()) + conv(ez, w1.abs())
    g = 0.5 * a1 * (1.0 + torch.erf(a1 / math.sqrt(2.0)))
    eg = GELU_SLOPE * e1 + 3.5 * U * (a1.abs() + e1) + U * g.abs()
    a2 = conv(g, w2) + bb2
    e2 = k * k * U * (conv(g.abs() + eg, w2.abs()) + bb2.abs()) + conv(eg, w2.abs())
    a2, e2 = a2.permute(0, 2, 3, 1).reshape(-1, D), e2.permute(0, 2, 3, 1).reshape(-1, D)
    y = x.double() + a2
    return y, (e2 + U * (y.abs() + e2)) * (1 + 1e-3)
