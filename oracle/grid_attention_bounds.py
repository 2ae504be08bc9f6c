"""fp64 references with a per-element error bound for the attention kernels over token grids and the kernels around
them: windows (Twins-SVT, MaxViT, CrossFormer), sub-sampled keys (Twins-SVT, CvT, ScalableViT), interactive windows
(ScalableViT), patch groups (MobileViT), the depthwise convolutional projection (CvT), window tokens and window mixing
(SepViT), region-to-local windows (RegionViT), the position-bias attention of LeViT, the positional encoding generator
(Twins-SVT, ScalableViT), the im2col gathers, and the SiLU GEMM epilogue and the head LayerNorm + GELU  --  TEST
INFRASTRUCTURE.

Every reference returns `(ref, bound)`: fp64 tensors on the device of its inputs, to be checked with
oracle.bounds.check.  The attention references gather each window's rows and hand them to
oracle.attention_bounds.attention_reference, whose bound models the bf16 probabilities the kernels round before P V;
the relative-position ones add the bias inside the score and bound it as the position-bias attention of LeViT.

The row maps (`window_rows`, `group_rows`, `region_window_rows`) and the bias index maps (`relpos_index`,
`region_bias_index`, `posbias_index`) are the kernels' address formulas; tests/test_grid_layer_trace.py and
tests/test_class_layer_trace.py tie each of them to the reference module's own rearranges and bias look-ups."""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch
import torch.nn.functional as F

from oracle.attention_bounds import attention_reference
from oracle.bounds import C_ACC, U, U_BF16, bf16_ulp
from oracle.row_bounds import layernorm_heads_reference

Tensor = torch.Tensor


def _f32(v: float) -> float:
    return float(torch.tensor(v, dtype=torch.float32))


# ------------------------------------------------------------------------------------------------------ row maps
def window_rows(B: int, gh: int, gw: int, wh: int, ww: int, device, dilated: bool = False) -> Tensor:
    """int64 [B * windows, wh*ww]: the map rows of every window of a gh x gw grid, windows in (b, wy, wx) order and
    tokens (u, v) inside.  Contiguous wh x ww blocks, or with `dilated` the dilated grids of
    b200vit_attention_window_relpos (token (u, v) of window (wy, wx) at map position (u * gh/wh + wy, v * gw/ww + wx))."""
    X, Y = gh // wh, gw // ww
    b, i, j, u, v = torch.meshgrid(*(torch.arange(n, device=device) for n in (B, X, Y, wh, ww)), indexing="ij")
    y = u * X + i if dilated else i * wh + u
    x = v * Y + j if dilated else j * ww + v
    return ((b * gh + y) * gw + x).reshape(B * X * Y, wh * ww)


def group_rows(B: int, gh: int, gw: int, ph: int, pw: int, device) -> Tensor:
    """[B*ph*pw, n] map rows of every patch group, group (b, i, j) in that order, token t = y'*(gw/pw) + x'."""
    hh, ww = gh // ph, gw // pw
    b, i, j, y, x = torch.meshgrid(*(torch.arange(n, device=device) for n in (B, ph, pw, hh, ww)), indexing="ij")
    return ((b * gh + y * ph + i) * gw + x * pw + j).reshape(B * ph * pw, hh * ww)


def region_window_rows(B: int, lh: int, lw: int, rh: int, rw: int, device) -> Tensor:
    """[B*rh*rw, 1 + wh*ww] stream rows of every region-to-local window in (b, i, j) order: the region row, then local
    (u, v)."""
    wh, ww = lh // rh, lw // rw
    b, i, j, u, v = torch.meshgrid(*(torch.arange(n, device=device) for n in (B, rh, rw, wh, ww)), indexing="ij")
    local = ((b * lh + i * wh + u) * lw + j * ww + v).reshape(B * rh * rw, wh * ww)
    region = B * lh * lw + torch.arange(B * rh * rw, device=device)
    return torch.cat((region[:, None], local), 1)


def relpos_index(w: int, device) -> Tensor:
    """[w*w, w*w] column of the [(2w-1)^2] bias table that b200vit_attention_window_relpos adds to the score of local
    query r = u*w + v and key r' = u'*w + v': row offset major, (u - u' + w - 1) (2w - 1) + (v - v' + w - 1)."""
    r = torch.arange(w * w, device=device)
    u, v = r // w, r % w
    return (u[:, None] - u[None, :] + w - 1) * (2 * w - 1) + (v[:, None] - v[None, :] + w - 1)


def region_bias_index(wh: int, ww: int, W: int, device) -> Tensor:
    """[wh*ww, wh*ww] column of the [(2W-1)^2] bias table that b200vit_attention_region_local adds between local
    tokens t = u*ww + v and t': column offset major, (u - u' + W - 1) + (v - v' + W - 1) (2W - 1)."""
    t = torch.arange(wh * ww, device=device)
    u, v = t // ww, t % ww
    return (u[:, None] - u[None, :] + W - 1) + (v[:, None] - v[None, :] + W - 1) * (2 * W - 1)


def _scatter(rows: Tensor, vals: Tensor, M: int) -> Tensor:
    out = torch.zeros(M, vals.shape[-1], dtype=torch.float64, device=vals.device)
    out[rows.reshape(-1)] = vals
    return out


# ------------------------------------------------------------------------------------------------------ windows
def window_reference(qkv: Tensor, B: int, gh: int, gw: int, p: int, H: int, dh: int,
                     scale: Optional[float] = None) -> Tuple[Tensor, Tensor]:
    """b200vit_attention_window (Twins-SVT's LocalAttention): attention_reference inside every p x p block."""
    scale = dh ** -0.5 if scale is None else scale
    I, rows = H * dh, window_rows(B, gh, gw, p, p, qkv.device)
    g = qkv[rows.reshape(-1)].view(rows.shape[0], p * p, 3, H, dh).permute(2, 0, 3, 1, 4)      # 3, W, H, n, dh
    q, k, v = (t.reshape(-1, p * p, dh) for t in g)
    ref, bound = attention_reference(q, k, v, scale)
    back = lambda t: t.view(rows.shape[0], H, p * p, dh).permute(0, 2, 1, 3).reshape(-1, I)   # noqa: E731
    M = B * gh * gw
    return _scatter(rows, back(ref), M), _scatter(rows, back(bound), M)


def _bias_attention(q: Tensor, k: Tensor, v: Tensor, bias: Tensor, scale: float, dh: int) -> Tuple[Tensor, Tensor]:
    """(out, bound) [G, H, n, dh] of softmax(scale q k^T + bias) v on fp64 q, k, v [G, H, n, dh], bounded as the
    position-bias attention of test_gpu_levit.py: the bf16 probabilities before P V, the fp32 scores and the rounding
    of the scale and the bias, fp32 accumulation, the output's bf16 rounding."""
    n = q.shape[-2]
    sc = _f32(scale)
    logits = sc * q @ k.transpose(-1, -2) + bias
    p = logits.softmax(-1)
    out = p @ v
    mag = p @ v.abs()
    dx = (C_ACC * dh + 4) * U * sc * (q.abs() @ k.abs().transpose(-1, -2)) + 4 * U * (bias.abs() + logits.abs())
    e = (2.0 ** -8 + 4 * dx.amax(-1, keepdim=True) + (C_ACC * n + n / 4 + 16) * U) * mag + 3 * U * out.abs()
    return out, e + bf16_ulp(out.abs() + e) / 2


def relpos_bias(table: Tensor, w: int) -> Tensor:
    """[H, w*w, w*w] fp64: the bias b200vit_attention_window_relpos adds, from its table [H, (2w-1)^2]."""
    return table.double()[:, relpos_index(w, table.device)]


def relpos_reference(qkv: Tensor, table: Tensor, B: int, gh: int, gw: int, w: int, grid: bool, H: int, dh: int,
                     scale: float) -> Tuple[Tensor, Tensor]:
    """fp64 (ref, bound) of b200vit_attention_window_relpos on the kernel's own bf16 inputs: w x w windows (dilated
    grids with `grid`) under the relative-position bias table [H, (2w-1)^2]."""
    rows = window_rows(B, gh, gw, w, w, qkv.device, dilated=grid)
    x = qkv.double()[rows]                                                   # windows, n, 3 H dh
    n = w * w
    q, k, v = (x[..., s * H * dh:(s + 1) * H * dh].reshape(-1, n, H, dh).transpose(1, 2) for s in range(3))
    out, bound = _bias_attention(q, k, v, relpos_bias(table, w), scale, dh)
    M = B * gh * gw
    return (_scatter(rows, out.transpose(1, 2).reshape(-1, H * dh), M),
            _scatter(rows, bound.transpose(1, 2).reshape(-1, H * dh), M))


def region_bias(table: Tensor, wh: int, ww: int, W: int) -> Tensor:
    """[H, n, n] fp64, n = 1 + wh*ww: the bias b200vit_attention_region_local adds inside a window (none on the region
    token's row and column), from its table [H, (2W-1)^2]."""
    H, n = table.shape[0], 1 + wh * ww
    bias = torch.zeros(H, n, n, dtype=torch.float64, device=table.device)
    bias[:, 1:, 1:] = table.double()[:, region_bias_index(wh, ww, W, table.device)]
    return bias


def region_local_reference(qkv: Tensor, table: Tensor, B: int, lh: int, lw: int, rh: int, rw: int, W: int, H: int,
                           scale: float, dh: int = 32) -> Tuple[Tensor, Tensor]:
    """fp64 (ref, bound) of b200vit_attention_region_local on the kernel's own bf16 inputs, bounded as the
    relative-position window attention (relpos_reference)."""
    rows = region_window_rows(B, lh, lw, rh, rw, qkv.device)
    n = rows.shape[1]
    x = qkv.double()[rows]                                                   # windows, n, 3 H dh
    q, k, v = (x[..., s * H * dh:(s + 1) * H * dh].reshape(-1, n, H, dh).transpose(1, 2) for s in range(3))
    out, bound = _bias_attention(q, k, v, region_bias(table, lh // rh, lw // rw, W), scale, dh)
    M = qkv.shape[0]
    return (_scatter(rows, out.transpose(1, 2).reshape(-1, H * dh), M),
            _scatter(rows, bound.transpose(1, 2).reshape(-1, H * dh), M))


# ---------------------------------------------------------------------------------------------------- sub-sampled keys
def kv_reference(q: Tensor, kv: Tensor, B: int, Nq: int, Nk: int, H: int, dh: int,
                 scale: Optional[float] = None) -> Tuple[Tensor, Tensor]:
    """b200vit_attention_kv: Nq queries per image against the image's Nk keys.  attention_reference takes as many
    queries as keys: the queries go in chunks of Nk (zero padded), each chunk a sequence of its own over the image's
    keys."""
    scale = dh ** -0.5 if scale is None else scale
    I, chunks = H * dh, -(-Nq // Nk)
    q4 = F.pad(q.reshape(B, Nq, H, dh), (0, 0, 0, 0, 0, chunks * Nk - Nq)).view(B, chunks, Nk, H, dh)
    qs = q4.permute(0, 3, 1, 2, 4).reshape(B * H * chunks, Nk, dh)
    k, v = (kv[:, o * I:(o + 1) * I].reshape(B, Nk, H, dh).permute(0, 2, 1, 3).reshape(B * H, Nk, dh) for o in (0, 1))
    ref, bound = attention_reference(qs, k.repeat_interleave(chunks, 0), v.repeat_interleave(chunks, 0), scale)
    back = lambda t: t.view(B, H, chunks * Nk, dh)[:, :, :Nq].permute(0, 2, 1, 3).reshape(B * Nq, I)   # noqa: E731
    return back(ref), back(bound)


def attention_ex_reference(q: Tensor, k: Tensor, v: Tensor, scale: float) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [G, n, dv] of attention_reference for key heads dk and value heads dv wide: both padded with zero
    columns to max(dk, dv) (zero q / k columns add exactly 0 to every score, the bound's score term grows with the
    width), the zero value columns dropped again."""
    dk, dv = q.shape[-1], v.shape[-1]
    W = max(dk, dv)
    pad = lambda t: F.pad(t, (0, W - t.shape[-1]))     # noqa: E731
    ref, bound = attention_reference(pad(q), pad(k), pad(v), scale, kb=64)
    return ref[..., :dv], bound[..., :dv]


def _kv_rows_reference(q: Tensor, k: Tensor, v: Tensor, scale: float) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [Nq, dv] of Nq queries against one set of Nk keys: attention_reference takes sequences with as many
    queries as keys and bounds every query row on its own, so the queries go in as ceil(Nq / Nk) sequences of Nk rows
    (the last one filled with repeats of the last query) over the same keys."""
    Nq, Nk = q.shape[0], k.shape[0]
    c = -(-Nq // Nk)
    qq = q[torch.arange(c * Nk, device=q.device).clamp_max(Nq - 1)].view(c, Nk, -1)
    r, b = attention_ex_reference(qq, k[None].expand(c, -1, -1).contiguous(), v[None].expand(c, -1, -1).contiguous(),
                                  scale)
    return r.reshape(c * Nk, -1)[:Nq], b.reshape(c * Nk, -1)[:Nq]


def kv_ex_reference(q: Tensor, kv: Tensor, B: int, Nq: int, Nk: int, H: int, dk: int, dv: int,
                    scale: float) -> Tuple[Tensor, Tensor]:
    """b200vit_attention_kv_ex: key heads dk wide, value heads dv wide (ScalableViT's SSA)."""
    qh = q.view(B, Nq, H, dk).transpose(1, 2).reshape(B * H, Nq, dk)
    kh = kv[:, :H * dk].reshape(B, Nk, H, dk).transpose(1, 2).reshape(B * H, Nk, dk)
    vh = kv[:, H * dk:].reshape(B, Nk, H, dv).transpose(1, 2).reshape(B * H, Nk, dv)
    outs, bounds = zip(*(_kv_rows_reference(qh[g], kh[g], vh[g], scale) for g in range(B * H)))
    ref = torch.stack(outs).view(B, H, Nq, dv).transpose(1, 2).reshape(B * Nq, H * dv)
    bnd = torch.stack(bounds).view(B, H, Nq, dv).transpose(1, 2).reshape(B * Nq, H * dv)
    return ref, bnd


# ------------------------------------------------------------------------------------------------- interactive windows
def with_added(ref: Tensor, bound: Tensor, lim: Tensor) -> Tuple[Tensor, Tensor]:
    """(ref, bound) of bf16(fma(O, 1 / l, lim)) from attention_reference's (ref, bound) of bf16(O / l): its fp32 error
    is at most bound - ulp(|ref|) / 2 (the rounding term it adds is at least that), plus the fma's rounding."""
    e32 = (bound - 0.5 * bf16_ulp(ref.abs())).clamp_min(0)
    tot = ref + lim.double()
    e = e32 + U * (tot.abs() + e32)
    return tot, e + 0.5 * bf16_ulp(tot.abs() + e)


def iwsa_reference(qkv: Tensor, lim: Tensor, B: int, gh: int, gw: int, wh: int, ww: int, H: int, dk: int, dv: int,
                   scale: float) -> Tuple[Tensor, Tensor]:
    """b200vit_attention_iwsa: attention inside wh x ww windows with q / k heads dk wide and v heads dv wide, plus the
    LIM term `lim` before the output's one rounding."""
    rows = window_rows(B, gh, gw, wh, ww, qkv.device)
    G, n = rows.shape
    x = qkv[rows.reshape(-1)].view(G, n, -1)
    q = x[..., :H * dk].reshape(G, n, H, dk).transpose(1, 2).reshape(G * H, n, dk)
    k = x[..., H * dk:2 * H * dk].reshape(G, n, H, dk).transpose(1, 2).reshape(G * H, n, dk)
    v = x[..., 2 * H * dk:2 * H * dk + H * dv].reshape(G, n, H, dv).transpose(1, 2).reshape(G * H, n, dv)
    r, b = attention_ex_reference(q, k, v, scale)
    r = r.view(G, H, n, dv).transpose(1, 2).reshape(G * n, H * dv)
    b = b.view(G, H, n, dv).transpose(1, 2).reshape(G * n, H * dv)
    M = B * gh * gw
    return with_added(_scatter(rows, r, M), _scatter(rows, b, M), lim)


# ------------------------------------------------------------------------------------------------------ patch groups
def groups_reference(qkv: Tensor, B: int, gh: int, gw: int, ph: int, pw: int, H: int, dh: int = 8,
                     scale: Optional[float] = None) -> Tuple[Tensor, Tensor]:
    """b200vit_attention_groups (MobileViT): attention inside every strided patch group."""
    scale = dh ** -0.5 if scale is None else scale
    rows = group_rows(B, gh, gw, ph, pw, qkv.device)
    G, n = rows.shape
    x = qkv[rows.reshape(-1)].view(G, n, 3, H, dh).permute(2, 0, 3, 1, 4).reshape(3, G * H, n, dh)
    r, b = attention_reference(x[0], x[1], x[2], scale, kb=64)
    M = B * gh * gw
    back = lambda t: t.view(G, H, n, dh).permute(0, 2, 1, 3).reshape(-1, H * dh)      # noqa: E731
    return _scatter(rows, back(r), M), _scatter(rows, back(b), M)


# ------------------------------------------------------------------------------------------------------ window tokens
def window_token_reference(qkv: Tensor, tok: Tensor, B: int, gh: int, gw: int, p: int, H: int, dh: int,
                           scale: Optional[float] = None) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """(ref, bound) of out [M, I] and tok_out [B*nw, I] of b200vit_attention_window_token: attention_reference over
    every (window, head) with the window token's q | k | v prepended as token 0."""
    scale = dh ** -0.5 if scale is None else scale
    I, rows = H * dh, window_rows(B, gh, gw, p, p, qkv.device)
    G, n = rows.shape
    x = qkv[rows.reshape(-1)].view(G, n, 3, H, dh)
    x = torch.cat((tok.view(1, 1, 3, H, dh).expand(G, 1, -1, -1, -1), x), 1)
    x = x.permute(2, 0, 3, 1, 4).reshape(3, G * H, n + 1, dh)
    r, b = attention_reference(x[0], x[1], x[2], scale, kb=64)
    r, b = r.view(G, H, n + 1, dh).transpose(1, 2), b.view(G, H, n + 1, dh).transpose(1, 2)
    M = B * gh * gw
    return (_scatter(rows, r[:, 1:].reshape(-1, I), M), _scatter(rows, b[:, 1:].reshape(-1, I), M),
            r[:, 0].reshape(G, I), b[:, 0].reshape(G, I))


def mix_reference(wqk: Tensor, o: Tensor, B: int, gh: int, gw: int, p: int, H: int, dh: int,
                  scale: Optional[float] = None) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [M, I] of b200vit_window_mix: attention_reference with q = wq, k = wk and v = each window's p*p*dh
    outputs of the head, taken dh columns (one window position) at a time."""
    scale = dh ** -0.5 if scale is None else scale
    I, rows = H * dh, window_rows(B, gh, gw, p, p, o.device)
    nw, pp = rows.shape[0] // B, p * p
    w = wqk.view(B, nw, H, 2, dh).permute(0, 2, 1, 3, 4)                 # b h n (q|k) d
    q, k = (w[..., c, :].reshape(B * H, 1, nw, dh).expand(-1, pp, -1, -1).reshape(-1, nw, dh) for c in (0, 1))
    v = o[rows.reshape(-1)].view(B, nw, pp, H, dh).permute(0, 3, 2, 1, 4).reshape(B * H * pp, nw, dh)
    r, b = attention_reference(q, k, v, scale, kb=64)                     # [(b h w), i, d]
    back = lambda t: t.view(B, H, pp, nw, dh).permute(0, 3, 2, 1, 4).reshape(-1, I)    # noqa: E731
    return _scatter(rows, back(r), B * gh * gw), _scatter(rows, back(b), B * gh * gw)


def head_layernorm_gelu_reference(x: Tensor, gamma: Tensor, beta: Tensor, H: int, dh: int,
                                  eps: float = 1e-5) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [T, H, dh] of b200vit_head_layernorm_gelu on bf16 x [T, H dh]: GELU(LN(head) gamma + beta), one
    LayerNorm over each head's dh values.  The head norm's fp32 bound (oracle/row_bounds.py) before its rounding, the
    shift's add, GELU's slope (below 1.13) and gelu_erf's 1.2e-5 (common.cuh) plus its products' roundings, then the
    output's bf16 rounding."""
    T = x.shape[0]
    ln, bnd = layernorm_heads_reference(x.reshape(T, H, dh), gamma.reshape(1, dh).expand(H, dh), eps)
    e_ln = (bnd - bf16_ulp(ln)) / (1 + U_BF16)           # the fp32 bound of the normalised value, before rounding
    pre = ln + beta.double().reshape(dh)
    e_pre = e_ln + U * (pre.abs() + e_ln)
    ref = 0.5 * pre * (1 + torch.erf(pre / math.sqrt(2)))
    e = 1.13 * e_pre + 1.2e-5 + 8 * U * ref.abs()
    return ref, bf16_ulp(ref.abs() + e) / 2 + e


# ------------------------------------------------------------------------------------------------------ convolutions
def conv_reference(x: Tensor, wt: Tensor, b: Tensor, B: int, h: int, w: int, k: int, s: int) -> Tuple[Tensor, Tensor]:
    """fp64 (ref, bound) of one half of b200vit_conv_proj_dw: the depthwise k x k convolution at stride s, zero padding
    k // 2, of the kernel's own bf16 input with its tap-major weights wt [k*k, C] and bias b, bounded by half a bf16 ulp
    of the fp64 value plus the fp32 accumulation of k*k products and the bias, about k^2 2^-23 sum |w x| + |b|."""
    C = x.shape[1]
    xi = x.double().reshape(B, h, w, C).permute(0, 3, 1, 2)
    wd = wt.double().t().reshape(C, 1, k, k)
    ref = F.conv2d(xi, wd, b.double(), stride=s, padding=k // 2, groups=C)
    mag = F.conv2d(xi.abs(), wd.abs(), b.double().abs(), stride=s, padding=k // 2, groups=C)
    ref, mag = (t.permute(0, 2, 3, 1).reshape(-1, C) for t in (ref, mag))
    e = (k * k + 1) * 2.0 ** -23 * mag
    return ref, e + bf16_ulp(ref.abs() + e) / 2


def peg_reference(x: Tensor, w: Tensor, b: Tensor, B: int, gh: int, gw: int, k: int) -> Tuple[Tensor, Tensor]:
    """fp64 (ref, bound) of b200vit_peg (Twins-SVT, ScalableViT): conv2d plus the identity, and per element the fp32
    error of k*k accumulated taps, the bias and the residual add."""
    C = x.shape[1]
    grid = x.double().view(B, gh, gw, C).permute(0, 3, 1, 2)
    wt = w.double().t().reshape(C, 1, k, k)
    ref = F.conv2d(grid, wt, b.double(), padding=k // 2, groups=C) + grid
    mag = F.conv2d(grid.abs(), wt.abs(), b.double().abs(), padding=k // 2, groups=C) + grid.abs()
    ref, mag = (t.permute(0, 2, 3, 1).reshape(-1, C) for t in (ref, mag))
    return ref, (k * k + 4) * U * mag + 1e-30


def im2col_reference(x: Tensor, B: int, H: int, W: int, k: int, s: int, pad: int) -> Tensor:
    """b200vit_conv_im2col_nhwc, exactly: the k x k patches at stride s, zero padding `pad`, of the NHWC map x
    [B*H*W, C] (a column slice allowed), one row per output position, columns (tap row, tap column, channel)."""
    C = x.shape[1]
    xi = x.reshape(B, H, W, C).permute(0, 3, 1, 2).double()
    cols = F.unfold(xi, k, padding=pad, stride=s)                          # B, C k k, L: columns (c, ky, kx)
    L = cols.shape[-1]
    return cols.view(B, C, k * k, L).permute(0, 3, 2, 1).reshape(B * L, k * k * C)


def im2col_nchw_reference(img: Tensor, k: int, s: int, pad: int) -> Tensor:
    """b200vit_conv_im2col_nchw, exactly: F.unfold(img, k, padding=pad, stride=s) of the NCHW image [B, C, H, W], one
    row per output position, columns (channel, tap row, tap column)."""
    cols = F.unfold(img.double(), k, padding=pad, stride=s)               # B, C k k, L
    return cols.transpose(1, 2).reshape(-1, cols.shape[1])


def posbias_index(F_: int, s: int, device=None) -> Tensor:
    """int64 [ceil(F / s)^2, F^2]: the bias-table column b200vit_attention_posbias adds to query (i, j) and key
    (y, x) of an F x F map, the query at map position (s i, s j): |s i - y| F + |s j - x|."""
    qy, qx = torch.meshgrid(torch.arange(0, F_, s, device=device), torch.arange(0, F_, s, device=device), indexing="ij")
    ky, kx = torch.meshgrid(torch.arange(F_, device=device), torch.arange(F_, device=device), indexing="ij")
    return (qy.reshape(-1, 1) - ky.reshape(1, -1)).abs() * F_ + (qx.reshape(-1, 1) - kx.reshape(1, -1)).abs()


def posbias_reference(qkv: Tensor, table: Tensor, B: int, F_: int, s: int, H: int, dk: int, dv: int, scale: float,
                      gelu: bool = True) -> Tuple[Tensor, Tensor]:
    """fp64 (ref, bound) of b200vit_attention_posbias (LeViT, levit.py:133-158) on the kernel's own bf16 inputs.  The
    bound counts: the bf16 rounding of the probabilities before P V (2^-8 relative per key, against sum_j p_j |v_j|),
    the score error (the fp32 dot products, C_ACC dk u sum |q||k| scaled, and the rounding of the scale, the bias and
    their sum: a relative change of the probabilities by e^(2 dx)), fp32 accumulation of P V and of l, then GELU
    (slope at most 1.13) and the output's bf16 rounding."""
    Fq = -(-F_ // s)
    x = qkv.double()[:B * F_ * F_].view(B, F_, F_, -1)
    q = x[:, ::s, ::s, :H * dk].reshape(B, Fq * Fq, H, dk).transpose(1, 2)
    k = x[..., H * dk:2 * H * dk].reshape(B, F_ * F_, H, dk).transpose(1, 2)
    v = x[..., 2 * H * dk:2 * H * dk + H * dv].reshape(B, F_ * F_, H, dv).transpose(1, 2)
    bias = table.double()[:, posbias_index(F_, s, qkv.device)]                       # H, Nq, Nk
    sc = float(torch.tensor(scale, dtype=torch.float32))
    logits = sc * q @ k.transpose(-1, -2) + bias
    p = logits.softmax(-1)
    out = p @ v
    mag = p @ v.abs()                                                                  # sum_j p_j |v_j|
    dx = (C_ACC * dk + 4) * U * sc * (q.abs() @ k.abs().transpose(-1, -2)) + 4 * U * (bias.abs() + logits.abs())
    dxm = dx.amax(-1, keepdim=True)
    nk = F_ * F_
    e_attn = (2.0 ** -8 + 4 * dxm + (C_ACC * nk + nk / 4 + 16) * U) * mag
    e_attn = e_attn + 3 * U * out.abs()
    if gelu:
        ref = torch.nn.functional.gelu(out)
        e = 1.13 * e_attn + 1e-6 * (ref.abs() + e_attn) + 1e-30
    else:
        ref, e = out, e_attn
    bound = e + bf16_ulp(ref.abs() + e) / 2
    back = lambda t: t.transpose(1, 2).reshape(B * Fq * Fq, H * dv)                   # noqa: E731
    return back(ref), back(bound)


# ------------------------------------------------------------------------------------------------------ epilogues
def silu_bound(y: Tensor, e_y: Tensor) -> Tuple[Tensor, Tensor]:
    """(ref, fp32 bound) of the SiLU epilogue y sigmoid(y) on a GEMM result y within e_y: SiLU's slope is below 1.1,
    plus its ex2 / rcp approximations and products."""
    ref = y * torch.sigmoid(y)
    return ref, 1.1 * e_y + 8 * U * ref.abs() + 4 * U * y.abs() + 1e-30
