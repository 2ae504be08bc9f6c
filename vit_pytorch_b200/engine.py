"""Host-side engine of the fused sm_90a forward: weight preparation, workspaces and the kernel schedule.

The nn.Modules in vit.py, simple_vit.py, na_vit.py, ... own the parameters (reference-compatible names); each
Transformer describes its layers to this file as EncoderLayer records, the only thing the engine knows about a model
family.  This file turns them into the flat bf16 / fp32 device buffers the C ABI (include/b200vit.h) consumes and
issues the launches on torch's current stream.  Nothing here computes on the host and nothing falls back: a missing
library or a failing call raises.

Schedule per encoder layer (reference vit.py:78-81) in the default LayerNorm mode, fold (see ln_mode), M = B*N token
rows, residual stream x in fp32 and xb, its bf16 copy, which the LN-folded GEMMs read with its per-row (sum, sum^2):
    qkv = LN1(x) Wqkv^T                        b200vit_gemm_bf16      LN-folded, bf16 out       (vit.py:52,54)
    o   = softmax(q k^T * scale) v             b200vit_attention      wgmma, online softmax     (vit.py:55-63)
    x  += o Wout^T + b                         b200vit_gemm_bf16      residual epilogue, + xb   (vit.py:64,80)
    h   = GELU(LN2(x) W1^T + b1)               b200vit_gemm_bf16      LN-folded, GELU epilogue  (vit.py:19-21)
    x  += h W2^T + b2                          b200vit_gemm_bf16      residual epilogue, + xb   (vit.py:23,81)
exact: b200vit_layernorm (x -> xb) and the plain GEMM in place of each LN-folded one, the reference's operator sequence.
"""
from __future__ import annotations

import ctypes
import os
from dataclasses import dataclass
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple, Union

import torch
from torch import nn

from . import _lib

_FORCE_EAGER_ENV = "B200VIT_DISABLE_FUSED"
_LN_MODE_ENV = "B200VIT_LN_MODE"      # "fold" (default) | "exact"
_PATCH_MODE_ENV = "B200VIT_PATCH_MODE"  # "tma" (default: im2col-free 16x16 patch embedding) | "gather"
_HOST_LOOP_ENV = "B200VIT_HOST_LOOP"    # "c" (default: all layers in one b200vit_encoder_blocks call) | "python"


def ln_mode() -> str:
    """'exact' : LayerNorm kernel -> bf16 -> GEMM, the literal operator sequence of the reference.
       'fold'  : (default) no standalone LayerNorm kernels inside the layer loop.  The residual GEMMs (out-proj, fc2) also emit
                 a bf16 copy of x plus per-row (sum, sum^2); the following GEMM multiplies that copy by gamma*W and
                 applies  rstd*(acc - mu*colsum) + (W beta + b)  in its epilogue.  The statistics are
                 written as per-tile partials (no atomics) and summed in a fixed order, so results are deterministic."""
    m = os.environ.get(_LN_MODE_ENV, "fold")
    if m not in ("fold", "exact"):
        raise ValueError(f"{_LN_MODE_ENV} must be 'fold' or 'exact', got {m!r}")
    return m


def on_device(t: torch.Tensor):
    """Context manager that makes t's GPU the current device for the duration of a fused forward: the library
    enqueues on torch's current stream of the CURRENT device and keeps its per-device state by cudaGetDevice, so a
    model on cuda:1 must not be launched while cuda:0 is current (ADVICE r1)."""
    return torch.cuda.device(t.device)


def _global_hooks() -> bool:
    """Hooks installed with torch.nn.modules.module.register_module_forward_hook & co. observe every submodule call,
    so they need the PyTorch graph exactly like per-module hooks do."""
    mod = torch.nn.modules.module
    return bool(getattr(mod, "_global_forward_hooks", None)) or bool(getattr(mod, "_global_forward_pre_hooks", None))


def _has_hooks(m: nn.Module) -> bool:
    return bool(m._forward_hooks) or bool(m._forward_pre_hooks) or bool(getattr(m, "_backward_hooks", None))


def hooks_inside(root: nn.Module, skip: Tuple[nn.Module, ...] = ()) -> bool:
    """True if any submodule strictly inside `root` carries a forward(-pre) hook (Recorder / Extractor style
    introspection, reference recorder.py:25-30): those need the materialised eager graph."""
    if _global_hooks():
        return True
    for m in root.modules():
        if m is root or any(m is s for s in skip):
            continue
        if _has_hooks(m):
            return True
    return False


def transformer_is_hooked(owner: nn.Module) -> bool:
    """A hook on the Transformer module ITSELF (reference extractor.py:50-59 registers one to read the embeddings):
    the fused forward then passes the tokens through `owner.transformer(...)` as a module call, so the hook fires
    with the real input / output while the blocks still run fused (hooks strictly inside it need the eager graph)."""
    return _has_hooks(owner.transformer)


def hooked_transformer_tokens(owner: nn.Module, x: torch.Tensor, B: int, N: int) -> torch.Tensor:
    """x fp32 [B*N, D] (assembled tokens) -> owner.transformer(tokens bf16 [B, N, D]) through Module.__call__."""
    tok = torch.empty(B * N, x.shape[1], device=x.device, dtype=torch.bfloat16)
    _lib.cast_f32_bf16(x.view(-1), tok.view(-1))
    return owner.transformer(tok.view(B, N, x.shape[1]))


def why_not_fused(params: List[torch.Tensor], x: torch.Tensor, *, training: bool, dropout_p: float) -> Optional[str]:
    """None if the fused path applies to this call, else the reason the eager PyTorch graph is used."""
    if os.environ.get(_FORCE_EAGER_ENV, "0") == "1":
        return f"{_FORCE_EAGER_ENV}=1"
    if not x.is_cuda:
        return "input is not on a CUDA device"
    if x.dtype != torch.bfloat16:
        return f"input dtype {x.dtype} (fused path is bf16)"
    for p in params:
        if p.device != x.device:
            return "parameters and input on different devices"
        if p.dtype != torch.bfloat16:
            return f"parameter dtype {p.dtype} (fused path is bf16)"
    if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params)):
        # also a frozen model fed by something trainable (prompts, an upstream module, saliency w.r.t. the input):
        # the fused kernels are forward only and would silently cut the graph
        return "autograd is recording (fused path is forward only)"
    if training and dropout_p > 0.0:
        return "dropout is active"
    if torch.cuda.get_device_capability(x.device) != (9, 0):
        return "device is not sm_90"
    return None


def common_reason(owner: nn.Module, x: torch.Tensor, *, encoders=(), dropout_p: float = 0.0,
                  skip: Tuple[nn.Module, ...] = (), inside: str = "model") -> Optional[str]:
    """The part of every drop-in module's fused_reason that does not depend on its input's shape: an empty encoder in
    `encoders`, then why_not_fused over all of `owner`'s parameters, then hooks on submodules of `owner` other than
    `skip` (`inside` names the owner in that reason: "model" or "transformer")."""
    if any(len(e.layers) == 0 for e in encoders):
        return "depth == 0"
    r = why_not_fused(list(owner.parameters()), x, training=owner.training, dropout_p=dropout_p)
    if r is None and hooks_inside(owner, skip):
        r = f"forward hooks registered inside the {inside}"
    return r


HEAD_WIDTHS = (32, 64, 80, 128)
HEADMIX_WIDTHS = (32, 48, 64, 80, 128)     # b200vit_attention_headmix
HEADMIX_MAX_HEADS, HEADMIX_MAX_INNER = 16, 1024
XCA_WIDTHS = (32, 48, 64, 80, 128)         # b200vit_attention_xca
LPI_KERNEL_SIZES = (1, 3, 5, 7)            # b200vit_local_patch_interaction
WINDOW_MAX_TOKENS = 64                     # b200vit_attention_window: tokens of one window
PEG_KERNEL_SIZES = (1, 3, 5, 7)            # b200vit_peg
CONV_PROJ_KERNEL_SIZES = (1, 3, 5, 7)      # b200vit_conv_proj_dw
GROUPS_WIDTHS = (8,)                       # b200vit_attention_groups
GROUPS_MAX_TOKENS = _lib.ATTN_GROUPS_MAX_TOKENS    # b200vit_attention_groups: tokens of one group
WINDOW_TOKEN_MAX_WINDOW = 7                # b200vit_attention_window_token: p*p tokens + the window token <= 64
WINDOW_MIX_MAX_WINDOWS = 64                # b200vit_window_mix: windows of one map
REGION_LOCAL_WIDTHS = (32,)                # b200vit_attention_region_local
REGION_LOCAL_MAX_TOKENS = 256              # b200vit_attention_region_local: a window's local tokens + its region token
REGION_MAX_TOKENS = 512                    # b200vit_attention over one image's region tokens
KV_EX_KEY_WIDTHS = (16, 32, 48, 64)        # b200vit_attention_kv_ex and b200vit_attention_iwsa: q / k head widths
KV_EX_VALUE_WIDTHS = (32, 64)              # ... and v head widths
ATTN_KV_MAX_KEYS = 16384                   # B200VIT_ATTN_KV_MAX_KEYS: keys per image or window


def head_width_reason(dh: int) -> Optional[str]:
    """None if the attention, head-norm and pooling kernels are built for heads `dh` wide, else the reason the eager
    PyTorch graph is used.  One rule for every model family."""
    if dh not in HEAD_WIDTHS:
        return f"dim_head={dh} (the attention kernels are built for 32, 64, 80 and 128)"
    return None


def headmix_reason(heads: int, dh: int) -> Optional[str]:
    """None if b200vit_attention_headmix is built for `heads` heads `dh` wide, else the reason the eager PyTorch graph
    is used."""
    if dh not in HEADMIX_WIDTHS:
        return f"dim_head={dh} (the head-mixing attention kernel is built for 32, 48, 64, 80 and 128)"
    if heads > HEADMIX_MAX_HEADS or heads * dh > HEADMIX_MAX_INNER:
        return (f"heads={heads} x dim_head={dh} (the head-mixing attention kernel takes at most "
                f"{HEADMIX_MAX_HEADS} heads and heads * dim_head <= {HEADMIX_MAX_INNER})")
    return None


def xca_reason(dh: int) -> Optional[str]:
    """None if b200vit_attention_xca is built for heads `dh` wide, else the reason the eager PyTorch graph is used."""
    if dh not in XCA_WIDTHS:
        return f"dim_head={dh} (the cross-covariance attention kernel is built for 32, 48, 64, 80 and 128)"
    return None


def lpi_reason(kernel_size: int, grid_w: int) -> Optional[str]:
    """None if b200vit_local_patch_interaction runs a k x k kernel over grid rows of `grid_w` tokens, else the reason
    the eager PyTorch graph is used.  The kernel keeps (3k - 1) padded grid rows of at least 4 channels in 100 KB of
    shared memory."""
    if kernel_size not in LPI_KERNEL_SIZES:
        return f"local_patch_kernel_size={kernel_size} (the local patch interaction kernel is built for 1, 3, 5 and 7)"
    if (3 * kernel_size - 1) * (grid_w + 2 * (kernel_size // 2)) * 4 * 4 > 100 * 1024:
        return f"a grid row of {grid_w} tokens is too wide for the local patch interaction kernel"
    return None


def kv_ex_reason(dk: int, dv: int, what: str) -> Optional[str]:
    """None if b200vit_attention_kv_ex / b200vit_attention_iwsa are built for key heads `dk` wide (after padding) and
    value heads `dv` wide, else the reason the eager PyTorch graph is used; `what` names the attention."""
    if dk not in KV_EX_KEY_WIDTHS or dv not in KV_EX_VALUE_WIDTHS:
        return (f"dim_key={dk}, dim_value={dv} (the {what} attention kernel is built for key heads 16, 32, 48 or 64 "
                f"and value heads 32 or 64 wide)")
    return None


def value_width(L: "EncoderLayer") -> int:
    """The width of layer L's value heads: L.dim_head, unless its attention record says otherwise."""
    A = L.attention
    return A.value_width(L) if hasattr(A, "value_width") else L.dim_head


def _rows_of(buf: torch.Tensor, cols: int) -> torch.Tensor:
    """A contiguous [rows, cols] view at the start of the workspace buffer `buf` (at least as many elements)."""
    if buf.shape[1] == cols:
        return buf
    return buf.view(-1)[: buf.shape[0] * cols].view(buf.shape[0], cols)


class Norm(NamedTuple):
    """A LayerNorm over the feature dim.  beta None: the norm has no shift."""
    gamma: torch.Tensor
    beta: Optional[torch.Tensor]
    eps: float

    @staticmethod
    def of(ln: nn.LayerNorm) -> "Norm":
        return Norm(ln.weight, ln.bias, ln.eps)


class AttnBlock(NamedTuple):
    """A second pre-LN attention sub-block of a layer (same heads, dim_head and scale as the first):
        x += out(attention(qkv(LN(x))))"""
    ln: Norm
    qkv_w: torch.Tensor                            # [3 * heads * dim_head, D], rows q | k | v
    out_w: Optional[torch.Tensor]                  # None: to_out is the identity, as EncoderLayer.out_w
    out_b: Optional[torch.Tensor]


class LPIBlock(NamedTuple):
    """XCiT's local patch interaction between the attention and the feed-forward block (xcit.py:150-167, 208-211), on
    the h x w token grid:  x += scale * conv2(GELU(BatchNorm(conv1(LN(x))))), conv1 / conv2 depthwise k x k with zero
    padding k // 2 (b200vit_local_patch_interaction).  BatchNorm runs on its running statistics (eval)."""
    ln: Norm
    conv1_w: torch.Tensor                         # [D, 1, k, k]
    conv1_b: Optional[torch.Tensor]
    bn_w: torch.Tensor
    bn_b: torch.Tensor
    bn_mean: torch.Tensor                         # running_mean, a buffer
    bn_var: torch.Tensor                          # running_var, a buffer
    bn_eps: float
    conv2_w: torch.Tensor                         # [D, 1, k, k]
    conv2_b: Optional[torch.Tensor]
    scale: Optional[torch.Tensor]                 # LayerScale [D], or None
    kernel_size: int


def lpi_weights(P: LPIBlock) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """(w1, b1, w2, b2) fp32 of b200vit_local_patch_interaction: BatchNorm (eval) folded into conv1,
        w1' = w1 g / sqrt(var + eps),  b1' = (b1 - mean) g / sqrt(var + eps) + beta,
    LayerScale s into conv2, w2' = s w2, b2' = s b2 (all per channel: the convolutions are depthwise); the weights
    tap-major [k*k, D]."""
    D, kk = P.conv1_w.shape[0], P.kernel_size * P.kernel_size
    f = lambda t: t.detach().float()                                                    # noqa: E731
    zeros = torch.zeros(D, device=P.conv1_w.device, dtype=torch.float32)
    inv = f(P.bn_w) / torch.sqrt(f(P.bn_var) + P.bn_eps)
    w1 = f(P.conv1_w).reshape(D, kk) * inv[:, None]
    b1 = ((f(P.conv1_b) if P.conv1_b is not None else zeros) - f(P.bn_mean)) * inv + f(P.bn_b)
    s = f(P.scale).reshape(D) if P.scale is not None else torch.ones_like(zeros)
    w2 = f(P.conv2_w).reshape(D, kk) * s[:, None]
    b2 = (f(P.conv2_b) if P.conv2_b is not None else zeros) * s
    return w1.t().contiguous(), b1.contiguous(), w2.t().contiguous(), b2.contiguous()


# ------------------------------------------------------------------------------------------------ attention variants
# EncoderLayer.attention is None (softmax attention over the layer's sequences) or one of the records below, each of
# which holds its variant's parameters and what the engine knows about it:
#   kernel, rejects   the name attention_kernel() reports, and its ValueError for `axial` or a packed batch
#   reason(L)         why the kernels are not built for layer L's widths or window, or None
#   geometry_reason(L, N, grid, groups, regions, rows)   why run_blocks' token geometry does not suit it, or None;
#                     `rows` = (B, rows of x) in run_blocks, None in unsupported_reason
#   prepare(t, i, L)  its prepared weights of layer i, into t
#   launch(c, L, i)   its launches in the BlocksCall c up to the attention output; returns the buffer holding it
#   o2 = True         (WindowTokenBlock only) launch() needs the workspace's second attention output


class HeadMix(NamedTuple):
    """Softmax probabilities mixed across the head axis (b200vit_attention_headmix; DeepViT's re-attention,
    deepvit.py:61-62): post indexed [input head, output head], ln a LayerNorm over the heads of every (query, key)
    pair after the mix; pre (CaiT's talking heads, cait.py:94) mixes the scores the same way before the softmax."""
    post: torch.Tensor                            # [heads, heads]
    ln: Optional[Norm]                            # over `heads` values, or None
    pre: Optional[torch.Tensor] = None            # [heads, heads], or None
    kernel = "headmix"
    rejects = "head-mixing attention runs over B sequences of N tokens only"

    def reason(self, L: EncoderLayer) -> Optional[str]:
        return headmix_reason(L.heads, L.dim_head)

    def geometry_reason(self, L: EncoderLayer, N: int, grid, groups, regions, rows=None) -> Optional[str]:
        return None

    def prepare(self, t: Dict[str, torch.Tensor], i: int, L: EncoderLayer) -> None:
        t[f"{i}.post"] = _f32(self.post)
        if self.pre is not None:
            t[f"{i}.pre"] = _f32(self.pre)
        if self.ln is not None:
            t[f"{i}.hln.w"], t[f"{i}.hln.b"] = _f32(self.ln.gamma), _f32(self.ln.beta)

    def launch(self, c: BlocksCall, L: EncoderLayer, i: int) -> torch.Tensor:
        c.project(L, i)
        hln = None if self.ln is None else (c.t[f"{i}.hln.w"], c.t[f"{i}.hln.b"], self.ln.eps)
        _lib.attention_headmix(c.qkv, c.o, c.B, c.N, L.heads, L.dim_head, L.scale, c.t[f"{i}.post"], hln,
                               pre=c.t.get(f"{i}.pre"))
        return c.o


class CrossCovariance(NamedTuple):
    """Cross-covariance attention (XCiT, xcit.py:109-148; b200vit_attention_xca) with the per-head temperature
    exp(tau), read when the prepared weights are rebuilt."""
    tau: torch.Tensor                             # the temperature parameter [heads, 1, 1]
    kernel = "xca"
    rejects = "cross-covariance attention runs over B sequences of N tokens only"

    def reason(self, L: EncoderLayer) -> Optional[str]:
        return xca_reason(L.dim_head)

    def geometry_reason(self, L: EncoderLayer, N: int, grid, groups, regions, rows=None) -> Optional[str]:
        return None

    def prepare(self, t: Dict[str, torch.Tensor], i: int, L: EncoderLayer) -> None:
        t[f"{i}.tau"] = self.tau.detach().float().exp().reshape(-1).contiguous()

    def launch(self, c: BlocksCall, L: EncoderLayer, i: int) -> torch.Tensor:
        c.project(L, i)
        _lib.attention_xca(c.qkv, c.t[f"{i}.tau"], c.o, c.B, c.N, L.heads, L.dim_head)
        return c.o


class Windows(NamedTuple):
    """Attention inside non-overlapping size x size blocks of the token grid (Twins-SVT's LocalAttention,
    twins_svt.py:85-120; b200vit_attention_window).  With `rel_pos_bias`, the Embedding weight [(2 size - 1)^2, heads],
    a learned relative-position bias inside every window (MaxViT, max_vit.py:148-159; b200vit_attention_window_relpos);
    `dilated` then cuts the map into dilated grids instead of contiguous blocks ('b d (w1 x) (w2 y)', max_vit.py:269).
    run_blocks needs `grid`."""
    size: int
    rel_pos_bias: Optional[torch.Tensor] = None
    dilated: bool = False
    rejects = "windowed and sub-sampled-key attention run over B token grids only"

    @property
    def kernel(self) -> str:
        return "window" if self.rel_pos_bias is None else "window_relpos"

    def reason(self, L: EncoderLayer) -> Optional[str]:
        r = head_width_reason(L.dim_head)
        if r is None and self.size ** 2 > WINDOW_MAX_TOKENS:
            name, what = ("local_patch_size", "window") if self.rel_pos_bias is None else \
                ("window_size", "relative-position window")
            r = (f"{name}={self.size}: a window of {self.size ** 2} tokens (the {what} attention kernel takes at "
                 f"most {WINDOW_MAX_TOKENS})")
        return r

    def geometry_reason(self, L: EncoderLayer, N: int, grid, groups, regions, rows=None) -> Optional[str]:
        if grid is None or grid[0] * grid[1] != N:
            return "windowed and sub-sampled-key attention need `grid` = (h, w) with h * w == N"
        if grid[0] % self.size or grid[1] % self.size:
            return f"a {grid[0]} x {grid[1]} grid cannot be cut into {self.size} x {self.size} windows"
        return None

    def prepare(self, t: Dict[str, torch.Tensor], i: int, L: EncoderLayer) -> None:
        if self.rel_pos_bias is not None:
            t[f"{i}.relpos"] = self.rel_pos_bias.detach().float().t().contiguous()

    def launch(self, c: BlocksCall, L: EncoderLayer, i: int) -> torch.Tensor:
        c.project(L, i)
        if self.rel_pos_bias is None:
            _lib.attention_window(c.qkv, c.o, c.B, c.grid[0], c.grid[1], self.size, L.heads, L.dim_head, L.scale)
        else:
            _lib.attention_window_relpos(c.qkv, c.o, c.t[f"{i}.relpos"], c.B, c.grid[0], c.grid[1], self.size,
                                         self.dilated, L.heads, L.dim_head, L.scale)
        return c.o


class StridedKV(NamedTuple):
    """Keys and values from a stride x stride, stride-`stride` convolution of the normalised token grid (Twins-SVT's
    GlobalAttention, twins_svt.py:122-157; b200vit_attention_kv); EncoderLayer.qkv_w holds the query rows only.
    run_blocks needs `grid`.  The LayerNorm cannot be folded into the key / value projection (one convolution window
    spans tokens with different statistics): in both LayerNorm modes the layer runs layernorm(x -> xb), the query GEMM
    on xb, conv_im2col_nhwc of xb and the key / value GEMM (stride 1: the GEMM on xb itself), then attention_kv.
    `dim_value`: value heads of another width than L.dim_head, the key heads (ScalableViT's SSA, scalable_vit.py:71-124;
    b200vit_attention_kv_ex); kv_w then has heads * (dim_head + dim_value) rows and the output heads * dim_value
    columns.  None: dim_value == dim_head."""
    stride: int
    kv_w: torch.Tensor                            # the Conv2d weight [heads * (dk + dv), D, k, k], rows k | v
    dim_value: Optional[int] = None
    kernel = "kv"
    rejects = Windows.rejects

    def reason(self, L: EncoderLayer) -> Optional[str]:
        if self.dim_value is None:
            return head_width_reason(L.dim_head)
        return kv_ex_reason(L.dim_head, self.dim_value, "sub-sampled-key")

    def value_width(self, L: EncoderLayer) -> int:
        return L.dim_head if self.dim_value is None else self.dim_value

    def geometry_reason(self, L: EncoderLayer, N: int, grid, groups, regions, rows=None) -> Optional[str]:
        if grid is None or grid[0] * grid[1] != N:
            return "windowed and sub-sampled-key attention need `grid` = (h, w) with h * w == N"
        if min(grid) < self.stride:
            return f"a {grid[0]} x {grid[1]} grid cannot be cut into {self.stride} x {self.stride} key patches"
        return None

    def prepare(self, t: Dict[str, torch.Tensor], i: int, L: EncoderLayer) -> None:
        # the Conv2d weight in the column order of b200vit_conv_im2col_nhwc: (tap row, tap column, channel)
        t[f"{i}.kv.w"] = _bf16_rows(self.kv_w.detach().permute(0, 2, 3, 1).reshape(self.kv_w.shape[0], -1))

    def launch(self, c: BlocksCall, L: EncoderLayer, i: int) -> torch.Tensor:
        x, xb, t, k = c.x, c.xb, c.t, self.stride
        I, (gh, gw) = L.heads * L.dim_head, c.grid
        kh, kw = gh // k, gw // k
        _lib.layernorm(x, t[f"{i}.ln1.w"], t[f"{i}.ln1.b"], out_bf16=xb, eps=L.ln1.eps)
        q = c.qkv[:, :I]
        _lib.gemm(xb, t[f"{i}.qkv.w"], out_bf16=q)
        if k == 1:
            col = xb
        else:
            col = torch.empty(c.B * kh * kw, k * k * x.shape[1], device=x.device, dtype=torch.bfloat16)
            _lib.conv_im2col_nhwc(xb, col, c.B, gh, gw, k, k, 0)
        kv = torch.empty(c.B * kh * kw, self.kv_w.shape[0], device=x.device, dtype=torch.bfloat16)
        _lib.gemm(col, t[f"{i}.kv.w"], out_bf16=kv)
        if self.dim_value is None:
            _lib.attention_kv(q, kv, c.o, c.B, c.N, kh * kw, L.heads, L.dim_head, L.scale)
            return c.o
        o = _rows_of(c.o, L.heads * self.dim_value)
        _lib.attention_kv_ex(q, kv, o, c.B, c.N, kh * kw, L.heads, L.dim_head, self.dim_value, L.scale)
        return o


class InteractiveWindows(NamedTuple):
    """ScalableViT's interactive windowed self-attention (scalable_vit.py:126-194; b200vit_attention_iwsa): attention
    inside size x size windows of the token grid (None: the whole grid) plus the local interactive module, a dense
    3 x 3 convolution with bias and zero padding 1 of the value map, added to the attention output before the
    out-projection.  EncoderLayer.qkv_w holds the rows q | k | v, the q and k heads L.dim_head wide, the v heads
    lim_w.shape[0] / heads.  The layer runs the QKV projection (c.project), conv_im2col_nhwc over the v columns of
    qkv, the convolution's GEMM with its bias into a bf16 `lim` buffer, then attention_iwsa.  run_blocks needs `grid`."""
    size: Optional[int]
    lim_w: torch.Tensor                           # local_interactive_module.weight [heads * dv, heads * dv, 3, 3]
    lim_b: torch.Tensor
    kernel = "iwsa"
    rejects = "interactive windowed attention runs over B token grids only"

    def value_width(self, L: EncoderLayer) -> int:
        return self.lim_w.shape[0] // L.heads

    def window(self, grid: Tuple[int, int]) -> Tuple[int, int]:
        return (grid[0], grid[1]) if self.size is None else (self.size, self.size)

    def reason(self, L: EncoderLayer) -> Optional[str]:
        r = kv_ex_reason(L.dim_head, self.value_width(L), "interactive windowed")
        if r is None and self.size is not None and self.size ** 2 > ATTN_KV_MAX_KEYS:
            r = (f"window_size={self.size}: a window of {self.size ** 2} tokens (the interactive windowed attention "
                 f"kernel takes at most {ATTN_KV_MAX_KEYS})")
        return r

    def geometry_reason(self, L: EncoderLayer, N: int, grid, groups, regions, rows=None) -> Optional[str]:
        if grid is None or grid[0] * grid[1] != N:
            return "interactive windowed attention needs `grid` = (h, w) with h * w == N"
        wh, ww = self.window(grid)
        if grid[0] % wh or grid[1] % ww:
            # the reference's assertion (scalable_vit.py:161)
            return (f"height ({grid[0]}) or width ({grid[1]}) of feature map is not divisible by the window size "
                    f"({wh}, {ww})")
        if wh * ww > ATTN_KV_MAX_KEYS:
            return (f"a {wh} x {ww} window of {wh * ww} tokens (the interactive windowed attention kernel takes at "
                    f"most {ATTN_KV_MAX_KEYS})")
        return None

    def prepare(self, t: Dict[str, torch.Tensor], i: int, L: EncoderLayer) -> None:
        # the Conv2d weight in the column order of b200vit_conv_im2col_nhwc: (tap row, tap column, channel)
        w = self.lim_w.detach()
        t[f"{i}.lim.w"] = _bf16_rows(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1))
        t[f"{i}.lim.b"] = _f32(self.lim_b)

    def launch(self, c: BlocksCall, L: EncoderLayer, i: int) -> torch.Tensor:
        t, (gh, gw), M = c.t, c.grid, c.x.shape[0]
        Ik, dv = L.heads * L.dim_head, self.value_width(L)
        Iv = L.heads * dv
        qkv = _rows_of(c.qkv, L.qkv_w.shape[0])
        c.project(L, i, out=qkv)
        col = torch.empty(M, 9 * Iv, device=c.x.device, dtype=torch.bfloat16)
        _lib.conv_im2col_nhwc(qkv[:, 2 * Ik:], col, c.B, gh, gw, 3, 1, 1)
        lim = torch.empty(M, Iv, device=c.x.device, dtype=torch.bfloat16)
        _lib.gemm(col, t[f"{i}.lim.w"], out_bf16=lim, bias=t[f"{i}.lim.b"])
        o = _rows_of(c.o, Iv)
        wh, ww = self.window(c.grid)
        _lib.attention_iwsa(qkv, lim, o, c.B, gh, gw, wh, ww, L.heads, L.dim_head, dv, L.scale)
        return o


class PatchGroups(NamedTuple):
    """Attention inside the strided patch groups of the token grid, token (y'*ph + i, x'*pw + j) in group (i, j)
    (MobileViT, mobile_vit.py:150; b200vit_attention_groups); run_blocks needs `grid` and `groups` = (ph, pw).  It has
    no fields, so it is an empty tuple: test EncoderLayer.attention against None, never for truth."""
    kernel = "groups"
    rejects = "patch-group attention runs over B token grids only"

    def reason(self, L: EncoderLayer) -> Optional[str]:
        if L.dim_head not in GROUPS_WIDTHS:
            return f"dim_head={L.dim_head} (the patch-group attention kernel is built for 8)"
        return None

    def geometry_reason(self, L: EncoderLayer, N: int, grid, groups, regions, rows=None) -> Optional[str]:
        if grid is None or grid[0] * grid[1] != N or groups is None:
            return "patch-group attention needs `grid` = (h, w) with h * w == N and `groups`"
        if grid[0] % groups[0] or grid[1] % groups[1]:
            return f"a {grid[0]} x {grid[1]} grid cannot be cut into {groups[0]} x {groups[1]} patches"
        n = (grid[0] // groups[0]) * (grid[1] // groups[1])
        if not 1 <= n <= GROUPS_MAX_TOKENS:
            return f"{n} tokens per group (the patch-group attention kernel takes 1 to {GROUPS_MAX_TOKENS})"
        return None

    def prepare(self, t: Dict[str, torch.Tensor], i: int, L: EncoderLayer) -> None:
        pass

    def launch(self, c: BlocksCall, L: EncoderLayer, i: int) -> torch.Tensor:
        c.project(L, i)
        _lib.attention_groups(c.qkv, c.o, c.B, c.grid[0], c.grid[1], c.groups[0], c.groups[1], L.heads, L.dim_head,
                              L.scale)
        return c.o


class ConvProj(NamedTuple):
    """CvT's convolutional projections (cvt.py:51-60, 74-75) of the normalised h x w token grid: for the queries a
    depthwise k x k convolution at stride 1, for the keys / values one at stride `stride`, both bias-free with zero
    padding k // 2 and followed by a BatchNorm (eval, on its running statistics); the bias-free 1 x 1 convolutions
    after them are EncoderLayer.qkv_w (queries) and kv_proj_w (keys | values).  The attention runs b200vit_conv_proj_dw,
    then b200vit_attention_kv; run_blocks needs `grid`, of any h, w >= 1 (the projections pad)."""
    q_w: torch.Tensor                             # [D, 1, k, k]
    q_bn_w: torch.Tensor
    q_bn_b: torch.Tensor
    q_bn_mean: torch.Tensor                       # running_mean, a buffer
    q_bn_var: torch.Tensor                        # running_var, a buffer
    q_bn_eps: float
    kv_w: torch.Tensor                            # [D, 1, k, k]
    kv_bn_w: torch.Tensor
    kv_bn_b: torch.Tensor
    kv_bn_mean: torch.Tensor
    kv_bn_var: torch.Tensor
    kv_bn_eps: float
    kernel_size: int
    stride: int
    kv_proj_w: Optional[torch.Tensor] = None      # [2 * heads * dim_head, D], rows k | v; an encoder layer needs it
    kernel = "kv"
    rejects = Windows.rejects

    def grid(self, h: int, w: int) -> Tuple[int, int]:
        """The (h, w) of the key / value map of an h x w token grid."""
        return (h - 1) // self.stride + 1, (w - 1) // self.stride + 1

    def reason(self, L: EncoderLayer) -> Optional[str]:
        r = head_width_reason(L.dim_head)
        if r is None and self.kernel_size not in CONV_PROJ_KERNEL_SIZES:
            r = f"proj_kernel={self.kernel_size} (the convolutional-projection kernel is built for 1, 3, 5 and 7)"
        return r

    def geometry_reason(self, L: EncoderLayer, N: int, grid, groups, regions, rows=None) -> Optional[str]:
        if grid is None or grid[0] * grid[1] != N:
            return "windowed and sub-sampled-key attention need `grid` = (h, w) with h * w == N"
        return None

    def prepare(self, t: Dict[str, torch.Tensor], i: int, L: EncoderLayer) -> None:
        # the depthwise halves with their BatchNorms folded (tap-major) and the keys' / values' 1 x 1 rows
        t[f"{i}.cpq.w"], t[f"{i}.cpq.b"], t[f"{i}.cpkv.w"], t[f"{i}.cpkv.b"] = conv_proj_weights(self)
        t[f"{i}.kv.w"] = _bf16_rows(self.kv_proj_w.reshape(self.kv_proj_w.shape[0], -1))

    def launch(self, c: BlocksCall, L: EncoderLayer, i: int) -> torch.Tensor:
        """layernorm(x -> xb), both depthwise projections of xb in one pass (the LayerNorm cannot be folded: the
        padding taps must read zeros of the normalised map), the 1 x 1 GEMMs, attention_kv."""
        x, xb, t = c.x, c.xb, c.t
        I, D = L.heads * L.dim_head, x.shape[1]
        kh, kw = self.grid(*c.grid)
        _lib.layernorm(x, t[f"{i}.ln1.w"], t[f"{i}.ln1.b"], out_bf16=xb, eps=L.ln1.eps)
        aq = torch.empty(x.shape[0], D, device=x.device, dtype=torch.bfloat16)
        akv = torch.empty(c.B * kh * kw, D, device=x.device, dtype=torch.bfloat16)
        _lib.conv_proj_dw(xb, t[f"{i}.cpq.w"], t[f"{i}.cpq.b"], t[f"{i}.cpkv.w"], t[f"{i}.cpkv.b"], aq, akv, c.B,
                          c.grid[0], c.grid[1], self.kernel_size, self.stride)
        q = c.qkv[:, :I]
        _lib.gemm(aq, t[f"{i}.qkv.w"], out_bf16=q)
        kv = torch.empty(c.B * kh * kw, 2 * I, device=x.device, dtype=torch.bfloat16)
        _lib.gemm(akv, t[f"{i}.kv.w"], out_bf16=kv)
        _lib.attention_kv(q, kv, c.o, c.B, c.N, kh * kw, L.heads, L.dim_head, L.scale)
        return c.o


def conv_proj_weights(P: ConvProj) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """(wq, bq, wkv, bkv) fp32 of b200vit_conv_proj_dw: each BatchNorm (eval) folded into its bias-free depthwise
    convolution, w' = w g / sqrt(var + eps), b' = beta - mean g / sqrt(var + eps); the weights tap-major [k*k, D]."""
    f = lambda t: t.detach().float()                                                    # noqa: E731
    out = []
    for w, g, beta, mean, var, eps in ((P.q_w, P.q_bn_w, P.q_bn_b, P.q_bn_mean, P.q_bn_var, P.q_bn_eps),
                                       (P.kv_w, P.kv_bn_w, P.kv_bn_b, P.kv_bn_mean, P.kv_bn_var, P.kv_bn_eps)):
        inv = f(g) / torch.sqrt(f(var) + eps)
        out.append((f(w).reshape(w.shape[0], -1) * inv[:, None]).t().contiguous())
        out.append((f(beta) - f(mean) * inv).contiguous())
    return out[0], out[1], out[2], out[3]


class WindowTokenBlock(NamedTuple):
    """SepViT's window token and the attention across windows it drives (DSSA, sep_vit.py:91-102, 139-205): `token`
    [D] joins every p x p window as one more key, value and query of the layer's own (bias-free) qkv projection, not
    normalised; its per-head outputs pass `ln` (nn.LayerNorm(dim_head), shared by the heads), GELU and the 1 x 1
    convolution wqk_w [2I, I] + wqk_b over the heads' channels, whose output columns interleave per head (q of head h
    at [2h dh, 2h dh + dh), its k right after); softmax(scale wq wk^T) over the windows then mixes the windows' outputs
    position by position (b200vit_attention_window_token, b200vit_head_layernorm_gelu, GEMM, b200vit_window_mix).
    run_blocks needs `grid`, cut into at most 64 windows."""
    token: torch.Tensor                           # [D], a parameter
    ln: Norm                                      # over dim_head values
    wqk_w: torch.Tensor                           # [2I, I] (the Conv1d weight [2I, I, 1] reshaped)
    wqk_b: torch.Tensor                           # [2I]
    window: int
    kernel = "window_token"
    rejects = "window-token attention runs over B token grids only"
    o2 = True                                     # launch() writes the workspace's second attention output

    def reason(self, L: EncoderLayer) -> Optional[str]:
        r, p = head_width_reason(L.dim_head), self.window
        if r is None and p > WINDOW_TOKEN_MAX_WINDOW:
            r = (f"window_size={p}: a window of {p ** 2} tokens and its window token (the window-token attention "
                 f"kernel takes windows up to {WINDOW_TOKEN_MAX_WINDOW} x {WINDOW_TOKEN_MAX_WINDOW})")
        return r

    def geometry_reason(self, L: EncoderLayer, N: int, grid, groups, regions, rows=None) -> Optional[str]:
        p = self.window
        if grid is None or grid[0] * grid[1] != N:
            return "window-token attention needs `grid` = (h, w) with h * w == N"
        if grid[0] % p or grid[1] % p:
            return f"a {grid[0]} x {grid[1]} grid cannot be cut into {p} x {p} windows"
        nw = (grid[0] // p) * (grid[1] // p)
        if nw > WINDOW_MIX_MAX_WINDOWS:
            return (f"a {grid[0]} x {grid[1]} grid has {nw} windows of {p} x {p}, more than {WINDOW_MIX_MAX_WINDOWS} "
                    f"(the window-mixing kernel's limit)")
        return None

    def prepare(self, t: Dict[str, torch.Tensor], i: int, L: EncoderLayer) -> None:
        # the window token's q | k | v: the same for every window, so projected once, in fp32, then rounded
        t[f"{i}.tok_qkv"] = (L.qkv_w.detach().float() @ self.token.detach().float()).to(torch.bfloat16)
        t[f"{i}.wt.ln.w"], t[f"{i}.wt.ln.b"] = _f32(self.ln.gamma), _f32(self.ln.beta)
        t[f"{i}.wqk.w"], t[f"{i}.wqk.b"] = _bf16_rows(self.wqk_w), _f32(self.wqk_b)

    def launch(self, c: BlocksCall, L: EncoderLayer, i: int) -> torch.Tensor:
        """The QKV projection, then the windows' attention with their window token into o; with more than one window,
        the window tokens' outputs -> LayerNorm + GELU -> their q | k GEMM -> the attention across windows into o2."""
        c.project(L, i)
        t, I = c.t, L.heads * L.dim_head
        (gh, gw), p = c.grid, self.window
        nw = (gh // p) * (gw // p)
        if nw == 1:           # the window token is a key and a value, its own output unused (sep_vit.py:176-178)
            _lib.attention_window_token(c.qkv, t[f"{i}.tok_qkv"], c.o, None, c.B, gh, gw, p, L.heads, L.dim_head,
                                        L.scale)
            return c.o
        tok = torch.empty(c.B * nw, I, device=c.x.device, dtype=torch.bfloat16)
        _lib.attention_window_token(c.qkv, t[f"{i}.tok_qkv"], c.o, tok, c.B, gh, gw, p, L.heads, L.dim_head, L.scale)
        _lib.head_layernorm_gelu(tok, t[f"{i}.wt.ln.w"], t[f"{i}.wt.ln.b"], L.heads, L.dim_head, eps=self.ln.eps)
        wqk = torch.empty(c.B * nw, 2 * I, device=c.x.device, dtype=torch.bfloat16)
        _lib.gemm(tok, t[f"{i}.wqk.w"], out_bf16=wqk, bias=t[f"{i}.wqk.b"])
        mixed = c.ws["o2"]
        _lib.window_mix(wqk, c.o, mixed, c.B, gh, gw, p, L.heads, L.dim_head, L.scale)
        return mixed


class RegionLocalBlock(NamedTuple):
    """RegionViT's region-to-local attention (R2LTransformer, regionvit.py:114-190): the layer's attention runs over
    the region tokens alone, then inside every window of local tokens together with the window's region token, with
    the learned relative-position bias `bias` between local tokens (b200vit_attention, then
    b200vit_attention_region_local); `window` is the W the bias table was built for, (2W-1)^2 offsets.  run_blocks
    takes x = B*N local rows (the `grid` maps, N = h*w) followed by the B*rh*rw rows of the `regions` = (rh, rw) maps;
    the windows are (h/rh) x (w/rw) local tokens, at most 255."""
    bias: torch.Tensor                            # local_rel_pos_bias.weight [(2W-1)^2, heads], a parameter
    window: int
    kernel = "region_local"
    rejects = "region-to-local attention runs over B local and region token maps only"

    def reason(self, L: EncoderLayer) -> Optional[str]:
        r = head_width_reason(L.dim_head)
        if r is None and L.dim_head not in REGION_LOCAL_WIDTHS:
            r = f"dim_head={L.dim_head} (the region-to-local attention kernel is built for 32)"
        return r

    def geometry_reason(self, L: EncoderLayer, N: int, grid, groups, regions, rows=None) -> Optional[str]:
        if grid is None or regions is None or grid[0] * grid[1] != N:
            return "region-to-local attention needs `grid` = (h, w) with h * w == N and `regions` = (rh, rw)"
        (lh, lw), (rh, rw) = grid, regions
        if rows is not None and rows[1] != rows[0] * (N + rh * rw):
            return (f"x has {rows[1]} rows, not the B * (N + rh * rw) = {rows[0] * (N + rh * rw)} of B local and "
                    f"region maps")
        if lh % rh or lw % rw:
            return f"the {lh} x {lw} local map does not split into the {rh} x {rw} region map"
        wh, ww = lh // rh, lw // rw
        if wh > self.window or ww > self.window:
            return f"a {wh} x {ww} window is larger than window_size={self.window} of the relative-position bias"
        if wh * ww + 1 > REGION_LOCAL_MAX_TOKENS:
            return (f"a {wh} x {ww} window of {wh * ww} local tokens (the region-to-local attention kernel takes at "
                    f"most {REGION_LOCAL_MAX_TOKENS - 1})")
        if rh * rw > REGION_MAX_TOKENS:
            return f"a {rh} x {rw} region map (regional attention takes at most {REGION_MAX_TOKENS} tokens)"
        return None

    def prepare(self, t: Dict[str, torch.Tensor], i: int, L: EncoderLayer) -> None:
        t[f"{i}.r2l"] = self.bias.detach().float().t().contiguous()     # [heads, (2W-1)^2]

    def launch(self, c: BlocksCall, L: EncoderLayer, i: int) -> torch.Tensor:
        """The QKV GEMM, attention over each image's region tokens and the out-projection residual on the region rows
        alone (pointer offsets into x, its bf16 copy and its statistics), then the QKV GEMM over all rows and the
        region-to-local attention into o.  In fold mode the region residual writes the region rows' statistics where
        the next QKV GEMM reads them; right after a rowstats_cast prime (one part per row) the region rows take the
        exact LayerNorm and one rowstats_cast of the region rows writes their statistics instead."""
        t, x, xb, qkv, o = c.t, c.x, c.xb, c.qkv, c.o
        Ml, (rh, rw) = c.B * c.N, c.regions
        xr, xbr = x[Ml:], xb[Ml:]
        if c.fold and c.sums is None:
            c.sums = c.ws["stats_in"]
            _lib.rowstats_cast(x, xb, c.sums)
        sums = c.sums
        # the residual GEMMs' statistics: the folded GEMM reads them from row Ml on.  A rowstats_cast prime (one part
        # per row) is read there only 8 bytes per row in, which the GEMM's 16-byte rule does not allow for odd Ml: the
        # region rows then take the exact LayerNorm, and their new statistics a rowstats_cast
        gemm_stats = c.fold and sums is not c.ws["stats_in"]
        if gemm_stats:
            _lib.gemm(xbr, t[f"{i}.qkv.wg"], out_bf16=qkv[Ml:], bias=t[f"{i}.qkv.t"], ln_sums=sums[Ml:],
                      col_s=t[f"{i}.qkv.s"], ln_eps=L.ln1.eps)
        else:
            _lib.layernorm(xr, t[f"{i}.ln1.w"], t[f"{i}.ln1.b"], out_bf16=xbr, eps=L.ln1.eps)
            _lib.gemm(xbr, t[f"{i}.qkv.w"], out_bf16=qkv[Ml:])
        _lib.attention(qkv[Ml:], o[Ml:], c.B, rh * rw, L.heads, L.dim_head, L.scale)
        _lib.gemm(o[Ml:], t[f"{i}.out.w"], out_f32=xr, out_bf16=xbr if gemm_stats else None, bias=t[f"{i}.out.b"],
                  resid=xr, stats_out=sums[Ml:] if gemm_stats else None)
        if c.fold and not gemm_stats:
            _lib.rowstats_cast(xr, xbr, sums[Ml:])
        c.normed(x, f"{i}.ln1", L.ln1, f"{i}.qkv", qkv)
        _lib.attention_region_local(qkv, o, t[f"{i}.r2l"], c.B, c.grid[0], c.grid[1], rh, rw, self.window, L.heads,
                                    L.dim_head, L.scale)
        return o


AttentionVariant = Union[HeadMix, CrossCovariance, Windows, StridedKV, InteractiveWindows, ConvProj, PatchGroups,
                         WindowTokenBlock, RegionLocalBlock]


@dataclass
class EncoderLayer:
    """One pre-LN encoder layer as a model family describes it to the engine (reference vit.py:78-81):
        x += out(attention(qkv(LN1(x))))        x += fc2(GELU(fc1(LN2(x))))
    The tensors are the module's own parameters; TransformerEngine.prepared() derives the device copies from them."""
    ln1: Norm
    qkv_w: torch.Tensor                            # [3 * heads * dim_head, D], rows q | k | v
    out_w: Optional[torch.Tensor]                  # None: to_out is the identity (heads == 1 and dim_head == D)
    out_b: Optional[torch.Tensor]
    ln2: Norm
    fc1_w: torch.Tensor
    fc1_b: torch.Tensor
    fc2_w: torch.Tensor
    fc2_b: torch.Tensor
    heads: int
    dim_head: int
    scale: float                                   # softmax scale
    qk_norm: Optional[str] = None                  # per-head norm of q and k after the projection: None, "rms" or "ln"
    qk_gamma: Tuple[torch.Tensor, ...] = ()        # (q gamma, k gamma), each heads * dim_head values
    qk_eps: float = 0.0                            # eps of the "ln" head norm
    # attention along the time axis between the attention and the feed-forward block (ViViT's FactorizedTransformer,
    # reference vivit.py:144-150); run_blocks needs `axial` to address its sequences
    temporal: Optional[AttnBlock] = None
    # each query's own key excluded from its softmax (LSA, vit_for_small_dataset.py:53-57)
    mask_self: bool = False
    # the attention variant: None for softmax attention over the layer's sequences, else its record (see above)
    attention: Optional[AttentionVariant] = None
    # LayerScale (cait.py:31-45): the attention and feed-forward outputs multiplied by these [D] vectors before their
    # residual adds, folded into the rows and biases of out_w and fc2_w
    out_scale: Optional[torch.Tensor] = None
    ff_scale: Optional[torch.Tensor] = None
    # local patch interaction between the attention and the feed-forward block (XCiT); run_blocks needs `grid`
    lpi: Optional[LPIBlock] = None
    # `ln2` replaces the stream: x = LN2(x); x += fc2(GELU(fc1(x))) (cct.py:137-142)
    post_norm: bool = False
    # the feed-forward block's activation: "gelu" (vit.py:21) or "silu" (MobileViT's FeedForward, mobile_vit.py:28-34)
    ff_act: str = "gelu"
    # the feed-forward block runs before the attention: x += fc2(GELU(fc1(LN2(x)))); x += out(attention(...)) (the
    # second half of a ScalableViT layer, scalable_vit.py:228-236); not with lpi, post_norm or temporal
    ff_first: bool = False


def attention_kernel(L: EncoderLayer, axial: bool = False, packed: bool = False, key_blocks: bool = False) -> str:
    """Which kernel runs layer L's attention: its record's `kernel` ('headmix', 'xca', 'window', 'window_relpos', 'kv',
    'iwsa', 'groups', 'window_token' or 'region_local'), or for softmax attention 'axial' (a run_blocks call with
    `axial`, unless the layer's temporal sub-block runs there), 'varlen' (`key_blocks`: a packed batch, or more than 512
    keys) or 'plain'.  ValueError for an attention variant with `axial` or over a `packed` batch."""
    A = L.attention
    if A is not None:
        if axial or packed:
            raise ValueError(A.rejects)
        return A.kernel
    if axial and L.temporal is None:
        return "axial"
    return "varlen" if key_blocks else "plain"


class _Prepared:
    """What was derived from some parameters (usually flat device buffers) + the parameter versions it was built from."""

    def __init__(self) -> None:
        self.key: Optional[tuple] = None
        self.t = None

    def get(self, params: List[torch.Tensor], build, *extra_key):
        """build()'s result, rebuilt only when a version of `params` (or `extra_key`) has changed since the last call."""
        key = _version_key(params) + extra_key
        if self.key != key:
            self.t, self.key = build(), key
        return self.t


def cached(owner, name: str, params: List[torch.Tensor], build, *extra_key):
    """_Prepared.get on the _Prepared kept on `owner` under `name` (made on first use)."""
    prep = owner.__dict__.get(name)
    if prep is None:
        prep = owner.__dict__[name] = _Prepared()
    return prep.get(params, build, *extra_key)


# bumped by refresh_fused_weights(): part of every prepared-weight key, so one call invalidates every engine of the
# process.  (p._version catches in-place ops on the parameter; writes through `p.data` -- EMA updates, manual
# weight loading -- do NOT bump it, hence the explicit epoch; load_state_dict / .to() / .half() of the drop-in
# modules call refresh_fused_weights() themselves.)
_WEIGHT_EPOCH = [0]


def refresh_fused_weights() -> None:
    """Drop every cached bf16 / LN-folded copy of the parameters; the next fused forward rebuilds them."""
    _WEIGHT_EPOCH[0] += 1


def _version_key(params: List[torch.Tensor]) -> tuple:
    return (_WEIGHT_EPOCH[0],) + tuple((p.data_ptr(), p._version) for p in params)


class FusedWeightsMixin:
    """nn.Module mixin: state-changing entry points that bypass parameter versions invalidate the fused copies."""

    def refresh_fused_weights(self) -> None:
        refresh_fused_weights()

    def load_state_dict(self, *args, **kwargs):            # copy_ under no_grad bumps _version, but be explicit
        out = super().load_state_dict(*args, **kwargs)
        refresh_fused_weights()
        return out

    def _apply(self, fn, *args, **kwargs):                 # .to() / .cuda() / .bfloat16(): new storages
        out = super()._apply(fn, *args, **kwargs)
        refresh_fused_weights()
        return out


def _f32(p: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    return None if p is None else p.detach().float().contiguous()


def _bf16_rows(p: torch.Tensor, k_pad: Optional[int] = None) -> torch.Tensor:
    """[out, in] weight as contiguous bf16 with the K dim padded to `k_pad` (zeros) for TMA's 16-byte row rule."""
    w = p.detach()
    if k_pad is not None and k_pad != w.shape[1]:
        wp = torch.zeros(w.shape[0], k_pad, device=w.device, dtype=torch.bfloat16)
        wp[:, : w.shape[1]] = w
        return wp
    return w.to(torch.bfloat16).contiguous()


def _scaled_rows(w: torch.Tensor, b: Optional[torch.Tensor], scale: Optional[torch.Tensor]
                 ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """(bf16 weight, fp32 bias) of a Linear whose output is multiplied by `scale` [out] (LayerScale): rows and bias
    scaled in fp32, then rounded."""
    if scale is None:
        return _bf16_rows(w), _f32(b)
    s = scale.detach().float().reshape(-1)
    ws = (w.detach().float() * s[:, None]).to(torch.bfloat16).contiguous()
    return ws, None if b is None else (b.detach().float() * s).contiguous()


def _fold(t: Dict[str, torch.Tensor], prefix: str, w: torch.Tensor, b: Optional[torch.Tensor], ln: Norm) -> None:
    """LayerNorm folded into the Linear that follows it:
        LN(x) W^T + b  ==  rstd * (x (gamma*W)^T - mu * colsum) + (W beta + b)
    t[prefix + '.wg'] = gamma*W (bf16), '.s' = its row sums, '.t' = W beta + b (just b, or zeros, when beta is None)."""
    w32 = w.detach().float()
    wg = (w32 * ln.gamma.detach().float()[None, :]).to(torch.bfloat16).contiguous()
    t[prefix + ".wg"] = wg
    t[prefix + ".s"] = wg.float().sum(dim=1).contiguous()          # from the ROUNDED weights the MMA sees
    if ln.beta is None:
        # still a bias vector: the GEMM keeps its bias epilogue whether or not the LayerNorm has a shift
        t[prefix + ".t"] = _f32(b) if b is not None else torch.zeros(w.shape[0], device=w.device, dtype=torch.float32)
    else:
        tb = w32 @ ln.beta.detach().float()
        t[prefix + ".t"] = (tb + b.detach().float() if b is not None else tb).contiguous()


def depthwise_peg_weights(conv: nn.Conv2d) -> dict:
    """'w' fp32 [k*k, C] (the depthwise k x k weights tap major) and 'b' fp32 [C] of b200vit_peg, from the PEG's
    Conv2d(C, C, k, padding=k // 2, groups=C) (Twins-SVT, twins_svt.py:77-83; ScalableViT, scalable_vit.py:44-50)."""
    C, kk = conv.weight.shape[0], conv.kernel_size[0] ** 2
    bias = _f32(conv.bias) if conv.bias is not None else torch.zeros(C, device=conv.weight.device)
    return {"w": conv.weight.detach().float().reshape(C, kk).t().contiguous(), "b": bias}


class Workspace:
    """Scratch buffers of a TransformerEngine: `t` by name, `c` the _lib.EncoderWs over them, `key` what they were
    allocated for (rows, device, stream)."""

    def __init__(self) -> None:
        self.key: Optional[tuple] = None
        self.t: Dict[str, torch.Tensor] = {}
        self.c = None


class FusedEncoder:
    """nn.Module mixin of the Transformers the engine runs.  A class using it provides
        encoder_layers() -> (List[EncoderLayer], final Norm or None)
    and gets engine(), its TransformerEngine (made on first use, kept with the module)."""

    def engine(self) -> "TransformerEngine":
        eng = getattr(self, "_engine", None)
        if eng is None:
            eng = self._engine = TransformerEngine(self)
        return eng


class BlocksCall:
    """What the launches of one run_blocks call on the per-kernel loop share: the prepared weights `t`, the workspace
    `ws` and its buffers xb (the bf16 copy of x), qkv, o and h, the fp32 residual stream x, the call's arguments and
    `sums`, in fold mode the row sums of xb that the next LN-folded GEMM reads (None until a pass writes them)."""

    def __init__(self, t: Dict[str, torch.Tensor], ws: Dict[str, torch.Tensor], x: torch.Tensor, B: int, N: int,
                 grid, groups, regions, rope, axial, vl, fold: bool, primed: bool) -> None:
        self.t, self.ws, self.x, self.fold = t, ws, x, fold
        self.xb, self.qkv, self.o, self.h = ws["xn"], ws["qkv"], ws["o"], ws["h"]
        self.B, self.N, self.grid, self.groups, self.regions = B, N, grid, groups, regions
        self.rope, self.axial, self.vl = rope, axial, vl
        self.sums = ws["stats_in"] if primed else None

    def normed(self, src: torch.Tensor, ln: str, norm: Norm, w: str, out: torch.Tensor, **epi) -> None:
        """out = LN(src) W^T, LN = t[ln + '.w' / '.b'] with norm.eps, W the Linear t[w + ...].  fold: the LN-folded
        GEMM on xb and `sums` (made by one rowstats_cast pass if not primed); exact: layernorm(src -> xb), then the
        plain GEMM with the Linear's bias if it has one.  `epi` with head_gamma (a q / k norm): gemm_headnorm."""
        t, xb = self.t, self.xb
        if self.fold:
            if self.sums is None:
                self.sums = self.ws["stats_in"]
                _lib.rowstats_cast(src, xb, self.sums)
            wt, ln_kw = t[w + ".wg"], dict(bias=t[w + ".t"], ln_sums=self.sums, col_s=t[w + ".s"], ln_eps=norm.eps)
        else:
            _lib.layernorm(src, t[ln + ".w"], t[ln + ".b"], out_bf16=xb, eps=norm.eps)
            wt, ln_kw = t[w + ".w"], dict(bias=t.get(w + ".b"))
        fn = _lib.gemm_headnorm if "head_gamma" in epi else _lib.gemm_act if "act" in epi else _lib.gemm
        fn(xb, wt, out_bf16=out, **epi, **ln_kw)

    def stream_copy(self, slot: str) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """(bf16 copy, row sums) the kernel writing the stream also writes: fold (xb, ws[slot]), exact none."""
        if self.fold:
            self.sums = self.ws[slot]
            return self.xb, self.sums
        return None, None

    def residual(self, a: torch.Tensor, w: str, resid: torch.Tensor, slot: Optional[str]) -> None:
        """x = resid + a W^T + b (t[w + '.w' / '.b']) and stream_copy(slot); None: a local patch interaction
        follows and writes the copy of its own output."""
        copy, stats = self.stream_copy(slot) if slot is not None else (None, None)
        _lib.gemm(a, self.t[w + ".w"], out_f32=self.x, out_bf16=copy, bias=self.t[w + ".b"], resid=resid,
                  stats_out=stats)

    def project(self, L: EncoderLayer, i: int, out: Optional[torch.Tensor] = None) -> None:
        """qkv = LN1(x) Wqkv^T with layer L's q / k head norm, then the call's rotary positions; into `out` in place of
        the workspace's qkv when given."""
        head = {} if L.qk_norm is None else dict(head_gamma=self.t[f"{i}.gqk"], norm_heads=2 * L.heads, dh=L.dim_head,
                                                 head_layernorm_eps=L.qk_eps if L.qk_norm == "ln" else None)
        self.normed(self.x, f"{i}.ln1", L.ln1, f"{i}.qkv", self.qkv if out is None else out, **head)
        if self.rope is not None:
            _lib.rope_qk(self.qkv, self.rope[0], self.rope[1], L.heads, L.dim_head)

    def attend(self, kernel: str, L: EncoderLayer, i: int) -> None:
        """o = softmax attention of qkv through the kernel attention_kernel chose: 'axial', 'varlen' or 'plain'."""
        if kernel == "axial":
            G, T, key_mask, zero = self.axial
            _lib.attention_axial(self.qkv, self.o, key_mask, self.x.shape[0] // (T * G), T, G, L.heads, L.dim_head,
                                 L.scale, zero)
        elif kernel == "varlen":
            _lib.attention_varlen(self.qkv, self.o, *self.vl, L.heads, L.dim_head, L.scale, mask_self=L.mask_self)
        else:
            _lib.attention(self.qkv, self.o, self.B, self.N, L.heads, L.dim_head, L.scale, mask_self=L.mask_self)


class TransformerEngine:
    """Fused execution of the encoder layers a FusedEncoder module describes (reference vit.py:66-83)."""

    def __init__(self, transformer: nn.Module) -> None:
        self.mod = transformer
        self.prep = _Prepared()
        # what prepared() was built from: the layers and the final LayerNorm (simple_flash_attn_vit.py has none)
        self.layers: List[EncoderLayer] = []
        self.norm: Optional[Norm] = None
        self.slot = Workspace()                # may be shared with engines of the same shapes (share_workspace)
        self._vl_key: Optional[tuple] = None
        self._vl = None                        # varlen index of the fixed grid, for N > 512
        self.rows: Dict[tuple, torch.Tensor] = {}      # cls_row_index of the shapes pool() has seen

    def params(self) -> List[torch.Tensor]:
        """What the prepared weights are built from: the module's parameters and the buffers it names in
        `prepared_buffers()` (BatchNorm running statistics), so an in-place update of either rebuilds them."""
        extra = getattr(self.mod, "prepared_buffers", None)
        return list(self.mod.parameters()) + (list(extra()) if extra is not None else [])

    def unsupported_reason(self, N: int, grid: Optional[Tuple[int, int]] = None,
                           groups: Optional[Tuple[int, int]] = None,
                           regions: Optional[Tuple[int, int]] = None) -> Optional[str]:
        """None if the kernels are built for these layers over sequences of N tokens, else the reason the eager
        PyTorch graph is used.  Layers with an attention variant also check the token geometry, `grid`, `groups` and
        `regions` as run_blocks takes them, with the rule run_blocks raises on."""
        # only shapes are read, and a module's shapes are fixed at construction: any description of it serves
        for L in self.layers or self.mod.encoder_layers()[0]:
            A = L.attention
            r = head_width_reason(L.dim_head) if A is None else A.reason(L)
            if r is None and L.lpi is not None and L.lpi.kernel_size not in LPI_KERNEL_SIZES:
                r = lpi_reason(L.lpi.kernel_size, 1)
            if r is None and A is not None:
                r = A.geometry_reason(L, N, grid, groups, regions)
            if r is not None:
                return r
            if L.qkv_w.shape[1] % 8 or L.fc1_w.shape[0] % 8:
                return "dim / mlp_dim not multiples of 8"
        if N > 16384:
            return f"sequence length {N} > 16384"
        return None

    # -------------------------------------------------------------------------------------------- weights
    def prepared(self) -> Dict[str, torch.Tensor]:
        return self.prep.get(self.params(), self._build)

    def _build(self) -> Dict[str, torch.Tensor]:
        layers, norm = self.mod.encoder_layers()
        t: Dict[str, torch.Tensor] = {}
        for i, L in enumerate(layers):
            t[f"{i}.ln1.w"], t[f"{i}.ln1.b"] = _f32(L.ln1.gamma), _f32(L.ln1.beta)
            t[f"{i}.qkv.w"] = _bf16_rows(L.qkv_w)
            _fold(t, f"{i}.qkv", L.qkv_w, None, L.ln1)
            if L.qk_norm is not None:
                # per-head q / k norm: epilogue of the QKV GEMM
                t[f"{i}.gqk"] = torch.cat([_f32(g).reshape(-1) for g in L.qk_gamma])
            if L.out_w is None:
                # reference vit.py:34,46-49: heads == 1 and dim_head == dim -> to_out is nn.Identity.  The residual
                # GEMM then runs with an identity weight: bf16 x 1.0 products accumulate exactly, so x += o bit for bit
                eye = torch.eye(L.qkv_w.shape[1], device=L.qkv_w.device, dtype=torch.bfloat16)
                t[f"{i}.out.w"], t[f"{i}.out.b"] = _scaled_rows(eye, L.out_b, L.out_scale)
            else:
                t[f"{i}.out.w"], t[f"{i}.out.b"] = _scaled_rows(L.out_w, L.out_b, L.out_scale)
            if L.temporal is not None:
                T = L.temporal
                t[f"{i}.tln.w"], t[f"{i}.tln.b"] = _f32(T.ln.gamma), _f32(T.ln.beta)
                t[f"{i}.tqkv.w"] = _bf16_rows(T.qkv_w)
                _fold(t, f"{i}.tqkv", T.qkv_w, None, T.ln)
                t[f"{i}.tout.w"] = (torch.eye(T.qkv_w.shape[1], device=T.qkv_w.device, dtype=torch.bfloat16)
                                    if T.out_w is None else _bf16_rows(T.out_w))
                t[f"{i}.tout.b"] = _f32(T.out_b)
            if L.attention is not None:
                L.attention.prepare(t, i, L)
            if L.lpi is not None:
                P = L.lpi
                t[f"{i}.lpi.ln.w"], t[f"{i}.lpi.ln.b"] = _f32(P.ln.gamma), _f32(P.ln.beta)
                t[f"{i}.lpi.w1"], t[f"{i}.lpi.b1"], t[f"{i}.lpi.w2"], t[f"{i}.lpi.b2"] = lpi_weights(P)
            t[f"{i}.ln2.w"], t[f"{i}.ln2.b"] = _f32(L.ln2.gamma), _f32(L.ln2.beta)
            _fold(t, f"{i}.fc1", L.fc1_w, L.fc1_b, L.ln2)
            t[f"{i}.fc1.w"], t[f"{i}.fc1.b"] = _bf16_rows(L.fc1_w), _f32(L.fc1_b)
            t[f"{i}.fc2.w"], t[f"{i}.fc2.b"] = _scaled_rows(L.fc2_w, L.fc2_b, L.ff_scale)
        if norm is not None:
            t["norm.w"], t["norm.b"] = _f32(norm.gamma), _f32(norm.beta)
        self.layers, self.norm = layers, norm
        t["c_layers"] = self._c_layers(t)            # type: ignore[assignment]
        return t

    def _c_layers(self, t: Dict[str, torch.Tensor]):
        """(ctypes array of b200vit_layer, (heads, dh, hidden, scale), layer scales, attention flags) for the one-call
        encoder (b200vit_encoder_blocks), or None when it cannot run these layers: they are not uniform, one has a
        per-head LayerNorm (the one-call encoder has no EPI_HEADLN), a temporal sub-block, an attention variant, a
        local patch interaction or a post-norm step.  Layer scales: None when every layer has the same scale, else
        a ctypes float array for b200vit_encoder_blocks_ex (LSA's learned temperatures).  The pointers stay valid as
        long as `t` (which holds the tensors)."""
        sig = lambda L: (L.heads, L.dim_head, L.fc1_w.shape[0], L.mask_self)      # noqa: E731
        if any(L.qk_norm == "ln" or L.temporal is not None or L.attention is not None or L.lpi is not None
               or L.post_norm or L.ff_first or L.ff_act != "gelu" or sig(L) != sig(self.layers[0])
               for L in self.layers):
            return None
        arr = (_lib.Layer * len(self.layers))()
        p = lambda v: None if v is None else v.data_ptr()      # noqa: E731
        for i, L in enumerate(self.layers):
            c = arr[i]
            c.qkv_wg, c.qkv_t, c.qkv_s = p(t[f"{i}.qkv.wg"]), p(t[f"{i}.qkv.t"]), p(t[f"{i}.qkv.s"])
            c.qk_gamma = p(t.get(f"{i}.gqk"))
            c.out_w, c.out_b = p(t[f"{i}.out.w"]), p(t[f"{i}.out.b"])
            c.fc1_wg, c.fc1_t, c.fc1_s = p(t[f"{i}.fc1.wg"]), p(t[f"{i}.fc1.t"]), p(t[f"{i}.fc1.s"])
            c.fc2_w, c.fc2_b = p(t[f"{i}.fc2.w"]), p(t[f"{i}.fc2.b"])
            c.ln1_eps, c.ln2_eps = float(L.ln1.eps), float(L.ln2.eps)
        L0 = self.layers[0]
        scales = [float(L.scale) for L in self.layers]
        per_layer = None if all(sc == scales[0] for sc in scales) else (ctypes.c_float * len(scales))(*scales)
        return arr, (L0.heads, L0.dim_head, L0.fc1_w.shape[0], L0.scale), per_layer, \
            _lib.ATTN_MASK_SELF if L0.mask_self else 0

    # -------------------------------------------------------------------------------------------- workspaces
    def share_workspace(self, other: "TransformerEngine") -> None:
        """Run on `other`'s workspace from now on.  Only for encoders of identical shapes that never run at the same
        time: the stages of one CrossViT branch (cross_vit.py:151-153), which would otherwise each hold their own."""
        self.slot = other.slot

    def workspace(self, M: int, device: torch.device) -> Dict[str, torch.Tensor]:
        # one workspace per (rows, stream): two streams running the same model must not share scratch buffers.  The
        # other dimensions are the module's own and do not change.
        key = (M, device, torch.cuda.current_stream(device).cuda_stream)
        slot = self.slot
        if slot.key != key:
            self.prepared()
            L = self.layers[0]
            D, I, Hd = L.qkv_w.shape[1], L.heads * L.dim_head, L.fc1_w.shape[0]
            # layers whose q / k and v heads differ in width (ScalableViT) take views of other widths of these two
            Iqkv = max([3 * I] + [K.qkv_w.shape[0] for K in self.layers])
            Io = max([I] + [K.heads * value_width(K) for K in self.layers])
            bf = dict(device=device, dtype=torch.bfloat16)
            slot.t = {
                "xn": torch.empty(M, D, **bf),          # exact: LayerNorm output; fold: bf16 copy of x
                "qkv": torch.empty(M, Iqkv, **bf),
                "o": torch.empty(M, Io, **bf),
                "h": torch.empty(M, Hd, **bf),
                # LN-fold row statistics: [M, 1, 2] written by embed_tokens / rowstats_cast, [M, parts(D), 2] by GEMMs
                "stats_in": torch.empty(M, 1, 2, device=device, dtype=torch.float32),
                "stats_a": torch.empty(M, _lib.stats_parts(D), 2, device=device, dtype=torch.float32),
                "stats_b": torch.empty(M, _lib.stats_parts(D), 2, device=device, dtype=torch.float32),
            }
            if any(L.lpi is not None or L.post_norm for L in self.layers):
                # the stream the feed-forward block reads: the local patch interaction's or the post-norm's output
                slot.t["y"] = torch.empty(M, D, device=device, dtype=torch.float32)
            if any(getattr(L.attention, "o2", False) for L in self.layers):
                # a second attention output, out of place from "o" (the attention across windows)
                slot.t["o2"] = torch.empty(M, I, **bf)
            if any(L.lpi is not None for L in self.layers):
                # the local patch interaction's row statistics and its LayerNorm scratch
                slot.t["stats_l"] = torch.empty(M, 2, device=device, dtype=torch.float32)
                slot.t["lnst"] = torch.empty(M, 2, device=device, dtype=torch.float32)
            w = slot.t
            slot.c = _lib.EncoderWs(w["xn"].data_ptr(), w["qkv"].data_ptr(), w["o"].data_ptr(), w["h"].data_ptr(),
                                    w["stats_in"].data_ptr(), w["stats_a"].data_ptr(), w["stats_b"].data_ptr())
            slot.key = key
        return slot.t

    # -------------------------------------------------------------------------------------------- execution
    def _varlen_args(self, B: int, N: int, varlen: Optional[_lib.VarlenIndex], device: torch.device):
        """(cu_seqlens, tile_prefix, total_tiles) of the key-block (varlen) attention kernel, or None for the
        single-pass kernel: a packed batch always takes the varlen kernel, a fixed (B, N) grid does beyond 512 keys."""
        if varlen is not None:
            return varlen.cu, varlen.tile_prefix, varlen.total_tiles
        if N <= 512:
            return None
        key = (B, N, device)
        if self._vl_key != key:
            self._vl, self._vl_key = _lib.varlen_index([N] * B, device), key
        return self._vl

    def run_blocks(self, x: torch.Tensor, B: int = 0, N: int = 0, primed: bool = False,
                   varlen: Optional[_lib.VarlenIndex] = None,
                   rope: Optional[Tuple[torch.Tensor, int]] = None,
                   axial: Optional[Tuple[int, int, Optional[torch.Tensor], bool]] = None,
                   layers: Optional[Sequence[int]] = None, grid: Optional[Tuple[int, int]] = None,
                   groups: Optional[Tuple[int, int]] = None, regions: Optional[Tuple[int, int]] = None) -> None:
        """The encoder layers (all, or the indices in `layers`, in order: CaiT's layer dropout, cait.py:14-27), in place
        on the fp32 residual stream x[M, D] (no final LayerNorm).  Attention runs over
        B sequences of N tokens (M = B*N) or, `varlen` given, over the packed sequences it describes (M = varlen.T).
        `rope` = (table, rows): rotary positions on q and k after every QKV projection (and its head norm), token t
        using table row t % rows (_lib.rope_qk; the rotary ViTND, vit_nd_rotary.py:143-147).
        `axial` = (G, L, key_mask, zero_masked_rows): the sequences of _lib.attention_axial over the rows, token j of
        sequence b*G + p at row b*L*G + j*G + p, key_mask None or uint8 [M / (L*G), L].  Layers with a temporal
        sub-block run it there (the factorized layers of ViViT: spatial attention over the B sequences of N tokens,
        G = N); layers without one run their attention there instead of over the B x N sequences (ViViT's masked
        temporal transformer, G = 1).  These calls take the per-kernel loop below.
        `grid` = (h, w): the token grid of every sequence (N = h*w, token r*w + c), which layers with a local patch
        interaction (XCiT) or an attention variant on the grid need; `groups` and `regions` as those variants describe
        them (PatchGroups, RegionLocalBlock).  A layer's feed-forward block applies its `ff_act`.  A layer runs QKV ->
        rope -> attention (or its variant's launches) -> out-projection -> temporal sub-block (QKV, axial attention,
        out) -> local patch interaction x -> y, the stream the feed-forward block reads -> fc1 -> fc2 onto that stream,
        written to x.  A post-norm layer (CCT) writes y = LN2(x) and its bf16 copy instead, and its fc1 is the plain
        GEMM on that copy.  The call is checked first: a ValueError leaves x as it was.

        fold mode needs ws['xn'] (bf16 copy of x) and ws['stats_in'] (row sums of that copy) on entry: `primed` says
        the caller (embed_tokens / embed_varlen) already wrote them, otherwise one rowstats_cast pass produces them."""
        t = self.prepared()
        ws = self.workspace(x.shape[0], x.device)
        vl = self._varlen_args(B, N, varlen, x.device)
        fold = ln_mode() == "fold"
        if (fold and varlen is None and axial is None and layers is None and t["c_layers"] is not None
                and not _lib.profiling() and os.environ.get(_HOST_LOOP_ENV, "c") == "c"):
            # the whole layer loop below the language boundary: one ctypes call instead of 5 x depth
            arr, (heads, dh, hidden, scale), layer_scales, flags = t["c_layers"]
            _lib.encoder_blocks(arr, len(arr), x, self.slot.c, B, N, x.shape[1], heads, dh, hidden, scale, primed, vl,
                                rope=rope, layer_scales=layer_scales, attn_flags=flags)
            return
        run = range(len(self.layers)) if layers is None else layers
        kernels = []
        for i in run:
            L = self.layers[i]
            if L.temporal is not None and axial is None:
                raise ValueError("a layer with a temporal attention sub-block needs `axial` to address its sequences")
            kernels.append(attention_kernel(L, axial is not None, varlen is not None, vl is not None))
            if L.lpi is not None and (grid is None or grid[0] * grid[1] != N or axial is not None or varlen is not None):
                raise ValueError("a layer with a local patch interaction needs `grid` = (h, w) with h * w == N")
            if L.attention is not None:
                r = L.attention.geometry_reason(L, N, grid, groups, regions, rows=(B, x.shape[0]))
                if r is not None:
                    raise ValueError(r)
            if L.ff_first and (L.lpi is not None or L.post_norm or L.temporal is not None):
                raise ValueError("a layer whose feed-forward block runs first has no lpi, post_norm or temporal block")
        c = BlocksCall(t, ws, x, B, N, grid, groups, regions, rope, axial, vl, fold, primed)
        xb, h = c.xb, c.h
        for i, kernel in zip(run, kernels):
            L = self.layers[i]
            act = dict(act="silu") if L.ff_act == "silu" else dict(gelu=True)
            if L.ff_first:
                c.normed(x, f"{i}.ln2", L.ln2, f"{i}.fc1", h, **act)
                c.residual(h, f"{i}.fc2", x, "stats_a")
            if L.attention is None:
                c.project(L, i)
                c.attend(kernel, L, i)
                attn_out = c.o
            else:
                attn_out = L.attention.launch(c, L, i)
            c.residual(attn_out, f"{i}.out", x, "stats_b" if L.lpi is None and not L.post_norm else None)
            if L.temporal is not None:
                c.normed(x, f"{i}.tln", L.temporal.ln, f"{i}.tqkv", c.qkv)
                c.attend("axial", L, i)
                c.residual(c.o, f"{i}.tout", x, "stats_b")
            ff_in = x if L.lpi is None and not L.post_norm else ws["y"]
            if L.lpi is not None:
                yb, ys = c.stream_copy("stats_l")
                ln = (t[f"{i}.lpi.ln.w"], t[f"{i}.lpi.ln.b"], L.lpi.ln.eps)
                _lib.local_patch_interaction(x, ff_in, ws["lnst"], ln, t[f"{i}.lpi.w1"], t[f"{i}.lpi.b1"],
                                             t[f"{i}.lpi.w2"], t[f"{i}.lpi.b2"], B, grid[0], grid[1],
                                             L.lpi.kernel_size, y_bf16=yb, y_stats=ys)
            if L.ff_first:
                continue
            if L.post_norm:
                # the normalised stream and its bf16 copy; fc1 reads that copy as it is, with no LayerNorm of its own
                _lib.layernorm(x, t[f"{i}.ln2.w"], t[f"{i}.ln2.b"], out_f32=ff_in, out_bf16=xb, eps=L.ln2.eps)
                (_lib.gemm_act if "act" in act else _lib.gemm)(xb, t[f"{i}.fc1.w"], out_bf16=h, bias=t[f"{i}.fc1.b"],
                                                                **act)
            else:
                c.normed(ff_in, f"{i}.ln2", L.ln2, f"{i}.fc1", h, **act)
            c.residual(h, f"{i}.fc2", ff_in, "stats_a")

    def final_norm(self, x: torch.Tensor, *, out_bf16: Optional[torch.Tensor] = None,
                   out_f32: Optional[torch.Tensor] = None, row_index: Optional[torch.Tensor] = None) -> None:
        t = self.prepared()
        assert self.norm is not None
        _lib.layernorm(x, t["norm.w"], t["norm.b"], out_bf16=out_bf16, out_f32=out_f32, row_index=row_index,
                       eps=self.norm.eps)

    def stream_bf16(self, x: torch.Tensor) -> torch.Tensor:
        """The bf16 copy of the residual stream x after run_blocks: in fold mode the workspace's, which the last
        residual GEMM wrote; otherwise a new cast of x."""
        if ln_mode() == "fold":
            return self.workspace(x.shape[0], x.device)["xn"]
        xb = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)
        _lib.cast_f32_bf16(x.view(-1), xb.view(-1))
        return xb

    def entry_buffers(self, M: int, device: torch.device) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """(xb, stats) an embedding kernel writes for the first layer so that run_blocks(primed=True) can skip its
        rowstats_cast pass: the workspace's bf16 copy of x and its row sums in fold mode, (None, None) otherwise."""
        if ln_mode() != "fold":
            return None, None
        ws = self.workspace(M, device)
        return ws["xn"], ws["stats_in"]

    def pool(self, x: torch.Tensor, B: int, N: int, *, mean: bool, skip: int = 0, n_pool: Optional[int] = None,
             dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
        """After run_blocks on B sequences of N rows of x: the final LayerNorm (none if the Transformer has none), then
        per sequence its first row (mean=False) or the mean of `n_pool` rows (default N) from row `skip` on, as a new
        [B, D] tensor of `dtype`.  LayerNorm is per token, so first-row pooling normalises only those rows."""
        D, dev = x.shape[1], x.device
        out = torch.empty(B, D, device=dev, dtype=dtype)
        if not mean:
            rows = cls_row_index(self.rows, B, N, dev)
            if dtype == torch.bfloat16:
                self.final_norm(x, out_bf16=out, row_index=rows)
            else:
                self.final_norm(x, out_f32=out, row_index=rows)
            return out
        if self.norm is not None:
            xf = torch.empty_like(x)
            self.final_norm(x, out_f32=xf)
        else:
            xf = x
        pm = out if dtype == torch.float32 else torch.empty(B, D, device=dev, dtype=torch.float32)
        _lib.mean_pool(xf.view(-1)[skip * D:] if skip else xf, pm, B, N, D, n_pool=n_pool)
        if pm is not out:
            _lib.cast_f32_bf16(pm, out)
        return out

    def forward_tokens(self, tokens: torch.Tensor, rope: Optional[Tuple[torch.Tensor, int]] = None,
                       axial: Optional[Tuple[int, int, Optional[torch.Tensor], bool]] = None,
                       layers: Optional[Sequence[int]] = None, grid: Optional[Tuple[int, int]] = None,
                       groups: Optional[Tuple[int, int]] = None) -> torch.Tensor:
        """Transformer.forward on arbitrary bf16 tokens [B, N, D] (what MAE / SimMIM / Distill call,
        reference mae.py:74, simmim.py:70, distill.py:66); `rope`, `axial`, `layers`, `grid` and `groups` as in
        run_blocks."""
        B, N, D = tokens.shape
        with on_device(tokens):
            x = tokens.reshape(B * N, D).float().contiguous()
            self.run_blocks(x, B, N, rope=rope, axial=axial, layers=layers, grid=grid, groups=groups)
            out = torch.empty(B * N, D, device=tokens.device, dtype=torch.bfloat16)
            if self.norm is not None:
                self.final_norm(x, out_bf16=out)
            else:
                _lib.cast_f32_bf16(x.view(-1), out.view(-1))
        return out.view(B, N, D)


class PatchEmbedEngine:
    """Fused patch embedding + token assembly (reference vit.py:99-104,120-127 / simple_vit.py:90-95,113-114).  An
    owner whose to_patch_embedding is an SPT (vit_for_small_dataset.py:81-96: `to_patch_tokens` = Rearrange,
    LayerNorm, Linear, and no LayerNorm(dim)) gets the shifted-patch kernel instead of the plain patchify."""

    def __init__(self, owner: nn.Module) -> None:
        self.owner = owner
        self.prep = _Prepared()

    def cls_row(self) -> Optional[torch.Tensor]:
        """The owner's cls token if it opens every sequence: not for an owner with `cls_in_sequence = False` (CaiT's
        cls token joins only in its class-attention stage, cait.py:175-176)."""
        return getattr(self.owner, "cls_token", None) if getattr(self.owner, "cls_in_sequence", True) else None

    def params(self) -> List[torch.Tensor]:
        o = self.owner
        ps = list(o.to_patch_embedding.parameters())
        for name in ("cls_token", "pos_embedding", "register_tokens"):
            v = getattr(o, name, None)
            if isinstance(v, nn.Parameter):
                ps.append(v)
        return ps

    def prepared(self, device: torch.device) -> Dict[str, torch.Tensor]:
        return self.prep.get(self.params(), lambda: self._build(device), str(device))

    def _build(self, device: torch.device) -> Dict[str, torch.Tensor]:
        o = self.owner
        spt = getattr(o.to_patch_embedding, "to_patch_tokens", None)
        if spt is not None:
            ln1, lin, ln2 = spt[1], spt[2], None
        else:
            ln1, lin, ln2 = o.to_patch_embedding[1], o.to_patch_embedding[2], o.to_patch_embedding[3]
        pd = lin.weight.shape[1]
        kp = (pd + 63) // 64 * 64
        t = {
            "ln1.w": _f32(ln1.weight), "ln1.b": _f32(ln1.bias),
            "w": _bf16_rows(lin.weight, kp), "b": _f32(lin.bias),
            "ln2.w": None if ln2 is None else _f32(ln2.weight), "ln2.b": None if ln2 is None else _f32(ln2.bias),
        }
        t["kp"] = kp  # type: ignore[assignment]
        t["spt"] = spt is not None  # type: ignore[assignment]
        t["ln1.eps"], t["ln2.eps"] = ln1.eps, 1e-5 if ln2 is None else ln2.eps  # type: ignore[assignment]
        ph, pw = getattr(o, "fused_patch_box", None) or o.patch_size
        if spt is None and ph == 16 and pw == 16 and pd % 256 == 0:
            # im2col-free path (b200vit_patch_embed_tma): LayerNorm(patch) folded into the projection, weight columns
            # permuted from the reference's (p1 p2 c) order (vit.py:100) to the image's own (c p1 p2)
            C = pd // 256
            w32 = lin.weight.detach().float()
            wg = w32 * ln1.weight.detach().float()[None, :]
            t["tma.w"] = wg.view(-1, 256, C).permute(0, 2, 1).reshape(-1, pd).to(torch.bfloat16).contiguous()
            t["tma.s"] = t["tma.w"].float().sum(dim=1).contiguous()           # from the ROUNDED weights the MMA sees
            t["tma.b"] = (w32 @ ln1.bias.detach().float() + lin.bias.detach().float()).contiguous()
        cls = self.cls_row()
        t["cls"] = _f32(cls) if (cls is not None and cls.shape[0] > 0) else None
        reg = getattr(o, "register_tokens", None)          # simple_vit_with_register_tokens.py:103,124-126
        t["tail"] = _f32(reg) if (reg is not None and reg.shape[0] > 0) else None
        pos = getattr(o, "pos_embedding", None)
        t["pos"] = pos.detach().to(device=device, dtype=torch.float32).contiguous() if pos is not None else None
        return t

    def _pos_table(self, t: Dict[str, torch.Tensor], gh: int, gw: int, device: torch.device) -> torch.Tensor:
        """The module's positional table, or -- for the variants that build the sin-cos table from the input's own
        patch grid on every call (simple_flash_attn_vit.py:158-160) -- that table, cached per grid shape."""
        if t["pos"] is not None:
            return t["pos"]
        cache = self.__dict__.setdefault("_pos_cache", {})
        key = (gh, gw, str(device))
        if key not in cache:
            cache[key] = self.owner.fused_pos_table(gh, gw).to(device=device, dtype=torch.float32).contiguous()
        return cache[key]

    def run(self, img: torch.Tensor, xb: Optional[torch.Tensor] = None, stats: Optional[torch.Tensor] = None,
            patch: Optional[Tuple[int, int]] = None, pos: Optional[torch.Tensor] = None
            ) -> Tuple[torch.Tensor, int, int]:
        """img [B, C, H, W] bf16 -> (x fp32 [B*N, D], B, N); optionally also the bf16 copy of x and its row sums.
        `patch` / `pos` override the owner's patch size and positional table: the 1-D and 3-D front-ends
        (simple_vit_1d.py, simple_vit_3d.py) present their input as a [B, C, H', W'] view with its own patch box."""
        o = self.owner
        ph, pw = patch if patch is not None else o.patch_size
        B, C, H, W = img.shape
        if H % ph or W % pw:
            raise ValueError("Image dimensions must be divisible by the patch size.")
        t = self.prepared(img.device)
        n = (H // ph) * (W // pw)
        ncls = 0 if t["cls"] is None else t["cls"].shape[0]
        ntail = 0 if t["tail"] is None else t["tail"].shape[0]
        N = n + ncls + ntail
        D = t["w"].shape[0]
        if pos is None:
            pos = self._pos_table(t, H // ph, W // pw, img.device)
        if pos.shape[0] < n + ncls:
            raise ValueError(f"sequence of {n + ncls} tokens exceeds the positional table ({pos.shape[0]})")
        y = self.project(img, patch)
        x = torch.empty(B * N, D, device=img.device, dtype=torch.float32)
        _lib.embed_tokens(y, t["ln2.w"], t["ln2.b"], t["cls"], pos, x, B, n, ncls, xb=xb, stats=stats,
                          eps=t["ln2.eps"], tail=t["tail"])
        return x, B, N

    def project(self, img: torch.Tensor, patch: Optional[Tuple[int, int]] = None) -> torch.Tensor:
        """The patch projection alone (vit.py:100-102): img [B, C, H, W] bf16 -> y fp32 [B*n, D] = LayerNorm(patch)
        W^T + b, patches in row-major grid order, before the LayerNorm(dim) that token assembly applies."""
        o = self.owner
        ph, pw = patch if patch is not None else o.patch_size
        B, C, H, W = img.shape
        if H % ph or W % pw:
            raise ValueError("Image dimensions must be divisible by the patch size.")
        t = self.prepared(img.device)
        n = (H // ph) * (W // pw)
        D = t["w"].shape[0]
        dev = img.device
        y = torch.empty(B * n, D, device=dev, dtype=torch.float32)
        if ("tma.w" in t and (ph, pw) == (16, 16) and os.environ.get(_PATCH_MODE_ENV, "tma") == "tma"
                and W // pw <= 128 and D % 8 == 0):
            # the wgmma GEMM reads the image itself: no patch matrix, no LayerNorm pass
            stats_p = torch.empty(B * n, 2, device=dev, dtype=torch.float32)
            _lib.patch_embed_tma(img.contiguous(), t["tma.w"], t["tma.b"], t["tma.s"], stats_p, y, eps=t["ln1.eps"])
        else:
            a0 = torch.empty(B * n, t["kp"], device=dev, dtype=torch.bfloat16)
            if t["spt"]:
                # the five shifted copies are gathered straight from the image (vit_for_small_dataset.py:92-96)
                _lib.patchify_spt_ln(img.contiguous(), t["ln1.w"], t["ln1.b"], a0, ph, eps=t["ln1.eps"])
            else:
                _lib.patchify_ln(img.contiguous(), t["ln1.w"], t["ln1.b"], a0, ph, pw, eps=t["ln1.eps"])
            _lib.gemm(a0, t["w"], out_f32=y, bias=t["b"])
        return y

    def geometry(self, img: torch.Tensor, patch: Optional[Tuple[int, int]] = None) -> Tuple[int, int]:
        """(B, N) the image batch will produce, without running anything."""
        ph, pw = patch if patch is not None else self.owner.patch_size
        cls = self.cls_row()
        reg = getattr(self.owner, "register_tokens", None)
        extra = (cls.shape[0] if cls is not None else 0) + (reg.shape[0] if reg is not None else 0)
        return img.shape[0], (img.shape[2] // ph) * (img.shape[3] // pw) + extra


class HeadEngine:
    """Pooled-feature -> logits GEMM (reference vit.py:138 / simple_vit.py:120)."""

    def __init__(self, linear: nn.Linear) -> None:
        self.lin = linear
        self.prep = _Prepared()

    def params(self) -> List[torch.Tensor]:
        return list(self.lin.parameters())

    def run(self, pooled_bf16: torch.Tensor) -> torch.Tensor:
        t = self.prep.get(self.params(), lambda: {"w": _bf16_rows(self.lin.weight), "b": _f32(self.lin.bias)})
        out = torch.empty(pooled_bf16.shape[0], t["w"].shape[0], device=pooled_bf16.device, dtype=torch.bfloat16)
        _lib.gemm(pooled_bf16.contiguous(), t["w"], out_bf16=out, bias=t["b"])
        return out


class FeedForwardBlock(NamedTuple):
    """x += fc2(GELU(fc1(LN(x)))) (reference vit.py:15-28)."""
    ln: Norm
    fc1_w: torch.Tensor
    fc1_b: torch.Tensor
    fc2_w: torch.Tensor
    fc2_b: torch.Tensor


class CrossLayer(NamedTuple):
    """One direction of one class-token cross-attention layer (CrossViT, reference cross_vit.py:94-130), as the module
    describes it to CrossAttentionEngine: the cls row of stream A (width D_A) queries the patch rows of stream B
    (width D_B), in B's width:
        c    = project_in(cls_A)                                   (Identity when D_A == D_B)
        cn   = LN(c);  q = cn Wq^T;  [k | v] = [cn; ctx_B] Wkv^T  (kv_include_self)
        cls_A += project_out(to_out(softmax(q k^T * scale) v))
    Optional parts (CaiT's class attention, cait.py:83-122): talking heads `pre` / `post` around the softmax
    (b200vit_attention_cls_headmix), LayerScale `out_scale` on the to_out output, and a feed-forward sub-block `ff`
    on the cls rows afterwards, its output scaled by `ff_scale`.  They need D_A == D_B."""
    proj_in: Optional[Tuple[torch.Tensor, torch.Tensor]]       # (weight [D_B, D_A], bias) or None
    ln: Norm
    q_w: torch.Tensor                                           # [heads * dim_head, D_B]
    kv_w: torch.Tensor                                          # [2 * heads * dim_head, D_B], rows k | v
    out_w: torch.Tensor                                         # [D_B, heads * dim_head]
    out_b: Optional[torch.Tensor]
    proj_out: Optional[Tuple[torch.Tensor, torch.Tensor]]      # (weight [D_A, D_B], bias) or None
    heads: int
    dim_head: int
    scale: float
    pre: Optional[torch.Tensor] = None                          # [heads, heads], [input head, output head]
    post: Optional[torch.Tensor] = None                         # (pre and post: both or neither)
    out_scale: Optional[torch.Tensor] = None                    # [D_B]
    ff: Optional[FeedForwardBlock] = None
    ff_scale: Optional[torch.Tensor] = None                     # [D_A]


class CrossAttentionEngine:
    """Fused execution of one direction of a CrossTransformer (cls of stream A attends to stream B's patch rows).
    The owner module provides cross_layers(direction) -> List[CrossLayer] and cross_params(direction), the parameters
    they are made of.

    Per call: one GEMM of every layer's to_kv, stacked, over all rows of B's bf16 copy (the context never changes
    inside a CrossTransformer, cross_vit.py:121-130; B's cls rows are computed and skipped).  Per layer:
        projection:  project_in GEMM on A's cls rows (+ row statistics) -> LN-folded [to_q; to_kv] GEMM
        Identity:    LayerNorm of A's fp32 cls rows (row_index)        -> [to_q; to_kv] GEMM
        b200vit_attention_cls -> to_out GEMM -> project_out GEMM with the residual, in place on A's cls rows of the
        fp32 stream and its bf16 copy (Identity: to_out carries the residual);
        with a feed-forward sub-block: LayerNorm of the cls rows -> fc1 GEMM + GELU -> fc2 GEMM with the residual."""

    def __init__(self, owner: nn.Module, direction: int) -> None:
        self.owner, self.direction = owner, direction
        self.prep = _Prepared()
        self.layers: List[CrossLayer] = []

    def prepared(self) -> Dict[str, torch.Tensor]:
        return self.prep.get(self.owner.cross_params(self.direction), self._build)

    def _build(self) -> Dict[str, torch.Tensor]:
        layers = self.owner.cross_layers(self.direction)
        t: Dict[str, torch.Tensor] = {}
        for i, L in enumerate(layers):
            qkv_w = torch.cat([L.q_w.detach(), L.kv_w.detach()])
            if L.proj_in is not None:
                t[f"{i}.pin.w"], t[f"{i}.pin.b"] = _bf16_rows(L.proj_in[0]), _f32(L.proj_in[1])
                _fold(t, f"{i}.qkv", qkv_w, None, L.ln)
            else:
                t[f"{i}.ln.w"], t[f"{i}.ln.b"] = _f32(L.ln.gamma), _f32(L.ln.beta)
                t[f"{i}.qkv.w"] = _bf16_rows(qkv_w)
            t[f"{i}.out.w"], t[f"{i}.out.b"] = _scaled_rows(L.out_w, L.out_b, L.out_scale)
            if L.proj_out is not None:
                t[f"{i}.pout.w"], t[f"{i}.pout.b"] = _bf16_rows(L.proj_out[0]), _f32(L.proj_out[1])
            if L.pre is not None:
                t[f"{i}.pre"], t[f"{i}.post"] = _f32(L.pre), _f32(L.post)
            if L.ff is not None:
                F = L.ff
                t[f"{i}.ln2.w"], t[f"{i}.ln2.b"] = _f32(F.ln.gamma), _f32(F.ln.beta)
                t[f"{i}.fc1.w"], t[f"{i}.fc1.b"] = _bf16_rows(F.fc1_w), _f32(F.fc1_b)
                t[f"{i}.fc2.w"], t[f"{i}.fc2.b"] = _scaled_rows(F.fc2_w, F.fc2_b, L.ff_scale)
        t["ctx.w"] = _bf16_rows(torch.cat([L.kv_w.detach() for L in layers]))
        self.layers = layers
        return t

    def run(self, xa: torch.Tensor, xba: torch.Tensor, Na: int, xbb: torch.Tensor, Nb: int, B: int,
            cls_rows_a: torch.Tensor, skip: int = 1, layers: Optional[Sequence[int]] = None) -> None:
        """xa fp32 [B*Na, D_A] (stream A) and xba, its bf16 copy: cls rows updated in place.  xbb bf16 [B*Nb, D_B]:
        stream B, whose first `skip` rows per image are not part of the context (1: its cls token).  cls_rows_a int32
        [B] = b*Na.  `layers`: the indices of the layers to run, in order (default all)."""
        t = self.prepared()
        dev = xa.device
        bf = dict(device=dev, dtype=torch.bfloat16)
        Da = xa.shape[1]
        ctx = torch.empty(B * Nb, t["ctx.w"].shape[0], **bf)
        _lib.gemm(xbb, t["ctx.w"], out_bf16=ctx)
        a_cls, ab_cls = xa.view(B, Na, Da)[:, 0], xba.view(B, Na, Da)[:, 0]      # row stride Na * D_A
        for i in range(len(self.layers)) if layers is None else layers:
            L = self.layers[i]
            I, Dc = L.heads * L.dim_head, L.q_w.shape[1]
            qin = torch.empty(B, Dc, **bf)
            qkv = torch.empty(B, 3 * I, **bf)
            if L.proj_in is not None:
                st = torch.empty(B, _lib.stats_parts(Dc), 2, device=dev, dtype=torch.float32)
                _lib.gemm(ab_cls, t[f"{i}.pin.w"], out_bf16=qin, bias=t[f"{i}.pin.b"], stats_out=st)
                _lib.gemm(qin, t[f"{i}.qkv.wg"], out_bf16=qkv, bias=t[f"{i}.qkv.t"], ln_sums=st,
                          col_s=t[f"{i}.qkv.s"], ln_eps=L.ln.eps)
            else:
                _lib.layernorm(xa, t[f"{i}.ln.w"], t[f"{i}.ln.b"], out_bf16=qin, row_index=cls_rows_a, eps=L.ln.eps)
                _lib.gemm(qin, t[f"{i}.qkv.w"], out_bf16=qkv)
            o = torch.empty(B, I, **bf)
            ctx_i = ctx[:, 2 * I * i:2 * I * (i + 1)]
            if L.pre is not None:
                _lib.attention_cls_headmix(qkv, ctx_i, o, Nb, skip, Nb - skip, L.heads, L.dim_head, L.scale,
                                           t[f"{i}.pre"], t[f"{i}.post"])
            else:
                _lib.attention_cls(qkv, ctx_i, o, Nb, skip, Nb - skip, L.heads, L.dim_head, L.scale)
            if L.proj_out is not None:
                y = torch.empty(B, Dc, **bf)
                _lib.gemm(o, t[f"{i}.out.w"], out_bf16=y, bias=t[f"{i}.out.b"])
                _lib.gemm(y, t[f"{i}.pout.w"], out_f32=a_cls, out_bf16=ab_cls, bias=t[f"{i}.pout.b"], resid=a_cls)
            else:
                _lib.gemm(o, t[f"{i}.out.w"], out_f32=a_cls, out_bf16=ab_cls, bias=t[f"{i}.out.b"], resid=a_cls)
            if L.ff is not None:
                h = torch.empty(B, L.ff.fc1_w.shape[0], **bf)
                _lib.layernorm(xa, t[f"{i}.ln2.w"], t[f"{i}.ln2.b"], out_bf16=qin, row_index=cls_rows_a,
                               eps=L.ff.ln.eps)
                _lib.gemm(qin, t[f"{i}.fc1.w"], out_bf16=h, bias=t[f"{i}.fc1.b"], gelu=True)
                _lib.gemm(h, t[f"{i}.fc2.w"], out_f32=a_cls, out_bf16=ab_cls, bias=t[f"{i}.fc2.b"], resid=a_cls)


def cls_row_index(cache: Dict[tuple, torch.Tensor], B: int, N: int, device: torch.device) -> torch.Tensor:
    """int32 [B] = 0, N, 2N, ...: the cls rows of B images of N tokens, made once per shape so a steady-state forward
    (and a CUDA-graph capture) issues no allocation-and-fill for it."""
    key = (B, N, str(device))
    if key not in cache:
        cache[key] = torch.arange(0, B * N, N, device=device, dtype=torch.int32)
    return cache[key]


def fused_two_streams(stages, xs: torch.Tensor, xl: torch.Tensor, B: int, Ns: int, Nl: int, primed: bool,
                      rows: Tuple[torch.Tensor, torch.Tensor]) -> Tuple[List[torch.Tensor], List[torch.Tensor]]:
    """CrossViT's MultiScaleEncoder (reference cross_vit.py:157-162) on two fp32 residual streams xs [B*Ns, D_sm] and
    xl [B*Nl, D_lg].  `stages`: per multi-scale block (sm TransformerEngine, lg TransformerEngine, sm-attends-lg
    CrossAttentionEngine, lg-attends-sm CrossAttentionEngine); the engines of one branch share one workspace, whose
    'xn' holds that branch's bf16 copy.  Per block and branch: the encoder layers, then the Transformer's final
    LayerNorm (cross_vit.py:90), which REPLACES the stream -- written as a new fp32 stream and its bf16 copy; the next
    block's layers enter the folded chain from it.  Then both cross directions; they are independent (the lg->sm
    direction reads sm patch rows and lg cls, cross_vit.py:124-126).  `primed`: the embedding already wrote the first
    block's bf16 copies and row statistics.  `rows`: cls_row_index of either stream.
    Returns ([x_sm, x_lg], [xb_sm, xb_lg]): the final fp32 streams and their bf16 copies."""
    x, N = [xs, xl], (Ns, Nl)
    spare = [torch.empty_like(xs), torch.empty_like(xl)]
    xb: List[torch.Tensor] = [xs, xl]
    for i, (enc_s, enc_l, sm_lg, lg_sm) in enumerate(stages):
        for b, eng in enumerate((enc_s, enc_l)):
            eng.run_blocks(x[b], B, N[b], primed=primed and i == 0)
            xb[b] = eng.workspace(B * N[b], x[b].device)["xn"]
            eng.final_norm(x[b], out_f32=spare[b], out_bf16=xb[b])
            x[b], spare[b] = spare[b], x[b]
        sm_lg.run(x[0], xb[0], Ns, xb[1], Nl, B, rows[0])
        lg_sm.run(x[1], xb[1], Nl, xb[0], Ns, B, rows[1])
    return x, xb


def patch_engine(owner: nn.Module) -> PatchEmbedEngine:
    """The owner's PatchEmbedEngine, made on first use."""
    pe = owner.__dict__.get("_patch_engine")
    if pe is None:
        pe = owner._patch_engine = PatchEmbedEngine(owner)
    return pe


def head_engine(owner: nn.Module, linear: nn.Linear) -> HeadEngine:
    """The owner's HeadEngine over its classifier Linear `linear`, made on first use."""
    he = owner.__dict__.get("_head_engine")
    if he is None:
        he = owner._head_engine = HeadEngine(linear)
    return he


def classify(owner: nn.Module, linear: nn.Linear, pooled: torch.Tensor) -> torch.Tensor:
    """Logits of bf16 pooled features: owner.to_latent(pooled), which stays a called module (Dino / LeJEPA hook it),
    then the head GEMM of `linear`."""
    return head_engine(owner, linear).run(owner.to_latent(pooled))


def head_norm(owner: nn.Module, ln: nn.LayerNorm) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """fp32 (weight, bias) of the LayerNorm of the owner's head, cached by parameter version."""
    return cached(owner, "_head_norm", list(ln.parameters()), lambda: (_f32(ln.weight), _f32(ln.bias)))


def head_ln_pool(owner: nn.Module, ln: nn.LayerNorm, x: torch.Tensor, B: int, N: int, *, mean: bool) -> torch.Tensor:
    """x fp32 [B*N, D] encoder output of a Transformer without a final LayerNorm -> ln(x[:, 0]) or ln(x.mean(1)), bf16
    [B, D]: the models whose mlp_head starts with a LayerNorm (vit_for_small_dataset.py:134-140, deepvit.py:125-129)."""
    D = x.shape[1]
    dev = x.device
    g, b = head_norm(owner, ln)
    pooled = torch.empty(B, D, device=dev, dtype=torch.bfloat16)
    if mean:
        pm = torch.empty(B, D, device=dev, dtype=torch.float32)
        _lib.mean_pool(x, pm, B, N, D)
        _lib.layernorm(pm, g, b, out_bf16=pooled, eps=ln.eps)
    elif N == 1:                                   # x holds the cls rows only (CaiT's class-attention stage)
        _lib.layernorm(x, g, b, out_bf16=pooled, eps=ln.eps)
    else:                                          # LayerNorm is per token: normalise only the cls rows
        rows = cls_row_index(owner.transformer.engine().rows, B, N, dev)
        _lib.layernorm(x, g, b, out_bf16=pooled, row_index=rows, eps=ln.eps)
    return pooled


def fused_encode(owner: nn.Module, img: torch.Tensor, patch: Optional[Tuple[int, int]] = None,
                 pos: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, int, int]:
    """Patch embedding -> encoder blocks of the single-image models: (x, B, N) with x the fp32 residual stream
    [B*N, D] after the last layer, before the final LayerNorm.  In fold mode the patch embedding also writes the
    engine's bf16 copy of x and its row statistics, which the first layer reads.  Must run inside on_device(img)."""
    pe, eng = patch_engine(owner), owner.transformer.engine()
    B, N = pe.geometry(img, patch)
    xb, stats = eng.entry_buffers(B * N, img.device)
    x, B, N = pe.run(img, xb=xb, stats=stats, patch=patch, pos=pos)
    eng.run_blocks(x, B, N, primed=xb is not None)
    return x, B, N


def fused_mean_pooled_features(owner: nn.Module, img: torch.Tensor, pool_tokens: Optional[int] = None,
                               patch: Optional[Tuple[int, int]] = None, pos: Optional[torch.Tensor] = None
                               ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Shared body of the SimpleViT-family fused forwards (reference simple_vit.py:110-117 and its variants):
    patch embedding (+ register tokens) -> encoder blocks -> final LayerNorm if the Transformer has one -> mean over
    the first `pool_tokens` tokens of every image (all tokens by default).  Returns that mean as fp32 and as bf16,
    [B, D] each; must run inside on_device(img)."""
    if transformer_is_hooked(owner):
        x, B, N = patch_engine(owner).run(img, patch=patch, pos=pos)
        xf = hooked_transformer_tokens(owner, x, B, N).reshape(B * N, -1).float()
        pm = torch.empty(B, xf.shape[1], device=img.device, dtype=torch.float32)
        _lib.mean_pool(xf, pm, B, N, xf.shape[1], n_pool=pool_tokens)
    else:
        x, B, N = fused_encode(owner, img, patch=patch, pos=pos)
        pm = owner.transformer.engine().pool(x, B, N, mean=True, n_pool=pool_tokens, dtype=torch.float32)
    pooled = torch.empty(pm.shape, device=img.device, dtype=torch.bfloat16)
    _lib.cast_f32_bf16(pm, pooled)
    return pm, pooled
