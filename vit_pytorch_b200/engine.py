"""Host-side engine of the fused sm_90a forward: weight preparation, workspaces and the kernel schedule.

The nn.Modules in vit.py / simple_vit.py own the parameters (reference-compatible names); this file turns them into
the flat bf16 / fp32 device buffers the C ABI (include/b200vit.h) consumes and issues the launches on torch's current
stream.  Nothing here computes on the host and nothing falls back: a missing library or a failing call raises.

Schedule per encoder layer (reference vit.py:78-81), M = B*N token rows, residual stream x kept in fp32:
    xn  = LayerNorm(x)                         b200vit_layernorm      fp32 -> bf16              (vit.py:52)
    qkv = xn Wqkv^T                            b200vit_gemm_bf16      wgmma, bf16 out           (vit.py:54)
    o   = softmax(q k^T * scale) v             b200vit_attention      wgmma, online softmax     (vit.py:55-63)
    x  += o Wout^T + b                         b200vit_gemm_bf16      residual epilogue, fp32   (vit.py:64,80)
    xn  = LayerNorm(x)                         b200vit_layernorm                               (vit.py:19)
    h   = GELU(xn W1^T + b1)                   b200vit_gemm_bf16      bias+GELU epilogue        (vit.py:20-21)
    x  += h W2^T + b2                          b200vit_gemm_bf16      residual epilogue         (vit.py:23,81)
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Tuple

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


def _softmax_scale(attn) -> float:
    """dim_head ** -0.5 (vit.py:37,57) unless the module says otherwise (q/k-normalised attention uses 1)."""
    return float(getattr(attn, "softmax_scale", attn.scale))


class _Prepared:
    """Flat device buffers derived from one module's parameters + the parameter versions they were built from."""

    def __init__(self) -> None:
        self.key: Optional[tuple] = None
        self.t: Dict[str, torch.Tensor] = {}


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


def _f32(p: torch.Tensor) -> torch.Tensor:
    return p.detach().float().contiguous()


def _bf16_rows(p: torch.Tensor, k_pad: Optional[int] = None) -> torch.Tensor:
    """[out, in] weight as contiguous bf16 with the K dim padded to `k_pad` (zeros) for TMA's 16-byte row rule."""
    w = p.detach()
    if k_pad is not None and k_pad != w.shape[1]:
        wp = torch.zeros(w.shape[0], k_pad, device=w.device, dtype=torch.bfloat16)
        wp[:, : w.shape[1]] = w
        return wp
    return w.to(torch.bfloat16).contiguous()


class TransformerEngine:
    """Fused execution of a vit.Transformer / simple_vit.Transformer module (reference vit.py:66-83)."""

    def __init__(self, transformer: nn.Module) -> None:
        self.mod = transformer
        self.prep = _Prepared()
        self.ws_key: Optional[tuple] = None
        self.ws: Dict[str, torch.Tensor] = {}
        self.c_ws = None                       # _lib.EncoderWs over self.ws

    # -------------------------------------------------------------------------------------------- structure
    def _layers(self):
        for attn, ff in self.mod.layers:
            yield attn, ff

    def params(self) -> List[torch.Tensor]:
        return list(self.mod.parameters())

    def has_final_norm(self) -> bool:
        """simple_flash_attn_vit.py's Transformer has no final LayerNorm (its head carries one instead)."""
        return getattr(self.mod, "norm", None) is not None

    def unsupported_reason(self, N: int) -> Optional[str]:
        for attn, ff in self._layers():
            if attn.dim_head not in (64, 80):
                return f"dim_head={attn.dim_head} (the attention kernels are built for 64 and 80)"
            if attn.dim_head == 80 and (N > 512 or getattr(attn, "q_norm", None) is not None):
                return "dim_head=80 is built for the single-pass attention kernel (N <= 512, no q/k norm) only"
            if attn.dim % 8 or ff.hidden_dim % 8:
                return "dim / mlp_dim not multiples of 8"
        if N > 16384:
            return f"sequence length {N} > 16384"
        return None

    # -------------------------------------------------------------------------------------------- weights
    def prepared(self) -> Dict[str, torch.Tensor]:
        params = self.params()
        key = _version_key(params)
        if self.prep.key == key:
            return self.prep.t
        t: Dict[str, torch.Tensor] = {}

        def fold(prefix: str, lin_w: torch.Tensor, lin_b: Optional[torch.Tensor], g: torch.Tensor, b: torch.Tensor):
            # LN(x) W^T + bias  ==  rstd * (x (gamma*W)^T - mu * colsum) + (W beta + bias)
            w32 = lin_w.detach().float()
            wg = (w32 * g.detach().float()[None, :]).to(torch.bfloat16).contiguous()
            t[prefix + ".wg"] = wg
            t[prefix + ".s"] = wg.float().sum(dim=1).contiguous()          # from the ROUNDED weights the MMA sees
            tb = w32 @ b.detach().float()
            t[prefix + ".t"] = (tb + lin_b.detach().float() if lin_b is not None else tb).contiguous()

        for i, (attn, ff) in enumerate(self._layers()):
            t[f"{i}.ln1.w"], t[f"{i}.ln1.b"] = _f32(attn.norm.weight), _f32(attn.norm.bias)
            t[f"{i}.qkv.w"] = _bf16_rows(attn.to_qkv.weight)
            fold(f"{i}.qkv", attn.to_qkv.weight, None, attn.norm.weight, attn.norm.bias)
            fold(f"{i}.fc1", ff.parts()[1].weight, ff.parts()[1].bias, ff.parts()[0].weight, ff.parts()[0].bias)
            out_lin = attn.out_linear() if getattr(attn, "project_out", True) else None
            if out_lin is None:
                # reference vit.py:34,46-49: heads == 1 and dim_head == dim -> to_out is nn.Identity.  The residual
                # GEMM then runs with an identity weight: bf16 x 1.0 products accumulate exactly, so x += o bit for bit
                t[f"{i}.out.w"] = torch.eye(attn.dim, device=attn.to_qkv.weight.device, dtype=torch.bfloat16)
                t[f"{i}.out.b"] = None
            else:
                t[f"{i}.out.w"] = _bf16_rows(out_lin.weight)
                t[f"{i}.out.b"] = _f32(out_lin.bias) if out_lin.bias is not None else None
            if getattr(attn, "q_norm", None) is not None:
                # per-head q / k RMSNorm (simple_vit_with_qk_norm.py:29-37,60-67): epilogue of the QKV GEMM
                t[f"{i}.gqk"] = torch.cat([_f32(attn.q_norm.gamma).reshape(-1), _f32(attn.k_norm.gamma).reshape(-1)])
            ln, fc1, fc2 = ff.parts()
            t[f"{i}.ln2.w"], t[f"{i}.ln2.b"] = _f32(ln.weight), _f32(ln.bias)
            t[f"{i}.fc1.w"], t[f"{i}.fc1.b"] = _bf16_rows(fc1.weight), _f32(fc1.bias)
            t[f"{i}.fc2.w"], t[f"{i}.fc2.b"] = _bf16_rows(fc2.weight), _f32(fc2.bias)
        if self.has_final_norm():
            t["norm.w"], t["norm.b"] = _f32(self.mod.norm.weight), _f32(self.mod.norm.bias)
        t["c_layers"] = self._c_layers(t)            # type: ignore[assignment]
        self.prep.key, self.prep.t = key, t
        return t

    def _c_layers(self, t: Dict[str, torch.Tensor]):
        """(ctypes array of b200vit_layer, heads, dh, hidden, scale) for the one-call encoder (b200vit_encoder_blocks),
        or None when the layers are not uniform.  The pointers stay valid as long as `t` (which holds the tensors)."""
        layers = list(self._layers())
        a0, f0 = layers[0]
        sig = (a0.heads, a0.dim_head, f0.hidden_dim, _softmax_scale(a0))
        if any((a.heads, a.dim_head, f.hidden_dim, _softmax_scale(a)) != sig for a, f in layers):
            return None
        arr = (_lib.Layer * len(layers))()
        p = lambda v: None if v is None else v.data_ptr()      # noqa: E731
        for i, (attn, ff) in enumerate(layers):
            L = arr[i]
            L.qkv_wg, L.qkv_t, L.qkv_s = p(t[f"{i}.qkv.wg"]), p(t[f"{i}.qkv.t"]), p(t[f"{i}.qkv.s"])
            L.qk_gamma = p(t.get(f"{i}.gqk"))
            L.out_w, L.out_b = p(t[f"{i}.out.w"]), p(t[f"{i}.out.b"])
            L.fc1_wg, L.fc1_t, L.fc1_s = p(t[f"{i}.fc1.wg"]), p(t[f"{i}.fc1.t"]), p(t[f"{i}.fc1.s"])
            L.fc2_w, L.fc2_b = p(t[f"{i}.fc2.w"]), p(t[f"{i}.fc2.b"])
            L.ln1_eps, L.ln2_eps = float(attn.norm.eps), float(ff.parts()[0].eps)
        return arr, sig

    # -------------------------------------------------------------------------------------------- workspaces
    def workspace(self, M: int, device: torch.device) -> Dict[str, torch.Tensor]:
        attn0, ff0 = next(iter(self._layers()))
        D, I, Hd = attn0.dim, attn0.heads * attn0.dim_head, ff0.hidden_dim
        # one workspace per (shape, stream): two streams running the same model must not share scratch buffers
        key = (M, D, I, Hd, device, torch.cuda.current_stream(device).cuda_stream)
        if self.ws_key != key:
            bf = dict(device=device, dtype=torch.bfloat16)
            self.ws = {
                "xn": torch.empty(M, D, **bf),          # exact: LayerNorm output; fold: bf16 copy of x
                "qkv": torch.empty(M, 3 * I, **bf),
                "o": torch.empty(M, I, **bf),
                "h": torch.empty(M, Hd, **bf),
                # LN-fold row statistics: [M, 1, 2] written by embed_tokens / rowstats_cast, [M, parts(D), 2] by GEMMs
                "stats_in": torch.empty(M, 1, 2, device=device, dtype=torch.float32),
                "stats_a": torch.empty(M, _lib.stats_parts(D), 2, device=device, dtype=torch.float32),
                "stats_b": torch.empty(M, _lib.stats_parts(D), 2, device=device, dtype=torch.float32),
            }
            w = self.ws
            self.c_ws = _lib.EncoderWs(w["xn"].data_ptr(), w["qkv"].data_ptr(), w["o"].data_ptr(), w["h"].data_ptr(),
                                       w["stats_in"].data_ptr(), w["stats_a"].data_ptr(), w["stats_b"].data_ptr())
            self.ws_key = key
        return self.ws

    # -------------------------------------------------------------------------------------------- execution
    def _attention(self, ws: Dict[str, torch.Tensor], B: int, N: int, attn) -> None:
        """Single-pass kernel for N <= 512 keys, the key-block (varlen) kernel beyond."""
        if N <= 512:
            _lib.attention(ws["qkv"], ws["o"], B, N, attn.heads, attn.dim_head, _softmax_scale(attn))
            return
        key = (B, N, ws["qkv"].device)
        if getattr(self, "_vl_key", None) != key:
            self._vl = _lib.varlen_index([N] * B, ws["qkv"].device)
            self._vl_key = key
        cu, tp, tiles = self._vl
        _lib.attention_varlen(ws["qkv"], ws["o"], cu, tp, tiles, attn.heads, attn.dim_head, _softmax_scale(attn))

    def run_blocks(self, x: torch.Tensor, B: int, N: int, primed: bool = False) -> None:
        """All encoder layers, in place on the fp32 residual stream x[B*N, D] (no final LayerNorm).

        fold mode needs ws['xn'] (bf16 copy of x) and ws['stats_in'] (row sums of that copy) on entry: `primed` says
        the caller (embed_tokens) already wrote them, otherwise one rowstats_cast pass produces them."""
        t = self.prepared()
        M = B * N
        ws = self.workspace(M, x.device)
        if ln_mode() == "fold":
            xb, sa, sb = ws["xn"], ws["stats_a"], ws["stats_b"]
            if t["c_layers"] is not None and not _lib.profiling() and os.environ.get(_HOST_LOOP_ENV, "c") == "c":
                # the whole layer loop below the language boundary: one ctypes call instead of 5 x depth
                arr, (heads, dh, hidden, scale) = t["c_layers"]
                varlen = None
                if N > 512:
                    key = (B, N, x.device)
                    if getattr(self, "_vl_key", None) != key:
                        self._vl = _lib.varlen_index([N] * B, x.device)
                        self._vl_key = key
                    varlen = self._vl
                _lib.encoder_blocks(arr, len(arr), x, self.c_ws, B, N, x.shape[1], heads, dh, hidden, scale, primed,
                                    varlen)
                return
            if not primed:
                _lib.rowstats_cast(x, xb, ws["stats_in"])
            for i, (attn, ff) in enumerate(self._layers()):
                if f"{i}.gqk" in t:
                    _lib.gemm_headnorm(xb, t[f"{i}.qkv.wg"], out_bf16=ws["qkv"], bias=t[f"{i}.qkv.t"],
                                       ln_sums=ws["stats_in"] if i == 0 else sa, col_s=t[f"{i}.qkv.s"],
                                       ln_eps=attn.norm.eps, head_gamma=t[f"{i}.gqk"], norm_heads=2 * attn.heads)
                else:
                    _lib.gemm(xb, t[f"{i}.qkv.wg"], out_bf16=ws["qkv"], bias=t[f"{i}.qkv.t"],
                              ln_sums=ws["stats_in"] if i == 0 else sa, col_s=t[f"{i}.qkv.s"], ln_eps=attn.norm.eps)
                self._attention(ws, B, N, attn)
                _lib.gemm(ws["o"], t[f"{i}.out.w"], out_f32=x, out_bf16=xb, bias=t[f"{i}.out.b"], resid=x,
                          stats_out=sb)
                _lib.gemm(xb, t[f"{i}.fc1.wg"], out_bf16=ws["h"], bias=t[f"{i}.fc1.t"], gelu=True, ln_sums=sb,
                          col_s=t[f"{i}.fc1.s"], ln_eps=ff.parts()[0].eps)
                _lib.gemm(ws["h"], t[f"{i}.fc2.w"], out_f32=x, out_bf16=xb, bias=t[f"{i}.fc2.b"], resid=x,
                          stats_out=sa)
            return
        for i, (attn, ff) in enumerate(self._layers()):
            _lib.layernorm(x, t[f"{i}.ln1.w"], t[f"{i}.ln1.b"], out_bf16=ws["xn"], eps=attn.norm.eps)
            if f"{i}.gqk" in t:
                _lib.gemm_headnorm(ws["xn"], t[f"{i}.qkv.w"], out_bf16=ws["qkv"], head_gamma=t[f"{i}.gqk"],
                                   norm_heads=2 * attn.heads)
            else:
                _lib.gemm(ws["xn"], t[f"{i}.qkv.w"], out_bf16=ws["qkv"])
            self._attention(ws, B, N, attn)
            _lib.gemm(ws["o"], t[f"{i}.out.w"], out_f32=x, bias=t[f"{i}.out.b"], resid=x)
            _lib.layernorm(x, t[f"{i}.ln2.w"], t[f"{i}.ln2.b"], out_bf16=ws["xn"], eps=ff.parts()[0].eps)
            _lib.gemm(ws["xn"], t[f"{i}.fc1.w"], out_bf16=ws["h"], bias=t[f"{i}.fc1.b"], gelu=True)
            _lib.gemm(ws["h"], t[f"{i}.fc2.w"], out_f32=x, bias=t[f"{i}.fc2.b"], resid=x)

    def final_norm(self, x: torch.Tensor, *, out_bf16: Optional[torch.Tensor] = None,
                   out_f32: Optional[torch.Tensor] = None, row_index: Optional[torch.Tensor] = None) -> None:
        t = self.prepared()
        assert self.has_final_norm()
        _lib.layernorm(x, t["norm.w"], t["norm.b"], out_bf16=out_bf16, out_f32=out_f32, row_index=row_index,
                       eps=self.mod.norm.eps)

    def forward_tokens(self, tokens: torch.Tensor) -> torch.Tensor:
        """Transformer.forward on arbitrary bf16 tokens [B, N, D] (what MAE / SimMIM / Distill call,
        reference mae.py:74, simmim.py:70, distill.py:66)."""
        B, N, D = tokens.shape
        with on_device(tokens):
            x = tokens.reshape(B * N, D).float().contiguous()
            self.run_blocks(x, B, N)
            out = torch.empty(B * N, D, device=tokens.device, dtype=torch.bfloat16)
            if self.has_final_norm():
                self.final_norm(x, out_bf16=out)
            else:
                _lib.cast_f32_bf16(x.view(-1), out.view(-1))
        return out.view(B, N, D)


class PatchEmbedEngine:
    """Fused patch embedding + token assembly (reference vit.py:99-104,120-127 / simple_vit.py:90-95,113-114)."""

    def __init__(self, owner: nn.Module) -> None:
        self.owner = owner
        self.prep = _Prepared()

    def params(self) -> List[torch.Tensor]:
        o = self.owner
        ps = list(o.to_patch_embedding.parameters())
        for name in ("cls_token", "pos_embedding", "register_tokens"):
            v = getattr(o, name, None)
            if isinstance(v, nn.Parameter):
                ps.append(v)
        return ps

    def prepared(self, device: torch.device) -> Dict[str, torch.Tensor]:
        o = self.owner
        params = self.params()
        key = _version_key(params) + (str(device),)
        if self.prep.key == key:
            return self.prep.t
        ln1, lin, ln2 = o.to_patch_embedding[1], o.to_patch_embedding[2], o.to_patch_embedding[3]
        pd = lin.weight.shape[1]
        kp = (pd + 63) // 64 * 64
        t = {
            "ln1.w": _f32(ln1.weight), "ln1.b": _f32(ln1.bias),
            "w": _bf16_rows(lin.weight, kp), "b": _f32(lin.bias),
            "ln2.w": _f32(ln2.weight), "ln2.b": _f32(ln2.bias),
        }
        t["kp"] = kp  # type: ignore[assignment]
        ph, pw = getattr(o, "fused_patch_box", None) or o.patch_size
        if ph == 16 and pw == 16 and pd % 256 == 0:
            # im2col-free path (b200vit_patch_embed_tma): LayerNorm(patch) folded into the projection, weight columns
            # permuted from the reference's (p1 p2 c) order (vit.py:100) to the image's own (c p1 p2)
            C = pd // 256
            w32 = lin.weight.detach().float()
            wg = w32 * ln1.weight.detach().float()[None, :]
            t["tma.w"] = wg.view(-1, 256, C).permute(0, 2, 1).reshape(-1, pd).to(torch.bfloat16).contiguous()
            t["tma.s"] = t["tma.w"].float().sum(dim=1).contiguous()           # from the ROUNDED weights the MMA sees
            t["tma.b"] = (w32 @ ln1.bias.detach().float() + lin.bias.detach().float()).contiguous()
        cls = getattr(o, "cls_token", None)
        t["cls"] = _f32(cls) if (cls is not None and cls.shape[0] > 0) else None
        reg = getattr(o, "register_tokens", None)          # simple_vit_with_register_tokens.py:103,124-126
        t["tail"] = _f32(reg) if (reg is not None and reg.shape[0] > 0) else None
        pos = getattr(o, "pos_embedding", None)
        t["pos"] = pos.detach().to(device=device, dtype=torch.float32).contiguous() if pos is not None else None
        self.prep.key, self.prep.t = key, t
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
        dev = img.device
        y = torch.empty(B * n, D, device=dev, dtype=torch.float32)
        if ("tma.w" in t and (ph, pw) == (16, 16) and os.environ.get(_PATCH_MODE_ENV, "tma") == "tma"
                and W // pw <= 128 and D % 8 == 0):
            # the wgmma GEMM reads the image itself: no patch matrix, no LayerNorm pass
            stats_p = torch.empty(B * n, 2, device=dev, dtype=torch.float32)
            _lib.patch_embed_tma(img.contiguous(), t["tma.w"], t["tma.b"], t["tma.s"], stats_p, y,
                                 eps=o.to_patch_embedding[1].eps)
        else:
            a0 = torch.empty(B * n, t["kp"], device=dev, dtype=torch.bfloat16)
            _lib.patchify_ln(img.contiguous(), t["ln1.w"], t["ln1.b"], a0, ph, pw, eps=o.to_patch_embedding[1].eps)
            _lib.gemm(a0, t["w"], out_f32=y, bias=t["b"])
        x = torch.empty(B * N, D, device=dev, dtype=torch.float32)
        _lib.embed_tokens(y, t["ln2.w"], t["ln2.b"], t["cls"], pos, x, B, n, ncls, xb=xb, stats=stats,
                          eps=o.to_patch_embedding[3].eps, tail=t["tail"])
        return x, B, N

    def geometry(self, img: torch.Tensor, patch: Optional[Tuple[int, int]] = None) -> Tuple[int, int]:
        """(B, N) the image batch will produce, without running anything."""
        ph, pw = patch if patch is not None else self.owner.patch_size
        cls = getattr(self.owner, "cls_token", None)
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
        params = self.params()
        key = _version_key(params)
        if self.prep.key != key:
            self.prep.t = {"w": _bf16_rows(self.lin.weight),
                           "b": _f32(self.lin.bias) if self.lin.bias is not None else None}
            self.prep.key = key
        t = self.prep.t
        out = torch.empty(pooled_bf16.shape[0], t["w"].shape[0], device=pooled_bf16.device, dtype=torch.bfloat16)
        _lib.gemm(pooled_bf16.contiguous(), t["w"], out_bf16=out, bias=t["b"])
        return out


def fused_mean_pooled_features(owner: nn.Module, img: torch.Tensor, pool_tokens: Optional[int] = None,
                               patch: Optional[Tuple[int, int]] = None,
                               pos: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Shared body of the SimpleViT-family fused forwards (reference simple_vit.py:110-117 and its variants):
    patch embedding (+ register tokens) -> encoder blocks -> final LayerNorm if the Transformer has one -> mean over
    the first `pool_tokens` tokens of every image (all tokens by default).  Returns fp32 [B, D]; must run inside
    on_device(img)."""
    if getattr(owner, "_patch_engine", None) is None:
        owner._patch_engine = PatchEmbedEngine(owner)
    eng = owner.transformer.engine()
    B, N = owner._patch_engine.geometry(img, patch)
    if transformer_is_hooked(owner):
        x, B, N = owner._patch_engine.run(img, patch=patch, pos=pos)
        xf = hooked_transformer_tokens(owner, x, B, N).reshape(B * N, -1).float()
        pm = torch.empty(B, xf.shape[1], device=img.device, dtype=torch.float32)
        _lib.mean_pool(xf, pm, B, N, xf.shape[1], n_pool=pool_tokens)
        return pm
    primed = ln_mode() == "fold"
    ws = eng.workspace(B * N, img.device) if primed else None
    x, B, N = owner._patch_engine.run(img, xb=ws["xn"] if primed else None, stats=ws["stats_in"] if primed else None,
                                      patch=patch, pos=pos)
    D = x.shape[1]
    eng.run_blocks(x, B, N, primed=primed)
    if eng.has_final_norm():
        xf = torch.empty_like(x)
        eng.final_norm(x, out_f32=xf)
    else:
        xf = x
    pm = torch.empty(B, D, device=img.device, dtype=torch.float32)
    _lib.mean_pool(xf, pm, B, N, D, n_pool=pool_tokens)
    return pm
