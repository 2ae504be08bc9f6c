"""ctypes binding of libb200vit.so (the C ABI declared in include/b200vit.h).

No torch C++ headers are involved: tensors cross the boundary as raw device pointers + sizes, the stream as the
cudaStream_t handle of torch's current stream.  There is NO fallback here: if the library is missing or a call
fails, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path
from typing import Optional

import torch

_PKG = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ["B200VIT_LIB"]).resolve() if os.environ.get("B200VIT_LIB") else _PKG / "lib" / "libb200vit.so"

EPI_BIAS = 1
EPI_GELU = 2
EPI_RESIDUAL = 4
EPI_LNFOLD = 8
EPI_STATS = 16
EPI_HEADLN = 64

# every symbol include/b200vit.h declares (tests check that the library exports each of them)
SYMBOLS = [
    "b200vit_last_error", "b200vit_version", "b200vit_launch_count", "b200vit_reset_launch_count",
    "b200vit_device_ok", "b200vit_gemm_bf16", "b200vit_layernorm", "b200vit_patchify_ln", "b200vit_embed_tokens",
    "b200vit_attention", "b200vit_mean_pool", "b200vit_cast_f32_bf16", "b200vit_rowstats_cast", "b200vit_debug_set",
    "b200vit_stats_parts", "b200vit_attention_varlen", "b200vit_qk_rmsnorm", "b200vit_attn_pool",
    "b200vit_patchify_varlen_ln", "b200vit_rmsnorm_heads", "b200vit_embed_varlen",
    "b200vit_gemm_headnorm_bf16", "b200vit_layernorm_heads", "b200vit_patch_stats", "b200vit_patch_embed_tma",
    "b200vit_encoder_blocks",
]


class Layer(C.Structure):
    """struct b200vit_layer (include/b200vit.h): LN-folded weights of one encoder layer, raw device pointers."""
    _fields_ = [("qkv_wg", C.c_void_p), ("qkv_t", C.c_void_p), ("qkv_s", C.c_void_p), ("qk_gamma", C.c_void_p),
                ("out_w", C.c_void_p), ("out_b", C.c_void_p), ("fc1_wg", C.c_void_p), ("fc1_t", C.c_void_p),
                ("fc1_s", C.c_void_p), ("fc2_w", C.c_void_p), ("fc2_b", C.c_void_p),
                ("ln1_eps", C.c_float), ("ln2_eps", C.c_float)]


class EncoderWs(C.Structure):
    """struct b200vit_encoder_ws: scratch buffers of b200vit_encoder_blocks."""
    _fields_ = [("xb", C.c_void_p), ("qkv", C.c_void_p), ("o", C.c_void_p), ("h", C.c_void_p),
                ("stats_in", C.c_void_p), ("stats_a", C.c_void_p), ("stats_b", C.c_void_p)]

_lib: Optional[C.CDLL] = None


class B200VitError(RuntimeError):
    pass


def lib() -> C.CDLL:
    """Load (once) and return the shared library; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise B200VitError(
            f"{LIB_PATH} not found: build it with `python -m vit_pytorch_b200.build` "
            "(there is no fallback for the fused CUDA path)")
    L = C.CDLL(str(LIB_PATH))
    vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_int64, C.c_float
    L.b200vit_last_error.restype = C.c_char_p
    L.b200vit_last_error.argtypes = []
    L.b200vit_version.restype = i32
    L.b200vit_launch_count.restype = i64
    L.b200vit_reset_launch_count.restype = None
    L.b200vit_device_ok.restype = i32
    L.b200vit_device_ok.argtypes = [i32]
    L.b200vit_gemm_bf16.restype = i32
    L.b200vit_gemm_bf16.argtypes = [vp, i64, vp, i64, vp, vp, i64, vp, vp, vp, i32, f32, vp, vp, i32, i32, i32, i32,
                                    vp]
    L.b200vit_gemm_headnorm_bf16.restype = i32
    L.b200vit_gemm_headnorm_bf16.argtypes = [vp, i64, vp, i64, vp, i64, vp, vp, i32, f32, vp, vp, i32, i32, f32, i32,
                                             i32, i32, i32, vp]
    L.b200vit_layernorm_heads.restype = i32
    L.b200vit_layernorm_heads.argtypes = [vp, i64, vp, i32, i32, i32, f32, vp]
    L.b200vit_stats_parts.restype = i32
    L.b200vit_stats_parts.argtypes = [i32]
    L.b200vit_layernorm.restype = i32
    L.b200vit_layernorm.argtypes = [vp, i64, vp, vp, vp, vp, i64, vp, i32, i32, f32, vp]
    L.b200vit_patchify_ln.restype = i32
    L.b200vit_patchify_ln.argtypes = [vp, vp, vp, vp, i64, i32, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_patch_stats.restype = i32
    L.b200vit_patch_stats.argtypes = [vp, vp, i32, i32, i32, i32, vp]
    L.b200vit_patch_embed_tma.restype = i32
    L.b200vit_patch_embed_tma.argtypes = [vp, vp, vp, vp, vp, f32, vp, i64, i32, i32, i32, i32, i32, vp]
    L.b200vit_embed_tokens.restype = i32
    L.b200vit_embed_tokens.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_rowstats_cast.restype = i32
    L.b200vit_rowstats_cast.argtypes = [vp, vp, vp, i32, i32, vp]
    L.b200vit_debug_set.restype = i32
    L.b200vit_debug_set.argtypes = [i32, i32]
    L.b200vit_attention.restype = i32
    L.b200vit_attention.argtypes = [vp, vp, i32, i32, i32, i32, f32, vp]
    L.b200vit_attention_varlen.restype = i32
    L.b200vit_attention_varlen.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_patchify_varlen_ln.restype = i32
    L.b200vit_patchify_varlen_ln.argtypes = [vp, vp, vp, vp, vp, vp, i64, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_qk_rmsnorm.restype = i32
    L.b200vit_qk_rmsnorm.argtypes = [vp, vp, i32, i32, i32, vp]
    L.b200vit_rmsnorm_heads.restype = i32
    L.b200vit_rmsnorm_heads.argtypes = [vp, i64, vp, i32, i32, i32, vp]
    L.b200vit_embed_varlen.restype = i32
    L.b200vit_embed_varlen.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, i32, i32, i32, i32, f32, vp]
    L.b200vit_attn_pool.restype = i32
    L.b200vit_attn_pool.argtypes = [vp, vp, vp, vp, i32, i32, i32, vp]
    L.b200vit_mean_pool.restype = i32
    L.b200vit_mean_pool.argtypes = [vp, vp, i32, i32, i32, i32, vp]
    L.b200vit_cast_f32_bf16.restype = i32
    L.b200vit_cast_f32_bf16.argtypes = [vp, vp, i64, vp]
    L.b200vit_encoder_blocks.restype = i32
    L.b200vit_encoder_blocks.argtypes = [C.POINTER(Layer), i32, vp, C.POINTER(EncoderWs), i32, i32, i32, i32, i32, i32,
                                         f32, i32, vp, vp, i32, vp]
    _lib = L
    return L


def _check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().b200vit_last_error()
        raise B200VitError(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _stream() -> int:
    """cudaStream_t of torch's current stream on the CURRENT device.  Every fused forward runs inside
    `with torch.cuda.device(x.device)` (engine.on_device), so this is the stream of the tensors' device; the library
    itself never calls cudaSetDevice."""
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------------------------
# optional per-call CUDA-event timing (bench.py's roofline pass); None = off (the normal, un-instrumented path)
# ------------------------------------------------------------------------------------------------------------------
_prof: Optional[list] = None


def profile_start() -> None:
    global _prof
    _prof = []


def profile_stop() -> list:
    """Returns [(kernel, meta, milliseconds), ...] for every library call since profile_start()."""
    global _prof
    rec, _prof = _prof or [], None
    torch.cuda.synchronize()
    return [(name, meta, e0.elapsed_time(e1)) for name, meta, e0, e1 in rec]


class _Timed:
    def __init__(self, name: str, **meta) -> None:
        self.name, self.meta = name, meta

    def __enter__(self):
        if _prof is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if _prof is not None:
            self.e1.record()
            _prof.append((self.name, self.meta, self.e0, self.e1))
        return False


def profiling() -> bool:
    """True between profile_start() and profile_stop(): callers that batch several kernels into one library call
    (encoder_blocks) go call by call instead, so that every kernel gets its own events."""
    return _prof is not None


def encoder_blocks(layers, depth: int, x: torch.Tensor, ws: "EncoderWs", B: int, N: int, D: int, heads: int, dh: int,
                   hidden: int, scale: float, primed: bool, varlen=None) -> None:
    """All encoder layers in one library call (b200vit_encoder_blocks).  `layers`: ctypes array of Layer built from the
    prepared weights; `ws`: EncoderWs over the engine's workspace; `varlen`: (cu, tile_prefix, total_tiles) if N > 512."""
    _chk(x, torch.float32, "x")
    cu, tp, tiles = varlen if varlen is not None else (None, None, 0)
    rc = lib().b200vit_encoder_blocks(layers, depth, _ptr(x), C.byref(ws), B, N, D, heads, dh, hidden, float(scale),
                                      1 if primed else 0, _ptr(cu), _ptr(tp), int(tiles), _stream())
    _check(rc, "b200vit_encoder_blocks")


def launch_count() -> int:
    return int(lib().b200vit_launch_count())


def reset_launch_count() -> None:
    lib().b200vit_reset_launch_count()


def device_ok(dev: int) -> bool:
    return lib().b200vit_device_ok(int(dev)) == 0


def _chk(t: Optional[torch.Tensor], dtype, name: str) -> None:
    if t is None:
        return
    if not t.is_cuda or t.dtype != dtype:
        raise B200VitError(f"{name}: expected CUDA {dtype}, got {t.device} {t.dtype}")
    if t.device.index != torch.cuda.current_device():
        raise B200VitError(f"{name} lives on {t.device} but the current CUDA device is {torch.cuda.current_device()}: "
                           "wrap the call in `with torch.cuda.device(tensor.device)`")


def gemm(a: torch.Tensor, w: torch.Tensor, *, out_bf16: Optional[torch.Tensor] = None,
         out_f32: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None,
         resid: Optional[torch.Tensor] = None, gelu: bool = False, ln_sums: Optional[torch.Tensor] = None,
         ln_eps: float = 1e-5, col_s: Optional[torch.Tensor] = None, stats_out: Optional[torch.Tensor] = None,
         n: Optional[int] = None, k: Optional[int] = None) -> None:
    """out = epilogue(a[M,K] @ w[N,K]^T).  a, w bf16 row-major (last stride 1).

    ln_sums: [M, parts, 2] (or [M, 2]) partial row sums of `a`; stats_out: [M, stats_parts(N), 2], fully overwritten."""
    _chk(a, torch.bfloat16, "a"); _chk(w, torch.bfloat16, "w")
    _chk(out_bf16, torch.bfloat16, "out_bf16"); _chk(out_f32, torch.float32, "out_f32")
    for nm, t in (("bias", bias), ("resid", resid), ("ln_sums", ln_sums), ("col_s", col_s), ("stats_out", stats_out)):
        _chk(t, torch.float32, nm)
    assert a.dim() == 2 and w.dim() == 2 and a.stride(1) == 1 and w.stride(1) == 1
    M = a.shape[0]
    K = a.shape[1] if k is None else k
    N = w.shape[0] if n is None else n
    out = out_bf16 if out_bf16 is not None else out_f32
    assert out is not None and out.stride(1) == 1
    if out_bf16 is not None and out_f32 is not None:
        assert out_bf16.stride(0) == out_f32.stride(0)
    flags = 0
    if bias is not None:
        flags |= EPI_BIAS
    if gelu:
        flags |= EPI_GELU
    if resid is not None:
        flags |= EPI_RESIDUAL
        assert resid.stride(0) == out.stride(0)
    ln_parts = 0
    if ln_sums is not None:
        flags |= EPI_LNFOLD
        assert ln_sums.is_contiguous() and ln_sums.shape[0] == M and ln_sums.shape[-1] == 2
        ln_parts = 1 if ln_sums.dim() == 2 else ln_sums.shape[1]
    if stats_out is not None:
        flags |= EPI_STATS
        assert stats_out.is_contiguous() and tuple(stats_out.shape) == (M, stats_parts(N), 2), \
            f"stats_out must be [M, {stats_parts(N)}, 2]"
    with _Timed("gemm", M=M, N=N, K=K, flags=flags, flops=2.0 * M * N * K):
        rc = lib().b200vit_gemm_bf16(_ptr(a), a.stride(0), _ptr(w), w.stride(0), _ptr(out_bf16), _ptr(out_f32),
                                     out.stride(0), _ptr(bias), _ptr(resid), _ptr(ln_sums), ln_parts, float(ln_eps),
                                     _ptr(col_s), _ptr(stats_out), M, N, K, flags, _stream())
    _check(rc, "b200vit_gemm_bf16")


def gemm_headnorm(a: torch.Tensor, w: torch.Tensor, *, out_bf16: torch.Tensor, head_gamma: torch.Tensor,
                  norm_heads: int, dh: int = 64, bias: Optional[torch.Tensor] = None,
                  ln_sums: Optional[torch.Tensor] = None, ln_eps: float = 1e-5,
                  col_s: Optional[torch.Tensor] = None, head_layernorm_eps: Optional[float] = None) -> None:
    """out = epilogue(a @ w^T) with the first norm_heads heads of every row RMS-normalised (NaViT q / k norm), or --
    head_layernorm_eps given -- LayerNorm-ed without bias (nested-tensor NaViT)."""
    _chk(a, torch.bfloat16, "a"); _chk(w, torch.bfloat16, "w"); _chk(out_bf16, torch.bfloat16, "out_bf16")
    for nm, t in (("bias", bias), ("ln_sums", ln_sums), ("col_s", col_s), ("head_gamma", head_gamma)):
        _chk(t, torch.float32, nm)
    assert a.dim() == 2 and w.dim() == 2 and a.stride(1) == 1 and w.stride(1) == 1 and out_bf16.stride(1) == 1
    M, K = a.shape
    N = w.shape[0]
    assert head_gamma.is_contiguous() and head_gamma.numel() == norm_heads * dh
    flags = 0
    if bias is not None:
        flags |= EPI_BIAS
    ln_parts = 0
    if ln_sums is not None:
        flags |= EPI_LNFOLD
        assert ln_sums.is_contiguous() and ln_sums.shape[0] == M and ln_sums.shape[-1] == 2
        ln_parts = 1 if ln_sums.dim() == 2 else ln_sums.shape[1]
    head_eps = 0.0
    if head_layernorm_eps is not None:
        flags |= EPI_HEADLN
        head_eps = float(head_layernorm_eps)
    with _Timed("gemm", M=M, N=N, K=K, flags=flags, flops=2.0 * M * N * K):
        rc = lib().b200vit_gemm_headnorm_bf16(_ptr(a), a.stride(0), _ptr(w), w.stride(0), _ptr(out_bf16),
                                              out_bf16.stride(0), _ptr(bias), _ptr(ln_sums), ln_parts, float(ln_eps),
                                              _ptr(col_s), _ptr(head_gamma), norm_heads, dh, head_eps, M, N, K, flags,
                                              _stream())
    _check(rc, "b200vit_gemm_headnorm_bf16")


def stats_parts(n: int) -> int:
    return int(lib().b200vit_stats_parts(int(n)))


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: Optional[torch.Tensor], *,
              out_bf16: Optional[torch.Tensor] = None, out_f32: Optional[torch.Tensor] = None,
              row_index: Optional[torch.Tensor] = None, eps: float = 1e-5) -> None:
    _chk(x, torch.float32, "x"); _chk(gamma, torch.float32, "gamma"); _chk(beta, torch.float32, "beta")
    _chk(out_bf16, torch.bfloat16, "out_bf16"); _chk(out_f32, torch.float32, "out_f32")
    assert x.dim() == 2 and x.stride(1) == 1
    out = out_bf16 if out_bf16 is not None else out_f32
    assert out is not None
    M = out.shape[0]
    D = x.shape[1]
    if row_index is not None:
        assert row_index.dtype == torch.int32 and row_index.numel() == M
    else:
        assert x.shape[0] == M
    nbytes = M * D * (4 + (2 if out_bf16 is not None else 0) + (4 if out_f32 is not None else 0))
    with _Timed("layernorm", M=M, D=D, bytes=nbytes):
        rc = lib().b200vit_layernorm(_ptr(x), x.stride(0), _ptr(gamma), _ptr(beta), _ptr(out_bf16), _ptr(out_f32),
                                     out.stride(0), _ptr(row_index), M, D, float(eps), _stream())
    _check(rc, "b200vit_layernorm")


def patchify_ln(img: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, out_bf16: torch.Tensor, ph: int, pw: int,
                eps: float = 1e-5) -> None:
    _chk(img, torch.bfloat16, "img"); _chk(out_bf16, torch.bfloat16, "out")
    _chk(gamma, torch.float32, "gamma"); _chk(beta, torch.float32, "beta")
    assert img.is_contiguous() and img.dim() == 4
    B, Cc, H, W = img.shape
    with _Timed("patchify_ln", bytes=img.numel() * 2 + out_bf16.numel() * 2):
        rc = lib().b200vit_patchify_ln(_ptr(img), _ptr(gamma), _ptr(beta), _ptr(out_bf16), out_bf16.stride(0), B, Cc,
                                       H, W, ph, pw, float(eps), _stream())
    _check(rc, "b200vit_patchify_ln")


def patch_embed_tma(img: torch.Tensor, w_perm: torch.Tensor, bias: torch.Tensor, col_s: torch.Tensor,
                    stats: torch.Tensor, out_f32: torch.Tensor, eps: float = 1e-5) -> None:
    """out_f32[B*n, D] = LayerNorm(16x16 patches of img) @ W^T + b, the image read through a 5-D TMA map (no patch
    matrix in memory).  w_perm / bias / col_s: see include/b200vit.h; stats [B*n, 2] is scratch (fully overwritten)."""
    _chk(img, torch.bfloat16, "img"); _chk(w_perm, torch.bfloat16, "w_perm"); _chk(out_f32, torch.float32, "out")
    for nm, t in (("bias", bias), ("col_s", col_s), ("stats", stats)):
        _chk(t, torch.float32, nm)
    assert img.is_contiguous() and img.dim() == 4 and w_perm.is_contiguous() and out_f32.stride(1) == 1
    B, Cc, H, W = img.shape
    D = w_perm.shape[0]
    n = (H // 16) * (W // 16)
    assert w_perm.shape[1] == Cc * 256 and out_f32.shape == (B * n, D) and stats.is_contiguous() and stats.numel() == 2 * B * n
    with _Timed("patch_stats", bytes=img.numel() * 2):
        rc = lib().b200vit_patch_stats(_ptr(img), _ptr(stats), B, Cc, H, W, _stream())
    _check(rc, "b200vit_patch_stats")
    with _Timed("gemm", M=B * n, N=D, K=Cc * 256, flags=EPI_LNFOLD | EPI_BIAS, flops=2.0 * B * n * D * Cc * 256):
        rc = lib().b200vit_patch_embed_tma(_ptr(img), _ptr(w_perm), _ptr(bias), _ptr(col_s), _ptr(stats), float(eps),
                                           _ptr(out_f32), out_f32.stride(0), B, Cc, H, W, D, _stream())
    _check(rc, "b200vit_patch_embed_tma")


def embed_tokens(y: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, cls: Optional[torch.Tensor],
                 pos: torch.Tensor, x: torch.Tensor, B: int, n: int, ncls: int, eps: float = 1e-5,
                 xb: Optional[torch.Tensor] = None, stats: Optional[torch.Tensor] = None,
                 tail: Optional[torch.Tensor] = None) -> None:
    """tail [ntail, D]: rows appended after the n patch tokens of every image (register tokens, no pos)."""
    _chk(xb, torch.bfloat16, "xb"); _chk(stats, torch.float32, "stats")
    for nm, t in (("y", y), ("gamma", gamma), ("beta", beta), ("cls", cls), ("pos", pos), ("x", x), ("tail", tail)):
        _chk(t, torch.float32, nm)
    D = y.shape[1]
    ntail = 0 if tail is None else tail.shape[0]
    assert y.is_contiguous() and x.is_contiguous() and pos.is_contiguous() and (tail is None or tail.is_contiguous())
    assert x.shape[0] == B * (n + ncls + ntail) and pos.shape[0] >= n + ncls
    with _Timed("embed_tokens", bytes=(y.numel() + x.numel()) * 4):
        rc = lib().b200vit_embed_tokens(_ptr(y), _ptr(gamma), _ptr(beta), _ptr(cls), _ptr(pos), _ptr(tail), _ptr(x),
                                        _ptr(xb), _ptr(stats), B, n, ncls, ntail, D, float(eps), _stream())
    _check(rc, "b200vit_embed_tokens")


def rowstats_cast(x: torch.Tensor, xb: torch.Tensor, stats: torch.Tensor) -> None:
    _chk(x, torch.float32, "x"); _chk(xb, torch.bfloat16, "xb"); _chk(stats, torch.float32, "stats")
    assert x.is_contiguous() and xb.is_contiguous() and stats.is_contiguous()
    M, D = x.shape
    with _Timed("rowstats_cast", bytes=M * D * 6):
        rc = lib().b200vit_rowstats_cast(_ptr(x), _ptr(xb), _ptr(stats), M, D, _stream())
    _check(rc, "b200vit_rowstats_cast")


def attention(qkv: torch.Tensor, out: torch.Tensor, B: int, N: int, H: int, dh: int, scale: float) -> None:
    _chk(qkv, torch.bfloat16, "qkv"); _chk(out, torch.bfloat16, "out")
    assert qkv.is_contiguous() and out.is_contiguous()
    assert qkv.shape == (B * N, 3 * H * dh) and out.shape == (B * N, H * dh)
    with _Timed("attention", B=B, N=N, H=H, bytes=(qkv.numel() + out.numel()) * 2, flops=4.0 * B * H * N * N * dh):
        rc = lib().b200vit_attention(_ptr(qkv), _ptr(out), B, N, H, dh, float(scale), _stream())
    _check(rc, "b200vit_attention")


def varlen_index(lengths, device) -> tuple:
    """(cu_seqlens, tile_prefix, total_tiles) device int32 tensors for b200vit_attention_varlen."""
    cu, tp = [0], [0]
    for n in lengths:
        cu.append(cu[-1] + int(n))
        tp.append(tp[-1] + (int(n) + 127) // 128)
    return (torch.tensor(cu, dtype=torch.int32, device=device), torch.tensor(tp, dtype=torch.int32, device=device),
            tp[-1])


def attention_varlen(qkv: torch.Tensor, out: torch.Tensor, cu_seqlens: torch.Tensor, tile_prefix: torch.Tensor,
                     total_tiles: int, H: int, dh: int, scale: float) -> None:
    _chk(qkv, torch.bfloat16, "qkv"); _chk(out, torch.bfloat16, "out")
    assert qkv.is_contiguous() and out.is_contiguous()
    assert cu_seqlens.dtype == torch.int32 and tile_prefix.dtype == torch.int32 and cu_seqlens.is_cuda
    T = qkv.shape[0]
    S = cu_seqlens.numel() - 1
    assert qkv.shape[1] == 3 * H * dh and out.shape == (T, H * dh) and tile_prefix.numel() == S + 1
    with _Timed("attention_varlen", bytes=(qkv.numel() + out.numel()) * 2):
        rc = lib().b200vit_attention_varlen(_ptr(qkv), _ptr(out), _ptr(cu_seqlens), _ptr(tile_prefix), S, T,
                                            int(total_tiles), H, dh, float(scale), _stream())
    _check(rc, "b200vit_attention_varlen")


class VarlenIndex:
    """Device-side index arrays of a packed batch of variable-size images, built on the host and moved with ONE
    host->device copy: cu_seqlens[S+1] (token offsets), tile_prefix[S+1] (128-row query tiles, attention_varlen),
    dims[S][2] = (H, W) pixels, row_prefix[S+1] (patch rows), img_ptrs[S] (int64 addresses)."""

    def __init__(self, images, p: int, device) -> None:
        S = len(images)
        cu, tp, rows, dims, ptrs = [0], [0], [0], [], []
        for im in images:
            hh, ww = int(im.shape[-2]), int(im.shape[-1])
            n = (hh // p) * (ww // p)
            cu.append(cu[-1] + n)
            tp.append(tp[-1] + (n + 127) // 128)
            rows.append(rows[-1] + hh // p)
            dims += [hh, ww]
            ptrs.append(im.data_ptr())
        n32 = 3 * (S + 1) + 2 * S
        host = torch.empty(S + (n32 + 1) // 2, dtype=torch.int64)
        host[:S] = torch.tensor(ptrs, dtype=torch.int64)
        host[S:].view(torch.int32)[:n32] = torch.tensor(cu + tp + rows + dims, dtype=torch.int32)
        dev = host.to(device)
        i32 = dev[S:].view(torch.int32)
        self.img_ptrs = dev[:S]
        self.cu = i32[:S + 1]
        self.tile_prefix = i32[S + 1:2 * (S + 1)]
        self.row_prefix = i32[2 * (S + 1):3 * (S + 1)]
        self.dims = i32[3 * (S + 1):3 * (S + 1) + 2 * S]
        self.S, self.T, self.total_tiles, self.total_rows = S, cu[-1], tp[-1], rows[-1]
        self.max_w = max(dims[1::2])
        self.max_gh, self.max_gw = max(dims[0::2]) // p, max(dims[1::2]) // p      # largest patch grid (pos tables)
        self.lengths = [cu[i + 1] - cu[i] for i in range(S)]


def patchify_varlen_ln(images, gamma: torch.Tensor, out_bf16: torch.Tensor, cu_seqlens: torch.Tensor, p: int,
                       eps: float = 1e-5, index: Optional[VarlenIndex] = None) -> None:
    """images: list of contiguous CUDA bf16 [C, H, W] tensors (kept alive by the caller until the stream has run)."""
    _chk(gamma, torch.float32, "gamma"); _chk(out_bf16, torch.bfloat16, "out")
    dev = out_bf16.device
    C = images[0].shape[0]
    for im in images:
        assert im.is_cuda and im.dtype == torch.bfloat16 and im.is_contiguous() and im.shape[0] == C
    ix = index if index is not None else VarlenIndex(images, p, dev)
    with _Timed("patchify_varlen_ln", bytes=out_bf16.numel() * 4):
        rc = lib().b200vit_patchify_varlen_ln(_ptr(ix.img_ptrs), _ptr(ix.dims), _ptr(cu_seqlens), _ptr(ix.row_prefix),
                                              _ptr(gamma), _ptr(out_bf16), out_bf16.stride(0), len(images),
                                              ix.total_rows, ix.max_w, C, p, float(eps), _stream())
    _check(rc, "b200vit_patchify_varlen_ln")


def embed_varlen(y: torch.Tensor, gamma: torch.Tensor, pos_h: torch.Tensor, pos_w: torch.Tensor, index: VarlenIndex,
                 x: torch.Tensor, p: int, xb: Optional[torch.Tensor] = None, stats: Optional[torch.Tensor] = None,
                 eps: float = 1e-5) -> None:
    for nm, t in (("y", y), ("gamma", gamma), ("pos_h", pos_h), ("pos_w", pos_w), ("x", x), ("stats", stats)):
        _chk(t, torch.float32, nm)
    _chk(xb, torch.bfloat16, "xb")
    T, D = y.shape
    assert y.is_contiguous() and x.is_contiguous() and pos_h.is_contiguous() and pos_w.is_contiguous()
    assert T == index.T and x.shape == y.shape and pos_h.shape[1] == D and pos_w.shape[1] == D
    if index.max_gh > pos_h.shape[0] or index.max_gw > pos_w.shape[0]:
        raise IndexError(f"an image of {index.max_gh} x {index.max_gw} patches exceeds the positional tables "
                         f"({pos_h.shape[0]} x {pos_w.shape[0]})")
    assert xb is None or (xb.is_contiguous() and xb.shape == y.shape)
    assert stats is None or (stats.is_contiguous() and stats.numel() == 2 * T)
    with _Timed("embed_varlen", bytes=y.numel() * 10):
        rc = lib().b200vit_embed_varlen(_ptr(y), _ptr(gamma), _ptr(pos_h), _ptr(pos_w), pos_h.shape[0],
                                        pos_w.shape[0], _ptr(index.cu), _ptr(index.dims), _ptr(x), _ptr(xb),
                                        _ptr(stats), T, D, index.S, p, float(eps), _stream())
    _check(rc, "b200vit_embed_varlen")


def rmsnorm_heads(buf: torch.Tensor, gamma: torch.Tensor, nheads: int, dh: int) -> None:
    """In place on the first nheads*dh columns of every row of buf[T, ld]."""
    _chk(buf, torch.bfloat16, "buf"); _chk(gamma, torch.float32, "gamma")
    assert buf.dim() == 2 and buf.stride(1) == 1 and gamma.is_contiguous() and gamma.numel() == nheads * dh
    assert buf.shape[1] >= nheads * dh
    T = buf.shape[0]
    with _Timed("rmsnorm_heads", bytes=T * nheads * dh * 4):
        rc = lib().b200vit_rmsnorm_heads(_ptr(buf), buf.stride(0), _ptr(gamma), T, nheads, dh, _stream())
    _check(rc, "b200vit_rmsnorm_heads")


def qk_rmsnorm(qkv: torch.Tensor, gamma_qk: torch.Tensor, H: int, dh: int) -> None:
    _chk(qkv, torch.bfloat16, "qkv"); _chk(gamma_qk, torch.float32, "gamma_qk")
    assert qkv.is_contiguous() and gamma_qk.is_contiguous() and gamma_qk.numel() == 2 * H * dh
    T = qkv.shape[0]
    assert qkv.shape[1] == 3 * H * dh
    with _Timed("qk_rmsnorm", bytes=T * 2 * H * dh * 4):
        rc = lib().b200vit_qk_rmsnorm(_ptr(qkv), _ptr(gamma_qk), T, H, dh, _stream())
    _check(rc, "b200vit_qk_rmsnorm")


def attn_pool(kv: torch.Tensor, qn: torch.Tensor, cu_seqlens: torch.Tensor, out: torch.Tensor, H: int, dh: int) -> None:
    _chk(kv, torch.bfloat16, "kv"); _chk(qn, torch.float32, "qn"); _chk(out, torch.bfloat16, "out")
    assert kv.is_contiguous() and qn.is_contiguous() and out.is_contiguous() and cu_seqlens.dtype == torch.int32
    S = cu_seqlens.numel() - 1
    assert kv.shape[1] == 2 * H * dh and out.shape == (S, H * dh) and qn.numel() == H * dh
    with _Timed("attn_pool", bytes=kv.numel() * 2):
        rc = lib().b200vit_attn_pool(_ptr(kv), _ptr(qn), _ptr(cu_seqlens), _ptr(out), S, H, dh, _stream())
    _check(rc, "b200vit_attn_pool")


def mean_pool(x: torch.Tensor, out: torch.Tensor, B: int, N: int, D: int, n_pool: Optional[int] = None) -> None:
    """out[b] = mean of the first n_pool (default: all N) token rows of image b."""
    _chk(x, torch.float32, "x"); _chk(out, torch.float32, "out")
    assert x.is_contiguous() and out.is_contiguous()
    with _Timed("mean_pool", bytes=x.numel() * 4):
        rc = lib().b200vit_mean_pool(_ptr(x), _ptr(out), B, N, D, N if n_pool is None else int(n_pool), _stream())
    _check(rc, "b200vit_mean_pool")


def cast_f32_bf16(x: torch.Tensor, out: torch.Tensor) -> None:
    _chk(x, torch.float32, "x"); _chk(out, torch.bfloat16, "out")
    assert x.is_contiguous() and out.is_contiguous() and x.numel() == out.numel()
    with _Timed("cast", bytes=x.numel() * 6):
        rc = lib().b200vit_cast_f32_bf16(_ptr(x), _ptr(out), x.numel(), _stream())
    _check(rc, "b200vit_cast_f32_bf16")
