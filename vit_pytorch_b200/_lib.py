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
EPI_HARDSWISH = 32
EPI_HEADLN = 64
EPI_SILU = 128
EPI_SIGMOID = 256
ATTN_MASK_SELF = 1
ATTN_GELU_OUT = 4
ATTN_POSBIAS_MAX_KEYS = 4096    # B200VIT_ATTN_POSBIAS_MAX_KEYS
MBCONV_PART_ROWS = 64           # B200VIT_MBCONV_PART_ROWS
ATTN_GROUPS_MAX_TOKENS = 4096   # B200VIT_ATTN_GROUPS_MAX_TOKENS
ATTN_WIDE_MAX_TOKENS = 1024     # B200VIT_ATTN_WIDE_MAX_TOKENS
ATTN_WIDE_MAX_WIDTH = 4096      # B200VIT_ATTN_WIDE_MAX_WIDTH
ATS_MAX_TOKENS = 4096           # B200VIT_ATS_MAX_TOKENS
ATS_MAX_HEAD_TOKENS = 16384     # B200VIT_ATS_MAX_HEAD_TOKENS

# every symbol include/b200vit.h declares (tests check that the library exports each of them)
SYMBOLS = [
    "b200vit_last_error", "b200vit_version", "b200vit_launch_count", "b200vit_reset_launch_count",
    "b200vit_device_ok", "b200vit_gemm_bf16", "b200vit_layernorm", "b200vit_patchify_ln", "b200vit_embed_tokens",
    "b200vit_attention", "b200vit_mean_pool", "b200vit_cast_f32_bf16", "b200vit_rowstats_cast", "b200vit_debug_set",
    "b200vit_stats_parts", "b200vit_attention_varlen", "b200vit_qk_rmsnorm", "b200vit_attn_pool",
    "b200vit_patchify_varlen_ln", "b200vit_rmsnorm_heads", "b200vit_embed_varlen",
    "b200vit_gemm_headnorm_bf16", "b200vit_layernorm_heads", "b200vit_patch_stats", "b200vit_patch_embed_tma",
    "b200vit_encoder_blocks", "b200vit_patchify_nd", "b200vit_rope_qk", "b200vit_encoder_blocks_rope",
    "b200vit_attention_axial", "b200vit_embed_tokens_grouped", "b200vit_patchify_spt_ln", "b200vit_attention_ex",
    "b200vit_attention_varlen_ex", "b200vit_encoder_blocks_ex", "b200vit_attention_cls",
    "b200vit_attention_headmix", "b200vit_attention_headmix_ex", "b200vit_attention_cls_headmix",
    "b200vit_attention_xca", "b200vit_local_patch_interaction", "b200vit_unfold_patches", "b200vit_pit_pool",
    "b200vit_conv_im2col_nchw", "b200vit_conv_im2col_nhwc", "b200vit_relu_maxpool", "b200vit_seq_pool",
    "b200vit_attention_window", "b200vit_attention_kv", "b200vit_merge_patches_ln", "b200vit_peg",
    "b200vit_attention_posbias", "b200vit_attention_window_relpos", "b200vit_mbconv_dwconv", "b200vit_se_pool",
    "b200vit_se_scale", "b200vit_conv_proj_dw", "b200vit_cross_embed_nchw", "b200vit_mbconv_dwconv_ex",
    "b200vit_attention_groups", "b200vit_conv_im2col_nhwc_ex", "b200vit_attention_window_token",
    "b200vit_window_mix", "b200vit_head_layernorm_gelu", "b200vit_attention_region_local",
    "b200vit_nest_level_entry", "b200vit_nest_im2col", "b200vit_attention_kv_ex", "b200vit_attention_iwsa",
    "b200vit_t2t_unfold_image", "b200vit_t2t_unfold_tokens", "b200vit_attention_wide",
    "b200vit_attention_wide_workspace", "b200vit_ats_select", "b200vit_ats_gather", "b200vit_attention_kv_lens",
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
    L.b200vit_attention_cls.restype = i32
    L.b200vit_attention_cls.argtypes = [vp, vp, i64, i64, i32, i32, vp, i64, i32, i32, i32, f32, vp]
    L.b200vit_attention_headmix.restype = i32
    L.b200vit_attention_headmix.argtypes = [vp, vp, i32, i32, i32, i32, f32, vp, vp, vp, f32, vp]
    L.b200vit_attention_headmix_ex.restype = i32
    L.b200vit_attention_headmix_ex.argtypes = [vp, vp, i32, i32, i32, i32, f32, vp, vp, vp, vp, f32, vp]
    L.b200vit_attention_cls_headmix.restype = i32
    L.b200vit_attention_cls_headmix.argtypes = [vp, vp, i64, i64, i32, i32, vp, i64, i32, i32, i32, f32, vp, vp, vp]
    L.b200vit_attention_xca.restype = i32
    L.b200vit_attention_xca.argtypes = [vp, vp, vp, i32, i32, i32, i32, vp]
    L.b200vit_local_patch_interaction.restype = i32
    L.b200vit_local_patch_interaction.argtypes = [vp, vp, vp, vp, vp, vp, vp, f32, vp, vp, vp, vp, i32, i32, i32, i32,
                                                  i32, vp]
    L.b200vit_unfold_patches.restype = i32
    L.b200vit_unfold_patches.argtypes = [vp, vp, i64, i32, i32, i32, i32, i32, i32, vp]
    L.b200vit_pit_pool.restype = i32
    L.b200vit_pit_pool.argtypes = [vp, i64, i32, i32, i32, i32, vp, vp, vp, i64, vp, i64, vp]
    L.b200vit_conv_im2col_nchw.restype = i32
    L.b200vit_conv_im2col_nchw.argtypes = [vp, vp, i64, i32, i32, i32, i32, i32, i32, i32, vp]
    L.b200vit_conv_im2col_nhwc.restype = i32
    L.b200vit_conv_im2col_nhwc.argtypes = [vp, i64, vp, i64, i32, i32, i32, i32, i32, i32, i32, vp]
    L.b200vit_conv_im2col_nhwc_ex.restype = i32
    L.b200vit_conv_im2col_nhwc_ex.argtypes = [vp, i64, i64, vp, i64, i32, i32, i32, i32, i32, i32, i32, vp]
    L.b200vit_relu_maxpool.restype = i32
    L.b200vit_relu_maxpool.argtypes = [vp, i64, i32, i32, i32, i32, i32, i32, i32, vp, vp, i64, vp]
    L.b200vit_seq_pool.restype = i32
    L.b200vit_seq_pool.argtypes = [vp, i32, i32, i32, vp, vp, f32, vp, vp, vp, i64, vp]
    L.b200vit_attention_window.restype = i32
    L.b200vit_attention_window.argtypes = [vp, vp, i32, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_attention_kv.restype = i32
    L.b200vit_attention_kv.argtypes = [vp, i64, vp, i64, vp, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_attention_kv_ex.restype = i32
    L.b200vit_attention_kv_ex.argtypes = [vp, i64, vp, i64, vp, i32, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_attention_iwsa.restype = i32
    L.b200vit_attention_iwsa.argtypes = [vp, i64, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_merge_patches_ln.restype = i32
    L.b200vit_merge_patches_ln.argtypes = [vp, i64, vp, vp, vp, i64, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_peg.restype = i32
    L.b200vit_peg.argtypes = [vp, i64, vp, vp, vp, i32, i32, i32, i32, i32, vp]
    L.b200vit_attention_posbias.restype = i32
    L.b200vit_attention_posbias.argtypes = [vp, i64, vp, vp, i32, i32, i32, i32, i32, i32, f32, i32, vp]
    L.b200vit_attention_window_relpos.restype = i32
    L.b200vit_attention_window_relpos.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_mbconv_dwconv.restype = i32
    L.b200vit_mbconv_dwconv.argtypes = [vp, i64, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp]
    L.b200vit_mbconv_dwconv_ex.restype = i32
    L.b200vit_mbconv_dwconv_ex.argtypes = [vp, i64, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]
    L.b200vit_attention_groups.restype = i32
    L.b200vit_attention_groups.argtypes = [vp, vp, i32, i32, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_attention_window_token.restype = i32
    L.b200vit_attention_window_token.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_window_mix.restype = i32
    L.b200vit_window_mix.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_head_layernorm_gelu.restype = i32
    L.b200vit_head_layernorm_gelu.argtypes = [vp, i64, vp, vp, i32, i32, i32, f32, vp]
    L.b200vit_attention_region_local.restype = i32
    L.b200vit_attention_region_local.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_nest_level_entry.restype = i32
    L.b200vit_nest_level_entry.argtypes = [vp, i64, vp, vp, f32, vp, i32, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32,
                                           i32, vp]
    L.b200vit_nest_im2col.restype = i32
    L.b200vit_nest_im2col.argtypes = [vp, i64, vp, i64, i32, i32, i32, i32, i32, vp]
    L.b200vit_se_pool.restype = i32
    L.b200vit_se_pool.argtypes = [vp, vp, i32, i32, i32, f32, vp]
    L.b200vit_se_scale.restype = i32
    L.b200vit_se_scale.argtypes = [vp, vp, i32, i32, i32, vp]
    L.b200vit_conv_proj_dw.restype = i32
    L.b200vit_conv_proj_dw.argtypes = [vp, i64, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]
    L.b200vit_cross_embed_nchw.restype = i32
    L.b200vit_cross_embed_nchw.argtypes = [vp, vp, vp, vp, i64, i32, i32, i32, i32, i32, C.POINTER(i32),
                                           C.POINTER(i32), i32, vp]
    L.b200vit_mean_pool.restype = i32
    L.b200vit_mean_pool.argtypes = [vp, vp, i32, i32, i32, i32, vp]
    L.b200vit_cast_f32_bf16.restype = i32
    L.b200vit_cast_f32_bf16.argtypes = [vp, vp, i64, vp]
    L.b200vit_encoder_blocks.restype = i32
    L.b200vit_encoder_blocks.argtypes = [C.POINTER(Layer), i32, vp, C.POINTER(EncoderWs), i32, i32, i32, i32, i32, i32,
                                         f32, i32, vp, vp, i32, vp]
    L.b200vit_encoder_blocks_rope.restype = i32
    L.b200vit_encoder_blocks_rope.argtypes = [C.POINTER(Layer), i32, vp, C.POINTER(EncoderWs), i32, i32, i32, i32, i32,
                                              i32, f32, i32, vp, vp, i32, vp, i32, vp]
    L.b200vit_patchify_nd.restype = i32
    L.b200vit_patchify_nd.argtypes = [vp, vp, i64, i32, i32, i32, C.POINTER(i32), C.POINTER(i32), vp]
    L.b200vit_rope_qk.restype = i32
    L.b200vit_rope_qk.argtypes = [vp, vp, i32, i32, i32, i32, vp]
    L.b200vit_attention_axial.restype = i32
    L.b200vit_attention_axial.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, f32, i32, vp]
    L.b200vit_embed_tokens_grouped.restype = i32
    L.b200vit_embed_tokens_grouped.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, i32,
                                               i32, i32, vp]
    L.b200vit_patchify_spt_ln.restype = i32
    L.b200vit_patchify_spt_ln.argtypes = [vp, vp, vp, vp, i64, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_attention_ex.restype = i32
    L.b200vit_attention_ex.argtypes = [vp, vp, i32, i32, i32, i32, f32, i32, vp]
    L.b200vit_attention_varlen_ex.restype = i32
    L.b200vit_attention_varlen_ex.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, i32, vp]
    L.b200vit_encoder_blocks_ex.restype = i32
    L.b200vit_encoder_blocks_ex.argtypes = [C.POINTER(Layer), i32, vp, C.POINTER(EncoderWs), i32, i32, i32, i32, i32,
                                            i32, f32, i32, vp, vp, i32, vp, i32, C.POINTER(C.c_float), i32, vp]
    L.b200vit_t2t_unfold_image.restype = i32
    L.b200vit_t2t_unfold_image.argtypes = [vp, vp, vp, i64, i32, i32, i32, i32, i32, i32, i32, vp]
    L.b200vit_t2t_unfold_tokens.restype = i32
    L.b200vit_t2t_unfold_tokens.argtypes = [vp, i64, i32, i32, i32, vp, vp, i64, i32, i32, i32, vp]
    L.b200vit_attention_wide_workspace.restype = i64
    L.b200vit_attention_wide_workspace.argtypes = [i32, i32, i32]
    L.b200vit_attention_wide.restype = i32
    L.b200vit_attention_wide.argtypes = [vp, vp, vp, i64, i32, i32, i32, i32, f32, vp, i64, vp]
    L.b200vit_ats_select.restype = i32
    L.b200vit_ats_select.argtypes = [vp, i64, vp, vp, vp, i32, vp, vp, vp, i32, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_ats_gather.restype = i32
    L.b200vit_ats_gather.argtypes = [vp, i32, vp, i64, vp, i64, i32, vp, i64, vp, i64, i32, vp]
    L.b200vit_attention_kv_lens.restype = i32
    L.b200vit_attention_kv_lens.argtypes = [vp, i64, vp, i64, vp, i32, i32, i32, vp, i32, i32, f32, vp]
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
                   hidden: int, scale: float, primed: bool, varlen=None, rope=None, layer_scales=None,
                   attn_flags: int = 0) -> None:
    """All encoder layers in one library call (b200vit_encoder_blocks).  `layers`: ctypes array of Layer built from the
    prepared weights; `ws`: EncoderWs over the engine's workspace; `varlen`: (cu, tile_prefix, total_tiles) if N > 512;
    `rope`: (cs table, rows) of rope_qk, applied after every QKV GEMM (b200vit_encoder_blocks_rope);
    `layer_scales`: ctypes float array of `depth` softmax scales (None: `scale` for every layer) and `attn_flags`
    (ATTN_MASK_SELF) go to b200vit_encoder_blocks_ex."""
    _chk(x, torch.float32, "x")
    cu, tp, tiles = varlen if varlen is not None else (None, None, 0)
    if layer_scales is not None or attn_flags:
        cs, rows = rope if rope is not None else (None, 0)
        _chk(cs, torch.float32, "rope table")
        assert layer_scales is None or len(layer_scales) == depth
        rc = lib().b200vit_encoder_blocks_ex(layers, depth, _ptr(x), C.byref(ws), B, N, D, heads, dh, hidden,
                                             float(scale), 1 if primed else 0, _ptr(cu), _ptr(tp), int(tiles),
                                             _ptr(cs), int(rows), layer_scales, int(attn_flags), _stream())
        _check(rc, "b200vit_encoder_blocks_ex")
        return
    if rope is None:
        rc = lib().b200vit_encoder_blocks(layers, depth, _ptr(x), C.byref(ws), B, N, D, heads, dh, hidden,
                                          float(scale), 1 if primed else 0, _ptr(cu), _ptr(tp), int(tiles), _stream())
        _check(rc, "b200vit_encoder_blocks")
        return
    cs, rows = rope
    _chk(cs, torch.float32, "rope table")
    assert cs.is_contiguous()
    rc = lib().b200vit_encoder_blocks_rope(layers, depth, _ptr(x), C.byref(ws), B, N, D, heads, dh, hidden,
                                           float(scale), 1 if primed else 0, _ptr(cu), _ptr(tp), int(tiles), _ptr(cs),
                                           int(rows), _stream())
    _check(rc, "b200vit_encoder_blocks_rope")


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
    _gemm(a, w, out_bf16, out_f32, bias, resid, gelu, ln_sums, ln_eps, col_s, stats_out, n, k, 0)


def gemm_act(a: torch.Tensor, w: torch.Tensor, *, act: str, out_bf16: Optional[torch.Tensor] = None,
             out_f32: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None,
             ln_sums: Optional[torch.Tensor] = None, ln_eps: float = 1e-5, col_s: Optional[torch.Tensor] = None,
             stats_out: Optional[torch.Tensor] = None) -> None:
    """gemm with the activation `act` after the bias / LayerNorm fold: "gelu" (EPI_GELU) or "silu" (EPI_SILU:
    y / (1 + exp(-y)); MobileViT's convolutions and FeedForward), at any M, with the LN fold, fp32 / bf16 outputs and
    row statistics as gemm takes them (no residual)."""
    if act not in ("gelu", "silu"):
        raise B200VitError(f"gemm_act: act={act!r} (gelu or silu)")
    _gemm(a, w, out_bf16, out_f32, bias, None, act == "gelu", ln_sums, ln_eps, col_s, stats_out, None, None,
          EPI_SILU if act == "silu" else 0)


def gemm_hardswish(a: torch.Tensor, w: torch.Tensor, *, out_bf16: torch.Tensor, bias: Optional[torch.Tensor] = None
                   ) -> None:
    """out_bf16 = hardswish(a @ w^T + bias) (EPI_HARDSWISH: y * clamp(y + 3, 0, 6) / 6; LeViT's FeedForward)."""
    _gemm(a, w, out_bf16, None, bias, None, False, None, 1e-5, None, None, None, None, EPI_HARDSWISH)


def gemm_silu(a: torch.Tensor, w: torch.Tensor, *, out_bf16: torch.Tensor, bias: Optional[torch.Tensor] = None
              ) -> None:
    """out_bf16 = silu(a @ w^T + bias) (EPI_SILU: y / (1 + exp(-y)); MaxViT's squeeze-excitation)."""
    _gemm(a, w, out_bf16, None, bias, None, False, None, 1e-5, None, None, None, None, EPI_SILU)


def gemm_sigmoid(a: torch.Tensor, w: torch.Tensor, *, out_bf16: torch.Tensor, bias: Optional[torch.Tensor] = None
                 ) -> None:
    """out_bf16 = sigmoid(a @ w^T + bias) (EPI_SIGMOID: 1 / (1 + exp(-y)); MaxViT's squeeze-excitation gate)."""
    _gemm(a, w, out_bf16, None, bias, None, False, None, 1e-5, None, None, None, None, EPI_SIGMOID)


def _gemm(a, w, out_bf16, out_f32, bias, resid, gelu, ln_sums, ln_eps, col_s, stats_out, n, k, extra_flags) -> None:
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
    flags = extra_flags
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


def patchify_spt_ln(img: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, out_bf16: torch.Tensor, p: int,
                    eps: float = 1e-5) -> None:
    """Shifted patch tokenization + LayerNorm(5*C*p*p): img [B, C, H, W] bf16 -> out [B*n, ldo] bf16 rows of the
    '(p1 p2 c)' patches of cat(img, its four one-pixel shifts) over 5C channels, zero K padding."""
    _chk(img, torch.bfloat16, "img"); _chk(out_bf16, torch.bfloat16, "out")
    _chk(gamma, torch.float32, "gamma"); _chk(beta, torch.float32, "beta")
    assert img.is_contiguous() and img.dim() == 4 and out_bf16.dim() == 2 and out_bf16.stride(1) == 1
    B, Cc, H, W = img.shape
    with _Timed("patchify_spt_ln", bytes=img.numel() * 2 + out_bf16.numel() * 2):
        rc = lib().b200vit_patchify_spt_ln(_ptr(img), _ptr(gamma), _ptr(beta), _ptr(out_bf16), out_bf16.stride(0), B,
                                           Cc, H, W, int(p), float(eps), _stream())
    _check(rc, "b200vit_patchify_spt_ln")


def patchify_nd(img: torch.Tensor, out_bf16: torch.Tensor, patch) -> None:
    """img [B, C, S_0 .. S_{r-1}] bf16 -> out [B*n, ldo] with the (p0 .. p_{r-1} c) patch rows, zero K padding."""
    _chk(img, torch.bfloat16, "img"); _chk(out_bf16, torch.bfloat16, "out")
    assert img.is_contiguous() and out_bf16.dim() == 2 and out_bf16.stride(1) == 1
    B, Cc, *shape = img.shape
    r = len(shape)
    shp, pat = (C.c_int * max(r, 1))(*shape), (C.c_int * max(r, 1))(*patch)
    with _Timed("patchify_nd", bytes=img.numel() * 2 + out_bf16.shape[0] * out_bf16.stride(0) * 2):
        rc = lib().b200vit_patchify_nd(_ptr(img), _ptr(out_bf16), out_bf16.stride(0), B, Cc, r, shp, pat, _stream())
    _check(rc, "b200vit_patchify_nd")


def rope_qk(qkv: torch.Tensor, cs: torch.Tensor, rows: int, H: int, dh: int) -> None:
    """Rotate the q and k slices of qkv[T, 3*H*dh] in place with the (cos, sin) table cs[rows, H, dh/2, 2]; token t
    uses table row t % rows."""
    _chk(qkv, torch.bfloat16, "qkv"); _chk(cs, torch.float32, "cs")
    assert qkv.is_contiguous() and cs.is_contiguous() and cs.numel() == rows * H * dh
    T = qkv.shape[0]
    assert qkv.shape[1] == 3 * H * dh
    # q and k read and written once (bf16) + the table (fp32)
    with _Timed("rope_qk", bytes=T * 2 * H * dh * 4 + cs.numel() * 4):
        rc = lib().b200vit_rope_qk(_ptr(qkv), _ptr(cs), int(rows), T, H, dh, _stream())
    _check(rc, "b200vit_rope_qk")


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
                 pos: Optional[torch.Tensor], x: torch.Tensor, B: int, n: int, ncls: int, eps: float = 1e-5,
                 xb: Optional[torch.Tensor] = None, stats: Optional[torch.Tensor] = None,
                 tail: Optional[torch.Tensor] = None) -> None:
    """tail [ntail, D]: rows appended after the n patch tokens of every image (register tokens, no pos).
    pos None: no positional term.  gamma None: no LayerNorm (beta ignored)."""
    _chk(xb, torch.bfloat16, "xb"); _chk(stats, torch.float32, "stats")
    for nm, t in (("y", y), ("gamma", gamma), ("beta", beta), ("cls", cls), ("pos", pos), ("x", x), ("tail", tail)):
        _chk(t, torch.float32, nm)
    D = y.shape[1]
    ntail = 0 if tail is None else tail.shape[0]
    assert y.is_contiguous() and x.is_contiguous() and (tail is None or tail.is_contiguous())
    assert x.shape[0] == B * (n + ncls + ntail)
    assert pos is None or (pos.is_contiguous() and pos.shape[0] >= n + ncls)
    with _Timed("embed_tokens", bytes=(y.numel() + x.numel()) * 4):
        rc = lib().b200vit_embed_tokens(_ptr(y), _ptr(gamma), _ptr(beta), _ptr(cls), _ptr(pos), _ptr(tail), _ptr(x),
                                        _ptr(xb), _ptr(stats), B, n, ncls, ntail, D, float(eps), _stream())
    _check(rc, "b200vit_embed_tokens")


def embed_tokens_grouped(y: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, cls: Optional[torch.Tensor],
                         pos: Optional[torch.Tensor], x: torch.Tensor, groups: int, n: int, ncls: int, pos_period: int,
                         pos_stride: int, cls_pos: bool, eps: float = 1e-5, xb: Optional[torch.Tensor] = None,
                         stats: Optional[torch.Tensor] = None) -> None:
    """embed_tokens over `groups` token groups whose positions come from blocks of a larger table: group g reads the
    block at row (g % pos_period) * pos_stride; patch t reads row ncls + t of it (cls_pos) or row t, the cls rows then
    getting no position (ViViT's per-frame table, reference vivit.py:227-231)."""
    _chk(xb, torch.bfloat16, "xb"); _chk(stats, torch.float32, "stats")
    for nm, t in (("y", y), ("gamma", gamma), ("beta", beta), ("cls", cls), ("pos", pos), ("x", x)):
        _chk(t, torch.float32, nm)
    D = y.shape[1]
    assert y.is_contiguous() and x.is_contiguous() and y.shape[0] == groups * n and x.shape[0] == groups * (n + ncls)
    if pos is not None:
        last = (pos_period - 1) * pos_stride + n + (ncls if cls_pos else 0)
        assert pos.is_contiguous() and pos.shape[0] >= last, f"positional table of {pos.shape[0]} rows, {last} needed"
    with _Timed("embed_tokens", bytes=(y.numel() + x.numel()) * 4):
        rc = lib().b200vit_embed_tokens_grouped(_ptr(y), _ptr(gamma), _ptr(beta), _ptr(cls), _ptr(pos), None, _ptr(x),
                                                _ptr(xb), _ptr(stats), groups, n, ncls, 0, D, float(eps),
                                                int(pos_period), int(pos_stride), 1 if cls_pos else 0, _stream())
    _check(rc, "b200vit_embed_tokens_grouped")


def rowstats_cast(x: torch.Tensor, xb: torch.Tensor, stats: torch.Tensor) -> None:
    _chk(x, torch.float32, "x"); _chk(xb, torch.bfloat16, "xb"); _chk(stats, torch.float32, "stats")
    assert x.is_contiguous() and xb.is_contiguous() and stats.is_contiguous()
    M, D = x.shape
    with _Timed("rowstats_cast", bytes=M * D * 6):
        rc = lib().b200vit_rowstats_cast(_ptr(x), _ptr(xb), _ptr(stats), M, D, _stream())
    _check(rc, "b200vit_rowstats_cast")


def attention(qkv: torch.Tensor, out: torch.Tensor, B: int, N: int, H: int, dh: int, scale: float,
              mask_self: bool = False) -> None:
    """mask_self: each query's own key is excluded (b200vit_attention_ex with ATTN_MASK_SELF)."""
    _chk(qkv, torch.bfloat16, "qkv"); _chk(out, torch.bfloat16, "out")
    assert qkv.is_contiguous() and out.is_contiguous()
    assert qkv.shape == (B * N, 3 * H * dh) and out.shape == (B * N, H * dh)
    with _Timed("attention", B=B, N=N, H=H, bytes=(qkv.numel() + out.numel()) * 2, flops=4.0 * B * H * N * N * dh):
        if mask_self:
            rc = lib().b200vit_attention_ex(_ptr(qkv), _ptr(out), B, N, H, dh, float(scale), ATTN_MASK_SELF,
                                            _stream())
        else:
            rc = lib().b200vit_attention(_ptr(qkv), _ptr(out), B, N, H, dh, float(scale), _stream())
    _check(rc, "b200vit_attention")


def attention_axial(qkv: torch.Tensor, out: torch.Tensor, key_mask: Optional[torch.Tensor], B: int, L: int, G: int,
                    H: int, dh: int, scale: float, zero_masked_rows: bool) -> None:
    """Attention over the B*G sequences of L tokens of qkv[B*L*G, 3*H*dh], token j of sequence b*G + p at row
    b*L*G + j*G + p; key_mask: None or uint8 [B, L] (1 = keep), shared by the G sequences of b."""
    _chk(qkv, torch.bfloat16, "qkv"); _chk(out, torch.bfloat16, "out"); _chk(key_mask, torch.uint8, "key_mask")
    assert qkv.is_contiguous() and out.is_contiguous()
    assert qkv.shape == (B * L * G, 3 * H * dh) and out.shape == (B * L * G, H * dh)
    assert key_mask is None or (key_mask.is_contiguous() and key_mask.numel() == B * L)
    with _Timed("attention_axial", B=B, L=L, G=G, H=H, bytes=(qkv.numel() + out.numel()) * 2,
                flops=4.0 * B * G * H * L * L * dh):
        rc = lib().b200vit_attention_axial(_ptr(qkv), _ptr(out), _ptr(key_mask), B, L, G, H, dh, float(scale),
                                           1 if zero_masked_rows else 0, _stream())
    _check(rc, "b200vit_attention_axial")


def attention_window(qkv: torch.Tensor, out: torch.Tensor, B: int, gh: int, gw: int, p: int, H: int, dh: int,
                     scale: float) -> None:
    """Attention inside the p x p windows of B token maps of gh x gw tokens: qkv[B*gh*gw, 3*H*dh] packed q | k | v,
    token (b, y, x) at row (b*gh + y)*gw + x; out[B*gh*gw, H*dh]."""
    _chk(qkv, torch.bfloat16, "qkv"); _chk(out, torch.bfloat16, "out")
    assert qkv.is_contiguous() and out.is_contiguous()
    assert qkv.shape == (B * gh * gw, 3 * H * dh) and out.shape == (B * gh * gw, H * dh)
    with _Timed("attention_window", B=B, h=gh, w=gw, p=p, H=H, bytes=(qkv.numel() + out.numel()) * 2,
                flops=4.0 * B * gh * gw * H * p * p * dh):
        rc = lib().b200vit_attention_window(_ptr(qkv), _ptr(out), B, int(gh), int(gw), int(p), H, dh, float(scale),
                                            _stream())
    _check(rc, "b200vit_attention_window")


def attention_kv(q: torch.Tensor, kv: torch.Tensor, out: torch.Tensor, B: int, Nq: int, Nk: int, H: int, dh: int,
                 scale: float) -> None:
    """out[B*Nq, H*dh] = softmax(scale q k^T) v per image and head: q[B*Nq, H*dh] (any row stride), kv[B*Nk, 2*H*dh]
    packed k | v (any row stride), Nq and Nk independent."""
    _chk(q, torch.bfloat16, "q"); _chk(kv, torch.bfloat16, "kv"); _chk(out, torch.bfloat16, "out")
    assert q.dim() == 2 and q.stride(1) == 1 and kv.dim() == 2 and kv.stride(1) == 1 and out.is_contiguous()
    assert q.shape == (B * Nq, H * dh) and kv.shape == (B * Nk, 2 * H * dh) and out.shape == (B * Nq, H * dh)
    with _Timed("attention_kv", B=B, Nq=Nq, Nk=Nk, H=H, bytes=(q.numel() + kv.numel() + out.numel()) * 2,
                flops=4.0 * B * H * Nq * Nk * dh):
        rc = lib().b200vit_attention_kv(_ptr(q), q.stride(0), _ptr(kv), kv.stride(0), _ptr(out), B, int(Nq), int(Nk),
                                        H, dh, float(scale), _stream())
    _check(rc, "b200vit_attention_kv")


def attention_kv_ex(q: torch.Tensor, kv: torch.Tensor, out: torch.Tensor, B: int, Nq: int, Nk: int, H: int, dk: int,
                    dv: int, scale: float) -> None:
    """attention_kv with key heads dk wide and value heads dv wide: q[B*Nq, H*dk] (any row stride), kv[B*Nk, H*dk + H*dv]
    packed k | v (any row stride), out[B*Nq, H*dv]."""
    _chk(q, torch.bfloat16, "q"); _chk(kv, torch.bfloat16, "kv"); _chk(out, torch.bfloat16, "out")
    assert q.dim() == 2 and q.stride(1) == 1 and kv.dim() == 2 and kv.stride(1) == 1 and out.is_contiguous()
    assert q.shape == (B * Nq, H * dk) and kv.shape == (B * Nk, H * (dk + dv)) and out.shape == (B * Nq, H * dv)
    with _Timed("attention_kv_ex", B=B, Nq=Nq, Nk=Nk, H=H, dk=dk, dv=dv,
                bytes=(q.numel() + kv.numel() + out.numel()) * 2, flops=2.0 * B * H * Nq * Nk * (dk + dv)):
        rc = lib().b200vit_attention_kv_ex(_ptr(q), q.stride(0), _ptr(kv), kv.stride(0), _ptr(out), B, int(Nq), int(Nk),
                                           H, dk, dv, float(scale), _stream())
    _check(rc, "b200vit_attention_kv_ex")


def attention_iwsa(qkv: torch.Tensor, lim: torch.Tensor, out: torch.Tensor, B: int, gh: int, gw: int, wh: int, ww: int,
                   H: int, dk: int, dv: int, scale: float) -> None:
    """ScalableViT's windowed attention plus the local interactive module over B gh x gw maps in map order:
    qkv[B*gh*gw, >= H*(2dk + dv)] q | k | v (any row stride), lim and out [B*gh*gw, H*dv]; per wh x ww window and head
    out = softmax(scale q k^T) v + lim, summed in fp32 and rounded once."""
    _chk(qkv, torch.bfloat16, "qkv"); _chk(lim, torch.bfloat16, "lim"); _chk(out, torch.bfloat16, "out")
    M = B * gh * gw
    assert qkv.dim() == 2 and qkv.stride(1) == 1 and qkv.shape[0] == M and qkv.shape[1] >= H * (2 * dk + dv)
    assert lim.is_contiguous() and out.is_contiguous() and lim.shape == out.shape == (M, H * dv)
    with _Timed("attention_iwsa", B=B, h=gh, w=gw, wh=wh, ww=ww, H=H, dk=dk, dv=dv,
                bytes=(M * H * (2 * dk + dv) + 2 * M * H * dv) * 2, flops=2.0 * M * H * wh * ww * (dk + dv)):
        rc = lib().b200vit_attention_iwsa(_ptr(qkv), qkv.stride(0), _ptr(lim), _ptr(out), B, int(gh), int(gw), int(wh),
                                          int(ww), H, dk, dv, float(scale), _stream())
    _check(rc, "b200vit_attention_iwsa")


def attention_posbias(qkv: torch.Tensor, out: torch.Tensor, table: torch.Tensor, B: int, F: int, s: int, H: int,
                      dk: int, dv: int, scale: float, gelu_out: bool = False) -> None:
    """LeViT attention over B F x F token maps: qkv[B*F*F, ld] packed q (H*dk) | k (H*dk) | v (H*dv), any row stride;
    queries the tokens (s*i, s*j); out[B*Fq*Fq, H*dv] (Fq = ceil(F / s)) = [GELU] softmax(scale q k^T + bias) v, the
    bias table[h][|dy|*F + |dx|] from table fp32 [H, F*F]."""
    _chk(qkv, torch.bfloat16, "qkv"); _chk(out, torch.bfloat16, "out"); _chk(table, torch.float32, "table")
    Fq = -(-F // s)
    assert qkv.dim() == 2 and qkv.stride(1) == 1 and out.is_contiguous() and table.is_contiguous()
    assert qkv.shape == (B * F * F, H * (2 * dk + dv)) and out.shape == (B * Fq * Fq, H * dv)
    assert table.shape == (H, F * F)
    with _Timed("attention_posbias", B=B, F=F, s=s, H=H, bytes=(qkv.numel() + out.numel()) * 2,
                flops=2.0 * B * H * Fq * Fq * F * F * (dk + dv)):
        rc = lib().b200vit_attention_posbias(_ptr(qkv), qkv.stride(0), _ptr(out), _ptr(table), B, int(F), int(s), H,
                                             int(dk), int(dv), float(scale), ATTN_GELU_OUT if gelu_out else 0,
                                             _stream())
    _check(rc, "b200vit_attention_posbias")


def attention_window_relpos(qkv: torch.Tensor, out: torch.Tensor, table: torch.Tensor, B: int, gh: int, gw: int,
                            w: int, grid: bool, H: int, dh: int, scale: float) -> None:
    """MaxViT attention inside the w x w windows of B token maps of gh x gw tokens with a relative-position bias:
    qkv[B*gh*gw, 3*H*dh] packed q | k | v, token (b, y, x) at row (b*gh + y)*gw + x; out[B*gh*gw, H*dh].  grid False:
    window (i, j) is the block of map positions (i*w + u, j*w + v); True: the dilated grid (u*gh/w + i, v*gw/w + j).
    table fp32 [H, (2w-1)^2] = rel_pos_bias.weight^T, indexed by the local offset (du + w-1)*(2w-1) + dv + w-1."""
    _chk(qkv, torch.bfloat16, "qkv"); _chk(out, torch.bfloat16, "out"); _chk(table, torch.float32, "table")
    assert qkv.is_contiguous() and out.is_contiguous() and table.is_contiguous()
    assert qkv.shape == (B * gh * gw, 3 * H * dh) and out.shape == (B * gh * gw, H * dh)
    assert table.shape == (H, (2 * w - 1) ** 2)
    with _Timed("attention_window_relpos", B=B, h=gh, w=gw, window=w, grid=bool(grid), H=H,
                bytes=(qkv.numel() + out.numel()) * 2, flops=4.0 * B * gh * gw * H * w * w * dh):
        rc = lib().b200vit_attention_window_relpos(_ptr(qkv), _ptr(out), _ptr(table), B, int(gh), int(gw), int(w),
                                                   1 if grid else 0, H, dh, float(scale), _stream())
    _check(rc, "b200vit_attention_window_relpos")


def mbconv_parts(oh: int, ow: int) -> int:
    """Partial sums per image that mbconv_dwconv writes for an oh x ow output map."""
    return -(-(oh * ow) // MBCONV_PART_ROWS)


def mbconv_dwconv(x: torch.Tensor, w9: torch.Tensor, bias: torch.Tensor, y: torch.Tensor, part: torch.Tensor, B: int,
                  h: int, w: int, stride: int) -> None:
    """y = GELU(depthwise 3 x 3 convolution of x, zero padding 1, stride 1 or 2, + bias): x bf16 [B*h*w, C]
    channels-last, y bf16 [B*ceil(h/s)*ceil(w/s), C], w9 fp32 [9, C] tap-major and bias fp32 [C] with the BatchNorm
    folded in; part fp32 [B, mbconv_parts(oh, ow), C] gets the per-image channel sums of the rounded y, part by part."""
    _chk(x, torch.bfloat16, "x"); _chk(y, torch.bfloat16, "y")
    for nm, t in (("w9", w9), ("bias", bias), ("part", part)):
        _chk(t, torch.float32, nm)
    M, Cc = x.shape
    oh, ow = -(-h // stride), -(-w // stride)
    assert x.is_contiguous() and y.is_contiguous() and w9.is_contiguous() and bias.is_contiguous()
    assert y.shape == (B * oh * ow, Cc) and w9.shape == (9, Cc) and bias.numel() == Cc
    assert part.is_contiguous() and part.shape == (B, mbconv_parts(oh, ow), Cc)
    with _Timed("mbconv_dwconv", B=B, h=h, w=w, C=Cc, s=stride, bytes=(M + y.shape[0]) * Cc * 2):
        rc = lib().b200vit_mbconv_dwconv(_ptr(x), M, _ptr(w9), _ptr(bias), _ptr(y), _ptr(part), B, int(h), int(w), Cc,
                                         int(stride), _stream())
    _check(rc, "b200vit_mbconv_dwconv")


def mbconv_dwconv_ex(x: torch.Tensor, w9: torch.Tensor, bias: torch.Tensor, y: torch.Tensor,
                     part: Optional[torch.Tensor], B: int, h: int, w: int, stride: int, act: str = "gelu") -> None:
    """mbconv_dwconv with the activation `act` ("gelu" or "silu": y / (1 + exp(-y)), as the GEMM's EPI_SILU) and
    `part` optional (None: no channel sums; MobileViT's MV2Block, mobile_vit.py:108-127)."""
    _chk(x, torch.bfloat16, "x"); _chk(y, torch.bfloat16, "y")
    for nm, t in (("w9", w9), ("bias", bias), ("part", part)):
        _chk(t, torch.float32, nm)
    if act not in ("gelu", "silu"):
        raise B200VitError(f"mbconv_dwconv_ex: act={act!r} (gelu or silu)")
    M, Cc = x.shape
    oh, ow = -(-h // stride), -(-w // stride)
    assert x.is_contiguous() and y.is_contiguous() and w9.is_contiguous() and bias.is_contiguous()
    assert y.shape == (B * oh * ow, Cc) and w9.shape == (9, Cc) and bias.numel() == Cc
    assert part is None or (part.is_contiguous() and part.shape == (B, mbconv_parts(oh, ow), Cc))
    with _Timed("mbconv_dwconv", B=B, h=h, w=w, C=Cc, s=stride, act=act, bytes=(M + y.shape[0]) * Cc * 2):
        rc = lib().b200vit_mbconv_dwconv_ex(_ptr(x), M, _ptr(w9), _ptr(bias), _ptr(y), _ptr(part), B, int(h), int(w),
                                            Cc, int(stride), EPI_GELU if act == "gelu" else EPI_SILU, _stream())
    _check(rc, "b200vit_mbconv_dwconv_ex")


def attention_groups(qkv: torch.Tensor, out: torch.Tensor, B: int, gh: int, gw: int, ph: int, pw: int, H: int,
                     dh: int, scale: float) -> None:
    """MobileViT attention inside the strided patch groups of B token maps of gh x gw tokens: qkv[B*gh*gw, 3*H*dh]
    packed q | k | v, token (b, y, x) at row (b*gh + y)*gw + x; out[B*gh*gw, H*dh].  Group (b, i, j) is the tokens
    (y'*ph + i, x'*pw + j) (mobile_vit.py:150); dh = 8."""
    _chk(qkv, torch.bfloat16, "qkv"); _chk(out, torch.bfloat16, "out")
    assert qkv.is_contiguous() and out.is_contiguous()
    assert qkv.shape == (B * gh * gw, 3 * H * dh) and out.shape == (B * gh * gw, H * dh)
    n = (gh // ph) * (gw // pw) if ph > 0 and pw > 0 else 0
    with _Timed("attention_groups", B=B, h=gh, w=gw, ph=ph, pw=pw, H=H, n=n, bytes=(qkv.numel() + out.numel()) * 2,
                exps=B * ph * pw * H * n * n, flops=4.0 * B * ph * pw * H * n * n * dh):
        rc = lib().b200vit_attention_groups(_ptr(qkv), _ptr(out), B, int(gh), int(gw), int(ph), int(pw), H, dh,
                                            float(scale), _stream())
    _check(rc, "b200vit_attention_groups")


def attention_window_token(qkv: torch.Tensor, tok_qkv: torch.Tensor, out: torch.Tensor,
                           tok_out: Optional[torch.Tensor], B: int, gh: int, gw: int, p: int, H: int, dh: int,
                           scale: float) -> None:
    """SepViT attention inside the p x p windows of B token maps of gh x gw tokens, each window with one more token
    whose q | k | v is tok_qkv[3*H*dh] (the same for every window): qkv[B*gh*gw, 3*H*dh] packed q | k | v, token
    (b, y, x) at row (b*gh + y)*gw + x; out[B*gh*gw, H*dh]; tok_out None or [B*nw, H*dh], the window token's output
    of window (b, wy, wx) at row (b*gh/p + wy)*gw/p + wx (sep_vit.py:139-172)."""
    _chk(qkv, torch.bfloat16, "qkv"); _chk(tok_qkv, torch.bfloat16, "tok_qkv"); _chk(out, torch.bfloat16, "out")
    _chk(tok_out, torch.bfloat16, "tok_out")
    I = H * dh
    assert qkv.is_contiguous() and out.is_contiguous() and tok_qkv.is_contiguous() and tok_qkv.numel() == 3 * I
    assert qkv.shape == (B * gh * gw, 3 * I) and out.shape == (B * gh * gw, I)
    nw = (gh // p) * (gw // p) if p > 0 else 0
    assert tok_out is None or (tok_out.is_contiguous() and tok_out.shape == (B * nw, I))
    n = p * p + 1
    with _Timed("attention_window_token", B=B, h=gh, w=gw, p=p, H=H,
                bytes=(qkv.numel() + out.numel() + (0 if tok_out is None else tok_out.numel())) * 2,
                flops=4.0 * B * nw * H * n * n * dh):
        rc = lib().b200vit_attention_window_token(_ptr(qkv), _ptr(tok_qkv), _ptr(out), _ptr(tok_out), B, int(gh),
                                                  int(gw), int(p), H, dh, float(scale), _stream())
    _check(rc, "b200vit_attention_window_token")


def attention_region_local(qkv: torch.Tensor, out: torch.Tensor, table: torch.Tensor, B: int, lh: int, lw: int,
                           rh: int, rw: int, W: int, H: int, dh: int, scale: float) -> None:
    """RegionViT's region-to-local attention (regionvit.py:167-176): qkv[B*lh*lw + B*rh*rw, 3*H*dh] packed q | k | v,
    the local tokens (b, y, x) at rows (b*lh + y)*lw + x, then the region tokens (b, i, j) at rows
    B*lh*lw + (b*rh + i)*rw + j; window (b, i, j) is that region token and the (lh/rh) x (lw/rw) local tokens of its
    cell, attending together under table[H, (2W-1)^2] (the transposed local_rel_pos_bias weight) between local tokens;
    out [same rows, H*dh]."""
    _chk(qkv, torch.bfloat16, "qkv"); _chk(out, torch.bfloat16, "out"); _chk(table, torch.float32, "table")
    I = H * dh
    rows = B * (lh * lw + rh * rw)
    assert qkv.is_contiguous() and out.is_contiguous() and table.is_contiguous()
    assert qkv.shape == (rows, 3 * I) and out.shape == (rows, I) and table.shape == (H, (2 * W - 1) ** 2)
    n = (lh // rh) * (lw // rw) + 1 if rh > 0 and rw > 0 else 0
    with _Timed("attention_region_local", B=B, lh=lh, lw=lw, rh=rh, rw=rw, H=H, n=n,
                bytes=(qkv.numel() + out.numel()) * 2 + table.numel() * 4,
                flops=4.0 * B * rh * rw * H * n * n * dh):
        rc = lib().b200vit_attention_region_local(_ptr(qkv), _ptr(out), _ptr(table), B, int(lh), int(lw), int(rh),
                                                  int(rw), int(W), H, dh, float(scale), _stream())
    _check(rc, "b200vit_attention_region_local")


def window_mix(wqk: torch.Tensor, o: torch.Tensor, out: torch.Tensor, B: int, gh: int, gw: int, p: int, H: int,
               dh: int, scale: float) -> None:
    """SepViT attention across the nw windows of each map (sep_vit.py:182-205): per image and head P =
    softmax(scale wq wk^T) over the windows, wqk[B*nw, 2*H*dh] with head h's query at columns [2h dh, 2h dh + dh) and
    its key right after; out[(window i, position w)] = sum_j P_ij o[(window j, position w)], o and out [B*gh*gw, H*dh]
    in the map's row order, out of place."""
    _chk(wqk, torch.bfloat16, "wqk"); _chk(o, torch.bfloat16, "o"); _chk(out, torch.bfloat16, "out")
    I = H * dh
    nw = (gh // p) * (gw // p) if p > 0 else 0
    assert wqk.is_contiguous() and o.is_contiguous() and out.is_contiguous()
    assert wqk.shape == (B * nw, 2 * I) and o.shape == (B * gh * gw, I) and out.shape == (B * gh * gw, I)
    with _Timed("window_mix", B=B, h=gh, w=gw, p=p, H=H, nw=nw, bytes=(wqk.numel() + o.numel() + out.numel()) * 2,
                flops=2.0 * B * H * nw * nw * (dh + p * p * dh)):
        rc = lib().b200vit_window_mix(_ptr(wqk), _ptr(o), _ptr(out), B, int(gh), int(gw), int(p), H, dh, float(scale),
                                      _stream())
    _check(rc, "b200vit_window_mix")


def head_layernorm_gelu(buf: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, nheads: int, dh: int,
                        eps: float = 1e-5) -> None:
    """In place on buf[T, >= nheads*dh] bf16: every dh-wide head from column 0 <- GELU_erf(LayerNorm(head) gamma +
    beta), gamma and beta fp32 [dh] shared by the heads (SepViT's window_tokens_to_qk, sep_vit.py:96-98)."""
    _chk(buf, torch.bfloat16, "buf"); _chk(gamma, torch.float32, "gamma"); _chk(beta, torch.float32, "beta")
    assert buf.dim() == 2 and buf.stride(1) == 1 and gamma.is_contiguous() and beta.is_contiguous()
    assert gamma.numel() == dh and beta.numel() == dh
    T = buf.shape[0]
    with _Timed("head_layernorm_gelu", T=T, H=nheads, bytes=T * nheads * dh * 4):
        rc = lib().b200vit_head_layernorm_gelu(_ptr(buf), buf.stride(0), _ptr(gamma), _ptr(beta), T, int(nheads),
                                               int(dh), float(eps), _stream())
    _check(rc, "b200vit_head_layernorm_gelu")


def se_pool(part: torch.Tensor, pooled: torch.Tensor, n: int) -> None:
    """pooled bf16 [B, C] = the sum over the parts of part fp32 [B, P, C], in part order, divided by n."""
    _chk(part, torch.float32, "part"); _chk(pooled, torch.bfloat16, "pooled")
    B, P, Cc = part.shape
    assert part.is_contiguous() and pooled.is_contiguous() and pooled.shape == (B, Cc)
    with _Timed("se_pool", B=B, C=Cc, bytes=part.numel() * 4):
        rc = lib().b200vit_se_pool(_ptr(part), _ptr(pooled), B, P, Cc, 1.0 / n, _stream())
    _check(rc, "b200vit_se_pool")


def se_scale(h: torch.Tensor, gate: torch.Tensor, B: int, n: int) -> None:
    """In place h[b*n + t, c] *= gate[b, c], rounded to bf16: h bf16 [B*n, C], gate bf16 [B, C]."""
    _chk(h, torch.bfloat16, "h"); _chk(gate, torch.bfloat16, "gate")
    assert h.is_contiguous() and gate.is_contiguous() and h.shape[0] == B * n and gate.shape == (B, h.shape[1])
    with _Timed("se_scale", B=B, n=n, C=h.shape[1], bytes=h.numel() * 4):
        rc = lib().b200vit_se_scale(_ptr(h), _ptr(gate), B, int(n), h.shape[1], _stream())
    _check(rc, "b200vit_se_scale")


def varlen_index(lengths, device) -> tuple:
    """(cu_seqlens, tile_prefix, total_tiles) device int32 tensors for b200vit_attention_varlen."""
    cu, tp = [0], [0]
    for n in lengths:
        cu.append(cu[-1] + int(n))
        tp.append(tp[-1] + (int(n) + 127) // 128)
    return (torch.tensor(cu, dtype=torch.int32, device=device), torch.tensor(tp, dtype=torch.int32, device=device),
            tp[-1])


def attention_varlen(qkv: torch.Tensor, out: torch.Tensor, cu_seqlens: torch.Tensor, tile_prefix: torch.Tensor,
                     total_tiles: int, H: int, dh: int, scale: float, mask_self: bool = False) -> None:
    _chk(qkv, torch.bfloat16, "qkv"); _chk(out, torch.bfloat16, "out")
    assert qkv.is_contiguous() and out.is_contiguous()
    assert cu_seqlens.dtype == torch.int32 and tile_prefix.dtype == torch.int32 and cu_seqlens.is_cuda
    T = qkv.shape[0]
    S = cu_seqlens.numel() - 1
    assert qkv.shape[1] == 3 * H * dh and out.shape == (T, H * dh) and tile_prefix.numel() == S + 1
    with _Timed("attention_varlen", bytes=(qkv.numel() + out.numel()) * 2):
        if mask_self:
            rc = lib().b200vit_attention_varlen_ex(_ptr(qkv), _ptr(out), _ptr(cu_seqlens), _ptr(tile_prefix), S, T,
                                                   int(total_tiles), H, dh, float(scale), ATTN_MASK_SELF, _stream())
        else:
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


def attention_cls(qkv_self: torch.Tensor, ctx: Optional[torch.Tensor], out: torch.Tensor, rows_per_image: int,
                  first: int, n: int, H: int, dh: int, scale: float) -> None:
    """Class-token cross attention: the query of image b (row b of qkv_self[B, 3*H*dh], q | k | v) attends over its
    own k / v and rows b*rows_per_image + first + j (j < n) of the [k | v] matrix ctx (row stride ctx.stride(0)).
    out [B, H*dh] bf16, any row stride."""
    _chk(qkv_self, torch.bfloat16, "qkv_self"); _chk(ctx, torch.bfloat16, "ctx"); _chk(out, torch.bfloat16, "out")
    B = qkv_self.shape[0]
    assert qkv_self.is_contiguous() and qkv_self.shape[1] == 3 * H * dh
    assert out.dim() == 2 and out.stride(1) == 1 and out.shape == (B, H * dh)
    assert ctx is None or (ctx.dim() == 2 and ctx.stride(1) == 1 and ctx.shape[1] >= 2 * H * dh
                           and ctx.shape[0] >= (B - 1) * rows_per_image + first + n)
    with _Timed("attention_cls", B=B, n=n, H=H, bytes=(B * n * 2 * H * dh + qkv_self.numel() + out.numel()) * 2,
                flops=4.0 * B * H * (n + 1) * dh):
        rc = lib().b200vit_attention_cls(_ptr(qkv_self), _ptr(ctx), 0 if ctx is None else ctx.stride(0),
                                         int(rows_per_image), int(first), int(n), _ptr(out), out.stride(0), B, H, dh,
                                         float(scale), _stream())
    _check(rc, "b200vit_attention_cls")


def attention_headmix(qkv: torch.Tensor, out: torch.Tensor, B: int, N: int, H: int, dh: int, scale: float,
                       post: torch.Tensor, head_ln: Optional[tuple] = None, pre: Optional[torch.Tensor] = None) -> None:
    """Attention with heads mixed across the head axis (re-attention, talking heads) over B sequences of N tokens of
    qkv[B*N, 3*H*dh]: post (fp32 [H, H], indexed [input head, output head]) mixes the softmax probabilities; head_ln =
    (gamma [H], beta [H], eps) adds a LayerNorm over the heads of every (query, key) pair after the mix; pre (fp32
    [H, H], same indexing) mixes the scores before the softmax (b200vit_attention_headmix_ex)."""
    _chk(qkv, torch.bfloat16, "qkv"); _chk(out, torch.bfloat16, "out")
    _chk(post, torch.float32, "post"); _chk(pre, torch.float32, "pre")
    assert qkv.is_contiguous() and out.is_contiguous()
    assert qkv.shape == (B * N, 3 * H * dh) and out.shape == (B * N, H * dh)
    assert post.is_contiguous() and post.shape == (H, H)
    assert pre is None or (pre.is_contiguous() and pre.shape == (H, H))
    g = b = None
    eps = 0.0
    if head_ln is not None:
        g, b, eps = head_ln
        _chk(g, torch.float32, "head_ln gamma"); _chk(b, torch.float32, "head_ln beta")
        assert g.is_contiguous() and b.is_contiguous() and g.numel() == H and b.numel() == H
    with _Timed("attention_headmix", B=B, N=N, H=H, bytes=(qkv.numel() + out.numel()) * 2,
                flops=4.0 * B * H * N * N * dh):
        rc = lib().b200vit_attention_headmix_ex(_ptr(qkv), _ptr(out), B, N, H, dh, float(scale), _ptr(pre),
                                                _ptr(post), _ptr(g), _ptr(b), float(eps), _stream())
    _check(rc, "b200vit_attention_headmix_ex")


def attention_cls_headmix(qkv_self: torch.Tensor, ctx: Optional[torch.Tensor], out: torch.Tensor,
                          rows_per_image: int, first: int, n: int, H: int, dh: int, scale: float, pre: torch.Tensor,
                          post: torch.Tensor) -> None:
    """Class-token attention with talking heads: the addressing of attention_cls, with the heads mixed by pre (fp32
    [H, H], [input head, output head]) before the softmax and by post after it."""
    _chk(qkv_self, torch.bfloat16, "qkv_self"); _chk(ctx, torch.bfloat16, "ctx"); _chk(out, torch.bfloat16, "out")
    _chk(pre, torch.float32, "pre"); _chk(post, torch.float32, "post")
    B = qkv_self.shape[0]
    assert qkv_self.is_contiguous() and qkv_self.shape[1] == 3 * H * dh
    assert out.dim() == 2 and out.stride(1) == 1 and out.shape == (B, H * dh)
    assert ctx is None or (ctx.dim() == 2 and ctx.stride(1) == 1 and ctx.shape[1] >= 2 * H * dh
                           and ctx.shape[0] >= (B - 1) * rows_per_image + first + n)
    assert pre.is_contiguous() and pre.shape == (H, H) and post.is_contiguous() and post.shape == (H, H)
    with _Timed("attention_cls_headmix", B=B, n=n, H=H, bytes=(B * n * 2 * H * dh + qkv_self.numel() + out.numel()) * 2,
                flops=4.0 * B * H * (n + 1) * dh):
        rc = lib().b200vit_attention_cls_headmix(_ptr(qkv_self), _ptr(ctx), 0 if ctx is None else ctx.stride(0),
                                                 int(rows_per_image), int(first), int(n), _ptr(out), out.stride(0), B,
                                                 H, dh, float(scale), _ptr(pre), _ptr(post), _stream())
    _check(rc, "b200vit_attention_cls_headmix")


def attention_xca(qkv: torch.Tensor, tau: torch.Tensor, out: torch.Tensor, B: int, N: int, H: int, dh: int) -> None:
    """Cross-covariance attention over the channels of every head (XCiT): qkv[B*N, 3*H*dh] packed q | k | v, tau fp32
    [H] (temperature.exp()), out[B*N, H*dh]."""
    _chk(qkv, torch.bfloat16, "qkv"); _chk(tau, torch.float32, "tau"); _chk(out, torch.bfloat16, "out")
    assert qkv.is_contiguous() and out.is_contiguous() and tau.is_contiguous() and tau.numel() == H
    assert qkv.shape == (B * N, 3 * H * dh) and out.shape == (B * N, H * dh)
    with _Timed("attention_xca", B=B, N=N, H=H, bytes=(qkv.numel() + out.numel()) * 2, flops=4.0 * B * H * N * dh * dh):
        rc = lib().b200vit_attention_xca(_ptr(qkv), _ptr(tau), _ptr(out), B, N, H, dh, _stream())
    _check(rc, "b200vit_attention_xca")


def local_patch_interaction(x: torch.Tensor, y: torch.Tensor, ln_scratch: torch.Tensor, ln: tuple, w1: torch.Tensor,
                            b1: torch.Tensor, w2: torch.Tensor, b2: torch.Tensor, B: int, gh: int, gw: int, k: int,
                            y_bf16: Optional[torch.Tensor] = None, y_stats: Optional[torch.Tensor] = None) -> None:
    """y = x + conv2'(GELU(conv1'(LayerNorm(x)))) on B grids of gh x gw tokens of x fp32 [B*gh*gw, D] (XCiT's LPI).
    ln = (gamma, beta, eps); w1, w2 fp32 [k*k, D] tap-major depthwise weights, BatchNorm folded into w1 / b1 and
    LayerScale into w2 / b2.  y_bf16 / y_stats [M, 2]: the bf16 copy of y and its rowstats_cast statistics.
    ln_scratch fp32 [M, 2] is overwritten."""
    g, bt, eps = ln
    for nm, t in (("x", x), ("y", y), ("ln_scratch", ln_scratch), ("ln gamma", g), ("ln beta", bt), ("w1", w1),
                  ("b1", b1), ("w2", w2), ("b2", b2), ("y_stats", y_stats)):
        _chk(t, torch.float32, nm)
    _chk(y_bf16, torch.bfloat16, "y_bf16")
    M, D = x.shape
    assert M == B * gh * gw and y.shape == x.shape and x.is_contiguous() and y.is_contiguous()
    assert ln_scratch.is_contiguous() and ln_scratch.numel() >= 2 * M
    for t in (g, bt, b1, b2):
        assert t.is_contiguous() and t.numel() == D
    for t in (w1, w2):
        assert t.is_contiguous() and t.shape == (k * k, D)
    assert (y_bf16 is None) == (y_stats is None)
    assert y_bf16 is None or (y_bf16.is_contiguous() and y_bf16.shape == x.shape and y_stats.is_contiguous()
                              and y_stats.numel() == 2 * M)
    with _Timed("local_patch_interaction", B=B, h=gh, w=gw, D=D, k=k,
                bytes=M * D * (4 + 4 + (2 if y_bf16 is not None else 0))):
        rc = lib().b200vit_local_patch_interaction(_ptr(x), _ptr(y), _ptr(y_bf16), _ptr(y_stats), _ptr(ln_scratch),
                                                   _ptr(g), _ptr(bt), float(eps), _ptr(w1), _ptr(b1), _ptr(w2),
                                                   _ptr(b2), B, gh, gw, D, int(k), _stream())
    _check(rc, "b200vit_local_patch_interaction")


def unfold_patches(img: torch.Tensor, out_bf16: torch.Tensor, p: int, s: int) -> None:
    """img [B, C, H, W] bf16 -> out [B*oh*ow, ldo] bf16 rows of F.unfold(img, p, stride=s).transpose(1, 2) (columns
    (c, i, j), channel slowest), zero K padding up to ldo = out.stride(0)."""
    _chk(img, torch.bfloat16, "img"); _chk(out_bf16, torch.bfloat16, "out")
    assert img.is_contiguous() and img.dim() == 4 and out_bf16.dim() == 2 and out_bf16.stride(1) == 1
    B, Cc, H, W = img.shape
    rows = B * ((H - p) // s + 1) * ((W - p) // s + 1)
    assert out_bf16.shape[0] == rows and out_bf16.shape[1] >= Cc * p * p, \
        f"out must be [{rows}, >= {Cc * p * p}], got {tuple(out_bf16.shape)}"
    with _Timed("unfold_patches", bytes=img.numel() * 2 + rows * out_bf16.stride(0) * 2):
        rc = lib().b200vit_unfold_patches(_ptr(img), _ptr(out_bf16), out_bf16.stride(0), B, Cc, H, W, int(p), int(s),
                                          _stream())
    _check(rc, "b200vit_unfold_patches")


def pit_pool(x: torch.Tensor, B: int, h: int, w: int, w9: torch.Tensor, bias: torch.Tensor, a_bf16: torch.Tensor,
             cls_bf16: torch.Tensor) -> None:
    """PiT's Pool before its 1 x 1 convolution: x fp32 [B*(1 + h*w), D] (cls row, then the h x w grid) -> a_bf16
    [B*(1 + oh*ow), >= 2D] = the depthwise 3 x 3 / stride 2 / pad 1 convolution with channel multiplier 2 (+ bias) of
    every grid, cls slots zero filled, and cls_bf16 [B, >= D] = the bf16 cls rows.  w9 fp32 [9, 2D] tap major, bias
    fp32 [2D]."""
    for nm, t in (("x", x), ("w9", w9), ("bias", bias)):
        _chk(t, torch.float32, nm)
    _chk(a_bf16, torch.bfloat16, "a"); _chk(cls_bf16, torch.bfloat16, "cls")
    M, D = x.shape
    oh, ow = (h + 1) // 2, (w + 1) // 2
    assert x.is_contiguous() and w9.is_contiguous() and bias.is_contiguous()
    assert w9.shape == (9, 2 * D) and bias.numel() == 2 * D
    assert a_bf16.dim() == 2 and a_bf16.stride(1) == 1 and a_bf16.shape[0] == B * (1 + oh * ow) \
        and a_bf16.shape[1] >= 2 * D
    assert cls_bf16.dim() == 2 and cls_bf16.stride(1) == 1 and cls_bf16.shape[0] == B and cls_bf16.shape[1] >= D
    with _Timed("pit_pool", B=B, h=h, w=w, D=D, bytes=M * D * 4 + B * (1 + oh * ow) * 2 * D * 2):
        rc = lib().b200vit_pit_pool(_ptr(x), M, B, int(h), int(w), D, _ptr(w9), _ptr(bias), _ptr(a_bf16),
                                    a_bf16.stride(0), _ptr(cls_bf16), cls_bf16.stride(0), _stream())
    _check(rc, "b200vit_pit_pool")


def conv_out_size(n: int, k: int, s: int, p: int) -> int:
    """Output length of a Conv2d / MaxPool2d window along one axis (dilation 1, floor mode)."""
    return (n + 2 * p - k) // s + 1


def conv_im2col_nchw(img: torch.Tensor, out_bf16: torch.Tensor, k: int, s: int, p: int) -> None:
    """img [B, C, H, W] bf16 -> out [B*oh*ow, ldo] bf16 rows of F.unfold(img, k, padding=p, stride=s).transpose(1, 2)
    (columns (c, i, j), channel slowest), zero K padding up to ldo = out.stride(0)."""
    _chk(img, torch.bfloat16, "img"); _chk(out_bf16, torch.bfloat16, "out")
    assert img.is_contiguous() and img.dim() == 4 and out_bf16.dim() == 2 and out_bf16.stride(1) == 1
    B, Cc, H, W = img.shape
    rows = B * conv_out_size(H, k, s, p) * conv_out_size(W, k, s, p)
    assert out_bf16.shape[0] == rows and out_bf16.shape[1] >= Cc * k * k, \
        f"out must be [{rows}, >= {Cc * k * k}], got {tuple(out_bf16.shape)}"
    with _Timed("conv_im2col", bytes=img.numel() * 2 + rows * out_bf16.stride(0) * 2):
        rc = lib().b200vit_conv_im2col_nchw(_ptr(img), _ptr(out_bf16), out_bf16.stride(0), B, Cc, H, W, int(k), int(s),
                                            int(p), _stream())
    _check(rc, "b200vit_conv_im2col_nchw")


def conv_im2col_nhwc(x: torch.Tensor, out_bf16: torch.Tensor, B: int, H: int, W: int, k: int, s: int, p: int) -> None:
    """x [B*H*W, C] bf16 channels-last -> out [B*oh*ow, ldo] bf16, column (i*k + j)*C + c the channel c of tap (i, j)
    of the zero-padded k x k window at stride s, zero K padding up to ldo = out.stride(0).  x may be a column slice of
    a wider buffer (rows x.stride(0) apart: b200vit_conv_im2col_nhwc_ex)."""
    _chk(x, torch.bfloat16, "x"); _chk(out_bf16, torch.bfloat16, "out")
    assert x.dim() == 2 and x.stride(1) == 1 and out_bf16.dim() == 2 and out_bf16.stride(1) == 1
    M, Cc = x.shape
    rows = B * conv_out_size(H, k, s, p) * conv_out_size(W, k, s, p)
    assert out_bf16.shape[0] == rows and out_bf16.shape[1] >= Cc * k * k, \
        f"out must be [{rows}, >= {Cc * k * k}], got {tuple(out_bf16.shape)}"
    with _Timed("conv_im2col", bytes=x.numel() * 2 + rows * out_bf16.stride(0) * 2):
        if x.is_contiguous():
            rc = lib().b200vit_conv_im2col_nhwc(_ptr(x), M, _ptr(out_bf16), out_bf16.stride(0), B, H, W, Cc, int(k),
                                                int(s), int(p), _stream())
        else:
            rc = lib().b200vit_conv_im2col_nhwc_ex(_ptr(x), x.stride(0), M, _ptr(out_bf16), out_bf16.stride(0), B, H,
                                                   W, Cc, int(k), int(s), int(p), _stream())
    _check(rc, "b200vit_conv_im2col_nhwc")


def merge_patches_ln(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, out_bf16: torch.Tensor, B: int, gh: int,
                     gw: int, p: int, eps: float = 1e-5) -> None:
    """x fp32 [B*gh*gw, C] token map -> out [B*(gh/p)*(gw/p), ldo] bf16: every p x p block's tokens concatenated in
    (p1 p2 c) order, LayerNorm over all p*p*C values (gamma, beta in that order), zero K padding up to ldo."""
    for nm, t in (("x", x), ("gamma", gamma), ("beta", beta)):
        _chk(t, torch.float32, nm)
    _chk(out_bf16, torch.bfloat16, "out")
    M, Cc = x.shape
    K = p * p * Cc
    rows = B * (gh // p) * (gw // p)
    assert x.is_contiguous() and gamma.is_contiguous() and beta.is_contiguous() and gamma.numel() == beta.numel() == K
    assert out_bf16.dim() == 2 and out_bf16.stride(1) == 1 and out_bf16.shape[0] == rows and out_bf16.shape[1] >= K, \
        f"out must be [{rows}, >= {K}], got {tuple(out_bf16.shape)}"
    with _Timed("merge_patches_ln", B=B, h=gh, w=gw, C=Cc, p=p, bytes=M * Cc * 4 + rows * out_bf16.stride(0) * 2):
        rc = lib().b200vit_merge_patches_ln(_ptr(x), M, _ptr(gamma), _ptr(beta), _ptr(out_bf16), out_bf16.stride(0), B,
                                            int(gh), int(gw), Cc, int(p), float(eps), _stream())
    _check(rc, "b200vit_merge_patches_ln")


def peg(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, y: torch.Tensor, B: int, gh: int, gw: int, k: int) -> None:
    """y = x + depthwise k x k convolution (zero padding k // 2, + bias) of the B token maps x fp32 [B*gh*gw, C];
    w fp32 [k*k, C] tap major, bias fp32 [C]; y is another buffer."""
    for nm, t in (("x", x), ("w", w), ("bias", bias), ("y", y)):
        _chk(t, torch.float32, nm)
    M, Cc = x.shape
    assert x.is_contiguous() and y.is_contiguous() and y.shape == x.shape and w.is_contiguous() and bias.is_contiguous()
    assert w.shape == (k * k, Cc) and bias.numel() == Cc
    with _Timed("peg", B=B, h=gh, w=gw, C=Cc, k=k, bytes=M * Cc * 8):
        rc = lib().b200vit_peg(_ptr(x), M, _ptr(w), _ptr(bias), _ptr(y), B, int(gh), int(gw), Cc, int(k), _stream())
    _check(rc, "b200vit_peg")


def conv_proj_dw(x: torch.Tensor, wq: torch.Tensor, bq: torch.Tensor, wkv: torch.Tensor, bkv: torch.Tensor,
                 q_out: torch.Tensor, kv_out: torch.Tensor, B: int, h: int, w: int, k: int, s: int) -> None:
    """CvT's depthwise convolutional projections from one read of x bf16 [B*h*w, C] channels-last: q_out bf16
    [B*h*w, C] the k x k depthwise convolution (zero padding k // 2) at stride 1, kv_out bf16 [B*oh*ow, C]
    (oh = (h - 1) // s + 1, likewise ow) the same at stride s; wq, wkv fp32 [k*k, C] tap major and bq, bkv fp32 [C]
    with the BatchNorm folded in."""
    _chk(x, torch.bfloat16, "x"); _chk(q_out, torch.bfloat16, "q_out"); _chk(kv_out, torch.bfloat16, "kv_out")
    for nm, t in (("wq", wq), ("bq", bq), ("wkv", wkv), ("bkv", bkv)):
        _chk(t, torch.float32, nm)
    M, Cc = x.shape
    oh, ow = (h - 1) // s + 1, (w - 1) // s + 1
    assert x.is_contiguous() and q_out.is_contiguous() and kv_out.is_contiguous()
    assert q_out.shape == (M, Cc) and kv_out.shape == (B * oh * ow, Cc)
    for wt, bt in ((wq, bq), (wkv, bkv)):
        assert wt.is_contiguous() and bt.is_contiguous() and wt.shape == (k * k, Cc) and bt.numel() == Cc
    with _Timed("conv_proj_dw", B=B, h=h, w=w, C=Cc, k=k, s=s, bytes=(2 * M + kv_out.shape[0]) * Cc * 2):
        rc = lib().b200vit_conv_proj_dw(_ptr(x), M, _ptr(wq), _ptr(bq), _ptr(wkv), _ptr(bkv), _ptr(q_out),
                                        _ptr(kv_out), B, int(h), int(w), Cc, int(k), int(s), _stream())
    _check(rc, "b200vit_conv_proj_dw")


CROSS_EMBED_MAX_SCALES, CROSS_EMBED_MAX_KERNEL, CROSS_EMBED_MAX_CHANNELS = 4, 32, 4   # include/b200vit.h
CROSS_EMBED_MAX_STRIDE, CROSS_EMBED_MAX_WIDTH = 8, 64


def cross_embed_pack(weights) -> torch.Tensor:
    """The packed weight of b200vit_cross_embed_nchw from the scales' Conv2d weights [n_i, C, k_i, k_i]: bf16, scale
    after scale [n_i, Kp_i] with Kp_i = C*k_i^2 rounded up to a multiple of 64, columns (c, y, x), zeros past
    C*k_i^2."""
    parts = []
    for w in weights:
        w = w.detach().reshape(w.shape[0], -1)
        kp = (w.shape[1] + 63) // 64 * 64
        wp = torch.zeros(w.shape[0], kp, device=w.device, dtype=torch.bfloat16)
        wp[:, : w.shape[1]] = w
        parts.append(wp.reshape(-1))
    return torch.cat(parts)


def cross_embed_nchw(img: torch.Tensor, w_packed: torch.Tensor, bias: torch.Tensor, out: torch.Tensor,
                     kernel_sizes, widths, s: int) -> None:
    """CrossFormer's cross-scale embedding: img [B, C, H, W] bf16 -> out fp32 [B*oh*ow, ldo = out.stride(0)], columns
    [off_i, off_i + widths[i]) the Conv2d of kernel kernel_sizes[i], stride s, padding (k_i - s) // 2, plus its bias
    (bias fp32 [sum widths], output column order); w_packed from cross_embed_pack."""
    _chk(img, torch.bfloat16, "img"); _chk(w_packed, torch.bfloat16, "w"); _chk(bias, torch.float32, "bias")
    _chk(out, torch.float32, "out")
    assert img.is_contiguous() and img.dim() == 4 and out.dim() == 2 and out.stride(1) == 1
    assert w_packed.is_contiguous() and bias.is_contiguous() and len(kernel_sizes) == len(widths)
    B, Cc, H, W = img.shape
    S, D = len(kernel_sizes), sum(widths)
    p = (kernel_sizes[0] - s) // 2
    oh, ow = conv_out_size(H, kernel_sizes[0], s, p), conv_out_size(W, kernel_sizes[0], s, p)
    assert out.shape[0] == B * oh * ow and out.shape[1] >= D and bias.numel() == D
    assert w_packed.numel() == sum(n * ((Cc * k * k + 63) // 64 * 64) for k, n in zip(kernel_sizes, widths))
    ks = (C.c_int * S)(*[int(k) for k in kernel_sizes])
    ns = (C.c_int * S)(*[int(n) for n in widths])
    flops = 2.0 * B * oh * ow * sum(n * Cc * k * k for k, n in zip(kernel_sizes, widths))
    with _Timed("cross_embed_nchw", B=B, C=Cc, H=H, W=W, ks=tuple(kernel_sizes), ns=tuple(widths), s=s, flops=flops):
        rc = lib().b200vit_cross_embed_nchw(_ptr(img), _ptr(w_packed), _ptr(bias), _ptr(out), out.stride(0), B, Cc, H,
                                            W, S, ks, ns, int(s), _stream())
    _check(rc, "b200vit_cross_embed_nchw")


def relu_maxpool(y: torch.Tensor, B: int, H: int, W: int, pk: int, ps: int, pp: int, *,
                 out_bf16: Optional[torch.Tensor] = None, out_f32: Optional[torch.Tensor] = None) -> None:
    """y [B*H*W, C] bf16 channels-last -> relu(max_pool2d(y, pk, ps, pp)) channels-last [B*oh*ow, C] into exactly one
    of out_bf16 / out_f32 (row stride out.stride(0))."""
    _chk(y, torch.bfloat16, "y"); _chk(out_bf16, torch.bfloat16, "out_bf16"); _chk(out_f32, torch.float32, "out_f32")
    assert (out_bf16 is None) != (out_f32 is None)
    out = out_bf16 if out_bf16 is not None else out_f32
    assert y.is_contiguous() and y.dim() == 2 and out.dim() == 2 and out.stride(1) == 1
    M, Cc = y.shape
    rows = B * conv_out_size(H, pk, ps, pp) * conv_out_size(W, pk, ps, pp)
    assert out.shape[0] == rows and out.shape[1] >= Cc, f"out must be [{rows}, >= {Cc}], got {tuple(out.shape)}"
    with _Timed("relu_maxpool", bytes=M * Cc * 2 + rows * Cc * out.element_size()):
        rc = lib().b200vit_relu_maxpool(_ptr(y), M, B, H, W, Cc, int(pk), int(ps), int(pp), _ptr(out_bf16),
                                        _ptr(out_f32), out.stride(0), _stream())
    _check(rc, "b200vit_relu_maxpool")


NEST_POOL_MAX_KERNEL = 3      # B200VIT_NEST_POOL_MAX_KERNEL


def nest_level_entry(y: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, pos: torch.Tensor, x: torch.Tensor,
                     B: int, H: int, W: int, pk: int, ps: int, pp: int, nb: int, *, eps: float = 1e-5,
                     xb: Optional[torch.Tensor] = None, stats: Optional[torch.Tensor] = None) -> None:
    """NesT's level entry: y fp32 [B*H*W, D] in map order -> x fp32 [B*oh*ow, D] = max_pool2d(LN(y), pk, ps, pp) +
    pos[r], in the block-major order of nb x nb blocks (r the token's place in its block); with xb / stats (both or
    neither) also the bf16 copy of x and its row statistics, as rowstats_cast writes them."""
    for nm, t in (("y", y), ("gamma", gamma), ("beta", beta), ("pos", pos), ("x", x), ("stats", stats)):
        _chk(t, torch.float32, nm)
    _chk(xb, torch.bfloat16, "xb")
    M, D = y.shape
    for t in (y, x, gamma, beta, pos, xb, stats):
        assert t is None or t.is_contiguous()
    rows = B * conv_out_size(H, pk, ps, pp) * conv_out_size(W, pk, ps, pp)
    assert gamma.numel() == D and beta.numel() == D and x.shape == (rows, D), \
        f"x must be [{rows}, {D}], got {tuple(x.shape)}"
    assert xb is None or xb.shape == (rows, D)
    assert stats is None or stats.numel() == 2 * rows
    with _Timed("nest_level_entry", B=B, H=H, W=W, D=D, pk=pk, ps=ps, pp=pp, nb=nb,
                bytes=M * D * 4 + rows * D * (4 + (2 if xb is not None else 0)) + (rows * 8 if stats is not None else 0)):
        rc = lib().b200vit_nest_level_entry(_ptr(y), M, _ptr(gamma), _ptr(beta), float(eps), _ptr(pos), pos.numel(),
                                            _ptr(x), _ptr(xb), _ptr(stats), B, int(H), int(W), D, int(pk), int(ps),
                                            int(pp), int(nb), _stream())
    _check(rc, "b200vit_nest_level_entry")


def nest_im2col(x: torch.Tensor, out_bf16: torch.Tensor, B: int, H: int, W: int, nb: int) -> None:
    """x fp32 [B*H*W, D] block-major (nb x nb blocks) -> out bf16 [B*H*W, ldo] in map order, column (i*3 + j)*D + c the
    channel c of pixel (y - 1 + i, x - 1 + j) (zero outside the map), zero K padding up to ldo = out.stride(0)."""
    _chk(x, torch.float32, "x"); _chk(out_bf16, torch.bfloat16, "out")
    assert x.dim() == 2 and x.is_contiguous() and out_bf16.dim() == 2 and out_bf16.stride(1) == 1
    M, D = x.shape
    assert out_bf16.shape[0] == M and out_bf16.shape[1] >= 9 * D, \
        f"out must be [{M}, >= {9 * D}], got {tuple(out_bf16.shape)}"
    with _Timed("nest_im2col", B=B, H=H, W=W, D=D, nb=nb, bytes=M * D * 4 + M * out_bf16.stride(0) * 2):
        rc = lib().b200vit_nest_im2col(_ptr(x), M, _ptr(out_bf16), out_bf16.stride(0), B, int(H), int(W), D, int(nb),
                                       _stream())
    _check(rc, "b200vit_nest_im2col")


def seq_pool(x: torch.Tensor, B: int, n: int, gamma: torch.Tensor, beta: torch.Tensor, w: torch.Tensor,
             bias: torch.Tensor, out_bf16: torch.Tensor, eps: float = 1e-5) -> None:
    """x fp32 [B*n, D] -> out_bf16 [B, D] (any row stride) = sum_t softmax_t(LN(x_t) . w + bias) LN(x_t) per image
    (CCT's sequence pooling).  gamma, beta, w fp32 [D], bias fp32 [1]."""
    for nm, t in (("x", x), ("gamma", gamma), ("beta", beta), ("w", w), ("bias", bias)):
        _chk(t, torch.float32, nm)
    _chk(out_bf16, torch.bfloat16, "out")
    M, D = x.shape
    assert M == B * n and x.is_contiguous()
    for t in (gamma, beta, w):
        assert t.is_contiguous() and t.numel() == D
    assert bias.numel() == 1
    assert out_bf16.dim() == 2 and out_bf16.stride(1) == 1 and out_bf16.shape == (B, D)
    with _Timed("seq_pool", B=B, n=n, D=D, bytes=M * D * 4):
        rc = lib().b200vit_seq_pool(_ptr(x), B, n, D, _ptr(gamma), _ptr(beta), float(eps), _ptr(w), _ptr(bias),
                                    _ptr(out_bf16), out_bf16.stride(0), _stream())
    _check(rc, "b200vit_seq_pool")


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


def _unfold_out(out: torch.Tensor, rows: int, K: int, what: str):
    assert out.dim() == 2 and out.stride(1) == 1 and out.shape[0] == rows and out.shape[1] >= K, \
        f"{what}: out must be [{rows}, >= {K}], got {tuple(out.shape)}"
    if out.dtype == torch.float32:
        _chk(out, torch.float32, "out")
        return None, out
    _chk(out, torch.bfloat16, "out")
    return out, None


def t2t_unfold_image(img: torch.Tensor, out: torch.Tensor, k: int, s: int, p: int) -> None:
    """img [B, C, H, W] bf16 -> out [B*oh*ow, ldo] (bf16 or fp32) rows of F.unfold(img, k, padding=p, stride=s)
    .transpose(1, 2) (columns (c, i, j), channel slowest), zero K padding up to ldo = out.stride(0)."""
    _chk(img, torch.bfloat16, "img")
    assert img.is_contiguous() and img.dim() == 4
    B, Cc, H, W = img.shape
    rows = B * conv_out_size(H, k, s, p) * conv_out_size(W, k, s, p)
    ob, of = _unfold_out(out, rows, Cc * k * k, "t2t_unfold_image")
    with _Timed("t2t_unfold", bytes=img.numel() * 2 + rows * out.stride(0) * out.element_size()):
        rc = lib().b200vit_t2t_unfold_image(_ptr(img), _ptr(ob), _ptr(of), out.stride(0), B, Cc, H, W, int(k), int(s),
                                            int(p), _stream())
    _check(rc, "b200vit_t2t_unfold_image")


def t2t_unfold_tokens(x: torch.Tensor, grid, out: torch.Tensor, k: int, s: int, p: int) -> None:
    """x [B*n, C] bf16 (rows x.stride(0) apart), the token rows of B images read as the map grid = (h, w) that
    RearrangeImage makes of n = h*w tokens (pit.pool_grid; the library checks h == int(sqrt(n))) -> out [B*oh*ow, ldo]
    (bf16 or fp32) rows of the zero-padded unfold, as t2t_unfold_image."""
    _chk(x, torch.bfloat16, "x")
    h, w = grid
    n = h * w
    assert x.dim() == 2 and x.stride(1) == 1 and x.shape[0] % n == 0
    B, Cc = x.shape[0] // n, x.shape[1]
    rows = B * conv_out_size(h, k, s, p) * conv_out_size(w, k, s, p)
    ob, of = _unfold_out(out, rows, Cc * k * k, "t2t_unfold_tokens")
    with _Timed("t2t_unfold", bytes=x.shape[0] * Cc * 2 + rows * out.stride(0) * out.element_size()):
        rc = lib().b200vit_t2t_unfold_tokens(_ptr(x), x.stride(0), B, int(n), Cc, _ptr(ob), _ptr(of), out.stride(0),
                                             int(k), int(s), int(p), _stream())
    _check(rc, "b200vit_t2t_unfold_tokens")


def attention_wide_workspace(n: int, dp: int, images: int) -> int:
    """Bytes of the workspace b200vit_attention_wide needs to run `images` images per chunk."""
    return int(lib().b200vit_attention_wide_workspace(int(n), int(dp), int(images)))


def attention_wide(qkv: torch.Tensor, B: int, n: int, dp: int, scale: float, ws: torch.Tensor, *,
                   out: Optional[torch.Tensor] = None, x: Optional[torch.Tensor] = None,
                   n_resid: int = 0) -> None:
    """One head as wide as the token over B images of n tokens: qkv [B*n, 3*dp] bf16 -> out [B*n, dp] bf16 and/or, x
    fp32 given (rows x.stride(0) apart), x[:, :n_resid] += bf16(O[:, :n_resid]).  ws: uint8 scratch (any size holding
    one image, see attention_wide_workspace)."""
    _chk(qkv, torch.bfloat16, "qkv"); _chk(out, torch.bfloat16, "out"); _chk(x, torch.float32, "x")
    _chk(ws, torch.uint8, "ws")
    assert qkv.is_contiguous() and qkv.shape == (B * n, 3 * dp) and ws.is_contiguous()
    assert out is None or (out.is_contiguous() and out.shape == (B * n, dp))
    assert x is None or (x.dim() == 2 and x.stride(1) == 1 and x.shape[0] == B * n)
    with _Timed("attention_wide", B=B, N=n, H=1, bytes=(qkv.numel() + B * n * dp) * 2,
                flops=4.0 * B * n * n * dp):
        rc = lib().b200vit_attention_wide(_ptr(qkv), _ptr(out), _ptr(x), 0 if x is None else x.stride(0),
                                          int(n_resid), B, int(n), int(dp), float(scale), _ptr(ws), ws.numel(),
                                          _stream())
    _check(rc, "b200vit_attention_wide")


def _need(cond: bool, msg: str) -> None:
    """An argument check of the Adaptive Token Sampling wrappers: raises B200VitError (not an assert, which -O drops)."""
    if not cond:
        raise B200VitError(msg)


def _rows2d(t: Optional[torch.Tensor], name: str) -> None:
    _need(t is None or (t.dim() == 2 and t.stride(1) == 1), f"{name} must be 2-D with unit column stride")


def ats_select(qkv: torch.Tensor, lens: torch.Tensor, ids: torch.Tensor, u: torch.Tensor, src: torch.Tensor,
               lens_out: torch.Tensor, ids_out: torch.Tensor, B: int, S_in: int, K: int, H: int, dh: int,
               scale: float) -> None:
    """Adaptive Token Sampling's selection over B images of S_in-row slots (b200vit_ats_select): qkv [B*S_in, >= 3*H*dh]
    bf16 (any row stride), lens int32 [B] and ids int32 [B*S_in] in; u [B, K, S_in - 1] fp32 or bf16 uniforms; out
    src int32 [B*S_out], lens_out int32 [B], ids_out int32 [B*S_out], S_out = min(S_in, K + 1)."""
    S_out = min(S_in, K + 1)
    _rows2d(qkv, "qkv")
    _need(qkv.shape[0] == B * S_in and qkv.shape[1] >= 3 * H * dh,
          f"ats_select: qkv must be [{B * S_in}, >= {3 * H * dh}], got {tuple(qkv.shape)}")
    _need(u.dtype in (torch.float32, torch.bfloat16), f"ats_select: u must be fp32 or bf16 uniforms, got {u.dtype}")
    _need(u.is_contiguous() and tuple(u.shape) == (B, K, S_in - 1),
          f"ats_select: u must be contiguous [{B}, {K}, {S_in - 1}], got {tuple(u.shape)}")
    for t, name, n in ((lens, "lens", B), (ids, "ids", B * S_in), (src, "src", B * S_out),
                       (lens_out, "lens_out", B), (ids_out, "ids_out", B * S_out)):
        _need(t.dtype == torch.int32 and t.is_contiguous() and tuple(t.shape) == (n,),
              f"ats_select: {name} must be contiguous int32 [{n}], got {t.dtype} {tuple(t.shape)}")
    _need(lens.data_ptr() != lens_out.data_ptr() and ids.data_ptr() != ids_out.data_ptr(),
          "ats_select: lengths and ids cannot be updated in place")
    _chk(qkv, torch.bfloat16, "qkv")
    _chk(u, u.dtype, "u")
    for t, name in ((lens, "lens"), (ids, "ids"), (src, "src"), (lens_out, "lens_out"), (ids_out, "ids_out")):
        _chk(t, torch.int32, name)
    with _Timed("ats_select", B=B, S=S_in, K=K, H=H, bytes=B * S_in * 3 * H * dh * 2 + u.numel() * u.element_size()):
        rc = lib().b200vit_ats_select(_ptr(qkv), qkv.stride(0), _ptr(lens), _ptr(ids), _ptr(u),
                                      1 if u.dtype == torch.bfloat16 else 0, _ptr(src), _ptr(lens_out), _ptr(ids_out),
                                      B, int(S_in), int(S_out), int(K), H, dh, float(scale), _stream())
    _check(rc, "b200vit_ats_select")


def ats_gather(src: torch.Tensor, *, x: Optional[torch.Tensor] = None, x_out: Optional[torch.Tensor] = None,
               a: Optional[torch.Tensor] = None, a_out: Optional[torch.Tensor] = None, ncols: int = 0) -> None:
    """x_out[r] = x[src[r]] (fp32 rows) and / or a_out[r, :ncols] = a[src[r], :ncols] (bf16), r < src.numel(), as bit
    copies (b200vit_ats_gather); rows of any stride."""
    rows = src.numel()
    _need(src.dtype == torch.int32 and src.is_contiguous() and src.dim() == 1,
          f"ats_gather: src must be a contiguous int32 vector, got {src.dtype} {tuple(src.shape)}")
    _need((x is None) == (x_out is None) and (a is None) == (a_out is None) and (x is not None or a is not None),
          "ats_gather: give x with x_out and/or a with a_out")
    for t, name in ((x, "x"), (x_out, "x_out"), (a, "a"), (a_out, "a_out")):
        _rows2d(t, f"ats_gather: {name}")
    if x is not None:
        _need(x_out.shape == (rows, x.shape[1]), f"ats_gather: x_out must be [{rows}, {x.shape[1]}], "
              f"got {tuple(x_out.shape)}")
        _need(x.dtype == x_out.dtype == torch.float32, "ats_gather: x and x_out must be fp32")
    if a is not None:
        _need(a_out.shape[0] == rows and 0 < ncols <= min(a.shape[1], a_out.shape[1]),
              f"ats_gather: a_out must have {rows} rows and a, a_out at least ncols={ncols} columns")
        _need(a.dtype == a_out.dtype == torch.bfloat16, "ats_gather: a and a_out must be bf16")
    _chk(src, torch.int32, "src")
    _chk(x, torch.float32, "x"); _chk(x_out, torch.float32, "x_out")
    _chk(a, torch.bfloat16, "a"); _chk(a_out, torch.bfloat16, "a_out")
    D = 0 if x is None else x.shape[1]
    with _Timed("ats_gather", rows=rows, bytes=rows * (8 * D + 4 * ncols)):
        rc = lib().b200vit_ats_gather(_ptr(src), rows, _ptr(x), 0 if x is None else x.stride(0), _ptr(x_out),
                                      0 if x_out is None else x_out.stride(0), D, _ptr(a),
                                      0 if a is None else a.stride(0), _ptr(a_out),
                                      0 if a_out is None else a_out.stride(0), int(ncols), _stream())
    _check(rc, "b200vit_ats_gather")


def attention_kv_lens(q: torch.Tensor, kv: torch.Tensor, out: torch.Tensor, lens: torch.Tensor, B: int, Nq: int,
                      Nk: int, H: int, dh: int, scale: float) -> None:
    """attention_kv with image b attending over its first lens[b] keys (int32 [B] on the device, clamped to [1, Nk]):
    q[B*Nq, H*dh] (any row stride), kv[B*Nk, 2*H*dh] packed k | v (any row stride), out[B*Nq, H*dh]."""
    _rows2d(q, "attention_kv_lens: q")
    _rows2d(kv, "attention_kv_lens: kv")
    _need(tuple(q.shape) == (B * Nq, H * dh), f"attention_kv_lens: q must be [{B * Nq}, {H * dh}], got {tuple(q.shape)}")
    _need(tuple(kv.shape) == (B * Nk, 2 * H * dh),
          f"attention_kv_lens: kv must be [{B * Nk}, {2 * H * dh}], got {tuple(kv.shape)}")
    _need(out.is_contiguous() and tuple(out.shape) == (B * Nq, H * dh),
          f"attention_kv_lens: out must be contiguous [{B * Nq}, {H * dh}], got {tuple(out.shape)}")
    _need(lens.dtype == torch.int32 and lens.is_contiguous() and tuple(lens.shape) == (B,),
          f"attention_kv_lens: lens must be contiguous int32 [{B}], got {lens.dtype} {tuple(lens.shape)}")
    _chk(q, torch.bfloat16, "q"); _chk(kv, torch.bfloat16, "kv"); _chk(out, torch.bfloat16, "out")
    _chk(lens, torch.int32, "lens")
    with _Timed("attention_kv_lens", B=B, Nq=Nq, Nk=Nk, H=H, bytes=(q.numel() + kv.numel() + out.numel()) * 2,
                flops=4.0 * B * H * Nq * Nk * dh):
        rc = lib().b200vit_attention_kv_lens(_ptr(q), q.stride(0), _ptr(kv), kv.stride(0), _ptr(out), B, int(Nq),
                                             int(Nk), _ptr(lens), H, dh, float(scale), _stream())
    _check(rc, "b200vit_attention_kv_lens")
