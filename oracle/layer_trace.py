"""Every launch of TransformerEngine.run_blocks traced back to the reference layer  --  TEST INFRASTRUCTURE.

Whether the fused encoder computes what the reference module's forward defines splits into two questions that need no
error propagation through softmax, LayerNorm or GELU:

  provenance   every operand of every launch of a layer equals, bit for bit, the value the reference forward defines
               at that point: derived here from the module's own parameters (read through the attribute paths of
               the reference, `module_layers`) and from the snapshotted outputs of the launches before it -- the
               stream entering the layer, bf16(x), bf16(gamma W), ...  Row statistics are the one exception: they
               must be within the bound of the kernel that wrote them.  Scalars too: eps, softmax scale, heads,
               dim_head, mask_self, the key mask, the rotary table.  (`check_provenance`)
  accuracy     every output is within the fp64 bound its kernel already has, computed on the operands the kernel
               actually received.  (`expected`, `check_accuracy`)

Together they chain each layer back to the reference arithmetic: error enters only where the project chose it (the
bf16 operands, the folded LayerNorm's definition) and each kernel is held to its own bound.

The tracer (`trace`) wraps every _lib entry point run_blocks can reach, with the argument binding and the entry-point
list of tests/golden/make_engine_schedule.py; a launch is kept with its arguments, a clone of every tensor argument
taken before the call and a clone of every tensor it writes taken after it (the workspace buffers are overwritten
within a layer).  The clones go on the current stream.  `impl` runs a launch: the real kernels on the GPU, or
`emulate`, which writes the fp64 reference of `expected` rounded to the output's dtype, on a machine without one.  The
trace runs the per-kernel Python loop; the one-call C loop must be bit-identical to it.

The encoders that run outside a single run_blocks call are traced through their drivers (`trace_call`) and walked by
their own checks: CrossViT's two streams (`check_cross_vit_provenance`: each branch's layers, its final LayerNorm,
both class-attention directions), CaiT's and XCiT's forward_fused after the patch embedding
(`check_class_stage_provenance`: the patch encoder, the context, one CrossAttentionEngine.run against
`cross_module_layers`, the head), and LeViT's whole forward_fused (`check_levit_provenance`).

The ViT, SimpleViT-family, small-dataset ViT, DeepViT and NaViT forwards are walked from the pixels to the logits
(`check_forward_provenance`): the patch embedding in either patch mode, the token assembly, the layers, the final
LayerNorm, the pooling and the head, every operand read from the module's own attributes."""
from __future__ import annotations

import dataclasses
import inspect
import math
import os
import sys
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Tuple

import torch
from torch import nn

from oracle import attention_bounds as AB
from oracle import attention_fp32_bounds as FB
from oracle import bounds as Bd
from oracle import grid_attention_bounds as GB
from oracle import headmix_bounds as HB
from oracle import row_bounds as RB
from oracle import vit_oracle as O
from oracle.lpi_bounds import lpi_reference

Tensor = torch.Tensor
U = Bd.U
GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

# the tensors each entry point writes
OUTPUTS = {
    "gemm": ("out_f32", "out_bf16", "stats_out"),
    "gemm_headnorm": ("out_bf16",),
    "layernorm": ("out_f32", "out_bf16"),
    "rowstats_cast": ("xb", "stats"),
    "rope_qk": ("qkv",),
    "attention": ("out",),
    "attention_varlen": ("out",),
    "attention_axial": ("out",),
    "attention_headmix": ("out",),
    "attention_xca": ("out",),
    "local_patch_interaction": ("y", "y_bf16", "y_stats"),
    "gemm_act": ("out_f32", "out_bf16", "stats_out"),
    "conv_im2col_nhwc": ("out_bf16",),
    "attention_window": ("out",),
    "attention_window_relpos": ("out",),
    "attention_kv": ("out",),
    "attention_groups": ("out",),
    "conv_proj_dw": ("q_out", "kv_out"),
    "attention_kv_ex": ("out",),
    "attention_iwsa": ("out",),
    "attention_window_token": ("out", "tok_out"),
    "head_layernorm_gelu": ("buf",),
    "window_mix": ("out",),
    "attention_region_local": ("out",),
    "peg": ("y",),
    "attention_cls": ("out",),
    "attention_cls_headmix": ("out",),
    "attention_posbias": ("out",),
    "gemm_hardswish": ("out_bf16",),
    "mean_pool": ("out",),
    "cast_f32_bf16": ("out",),
    "conv_im2col_nchw": ("out_bf16",),
    "patch_embed_tma": ("stats", "out_f32"),
    "patchify_ln": ("out_bf16",),
    "patchify_spt_ln": ("out_bf16",),
    "patchify_nd": ("out_bf16",),
    "patchify_varlen_ln": ("out_bf16",),
    "embed_tokens": ("x", "xb", "stats"),
    "embed_tokens_grouped": ("x", "xb", "stats"),
    "embed_varlen": ("x", "xb", "stats"),
    "attn_pool": ("out",),
}
# the entry points of the attention records on token grids (engine.Windows, StridedKV, InteractiveWindows, ConvProj,
# PatchGroups, WindowTokenBlock, RegionLocalBlock), of the SiLU feed-forward block and of ScalableViT's positional
# encoding between two run_blocks calls, which make_engine_schedule.ENTRY_POINTS does not list
GRID_ENTRY_POINTS = ("gemm_act", "conv_im2col_nhwc", "attention_window", "attention_window_relpos", "attention_kv",
                     "attention_groups", "conv_proj_dw", "attention_kv_ex", "attention_iwsa", "attention_window_token",
                     "head_layernorm_gelu", "window_mix", "attention_region_local", "peg")
# the entry points of the class-token cross attention (engine.CrossAttentionEngine) and of LeViT's forward_fused
CLASS_ENTRY_POINTS = ("attention_cls", "attention_cls_headmix", "attention_posbias", "gemm_hardswish", "mean_pool",
                      "conv_im2col_nchw")
# the entry points of the patch embeddings, token assembly and NaViT's attention pooling (a whole forward_fused)
FRONT_ENTRY_POINTS = ("patch_embed_tma", "patchify_ln", "patchify_spt_ln", "patchify_nd", "patchify_varlen_ln",
                      "embed_tokens", "embed_tokens_grouped", "embed_varlen", "attn_pool")


def schedule():
    """tests/golden/make_engine_schedule.py: ENTRY_POINTS, Recorder, recording, CASES."""
    if GOLDEN not in sys.path:
        sys.path.insert(0, GOLDEN)
    import make_engine_schedule
    return make_engine_schedule


def f32(eps: float) -> float:
    """A Python float as the C ABI's float receives it."""
    return torch.tensor(eps, dtype=torch.float32).item()


# ------------------------------------------------------------------------------------------------------ tracing
@dataclass
class Launch:
    name: str
    args: dict                                    # bound arguments, the live objects
    pre: dict                                     # argument name -> clone before the call (tensors, tuples of them)
    post: dict = field(default_factory=dict)      # written argument name -> clone after the call


def _clone(v):
    if isinstance(v, torch.Tensor):
        return v.detach().clone()
    if isinstance(v, tuple):
        return tuple(_clone(e) for e in v)
    return v


def tracer(impl: Callable[[str, Callable], Callable]):
    """A make_engine_schedule.Recorder whose entry points run `impl(name, real)` and keep Launch records in
    `launches`."""
    S = schedule()

    class Tracer(S.Recorder):
        def __init__(self, eng, owners) -> None:
            super().__init__(eng, owners)
            self.launches: List[Launch] = []

        def recorder(self, name: str, real: Callable) -> Callable:
            sig, run = inspect.signature(real), impl(name, real)

            def call(*args, **kwargs):
                a = self.bind(sig, args, kwargs)
                rec = Launch(name, a, {k: _clone(v) for k, v in a.items()})
                run(**a)
                rec.post = {k: _clone(a[k]) for k in OUTPUTS.get(name, ()) if a.get(k) is not None}
                self.launches.append(rec)
            return call
    return Tracer


def real_impl(name: str, real: Callable) -> Callable:
    return real


def emulate_impl(name: str, real: Callable) -> Callable:
    """The launch emulated: its outputs get the fp64 reference of `expected`, rounded to their dtype.  An output that
    the reference on these operands does not fit (a wrong map size or stride passed with the right buffers) is
    written as NaN, so that the provenance walk, not the emulation, names the operand."""
    def run(**a):
        if name not in OUTPUTS:
            raise NotImplementedError(f"no emulation of _lib.{name}")
        pre = {k: _clone(v) for k, v in a.items()}
        got: Dict[str, Tensor] = {}

        def written(k, v):                        # expected() reads earlier outputs through `got`
            if v.numel() != a[k].numel():
                a[k].fill_(math.nan)
            else:
                a[k].copy_(v.reshape(a[k].shape).to(a[k].dtype))
            got[k] = a[k].detach().clone()
        expected(name, pre, got, on_output=written)
    return run


def trace(eng, x: Tensor, kw: dict, ln_mode: str, impl=real_impl, prime: Optional[Callable] = None,
          call: Optional[Callable[[], object]] = None) -> List[Launch]:
    """Run call() -- by default eng.run_blocks(x, **kw); a module's own driver of several run_blocks calls and the
    launches between them (ScalableViT's Transformer.run_fused) -- on the per-kernel loop in `ln_mode` with every
    launch traced.  In fold mode with kw['primed'], prime(x, xb, stats) first writes the workspace's bf16 copy of x and
    its row statistics (not traced), as an embedding kernel would; every other workspace buffer starts as NaN."""
    S = schedule()
    with S.recording(eng, S.caller_buffers(eng, x, kw), ln_mode, "python", extra_entry_points=GRID_ENTRY_POINTS,
                     recorder=tracer(impl)) as rec:
        for buf in eng.workspace(x.shape[0], x.device).values():      # a launch reading a stale buffer reads NaN
            buf.fill_(math.nan)
        if kw.get("primed"):
            xb, st = eng.entry_buffers(x.shape[0], x.device)
            if xb is not None:
                prime(x, xb, st)
        if call is None:
            eng.run_blocks(x, **kw)
        else:
            call()
    return rec.launches


def prime_exact(x: Tensor, xb: Tensor, stats: Tensor) -> None:
    """The embedding's bf16 copy of x and its row statistics, from their fp64 reference."""
    xb.copy_(x.bfloat16())
    stats.copy_(RB.row_stats_reference(xb)[0].view(stats.shape).float())


# ------------------------------------------------------------------------------------------------------ references
def rope_reference(qkv: Tensor, cs: Tensor, rows: int, H: int, dh: int) -> Tensor:
    """b200vit_rope_qk's arithmetic (GoldenGateRoPENd, vit_nd_rotary.py:79-96) on the packed buffer qkv[T, 3 H dh], in
    fp32: q and k of token t rotated by table row t % rows, v as it was."""
    T = qkv.shape[0]
    t = qkv.view(T, 3, H, dh).float()
    r = torch.arange(T, device=qkv.device) % rows
    c, s = cs[r][..., 0][:, None], cs[r][..., 1][:, None]
    a, b = t[:, :2, :, : dh // 2], t[:, :2, :, dh // 2:]
    out = qkv.view(T, 3, H, dh).clone()
    out[:, :2] = torch.cat((a * c - b * s, a * s + b * c), dim=-1).bfloat16()
    return out.view(T, -1)


def tma_patches(img: Tensor) -> Tensor:
    """The 16 x 16 patch rows [B n, C 256] of img [B, C, H, W] in the (c p1 p2) column order b200vit_patch_embed_tma
    reads the image in (the reference's Rearrange writes (p1 p2 c), vit.py:100)."""
    B, C, H, W = img.shape
    return img.reshape(B, C, H // 16, 16, W // 16, 16).permute(0, 2, 4, 1, 3, 5).reshape(-1, C * 256)


def spt_patches(img: Tensor, p: int) -> Tensor:
    """The (p1 p2 c) patch rows of cat(img, its four one-pixel shifts) over 5 C channels (vit_for_small_dataset.py:
    96-112), zero-filled shifts as F.pad makes them."""
    from vit_pytorch_b200.vit_for_small_dataset import SPT_SHIFTS
    xs = torch.cat([img] + [torch.nn.functional.pad(img, s) for s in SPT_SHIFTS], dim=1)
    return O.patchify(xs, p, p).reshape(-1, 5 * img.shape[1] * p * p)


def nd_patches(img: Tensor, patch) -> Tensor:
    """The (p0 .. p_{r-1} c) patch rows of img [B, C, S_0 .. S_{r-1}] (vit_nd.py's Rearrange), grid row-major."""
    B, C, *shape = img.shape
    r = len(shape)
    v = img.reshape(B, C, *[e for s, p in zip(shape, patch) for e in (s // p, p)])
    perm = [0] + [2 + 2 * i for i in range(r)] + [3 + 2 * i for i in range(r)] + [1]
    return v.permute(*perm).reshape(-1, C * math.prod(patch))


def varlen_patches(images, p: int) -> Tensor:
    """The (c p1 p2) patch rows of every image of a packed batch, in order (na_vit.py: _tokenise_row)."""
    rows = []
    for im in images:
        C, h, w = im.shape
        rows.append(im.reshape(C, h // p, p, w // p, p).permute(1, 3, 0, 2, 4).reshape(-1, C * p * p))
    return torch.cat(rows)


def _padded(rb: Tuple[Tensor, Tensor], width: int) -> Tuple[Tensor, Tensor]:
    """(ref, bound) of rows written with zero K padding up to `width` columns: the padding exactly 0."""
    pad = lambda t: torch.nn.functional.pad(t, (0, width - t.shape[1]))                 # noqa: E731
    return pad(rb[0]), pad(rb[1])


def _exact(v: Tensor) -> Tuple[Tensor, Tensor]:
    return v.double(), torch.zeros(v.shape, dtype=torch.float64, device=v.device)


def _stats(xb: Tensor, like: Tensor) -> Tuple[Tensor, Tensor]:
    """(ref, bound) of row statistics `like` ([M, 2], [M, 1, 2] or [M, parts, 2]) of the bf16 rows xb: one part, the
    emit_row_stats writers (rowstats_cast, the embedding, the local patch interaction); several, a GEMM's EPI_STATS."""
    parts = like.numel() // (2 * xb.shape[0])
    if parts == 1:
        r, b = RB.row_stats_reference(xb)
    else:
        r, b = Bd.stats_reference(xb, parts)
    return r.view(like.shape), b.view(like.shape)


def expected(name: str, a: dict, got: dict, on_output: Optional[Callable] = None, plain: Optional[Tensor] = None
             ) -> Dict[str, Tuple[Tensor, Tensor]]:
    """(ref, bound) of every output of launch `name` on its operands `a` (the clones taken before it), from the
    existing fp64 oracle of its kernel.  Outputs that derive from another output (a bf16 copy, row statistics) are
    referred to the kernel's own value of it in `got`.  on_output(name, ref) runs as each is made (the emulation
    writes it and adds it to `got`).  gemm_headnorm: `plain`, the same launch's bf16 output without the head norm
    (its norm is bounded on those values); the emulation rounds the GEMM's reference."""
    out: Dict[str, Tuple[Tensor, Tensor]] = {}

    def put(k, rb):
        out[k] = rb
        if on_output is not None:
            on_output(k, rb[0])

    if name in ("gemm", "gemm_headnorm"):
        w = a["w"]
        K = a.get("k") or w.shape[1]
        kw = dict(bias=a["bias"], ln_sums=a["ln_sums"], col_s=a["col_s"], ln_eps=f32(a["ln_eps"]))
        if name == "gemm":
            kw.update(resid=a["resid"], gelu=a["gelu"])
            if a["out_f32"] is not None:
                put("out_f32", Bd.gemm_reference(a["a"][:, :K], w[:, :K], **kw))
                if a["out_bf16"] is not None:       # the bf16 copy of the kernel's own fp32 result
                    put("out_bf16", _exact(got["out_f32"].bfloat16()))
            elif a["out_bf16"] is not None:
                put("out_bf16", Bd.gemm_reference(a["a"][:, :K], w[:, :K], bf16_out=True, **kw))
            if a["stats_out"] is not None:
                put("stats_out", _stats(got["out_bf16"], a["stats_out"]))
            return out
        ref, bnd = Bd.gemm_reference(a["a"][:, :K], w[:, :K], bf16_out=True, **kw)
        out["plain"] = (ref, bnd)
        p = ref.float().bfloat16() if plain is None else plain
        M, nh, dh = p.shape[0], a["norm_heads"], a["dh"]
        heads = p[:, :nh * dh].reshape(M, nh, dh)
        g = a["head_gamma"].view(nh, dh)
        eps = a["head_layernorm_eps"]
        r, b = RB.rmsnorm_heads_reference(heads, g) if eps is None else RB.layernorm_heads_reference(heads, g, f32(eps))
        ref, bnd = _exact(p)
        ref[:, :nh * dh], bnd[:, :nh * dh] = r.reshape(M, -1), b.reshape(M, -1)
        put("out_bf16", (ref, bnd))
        return out
    if name == "gemm_act":
        kw = dict(bias=a["bias"], ln_sums=a["ln_sums"], col_s=a["col_s"], ln_eps=f32(a["ln_eps"]))
        if a["act"] == "gelu":
            y, e = Bd.gemm_reference(a["a"], a["w"], gelu=True, **kw)
        else:
            y, e = GB.silu_bound(*Bd.gemm_reference(a["a"], a["w"], **kw))
        if a["out_f32"] is not None:
            put("out_f32", (y, e))
            if a["out_bf16"] is not None:
                put("out_bf16", _exact(got["out_f32"].bfloat16()))
        elif a["out_bf16"] is not None:
            put("out_bf16", (y, Bd.bf16_bound(y, e)))
        if a["stats_out"] is not None:
            put("stats_out", _stats(got["out_bf16"], a["stats_out"]))
        return out
    if name == "gemm_hardswish":
        put("out_bf16", Bd.gemm_reference(a["a"], a["w"], bias=a["bias"], hardswish=True, bf16_out=True))
        return out
    if name == "conv_im2col_nchw":
        col = GB.im2col_nchw_reference(a["img"], a["k"], a["s"], a["p"])
        put("out_bf16", _exact(torch.nn.functional.pad(col, (0, a["out_bf16"].shape[1] - col.shape[1]))))
        return out
    if name == "attention_cls":
        put("out", FB.cls_reference(a["qkv_self"], a["ctx"], a["rows_per_image"], a["first"], a["n"], a["H"], a["dh"],
                                    a["scale"]))
        return out
    if name == "attention_cls_headmix":
        put("out", FB.cls_headmix_reference(a["qkv_self"], a["ctx"], a["rows_per_image"], a["first"], a["n"], a["H"],
                                            a["dh"], a["scale"], a["pre"], a["post"]))
        return out
    if name == "attention_posbias":
        put("out", GB.posbias_reference(a["qkv"], a["table"], a["B"], a["F"], a["s"], a["H"], a["dk"], a["dv"],
                                        a["scale"], gelu=a["gelu_out"]))
        return out
    if name == "mean_pool":
        B, N, D = a["B"], a["N"], a["D"]
        flat = a["x"].reshape(-1)[:B * N * D]           # read at a row offset: the last rows past the view are not read
        flat = torch.nn.functional.pad(flat, (0, B * N * D - flat.numel()), value=math.nan)
        put("out", RB.mean_pool_reference(flat.view(B, N, D), N if a["n_pool"] is None else a["n_pool"]))
        return out
    if name == "cast_f32_bf16":
        put("out", _exact(a["x"].bfloat16()))
        return out
    if name == "conv_im2col_nhwc":
        col = GB.im2col_reference(a["x"], a["B"], a["H"], a["W"], a["k"], a["s"], a["p"])
        put("out_bf16", _exact(torch.nn.functional.pad(col, (0, a["out_bf16"].shape[1] - col.shape[1]))))
        return out
    if name == "attention_window":
        put("out", GB.window_reference(a["qkv"], a["B"], a["gh"], a["gw"], a["p"], a["H"], a["dh"], f32(a["scale"])))
        return out
    if name == "attention_window_relpos":
        put("out", GB.relpos_reference(a["qkv"], a["table"], a["B"], a["gh"], a["gw"], a["w"], a["grid"], a["H"],
                                       a["dh"], a["scale"]))
        return out
    if name == "attention_kv":
        put("out", GB.kv_reference(a["q"], a["kv"], a["B"], a["Nq"], a["Nk"], a["H"], a["dh"], f32(a["scale"])))
        return out
    if name == "attention_groups":
        put("out", GB.groups_reference(a["qkv"], a["B"], a["gh"], a["gw"], a["ph"], a["pw"], a["H"], a["dh"],
                                       f32(a["scale"])))
        return out
    if name == "conv_proj_dw":
        geo = (a["B"], a["h"], a["w"], a["k"])
        put("q_out", GB.conv_reference(a["x"], a["wq"], a["bq"], *geo, 1))
        put("kv_out", GB.conv_reference(a["x"], a["wkv"], a["bkv"], *geo, a["s"]))
        return out
    if name == "attention_kv_ex":
        put("out", GB.kv_ex_reference(a["q"], a["kv"], a["B"], a["Nq"], a["Nk"], a["H"], a["dk"], a["dv"],
                                      f32(a["scale"])))
        return out
    if name == "attention_iwsa":
        put("out", GB.iwsa_reference(a["qkv"], a["lim"], a["B"], a["gh"], a["gw"], a["wh"], a["ww"], a["H"], a["dk"],
                                     a["dv"], f32(a["scale"])))
        return out
    if name == "attention_window_token":
        r, b, tr, tb = GB.window_token_reference(a["qkv"], a["tok_qkv"], a["B"], a["gh"], a["gw"], a["p"], a["H"],
                                                 a["dh"], f32(a["scale"]))
        put("out", (r, b))
        if a["tok_out"] is not None:
            put("tok_out", (tr, tb))
        return out
    if name == "head_layernorm_gelu":                 # in place on the first nheads * dh columns of buf
        buf, n = a["buf"], a["nheads"] * a["dh"]
        r, b = GB.head_layernorm_gelu_reference(buf[:, :n], a["gamma"], a["beta"], a["nheads"], a["dh"], f32(a["eps"]))
        ref, bnd = _exact(buf)
        ref[:, :n], bnd[:, :n] = r.reshape(-1, n), b.reshape(-1, n)
        put("buf", (ref, bnd))
        return out
    if name == "window_mix":
        put("out", GB.mix_reference(a["wqk"], a["o"], a["B"], a["gh"], a["gw"], a["p"], a["H"], a["dh"],
                                    f32(a["scale"])))
        return out
    if name == "attention_region_local":
        put("out", GB.region_local_reference(a["qkv"], a["table"], a["B"], a["lh"], a["lw"], a["rh"], a["rw"], a["W"],
                                             a["H"], f32(a["scale"]), a["dh"]))
        return out
    if name == "peg":
        put("y", GB.peg_reference(a["x"], a["w"], a["bias"], a["B"], a["gh"], a["gw"], a["k"]))
        return out
    if name == "layernorm":
        kw = dict(row_index=a["row_index"], eps=f32(a["eps"]))
        if a["out_f32"] is not None:
            put("out_f32", RB.layernorm_reference(a["x"], a["gamma"], a["beta"], **kw))
        if a["out_bf16"] is not None:
            put("out_bf16", RB.layernorm_reference(a["x"], a["gamma"], a["beta"], bf16_out=True, **kw))
        return out
    if name == "rowstats_cast":
        put("xb", _exact(a["x"].bfloat16()))
        put("stats", _stats(got["xb"], a["stats"]))
        return out
    if name == "rope_qk":
        put("qkv", _exact(rope_reference(a["qkv"], a["cs"], a["rows"], a["H"], a["dh"])))
        return out
    if name == "attention":
        put("out", AB.qkv_attention_reference(a["qkv"], [a["N"]] * a["B"], a["H"], a["dh"], a["scale"],
                                              mask_self=a["mask_self"]))
        return out
    if name == "attention_varlen":
        lengths = a["cu_seqlens"].diff().tolist()
        put("out", AB.qkv_attention_reference(a["qkv"], lengths, a["H"], a["dh"], a["scale"],
                                              mask_self=a["mask_self"]))
        return out
    if name == "attention_axial":
        put("out", AB.axial_reference(a["qkv"], a["key_mask"], a["B"], a["L"], a["G"], a["H"], a["dh"], a["scale"],
                                      a["zero_masked_rows"]))
        return out
    if name == "attention_headmix":
        ref, bnd = HB.headmix_reference(a["qkv"], a["B"], a["N"], a["H"], a["dh"], a["scale"], a["pre"], a["post"],
                                        a["head_ln"])
        put("out", (ref.reshape(a["B"] * a["N"], -1), bnd.reshape(a["B"] * a["N"], -1)))
        return out
    if name == "attention_xca":
        put("out", FB.xca_reference(a["qkv"], a["tau"], a["B"], a["N"], a["H"], a["dh"]))
        return out
    if name == "local_patch_interaction":
        put("y", lpi_reference(a["x"], a["ln"], a["w1"], a["b1"], a["w2"], a["b2"], a["B"], a["gh"], a["gw"], a["k"]))
        if a["y_bf16"] is not None:
            put("y_bf16", _exact(got["y"].bfloat16()))
            put("y_stats", _stats(got["y_bf16"], a["y_stats"]))
        return out
    if name == "patch_embed_tma":                     # the patch statistics, then the LN-folded GEMM reading them
        rows = tma_patches(a["img"])
        put("stats", Bd.patch_stats_reference(rows))
        put("out_f32", Bd.gemm_reference(rows, a["w_perm"], bias=a["bias"], ln_sums=got["stats"], col_s=a["col_s"],
                                         ln_eps=f32(a["eps"])))
        return out
    if name in ("patchify_ln", "patchify_spt_ln", "patchify_varlen_ln"):
        if name == "patchify_ln":
            rows = O.patchify(a["img"], a["ph"], a["pw"])
            rows = rows.reshape(-1, rows.shape[-1])
        elif name == "patchify_spt_ln":
            rows = spt_patches(a["img"], a["p"])
        else:
            rows = varlen_patches(a["images"], a["p"])
        rb = Bd.layernorm_reference(rows, a["gamma"], a.get("beta"), f32(a["eps"]))
        put("out_bf16", _padded(rb, a["out_bf16"].shape[1]))
        return out
    if name == "patchify_nd":                         # a pure gather: exact
        put("out_bf16", _padded(_exact(nd_patches(a["img"], list(a["patch"]))), a["out_bf16"].shape[1]))
        return out
    if name in ("embed_tokens", "embed_tokens_grouped", "embed_varlen"):
        if name == "embed_varlen":
            ix = a["index"]
            dims = [tuple(d) for d in ix.dims.view(-1, 2).tolist()]
            put("x", RB.embed_varlen_reference(a["y"], a["gamma"], a["pos_h"], a["pos_w"], ix.lengths, dims, a["p"],
                                               f32(a["eps"])))
        elif name == "embed_tokens":                  # cls and pos: rows of D values, whatever their view's shape
            rows = lambda t: None if t is None else t.reshape(-1, a["y"].shape[1])              # noqa: E731
            put("x", RB.embed_tokens_reference(a["y"], a["gamma"], a["beta"], rows(a["cls"]), rows(a["pos"]), a["B"],
                                               a["n"], a["ncls"], tail=a["tail"], eps=f32(a["eps"])))
        else:
            put("x", RB.embed_tokens_reference(a["y"], a["gamma"], a["beta"], a["cls"], a["pos"], a["groups"], a["n"],
                                               a["ncls"], eps=f32(a["eps"]), pos_period=a["pos_period"],
                                               pos_stride=a["pos_stride"], cls_pos=a["cls_pos"]))
        if a["xb"] is not None:                       # the first layer's bf16 copy and row statistics
            put("xb", _exact(got["x"].bfloat16()))
            put("stats", _stats(got["xb"], a["stats"]))
        return out
    if name == "attn_pool":
        put("out", FB.navit_pool_reference(a["kv"], a["qn"], a["cu_seqlens"].diff().tolist(), a["H"], a["dh"]))
        return out
    raise NotImplementedError(f"no reference of _lib.{name}")


def launch_kind(c: Launch) -> str:
    """A short name of what the launch does, for the accuracy report."""
    if c.name == "gemm":
        a = c.args
        what = "ln-fold" if a["ln_sums"] is not None else "residual" if a["resid"] is not None else "plain"
        return f"gemm {what}{' gelu' if a['gelu'] else ''}"
    if c.name == "gemm_headnorm":
        return "gemm_headnorm " + ("ln" if c.args["head_layernorm_eps"] is not None else "rms")
    if c.name == "gemm_act":
        return f"gemm_act {'ln-fold ' if c.args['ln_sums'] is not None else ''}{c.args['act']}"
    if c.name == "attention_window_relpos":
        return f"attention_window_relpos {'dilated' if c.args['grid'] else 'block'}"
    return c.name


def check_accuracy(launches: List[Launch], what: str, rerun_plain: Optional[Callable] = None
                   ) -> Dict[str, float]:
    """Every traced output within its kernel's bound on the operands it received; worst |got - ref| / bound per
    launch kind.  rerun_plain(pre): the bf16 output of a gemm_headnorm launch's GEMM without the head norm."""
    worst: Dict[str, float] = {}
    for n, c in enumerate(launches):
        plain = rerun_plain(c.pre) if c.name == "gemm_headnorm" and rerun_plain is not None else None
        exp = expected(c.name, c.pre, c.post, plain=plain)
        kind = launch_kind(c)
        for k, (ref, bnd) in exp.items():
            got = plain if k == "plain" else c.post.get(k)
            if got is None:
                continue
            r = Bd.check(got.reshape(ref.shape), ref, bnd, f"{what}: launch {n} {kind}: {k}")
            worst[kind] = max(worst.get(kind, 0.0), r)
    return worst


# ------------------------------------------------------------------------------------------------------ module layers
@dataclass
class Ln:
    gamma: Tensor
    beta: Optional[Tensor]
    eps: float


def _ln(m: nn.Module) -> Ln:
    if isinstance(m, nn.LayerNorm):
        return Ln(m.weight, m.bias, m.eps)
    return Ln(m.gamma, None, 1e-5)              # NaViT's LayerNorm: F.layer_norm with gamma and a zero beta buffer


def _linears(seq: nn.Module) -> List[nn.Linear]:
    return [m for m in seq if isinstance(m, nn.Linear)]


def _out(attn: nn.Module) -> Optional[nn.Linear]:
    """to_out's Linear, None for the identity (heads == 1 and dim_head == dim, reference vit.py:46-49)."""
    o = attn.to_out
    if isinstance(o, nn.Identity):
        return None
    return o[0] if isinstance(o, nn.Sequential) else o


@dataclass
class RefLayer:
    """One layer of the reference module, read through the reference's own attribute paths.  The tensors are the
    module's parameters (concatenations where the reference projects q, k and v separately); the walk of
    check_provenance reads nothing else."""
    ln1: Ln
    qkv_w: Tensor
    out: Optional[Tuple[Tensor, Optional[Tensor]]]          # None: to_out is the identity
    ln2: Ln
    fc1: Tuple[Tensor, Tensor]
    fc2: Tuple[Tensor, Tensor]
    heads: int
    dim_head: int
    scale: float
    mask_self: bool = False
    qk: Optional[Tuple[str, Tensor, Tensor, float]] = None   # (kind 'rms' | 'ln', q gamma [H, dh], k gamma, eps)
    headmix: Optional[Tuple[Tensor, Optional[Tensor], Optional[Ln]]] = None   # (post, pre, LayerNorm over heads)
    tau: Optional[Tensor] = None                             # XCiT's temperature
    temporal: Optional[Tuple[Ln, Tensor, Optional[Tuple[Tensor, Optional[Tensor]]]]] = None  # (ln, qkv_w, out)
    out_scale: Optional[Tensor] = None
    ff_scale: Optional[Tensor] = None
    lpi: Optional[dict] = None                               # ln, conv1, bn, conv2, scale
    post_norm: bool = False
    cat: Tuple[str, ...] = ()                                # fields the engine gets as a concatenation, not `is`
    grid: Optional[dict] = None                              # the attention on the token grid, by `kind` (_grid_*)
    ff_act: str = "gelu"                                     # the feed-forward block's activation
    ff_first: bool = False                                   # the feed-forward block runs before the attention
    peg: Optional[nn.Conv2d] = None                          # the depthwise PEG convolution that runs after the layer


def _plain(attn, ff, qkv_w: Optional[Tensor] = None, scale: Optional[float] = None, **kw) -> RefLayer:
    """A pre-LN layer of `attn` (norm, to_qkv, to_out, heads, dim_head, scale) and `ff` (net: LayerNorm, Linear,
    ..., Linear); qkv_w / scale in place of the attention's own to_qkv / scale."""
    o = _out(attn)
    fc1, fc2 = _linears(ff.net)
    return RefLayer(ln1=_ln(attn.norm), qkv_w=attn.to_qkv.weight if qkv_w is None else qkv_w,
                    out=None if o is None else (o.weight, o.bias), ln2=_ln(ff.net[0]), fc1=(fc1.weight, fc1.bias),
                    fc2=(fc2.weight, fc2.bias), heads=attn.heads, dim_head=attn.dim_head,
                    scale=float(attn.scale) if scale is None else scale, **kw)


def _chan_ln(m: nn.Module) -> Ln:
    """The channel LayerNorm of an NCHW map (twins_svt.py:33-43, cvt.py:25-35): g and b of shape (1, dim, 1, 1)."""
    return Ln(m.g.reshape(-1), m.b.reshape(-1), m.eps)


def _conv_layer(attn: nn.Module, ff: nn.Sequential, qkv_w: Tensor, grid: dict, cat=()) -> RefLayer:
    """A layer of 1 x 1 convolutions over an NCHW map: `attn` (norm, to_out[0], heads, scale) and `ff` (channel
    LayerNorm, Conv2d, GELU, Dropout, Conv2d) (twins_svt.py:45-57, cvt.py:37-49)."""
    o, c1, c2 = attn.to_out[0], ff[1], ff[4]
    I, D = o.weight.shape[1], o.weight.shape[0]
    return RefLayer(ln1=_chan_ln(attn.norm), qkv_w=qkv_w, out=(o.weight.reshape(D, I), o.bias), ln2=_chan_ln(ff[0]),
                    fc1=(c1.weight.reshape(-1, D), c1.bias), fc2=(c2.weight.reshape(D, -1), c2.bias),
                    heads=attn.heads, dim_head=I // attn.heads, scale=float(attn.scale), grid=grid, cat=cat)


def padded_key_width(dk: int) -> int:
    """The width the key-head kernels (attention_kv_ex, attention_iwsa) are built for that runs a dim_key: dk rounded
    up to a multiple of 16."""
    return -(-dk // 16) * 16


def _padded_heads(w: Tensor, H: int, dp: int) -> Tensor:
    """w [H d, ...] with dp - d zero rows after each head's d rows: [H dp, ...].  A zero q or k column adds exactly 0
    to every score, so the padded heads' attention is the module's."""
    d, rest = w.shape[0] // H, tuple(w.shape[1:])
    out = torch.zeros((H, dp) + rest, dtype=w.dtype, device=w.device)
    out[:, :d] = w.detach().reshape((H, d) + rest)
    return out.reshape((H * dp,) + rest)


def _scalable_layers(mod: nn.Module) -> List[RefLayer]:
    """ScalableViT's Transformer (scalable_vit.py:214-236): each reference layer's modules [SSA, FeedForward, PEG,
    FeedForward, IWSA] run in that order (its loop binds the 4th, a FeedForward, to `iwsa` and the 5th to `ff2`): two
    layers, (SSA, FeedForward) and, feed-forward first, (FeedForward, IWSA); the first reference layer's PEG after the
    first.  The q and k heads run dim_key wide padded to padded_key_width; the softmax scale stays dim_key ** -0.5."""
    out = []
    for ssa, ff1, peg, ff2, iwsa in mod.layers:
        for a, ff, first in ((ssa, ff1, False), (iwsa, ff2, True)):
            H, D = a.heads, a.to_q.in_channels
            dk, dv = a.to_q.out_channels // H, a.to_v.out_channels // H
            dp = padded_key_width(dk)
            q = _padded_heads(a.to_q.weight.reshape(H * dk, D), H, dp)
            if a is ssa:                                    # scalable_vit.py:117-146: keys / values r x r, stride r
                qkv_w = q
                grid = dict(kind="strided", conv=a.to_k, kv=torch.cat((_padded_heads(a.to_k.weight, H, dp),
                                                                        a.to_v.weight.detach())), dv=dv)
            else:                                           # scalable_vit.py:149-196
                qkv_w = torch.cat((q, _padded_heads(a.to_k.weight.reshape(H * dk, D), H, dp),
                                   a.to_v.weight.detach().reshape(H * dv, D)))
                grid = dict(kind="iwsa", module=a, dv=dv)
            o, c1, c2 = a.to_out[0], ff.net[1], ff.net[4]
            out.append(RefLayer(
                ln1=_chan_ln(a.norm), qkv_w=qkv_w, out=(o.weight.reshape(D, H * dv), o.bias), ln2=_chan_ln(ff.net[0]),
                fc1=(c1.weight.reshape(-1, D), c1.bias), fc2=(c2.weight.reshape(D, -1), c2.bias), heads=H,
                dim_head=dp, scale=dk ** -0.5, grid=grid, cat=("qkv_w",), ff_first=first,
                peg=peg.proj if peg is not None and a is ssa else None))
    return out


def module_layers(mod: nn.Module) -> List[RefLayer]:
    """The layers of a reference Transformer, by family (the module's class)."""
    from vit_pytorch_b200 import (cait, cct, cross_vit, crossformer, cvt, deepvit, max_vit, mobile_vit, na_vit,
                                  na_vit_nested_tensor, nest, pit, regionvit, scalable_vit, sep_vit,
                                  simple_flash_attn_vit, simple_vit, simple_vit_with_qk_norm, twins_svt, vit,
                                  vit_for_small_dataset, vit_nd_rotary, vivit, xcit)
    t = type(mod)
    if t is scalable_vit.Transformer:
        return _scalable_layers(mod)
    if t is sep_vit.Transformer:                                            # sep_vit.py:208-235, DSSA :91-205
        out = []
        for a, ff in mod.layers:
            I, D = a.to_qkv.out_channels // 3, a.to_qkv.in_channels
            out.append(_conv_layer(a, ff.net, a.to_qkv.weight.reshape(3 * I, D), dict(kind="window_token", module=a)))
        return out
    if t is regionvit.R2LTransformer:                                       # regionvit.py:114-190
        out = []
        for a, ff in mod.layers:
            fc1, fc2 = _linears(ff)
            o = a.to_out[0]
            out.append(RefLayer(
                ln1=_ln(a.norm), qkv_w=a.to_qkv.weight, out=(o.weight, o.bias), ln2=_ln(ff[0]),
                fc1=(fc1.weight, fc1.bias), fc2=(fc2.weight, fc2.bias), heads=a.heads, dim_head=a.dim_head,
                scale=float(a.scale), grid=dict(kind="region_local", table=mod.local_rel_pos_bias.weight,
                                                window=mod.window_size)))
        return out
    if t is twins_svt.Transformer:                                          # twins_svt.py:159-176
        out = []
        for local_attn, ff1, global_attn, ff2 in mod.layers:
            if not isinstance(local_attn, nn.Identity):                     # LocalAttention, twins_svt.py:85-120
                a = local_attn.fn
                I, D = a.to_q.weight.shape[:2]
                out.append(_conv_layer(a, ff1.fn.net, torch.cat([a.to_q.weight, a.to_kv.weight]).reshape(3 * I, D),
                                       dict(kind="window", size=a.patch_size), cat=("qkv_w",)))
            a = global_attn.fn                                              # GlobalAttention, twins_svt.py:122-157
            I, D = a.to_q.weight.shape[:2]
            out.append(_conv_layer(a, ff2.fn.net, a.to_q.weight.reshape(I, D), dict(kind="strided", conv=a.to_kv)))
        return out
    if issubclass(t, max_vit._BlockAttention):                              # max_vit.py:262-273: block[2:4], [6:8]
        out = []
        for ai, fi, dilated in ((2, 3, False), (6, 7, True)):
            a, ff = mod.block[ai].fn, mod.block[fi].fn
            out.append(_plain(a, ff, grid=dict(kind="relpos", module=a, size=a.window_size, dilated=dilated,
                                               windows=mod.block[ai - 1])))
        return out
    if t is crossformer.Transformer:                                        # crossformer.py:167-199
        out = []
        for step in mod.layers:
            for a, ff in ((step[0], step[1]), (step[2], step[3])):         # Attention crossformer.py:101-165
                I, D = a.to_qkv.out_channels // 3, a.to_qkv.in_channels
                o, c1, c2 = a.to_out, ff[1], ff[4]
                out.append(RefLayer(
                    ln1=_chan_ln(a.norm), qkv_w=a.to_qkv.weight.reshape(3 * I, D),
                    out=(o.weight.reshape(D, I), o.bias), ln2=_chan_ln(ff[0]), fc1=(c1.weight.reshape(-1, D), c1.bias),
                    fc2=(c2.weight.reshape(D, -1), c2.bias), heads=a.heads, dim_head=I // a.heads, scale=float(a.scale),
                    grid=dict(kind="relpos", module=a, size=a.window_size, dilated=a.attn_type == "long", dpb=True)))
        return out
    if t is cvt.Transformer:                                                # cvt.py:99-112, Attention cvt.py:62-97
        out = []
        for a, ff in mod.layers:
            pq, pkv = a.to_q.net[2], a.to_kv.net[2]
            I, D = pq.weight.shape[:2]
            out.append(_conv_layer(a, ff.net, pq.weight.reshape(I, D),
                                   dict(kind="convproj", q=a.to_q.net, kv=a.to_kv.net,
                                        kv_w=pkv.weight.reshape(2 * I, D))))
        return out
    if t is mobile_vit.Transformer:                                         # mobile_vit.py:79-96, FeedForward :28-34
        return [dataclasses.replace(_plain(a, ff, grid=dict(kind="groups")), ff_act="silu") for a, ff in mod.layers]
    if t is vit.Transformer or t is pit.Transformer:                        # vit.py:66-83, pit.py:69-82
        return [_plain(attn, ff) for attn, ff in mod.layers]
    if t is simple_vit.Transformer or t is simple_flash_attn_vit.Transformer:
        # simple_vit.py:32-77, simple_flash_attn_vit.py:36-66: to_out a Linear without bias
        return [_plain(attn, ff) for attn, ff in mod.layers]
    if t is cross_vit.Transformer:                                          # cross_vit.py:34-90: to_q | to_kv
        return [_plain(attn, ff, qkv_w=torch.cat([attn.to_q.weight, attn.to_kv.weight]), cat=("qkv_w",))
                for attn, ff in mod.layers]
    if t is nest.Transformer:                                               # nest.py:84-104: 1 x 1 convs on NCHW
        out = []
        for attn, ff in mod.layers:
            I, D = attn.to_qkv.out_channels // 3, attn.to_qkv.in_channels
            out.append(_conv_layer(attn, ff.net, attn.to_qkv.weight.reshape(3 * I, D), None))
        return out
    if t is vit_nd_rotary.Transformer:                                      # vit_nd_rotary.py:115-156: to_qk | to_v
        return [_plain(attn, ff, qkv_w=torch.cat([attn.to_qk.weight, attn.to_v.weight]), cat=("qkv_w",))
                for attn, ff in mod.layers]
    if t is simple_vit_with_qk_norm.Transformer:                            # simple_vit_with_qk_norm.py:66-77
        return [_plain(attn, ff, qk=("rms", attn.q_norm.gamma, attn.k_norm.gamma, 0.0)) for attn, ff in mod.layers]
    if t is vit_for_small_dataset.Transformer:                              # LSA, vit_for_small_dataset.py:53-63
        return [_plain(attn, ff, scale=float(attn.temperature.detach().exp()), mask_self=True)
                for attn, ff in mod.layers]
    if t is na_vit.Transformer:                                             # na_vit.py:115-169: softmax scale 1
        out = []
        for attn, ff in mod.layers:
            fc1, fc2 = _linears(ff)
            H = attn.heads
            out.append(RefLayer(
                ln1=_ln(attn.norm), qkv_w=torch.cat([attn.to_q.weight, attn.to_kv.weight]),
                out=(attn.to_out[0].weight, attn.to_out[0].bias), ln2=_ln(ff[0]), fc1=(fc1.weight, fc1.bias),
                fc2=(fc2.weight, fc2.bias), heads=H, dim_head=attn.to_q.weight.shape[0] // H, scale=1.0,
                qk=("rms", attn.q_norm.gamma, attn.k_norm.gamma, 0.0), cat=("qkv_w",)))
        return out
    if t is na_vit_nested_tensor.Transformer:                               # na_vit_nested_tensor.py: q / k LayerNorm
        out = []
        for attn, ff in mod.layers:
            fc1, fc2 = _linears(ff)
            H, dh = attn.heads, attn.dim_head
            qn = attn.query_norm
            qk = None if isinstance(qn, nn.Identity) else \
                ("ln", qn.weight.expand(H, dh), attn.key_norm.weight.expand(H, dh), qn.eps)
            out.append(RefLayer(
                ln1=_ln(attn.norm), qkv_w=torch.cat([attn.to_queries.weight, attn.to_keys.weight,
                                                     attn.to_values.weight]),
                out=(attn.to_out.weight, attn.to_out.bias), ln2=_ln(ff[0]), fc1=(fc1.weight, fc1.bias),
                fc2=(fc2.weight, fc2.bias), heads=H, dim_head=dh, scale=dh ** -0.5, qk=qk, cat=("qkv_w", "qk")))
        return out
    if t is vivit.Transformer:                                              # vivit.py:75-89
        return [_plain(attn, ff) for attn, ff in mod.layers]
    if t is vivit.FactorizedTransformer:                                    # vivit.py:144-150
        out = []
        for sa, ta, ff in mod.layers:
            o = _out(ta)
            out.append(_plain(sa, ff, temporal=(_ln(ta.norm), ta.to_qkv.weight,
                                                None if o is None else (o.weight, o.bias))))
        return out
    if t is deepvit.Transformer:                                            # deepvit.py:40-75
        return [_plain(attn, ff, headmix=(attn.reattn_weights, None, _ln(attn.reattn_norm[1])))
                for attn, ff in mod.layers]
    if t is cait.Transformer:                                               # cait.py:31-45, 83-122
        out = []
        for ls_attn, ls_ff in mod.layers:
            attn, ff = ls_attn.fn, ls_ff.fn
            out.append(_plain(attn, ff, qkv_w=torch.cat([attn.to_q.weight, attn.to_kv.weight]),
                              headmix=(attn.mix_heads_post_attn, attn.mix_heads_pre_attn, None),
                              out_scale=ls_attn.scale, ff_scale=ls_ff.scale, cat=("qkv_w",)))
        return out
    if t is xcit.XCATransformer:                                            # xcit.py:109-167, 196-212
        out = []
        for ls_attn, ls_lpi, ls_ff in mod.layers:
            attn, net = ls_attn.fn, ls_lpi.fn.net
            lpi = dict(ln=_ln(net[0]), conv1=net[2], bn=net[3], conv2=net[5], scale=ls_lpi.scale)
            out.append(_plain(attn, ls_ff.fn, scale=1.0, tau=attn.temperature, out_scale=ls_attn.scale,
                              ff_scale=ls_ff.scale, lpi=lpi))
        return out
    if t is cct.TransformerClassifier:                                      # cct.py:84-111, 137-142
        out = []
        for blk in mod.blocks:
            a = blk.self_attn
            D = a.qkv.in_features
            out.append(RefLayer(
                ln1=_ln(blk.pre_norm), qkv_w=a.qkv.weight, out=(a.proj.weight, a.proj.bias), ln2=_ln(blk.norm1),
                fc1=(blk.linear1.weight, blk.linear1.bias), fc2=(blk.linear2.weight, blk.linear2.bias),
                heads=a.heads, dim_head=D // a.heads, scale=float(a.scale), post_norm=True))
        return out
    raise NotImplementedError(f"no reference layer table for {t.__module__}.{t.__name__}")


def _aliases(got: Tensor, want: Tensor) -> bool:
    """got views the same elements of the same storage as want (a reshape of the parameter, not a copy of it)."""
    return (got.untyped_storage().data_ptr() == want.untyped_storage().data_ptr()
            and got.storage_offset() == want.storage_offset() and got.stride() == want.stride())


def check_identity(mod: nn.Module, case: str = "") -> None:
    """Each EncoderLayer field the module describes to the engine IS the reference module's parameter (`is`, or a view
    of the same elements of its storage: the reshaped 1 x 1 convolutions and channel LayerNorms; equal values for the
    concatenations), so a swapped LayerNorm or a wrong layer index cannot hide behind a self-consistent
    description."""
    layers, _ = mod.encoder_layers()
    refs = module_layers(mod)
    if len(layers) != len(refs):
        raise AssertionError(f"{case}: encoder_layers() describes {len(layers)} layers, the module has {len(refs)}")

    def same(i, what, got, want, cat=False):
        if got is None and want is None:
            return
        ok = got is want or (got is not None and want is not None and got.shape == want.shape
                             and (cat or _aliases(got, want)) and torch.equal(got, want))
        if not ok:
            raise AssertionError(f"{case}: layer {i}: EncoderLayer.{what} is not the module's parameter")

    for i, (L, R) in enumerate(zip(layers, refs)):
        for nm, got, want in (("ln1", L.ln1, R.ln1), ("ln2", L.ln2, R.ln2)):
            same(i, f"{nm}.gamma", got.gamma, want.gamma)
            same(i, f"{nm}.beta", got.beta, want.beta)
        same(i, "qkv_w", L.qkv_w, R.qkv_w, "qkv_w" in R.cat)
        same(i, "out_w", L.out_w, None if R.out is None else R.out[0])
        same(i, "out_b", L.out_b, None if R.out is None else R.out[1])
        same(i, "fc1_w", L.fc1_w, R.fc1[0])
        same(i, "fc1_b", L.fc1_b, R.fc1[1])
        same(i, "fc2_w", L.fc2_w, R.fc2[0])
        same(i, "fc2_b", L.fc2_b, R.fc2[1])
        same(i, "out_scale", L.out_scale, R.out_scale)
        same(i, "ff_scale", L.ff_scale, R.ff_scale)
        if R.qk is not None:
            same(i, "qk_gamma[0]", L.qk_gamma[0], R.qk[1], "qk" in R.cat)
            same(i, "qk_gamma[1]", L.qk_gamma[1], R.qk[2], "qk" in R.cat)
        if R.headmix is not None:
            same(i, "attention.post", L.attention.post, R.headmix[0])
            same(i, "attention.pre", L.attention.pre, R.headmix[1])
            if R.headmix[2] is not None:
                same(i, "attention.ln.gamma", L.attention.ln.gamma, R.headmix[2].gamma)
                same(i, "attention.ln.beta", L.attention.ln.beta, R.headmix[2].beta)
        if R.tau is not None:
            same(i, "attention.tau", L.attention.tau, R.tau)
        if R.temporal is not None:
            T = L.temporal
            same(i, "temporal.ln.gamma", T.ln.gamma, R.temporal[0].gamma)
            same(i, "temporal.ln.beta", T.ln.beta, R.temporal[0].beta)
            same(i, "temporal.qkv_w", T.qkv_w, R.temporal[1])
            same(i, "temporal.out_w", T.out_w, None if R.temporal[2] is None else R.temporal[2][0])
            same(i, "temporal.out_b", T.out_b, None if R.temporal[2] is None else R.temporal[2][1])
        if R.lpi is not None:
            P, r = L.lpi, R.lpi
            for what, got, want in (("ln.gamma", P.ln.gamma, r["ln"].gamma), ("ln.beta", P.ln.beta, r["ln"].beta),
                                    ("conv1_w", P.conv1_w, r["conv1"].weight), ("conv1_b", P.conv1_b, r["conv1"].bias),
                                    ("bn_w", P.bn_w, r["bn"].weight), ("bn_b", P.bn_b, r["bn"].bias),
                                    ("bn_mean", P.bn_mean, r["bn"].running_mean),
                                    ("bn_var", P.bn_var, r["bn"].running_var),
                                    ("conv2_w", P.conv2_w, r["conv2"].weight), ("conv2_b", P.conv2_b, r["conv2"].bias),
                                    ("scale", P.scale, r["scale"])):
                same(i, f"lpi.{what}", got, want)
        if L.ff_first != R.ff_first:
            raise AssertionError(f"{case}: layer {i}: EncoderLayer.ff_first is {L.ff_first}, the module's feed-forward "
                                 f"block runs {'first' if R.ff_first else 'after the attention'}")
        g, A = R.grid or {}, L.attention
        kind = g.get("kind")
        if kind == "strided":                  # Twins-SVT's to_kv as it is, ScalableViT's padded to_k | to_v
            same(i, "attention.kv_w", A.kv_w, g.get("kv", g["conv"].weight), "kv" in g)
        elif kind == "iwsa":
            lim = g["module"].local_interactive_module
            same(i, "attention.lim_w", A.lim_w, lim.weight)
            same(i, "attention.lim_b", A.lim_b, lim.bias)
        elif kind == "window_token":
            m = g["module"]
            ln, conv = m.window_tokens_to_qk[0], m.window_tokens_to_qk[3]
            for what, got, want in (("token", A.token, m.window_tokens), ("ln.gamma", A.ln.gamma, ln.weight),
                                    ("ln.beta", A.ln.beta, ln.bias), ("wqk_w", A.wqk_w, conv.weight.reshape(
                                        conv.out_channels, conv.in_channels)), ("wqk_b", A.wqk_b, conv.bias)):
                same(i, f"attention.{what}", got, want)
        elif kind == "region_local":
            same(i, "attention.bias", A.bias, g["table"])


# ------------------------------------------------------------------------------------------------------ provenance
def _bits(t: Tensor) -> Tensor:
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float64: torch.int64}.get(
        t.dtype, t.dtype)) if t.dtype in (torch.float32, torch.bfloat16, torch.float64) else t


def _lpi_folded(P: dict, k: int):
    """(w1, b1, w2, b2) fp64 [k k, D] / [D] of the local patch interaction recomputed from the module's conv and
    BatchNorm parameters (xcit.py:150-167): BatchNorm (eval) into conv1, LayerScale into conv2; and (bound) the fp32
    rounding the host's fold may add: 5 u for w' = w g / sqrt(var + eps), 6 u |(b - mean) inv| + u |b1| for b1,
    u for each product with the scale."""
    d = lambda t: t.detach().double()                                                   # noqa: E731
    c1, bn, c2 = P["conv1"], P["bn"], P["conv2"]
    D = c1.weight.shape[0]
    zeros = torch.zeros(D, dtype=torch.float64, device=c1.weight.device)
    inv = d(bn.weight) / torch.sqrt(d(bn.running_var) + f32(bn.eps))
    w1 = (d(c1.weight).reshape(D, k * k) * inv[:, None]).t()
    cb = (d(c1.bias) if c1.bias is not None else zeros) - d(bn.running_mean)
    b1 = cb * inv + d(bn.bias)
    s = d(P["scale"]).reshape(D) if P["scale"] is not None else torch.ones_like(zeros)
    w2 = (d(c2.weight).reshape(D, k * k) * s[:, None]).t()
    b2 = (d(c2.bias) if c2.bias is not None else zeros) * s
    return [(w1, 5 * U * w1.abs()), (b1, 6 * U * (cb * inv).abs() + U * (b1.abs() + d(bn.bias).abs())),
            (w2, U * w2.abs()), (b2, U * b2.abs())]


def dpb_table_reference(attn: nn.Module) -> Tuple[Tensor, Tensor]:
    """(table, bound) fp64 [(2w-1)^2, heads] of CrossFormer's relative-position table (crossformer.py:195-215): the
    module's DynamicPositionBias evaluated in fp64 at the (2w+1)^2 offsets of _rel_offsets, the outputs that its
    rel_pos_indices (stride 2w-1) address -- the first (2w-1)^2 -- shared by the heads.  The bound is the error of the
    host's fp32 evaluation, carried layer by layer as a per-element bound e on the fp64 values v:
      Linear (K inputs)   e' = |W| e + (K + 2) u (|W| |v| + |b|)   (any order of the K fp32 products and sums);
      LayerNorm (D)       xhat = (v - mean) / sigma moves under a perturbation d of v by
                          (d_j - mean(d) - xhat_j mean(xhat d)) / sigma to first order (sigma = sqrt(var + eps) of the
                          fp64 input), so e' = |g| 1.01 (e + mean(e) + |xhat| mean(|xhat| e)) / sigma, the 1.01 for the
                          higher orders (e / sigma stays below 1e-4 here), plus (D + 8) u |g| (1 + |xhat|) + 2 u |v'|
                          for the mean, the variance's D-term sums, rsqrt and the products;
      ReLU                e' = e (1-Lipschitz, exact), 0 where v + e < 0 (both evaluations give exactly 0)."""
    from vit_pytorch_b200.crossformer import _rel_offsets
    w = attn.window_size
    d = lambda t: t.detach().double()                                                   # noqa: E731
    v = _rel_offsets(w, attn.rel_pos_indices.device).double()
    e = torch.zeros_like(v)
    for m in attn.dpb:
        if isinstance(m, nn.Linear):
            W, b = d(m.weight), d(m.bias)
            v, e = v @ W.t() + b, e @ W.abs().t() + (W.shape[1] + 2) * U * (v.abs() @ W.abs().t() + b.abs())
        elif isinstance(m, nn.LayerNorm):
            mu, var = v.mean(-1, keepdim=True), v.var(-1, unbiased=False, keepdim=True)
            sig = torch.sqrt(var + m.eps)
            xh = (v - mu) / sig
            v = xh * d(m.weight) + d(m.bias)
            g = d(m.weight).abs()
            dx = (e + e.mean(-1, keepdim=True) + xh.abs() * (xh.abs() * e).mean(-1, keepdim=True)) / sig
            e = g * 1.01 * dx + (v.shape[-1] + 8) * U * g * (1 + xh.abs()) + 2 * U * v.abs()
        elif isinstance(m, nn.ReLU):
            v, e = v.clamp_min(0), torch.where(v + e < 0, torch.zeros_like(e), e)
        else:
            v, e = m(v), m(e)
    n = (2 * w - 1) ** 2
    return v[:n, None].expand(-1, attn.heads), e[:n, None].expand(-1, attn.heads)


def _bn_folded(conv: nn.Conv2d, bn: nn.BatchNorm2d, tap_major: bool = True, bf16: bool = False):
    """((w, bound), (b, bound)) fp64 of a convolution with the BatchNorm (eval) after it folded in, recomputed from the
    module's parameters and its eps: w' = w g / sqrt(var + eps), b' = (b - mean) g / sqrt(var + eps) + beta, b the
    convolution's bias (0 without one).  w' [out, in k k], or tap_major [k k, out] (CvT's bias-free depthwise
    convolutions, cvt.py:51-60); LeViT's 1 x 1 convolutions take [out, in] (levit.py:92-108).  The bound is the fp32
    rounding the host's fold may add: 5 u for w' (the sum, sqrt, quotient and product), 5 u |(b - mean) inv| (6 u with
    the bias's subtraction) + u (|b'| + |beta|) for b'; bf16: w' then rounded to bf16."""
    d = lambda t: t.detach().double()                                                   # noqa: E731
    C = conv.weight.shape[0]
    inv = d(bn.weight) / torch.sqrt(d(bn.running_var) + f32(bn.eps))
    w = d(conv.weight).reshape(C, -1) * inv[:, None]
    if tap_major:
        w = w.t()
    cb = (d(conv.bias) if conv.bias is not None else torch.zeros_like(inv)) - d(bn.running_mean)
    b = cb * inv + d(bn.bias)
    wb = 5 * U * w.abs()
    return ((w, Bd.bf16_bound(w, wb) if bf16 else wb),
            (b, (6 if conv.bias is not None else 5) * U * (cb * inv).abs() + U * (b.abs() + d(bn.bias).abs())))


class ProvenanceError(AssertionError):
    pass


class Walk:
    """The provenance walk of one trace (check_provenance)."""

    def __init__(self, case: str, launches: List[Launch], fold: bool, kw: dict) -> None:
        self.case, self.calls, self.fold, self.kw = case, launches, fold, kw
        self.pos, self.where, self.cur = 0, "", None
        self.ratios: Dict[str, float] = {}            # operand -> worst |got - ref| / bound of its `within` checks
        self.have_stats = fold and bool(kw.get("primed"))
        # the statistics the next folded GEMM reads are the entry ones, one part per row (the prime or a rowstats_cast),
        # not a residual GEMM's
        self.entry_stats = self.have_stats

    # ---------------------------------------------------------------- failures and comparisons
    def fail(self, op: str, msg: str):
        c = self.cur
        launch = f"launch {self.pos - 1} {c.name}" if c is not None else "no launch"
        raise ProvenanceError(f"{self.case}: {self.where}: {launch}: operand {op}: {msg}")

    def take(self, *names: str) -> Launch:
        if self.pos >= len(self.calls):
            self.cur = None
            self.fail("-", f"the trace ended, {' or '.join(names)} expected")
        c = self.calls[self.pos]
        self.pos, self.cur = self.pos + 1, c
        if c.name not in names:
            self.fail("-", f"{' or '.join(names)} expected")
        return c

    def peek(self) -> Optional[str]:
        return self.calls[self.pos].name if self.pos < len(self.calls) else None

    def same(self, op: str, got, want) -> None:
        """Bit for bit (None only as None)."""
        if want is None or got is None:
            if got is not want:
                self.fail(op, f"got {'None' if got is None else 'a tensor'}, want "
                              f"{'None' if want is None else 'a tensor'}")
            return
        if got.dtype != want.dtype or tuple(got.shape) != tuple(want.shape):
            self.fail(op, f"got {got.dtype} {tuple(got.shape)}, want {want.dtype} {tuple(want.shape)}")
        want = want.to(got.device)
        bad = _bits(got.contiguous()) != _bits(want.contiguous())
        if bool(bad.any()):
            i = tuple(bad.nonzero()[0].tolist())
            self.fail(op, f"{int(bad.sum())} of {bad.numel()} elements differ, first at {i}: got {got[i].item()!r}, "
                          f"want {want[i].item()!r}")

    def within(self, op: str, got: Tensor, ref: Tensor, bound: Tensor) -> None:
        ref, bound = ref.to(got.device), bound.to(got.device)
        d = (got.double().reshape(ref.shape) - ref).abs()
        bad = ~(d <= bound)
        self.ratios[op] = max(self.ratios.get(op, 0.0), Bd.excess(got.reshape(ref.shape), ref, bound))
        if bool(bad.any()):
            i = tuple(bad.nonzero()[0].tolist())
            self.fail(op, f"{int(bad.sum())} of {bad.numel()} elements outside the bound, first at {i}: got "
                          f"{got.reshape(ref.shape)[i].item()!r}, want {ref[i].item()!r} +- {bound[i].item():.3e}")

    def value(self, op: str, got, want) -> None:
        if isinstance(want, float) and isinstance(got, (int, float)) and not isinstance(got, bool):
            ok = f32(got) == f32(want)
        else:
            ok = got == want and type(got) is type(want)
        if not ok:
            self.fail(op, f"got {got!r}, want {want!r}")

    def stats(self, op: str, got: Tensor, xb: Tensor) -> None:
        self.within(op, got, *_stats(xb, got))

    # ---------------------------------------------------------------- steps
    def entry_cast(self, S: Tensor) -> None:
        """rowstats_cast(S): the bf16 copy and the one-part row statistics the next folded GEMM reads."""
        c = self.take("rowstats_cast")
        self.same("x", c.pre["x"], S)
        self.have_stats = self.entry_stats = True

    def folded(self, a: dict, S: Tensor, ln: Ln, W: Tensor, b: Optional[Tensor]) -> None:
        """The operands of a LayerNorm-folded GEMM computing LN(S) W^T + b: bf16(S), its row statistics, gamma W,
        its column sums and W beta + b."""
        d = lambda t: t.detach().double()                                               # noqa: E731
        self.same("a", a["a"], S.bfloat16())
        self.stats("ln_sums", a["ln_sums"], a["a"])
        self.value("ln_eps", a["ln_eps"], float(ln.eps))
        wg = (d(W) * d(ln.gamma)[None]).float().bfloat16()
        self.same("w (gamma W)", a["w"], wg)
        K = W.shape[1]
        wd = wg.double()
        self.within("col_s", a["col_s"], wd.sum(1), K * U * wd.abs().sum(1))
        t = torch.zeros(W.shape[0], dtype=torch.float64, device=W.device)
        tb = torch.zeros_like(t)
        if ln.beta is not None:
            t, tb = d(W) @ d(ln.beta), d(W).abs() @ d(ln.beta).abs()
        if b is not None:
            t, tb = t + d(b), tb + d(b).abs()
        self.within("bias (W beta + b)", a["bias"], t, (K + 1) * U * tb)

    def normed(self, S: Tensor, ln: Ln, W: Tensor, b: Optional[Tensor], gelu: bool = False,
               head: Optional[tuple] = None, heads: int = 0, dh: int = 0, act: Optional[str] = None) -> Tensor:
        """out = LN(S) W^T + b (reference vit.py:19-21 / :52-54): the bf16 output of its GEMM; `act` "silu": the
        activation of gemm_act (MobileViT's FeedForward, mobile_vit.py:28-34)."""
        gemm = "gemm_headnorm" if head is not None else "gemm_act" if act is not None else "gemm"
        if self.fold:
            # a stream no launch has copied since it changed takes one rowstats_cast; without it the GEMM's operands
            # below show what it read instead
            if not self.have_stats and self.peek() == "rowstats_cast":
                self.entry_cast(S)
            c = self.take(gemm)
            a = c.pre
            self.folded(a, S, ln, W, b)
        else:
            c = self.take("layernorm")
            a = c.pre
            self.same("x", a["x"], S)
            self.same("gamma", a["gamma"], ln.gamma.detach().float())
            self.same("beta", a["beta"], None if ln.beta is None else ln.beta.detach().float())
            self.value("eps", a["eps"], float(ln.eps))
            self.same("row_index", a["row_index"], None)
            self.same("out_f32", a["out_f32"], None)
            xn = c.post["out_bf16"]
            c = self.take(gemm)
            a = c.pre
            self.same("a", a["a"], xn)
            self.same("w", a["w"], W.detach().bfloat16())
            self.same("bias", a["bias"], None if b is None else b.detach().float())
            self.same("ln_sums", a["ln_sums"], None)
        if act is not None:
            self.value("act", a["act"], act)
            self.same("out_f32", a["out_f32"], None)
            self.same("stats_out", a["stats_out"], None)
        elif head is None:
            self.value("gelu", a["gelu"], gelu)
            self.same("resid", a["resid"], None)
            self.same("out_f32", a["out_f32"], None)
        else:
            kind, gq, gk, eps = head
            self.same("head_gamma", a["head_gamma"], torch.cat([gq.detach().float().reshape(-1),
                                                                gk.detach().float().reshape(-1)]))
            self.value("norm_heads", a["norm_heads"], 2 * heads)
            self.value("dh", a["dh"], dh)
            self.value("head_layernorm_eps", a["head_layernorm_eps"], float(eps) if kind == "ln" else None)
        return c.post["out_bf16"]

    def residual(self, A: Tensor, out: Optional[Tuple[Tensor, Optional[Tensor]]], s: Optional[Tensor],
                 resid: Tensor, copy: bool, D: int) -> Tensor:
        """resid + (A W^T + b) s (reference vit.py:64,80-81; LayerScale cait.py:31-45): the new fp32 stream."""
        c = self.take("gemm")
        a = c.pre
        d = lambda t: t.detach().double()                                               # noqa: E731
        W, b = (None, None) if out is None else out
        Wd = torch.eye(D, dtype=torch.float64, device=resid.device) if W is None else d(W)
        bd = None if b is None else d(b)
        if s is not None:
            Wd, bd = Wd * d(s).reshape(-1, 1), None if bd is None else bd * d(s).reshape(-1)
        self.same("a", a["a"], A)
        self.same("w", a["w"], Wd.float().bfloat16())
        self.same("bias", a["bias"], None if bd is None else bd.float())
        self.same("resid", a["resid"], resid)
        self.same("ln_sums", a["ln_sums"], None)
        self.value("gelu", a["gelu"], False)
        if a["out_f32"] is None:
            self.fail("out_f32", "the residual GEMM writes no fp32 stream")
        new = c.post["out_f32"]
        if copy and self.fold:
            for op, what in (("out_bf16", "bf16 copy"), ("stats_out", "row statistics")):
                if a[op] is None:
                    self.fail(op, f"the stream's {what} the next folded GEMM reads is not written")
            self.same("out_bf16", c.post["out_bf16"], new.bfloat16())
            self.stats("stats_out", c.post["stats_out"], c.post["out_bf16"])
            self.have_stats, self.entry_stats = True, False
        else:
            self.same("out_bf16", a["out_bf16"], None)
            self.same("stats_out", a["stats_out"], None)
        return new

    def attention(self, R: RefLayer, qkv: Tensor, M: int, temporal: bool = False) -> Tensor:
        kw = self.kw
        axial = kw.get("axial")
        if R.headmix is not None:
            c = self.take("attention_headmix")
        elif R.tau is not None:
            c = self.take("attention_xca")
        elif temporal or (axial is not None and R.temporal is None):
            c = self.take("attention_axial")
        else:
            c = self.take("attention", "attention_varlen")
        a = c.pre
        self.same("qkv", a["qkv"], qkv)
        self.value("H", a["H"], R.heads)
        self.value("dh", a["dh"], R.dim_head)
        if c.name != "attention_xca":
            self.value("scale", a["scale"], float(R.scale))
        if c.name in ("attention", "attention_headmix", "attention_xca"):
            self.value("B", a["B"], kw["B"])
            self.value("N", a["N"], kw["N"])
        if c.name in ("attention", "attention_varlen"):
            self.value("mask_self", a["mask_self"], R.mask_self)
        if c.name == "attention_varlen":
            vl = kw.get("varlen")
            want = vl.cu if vl is not None else torch.arange(0, kw["B"] * kw["N"] + 1, kw["N"], dtype=torch.int32)
            self.same("cu_seqlens", a["cu_seqlens"], want.to(a["cu_seqlens"].device))
        if c.name == "attention_axial":
            G, T, km, zero = axial
            self.value("L", a["L"], T)
            self.value("G", a["G"], G)
            self.value("B", a["B"], M // (T * G))
            self.value("zero_masked_rows", a["zero_masked_rows"], zero)
            self.same("key_mask", a["key_mask"], km)
        if c.name == "attention_headmix":
            post, pre, hln = R.headmix
            self.same("post", a["post"], post.detach().float())
            self.same("pre", a["pre"], None if pre is None else pre.detach().float())
            if hln is None:
                self.value("head_ln", a["head_ln"], None)
            else:
                self.same("head_ln gamma", a["head_ln"][0], hln.gamma.detach().float())
                self.same("head_ln beta", a["head_ln"][1], hln.beta.detach().float())
                self.value("head_ln eps", a["head_ln"][2], float(hln.eps))
        if c.name == "attention_xca":
            tau = R.tau.detach().double().exp().reshape(-1)
            self.within("tau (exp temperature)", a["tau"], tau, 4 * U * tau)
        return c.post["out"]

    # ---------------------------------------------------------------- attention on the token grid
    def exact_ln(self, S: Tensor, ln: Ln) -> Tensor:
        """bf16(LN(S)) by the exact layernorm, in both modes: the normalised map a convolution reads."""
        c = self.take("layernorm")
        a = c.pre
        self.same("x", a["x"], S)
        self.same("gamma", a["gamma"], ln.gamma.detach().float())
        self.same("beta", a["beta"], None if ln.beta is None else ln.beta.detach().float())
        self.value("eps", a["eps"], float(ln.eps))
        self.same("row_index", a["row_index"], None)
        self.same("out_f32", a["out_f32"], None)
        return c.post["out_bf16"]

    def plain_gemm(self, A: Tensor, W: Tensor, b: Optional[Tensor] = None, gelu: bool = False) -> Tensor:
        """[GELU](A W^T + b) and no LayerNorm: a 1 x 1 convolution on a bf16 map, or a convolution on its im2col."""
        return self.prepared_gemm(A, W.detach().bfloat16(), None if b is None else b.detach().float(), gelu)

    def prepared_gemm(self, A: Tensor, W: Tensor, b: Optional[Tensor], gelu: bool = False, what: str = "w",
                      stats: bool = False) -> Tensor:
        """[GELU](A W^T + b) into a bf16 output alone, W and b as prepared (bf16, fp32), no LayerNorm and no residual;
        stats: with the row statistics of that output (a LayerNorm-folded GEMM reads them next)."""
        c = self.take("gemm")
        a = c.pre
        self.same("a", a["a"], A)
        self.same(what, a["w"], W)
        self.same("bias", a["bias"], b)
        for op in ("resid", "ln_sums", "out_f32"):
            self.same(op, a[op], None)
        self.value("gelu", a["gelu"], gelu)
        if not stats:
            self.same("stats_out", a["stats_out"], None)
        elif a["stats_out"] is None:
            self.fail("stats_out", "the row statistics the folded GEMM reads are not written")
        else:
            self.stats("stats_out", c.post["stats_out"], c.post["out_bf16"])
        return c.post["out_bf16"]

    def written_residual(self, A: Tensor, W: Tensor, b: Optional[Tensor], resid: Tensor) -> Tensor:
        """resid + A W^T + b with the prepared W (bf16) and b (fp32), written in fp32 and as its bf16 copy, with no row
        statistics (the cls rows of CrossAttentionEngine's stream A, LeViT's stream): the new fp32 rows."""
        c = self.take("gemm")
        a = c.pre
        self.same("a", a["a"], A)
        self.same("w", a["w"], W)
        self.same("bias", a["bias"], b)
        self.same("resid", a["resid"], resid)
        for op in ("ln_sums", "stats_out"):
            self.same(op, a[op], None)
        self.value("gelu", a["gelu"], False)
        if a["out_f32"] is None or a["out_bf16"] is None:
            self.fail("out_f32", "the cls rows and their bf16 copy are not both written")
        new = c.post["out_f32"]
        self.same("out_bf16", c.post["out_bf16"], new.bfloat16())
        return new

    def grid_geometry(self, a: dict, B: bool = True) -> None:
        gh, gw = self.kw["grid"]
        if B:
            self.value("B", a["B"], self.kw["B"])
        self.value("gh", a["gh"], gh)
        self.value("gw", a["gw"], gw)

    def heads(self, a: dict, R: RefLayer) -> None:
        self.value("H", a["H"], R.heads)
        self.value("dh", a["dh"], R.dim_head)
        self.value("scale", a["scale"], float(R.scale))

    def grid_attention(self, R: RefLayer, S: Tensor, i: int) -> Tuple[Tensor, Tensor]:
        """(the attention output of layer R on the stream S, by the kind of its attention on the grid; the stream,
        which RegionViT's region pass updates first)."""
        g, kind = R.grid, R.grid["kind"]
        if kind in ("window", "relpos", "groups"):
            qkv = self.normed(S, R.ln1, R.qkv_w, None)
            self.where = f"layer {i} attention"
            if kind == "window":                            # twins_svt.py:104-116: p x p blocks of the map
                c = self.take("attention_window")
                self.value("p", c.pre["p"], g["size"])
            elif kind == "relpos":                          # max_vit.py:247-272, block or dilated windows
                c = self.take("attention_window_relpos")
                self.value("w", c.pre["w"], g["size"])
                self.value("dilated", c.pre["grid"], g["dilated"])
                if g.get("dpb"):                            # crossformer.py:195-215: dpb at the offsets, host fp32
                    ref, bnd = dpb_table_reference(g["module"])
                    self.within("table (dpb)", c.pre["table"], ref.t(), bnd.t())
                else:
                    self.same("table", c.pre["table"], g["module"].rel_pos_bias.weight.detach().float().t())
            else:                                           # mobile_vit.py:150: strided patch groups
                c = self.take("attention_groups")
                ph, pw = self.kw["groups"]
                self.value("ph", c.pre["ph"], ph)
                self.value("pw", c.pre["pw"], pw)
            self.same("qkv", c.pre["qkv"], qkv)
            self.grid_geometry(c.pre)
            self.heads(c.pre, R)
            return c.post["out"], S
        if kind == "iwsa":
            return self.interactive_windows(R, S, i), S
        if kind == "window_token":
            return self.window_tokens(R, S, i), S
        if kind == "region_local":
            S = self.region_pass(R, S, i)
            qkv = self.normed(S, R.ln1, R.qkv_w, None)
            self.where = f"layer {i} attention"
            c = self.take("attention_region_local")
            a = c.pre
            self.same("qkv", a["qkv"], qkv)
            # regionvit.py:260-270: local_rel_pos_bias(bias_indices), whose table the kernel reads transposed
            self.same("table", a["table"], g["table"].detach().float().t())
            (lh, lw), (rh, rw) = self.kw["grid"], self.kw["regions"]
            self.value("B", a["B"], self.kw["B"])
            for op, v in (("lh", lh), ("lw", lw), ("rh", rh), ("rw", rw), ("W", g["window"])):
                self.value(op, a[op], v)
            self.heads(a, R)
            return c.post["out"], S
        gh, gw = self.kw["grid"]
        B = self.kw["B"]
        xn = self.exact_ln(S, R.ln1)
        if kind == "strided":       # twins_svt.py:140-157, scalable_vit.py:126-146: keys from a k x k, stride-k conv
            conv = g["conv"]
            k, s = conv.kernel_size[0], conv.stride[0]
            self.where = f"layer {i} queries"
            q = self.plain_gemm(xn, R.qkv_w)
            col = xn
            if k > 1:
                self.where = f"layer {i} key patches"
                c = self.take("conv_im2col_nhwc")
                a = c.pre
                self.same("x", a["x"], xn)
                self.value("B", a["B"], B)
                self.value("H", a["H"], gh)
                self.value("W", a["W"], gw)
                self.value("k", a["k"], k)
                self.value("s", a["s"], s)
                self.value("p", a["p"], conv.padding[0])
                col = c.post["out_bf16"]
            self.where = f"layer {i} keys and values"
            # the Conv2d weight (ScalableViT: to_k's, heads padded, then to_v's) in the im2col column order (tap row,
            # tap column, channel)
            kvw = g.get("kv", conv.weight)
            kv = self.plain_gemm(col, kvw.permute(0, 2, 3, 1).reshape(kvw.shape[0], -1))
            kh, kw = (gh + 2 * conv.padding[0] - k) // s + 1, (gw + 2 * conv.padding[1] - k) // s + 1
        else:                                               # cvt.py:51-60, 74-75: depthwise convs + BatchNorm, 1 x 1
            dq, bq, _ = g["q"]
            dkv, bkv, _ = g["kv"]
            k, s = dq.kernel_size[0], dkv.stride[0]
            self.where = f"layer {i} convolutional projection"
            if any(m.bias is not None for m in (dq, dkv, g["q"][2], g["kv"][2])):
                self.fail("-", "a convolution of the module's projections has a bias, which the fold drops")
            c = self.take("conv_proj_dw")
            a = c.pre
            self.same("x", a["x"], xn)
            for op, conv, bn in (("q", dq, bq), ("kv", dkv, bkv)):
                (w, wb), (b, bb) = _bn_folded(conv, bn)
                self.within(f"w{op} (BatchNorm folded)", a[f"w{op}"], w, wb)
                self.within(f"b{op} (BatchNorm folded)", a[f"b{op}"], b, bb)
            self.value("B", a["B"], B)
            self.value("h", a["h"], gh)
            self.value("w", a["w"], gw)
            self.value("k", a["k"], k)
            self.value("s", a["s"], s)
            if dq.stride[0] != 1 or dq.padding[0] != k // 2 or dkv.padding[0] != k // 2:
                self.fail("-", "the module's query convolution is not stride 1, or a padding is not k // 2")
            aq, akv = c.post["q_out"], c.post["kv_out"]
            self.where = f"layer {i} queries"
            q = self.plain_gemm(aq, R.qkv_w)
            self.where = f"layer {i} keys and values"
            kv = self.plain_gemm(akv, g["kv_w"])
            kh, kw = (gh + 2 * dkv.padding[0] - k) // s + 1, (gw + 2 * dkv.padding[1] - k) // s + 1
        self.where = f"layer {i} attention"
        c = self.take("attention_kv_ex" if "dv" in g else "attention_kv")
        a = c.pre
        self.same("q", a["q"], q)
        self.same("kv", a["kv"], kv)
        self.value("B", a["B"], B)
        self.value("Nq", a["Nq"], gh * gw)
        self.value("Nk", a["Nk"], kh * kw)
        if "dv" in g:                                       # ScalableViT: value heads of their own width
            self.value("H", a["H"], R.heads)
            self.value("dk", a["dk"], R.dim_head)
            self.value("dv", a["dv"], g["dv"])
            self.value("scale", a["scale"], float(R.scale))
        else:
            self.heads(a, R)
        return c.post["out"], S

    def interactive_windows(self, R: RefLayer, S: Tensor, i: int) -> Tensor:
        """ScalableViT's IWSA (scalable_vit.py:170-196): q | k | v of LN(S), the local interactive module (a 3 x 3
        convolution with bias) of the v map as im2col + GEMM, attention inside each window plus that term."""
        g = R.grid
        m, dv = g["module"], g["dv"]
        lim = m.local_interactive_module
        H, dp = R.heads, R.dim_head
        Ik, Iv = H * dp, H * dv
        (gh, gw), B = self.kw["grid"], self.kw["B"]
        qkv = self.normed(S, R.ln1, R.qkv_w, None)
        self.where = f"layer {i} local interactive module"
        c = self.take("conv_im2col_nhwc")
        a = c.pre
        self.same("x (the v columns of qkv)", a["x"], qkv[:, 2 * Ik:2 * Ik + Iv])
        self.value("B", a["B"], B)
        self.value("H", a["H"], gh)
        self.value("W", a["W"], gw)
        self.value("k", a["k"], lim.kernel_size[0])
        self.value("s", a["s"], lim.stride[0])
        self.value("p", a["p"], lim.padding[0])
        w = lim.weight
        lo = self.plain_gemm(c.post["out_bf16"], w.permute(0, 2, 3, 1).reshape(w.shape[0], -1), lim.bias)
        self.where = f"layer {i} attention"
        c = self.take("attention_iwsa")
        a = c.pre
        self.same("qkv", a["qkv"], qkv)
        self.same("lim", a["lim"], lo)
        self.grid_geometry(a)
        ws = m.window_size                                  # default(wsz, height), default(wsz, width)
        self.value("wh", a["wh"], gh if ws is None else ws)
        self.value("ww", a["ww"], gw if ws is None else ws)
        self.value("H", a["H"], H)
        self.value("dk", a["dk"], dp)
        self.value("dv", a["dv"], dv)
        self.value("scale", a["scale"], float(R.scale))
        return c.post["out"]

    def window_tokens(self, R: RefLayer, S: Tensor, i: int) -> Tensor:
        """SepViT's DSSA (sep_vit.py:168-219): the windows' attention with the window token, then, with more than one
        window, the window tokens' LayerNorm + GELU, their q | k projection and the attention across windows."""
        m = R.grid["module"]
        H, dh = R.heads, R.dim_head
        I, p = H * dh, m.window_size
        gh, gw = self.kw["grid"]
        qkv = self.normed(S, R.ln1, R.qkv_w, None)
        self.where = f"layer {i} attention"
        c = self.take("attention_window_token")
        a = c.pre
        self.same("qkv", a["qkv"], qkv)
        # the window token joins each window after the LayerNorm (sep_vit.py:175-184): to_qkv of the raw token, an
        # fp32 dot product of D terms rounded to bf16
        W, t = R.qkv_w.detach().double(), m.window_tokens.detach().double()
        ref = W @ t
        self.within("tok_qkv", a["tok_qkv"], ref, Bd.bf16_bound(ref, W.shape[1] * U * (W.abs() @ t.abs())))
        self.value("p", a["p"], p)
        self.grid_geometry(a)
        self.heads(a, R)
        o = c.post["out"]
        if (gh // p) * (gw // p) == 1:                      # sep_vit.py:202-203: no attention across windows
            self.same("tok_out", a["tok_out"], None)
            return o
        if a["tok_out"] is None:
            self.fail("tok_out", "the window tokens' outputs are not written")
        tok = c.post["tok_out"]
        self.where = f"layer {i} window tokens"
        c = self.take("head_layernorm_gelu")
        a = c.pre
        ln, act, conv = m.window_tokens_to_qk[0], m.window_tokens_to_qk[1], m.window_tokens_to_qk[3]
        if not isinstance(act, nn.GELU) or act.approximate != "none":
            self.fail("-", "the window tokens' activation is not the erf GELU the kernel computes")
        self.same("buf", a["buf"], tok)
        self.same("gamma", a["gamma"], ln.weight.detach().float())
        self.same("beta", a["beta"], ln.bias.detach().float())
        self.value("eps", a["eps"], float(ln.eps))
        self.value("nheads", a["nheads"], H)
        self.value("dh", a["dh"], dh)
        # the rows of the window tokens' q | k in the order window_mix reads (head h's q, then its k): the
        # convolution's output channels through the module's own _ChannelsToHeads and chunk(2, dim=-1)
        chan = torch.arange(2 * I, dtype=torch.float64).view(1, 2 * I, 1)
        wq, wk = m.window_tokens_to_qk[4](chan).chunk(2, dim=-1)          # [1, H, 1, dh] each
        order = torch.cat((wq, wk), -1).reshape(-1).long()
        wqk = self.plain_gemm(c.post["buf"], conv.weight.reshape(2 * I, I)[order.to(conv.weight.device)], conv.bias)
        self.where = f"layer {i} window mixing"
        c = self.take("window_mix")
        a = c.pre
        self.same("wqk", a["wqk"], wqk)
        self.same("o", a["o"], o)
        self.value("p", a["p"], p)
        self.grid_geometry(a)
        self.heads(a, R)
        return c.post["out"]

    def region_pass(self, R: RefLayer, S: Tensor, i: int) -> Tensor:
        """RegionViT's regional attention (regionvit.py:275): the layer's attention over each image's region tokens
        alone, with its residual, on the rows after the local ones; returns the stream with them updated.  In fold
        mode the region rows take the exact LayerNorm while the statistics are the entry ones (their one part per
        row is not read at a row offset), then a rowstats_cast of the new rows; after a residual GEMM wrote them, the
        folded QKV reads them and the region residual writes the new ones."""
        Ml = self.kw["B"] * self.kw["N"]
        rh, rw = self.kw["regions"]
        Sr = S[Ml:]
        self.where = f"layer {i} region qkv"
        if self.fold and not self.have_stats and self.peek() == "rowstats_cast":
            self.entry_cast(S)
        gemm_stats = self.fold and not self.entry_stats
        if gemm_stats:
            c = self.take("gemm")
            a = c.pre
            self.folded(a, Sr, R.ln1, R.qkv_w, None)
            for op in ("resid", "out_f32", "stats_out"):
                self.same(op, a[op], None)
            self.value("gelu", a["gelu"], False)
            qkv = c.post["out_bf16"]
        else:
            qkv = self.plain_gemm(self.exact_ln(Sr, R.ln1), R.qkv_w)
        self.where = f"layer {i} region attention"
        c = self.take("attention")
        a = c.pre
        self.same("qkv", a["qkv"], qkv)
        self.value("B", a["B"], self.kw["B"])
        self.value("N", a["N"], rh * rw)
        self.value("mask_self", a["mask_self"], False)
        self.heads(a, R)
        self.where = f"layer {i} region out"
        new = self.residual(c.post["out"], R.out, R.out_scale, Sr, copy=gemm_stats, D=S.shape[1])
        if self.fold and not gemm_stats:
            self.where = f"layer {i} region statistics"
            self.entry_cast(new)
        return torch.cat((S[:Ml], new))

    def feed_forward(self, R: RefLayer, S: Tensor, i: int) -> Tensor:
        """S + fc2(act(fc1(LN2(S)))): the new stream."""
        self.where = f"layer {i} fc1"
        act = None if R.ff_act == "gelu" else R.ff_act
        h = self.normed(S, R.ln2, R.fc1[0], R.fc1[1], gelu=act is None, act=act)
        self.where = f"layer {i} fc2"
        return self.residual(h, R.fc2, R.ff_scale, S, copy=True, D=S.shape[1])

    def peg(self, conv: nn.Conv2d, S: Tensor, i: int) -> Tensor:
        """y = S + conv(S), the depthwise PEG (scalable_vit.py:85-91, 313-314) between two layers, into a new stream;
        in fold mode a rowstats_cast of y then primes the next run_blocks call."""
        self.where = f"layer {i} positional encoding"
        c = self.take("peg")
        a = c.pre
        k, C = conv.kernel_size[0], conv.out_channels
        if conv.groups != C or conv.stride[0] != 1 or conv.padding[0] != k // 2:
            self.fail("-", "the PEG is not a depthwise k x k convolution at stride 1 with padding k // 2")
        self.same("x", a["x"], S)
        self.same("w (tap major)", a["w"], conv.weight.detach().float().reshape(C, k * k).t())
        self.same("bias", a["bias"], conv.bias.detach().float() if conv.bias is not None else
                  torch.zeros(C, dtype=torch.float32, device=S.device))
        self.grid_geometry(a)
        self.value("k", a["k"], k)
        y = c.post["y"]
        self.have_stats = False                 # the bf16 copy and statistics are S's
        if self.fold and self.peek() == "rowstats_cast":
            self.entry_cast(y)
        return y

    def lpi(self, R: RefLayer, S: Tensor) -> Tensor:
        """y = S + LPI(S) (xcit.py:150-167, 208-211)."""
        c = self.take("local_patch_interaction")
        a, P = c.pre, R.lpi
        k = P["conv1"].kernel_size[0]
        self.same("x", a["x"], S)
        self.same("ln gamma", a["ln"][0], P["ln"].gamma.detach().float())
        self.same("ln beta", a["ln"][1], P["ln"].beta.detach().float())
        self.value("ln eps", a["ln"][2], float(P["ln"].eps))
        for op, (ref, bnd) in zip(("w1", "b1", "w2", "b2"), _lpi_folded(P, k)):
            self.within(op, a[op], ref, bnd)
        grid = self.kw["grid"]
        self.value("B", a["B"], self.kw["B"])
        self.value("gh", a["gh"], grid[0])
        self.value("gw", a["gw"], grid[1])
        self.value("k", a["k"], k)
        y = c.post["y"]
        if self.fold:
            self.same("y_bf16", c.post.get("y_bf16"), y.bfloat16())
            self.stats("y_stats", c.post["y_stats"], c.post["y_bf16"])
            self.have_stats, self.entry_stats = True, False
        else:
            self.same("y_bf16", a["y_bf16"], None)
        return y

    def post_norm(self, R: RefLayer, S: Tensor) -> Tuple[Tensor, Tensor]:
        """x = LN2(x); h = GELU(fc1(x)) (cct.py:137-142): (the new stream, h)."""
        c = self.take("layernorm")
        a = c.pre
        self.same("x", a["x"], S)
        self.same("gamma", a["gamma"], R.ln2.gamma.detach().float())
        self.same("beta", a["beta"], R.ln2.beta.detach().float())
        self.value("eps", a["eps"], float(R.ln2.eps))
        if a["out_f32"] is None or a["out_bf16"] is None:
            self.fail("out_f32", "the post-norm writes the stream and its bf16 copy")
        y, yb = c.post["out_f32"], c.post["out_bf16"]
        c = self.take("gemm")
        a = c.pre
        self.same("a", a["a"], yb)
        self.same("w", a["w"], R.fc1[0].detach().bfloat16())
        self.same("bias", a["bias"], R.fc1[1].detach().float())
        self.value("gelu", a["gelu"], True)
        self.same("ln_sums", a["ln_sums"], None)
        self.have_stats = False
        return y, c.post["out_bf16"]


def walk_blocks(w: Walk, mod: nn.Module, x0: Tensor) -> Tensor:
    """The launches of one run_blocks(x0, **w.kw) call on the layers of `mod`, from w.pos on, walked in the reference
    forward's order (reference vit.py:78-81 and the family lines cited in module_layers); returns the fp32 stream the
    last launch wrote (x0 when no layer runs)."""
    kw = w.kw
    refs = module_layers(mod)
    S = x0
    M, D = x0.shape
    rope = kw.get("rope")
    run = kw.get("layers")
    for i in (range(len(refs)) if run is None else run):
        R = refs[i]
        w.where = f"layer {i} qkv"
        if R.grid is not None:
            if R.ff_first:                                     # scalable_vit.py:316-317
                S = w.feed_forward(R, S, i)
                w.where = f"layer {i} qkv"
            o, S = w.grid_attention(R, S, i)
            w.where = f"layer {i} out"
            S = w.residual(o, R.out, R.out_scale, S, copy=True, D=D)
            if not R.ff_first:
                S = w.feed_forward(R, S, i)
            if R.peg is not None:
                S = w.peg(R.peg, S, i)
            continue
        head = None if R.qk is None else R.qk
        qkv = w.normed(S, R.ln1, R.qkv_w, None, head=head, heads=R.heads, dh=R.dim_head)
        if rope is not None:                                   # vit_nd_rotary.py:143-147
            w.where = f"layer {i} rope"
            c = w.take("rope_qk")
            w.same("qkv", c.pre["qkv"], qkv)
            w.same("cs", c.pre["cs"], rope[0])
            w.value("rows", c.pre["rows"], rope[1])
            w.value("H", c.pre["H"], R.heads)
            w.value("dh", c.pre["dh"], R.dim_head)
            qkv = c.post["qkv"]
        w.where = f"layer {i} attention"
        o = w.attention(R, qkv, M)
        w.where = f"layer {i} out"
        S = w.residual(o, R.out, R.out_scale, S, copy=R.lpi is None and not R.post_norm, D=D)
        if R.temporal is not None:                             # vivit.py:144-150
            ln, tw, tout = R.temporal
            w.where = f"layer {i} temporal qkv"
            tq = w.normed(S, ln, tw, None)
            w.where = f"layer {i} temporal attention"
            to = w.attention(R, tq, M, temporal=True)
            w.where = f"layer {i} temporal out"
            S = w.residual(to, tout, None, S, copy=True, D=D)
        Y = S
        if R.lpi is not None:
            w.where = f"layer {i} local patch interaction"
            Y = w.lpi(R, S)
        if R.post_norm:
            w.where = f"layer {i} post-norm fc1"
            Y, h = w.post_norm(R, S)
        else:
            w.where = f"layer {i} fc1"
            h = w.normed(Y, R.ln2, R.fc1[0], R.fc1[1], gelu=True)
        w.where = f"layer {i} fc2"
        S = w.residual(h, R.fc2, R.ff_scale, Y, copy=True, D=D)
    return S


def _end(w: Walk) -> int:
    """Every launch walked: the number of launches; else a failure naming the first one left."""
    if w.pos != len(w.calls):
        w.where, w.cur = "after the last layer", w.calls[w.pos]
        w.pos += 1
        w.fail("-", "a launch the reference forward does not define")
    return w.pos


def check_provenance(mod: nn.Module, x0: Tensor, kw: dict, launches: List[Launch], ln_mode: str,
                     case: str = "") -> int:
    """Walk the trace of run_blocks(x0, **kw) through the layers of the reference module `mod` in its forward's
    order (walk_blocks) and assert every launch received what that forward defines.  Returns the number of launches
    checked; raises ProvenanceError naming the case, the layer, the launch, the operand and the first differing
    element."""
    check_identity(mod, case)
    w = Walk(case, launches, ln_mode == "fold", kw)
    walk_blocks(w, mod, x0)
    return _end(w)


# ------------------------------------------------------------------------------------------------------ class attention
def trace_call(call: Callable[[], object], ln_mode: str, impl=real_impl, setup: Optional[Callable[[], None]] = None
               ) -> List[Launch]:
    """Run call() -- a driver of several engines' launches: CrossViT's fused_two_streams, a CrossAttentionEngine.run,
    LeViT.forward_fused -- in `ln_mode` with every launch traced; setup() first, inside the tracing (it fills the
    workspaces the call will use with NaN)."""
    S = schedule()
    with S.recording(None, lambda: [], ln_mode, "python",
                     extra_entry_points=GRID_ENTRY_POINTS + CLASS_ENTRY_POINTS + FRONT_ENTRY_POINTS,
                     recorder=tracer(impl)) as rec:
        if setup is not None:
            setup()
        call()
    return rec.launches


@dataclass
class RefCross:
    """One class-attention layer of a reference module (CrossLayer's reference), read through its own attribute
    paths: the cls rows of stream A attend to [LN(project_in(cls)); context rows of stream B]."""
    proj_in: Optional[nn.Linear]
    ln: Ln
    q_w: Tensor
    kv_w: Tensor
    out: Tuple[Tensor, Optional[Tensor]]
    proj_out: Optional[nn.Linear]
    heads: int
    dim_head: int
    scale: float
    skip: int                                     # leading rows of each image of B that are not context
    talking: Optional[Tuple[Tensor, Tensor]] = None          # (pre, post), [input head, output head]
    out_scale: Optional[Tensor] = None
    ff: Optional[Tuple[Ln, nn.Linear, nn.Linear]] = None
    ff_scale: Optional[Tensor] = None


def cross_module_layers(mod: nn.Module, direction: int = 0) -> List[RefCross]:
    """The class-attention layers of a reference module, by family: CrossViT's CrossTransformer (direction 0: sm cls
    attends to lg, 1: lg cls attends to sm), CaiT's and XCiT's class-attention Transformer."""
    from vit_pytorch_b200 import cait, cross_vit, xcit
    t = type(mod)
    out = []
    if t is cross_vit.CrossTransformer:                     # cross_vit.py:94-130: context = the patch rows t[:, 1:]
        for layer in mod.layers:
            pio = layer[direction]
            a = pio.fn
            pin = None if isinstance(pio.project_in, nn.Identity) else pio.project_in
            pout = None if isinstance(pio.project_out, nn.Identity) else pio.project_out
            out.append(RefCross(pin, _ln(a.norm), a.to_q.weight, a.to_kv.weight, (a.to_out[0].weight, a.to_out[0].bias),
                                pout, a.heads, a.dim_head, float(a.scale), skip=1))
        return out
    if t is cait.Transformer or t is xcit.Transformer:      # cait.py:61-122, xcit.py:72-107, 169-189: every row
        for ls_attn, ls_ff in mod.layers:
            a, ff = ls_attn.fn, ls_ff.fn
            talking = (a.mix_heads_pre_attn, a.mix_heads_post_attn) if t is cait.Transformer else None
            fc1, fc2 = _linears(ff.net)
            out.append(RefCross(None, _ln(a.norm), a.to_q.weight, a.to_kv.weight,
                                (a.to_out[0].weight, a.to_out[0].bias), None, a.heads, a.dim_head, float(a.scale),
                                skip=0, talking=talking, out_scale=ls_attn.scale, ff=(_ln(ff.net[0]), fc1, fc2),
                                ff_scale=ls_ff.scale))
        return out
    raise NotImplementedError(f"no reference class-attention table for {t.__module__}.{t.__name__}")


def _scaled(W: Tensor, b: Optional[Tensor], s: Optional[Tensor]) -> Tuple[Tensor, Optional[Tensor]]:
    """bf16(W s) and fp32 b s of a Linear whose output is scaled by LayerScale s (cait.py:31-45), from fp64."""
    d = lambda t: t.detach().double()                                                   # noqa: E731
    Wd, bd = d(W), None if b is None else d(b)
    if s is not None:
        Wd, bd = Wd * d(s).reshape(-1, 1), None if bd is None else bd * d(s).reshape(-1)
    return Wd.float().bfloat16(), None if bd is None else bd.float()


def _cls_rows(S: Tensor, B: int, N: int) -> Tensor:
    return S.view(B, N, -1)[:, 0]


def _with_cls(S: Tensor, B: int, N: int, cls: Tensor) -> Tensor:
    out = S.clone()
    out.view(B, N, -1)[:, 0] = cls
    return out


def walk_cross(w: Walk, mod: nn.Module, direction: int, xa: Tensor, xba: Tensor, Na: int, xbb: Tensor, Nb: int,
               B: int, layers: Optional[List[int]] = None, tag: str = "") -> Tuple[Tensor, Tensor]:
    """The launches of one CrossAttentionEngine.run from w.pos on, against the class-attention layers of the reference
    module `mod`: stream A fp32 xa [B Na, D_A] and its bf16 copy xba, stream B's bf16 copy xbb [B Nb, D_B] (the keys and
    values); `layers` the indices run.  Returns A's stream and its bf16 copy with the new cls rows."""
    refs = cross_module_layers(mod, direction)
    d = lambda t: t.detach().double()                                                   # noqa: E731
    w.where = f"{tag}context"
    # cross_vit.py:65 / cait.py:91: to_kv of the raw context rows, every layer's in one GEMM over all of B's rows
    ctx = w.prepared_gemm(xbb, torch.cat([R.kv_w.detach() for R in refs]).bfloat16(), None,
                          what="w (every layer's to_kv)")
    rows = torch.arange(0, B * Na, Na, dtype=torch.int32)
    for i in (range(len(refs)) if layers is None else layers):
        R = refs[i]
        I = R.heads * R.dim_head
        Wqkv = torch.cat([R.q_w, R.kv_w])
        cls, clsb = _cls_rows(xa, B, Na), _cls_rows(xba, B, Na)
        w.where = f"{tag}layer {i} qkv"
        if R.proj_in is not None:                           # cross_vit.py:104-107: project_in, then the LayerNorm
            w.where = f"{tag}layer {i} project_in"
            qin = w.prepared_gemm(clsb, R.proj_in.weight.detach().bfloat16(), R.proj_in.bias.detach().float(),
                                  stats=True)
            w.where = f"{tag}layer {i} qkv"
            c = w.take("gemm")
            a = c.pre
            w.folded(a, qin, R.ln, Wqkv, None)
            for op in ("resid", "out_f32", "stats_out"):
                w.same(op, a[op], None)
            w.value("gelu", a["gelu"], False)
            qkv = c.post["out_bf16"]
        else:                                               # the LayerNorm of A's fp32 cls rows
            c = w.take("layernorm")
            a = c.pre
            w.same("x", a["x"], xa)
            w.same("gamma", a["gamma"], R.ln.gamma.detach().float())
            w.same("beta", a["beta"], R.ln.beta.detach().float())
            w.value("eps", a["eps"], float(R.ln.eps))
            w.same("row_index (the cls rows)", a["row_index"], rows.to(xa.device))
            w.same("out_f32", a["out_f32"], None)
            qkv = w.plain_gemm(c.post["out_bf16"], Wqkv)
        w.where = f"{tag}layer {i} attention"
        c = w.take("attention_cls_headmix" if R.talking is not None else "attention_cls")
        a = c.pre
        w.same("qkv_self", a["qkv_self"], qkv)
        w.same("ctx (the layer's to_kv columns)", a["ctx"], ctx[:, 2 * I * i:2 * I * (i + 1)])
        w.value("rows_per_image", a["rows_per_image"], Nb)
        w.value("first", a["first"], R.skip)
        w.value("n", a["n"], Nb - R.skip)
        w.value("H", a["H"], R.heads)
        w.value("dh", a["dh"], R.dim_head)
        w.value("scale", a["scale"], float(R.scale))
        if R.talking is not None:                           # cait.py:95-97: pre before the softmax, post after it
            w.same("pre", a["pre"], R.talking[0].detach().float())
            w.same("post", a["post"], R.talking[1].detach().float())
        o = c.post["out"]
        Wo, bo = _scaled(R.out[0], R.out[1], R.out_scale)
        if R.proj_out is not None:
            w.where = f"{tag}layer {i} out"
            y = w.prepared_gemm(o, Wo, bo)
            w.where = f"{tag}layer {i} project_out"
            new = w.written_residual(y, R.proj_out.weight.detach().bfloat16(), R.proj_out.bias.detach().float(), cls)
        else:
            w.where = f"{tag}layer {i} out"
            new = w.written_residual(o, Wo, bo, cls)
        xa, xba = _with_cls(xa, B, Na, new), _with_cls(xba, B, Na, new.bfloat16())
        if R.ff is not None:                                # cait.py:120-121: x = ff(x) + x on the cls rows
            ln, fc1, fc2 = R.ff
            w.where = f"{tag}layer {i} ff LayerNorm"
            c = w.take("layernorm")
            a = c.pre
            w.same("x", a["x"], xa)
            w.same("gamma", a["gamma"], ln.gamma.detach().float())
            w.same("beta", a["beta"], ln.beta.detach().float())
            w.value("eps", a["eps"], float(ln.eps))
            w.same("row_index (the cls rows)", a["row_index"], rows.to(xa.device))
            w.same("out_f32", a["out_f32"], None)
            w.where = f"{tag}layer {i} fc1"
            h = w.plain_gemm(c.post["out_bf16"], fc1.weight, fc1.bias, gelu=True)
            w.where = f"{tag}layer {i} fc2"
            W2, b2 = _scaled(fc2.weight, fc2.bias, R.ff_scale)
            new = w.written_residual(h, W2, b2, _cls_rows(xa, B, Na))
            xa, xba = _with_cls(xa, B, Na, new), _with_cls(xba, B, Na, new.bfloat16())
    return xa, xba


def check_class_stage_provenance(model: nn.Module, x0: Tensor, B: int, grid: Tuple[int, int], launches: List[Launch],
                                 ln_mode: str, case: str = "") -> int:
    """Walk the trace of CaiT's or XCiT's forward_fused after its patch embedding (cait.py:246-255, xcit.py:380-393):
    the patch encoder's layers on the embedded stream x0 [B N, D] of the (h, w) patch `grid` (walk_blocks, the layers its kept_layers() names),
    the context the class attention reads -- CaiT: bf16 of the encoder's output (the cast of it in exact mode), XCiT:
    its final_norm -- then the class-attention layers (walk_cross: the cls token of every image attends to
    [LN(cls); context], cls_transformer.kept_layers()), and the head's LayerNorm and Linear on the cls rows.  The number
    of launches checked."""
    from vit_pytorch_b200 import xcit
    is_xcit = isinstance(model, xcit.XCiT)
    enc = model.xcit_transformer if is_xcit else model.patch_transformer
    fold = ln_mode == "fold"
    check_identity(enc, case)
    N = grid[0] * grid[1]
    kw = dict(B=B, N=N, primed=fold, layers=enc.kept_layers())
    if is_xcit:
        kw["grid"] = grid
    w = Walk(case, launches, fold, kw)
    S = walk_blocks(w, enc, x0)
    w.where = "context"
    if is_xcit:                                             # xcit.py:388: final_norm of the patch rows
        fn = model.final_norm
        w.where = "context (final_norm)"
        c = w.take("layernorm")
        a = c.pre
        w.same("x", a["x"], S)
        w.same("gamma", a["gamma"], fn.weight.detach().float())
        w.same("beta", a["beta"], fn.bias.detach().float())
        w.value("eps", a["eps"], float(fn.eps))
        for op in ("row_index", "out_f32"):
            w.same(op, a[op], None)
        ctx = c.post["out_bf16"]
    else:                                                   # cait.py:252: the patch rows as they leave the encoder
        if not fold:
            c = w.take("cast_f32_bf16")
            w.same("x", c.pre["x"].reshape(S.shape), S)
        ctx = S.bfloat16()
    D = S.shape[1]
    cls = model.cls_token.detach().reshape(1, D).float().expand(B, D).contiguous()
    clsb = torch.full((B, D), math.nan, dtype=torch.bfloat16, device=S.device)
    w2 = Walk(case, launches, fold, {})
    w2.pos = w.pos
    cls, _ = walk_cross(w2, model.cls_transformer, 0, cls, clsb, 1, ctx, N, B,
                        layers=model.cls_transformer.kept_layers())
    w2.where = "head"                                       # cait.py:255 / xcit.py:393: mlp_head(x[:, 0])
    ln, lin = model.mlp_head[0], model.mlp_head[1]
    c = w2.take("layernorm")
    a = c.pre
    w2.same("x (the cls rows)", a["x"], cls)
    w2.same("gamma", a["gamma"], ln.weight.detach().float())
    w2.same("beta", a["beta"], ln.bias.detach().float())
    w2.value("eps", a["eps"], float(ln.eps))
    for op in ("row_index", "out_f32"):
        w2.same(op, a[op], None)
    w2.prepared_gemm(c.post["out_bf16"], lin.weight.detach().bfloat16(), lin.bias.detach().float())
    return _end(w2)


def check_cross_vit_provenance(mse: nn.Module, xs: Tensor, xl: Tensor, B: int, Ns: int, Nl: int, primed: bool,
                               launches: List[Launch], ln_mode: str, case: str = "") -> int:
    """Walk the trace of CrossViT's MultiScaleEncoder (engine.fused_two_streams; reference cross_vit.py:134-162): per
    block, each branch's encoder layers (walk_blocks), its final LayerNorm, which replaces the stream, then the
    sm-attends-lg and lg-attends-sm class attention (walk_cross) on the updated streams."""
    fold = ln_mode == "fold"
    x, xb, N = [xs, xl], [None, None], (Ns, Nl)
    pos = 0
    for k, (sm_enc, lg_enc, cross) in enumerate(mse.layers):
        for b, enc in enumerate((sm_enc, lg_enc)):
            branch = f"block {k} {'sm' if b == 0 else 'lg'} "
            check_identity(enc, case + " | " + branch)
            w = Walk(case, launches, fold, dict(B=B, N=N[b], primed=primed and k == 0))
            w.pos = pos
            S = walk_blocks(w, enc, x[b])
            w.where = branch + "final LayerNorm"                    # cross_vit.py:90: replaces the stream
            c = w.take("layernorm")
            a = c.pre
            w.same("x", a["x"], S)
            w.same("gamma", a["gamma"], enc.norm.weight.detach().float())
            w.same("beta", a["beta"], enc.norm.bias.detach().float())
            w.value("eps", a["eps"], float(enc.norm.eps))
            w.same("row_index", a["row_index"], None)
            if a["out_f32"] is None or a["out_bf16"] is None:
                w.fail("out_f32", "the final LayerNorm writes the new stream and its bf16 copy")
            x[b], xb[b] = c.post["out_f32"], c.post["out_bf16"]
            w.same("out_bf16", xb[b], x[b].bfloat16())
            pos = w.pos
        for direction, (A, Bs) in enumerate(((0, 1), (1, 0))):
            w = Walk(case, launches, fold, {})
            w.pos = pos
            x[A], xb[A] = walk_cross(w, cross, direction, x[A], xb[A], N[A], xb[Bs], N[Bs], B,
                                     tag=f"block {k} {('sm attends lg', 'lg attends sm')[direction]} ")
            pos = w.pos
    w = Walk(case, launches, fold, {})
    w.pos = pos
    return _end(w)


# ------------------------------------------------------------------------------------------------------ LeViT
def check_levit_provenance(mod: nn.Module, img: Tensor, launches: List[Launch], case: str = "") -> int:
    """Walk the trace of LeViT.forward_fused(img) through the reference LeViT (levit.py:27-195): the four stride-2
    convolutions of conv_embedding as im2col + GEMM; per Transformer layer the QKV GEMM of [to_q; to_k; to_v] with
    their BatchNorms folded (the module's eps), the position-bias attention (the bias table pos_bias.weight^T / scale,
    the module's pos_indices against the kernel's |s i - y| F + |s j - x| on the key grid, the stride of to_q), the
    to_out GEMM with its BatchNorm folded onto the residual or into a fresh stream, the Hardswish fc1 and the fc2
    residual; then the mean over the map, its bf16 cast and the [mlp_head; distill_head] GEMM.  The number of launches
    checked."""
    from vit_pytorch_b200 import levit
    w = Walk(case, launches, False, {})
    d = lambda t: t.detach().double()                                                   # noqa: E731
    B = img.shape[0]
    src = img.contiguous()
    H, W = img.shape[2:]
    S = Sb = None
    for i, conv in enumerate(mod.conv_embedding):                  # levit.py:153-158
        w.where = f"conv_embedding {i}"
        k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        c = w.take("conv_im2col_nchw" if i == 0 else "conv_im2col_nhwc")
        a = c.pre
        if i == 0:
            w.same("img", a["img"], src)
        else:
            w.same("x", a["x"], src)
            w.value("B", a["B"], B)
            w.value("H", a["H"], H)
            w.value("W", a["W"], W)
        w.value("k", a["k"], k)
        w.value("s", a["s"], s)
        w.value("p", a["p"], p)
        col = c.post["out_bf16"]
        # the weight in the gather's column order, (channel, tap) of the image, (tap, channel) of a channels-last map
        cw = conv.weight.detach() if i == 0 else conv.weight.detach().permute(0, 2, 3, 1)
        cw = cw.reshape(conv.out_channels, -1)
        cw = torch.nn.functional.pad(cw, (0, col.shape[1] - cw.shape[1])).bfloat16()
        c = w.take("gemm")
        a = c.pre
        w.same("a", a["a"], col)
        w.same("w", a["w"], cw)
        w.same("bias", a["bias"], conv.bias.detach().float())
        for op in ("resid", "ln_sums", "stats_out"):
            w.same(op, a[op], None)
        w.value("gelu", a["gelu"], False)
        H, W = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
        if i + 1 < len(mod.conv_embedding):
            w.same("out_f32", a["out_f32"], None)
            src = c.post["out_bf16"]
        else:
            if a["out_f32"] is None:
                w.fail("out_f32", "the last convolution writes no fp32 stream")
            S, Sb = c.post["out_f32"], c.post["out_bf16"]
            w.same("out_bf16", Sb, S.bfloat16())
    F_ = H
    for ti, tr in enumerate(mod.backbone):
        for li, (attn, ff) in enumerate(tr.layers):
            tag = f"transformer {ti} layer {li}"
            w.where = f"{tag} qkv"
            Hh = attn.heads
            dk, dv = attn.to_q[0].out_channels // Hh, attn.to_v[0].out_channels // Hh
            s = attn.to_q[0].stride[0]
            c = w.take("gemm")
            a = c.pre
            w.same("a", a["a"], Sb)
            parts = [_bn_folded(seq[0], seq[1], tap_major=False, bf16=True)
                     for seq in (attn.to_q, attn.to_k, attn.to_v)]
            w.within("w ([to_q; to_k; to_v], BatchNorm folded)", a["w"], torch.cat([p_[0][0] for p_ in parts]),
                     torch.cat([p_[0][1] for p_ in parts]))
            w.within("bias (BatchNorm folded)", a["bias"], torch.cat([p_[1][0] for p_ in parts]),
                     torch.cat([p_[1][1] for p_ in parts]))
            for op in ("resid", "ln_sums", "out_f32", "stats_out"):
                w.same(op, a[op], None)
            w.value("gelu", a["gelu"], False)
            qkv = c.post["out_bf16"]
            w.where = f"{tag} attention"
            c = w.take("attention_posbias")
            a = c.pre
            w.same("qkv", a["qkv"], qkv)
            # levit.py:110-136: pos_bias(pos_indices) / scale added to the scores; the kernel reads table[h][index]
            tbl = d(attn.pos_bias.weight).t() / f32(attn.scale)
            w.within("table (pos_bias^T / scale)", a["table"], tbl, 2 * U * tbl.abs())
            want = GB.posbias_index(F_, s, attn.pos_indices.device)
            if tuple(attn.pos_indices.shape) != tuple(want.shape) or not torch.equal(attn.pos_indices, want):
                w.fail("table (pos_indices)", f"the module's pos_indices {tuple(attn.pos_indices.shape)} are not the "
                                              f"kernel's |s i - y| F + |s j - x| (F {F_}, s {s}) of shape "
                                              f"{tuple(want.shape)}")
            w.value("B", a["B"], B)
            w.value("F", a["F"], F_)
            w.value("s (to_q's stride)", a["s"], s)
            w.value("H", a["H"], Hh)
            w.value("dk", a["dk"], dk)
            w.value("dv", a["dv"], dv)
            w.value("scale", a["scale"], float(attn.scale))
            w.value("gelu_out", a["gelu_out"], isinstance(attn.to_out[0], nn.GELU))
            o = c.post["out"]
            Fq = -(-F_ // s)
            w.where = f"{tag} out"
            c = w.take("gemm")
            a = c.pre
            w.same("a", a["a"], o)
            (ow, owb), (ob, obb) = _bn_folded(attn.to_out[1], attn.to_out[2], tap_major=False, bf16=True)
            w.within("w (to_out, BatchNorm folded)", a["w"], ow, owb)
            w.within("bias (BatchNorm folded)", a["bias"], ob, obb)
            w.same("resid", a["resid"], S if tr.attn_residual else None)     # levit.py:178-179
            for op in ("ln_sums", "stats_out"):
                w.same(op, a[op], None)
            w.value("gelu", a["gelu"], False)               # the GELU runs before to_out (attention_posbias)
            if a["out_f32"] is None or a["out_bf16"] is None:
                w.fail("out_f32", "the stream and its bf16 copy are not both written")
            S, Sb = c.post["out_f32"], c.post["out_bf16"]
            w.same("out_bf16", Sb, S.bfloat16())
            F_ = Fq
            w.where = f"{tag} fc1"
            fc1, act, fc2 = ff.net[0], ff.net[1], ff.net[3]
            if not isinstance(act, nn.Hardswish):
                w.fail("-", "the feed-forward activation is not the Hardswish the GEMM epilogue computes")
            c = w.take("gemm_hardswish")
            a = c.pre
            w.same("a", a["a"], Sb)
            w.same("w", a["w"], fc1.weight.detach().reshape(fc1.out_channels, -1).bfloat16())
            w.same("bias", a["bias"], fc1.bias.detach().float())
            h = c.post["out_bf16"]
            w.where = f"{tag} fc2"
            # levit.py:180: x = ff(x) + x, the bf16 copy written beside it
            S = w.written_residual(h, fc2.weight.detach().reshape(fc2.out_channels, -1).bfloat16(),
                                   fc2.bias.detach().float(), S)
            Sb = S.bfloat16()
    w.where = "head"                                                # levit.py:174-195
    D = S.shape[1]
    c = w.take("mean_pool")
    a = c.pre
    w.same("x", a["x"], S)
    w.value("B", a["B"], B)
    w.value("N", a["N"], F_ * F_)
    w.value("D", a["D"], D)
    w.value("n_pool", a["n_pool"], None)
    pm = c.post["out"]
    c = w.take("cast_f32_bf16")
    w.same("x", c.pre["x"], pm)
    pooled = c.post["out"]
    heads = [mod.mlp_head] + ([mod.distill_head] if isinstance(mod.distill_head, nn.Linear) else [])
    w.prepared_gemm(pooled, torch.cat([h_.weight.detach() for h_ in heads]).bfloat16(),
                    torch.cat([h_.bias.detach().float() for h_ in heads]), what="w ([mlp_head; distill_head])")
    return _end(w)



# ------------------------------------------------------------------------------------------------------ whole forwards
def _d(t: Tensor) -> Tensor:
    return t.detach().double()


def _f(t: Optional[Tensor]) -> Optional[Tensor]:
    return None if t is None else t.detach().float()


def _layernorm_launch(w: Walk, x: Tensor, ln: Ln, *, f32_out: bool = False, row_index: Optional[Tensor] = None
                      ) -> Tensor:
    """One b200vit_layernorm of the rows x (row_index: of those rows) with the LayerNorm ln: its bf16 output, or with
    f32_out its fp32 one (and no bf16 output)."""
    c = w.take("layernorm")
    a = c.pre
    w.same("x", a["x"], x)
    w.same("gamma", a["gamma"], _f(ln.gamma))
    w.same("beta", a["beta"], _f(ln.beta))
    w.value("eps", a["eps"], float(ln.eps))
    w.same("row_index", a["row_index"], None if row_index is None else row_index.to(x.device))
    if f32_out:
        w.same("out_bf16", a["out_bf16"], None)
        if a["out_f32"] is None:
            w.fail("out_f32", "the LayerNorm's fp32 output is not written")
        return c.post["out_f32"]
    w.same("out_f32", a["out_f32"], None)
    return c.post["out_bf16"]


def _head_gemm(w: Walk, A: Tensor, lin: nn.Linear, what: str) -> Tensor:
    """logits = A W^T + b of the classifier Linear `lin` into a bf16 output (engine.HeadEngine)."""
    return w.prepared_gemm(A, lin.weight.detach().bfloat16(), _f(lin.bias), what=f"w ({what})")


def _mean_pool(w: Walk, x: Tensor, B: int, N: int, n_pool: Optional[int], D: Optional[int] = None) -> Tensor:
    """mean_pool of the rows x (a flat view: read from a row offset, D its width)."""
    c = w.take("mean_pool")
    a = c.pre
    w.same("x", a["x"], x)
    w.value("B", a["B"], B)
    w.value("N", a["N"], N)
    w.value("D", a["D"], x.shape[1] if D is None else D)
    w.value("n_pool", a["n_pool"], n_pool)
    return c.post["out"]


def _cast(w: Walk, x: Tensor) -> Tensor:
    c = w.take("cast_f32_bf16")
    w.same("x", c.pre["x"].reshape(x.shape), x)
    return c.post["out"]


def walk_patch_projection(w: Walk, model: nn.Module, img: Tensor, box: Optional[Tuple[int, int]] = None) -> Tensor:
    """y = LayerNorm(patch) W^T + b of every patch of img (vit.py:99-102; the SPT's shifted patches,
    vit_for_small_dataset.py:96-112): the 16 x 16 TMA launch with LayerNorm(patch) folded into the projection -- gamma W
    with its columns permuted from the Rearrange's (p1 p2 c) to the image's (c p1 p2), their column sums, W beta + b
    -- or the patchify kernel and a GEMM at K padded to a multiple of 64.  `box`: the patch of img when it is not the
    module's patch_size (the 1-D and 3-D front ends' [B, C, H', W'] views).  Returns y fp32 [B n, D]."""
    pe = model.to_patch_embedding
    spt = getattr(pe, "to_patch_tokens", None)
    ln1, lin = (spt[1], spt[2]) if spt is not None else (pe[1], pe[2])
    ph, pw = box if box is not None else model.patch_size
    src = img.contiguous()
    D, K = lin.weight.shape
    w.where = "patch embedding"
    if w.peek() == "patch_embed_tma":
        c = w.take("patch_embed_tma")
        a = c.pre
        if spt is not None or (ph, pw) != (16, 16):
            w.fail("-", f"the 16 x 16 TMA patch embedding runs for {ph} x {pw}{' shifted' if spt else ''} patches")
        w.same("img", a["img"], src)
        C = K // 256
        wg = (_d(lin.weight) * _d(ln1.weight)[None]).float().bfloat16()
        w.same("w_perm (gamma W, columns (c p1 p2))", a["w_perm"], wg.view(D, 256, C).permute(0, 2, 1).reshape(D, K))
        wd = a["w_perm"].double()
        w.within("col_s (column sums of the bf16 w_perm)", a["col_s"], wd.sum(1), K * U * wd.abs().sum(1))
        t = _d(lin.weight) @ _d(ln1.bias) + _d(lin.bias)
        tb = _d(lin.weight).abs() @ _d(ln1.bias).abs() + _d(lin.bias).abs()
        w.within("bias (W beta + b)", a["bias"], t, (K + 1) * U * tb)
        w.value("eps", a["eps"], float(ln1.eps))
        return c.post["out_f32"]
    if spt is not None:
        c = w.take("patchify_spt_ln")
        w.value("p", c.pre["p"], ph)
    else:
        c = w.take("patchify_ln")
        w.value("ph", c.pre["ph"], ph)
        w.value("pw", c.pre["pw"], pw)
    a = c.pre
    w.same("img", a["img"], src)
    w.same("gamma", a["gamma"], _f(ln1.weight))
    w.same("beta", a["beta"], _f(ln1.bias))
    w.value("eps", a["eps"], float(ln1.eps))
    a0 = c.post["out_bf16"]
    kp = a0.shape[1]
    c = w.take("gemm")
    a = c.pre
    w.same("a", a["a"], a0)
    w.same("w (Linear, K padded)", a["w"], torch.nn.functional.pad(lin.weight.detach(), (0, kp - K)).bfloat16())
    w.same("bias", a["bias"], _f(lin.bias))
    for op in ("resid", "ln_sums", "out_bf16", "stats_out"):
        w.same(op, a[op], None)
    w.value("gelu", a["gelu"], False)
    if a["out_f32"] is None:
        w.fail("out_f32", "the patch projection writes no fp32 output")
    return c.post["out_f32"]


def walk_tokens(w: Walk, model: nn.Module, y: Tensor, B: int, grid: Tuple[int, int], pos: Optional[Tensor] = None,
                ln2: Optional[nn.Module] = None) -> Tuple[Tensor, int]:
    """embed_tokens: [cls; LayerNorm(dim)(y) + pos; register tokens] per image (vit.py:103,122-124,
    simple_vit_with_register_tokens.py:116-126; no LayerNorm(dim) after an SPT), with the first layer's bf16 copy and
    row statistics in fold mode.  `pos`: the positional table when the module builds it in its forward (the 1-D and
    3-D sin-cos tables); `ln2`: LayerNorm(dim) when it is not to_patch_embedding[3].  Returns (x fp32 [B N, D], N)."""
    pe = model.to_patch_embedding
    if ln2 is None:
        ln2 = None if hasattr(pe, "to_patch_tokens") else pe[3]
    ln2 = None if ln2 is None else _ln(ln2)
    D = y.shape[1]
    cls = getattr(model, "cls_token", None) if getattr(model, "cls_in_sequence", True) else None
    cls = None if cls is None or cls.numel() == 0 else cls.detach().float().reshape(-1, D)
    reg = getattr(model, "register_tokens", None)
    reg = None if reg is None or reg.numel() == 0 else reg.detach().float()
    if pos is None:
        pos = getattr(model, "pos_embedding", None)
    if pos is None and hasattr(model, "fused_pos_table"):    # the sin-cos table of the input's own patch grid
        pos = O.posemb_sincos_2d(*grid, D)                  # (simple_flash_attn_vit.py:110-114)
    ncls, ntail = 0 if cls is None else cls.shape[0], 0 if reg is None else reg.shape[0]
    w.where = "token assembly"
    c = w.take("embed_tokens")
    a = c.pre
    w.same("y", a["y"], y)
    w.same("gamma (LayerNorm(dim))", a["gamma"], None if ln2 is None else _f(ln2.gamma))
    if ln2 is not None:
        w.same("beta (LayerNorm(dim))", a["beta"], _f(ln2.beta))
        w.value("eps (LayerNorm(dim))", a["eps"], float(ln2.eps))
    rows = lambda t: None if t is None else t.reshape(-1, D)                            # noqa: E731
    w.same("cls", rows(a["cls"]), cls)
    w.same("pos", rows(a["pos"]), None if pos is None else pos.detach().float().reshape(-1, D))
    w.same("tail (register tokens)", a["tail"], reg)
    w.value("B", a["B"], B)
    n = math.prod(grid)
    w.value("n", a["n"], n)
    w.value("ncls", a["ncls"], ncls)
    x = c.post["x"]
    _entry_copy(w, c, x)
    return x, n + ncls + ntail


def _entry_copy(w: Walk, c: Launch, x: Tensor) -> None:
    """The bf16 copy of x and its row statistics the first folded GEMM reads, written by the embedding in fold mode."""
    a = c.pre
    if not w.fold:
        w.same("xb", a["xb"], None)
        w.same("stats", a["stats"], None)
        return
    if a["xb"] is None or a["stats"] is None:
        w.fail("xb", "the first layer's bf16 copy and row statistics are not written")
    w.same("xb", c.post["xb"], x.bfloat16())
    w.stats("stats", c.post["stats"], c.post["xb"])


def walk_head(w: Walk, model: nn.Module, S: Tensor, B: int, N: int, n: int) -> None:
    """After the last layer on the fp32 stream S: the final LayerNorm, the pooling and the head, by family --
    ViT (vit.py:129-138): LayerNorm of the cls rows (row_index) or of every row then the mean; the SimpleViT family
    (simple_vit.py:116-120 and its variants): LayerNorm, the mean over the patch tokens (not the register tokens), its
    bf16 cast, the head GEMM or the head LayerNorm; a LayerNorm + Linear mlp_head without a final LayerNorm
    (vit_for_small_dataset.py:173-178, deepvit.py:162-167): the cls rows or the mean, then mlp_head[0] and
    mlp_head[1]."""
    from vit_pytorch_b200 import deepvit, simple_vit_with_qk_norm, simple_vit_with_register_tokens, vit
    from vit_pytorch_b200 import vit_for_small_dataset, vit_nd, vit_nd_rotary
    enc = model.transformer
    norm = getattr(enc, "norm", None)
    rows = torch.arange(0, B * N, N, dtype=torch.int32)
    w.where = "head"
    if isinstance(model, (vit_for_small_dataset.ViT, deepvit.DeepViT)):
        ln, lin = _ln(model.mlp_head[0]), model.mlp_head[1]
        if model.pool == "mean":
            pooled = _layernorm_launch(w, _mean_pool(w, S, B, N, None), ln)
        else:
            pooled = _layernorm_launch(w, S, ln, row_index=rows)
        _head_gemm(w, pooled, lin, "mlp_head[1]")
        return
    if isinstance(model, (vit_nd.ViTND, vit_nd_rotary.ViTND)):
        # vit_nd.py:213-216: the mean over the patch tokens x[:, 1:] or the cls row; vit_nd_rotary.py:277: the mean
        if isinstance(model, vit_nd_rotary.ViTND) or model.pool == "mean":
            skip = 0 if isinstance(model, vit_nd_rotary.ViTND) else N - n
            xf = _layernorm_launch(w, S, _ln(norm), f32_out=True)
            flat = xf.reshape(-1)[skip * S.shape[1]:] if skip else xf
            pooled = _cast(w, _mean_pool(w, flat, B, N, None if skip == 0 else n, D=S.shape[1]))
        else:
            pooled = _layernorm_launch(w, S, _ln(norm), row_index=rows)
        _head_gemm(w, pooled, model.mlp_head, "mlp_head")
        return
    if isinstance(model, vit.ViT):
        if model.pool == "mean":
            pooled = _cast(w, _mean_pool(w, _layernorm_launch(w, S, _ln(norm), f32_out=True), B, N, None))
        else:
            pooled = _layernorm_launch(w, S, _ln(norm), row_index=rows)
        _head_gemm(w, pooled, model.mlp_head, "mlp_head")
        return
    xf = S if norm is None else _layernorm_launch(w, S, _ln(norm), f32_out=True)
    registers = isinstance(model, simple_vit_with_register_tokens.SimpleViT)
    pm = _mean_pool(w, xf, B, N, n if registers else None)
    pooled = _cast(w, pm)
    if isinstance(model, simple_vit_with_qk_norm.SimpleViT):       # linear_head is a LayerNorm (sic, reference :128)
        _layernorm_launch(w, pm, _ln(model.linear_head))
        return
    if isinstance(model.linear_head, nn.Sequential):     # simple_flash_attn_vit.py:116-117: LayerNorm, Linear
        _head_gemm(w, _layernorm_launch(w, pm, _ln(model.linear_head[0])), model.linear_head[1], "linear_head[1]")
        return
    _head_gemm(w, pooled, model.linear_head, "linear_head")


def _navit_query_reference(model: nn.Module) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [H dh] of NaViT's pooling query after its LayerNorm, to_q and per-head RMSNorm (na_vit.py:105-112,
    the same for every image), which the host computes in fp32 once per weight version.  The fp32 LayerNorm of D values
    is within layernorm_e32 at depth D, to_q adds D u |W| |ln| (any order of its sums), and the normalised head
    qh / ||qh|| moves by e / ||qh|| + |qh| ||e|| / ||qh||^2 under an error e of qh (first order, 1.01 for the rest);
    then (dh + 6) u |ref| for the norm, the quotient and the products with scale and gamma."""
    pool = model.attn_pool
    H = pool.heads
    q = _d(model.attn_pool_queries)[None]
    ln, e_ln = Bd.layernorm_e32(q, _d(pool.norm.gamma), None, 1e-5, q.shape[1])
    W = _d(pool.to_q.weight)
    qh = (W @ ln[0]).view(H, -1)
    e = (W.abs() @ e_ln[0] + W.shape[1] * U * (W.abs() @ ln[0].abs())).view(H, -1)
    nrm = torch.linalg.vector_norm(qh, dim=-1, keepdim=True)
    g = _d(pool.q_norm.gamma).view(H, -1) * pool.q_norm.scale
    ref = qh / nrm * g
    dh = qh.shape[1]
    bound = 1.01 * g.abs() * (e / nrm + qh.abs() * torch.linalg.vector_norm(e, dim=-1, keepdim=True) / nrm ** 2)
    return ref.reshape(-1), (bound + (dh + 6) * U * ref.abs()).reshape(-1)


def check_navit_provenance(model: nn.Module, images: List[Tensor], launches: List[Launch], ln_mode: str,
                           case: str = "", ratios: Optional[dict] = None) -> int:
    """Walk the trace of na_vit.NaViT.forward_fused(images) (na_vit.py:254-308) through the reference NaViT
    (reference na_vit.py:270-328): the packed (c p1 p2) patch rows of every image and their bias-free LayerNorm, the
    projection, LayerNorm(dim) + pos_embed_height[row] + pos_embed_width[col] of each token's place in its own image's
    grid, the encoder layers over the packed sequences, the final LayerNorm, the attention pooling -- to_kv of the
    normalised tokens with k_norm on the k half, one query per image, + the queries -- and the bias-free head LayerNorm
    and Linear.  The number of launches checked."""
    fold = ln_mode == "fold"
    p = model.patch_size
    pe = model.to_patch_embedding
    lengths = [(im.shape[-2] // p) * (im.shape[-1] // p) for im in images]
    cu = torch.tensor([0] + lengths, dtype=torch.int32).cumsum(0).to(torch.int32)
    dims = [(im.shape[-2], im.shape[-1]) for im in images]
    T, S_ = sum(lengths), len(images)
    w = Walk(case, launches, fold, dict(primed=fold, varlen=None))
    w.ratios = w.ratios if ratios is None else ratios
    w.where = "patch embedding"
    c = w.take("patchify_varlen_ln")
    a = c.pre
    if len(a["images"]) != S_:
        w.fail("images", f"{len(a['images'])} images, want {S_}")
    for i, (got, im) in enumerate(zip(a["images"], images)):
        w.same(f"images[{i}]", got, im.contiguous())
    w.same("gamma", a["gamma"], _f(_ln(pe[0]).gamma))
    w.same("cu_seqlens", a["cu_seqlens"], cu.to(a["cu_seqlens"].device))
    w.value("p", a["p"], p)
    w.value("eps", a["eps"], float(_ln(pe[0]).eps))
    a0 = c.post["out_bf16"]
    lin = pe[1]
    c = w.take("gemm")
    a = c.pre
    w.same("a", a["a"], a0)
    w.same("w", a["w"], lin.weight.detach().bfloat16())
    w.same("bias", a["bias"], _f(lin.bias))
    for op in ("resid", "ln_sums", "out_bf16", "stats_out"):
        w.same(op, a[op], None)
    if a["out_f32"] is None:
        w.fail("out_f32", "the patch projection writes no fp32 output")
    y = c.post["out_f32"]
    w.where = "token assembly"
    c = w.take("embed_varlen")
    a = c.pre
    ix = a["index"]
    w.same("y", a["y"], y)
    w.same("gamma (LayerNorm(dim))", a["gamma"], _f(_ln(pe[2]).gamma))
    w.same("pos_h (pos_embed_height)", a["pos_h"], _f(model.pos_embed_height))
    w.same("pos_w (pos_embed_width)", a["pos_w"], _f(model.pos_embed_width))
    w.same("index.cu", ix.cu, cu.to(ix.cu.device))
    w.same("index.dims", ix.dims, torch.tensor(dims, dtype=torch.int32).reshape(-1).to(ix.dims.device))
    w.value("p", a["p"], p)
    w.value("eps", a["eps"], float(_ln(pe[2]).eps))
    x = c.post["x"]
    _entry_copy(w, c, x)
    enc = model.transformer
    check_identity(enc, case)
    w.kw["varlen"] = ix                        # its cu_seqlens checked above
    S = walk_blocks(w, enc, x)
    w.where = "final LayerNorm"
    xn = _layernorm_launch(w, S, _ln(enc.norm))
    pool = model.attn_pool
    H = pool.heads
    I = pool.to_q.weight.shape[0]
    dh = I // H
    w.where = "attention pooling keys and values"        # na_vit.py:111-112: to_kv of the context, k_norm on k
    c = w.take("gemm_headnorm")
    a = c.pre
    w.same("a", a["a"], xn)
    w.same("w (to_kv)", a["w"], pool.to_kv.weight.detach().bfloat16())
    for op in ("bias", "ln_sums"):
        w.same(op, a[op], None)
    w.same("head_gamma (k_norm)", a["head_gamma"], _f(pool.k_norm.gamma).reshape(-1))
    w.value("norm_heads", a["norm_heads"], H)
    w.value("dh", a["dh"], dh)
    w.value("head_layernorm_eps", a["head_layernorm_eps"], None)
    kv = c.post["out_bf16"]
    w.where = "attention pooling"
    c = w.take("attn_pool")
    a = c.pre
    w.same("kv", a["kv"], kv)
    w.within("qn (the normalised query)", a["qn"], *_navit_query_reference(model))
    w.same("cu_seqlens", a["cu_seqlens"], cu.to(a["cu_seqlens"].device))
    w.value("H", a["H"], H)
    w.value("dh", a["dh"], dh)
    pooled = c.post["out"]
    w.where = "attention pooling out"                    # na_vit.py:384: attn_pool(...) + queries
    queries = _f(model.attn_pool_queries)[None].expand(S_, -1).to(S.device)
    out = pool.to_out[0]
    c = w.take("gemm")
    a = c.pre
    w.same("a", a["a"], pooled)
    w.same("w (to_out)", a["w"], out.weight.detach().bfloat16())
    w.same("bias", a["bias"], _f(out.bias))
    w.same("resid (the queries)", a["resid"], queries)
    for op in ("ln_sums", "out_bf16", "stats_out"):
        w.same(op, a[op], None)
    if a["out_f32"] is None:
        w.fail("out_f32", "the pooled rows are not written in fp32")
    z = c.post["out_f32"]
    w.where = "head"
    zl = _layernorm_launch(w, z, _ln(model.mlp_head[0]))
    _head_gemm(w, zl, model.mlp_head[1], "mlp_head[1]")
    return _end(w)


def walk_nd_projection(w: Walk, model: nn.Module, img: Tensor) -> Tensor:
    """y = (p0 .. p_{r-1} c) patches of img W^T + b (vit_nd.py:160-167, vit_nd_rotary.py:197-202): the N-d gather and
    a GEMM at K padded to a multiple of 64, no LayerNorm of the patches.  Returns y fp32 [B n, D]."""
    pe = model.to_patch_embedding
    lin = pe[1]
    D, K = lin.weight.shape
    w.where = "patch embedding"
    c = w.take("patchify_nd")
    a = c.pre
    w.same("img", a["img"], img.contiguous())
    w.value("patch", tuple(a["patch"]), tuple(pe[0].patch_size))
    a0 = c.post["out_bf16"]
    kp = a0.shape[1]
    c = w.take("gemm")
    a = c.pre
    w.same("a", a["a"], a0)
    w.same("w (Linear, K padded)", a["w"], torch.nn.functional.pad(lin.weight.detach(), (0, kp - K)).bfloat16())
    w.same("bias", a["bias"], _f(lin.bias))
    for op in ("resid", "ln_sums", "out_bf16", "stats_out"):
        w.same(op, a[op], None)
    if a["out_f32"] is None:
        w.fail("out_f32", "the patch projection writes no fp32 output")
    return c.post["out_f32"]


def _video_view(model: nn.Module, video: Tensor) -> Tuple[Tensor, Tuple[int, int], Tuple[int, int, int]]:
    """(the [b, c, (f pf h p1), w p2] view whose (pf p1) x p2 boxes hold the (pf p1 p2 c) patches of the reference's
    Rearrange (simple_vit_3d.py:97, vivit.py:196), the box, the (f, h, w) grid)."""
    pf = model.frame_patch_size if hasattr(model, "frame_patch_size") else model._pf
    p1, p2 = model.patch_size
    b, c, ft, ht, wt = video.shape
    f, h = ft // pf, ht // p1
    img = video.reshape(b, c, f, pf, h, p1, wt).permute(0, 1, 2, 4, 3, 5, 6).reshape(b, c, ft * ht, wt)
    return img, (pf * p1, p2), (f, h, wt // p2)


def check_vivit_provenance(model: nn.Module, video: Tensor, launches: List[Launch], ln_mode: str, case: str = "",
                           ratios: Optional[dict] = None) -> int:
    """Walk the trace of vivit.ViViT.forward_fused(video) (no mask) through the reference ViViT (vivit.py:214-262):
    the (pf p1 p2 c) tubelet embedding, the token assembly of every frame -- the spatial cls token without a position,
    the frame's block of pos_embedding (embed_tokens_grouped) -- then, factorized encoder: the spatial layers over
    every frame, the frame's cls row or mean, the temporal cls token and the temporal layers over the frames, the
    pooling and the head; factorized self-attention: the layers with their axial attention over the frames, then the
    pooling and the head."""
    from vit_pytorch_b200 import vivit
    fold = ln_mode == "fold"
    img, box, (f, h, wg) = _video_view(model, video)
    b, n = video.shape[0], h * wg
    w = Walk(case, launches, fold, dict(primed=fold))
    w.ratios = w.ratios if ratios is None else ratios
    y = walk_patch_projection(w, model, img, box)
    D = y.shape[1]
    cls = not model.global_average_pool
    ncls = int(cls)
    N = n + ncls
    ln2 = _ln(model.to_patch_embedding[3])
    w.where = "token assembly"
    c = w.take("embed_tokens_grouped")
    a = c.pre
    w.same("y", a["y"], y)
    w.same("gamma (LayerNorm(dim))", a["gamma"], _f(ln2.gamma))
    w.same("beta (LayerNorm(dim))", a["beta"], _f(ln2.beta))
    w.value("eps (LayerNorm(dim))", a["eps"], float(ln2.eps))
    w.same("cls (spatial_cls_token)", None if a["cls"] is None else a["cls"].reshape(-1, D),
           _f(model.spatial_cls_token.reshape(-1, D)) if cls else None)
    w.same("pos (pos_embedding)", a["pos"].reshape(-1, D), _f(model.pos_embedding.reshape(-1, D)))
    for op, v in (("groups", b * f), ("n", n), ("ncls", ncls), ("pos_period", f),
                  ("pos_stride", model.pos_embedding.shape[2]), ("cls_pos", False)):
        w.value(op, a[op], v)
    x = c.post["x"]
    _entry_copy(w, c, x)
    rows = lambda B_, N_: torch.arange(0, B_ * N_, N_, dtype=torch.int32)               # noqa: E731
    if model.variant == "factorized_encoder":
        sp, tr = model.spatial_transformer, model.temporal_transformer
        check_identity(sp, case)
        w.kw.update(B=b * f, N=N)
        S = walk_blocks(w, sp, x)
        w.where = "spatial pooling"                        # vivit.py:245-247: x[:, 0] or the mean, per frame
        if cls:
            xs = _layernorm_launch(w, S, _ln(sp.norm), f32_out=True, row_index=rows(b * f, N))
        else:
            xs = _mean_pool(w, _layernorm_launch(w, S, _ln(sp.norm), f32_out=True), b * f, N, None)
        if cls:                                            # vivit.py:251-254: the temporal cls token, then the frames
            xt = torch.cat((_f(model.temporal_cls_token).reshape(1, 1, D).expand(b, 1, D).to(xs.device),
                            xs.view(b, f, D)), 1).reshape(b * (f + 1), D)
        else:
            xt = xs
        Lt = f + ncls
        check_identity(tr, case)
        w.kw, w.have_stats, w.entry_stats = dict(B=b, N=Lt), False, False
        S = walk_blocks(w, tr, xt)
        w.where = "head"
        if cls:
            pooled = _layernorm_launch(w, S, _ln(tr.norm), row_index=rows(b, Lt))
        else:
            pooled = _cast(w, _mean_pool(w, _layernorm_launch(w, S, _ln(tr.norm), f32_out=True), b, Lt, None))
    else:
        tr = model.factorized_transformer
        check_identity(tr, case)
        w.kw.update(B=b * f, N=N, axial=(N, f, None, bool(vivit._flash_mode(tr))))
        S = walk_blocks(w, tr, x)
        w.where = "head"                                   # vivit.py:258-260: the first frame's cls row, or the mean
        if cls:
            pooled = _layernorm_launch(w, S, _ln(tr.norm), row_index=rows(b, f * N))
        else:
            pooled = _cast(w, _mean_pool(w, _layernorm_launch(w, S, _ln(tr.norm), f32_out=True), b, f * N, None))
    _head_gemm(w, pooled, model.mlp_head, "mlp_head")
    return _end(w)


def check_forward_provenance(model: nn.Module, inputs, launches: List[Launch], ln_mode: str, case: str = "",
                             ratios: Optional[dict] = None) -> int:
    """Walk the trace of model.forward_fused(inputs) from the pixels to the logits through the reference module's
    forward: the patch embedding (walk_patch_projection; the N-d gather, walk_nd_projection), the token assembly
    (walk_tokens), the encoder layers (walk_blocks, with the embedding's bf16 copy and row statistics in fold mode), the
    final LayerNorm, pooling and head (walk_head); NaViT by check_navit_provenance, ViViT by check_vivit_provenance.
    Every operand comes from the module's own attributes (to_patch_embedding, cls_token, pos_embedding,
    register_tokens, the head) or the tables its forward builds from the input's grid, never from the engine's
    prepared tensors.  Returns the number of launches checked; raises ProvenanceError naming the launch and the
    operand.  ratios: filled with the worst |got - ref| / bound of each operand checked within a bound (the host's
    fp32 weight preparation, the row statistics)."""
    from vit_pytorch_b200 import na_vit, simple_vit_1d, simple_vit_3d, vit_nd, vit_nd_rotary, vivit
    if isinstance(model, na_vit.NaViT):
        return check_navit_provenance(model, inputs, launches, ln_mode, case, ratios)
    if isinstance(model, vivit.ViViT):
        return check_vivit_provenance(model, inputs, launches, ln_mode, case, ratios)
    fold = ln_mode == "fold"
    w = Walk(case, launches, fold, dict(primed=fold))
    w.ratios = w.ratios if ratios is None else ratios
    B, rope = inputs.shape[0], None
    if isinstance(model, (vit_nd.ViTND, vit_nd_rotary.ViTND)):
        grid = tuple(s // p for s, p in zip(inputs.shape[2:], model.to_patch_embedding[0].patch_size))
        y = walk_nd_projection(w, model, inputs)
        x, N = walk_tokens(w, model, y, B, grid, ln2=model.to_patch_embedding[2])
        if isinstance(model, vit_nd_rotary.ViTND):        # vit_nd_rotary.py:143-147: the grid's rotary table
            cs = model.grid_table(grid, inputs.device)
            rope = (cs, cs.shape[0])
    else:
        if isinstance(model, simple_vit_1d.SimpleViT):    # simple_vit_1d.py:84-90: 'b c (n p) -> b n (p c)'
            b, ch, L = inputs.shape
            p = model.fused_patch_box[1]
            img, box, grid = inputs.contiguous().view(b, ch, 1, L), (1, p), (1, L // p)
            # posemb_sincos_1d / _3d build the table on the input's device (simple_vit_1d.py:21-25)
            pos = simple_vit_1d.sincos_table_1d(L // p, model.linear_head.in_features, device=inputs.device)
        elif isinstance(model, simple_vit_3d.SimpleViT):
            img, box, grid = _video_view(model, inputs)
            pos = simple_vit_3d.sincos_table_3d(*grid, model.linear_head.in_features, device=inputs.device)
        else:
            img, box = inputs, model.patch_size
            grid, pos = (img.shape[2] // box[0], img.shape[3] // box[1]), None
        y = walk_patch_projection(w, model, img, box)
        x, N = walk_tokens(w, model, y, B, grid, pos=None if pos is None else pos.to(y.device))
    enc = model.transformer
    check_identity(enc, case)
    w.kw.update(B=B, N=N, rope=rope)
    S = walk_blocks(w, enc, x)
    walk_head(w, model, S, B, N, math.prod(grid))
    return _end(w)
