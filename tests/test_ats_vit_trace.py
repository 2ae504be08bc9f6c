"""The Adaptive Token Sampling ViT's fused forward traced back to the reference layers, without a GPU: ViT.forward_fused
runs on CPU with every library launch traced (oracle/layer_trace.tracer) and emulated (test_ats_vit.ats_impl: the
encoder kernels by their fp64 references, the select, gather and key-count attention by oracle/ats_bounds.py), with
the fixture's uniforms replayed.

Then every launch is attributed to its reference layer and its operands checked bit for bit (`walk`): the patch
embedding's LayerNorm(dim), cls token and positional rows; per encoder layer Attention.norm (a LayerNorm launch, or in
fold mode its gamma folded into to_qkv's rows and its beta into the bias), to_qkv, then either the plain attention or
AdaptiveTokenSampling -- the select on that layer's qkv with its K, heads and scale, the lengths and ids the previous
select wrote, the gather of the stream entering the layer and of the qkv, the attention of the gathered queries (or
the qkv's own, on a layer that cannot sample) over that qkv's keys with the lengths the layer started from --
to_out onto the gathered stream, FeedForward.net (LayerNorm, Linear, GELU, Linear) and finally mlp_head (its LayerNorm
on every image's row 0, its Linear).  Each stream, bf16 copy and row-sum slot a launch reads must be the one the
launch before it wrote.  The emulated logits must match the module's own fp32 graph on the same draws, and a planted
miswiring is named."""
import math
import sys

import pytest
import torch

import test_ats_vit as TA
from conftest import GOLDEN_DIR, load_golden
from vit_pytorch_b200 import ats_vit as A

sys.path.insert(0, GOLDEN_DIR)
from ats_vit_spec import ATS_CASES, FAMILY  # noqa: E402


class Walk:
    def __init__(self, launches, case: str) -> None:
        self.launches, self.i, self.case = launches, 0, case

    def take(self, *names):
        c = self.launches[self.i]
        assert c.name in names, f"{self.case}: launch {self.i} is {c.name}, expected one of {names}"
        self.i += 1
        return c

    def peek(self) -> str:
        return self.launches[self.i].name if self.i < len(self.launches) else ""

    def same(self, what: str, got, want) -> None:
        if isinstance(want, torch.Tensor):
            ok = (isinstance(got, torch.Tensor) and got.shape == want.shape and got.dtype == want.dtype
                  and torch.equal(got, want))
        else:
            ok = got == want
        assert ok, f"{self.case}: launch {self.i - 1}: {what} is not the reference layer's"


def _f32(p):
    return p.detach().float()


def _bf(p):
    return p.detach().to(torch.bfloat16)


def normed_gemm(w: Walk, where: str, ln, lin, stream, xb, sums, fold: bool, **epi):
    """LN(stream) lin^T through a LayerNorm launch and the plain GEMM, or (fold) the LN-folded GEMM on the bf16 copy
    xb with the row sums `sums`; returns the GEMM launch."""
    if not fold:
        c = w.take("layernorm")
        w.same(f"{where} input stream", c.pre["x"], stream)
        w.same(f"{where} gamma", c.pre["gamma"], _f32(ln.weight))
        w.same(f"{where} beta", c.pre["beta"], _f32(ln.bias))
        w.same(f"{where} eps", c.args["eps"], ln.eps)
        g = w.take("gemm")
        w.same(f"{where} normalised rows", g.pre["a"], c.post["out_bf16"])
        w.same(f"{lin[0]} weight", g.pre["w"], _bf(lin[1].weight))
        w.same(f"{lin[0]} bias", g.pre["bias"], None if lin[1].bias is None else _f32(lin[1].bias))
    else:
        g = w.take("gemm")
        w.same(f"{where} bf16 copy of the stream", g.pre["a"], xb)
        w.same(f"{where} row sums", g.pre["ln_sums"], sums)
        w.same(f"{where} gamma folded into {lin[0]}",
               g.pre["w"], (_f32(lin[1].weight) * _f32(ln.weight)[None, :]).to(torch.bfloat16))
        t = _f32(lin[1].weight) @ _f32(ln.bias)
        w.same(f"{where} beta folded into {lin[0]}'s bias", g.pre["bias"],
               t if lin[1].bias is None else t + _f32(lin[1].bias))
        w.same(f"{where} eps", g.args["ln_eps"], ln.eps)
    for k, v in epi.items():
        w.same(f"{lin[0]} {k}", bool(g.args[k]), v)
    return g


def walk(model: A.ViT, launches, ln_mode: str, case: str) -> None:
    fold = ln_mode == "fold"
    w = Walk(launches, case)
    emb = model.to_patch_embedding
    if w.take("patchify_ln", "patch_embed_tma").name == "patchify_ln":
        w.take("gemm")                               # the patch projection
    e = w.take("embed_tokens")
    w.same("to_patch_embedding[3] gamma", e.pre["gamma"], _f32(emb[3].weight))
    w.same("to_patch_embedding[3] beta", e.pre["beta"], _f32(emb[3].bias))
    w.same("cls_token", e.pre["cls"].reshape(-1), _f32(model.cls_token).reshape(-1))
    n = e.args["n"]
    w.same("pos_embedding[:, :n + 1]", e.pre["pos"][:n + 1], _f32(model.pos_embedding)[0, :n + 1])
    stream, xb, sums = e.post["x"], e.post.get("xb"), e.post.get("stats")
    B = e.args["B"]
    lens, ids = torch.full((B,), n + 1, dtype=torch.int32), None
    for i, (attn, ff) in enumerate(model.transformer.layers):
        L = f"layer {i}"
        H, dh = attn.heads, attn.dim_head
        I = H * dh
        S_in = stream.shape[0] // B
        if fold and xb is None:                      # the un-primed fold chain opens with one statistics pass
            r = w.take("rowstats_cast")
            w.same(f"{L} rowstats input", r.pre["x"], stream)
            xb, sums = r.post["xb"], r.post["stats"]
        g = normed_gemm(w, f"{L} Attention.norm", attn.norm, ("to_qkv", attn.to_qkv), stream, xb, sums, fold)
        qkv = g.post["out_bf16"]
        if w.peek() == "attention":
            c = w.take("attention")
            w.same(f"{L} attention qkv", c.pre["qkv"], qkv)
            w.same(f"{L} heads / dim_head / scale", (c.args["H"], c.args["dh"], c.args["scale"]),
                   (H, dh, attn.scale))
            o, new_stream = c.post["out"], stream
        else:
            keys = lens
            if w.peek() == "ats_select":
                c = w.take("ats_select")
                w.same(f"{L} AdaptiveTokenSampling qkv", c.pre["qkv"], qkv)
                w.same(f"{L} AdaptiveTokenSampling K", c.args["K"], attn.output_num_tokens)
                w.same(f"{L} heads / dim_head / scale", (c.args["H"], c.args["dh"], c.args["scale"]),
                       (H, dh, attn.scale))
                w.same(f"{L} lengths entering the select", c.pre["lens"], lens)
                if ids is not None:
                    w.same(f"{L} token ids entering the select", c.pre["ids"], ids)
                src, lens, ids = c.post["src"], c.post["lens_out"], c.post["ids_out"]
                gth = w.take("ats_gather")
                w.same(f"{L} gather row map", gth.pre["src"], src)
                w.same(f"{L} gathered stream", gth.pre["x"], stream)
                w.same(f"{L} gathered qkv", gth.pre["a"], qkv)
                w.same(f"{L} gathered query columns", gth.args["ncols"], I)
                new_stream, q = gth.post["x_out"], gth.post["a_out"][:, :I]
            else:
                new_stream, q = stream, qkv[:, :I]
            c = w.take("attention_kv_lens")
            w.same(f"{L} attention queries", c.pre["q"], q)
            w.same(f"{L} attention keys and values", c.pre["kv"], qkv[:, I:3 * I])
            w.same(f"{L} attention key counts", c.pre["lens"], keys)
            w.same(f"{L} heads / dim_head / scale", (c.args["H"], c.args["dh"], c.args["scale"]),
                   (H, dh, attn.scale))
            w.same(f"{L} key slot", c.args["Nk"], S_in)
            o = c.post["out"]
        r = w.take("gemm")
        w.same(f"{L} to_out input", r.pre["a"], o)
        w.same(f"{L} to_out weight", r.pre["w"], _bf(attn.to_out[0].weight))
        w.same(f"{L} to_out bias", r.pre["bias"], _f32(attn.to_out[0].bias))
        w.same(f"{L} residual stream of to_out", r.pre["resid"], new_stream)
        stream, xb = r.post["out_f32"], r.post.get("out_bf16")
        sums = r.post.get("stats_out")
        g = normed_gemm(w, f"{L} FeedForward.net[0]", ff.net[0], ("FeedForward.net[1]", ff.net[1]), stream, xb, sums,
                        fold, gelu=True)
        r = w.take("gemm")
        w.same(f"{L} FeedForward.net[4] input", r.pre["a"], g.post["out_bf16"])
        w.same(f"{L} FeedForward.net[4] weight", r.pre["w"], _bf(ff.net[4].weight))
        w.same(f"{L} FeedForward.net[4] bias", r.pre["bias"], _f32(ff.net[4].bias))
        w.same(f"{L} residual stream of FeedForward", r.pre["resid"], stream)
        stream, xb, sums = r.post["out_f32"], r.post.get("out_bf16"), r.post.get("stats_out")
    c = w.take("layernorm")
    S = stream.shape[0] // B
    w.same("mlp_head[0] input stream", c.pre["x"], stream)
    w.same("mlp_head[0] gamma", c.pre["gamma"], _f32(model.mlp_head[0].weight))
    w.same("mlp_head[0] beta", c.pre["beta"], _f32(model.mlp_head[0].bias))
    w.same("mlp_head[0] rows (every image's row 0)", c.pre["row_index"],
           torch.arange(0, B * S, S, dtype=torch.int32))
    g = w.take("gemm")
    w.same("mlp_head[1] input", g.pre["a"], c.post["out_bf16"])
    w.same("mlp_head[1] weight", g.pre["w"], _bf(model.mlp_head[1].weight))
    w.same("mlp_head[1] bias", g.pre["bias"], _f32(model.mlp_head[1].bias))
    assert w.i == len(launches), f"{case}: {len(launches) - w.i} launches after the head"


def reference_logits(name: str) -> torch.Tensor:
    """The module's own fp32 graph on the case's recorded draws (the fixture's logits)."""
    return load_golden("ats_vit")["cases"][name]["logits_sampled"]


CASES = ["readme", "stays_off", "ragged", "no_sampling", "dh80"]


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("name", CASES)
def test_forward_traces_to_the_reference_layers(name, ln_mode, monkeypatch):
    spec, case = ATS_CASES[name], load_golden("ats_vit")["cases"][name]
    model = FAMILY.build(spec).bfloat16()
    img = FAMILY.input(spec)
    launches, (logits, _, _) = TA.trace(model, img, ln_mode, monkeypatch, case)
    walk(model, launches, ln_mode, f"{name} {ln_mode}")
    d = (logits.float() - reference_logits(name)).abs().max().item()
    assert d < 3e-2, (name, ln_mode, d)


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
def test_a_miswired_operand_is_named(ln_mode, monkeypatch):
    """The walk names a launch whose operand is not the reference layer's: layer 3's FeedForward LayerNorm with its
    Attention.norm's gamma (the prepared weights are built from that, and then the module differs from them)."""
    spec, case = ATS_CASES["readme"], load_golden("ats_vit")["cases"]["readme"]
    model = FAMILY.build(spec).bfloat16()
    img = FAMILY.input(spec)
    attn, ff = model.transformer.layers[3]
    with torch.no_grad():
        ff.net[0].weight.copy_(attn.norm.weight)
    launches, _ = TA.trace(model, img, ln_mode, monkeypatch, case)
    with torch.no_grad():
        ff.net[0].weight.add_(1.0)
    with pytest.raises(AssertionError, match="layer 3 FeedForward.net\\[0\\] gamma"):
        walk(model, launches, ln_mode, "miswired")
    assert math.isfinite(float(launches[-1].post["out_bf16"].float().sum()))


def test_a_miswired_stream_is_named(monkeypatch):
    """A sampling layer whose attention reads the key counts the select just wrote instead of the ones the layer
    started from is named."""
    spec, case = ATS_CASES["readme"], load_golden("ats_vit")["cases"]["readme"]
    model = FAMILY.build(spec).bfloat16()
    img = FAMILY.input(spec)
    lib = A._lib

    class Miswired:
        """ats_vit's view of the library with the attention handed the select's new key counts."""
        new = None

        def __getattr__(self, name):
            return getattr(lib, name)

        def ats_select(self, qkv, lens, ids, u, src, lens_out, *a, **k):
            Miswired.new = lens_out
            return lib.ats_select(qkv, lens, ids, u, src, lens_out, *a, **k)

        def attention_kv_lens(self, q, kv, out, lens, *a, **k):
            return lib.attention_kv_lens(q, kv, out, Miswired.new if Miswired.new is not None else lens, *a, **k)
    monkeypatch.setattr(A, "_lib", Miswired())
    launches, _ = TA.trace(model, img, "exact", monkeypatch, case)
    with pytest.raises(AssertionError, match="layer 3 attention key counts"):
        walk(model, launches, "exact", "miswired stream")
