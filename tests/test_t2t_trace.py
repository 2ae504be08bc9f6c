"""T2T-ViT's fused forward traced back to the reference layers, without a GPU: T2TViT.forward_fused runs on CPU with
every library launch traced (oracle/layer_trace.tracer, the recording of make_engine_schedule) and emulated -- each
output gets the fp64 reference of its kernel on the operands the launch actually received, rounded to the output's
dtype (oracle/layer_trace.emulate_impl, and below for the T2T entry points: the unfold as F.unfold, the wide attention
from oracle/wide_attention_bounds.py).

Then every launch of every soft split is attributed to its reference layer and its operands checked bit for bit
(`check_soft_splits`): the unfold reads the image or the previous soft split's final LayerNorm output on the map
RearrangeImage makes of it; LN1 reads the stream with Attention.norm's affine; the QKV GEMM reads LN1's output with
to_qkv's rows (q | k | v each padded to dp by zero rows) at K = w; the attention reads that qkv at width dp with the
scale of the true width, one head, one sequence per image; the identity to_out adds it to the stream (the residual
GEMM with the identity on w rows, or the wide kernel's own epilogue on w columns); LN2 and the two FeedForward GEMMs
carry FeedForward.net's parameters; the final LayerNorm is Transformer.norm's.  Then the last unfold, the final Linear,
the cls row and positions.  The main encoder after them is the ViT path that tests/test_layer_trace.py traces; here
its emulated logits must match the module's own fp32 PyTorch graph."""
import math
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN_DIR
from oracle import layer_trace as LT
from oracle.wide_attention_bounds import qkv_wide_reference
from vit_pytorch_b200.pit import pool_grid
from vit_pytorch_b200.t2t import T2TViT, soft_split_width

sys.path.insert(0, GOLDEN_DIR)
import make_engine_schedule as S  # noqa: E402
from t2t_spec import FAMILY, T2T_CASES  # noqa: E402

T2T_ENTRY_POINTS = ("t2t_unfold_image", "t2t_unfold_tokens", "attention_wide")


def _unfold_ref(src: torch.Tensor, k: int, s: int, p: int) -> torch.Tensor:
    """[B, C, h, w] -> the rows of F.unfold, channel-major columns."""
    return F.unfold(src.double(), k, padding=p, stride=s).transpose(1, 2).reshape(-1, src.shape[1] * k * k)


def _write(dst: torch.Tensor, val: torch.Tensor) -> None:
    dst.zero_()
    dst[:, :val.shape[1]] = val.to(dst.dtype)


def t2t_impl(name, real):
    """The T2T entry points emulated, every other one (token assembly included) by oracle/layer_trace.emulate_impl."""
    if name == "t2t_unfold_image":
        def run(img, out, k, s, p):
            _write(out, _unfold_ref(img, k, s, p))
        return run
    if name == "t2t_unfold_tokens":
        def run(x, grid, out, k, s, p):
            h, w = grid
            B = x.shape[0] // (h * w)
            _write(out, _unfold_ref(x.reshape(B, h, w, -1).permute(0, 3, 1, 2), k, s, p))
        return run
    if name == "attention_wide":
        def run(qkv, B, n, dp, scale, ws, out=None, x=None, n_resid=0):
            o = qkv_wide_reference(qkv, B, n, dp, LT.f32(scale))[0].bfloat16()
            if out is not None:
                out.copy_(o)
            if x is not None:
                x[:, :n_resid] += o[:, :n_resid].float()
        return run
    return LT.emulate_impl(name, real)


# what the T2T entry points write, for the tracer's after-call clones
T2T_OUTPUTS = {"t2t_unfold_image": ("out",), "t2t_unfold_tokens": ("out",), "attention_wide": ("out", "x")}


def trace(model: T2TViT, img: torch.Tensor, ln_mode: str, monkeypatch, impl=t2t_impl):
    """(launches, logits) of model.forward_fused(img), every launch run by impl (LT.real_impl: the real kernels)."""
    outs = []
    for k, v in T2T_OUTPUTS.items():
        monkeypatch.setitem(LT.OUTPUTS, k, v)
    with S.recording(None, lambda: [], ln_mode, "python", LT.GRID_ENTRY_POINTS + LT.CLASS_ENTRY_POINTS +
                     LT.FRONT_ENTRY_POINTS + T2T_ENTRY_POINTS, recorder=LT.tracer(impl)) as rec:
        with torch.inference_mode():
            outs.append(model.forward_fused(img))
    return rec.launches, outs[0]


class Walk:
    def __init__(self, launches, case: str) -> None:
        self.launches, self.i, self.case = launches, 0, case

    def take(self, *names):
        c = self.launches[self.i]
        assert c.name in names, f"{self.case}: launch {self.i} is {c.name}, expected {names}"
        self.i += 1
        return c

    def same(self, what: str, got, want) -> None:
        if isinstance(want, torch.Tensor):
            ok = got is not None and got.shape == want.shape and torch.equal(got.double(), want.to(got.device).double())
        else:
            ok = got == want
        assert ok, f"{self.case}: launch {self.i - 1} ({self.launches[self.i - 1].name}): {what} differs"

    def ln(self, what: str, c, m: torch.nn.LayerNorm, x: torch.Tensor) -> torch.Tensor:
        w = m.normalized_shape[0]
        self.same(f"{what} input", c.pre["x"], x[:, :w])
        self.same(f"{what} gamma", c.pre["gamma"], m.weight.float())
        self.same(f"{what} beta", c.pre["beta"], m.bias.float())
        self.same(f"{what} eps", c.args["eps"], m.eps)
        return c.post["out_bf16"]

    def gemm(self, what: str, c, a: torch.Tensor, lin_w: torch.Tensor, bias, K: int, rows=None) -> None:
        self.same(f"{what} K", c.args["k"], K)
        self.same(f"{what} A", c.pre["a"][:, :K], a[:, :K])
        W = c.pre["w"]
        want = torch.zeros(W.shape[0], K, dtype=torch.bfloat16, device=W.device)
        if rows is None:
            want[:lin_w.shape[0]] = lin_w[:, :K].bfloat16()
        else:
            for dst, src0, cnt in rows:
                want[dst:dst + cnt] = lin_w[src0:src0 + cnt, :K].bfloat16()
        self.same(f"{what} weight", W[:, :K], want)
        if bias is None:
            self.same(f"{what} bias", c.pre["bias"], None)
        else:
            b = c.pre["bias"]
            self.same(f"{what} bias", b[:bias.shape[0]], bias.float())
            assert (b[bias.shape[0]:] == 0).all(), f"{self.case}: {what} bias padding"


def check_soft_splits(model: T2TViT, img: torch.Tensor, launches, case: str) -> int:
    """Attribute every soft-split launch and the token assembly to the reference layers; returns the index of the
    first launch of the main encoder."""
    wk = Walk(launches, case)
    B, width = img.shape[0], img.shape[1]
    geo = model.stage_geometry(img.shape[2], img.shape[3])
    src = None
    for i, ((k, s), t, (h, w_, oh, ow)) in enumerate(zip(model.t2t_layers, model.soft_splits(), geo)):
        w, n = width * k * k, oh * ow
        if i == 0:
            c = wk.take("t2t_unfold_image")
            wk.same("image", c.pre["img"], img)
            want = _unfold_ref(img, k, s, s // 2)
        else:
            c = wk.take("t2t_unfold_tokens")
            wk.same("map", tuple(c.args["grid"]), pool_grid(h * w_))            # RearrangeImage's int(sqrt(n)) rows
            wk.same("token rows", c.pre["x"], src[:, :width])
            want = _unfold_ref(src[:, :width].reshape(B, h, w_, width).permute(0, 3, 1, 2), k, s, s // 2)
        wk.same("window", (c.args["k"], c.args["s"], c.args["p"]), (k, s, s // 2))
        x, x_ptr = c.post["out"], c.args["out"].data_ptr()
        wk.same("unfold", x[:, :w], want)
        assert (x[:, w:] == 0).all(), f"{case}: unfold padding"
        width = w
        if t is None:
            src = x
            break
        attn, ff = t.layers[0]
        dp = soft_split_width(w)
        xa = wk.ln("Attention.norm", wk.take("layernorm"), attn.norm, x)
        c = wk.take("gemm")
        wk.gemm("to_qkv", c, xa, attn.to_qkv.weight, None, w, rows=[(j * dp, j * w, w) for j in range(3)])
        qkv = c.post["out_bf16"]
        if dp <= 160:
            c = wk.take("attention_varlen")
            wk.same("qkv", c.pre["qkv"], qkv)
            wk.same("heads, width, scale", (c.args["H"], c.args["dh"], c.args["scale"]), (1, dp, attn.scale))
            wk.same("sequences", c.pre["cu_seqlens"].tolist(), list(range(0, (B + 1) * n, n)))
            o = c.post["out"]
            c = wk.take("gemm")                                         # to_out = nn.Identity: x += o
            wk.gemm("identity to_out", c, o, torch.eye(w), None, w)
            wk.same("residual", c.pre["resid"], x)
            wk.same("stream", c.args["out_f32"].data_ptr(), c.args["resid"].data_ptr())
            x = c.post["out_f32"]
        else:
            c = wk.take("attention_wide")
            wk.same("qkv", c.pre["qkv"], qkv)
            wk.same("images, tokens, width, scale, columns",
                    (c.args["B"], c.args["n"], c.args["dp"], c.args["scale"], c.args["n_resid"]),
                    (B, n, dp, attn.scale, w))
            wk.same("stream in", c.pre["x"], x)
            wk.same("stream", c.args["x"].data_ptr(), x_ptr)
            x = c.post["x"]
        xf = wk.ln("FeedForward.net[0]", wk.take("layernorm"), ff.net[0], x)
        fc1, fc2 = ff.net[1], ff.net[4]
        c = wk.take("gemm")
        wk.gemm("FeedForward.net[1]", c, xf, fc1.weight, fc1.bias, w)
        wk.same("GELU", c.args["gelu"], True)
        hid = c.post["out_bf16"]
        c = wk.take("gemm")
        wk.gemm("FeedForward.net[4]", c, hid, fc2.weight, fc2.bias, w)
        wk.same("residual", c.pre["resid"], x)
        x = c.post["out_f32"]
        src = wk.ln("Transformer.norm", wk.take("layernorm"), t.norm, x)
    lin = model.to_patch_embedding[-1]
    c = wk.take("gemm")
    wk.gemm("to_patch_embedding[-1]", c, src, lin.weight, lin.bias, width)
    y = c.post["out_f32"]
    c = wk.take("embed_tokens")
    wk.same("patch tokens", c.pre["y"], y)
    wk.same("cls_token", c.pre["cls"], model.cls_token.float().reshape(1, -1))
    wk.same("pos_embedding", c.pre["pos"], model.pos_embedding.float().reshape(-1, lin.out_features))
    wk.same("no LayerNorm", c.pre["gamma"], None)
    return wk.i


CASES = {
    # narrow (27 wide, dp 32) and wide (243, dp 256) soft splits
    "k3_small": T2T_CASES["k3_small"],
    # the README widths: 147 (dp 160) and 1323 (dp 1344)
    "pool_mean": T2T_CASES["pool_mean"],
    "isqrt_4x16": T2T_CASES["isqrt_4x16"],
}


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_soft_splits_trace_to_the_reference_layers(name, ln_mode, monkeypatch):
    spec = CASES[name]
    ref = FAMILY.build(spec)
    model = FAMILY.build(spec).bfloat16()
    img = FAMILY.input(spec)
    launches, logits = trace(model, img, ln_mode, monkeypatch)
    first_main = check_soft_splits(model, img, launches, f"{name} {ln_mode}")
    assert first_main < len(launches) and launches[-1].name == "gemm"
    with torch.inference_mode():
        want = ref(img.float())
    d = (logits.float() - want).abs().max().item()
    assert d < 5e-2, (name, ln_mode, d)


def test_a_miswired_operand_is_named(monkeypatch):
    """The walk names a launch whose operand is not the reference layer's: the soft split's LN2 with LN1's affine."""
    spec = CASES["k3_small"]
    model = FAMILY.build(spec).bfloat16()
    img = FAMILY.input(spec)
    t = model.soft_splits()[0]
    with torch.no_grad():
        t.layers[0][1].net[0].weight.copy_(t.layers[0][0].norm.weight)   # the prepared weights, as the driver reads
    launches, _ = trace(model, img, "exact", monkeypatch)
    with torch.no_grad():
        t.layers[0][1].net[0].weight.add_(1.0)                          # ... and a module that differs from them
    with pytest.raises(AssertionError, match="FeedForward.net\\[0\\] gamma"):
        check_soft_splits(model, img, launches, "miswired")
    assert math.isfinite(float(launches[0].post["out"].float().sum()))
