"""The encoder layers that attend over a token grid traced back to their reference layers without a GPU
(oracle/layer_trace.py, as tests/test_layer_trace.py does for the sequence families): Twins-SVT's local windows and
strided keys, MaxViT's block and dilated windows under a relative-position bias, CvT's convolutional projections,
MobileViT's patch groups with its SiLU feed-forward block, ScalableViT's sub-sampled keys and interactive windows (its
padded key heads, its feed-forward-first layers, and the PEG and entry prime between the run_blocks calls of
Transformer.run_fused), SepViT's window tokens and window mixing, and RegionViT's region pass and region-to-local
windows.

Every case runs in both LayerNorm modes with per-LayerNorm eps (set_eps, the channel LayerNorms included) and
BatchNorm eps 1e-3; the provenance walk must accept every launch and the emulated outputs must sit within their
bounds.  Planted wiring and weight-preparation defects must be named by layer, launch and operand.

The kernels' oracles (oracle/grid_attention_bounds.py) rebuild window membership, key patches and the bias look-up
from the kernels' address formulas; the geometry tests here hold those formulas to the modules' own eager rearranges,
convolutions and bias look-ups, which the family parity tests hold to the reference's logits, on integer index
maps."""
import copy
import dataclasses

import pytest
import torch
from torch import nn

from oracle import grid_attention_bounds as GB
from oracle import layer_trace as LT
from test_layer_trace import lib, make  # noqa: F401  (lib: the module fixture that builds the library)
from test_layer_trace import run as run_blocks_traced
from vit_pytorch_b200 import (_lib, crossformer, cvt, engine, max_vit, mobile_vit, regionvit, scalable_vit, sep_vit,
                              twins_svt)

S = LT.schedule()
D, B = S.D, 2


class MaxViTBlock(max_vit._BlockAttention, nn.Module):
    """The attention half of a MaxViT block (max_vit.py:262-273) as a module of its own: the block's Sequential with an
    identity where the MBConv stands."""

    def __init__(self, w: int, dim: int = D, dim_head: int = 32, mult: int = 2) -> None:
        nn.Module.__init__(self)
        attn = lambda: max_vit.Attention(dim, dim_head=dim_head, window_size=w)       # noqa: E731
        ff = lambda: max_vit.FeedForward(dim, mult=mult)                              # noqa: E731
        self.block = nn.Sequential(nn.Identity(), max_vit._ToWindows(w, grid=False), max_vit.Residual(dim, attn()),
                                   max_vit.Residual(dim, ff()), max_vit._FromWindows(grid=False),
                                   max_vit._ToWindows(w, grid=True), max_vit.Residual(dim, attn()),
                                   max_vit.Residual(dim, ff()), max_vit._FromWindows(grid=True))
        self.layers = (self.block[2], self.block[6])

    def parameters(self, recurse: bool = True):
        return nn.Module.parameters(self, recurse)


def _twins(p, k, local=True, depth=1):
    return lambda: twins_svt.Transformer(D, depth, heads=2, dim_head=32, mlp_mult=2, local_patch_size=p, global_k=k,
                                         has_local=local)


def _crossformer(local, glob, depth=1):
    return lambda: crossformer.Transformer(D, local_window_size=local, global_window_size=glob, depth=depth, dim_head=32)


def _cvt(heads, k=3, s=2):
    return lambda: cvt.Transformer(D, proj_kernel=k, kv_proj_stride=s, depth=2, heads=heads, dim_head=32, mlp_mult=2)


def _mobile():
    return mobile_vit.Transformer(D, 2, heads=2, dim_head=8, mlp_dim=2 * D)


def _scalable(dk, r, window, dv=32, depth=1):
    return lambda: scalable_vit.Transformer(D, depth, heads=2, ff_expansion_factor=2, ssa_dim_key=dk, ssa_dim_value=dv,
                                            ssa_reduction_factor=r, iwsa_dim_key=dk, iwsa_dim_value=dv,
                                            iwsa_window_size=window)


def _sep(depth=1):
    return lambda: sep_vit.Transformer(D, depth, dim_head=32, heads=2, ff_mult=2)


def _region(W, depth=2):
    return lambda: regionvit.R2LTransformer(D, window_size=W, depth=depth, heads=2)


def _case(name, module, grid, primed=False, **kw):
    gh, gw = grid
    return S.Case(name, module, B * gh * gw, lambda: dict(B=B, N=gh * gw, grid=grid, primed=primed, **kw), False)


def _region_case(name, module, grid, regions, b=B, primed=False):
    """B local maps (the `grid`) followed by B region maps, in one stream."""
    (lh, lw), (rh, rw) = grid, regions
    return S.Case(name, module, b * (lh * lw + rh * rw),
                  lambda: dict(B=b, N=lh * lw, grid=grid, regions=regions, primed=primed), False)


CASES = [
    # global k = 4 on a 6 x 10 grid: 1 x 2 key patches, the rest of the map dropped (floor, as Conv2d)
    _case("twins local 2 global 4 on 6x10", _twins(2, 4, depth=2), (6, 10)),
    _case("twins local 3 global 3 on 6x9 primed", _twins(3, 3), (6, 9), primed=True),
    _case("twins global 1 (no im2col) on 4x6", _twins(1, 1, local=False, depth=2), (4, 6), primed=True),
    # 3 x 3 windows on a 6 x 9 map: the blocks and the dilated grids differ
    _case("max_vit block + dilated w3 on 6x9", lambda: MaxViTBlock(3), (6, 9)),
    _case("max_vit block + dilated w2 on 4x4 primed", lambda: MaxViTBlock(2), (4, 4), primed=True),
    # short 3 x 3 blocks and long 2 x 2 dilated grids of a 6 x 12 map, where blocks and dilated grids differ
    _case("crossformer short 3 long 2 on 6x12", _crossformer(3, 2, depth=2), (6, 12)),
    _case("crossformer short 2 long 4 on 8x4 primed", _crossformer(2, 4), (8, 4), primed=True),
    _case("cvt 1 head stride 2 on 5x7", _cvt(1), (5, 7)),
    _case("cvt 2 heads stride 2 on 7x5 primed", _cvt(2), (7, 5), primed=True),
    _case("cvt 2 heads k5 stride 3 on 4x6", _cvt(2, k=5, s=3), (4, 6)),
    _case("mobile_vit groups 2x2 on 4x6", _mobile, (4, 6), groups=(2, 2)),
    _case("mobile_vit groups 1x2 on 3x4 primed", _mobile, (3, 4), primed=True, groups=(1, 2)),
    # dim_key 40 (run at 48) with value heads 64; 2 x 2 key patches of a 6 x 9 map (the last column dropped, as
    # Conv2d); 3 x 3 windows; depth 2: the PEG and the entry prime between the first two layers
    _case("scalable_vit dk40 dv64 reduction 2 window 3 on 6x9 depth 2", _scalable(40, 2, 3, dv=64, depth=2), (6, 9)),
    _case("scalable_vit reduction 1 whole-map window on 4x6", _scalable(32, 1, None), (4, 6)),
    # SepViT's windows are 7 x 7 (DSSA's default window_size)
    _case("sep_vit 4 windows 2 heads on 14x14 depth 2", _sep(depth=2), (14, 14)),
    _case("sep_vit single window on 7x7 primed", _sep(), (7, 7), primed=True),
    _region_case("regionvit 4x4 windows on 8x8 / 2x2 depth 2", _region(4), (8, 8), (2, 2)),
    _region_case("regionvit odd rows 3x5 / 1x1 primed", _region(5), (3, 5), (1, 1), b=3, primed=True),
    _region_case("regionvit 2x3 windows on 4x6 / 2x2 primed", _region(3), (4, 6), (2, 2), primed=True),
]


def _run_fused(mod, x, kw):
    gh, gw = kw["grid"]
    mod.run_fused(x, kw["B"], gh, gw)


def run(case, ln_mode, plant=None):
    """test_layer_trace.run; ScalableViT through its Transformer.run_fused: the first layer, the PEG and (fold) the
    entry prime, the other layers."""
    call = _run_fused if case.name.startswith("scalable_vit") else None
    return run_blocks_traced(case, ln_mode, plant, call=call)


def _named(name):
    return next(c for c in CASES if c.name == name)


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_every_grid_launch_traces_back_to_the_reference_layer(case, ln_mode):
    mod, x0, kw, launches = run(case, ln_mode)
    assert LT.check_provenance(mod, x0, kw, launches, ln_mode, case.name) == len(launches) > 0
    LT.check_accuracy(launches, f"{case.name} | {ln_mode}")


def test_every_case_eps_differs_between_its_layer_norms():
    for case in CASES:
        layers, _ = make(case).encoder_layers()
        assert all(L.ln1.eps != L.ln2.eps for L in layers), case.name
        for L in layers:
            A = L.attention
            if isinstance(A, engine.ConvProj):
                assert A.q_bn_eps == A.kv_bn_eps == 1e-3, case.name


def test_identity_accepts_views_of_the_parameters_and_rejects_copies():
    mod = make(_named("cvt 1 head stride 2 on 5x7"))
    LT.check_identity(mod, "views")
    orig = cvt.Transformer.encoder_layers

    def copied(self):
        layers, norm = orig(self)
        L = layers[1]
        return layers[:1] + [dataclasses.replace(L, ln1=L.ln1._replace(gamma=L.ln1.gamma.detach().clone()))], norm
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(cvt.Transformer, "encoder_layers", copied)
        with pytest.raises(AssertionError, match="layer 1: EncoderLayer.ln1.gamma"):
            LT.check_identity(mod, "copy")


# ------------------------------------------------------------------------------------------------------ planted defects
def _bn_default_eps(mp):
    orig = engine.conv_proj_weights
    mp.setattr(engine, "conv_proj_weights", lambda P: orig(P._replace(q_bn_eps=1e-5, kv_bn_eps=1e-5)))


def _strided_kv_channel_major(mp):
    def bad(self, t, i, L):
        t[f"{i}.kv.w"] = engine._bf16_rows(self.kv_w.detach().reshape(self.kv_w.shape[0], -1))
    mp.setattr(engine.StridedKV, "prepare", bad)


def _dilated_swapped(mp):
    orig = max_vit._BlockAttention.encoder_layers

    def bad(self):
        layers, norm = orig(self)
        return [dataclasses.replace(L, attention=L.attention._replace(dilated=not L.attention.dilated))
                for L in layers], norm
    mp.setattr(max_vit._BlockAttention, "encoder_layers", bad)


def _dpb_stride_2w_plus_1(mp):
    """The DPB table read with the stride 2w + 1 of the evaluated offset grid: the offsets in [-(w-1), w-1]^2."""
    def bad(attn):
        w = attn.window_size
        full = crossformer._rel_offsets(w, attn.rel_pos_indices.device)
        x = full
        with torch.no_grad():
            for m in attn.dpb:
                x = m(x)
        x = x.view(2 * w + 1, 2 * w + 1)[1:-1, 1:-1].reshape(-1)
        return x[:, None].expand(-1, attn.heads).float().contiguous()
    mp.setattr(crossformer, "dpb_table", bad)


def _gelu_feed_forward(mp):
    orig = mobile_vit.Transformer.encoder_layers

    def bad(self):
        layers, norm = orig(self)
        return [dataclasses.replace(L, ff_act="gelu") for L in layers], norm
    mp.setattr(mobile_vit.Transformer, "encoder_layers", bad)


def _iwsa_scale_padded(mp):
    """The IWSA softmax scale from the padded key width (48) instead of dim_key (40)."""
    orig = scalable_vit.Transformer.encoder_layers

    def bad(self):
        layers, norm = orig(self)
        return [dataclasses.replace(L, scale=L.dim_head ** -0.5) if L.ff_first else L for L in layers], norm
    mp.setattr(scalable_vit.Transformer, "encoder_layers", bad)


def _lim_reads_k(mp):
    """InteractiveWindows.launch with the LIM convolution's im2col over the k columns of qkv instead of the v."""
    def bad(self, c, L, i):
        t, (gh, gw), M = c.t, c.grid, c.x.shape[0]
        Ik, dv = L.heads * L.dim_head, self.value_width(L)
        Iv = L.heads * dv
        qkv = engine._rows_of(c.qkv, L.qkv_w.shape[0])
        c.project(L, i, out=qkv)
        col = torch.empty(M, 9 * Iv, device=c.x.device, dtype=torch.bfloat16)
        _lib.conv_im2col_nhwc(qkv[:, Ik:Ik + Iv], col, c.B, gh, gw, 3, 1, 1)
        lim = torch.empty(M, Iv, device=c.x.device, dtype=torch.bfloat16)
        _lib.gemm(col, t[f"{i}.lim.w"], out_bf16=lim, bias=t[f"{i}.lim.b"])
        o = engine._rows_of(c.o, Iv)
        wh, ww = self.window(c.grid)
        _lib.attention_iwsa(qkv, lim, o, c.B, gh, gw, wh, ww, L.heads, L.dim_head, dv, L.scale)
        return o
    mp.setattr(engine.InteractiveWindows, "launch", bad)


class _Without:
    """The _lib module as a model file sees it, with one entry point replaced."""

    def __init__(self, name, fn):
        self.name, self.fn = name, fn

    def __getattr__(self, name):
        return self.fn if name == self.name else getattr(_lib, name)


def _peg_prime_dropped(mp):
    """run_fused without the rowstats_cast after the PEG: the second run_blocks call, primed, reads the bf16 copy and
    statistics of the stream before the PEG."""
    mp.setattr(scalable_vit, "_lib", _Without("rowstats_cast", lambda *a, **k: None))


def _head_ln_default_eps(mp):
    orig = sep_vit.Transformer.encoder_layers

    def bad(self):
        layers, norm = orig(self)
        return [dataclasses.replace(L, attention=L.attention._replace(ln=L.attention.ln._replace(eps=1e-5)))
                for L in layers], norm
    mp.setattr(sep_vit.Transformer, "encoder_layers", bad)


def _window_token_normalised(mp):
    """The window token's q | k | v projected from the token after the layer's LayerNorm."""
    orig = engine.WindowTokenBlock.prepare

    def bad(self, t, i, L):
        orig(self, t, i, L)
        f = lambda p: p.detach().float()                                                # noqa: E731
        tok = torch.nn.functional.layer_norm(f(self.token), self.token.shape, f(L.ln1.gamma), f(L.ln1.beta), L.ln1.eps)
        t[f"{i}.tok_qkv"] = (L.qkv_w.detach().float() @ tok).to(torch.bfloat16)
    mp.setattr(engine.WindowTokenBlock, "prepare", bad)


def _wqk_blocked(mp):
    """The window tokens' q | k rows as all heads' q, then all heads' k."""
    orig = engine.WindowTokenBlock.prepare

    def bad(self, t, i, L):
        orig(self, t, i, L)
        H, dh = L.heads, L.dim_head
        w, b = t[f"{i}.wqk.w"], t[f"{i}.wqk.b"]
        t[f"{i}.wqk.w"] = w.view(H, 2, dh, -1).transpose(0, 1).reshape(w.shape).contiguous()
        t[f"{i}.wqk.b"] = b.view(H, 2, dh).transpose(0, 1).reshape(-1).contiguous()
    mp.setattr(engine.WindowTokenBlock, "prepare", bad)


def _region_residual_without_stats(mp):
    """The region rows' out-projection residual (its fp32 stream a view at a row offset of x) writes no statistics."""
    def gemm(*args, stats_out=None, resid=None, **kw):
        if resid is not None and resid.storage_offset() > 0:
            stats_out = None
        return _lib.gemm(*args, stats_out=stats_out, resid=resid, **kw)
    mp.setattr(engine, "_lib", _Without("gemm", gemm))


def _r2l_table_reshaped(mp):
    def bad(self, t, i, L):
        t[f"{i}.r2l"] = self.bias.detach().float().reshape(self.bias.shape[1], -1).contiguous()
    mp.setattr(engine.RegionLocalBlock, "prepare", bad)


SCALABLE_A, SCALABLE_B = ("scalable_vit dk40 dv64 reduction 2 window 3 on 6x9 depth 2",
                          "scalable_vit reduction 1 whole-map window on 4x6")
SEP, REGION = "sep_vit 4 windows 2 heads on 14x14 depth 2", "regionvit 4x4 windows on 8x8 / 2x2 depth 2"

# name: (case, LayerNorm mode, plant(monkeypatch), what the failure must name)
DEFECTS = {
    "CvT BatchNorm folded with eps 1e-5 instead of the module's":
        ("cvt 1 head stride 2 on 5x7", "exact", _bn_default_eps,
         ("layer 0 convolutional projection", "conv_proj_dw", "operand wq")),
    "StridedKV weight in (channel, tap) order":
        ("twins local 2 global 4 on 6x10", "fold", _strided_kv_channel_major,
         ("layer 1 keys and values", "gemm", "operand w")),
    "MaxViT block and grid windows swapped":
        ("max_vit block + dilated w3 on 6x9", "fold", _dilated_swapped,
         ("layer 0 attention", "attention_window_relpos", "operand dilated")),
    "CrossFormer DPB table taken with stride 2w + 1":
        ("crossformer short 3 long 2 on 6x12", "fold", _dpb_stride_2w_plus_1,
         ("layer 0 attention", "attention_window_relpos", "operand table (dpb)")),
    "MobileViT feed-forward with GELU instead of SiLU":
        ("mobile_vit groups 2x2 on 4x6", "exact", _gelu_feed_forward, ("layer 0 fc1", "gemm_act expected")),
    "IWSA scale from the padded key width":
        (SCALABLE_A, "exact", _iwsa_scale_padded, ("layer 1 attention", "attention_iwsa", "operand scale")),
    "LIM im2col over the k columns":
        (SCALABLE_B, "fold", _lim_reads_k, ("layer 1 local interactive module", "conv_im2col_nhwc", "operand x")),
    "no rowstats_cast after the PEG":
        (SCALABLE_A, "fold", _peg_prime_dropped, ("layer 1 fc1", "gemm", "operand a")),
    "SepViT head LayerNorm at the default eps":
        (SEP, "fold", _head_ln_default_eps, ("layer 0 window tokens", "head_layernorm_gelu", "operand eps")),
    "window token projected after the LayerNorm":
        (SEP, "exact", _window_token_normalised, ("layer 0 attention", "attention_window_token", "operand tok_qkv")),
    "window tokens' q | k rows blocked, not interleaved per head":
        (SEP, "fold", _wqk_blocked, ("layer 0 window tokens", "gemm", "operand w")),
    "region residual writes no statistics":
        (REGION, "fold", _region_residual_without_stats, ("layer 1 region out", "gemm", "operand stats_out")),
    "r2l table reshaped, not transposed":
        (REGION, "exact", _r2l_table_reshaped, ("layer 0 attention", "attention_region_local", "operand table")),
}


@pytest.mark.parametrize("name", list(DEFECTS))
def test_planted_defect_is_named(name, monkeypatch):
    case, ln_mode, plant, want = DEFECTS[name]
    mod, x0, kw, launches = run(_named(case), ln_mode, plant=lambda m, eng: plant(monkeypatch))
    with pytest.raises(AssertionError) as e:
        LT.check_provenance(mod, x0, kw, launches, ln_mode, case)
    msg = str(e.value)
    assert all(w in msg for w in want), msg


# ------------------------------------------------------------------------------------------------------ geometry
def _index_map(gh, gw):
    """float64 [B, 1, gh, gw]: every token's row in the stream, (b gh + y) gw + x."""
    return torch.arange(B * gh * gw, dtype=torch.float64).view(B, 1, gh, gw)


def check_relpos_geometry(case):
    """Each relative-position launch of a traced MaxViT block: the [n, n] bias its oracle adds (GB.relpos_bias of the
    traced table) is the bias the module's eager forward adds, rel_pos_bias(rel_pos_indices) (max_vit.py:247-272), and
    the oracle's windows of the launch's `grid` flag (GB.window_rows) are the module's own _ToWindows of the map."""
    mod, _, kw, launches = run(case, "exact")
    gh, gw = kw["grid"]
    rel = [c for c in launches if c.name == "attention_window_relpos"]
    assert len(rel) == 2
    for c, ai in zip(rel, (2, 6)):
        a = mod.block[ai].fn
        w = a.window_size
        want = a.rel_pos_bias(a.rel_pos_indices).permute(2, 0, 1).double()
        got = GB.relpos_bias(c.pre["table"], w)
        assert torch.equal(got, want), f"{case.name}: layer {ai // 4}: the oracle's bias is not the module's"
        windows = mod.block[ai - 1](_index_map(gh, gw))               # b x y w1 w2 1
        want_rows = windows.reshape(-1, w * w).long()
        got_rows = GB.window_rows(B, gh, gw, w, w, "cpu", dilated=c.pre["grid"])
        assert torch.equal(got_rows, want_rows), \
            f"{case.name}: layer {ai // 4}: the oracle's windows are not the module's"


@pytest.mark.parametrize("name", ["max_vit block + dilated w3 on 6x9", "max_vit block + dilated w2 on 4x4 primed"])
def test_relpos_bias_and_windows_are_the_modules(name):
    check_relpos_geometry(_named(name))


class _Captured(Exception):
    pass


class _Capture(nn.Module):
    """Keeps its input and stops the forward there."""

    def forward(self, t):
        self.seen = t
        raise _Captured


def test_twins_windows_are_the_local_attentions():
    """GB.window_rows of each traced attention_window launch is the window cut of LocalAttention.forward
    (twins_svt.py:104-116), seen at the input of its to_q on the index map."""
    case = _named("twins local 3 global 3 on 6x9 primed")
    mod, _, kw, launches = run(case, "fold")
    gh, gw = kw["grid"]
    for c, (local_attn, *_rest) in zip([c for c in launches if c.name == "attention_window"], mod.layers):
        a = copy.deepcopy(local_attn.fn)
        a.norm, a.to_q = nn.Identity(), _Capture()
        with pytest.raises(_Captured):
            a(_index_map(gh, gw))
        p = c.pre["p"]
        assert torch.equal(GB.window_rows(B, gh, gw, p, p, "cpu"), a.to_q.seen.reshape(-1, p * p).long())


def test_mobile_vit_groups_are_the_modules():
    """GB.group_rows of each traced attention_groups launch is mobile_vit.to_groups (mobile_vit.py:150) of the map."""
    for name in ("mobile_vit groups 2x2 on 4x6", "mobile_vit groups 1x2 on 3x4 primed"):
        _, _, kw, launches = run(_named(name), "exact")
        (gh, gw), (ph, pw) = kw["grid"], kw["groups"]
        for c in (c for c in launches if c.name == "attention_groups"):
            want = mobile_vit.to_groups(_index_map(gh, gw), ph, pw).reshape(B * ph * pw, -1).long()
            assert torch.equal(GB.group_rows(B, gh, gw, c.pre["ph"], c.pre["pw"], "cpu"), want)


def _swapped_digits(w, device):
    r = torch.arange(w * w, device=device)
    u, v = r // w, r % w
    return (u[:, None] - u[None, :] + w - 1) + (v[:, None] - v[None, :] + w - 1) * (2 * w - 1)


def _block_windows_only(orig):
    return lambda B, gh, gw, wh, ww, device, dilated=False: orig(B, gh, gw, wh, ww, device)


@pytest.mark.parametrize("defect", ["relpos offset digits swapped", "block windows for the dilated grid"])
def test_oracle_side_geometry_defect_is_flagged(defect, monkeypatch):
    if defect == "relpos offset digits swapped":
        monkeypatch.setattr(GB, "relpos_index", _swapped_digits)
        want = "the oracle's bias is not the module's"
    else:
        monkeypatch.setattr(GB, "window_rows", _block_windows_only(GB.window_rows))
        want = "layer 1: the oracle's windows are not the module's"
    with pytest.raises(AssertionError, match=want):
        check_relpos_geometry(_named("max_vit block + dilated w3 on 6x9"))


@pytest.mark.parametrize("name", ["crossformer short 3 long 2 on 6x12", "crossformer short 2 long 4 on 8x4 primed"])
def test_dpb_bias_and_windows_are_the_modules(name):
    """Each relative-position launch of a traced CrossFormer: the [n, n] bias its oracle adds (GB.relpos_bias of the
    traced table) is, within the table's fp32 rounding, the bias the module's eager forward adds,
    dpb(_rel_offsets(w))[rel_pos_indices] (crossformer.py:195-215), and the oracle's windows of the launch's `grid`
    flag are crossformer._to_windows (short and long) of the map."""
    mod, _, kw, launches = run(_named(name), "exact")
    gh, gw = kw["grid"]
    rel = [c for c in launches if c.name == "attention_window_relpos"]
    attns = [a for step in mod.layers for a in (step[0], step[2])]
    assert len(rel) == len(attns) > 0
    for c, a in zip(rel, attns):
        w = a.window_size
        with torch.no_grad():
            d = copy.deepcopy(a.dpb).double()
            want = d(crossformer._rel_offsets(w, "cpu").double())[a.rel_pos_indices]
        ref, bnd = LT.dpb_table_reference(a)
        got = GB.relpos_bias(c.pre["table"], w)
        lim = GB.relpos_bias(bnd.t(), w)
        assert ((got - want[None]).abs() <= lim).all(), f"{name}: the oracle's bias is not the module's"
        windows = crossformer._to_windows(_index_map(gh, gw), w, a.attn_type == "long")      # (b x y) 1 w w
        assert torch.equal(GB.window_rows(B, gh, gw, w, w, "cpu", dilated=c.pre["grid"]),
                           windows.reshape(-1, w * w).long()), f"{name}: the oracle's windows are not the module's"


class _CaptureBias(nn.Module):
    """Stands in for a region-to-local Attention: the regional call passes, the windowed call keeps its bias and its
    tokens and stops the forward."""

    def forward(self, x, rel_pos_bias=None):
        if rel_pos_bias is None:
            return torch.zeros_like(x)
        self.bias, self.tokens = rel_pos_bias, x
        raise _Captured


@pytest.mark.parametrize("lh,lw,rh,rw,W", [(6, 8, 2, 2, 4), (7, 4, 1, 1, 7), (4, 6, 2, 3, 3)])
def test_region_local_bias_and_windows_are_the_modules(lh, lw, rh, rw, W):
    """GB.region_bias (the column-major index of b200vit_attention_region_local) of the table the engine prepares is the
    bias R2LTransformer's eager forward adds (bias_indices, regionvit.py:260-270), and GB.region_window_rows is the
    window the eager forward builds from the local map and its region token (regionvit.py:279-284), on index maps."""
    torch.manual_seed(0)
    mod = regionvit.R2LTransformer(D, window_size=W, depth=1, heads=2).eval()
    t = mod.engine().prepared()
    m = copy.deepcopy(mod)
    m.layers[0][0] = _CaptureBias()
    local = torch.arange(B * lh * lw, dtype=torch.float64).view(B, 1, lh, lw)
    region = (B * lh * lw + torch.arange(B * rh * rw, dtype=torch.float64)).view(B, 1, rh, rw)
    with torch.no_grad(), pytest.raises(_Captured):
        m.forward_eager(local, region)
    cap = m.layers[0][0]
    bias = GB.region_bias(t["0.r2l"], lh // rh, lw // rw, W)
    assert torch.equal(bias[None], cap.bias.double()), "the oracle's bias is not the module's"
    assert torch.equal(GB.region_window_rows(B, lh, lw, rh, rw, "cpu"), cap.tokens[..., 0].long())


class _Ones(nn.Module):
    def forward(self, t):
        return torch.ones_like(t)


@pytest.mark.parametrize("name", [SCALABLE_A, SCALABLE_B])
def test_iwsa_windows_are_the_modules(name):
    """GB.window_rows of each traced attention_iwsa launch (its wh x ww) is the window cut of
    InteractiveWindowedSelfAttention.forward's windows() (scalable_vit.py:180-187) on the index map, seen in its
    scores with q the map, k ones and scale 1: score (i, j) of window w is the map row of its token i."""
    mod, _, kw, launches = run(_named(name), "exact")
    gh, gw = kw["grid"]
    iwsa = [c for c in launches if c.name == "attention_iwsa"]
    assert len(iwsa) == len(mod.layers) > 0
    for c, layer in zip(iwsa, mod.layers):
        a = copy.deepcopy(layer[4])
        a.norm, a.to_q, a.to_k, a.to_v, a.local_interactive_module = (nn.Identity(), nn.Identity(), _Ones(),
                                                                       nn.Identity(), nn.Identity())
        a.scale, a.attend = 1.0, _Capture()
        with torch.no_grad(), pytest.raises(_Captured):
            a(_index_map(gh, gw).expand(-1, a.heads, -1, -1))
        got = a.attend.seen[:, 0, :, 0].long()                            # (b x y), heads, w1 w2, w1 w2
        assert torch.equal(GB.window_rows(B, gh, gw, c.pre["wh"], c.pre["ww"], "cpu"), got), \
            f"{name}: the oracle's windows are not the module's"


def check_ssa_key_patches(mod, kw, launches):
    """The key / value operands the walk derives for each SSA -- GB.im2col_reference of the traced key-patch
    conv_im2col_nhwc launch (the oracle of that kernel's addresses) times the module's to_k (heads padded) | to_v
    weights in tap order -- are to_k's and to_v's own Conv2d of the map (scalable_vit.py:127-128, 138), exactly, on an
    integer map (the weights are multiples of 1/64: every sum is exact in fp64)."""
    gh, gw = kw["grid"]
    patches = [c for c in launches if c.name == "conv_im2col_nhwc" and c.pre["p"] == 0]
    refs = [R for R in LT.module_layers(mod) if R.grid["kind"] == "strided"]
    assert len(patches) == len(refs) == len(mod.layers) > 0
    x = torch.randint(-8, 9, (B * gh * gw, D), generator=torch.Generator().manual_seed(1)).double()
    xm = x.view(B, gh, gw, D).permute(0, 3, 1, 2)
    for c, R, (ssa, *_rest) in zip(patches, refs, mod.layers):
        a = c.pre
        col = GB.im2col_reference(x, a["B"], a["H"], a["W"], a["k"], a["s"], a["p"])
        kvw = R.grid["kv"].double()
        got = col @ kvw.permute(0, 2, 3, 1).reshape(kvw.shape[0], -1).t()
        H, dk, dp = ssa.heads, ssa.to_q.out_channels // ssa.heads, R.dim_head
        with torch.no_grad():
            k, v = (copy.deepcopy(m).double()(xm).permute(0, 2, 3, 1).reshape(got.shape[0], -1)
                    for m in (ssa.to_k, ssa.to_v))
        heads = got[:, :H * dp].reshape(-1, H, dp)
        assert torch.equal(heads[..., :dk].reshape(-1, H * dk), k), "the oracle's key patches are not to_k's"
        assert (heads[..., dk:] == 0).all(), "a padded key column is not zero"
        assert torch.equal(got[:, H * dp:], v), "the oracle's key patches are not to_v's"


def test_ssa_key_patches_are_the_modules_convolutions():
    mod, _, kw, launches = run(_named(SCALABLE_A), "exact")
    check_ssa_key_patches(mod, kw, launches)


def _im2col_channel_major(x, B, H, W, k, s, pad):
    """im2col with its columns in (channel, tap row, tap column) order, the Conv2d weight's own."""
    C = x.shape[1]
    cols = torch.nn.functional.unfold(x.reshape(B, H, W, C).permute(0, 3, 1, 2).double(), k, padding=pad, stride=s)
    return cols.permute(0, 2, 1).reshape(-1, C * k * k)


def test_oracle_side_key_patch_defect_is_flagged(monkeypatch):
    mod, _, kw, launches = run(_named(SCALABLE_A), "exact")
    monkeypatch.setattr(GB, "im2col_reference", _im2col_channel_major)
    with pytest.raises(AssertionError, match="the oracle's key patches are not to_k's"):
        check_ssa_key_patches(mod, kw, launches)


@pytest.mark.parametrize("name", [SEP, "sep_vit single window on 7x7 primed"])
def test_sep_vit_windows_are_the_modules(name):
    """GB.window_rows of each traced attention_window_token launch -- the windows, and their order, that its oracle
    (window_token_reference) and window_mix's (mix_reference) read -- is DSSA.forward's window cut and window order
    with the window token first (sep_vit.py:178-184), seen at the input of its to_qkv on the index map."""
    mod, _, kw, launches = run(_named(name), "exact")
    gh, gw = kw["grid"]
    wt = [c for c in launches if c.name == "attention_window_token"]
    assert len(wt) == len(mod.layers) > 0
    for c, (attn, _ff) in zip(wt, mod.layers):
        a = copy.deepcopy(attn)
        a.norm, a.to_qkv = nn.Identity(), _Capture()
        a.window_tokens = nn.Parameter(torch.full((1,), -1.0, dtype=torch.float64))
        with torch.no_grad(), pytest.raises(_Captured):
            a(_index_map(gh, gw))
        seen = a.to_qkv.seen                                                   # (b x y), 1, 1 + w1 w2
        p = c.pre["p"]
        assert (seen[:, 0, 0] == -1).all(), f"{name}: the window token is not each window's first token"
        assert torch.equal(GB.window_rows(B, gh, gw, p, p, "cpu"), seen[:, 0, 1:].long()), \
            f"{name}: the oracle's windows are not the module's"
