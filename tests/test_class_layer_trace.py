"""The remaining fused encoders traced back to their reference layers without a GPU (oracle/layer_trace.py, as
tests/test_layer_trace.py does for the sequence families): SimpleViT, flash-attention SimpleViT, PiT and NesT through
run_blocks; CrossViT's MultiScaleEncoder through engine.fused_two_streams (each branch's layers, its final LayerNorm,
both class-attention directions, with and without the projection between the widths); the class-attention stage of
CaiT (talking heads, layer subsets) and XCiT through their forward_fused after the patch embedding; and LeViT's whole forward_fused (stem,
folded BatchNorms, position-bias attention with a downsampling layer, Hardswish feed-forward, pooled head with a
distill head).

Every case runs in both LayerNorm modes with per-LayerNorm eps (test_layer_trace.set_eps) and BatchNorm eps 1e-3; the
provenance walk must accept every launch and the emulated outputs must sit within their bounds.  Planted wiring and
weight-preparation defects must be named by layer, launch and operand.  A completeness guard holds every fused encoder
class of the package to a traced case here or in the other two trace files."""
import importlib
import inspect
import pkgutil
import textwrap

import pytest
import torch

import test_grid_layer_trace as G
import test_layer_trace as T
import vit_pytorch_b200
from oracle import grid_attention_bounds as GB
from oracle import layer_trace as LT
from test_layer_trace import lib, make  # noqa: F401  (lib: the module fixture that builds the library)
from vit_pytorch_b200 import cait, cross_vit, engine, levit, xcit

S = LT.schedule()
D, HEADS, DH, MLP = S.D, S.HEADS, S.DH, S.MLP
B = 2


def _nest():
    from vit_pytorch_b200.nest import Transformer
    return Transformer(D, 16, 2, HEADS, 2)


def _m(path, *args, **kw):
    def build():
        mod, cls = path.rsplit(".", 1)
        return getattr(importlib.import_module(f"vit_pytorch_b200.{mod}"), cls)(*args, **kw)
    return build


# run_blocks cases, as make_engine_schedule.CASES
BLOCK_CASES = [
    S.Case("simple_vit", _m("simple_vit.Transformer", D, 2, HEADS, DH, MLP), B * 16,
           lambda: dict(B=B, N=16, primed=True), True),
    S.Case("simple_flash_attn_vit", _m("simple_flash_attn_vit.Transformer", D, 2, HEADS, DH, MLP, True), B * 16,
           lambda: dict(B=B, N=16), True),
    S.Case("pit stage", _m("pit.Transformer", D, 2, HEADS, DH, MLP), B * 17, lambda: dict(B=B, N=17, primed=True),
           True),
    # 2 images of 2 x 2 blocks of 4 x 4 tokens
    S.Case("nest level", _nest, 4 * B * 16, lambda: dict(B=4 * B, N=16, primed=True), True),
]


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("case", BLOCK_CASES, ids=[c.name for c in BLOCK_CASES])
def test_every_block_launch_traces_back_to_the_reference_layer(case, ln_mode):
    mod, x0, kw, launches = T.run(case, ln_mode)
    assert LT.check_provenance(mod, x0, kw, launches, ln_mode, case.name) == len(launches) > 0
    LT.check_accuracy(launches, f"{case.name} | {ln_mode}")


# ------------------------------------------------------------------------------------------------------ class attention
def _mse(sm_dim, lg_dim, cross_depth=2):
    enc = dict(depth=1, heads=HEADS, mlp_dim=MLP, dim_head=DH)
    return lambda: cross_vit.MultiScaleEncoder(depth=2, sm_dim=sm_dim, lg_dim=lg_dim, sm_enc_params=enc,
                                               lg_enc_params=dict(enc, mlp_dim=2 * MLP), cross_attn_heads=HEADS,
                                               cross_attn_depth=cross_depth, cross_attn_dim_head=DH)


# name: (module, sm rows per image, lg rows per image, primed)
CROSS_VIT = {
    "cross_vit projection sm 64 lg 96 cross depth 2": (_mse(D, 96), 17, 10, False),
    "cross_vit same width primed": (_mse(D, D, cross_depth=1), 10, 5, True),
}


def _streams(name, mse, ln_mode, plant=None):
    """(module, xs, xl, launches) of one emulated fused_two_streams call."""
    _, Ns, Nl, primed = CROSS_VIT[name]
    if plant is not None:
        plant(mse)
    g = torch.Generator().manual_seed(len(name))
    Ds, Dl = mse.layers[0][0].norm.normalized_shape[0], mse.layers[0][1].norm.normalized_shape[0]
    xs, xl = torch.randn(B * Ns, Ds, generator=g), torch.randn(B * Nl, Dl, generator=g)
    xs0, xl0 = xs.clone(), xl.clone()
    stages = mse.stages()

    def setup():
        for es, el, _, _ in stages[:1]:
            for eng, x in ((es, xs), (el, xl)):
                for buf in eng.workspace(x.shape[0], x.device).values():
                    buf.fill_(float("nan"))
                if primed:
                    xb, st = eng.entry_buffers(x.shape[0], x.device)
                    if xb is not None:
                        LT.prime_exact(x, xb, st)
    launches = LT.trace_call(lambda: engine.fused_two_streams(stages, xs, xl, B, Ns, Nl, primed,
                                                              mse.cls_rows(B, Ns, Nl, xs.device)),
                             ln_mode, LT.emulate_impl, setup=setup)
    return xs0, xl0, launches


def run_cross_vit(name, ln_mode, plant=None):
    mse = make(S.Case(name, CROSS_VIT[name][0], 0, dict, False))
    xs0, xl0, launches = _streams(name, mse, ln_mode, plant)
    return mse, xs0, xl0, launches


def check_cross_vit(name, ln_mode, mse, xs0, xl0, launches):
    _, Ns, Nl, primed = CROSS_VIT[name]
    return LT.check_cross_vit_provenance(mse, xs0, xl0, B, Ns, Nl, primed, launches, ln_mode, name)


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("name", list(CROSS_VIT))
def test_cross_vit_launches_trace_back_to_the_reference_layers(name, ln_mode):
    mse, xs0, xl0, launches = run_cross_vit(name, ln_mode)
    assert check_cross_vit(name, ln_mode, mse, xs0, xl0, launches) == len(launches) > 0
    kinds = {c.name for c in launches}
    assert "attention_cls" in kinds and "layernorm" in kinds
    LT.check_accuracy(launches, f"{name} | {ln_mode}")


def embedded(mp, x0, prime):
    """PatchEmbedEngine.run replaced by the stream x0 (the patch embedding is not part of these walks): a fresh copy of
    x0 and, when the caller passes them, its bf16 copy and row statistics written by prime(x, xb, stats)."""
    def run(self, img, xb=None, stats=None, patch=None, pos=None):
        x = x0.clone()
        if xb is not None:
            prime(x, xb, stats)
        return x, img.shape[0], x0.shape[0] // img.shape[0]
    mp.setattr(engine.PatchEmbedEngine, "run", run)


def trace_class_model(mp, model, img, x0, ln_mode, impl=LT.emulate_impl, prime=LT.prime_exact):
    """(launches, logits) of model.forward_fused(img) -- CaiT or XCiT -- after its patch embedding, which yields x0."""
    enc = getattr(model, "xcit_transformer", None) or model.patch_transformer
    embedded(mp, x0, prime)
    outs = []

    def setup():
        for buf in enc.engine().workspace(x0.shape[0], x0.device).values():
            buf.fill_(float("nan"))
    launches = LT.trace_call(lambda: outs.append(model.forward_fused(img)), ln_mode, impl, setup=setup)
    return launches, outs[0]


def _kept(model, patch, cls):
    """The layers each stage runs, fixed as layer dropout would draw them (cait.py:14-27); and set_eps on each stage
    (the patch LayerNorm of the embedding is wider than the model, so set_eps of the whole model would give every
    LayerNorm of the stages one eps)."""
    enc = getattr(model, "xcit_transformer", None) or model.patch_transformer
    T.set_eps(enc)
    T.set_eps(model.cls_transformer)
    enc.kept_layers = lambda: list(patch)
    model.cls_transformer.kept_layers = lambda: list(cls)
    return model


# name: (model, image (h, w), patch grid (h, w), layers the patch encoder runs, layers the class stage runs)
CLASS_MODELS = {
    "cait layer subsets": (lambda: cait.CaiT(image_size=32, patch_size=8, num_classes=10, dim=D, depth=3, cls_depth=3,
                                             heads=4, mlp_dim=MLP, dim_head=DH), (32, 32), (4, 4), [0, 2], [0, 2]),
    "xcit class depth 2": (lambda: xcit.XCiT(image_size=32, patch_size=8, num_classes=10, dim=D, depth=2, cls_depth=2,
                                             heads=HEADS, mlp_dim=MLP, dim_head=DH), (24, 32), (3, 4), [0, 1], [0, 1]),
}


def run_class_model(mp, name, ln_mode, plant=None):
    """(model, x0, launches) of one emulated CaiT or XCiT forward_fused after the patch embedding."""
    build, (ih, iw), (gh, gw), patch, cls = CLASS_MODELS[name]
    model = _kept(make(S.Case(name, build, 0, dict, False)), patch, cls)
    if plant is not None:
        plant(model)
    g = torch.Generator().manual_seed(len(name))
    img = torch.randn(B, 3, ih, iw, generator=g).bfloat16()
    x0 = torch.randn(B * gh * gw, D, generator=g)
    launches, _ = trace_class_model(mp, model, img, x0, ln_mode)
    return model, x0, launches


def check_class_model(name, ln_mode, model, x0, launches):
    return LT.check_class_stage_provenance(model, x0, B, CLASS_MODELS[name][2], launches, ln_mode, name)


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("name", list(CLASS_MODELS))
def test_class_attention_stage_traces_back_to_the_reference_layers(name, ln_mode, monkeypatch):
    model, x0, launches = run_class_model(monkeypatch, name, ln_mode)
    assert check_class_model(name, ln_mode, model, x0, launches) == len(launches) > 0
    assert sum(c.name.startswith("attention_cls") for c in launches) == len(CLASS_MODELS[name][4])
    for stage in (getattr(model, "xcit_transformer", None) or model.patch_transformer, model.cls_transformer):
        eps = [m.eps for m in stage.modules() if isinstance(m, torch.nn.LayerNorm)]
        assert len(set(eps)) == 3, eps
    LT.check_accuracy(launches, f"{name} | {ln_mode}")


# ------------------------------------------------------------------------------------------------------ LeViT
LEVIT = {
    # an 80 x 80 image: a 5 x 5 map, a downsampling layer to 3 x 3 (odd: the last query row and column at 4), a
    # distill head
    "levit downsampling distill": dict(image_size=80, num_classes=10, dim=(D, 96), depth=(2, 1), heads=(2, 3),
                                       mlp_mult=2, stages=2, dim_key=16, dim_value=32, num_distill_classes=7),
    "levit 3 stages": dict(image_size=64, num_classes=5, dim=(D, 96, 128), depth=1, heads=2, mlp_mult=2, stages=3,
                           dim_key=32, dim_value=32),
}


def run_levit(name, ln_mode="fold", plant=None):
    mod = make(S.Case(name, lambda: levit.LeViT(**LEVIT[name]), 0, dict, False))
    if plant is not None:
        plant(mod)
    s = LEVIT[name]["image_size"]
    img = torch.randn(B, 3, s, s, generator=torch.Generator().manual_seed(s)).bfloat16()
    launches = LT.trace_call(lambda: mod.forward_fused(img), ln_mode, LT.emulate_impl)
    return mod, img, launches


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("name", list(LEVIT))
def test_levit_forward_traces_back_to_the_reference(name, ln_mode):
    mod, img, launches = run_levit(name, ln_mode)
    assert LT.check_levit_provenance(mod, img, launches, name) == len(launches) > 0
    assert sum(c.name == "attention_posbias" and c.args["s"] == 2 for c in launches) == len(LEVIT[name]["dim"]) - 1
    LT.check_accuracy(launches, f"{name} | {ln_mode}")


def test_levit_pos_indices_are_the_kernels_bias_addresses():
    """The module's own pos_indices (levit.py:114-126, the reference's bias look-up) equal the kernel's address
    formula GB.posbias_index for the full-grid and the strided queries, at even and odd map sizes."""
    for F, down in ((4, False), (5, True), (7, True), (6, True)):
        a = levit.Attention(D, fmap_size=F, heads=2, dim_key=16, dim_value=32, downsample=down)
        assert torch.equal(a.pos_indices, GB.posbias_index(F, a.stride)), (F, down)


# ------------------------------------------------------------------------------------------------------ planted defects
def _source_patched(mp, cls, name, old, new):
    """cls.name recompiled from its own source with `old` replaced by `new` (exactly once)."""
    fn = getattr(cls, name)
    src = textwrap.dedent(inspect.getsource(fn))
    assert src.count(old) == 1, (name, old)
    ns = {}
    exec(compile(src.replace(old, new), inspect.getsourcefile(fn), "exec"), vars(inspect.getmodule(fn)), ns)
    mp.setattr(cls, name, ns[name])


def _context_with_cls(mp):
    _source_patched(mp, engine, "fused_two_streams", "sm_lg.run(x[0], xb[0], Ns, xb[1], Nl, B, rows[0])",
                    "sm_lg.run(x[0], xb[0], Ns, xb[1], Nl, B, rows[0], skip=0)")


def _other_layers_context(mp):
    _source_patched(mp, engine.CrossAttentionEngine, "run", "ctx_i = ctx[:, 2 * I * i:2 * I * (i + 1)]",
                    "ctx_i = ctx[:, :2 * I]")


def _talking_heads_swapped(mp):
    _source_patched(mp, engine.CrossAttentionEngine, "run", 't[f"{i}.pre"], t[f"{i}.post"])',
                    't[f"{i}.post"], t[f"{i}.pre"])')


def _class_subset_wrong_layer(mp):
    _source_patched(mp, engine.CrossAttentionEngine, "run", "for i in range(len(self.layers)) if layers is None else "
                    "layers:", "for i in range(len(self.layers)) if layers is None else range(len(layers)):")


def _levit_bn_default_eps(mp):
    orig = levit.fold_bn

    def bad(w, b, bn):
        saved = bn.eps
        bn.eps = 1e-5
        try:
            return orig(w, b, bn)
        finally:
            bn.eps = saved
    mp.setattr(levit, "fold_bn", bad)


def _levit_query_grid_indices(mod):
    """The downsampling layer's pos_indices built on the query grid, query (i, j) at (i, j) and not at (2 i, 2 j): the
    module's reference look-up no longer matches the kernel's addresses."""
    a = mod.backbone[1].layers[0][0]
    F, Fq = a.fmap_size, -(-a.fmap_size // 2)
    qy, qx = torch.meshgrid(torch.arange(Fq), torch.arange(Fq), indexing="ij")
    ky, kx = torch.meshgrid(torch.arange(F), torch.arange(F), indexing="ij")
    a.pos_indices.copy_((qy.reshape(-1, 1) - ky.reshape(1, -1)).abs() * F
                        + (qx.reshape(-1, 1) - kx.reshape(1, -1)).abs())


def _levit_queries_unstrided(mp):
    _source_patched(mp, levit.LeViT, "forward_fused", "B, F, s, Hh, dk, dv", "B, F, 1, Hh, dk, dv")


def _final_norm_kept_stream(mp):
    _source_patched(mp, engine, "fused_two_streams", "x[b], spare[b] = spare[b], x[b]", "pass")


def _cait_context_skips_a_row(mp):
    _source_patched(mp, cait.CaiT, "forward_fused", "skip=0,", "skip=1,")


def _xcit_context_before_final_norm(mp):
    _source_patched(mp, xcit.XCiT, "forward_fused", "_lib.layernorm(x, g, bt, out_bf16=ctx, eps=fn.eps)",
                    "_lib.cast_f32_bf16(x.view(-1), ctx.view(-1))")


def _context_gemm_gelu(mp):
    _source_patched(mp, engine.CrossAttentionEngine, "run", '_lib.gemm(xbb, t["ctx.w"], out_bf16=ctx)',
                    '_lib.gemm(xbb, t["ctx.w"], out_bf16=ctx, gelu=True)')


def _levit_out_gemm_gelu(mp):
    _source_patched(mp, levit.LeViT, "forward_fused", 'bias=t[p + "out.b"], resid=x)',
                    'bias=t[p + "out.b"], resid=x, gelu=True)')


CROSS_CASE = "cross_vit projection sm 64 lg 96 cross depth 2"
LEVIT_CASE = "levit downsampling distill"
# name: (kind, case, LayerNorm mode, plant(monkeypatch), plant(module), what the failure must name)
DEFECTS = {
    "the class attention's context includes the other stream's cls row":
        ("cross_vit", CROSS_CASE, "fold", _context_with_cls, None,
         ("block 0 sm attends lg layer 0 attention", "operand first")),
    "a class-attention layer reads another layer's slice of the stacked context GEMM":
        ("cross_vit", CROSS_CASE, "exact", _other_layers_context, None,
         ("block 0 sm attends lg layer 1 attention", "operand ctx")),
    "CrossViT block's final LayerNorm does not replace the stream":
        ("cross_vit", CROSS_CASE, "fold", _final_norm_kept_stream, None,
         ("block 0 sm attends lg layer 0 project_out", "operand resid")),
    "talking heads pre and post swapped":
        ("class", "cait layer subsets", "fold", _talking_heads_swapped, None,
         ("layer 0 attention", "attention_cls_headmix", "operand pre")),
    "class attention's LayerScale on the rows but not the bias":
        ("class", "xcit class depth 2", "fold", T._layerscale_rows_only, None, ("layer 0 out", "operand bias")),
    "class-attention layer subset runs the wrong layer":
        ("class", "cait layer subsets", "exact", _class_subset_wrong_layer, None, ("layer 2 qkv", "operand gamma")),
    "CaiT's class attention skips the first patch row of the context":
        ("class", "cait layer subsets", "fold", _cait_context_skips_a_row, None,
         ("layer 0 attention", "operand first")),
    "XCiT's class attention reads the patch rows before final_norm":
        ("class", "xcit class depth 2", "exact", _xcit_context_before_final_norm, None,
         ("context (final_norm)", "cast_f32_bf16", "layernorm expected")),
    "the stacked context GEMM applies GELU":
        ("class", "cait layer subsets", "fold", _context_gemm_gelu, None, ("context", "operand gelu")),
    "LeViT BatchNorm folded with the default eps":
        ("levit", LEVIT_CASE, "fold", _levit_bn_default_eps, None,
         ("transformer 0 layer 0 qkv", "launch 8 gemm", "operand w ([to_q; to_k; to_v]")),
    "LeViT's downsampling attention run with unstrided queries":
        ("levit", LEVIT_CASE, "fold", _levit_queries_unstrided, None,
         ("transformer 1 layer 0 attention", "attention_posbias", "operand s (to_q's stride)")),
    "LeViT's to_out GEMM applies GELU":
        ("levit", LEVIT_CASE, "exact", _levit_out_gemm_gelu, None, ("transformer 0 layer 0 out", "operand gelu")),
    "LeViT's pos_indices built on the query grid, not the kernel's key-grid addresses":
        ("levit", LEVIT_CASE, "fold", None, _levit_query_grid_indices,
         ("transformer 1 layer 0 attention", "attention_posbias", "operand table (pos_indices)")),
}


@pytest.mark.parametrize("name", list(DEFECTS))
def test_planted_defect_is_named(name, monkeypatch):
    kind, case, ln_mode, plant, plant_mod, want = DEFECTS[name]
    if plant is not None:
        plant(monkeypatch)
    with pytest.raises(AssertionError) as e:
        if kind == "cross_vit":
            mse, xs0, xl0, launches = run_cross_vit(case, ln_mode, plant_mod)
            check_cross_vit(case, ln_mode, mse, xs0, xl0, launches)
        elif kind == "class":
            model, x0, launches = run_class_model(monkeypatch, case, ln_mode, plant_mod)
            check_class_model(case, ln_mode, model, x0, launches)
        else:
            mod, img, launches = run_levit(case, ln_mode, plant_mod)
            LT.check_levit_provenance(mod, img, launches, case)
    msg = str(e.value)
    assert isinstance(e.value, LT.ProvenanceError), msg
    assert all(w in msg for w in want), msg


# ------------------------------------------------------------------------------------------------------ completeness
def _package_classes():
    for info in pkgutil.iter_modules(vit_pytorch_b200.__path__):
        mod = importlib.import_module(f"vit_pytorch_b200.{info.name}")
        for _, cls in inspect.getmembers(mod, inspect.isclass):
            if cls.__module__ == mod.__name__:
                yield cls


def _own_layer_loop(cls) -> bool:
    """A class whose fused forward launches an attention kernel itself rather than through an engine (LeViT)."""
    fwd = cls.__dict__.get("forward_fused")
    return fwd is not None and "_lib.attention" in inspect.getsource(fwd)


def _traced_modules():
    """(run_blocks modules, class-attention modules, own-loop modules) of every traced case of the three trace files."""
    blocks = [make(c) for c in T.CASES + G.CASES + BLOCK_CASES]
    cross = []
    for name, (build, _, _, _) in CROSS_VIT.items():
        mse = build()
        cross.append(mse)
        for sm, lg, ct in mse.layers:
            blocks += [sm, lg]
            cross.append(ct)
    cross += [build().cls_transformer for build, *_ in CLASS_MODELS.values()]
    own = [levit.LeViT(**kw) for kw in LEVIT.values()]
    return blocks, cross, own


def test_every_fused_encoder_class_has_a_traced_case():
    blocks, cross, own = _traced_modules()
    for m in blocks:                                    # a reference layer table: module_layers names a missing one
        LT.module_layers(m)
    for m in cross:
        if hasattr(m, "cross_layers"):
            LT.cross_module_layers(m)
    missing = []
    for cls in _package_classes():
        if cls is engine.FusedEncoder:
            continue
        if issubclass(cls, engine.FusedEncoder) and not any(isinstance(m, cls) for m in blocks):
            missing.append(f"{cls.__module__}.{cls.__name__} (FusedEncoder)")
        if "cross_layers" in vars(cls) and not any(isinstance(m, cls) for m in cross):
            missing.append(f"{cls.__module__}.{cls.__name__} (cross_layers)")
        if _own_layer_loop(cls) and not any(isinstance(m, cls) for m in own):
            missing.append(f"{cls.__module__}.{cls.__name__} (its own layer loop)")
    assert not missing, f"fused encoder classes without a traced case: {', '.join(missing)}"


def test_the_guard_sees_every_kind():
    classes = list(_package_classes())
    assert levit.LeViT in classes and _own_layer_loop(levit.LeViT)
    assert {cross_vit.CrossTransformer, cait.Transformer, xcit.Transformer} <= {
        c for c in classes if "cross_layers" in vars(c)}
