"""Each launch of TransformerEngine.run_blocks traced back to the reference layer without a GPU (oracle/layer_trace.py).

Every _lib entry point is replaced by an emulation that writes the fp64 reference of the kernel's existing oracle into
its outputs, rounded to their dtype, and torch.cuda.current_stream is stubbed as in
tests/golden/make_engine_schedule.py.  Each launch schedule case (and a post-norm CCT case) runs in both LayerNorm
modes with per-LayerNorm eps of 1e-5, 1e-6 and 1e-3 in turn, so that a swapped eps is a wrong argument; the
provenance walk must accept every launch, and the emulated outputs must sit within their bounds.  Then each wiring or
weight-preparation defect that moves a model's logits by less than its parity tolerance is planted in the engine, and
the walk must name the launch and the operand it corrupts."""
import dataclasses

import pytest
import torch
from torch import nn

from oracle import layer_trace as LT
from vit_pytorch_b200 import _lib, build, engine

S = LT.schedule()
EPS = (1e-5, 1e-6, 1e-3)


@pytest.fixture(scope="module", autouse=True)
def lib():
    # _lib.stats_parts, which sizes the workspace, is the real library call
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def _cct():
    from vit_pytorch_b200.cct import TransformerClassifier
    return TransformerClassifier(seq_pool=True, embedding_dim=S.D, num_layers=2, num_heads=S.HEADS, mlp_ratio=2.0,
                                 num_classes=3, dropout_rate=0.0, attention_dropout=0.0, stochastic_depth_rate=0.0,
                                 positional_embedding="none")


CASES = S.CASES + [S.Case("cct post-norm", _cct, 2 * 17, lambda: dict(B=2, N=17), False)]


def _case(name):
    return next(c for c in CASES if c.name == name)


def _ln_width(m):
    """The width of a LayerNorm: nn.LayerNorm's, or the channels of a channel LayerNorm over an NCHW map (Twins-SVT,
    CvT: `g` of shape (1, dim, 1, 1) and `eps`); None for any other module."""
    if isinstance(m, nn.LayerNorm):
        return m.normalized_shape[0]
    if isinstance(getattr(m, "g", None), nn.Parameter) and isinstance(getattr(m, "eps", None), float):
        return m.g.numel()
    return None


def set_eps(mod):
    """The LayerNorms over the model width take eps 1e-5, 1e-6, 1e-3 in module order, the narrower ones (q / k head
    norms, DeepViT's norm over heads) 1e-6."""
    norms = [m for m in mod.modules() if _ln_width(m) is not None]
    width = max(_ln_width(m) for m in norms) if norms else 0
    j = 0
    for m in norms:
        if _ln_width(m) == width:
            m.eps, j = EPS[j % len(EPS)], j + 1
        else:
            m.eps = EPS[1]


def make(case):
    """The case's module with per-LayerNorm eps (set_eps) and BatchNorm eps 1e-3."""
    mod = S.build(case)
    set_eps(mod)
    for m in mod.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.eps = 1e-3
    return mod


def run(case, ln_mode, plant=None, call=None):
    """(module, x before run_blocks, run_blocks' arguments, traced launches) of one emulated run; plant(mod, eng) runs
    before it; call(mod, x, kw) in place of eng.run_blocks(x, **kw) (LT.trace)."""
    mod = make(case)
    eng = mod.engine()
    if plant is not None:
        plant(mod, eng)
    x = torch.randn(case.rows, S.D, generator=torch.Generator().manual_seed(len(case.name)))
    kw = case.kwargs()
    x0 = x.clone()
    launches = LT.trace(eng, x, kw, ln_mode, LT.emulate_impl, prime=LT.prime_exact,
                        call=None if call is None else lambda: call(mod, x, kw))
    return mod, x0, kw, launches


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_every_launch_traces_back_to_the_reference_layer(case, ln_mode):
    mod, x0, kw, launches = run(case, ln_mode)
    assert LT.check_provenance(mod, x0, kw, launches, ln_mode, case.name) == len(launches) > 0
    # the emulated outputs are their references rounded once: within every bound the GPU test applies
    LT.check_accuracy(launches, f"{case.name} | {ln_mode}")


def test_every_case_eps_differs_between_its_layer_norms():
    for case in CASES:
        layers, _ = make(case).encoder_layers()
        if not case.name.startswith("navit varlen"):          # NaViT's LayerNorm is F.layer_norm's, eps 1e-5
            assert all(L.ln1.eps != L.ln2.eps for L in layers), case.name


# ------------------------------------------------------------------------------------------------------ planted defects
def _fc1_reads_stats_a(mp):
    orig = engine.BlocksCall.stream_copy

    def bad(self, slot):
        r = orig(self, slot)
        if slot == "stats_b":
            self.sums = self.ws["stats_a"]
        return r
    mp.setattr(engine.BlocksCall, "stream_copy", bad)


def _qkv_gets_ln2_eps(mp, eng):
    orig = engine.BlocksCall.normed

    def bad(self, src, ln, norm, w, out, **epi):
        if w.endswith(".qkv"):
            norm = norm._replace(eps=eng.layers[int(w.split(".")[0])].ln2.eps)
        return orig(self, src, ln, norm, w, out, **epi)
    mp.setattr(engine.BlocksCall, "normed", bad)


def _colsum_unrounded(mp):
    orig = engine._fold

    def bad(t, prefix, w, b, ln):
        orig(t, prefix, w, b, ln)
        t[prefix + ".s"] = (w.detach().float() * ln.gamma.detach().float()[None, :]).sum(dim=1).contiguous()
    mp.setattr(engine, "_fold", bad)


def _layerscale_rows_only(mp):
    orig = engine._scaled_rows

    def bad(w, b, scale):
        ws, bs = orig(w, b, scale)
        return ws, (bs if scale is None or b is None else b.detach().float().contiguous())
    mp.setattr(engine, "_scaled_rows", bad)


def _subset_wrong_layer(mp):
    orig = engine.TransformerEngine.run_blocks

    def bad(self, x, *args, layers=None, **kw):
        return orig(self, x, *args, layers=None if layers is None else list(range(len(layers))), **kw)
    mp.setattr(engine.TransformerEngine, "run_blocks", bad)


def _one_lsa_temperature(mp):
    from vit_pytorch_b200 import vit_for_small_dataset as V
    orig = V.Transformer.encoder_layers

    def bad(self):
        layers, norm = orig(self)
        return [dataclasses.replace(L, scale=layers[0].scale) for L in layers], norm
    mp.setattr(V.Transformer, "encoder_layers", bad)


def _bn_default_eps(mp):
    orig = engine.lpi_weights
    mp.setattr(engine, "lpi_weights", lambda P: orig(P._replace(bn_eps=1e-5)))


def _swapped_layer_norms(mp):
    from vit_pytorch_b200 import vit as V
    orig = V.Transformer.encoder_layers

    def bad(self):
        layers, norm = orig(self)
        return [layers[0], dataclasses.replace(layers[1], ln1=layers[1].ln2, ln2=layers[1].ln1)], norm
    mp.setattr(V.Transformer, "encoder_layers", bad)


def _exact_gemm_reads_o(mp):
    orig = engine.BlocksCall.normed

    def bad(self, src, ln, norm, w, out, **epi):
        if self.fold:
            return orig(self, src, ln, norm, w, out, **epi)
        t = self.t
        _lib.layernorm(src, t[ln + ".w"], t[ln + ".b"], out_bf16=self.xb, eps=norm.eps)
        fn = _lib.gemm_headnorm if "head_gamma" in epi else _lib.gemm
        fn(self.o, t[w + ".w"], out_bf16=out, bias=t.get(w + ".b"), **epi)
    mp.setattr(engine.BlocksCall, "normed", bad)


# name: (case, LayerNorm mode, plant(monkeypatch, engine), what the failure must name)
DEFECTS = {
    "fc1 LayerNorm reads the statistics from before the attention residual":
        ("vit cls primed", "fold", lambda mp, eng: _fc1_reads_stats_a(mp), ("layer 0 fc1", "operand ln_sums")),
    "QKV GEMM gets ln2's eps":
        ("vit cls", "fold", _qkv_gets_ln2_eps, ("layer 0 qkv", "operand ln_eps")),
    "fold column sums from the unrounded gamma W":
        ("simple_vit qk rmsnorm", "fold", lambda mp, eng: _colsum_unrounded(mp), ("layer 0 qkv", "operand col_s")),
    "LayerScale on the rows but not the bias":
        ("cait layer subset", "fold", lambda mp, eng: _layerscale_rows_only(mp), ("layer 0 out", "operand bias")),
    "layer subset runs the wrong layer's weights":
        ("cait layer subset", "fold", lambda mp, eng: _subset_wrong_layer(mp), ("layer 2 qkv", "operand ln_eps")),
    "one LSA temperature for every layer":
        ("vit small dataset", "fold", lambda mp, eng: _one_lsa_temperature(mp),
         ("layer 1 attention", "operand scale")),
    "local patch interaction's BatchNorm folded with the default eps":
        ("xcit layer subset", "fold", lambda mp, eng: _bn_default_eps(mp),
         ("layer 0 local patch interaction", "operand w1")),
    "encoder_layers() swaps a layer's LayerNorms":
        ("vit cls", "exact", lambda mp, eng: _swapped_layer_norms(mp), ("layer 1", "EncoderLayer.ln1.gamma")),
    "exact mode: the QKV GEMM reads the attention output buffer":
        ("vit cls", "exact", lambda mp, eng: _exact_gemm_reads_o(mp), ("layer 0 qkv", "operand a")),
}


@pytest.mark.parametrize("name", list(DEFECTS))
def test_planted_defect_is_named(name, monkeypatch):
    case, ln_mode, plant, want = DEFECTS[name]
    mod, x0, kw, launches = run(_case(case), ln_mode, plant=lambda m, eng: plant(monkeypatch, eng))
    with pytest.raises(AssertionError) as e:
        LT.check_provenance(mod, x0, kw, launches, ln_mode, case)
    msg = str(e.value)
    assert all(w in msg for w in want), msg
