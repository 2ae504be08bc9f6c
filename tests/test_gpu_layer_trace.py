"""-m gpu: every launch of TransformerEngine.run_blocks on the real kernels, traced back to the reference layer
(oracle/layer_trace.py) at production-like shapes: D 384 in 6 heads of 64 (the GEMMs run several tiles per CTA) and
token counts that are not multiples of 128.

For each case and LayerNorm mode: every operand of every launch is what the reference module's forward defines there
(provenance), and every output is within its kernel's existing fp64 bound on the operands it received.  The worst
|got - ref| / bound per (case, launch kind) is printed at the end of the module.  Where the one-call C loop applies and
no other test compares it, its final x, bf16 copy and row statistics must equal the per-kernel loop's bit for bit.  Two
planted defects are re-run through the real kernels: the walk must name them; whether a model-level max-abs criterion
would have seen them is printed, not asserted."""

import pytest
import torch

from oracle import layer_trace as LT
from test_layer_trace import _colsum_unrounded, _layerscale_rows_only, set_eps
from vit_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda"
D, H, DH, MLP = 384, 6, 64, 1536
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nworst |got - ref| / bound per case, LayerNorm mode and launch kind:")
    for key in sorted(WORST):
        print(f"  {' | '.join(key)}: {WORST[key]:.3f}")


def _images(sizes):
    return _lib.VarlenIndex([torch.empty(3, h, w, device=DEV) for h, w in sizes], 16, torch.device(DEV))


def _rope(N):
    theta = 3 * torch.randn(N, H, DH // 2, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    return torch.stack((theta.cos(), theta.sin()), dim=-1).contiguous(), N


def _mask():
    return torch.tensor([[1, 0, 1, 1], [1, 1, 0, 0]], dtype=torch.uint8, device=DEV)


def _m(path, *args, **kw):
    def make():
        import importlib
        mod, cls = path.rsplit(".", 1)
        return getattr(importlib.import_module(f"vit_pytorch_b200.{mod}"), cls)(*args, **kw)
    return make


def _cct():
    from vit_pytorch_b200.cct import TransformerClassifier
    return TransformerClassifier(seq_pool=True, embedding_dim=D, num_layers=2, num_heads=H, mlp_ratio=4.0,
                                 num_classes=3, dropout_rate=0.0, attention_dropout=0.0, stochastic_depth_rate=0.0,
                                 positional_embedding="none")


# name: (module, rows of x, run_blocks' keyword arguments, C loop applies and no other test compares it)
CASES = {
    "vit": (_m("vit.Transformer", D, 2, H, DH, MLP), 3 * 197, lambda: dict(B=3, N=197), False),
    "vit identity out": (_m("vit.Transformer", 128, 2, 1, 128, 512), 3 * 197, lambda: dict(B=3, N=197, primed=True),
                         True),
    "vit N 785 (varlen)": (_m("vit.Transformer", D, 2, H, DH, MLP), 2 * 785, lambda: dict(B=2, N=785), True),
    "simple_vit qk rmsnorm": (_m("simple_vit_with_qk_norm.Transformer", D, 2, H, DH, MLP), 3 * 196,
                              lambda: dict(B=3, N=196, primed=True), True),
    "navit packed": (_m("na_vit.Transformer", D, 2, H, DH, MLP), 196 + 128 + 60 + 15,
                     lambda: dict(primed=True, varlen=_images([(224, 224), (128, 256), (96, 160), (48, 80)])), False),
    "navit nested qk layernorm": (_m("na_vit_nested_tensor.Transformer", D, 2, H, DH, MLP), 196 + 128 + 60 + 15,
                                  lambda: dict(primed=True, varlen=_images([(224, 224), (128, 256), (96, 160),
                                                                            (48, 80)])), False),
    "vit_nd rotary": (_m("vit_nd_rotary.Transformer", D, 2, H, DH, MLP), 3 * 196,
                      lambda: dict(B=3, N=196, primed=True, rope=_rope(196)), False),
    "vit small dataset (LSA)": (_m("vit_for_small_dataset.Transformer", D, 2, H, DH, MLP), 5 * 65,
                                lambda: dict(B=5, N=65, primed=True), False),
    "vivit factorized": (_m("vivit.FactorizedTransformer", D, 2, H, DH, MLP), 8 * 197,
                         lambda: dict(B=8, N=197, primed=True, axial=(197, 4, None, True)), False),
    "vivit factorized masked": (_m("vivit.FactorizedTransformer", D, 2, H, DH, MLP), 8 * 197,
                                lambda: dict(B=8, N=197, primed=True, axial=(197, 4, _mask(), False)), False),
    "deepvit": (_m("deepvit.Transformer", D, 2, H, DH, MLP), 3 * 197, lambda: dict(B=3, N=197, primed=True), False),
    "cait": (_m("cait.Transformer", D, 3, H, DH, MLP), 3 * 196, lambda: dict(B=3, N=196, primed=True), False),
    "cait layer subset": (_m("cait.Transformer", D, 3, H, DH, MLP), 3 * 196,
                          lambda: dict(B=3, N=196, primed=True, layers=[0, 2]), False),
    "xcit": (_m("xcit.XCATransformer", D, 2, H, DH, MLP, local_patch_kernel_size=3), 3 * 196,
             lambda: dict(B=3, N=196, primed=True, grid=(14, 14)), False),
    "cct": (_cct, 3 * 196, lambda: dict(B=3, N=196), False),
}


def make(name, seed=0):
    """The case's module on the GPU (fp32 parameters): default init moved by noise so that LayerNorm gains and shifts,
    LayerScales and temperatures are not their constants, LayerNorm eps as test_layer_trace.set_eps sets them, BatchNorm
    running statistics away from (0, 1)."""
    return perturbed(CASES[name][0], seed)


def perturbed(module, seed=0):
    """module() as make() initialises it."""
    torch.manual_seed(seed)
    mod = module().eval()
    with torch.no_grad():
        for p in mod.parameters():
            p.add_(0.05 * torch.randn_like(p))
        for m in mod.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.normal_(0, 0.2)
                m.running_var.uniform_(0.5, 2.0)
                m.eps = 1e-3
    set_eps(mod)
    return mod.to(DEV)


def inputs(name):
    rows = CASES[name][1]
    x = torch.randn(rows, D if "identity" not in name else 128, device=DEV,
                    generator=torch.Generator(device=DEV).manual_seed(rows))
    return x, CASES[name][2]()


REAL_ROWSTATS, REAL_GEMM = _lib.rowstats_cast, _lib.gemm


def traced(mod, x, kw, ln_mode, call=None):
    eng = mod.engine()
    launches = LT.trace(eng, x, kw, ln_mode, LT.real_impl, prime=lambda a, b, s: REAL_ROWSTATS(a, b, s), call=call)
    torch.cuda.synchronize()
    return launches


def rerun_plain(pre):
    out = torch.empty_like(pre["out_bf16"])
    REAL_GEMM(pre["a"], pre["w"], out_bf16=out, bias=pre["bias"], ln_sums=pre["ln_sums"], col_s=pre["col_s"],
              ln_eps=pre["ln_eps"])
    return out


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("name", list(CASES))
def test_layer_launches_trace_back_and_stay_within_bounds(name, ln_mode):
    mod = make(name)
    x, kw = inputs(name)
    x0 = x.clone()
    with torch.no_grad():
        launches = traced(mod, x, kw, ln_mode)
        n = LT.check_provenance(mod, x0, kw, launches, ln_mode, f"{name} | {ln_mode}")
        assert n == len(launches) > 0
        for kind, r in LT.check_accuracy(launches, f"{name} | {ln_mode}", rerun_plain=rerun_plain).items():
            WORST[(name, ln_mode, kind)] = max(WORST.get((name, ln_mode, kind), 0.0), r)


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c[3]])
def test_c_loop_is_bit_identical_to_the_python_loop(name, monkeypatch):
    mod = make(name)
    eng = mod.engine()
    x0, kw = inputs(name)
    monkeypatch.setenv("B200VIT_LN_MODE", "fold")
    got = {}
    with torch.no_grad():
        for loop in ("python", "c"):
            monkeypatch.setenv("B200VIT_HOST_LOOP", loop)
            x = x0.clone()
            if kw.get("primed"):
                xb, st = eng.entry_buffers(x.shape[0], x.device)
                _lib.rowstats_cast(x, xb, st)
            _lib.reset_launch_count()
            eng.run_blocks(x, **kw)
            torch.cuda.synchronize()
            ws = eng.workspace(x.shape[0], x.device)
            got[loop] = (x, ws["xn"].clone(), ws["stats_a"].clone(), _lib.launch_count())
    assert got["c"][3] > 0
    for i, what in enumerate(("x", "xn", "stats_a")):
        assert torch.equal(got["c"][i], got["python"][i]), f"{name}: {what} differs between the C and Python loops"


def _eager(mod, x0, kw):
    """The module's own fp32 forward over the same tokens (the reference's operator sequence), final LayerNorm
    included; CaiT's layer subset as cait.py:14-27 runs it."""
    B, N = kw["B"], kw["N"]
    tokens = x0.view(B, N, -1)
    if kw.get("layers") is not None:
        want = tokens
        for i in kw["layers"]:
            ls_attn, ls_ff = mod.layers[i]
            want = ls_attn(want) + want
            want = ls_ff(want) + want
        return want.reshape(B * N, -1)
    return mod(tokens).reshape(B * N, -1)


# name: (case, plant, what the failure must name)
GPU_DEFECTS = {
    "fold column sums from the unrounded gamma W": ("vit", _colsum_unrounded, ("layer 0 qkv", "operand col_s")),
    "LayerScale on the rows but not the bias": ("cait", _layerscale_rows_only, ("layer 0 out", "operand bias")),
}


@pytest.mark.parametrize("defect", list(GPU_DEFECTS))
def test_planted_defect_is_named_on_the_real_kernels(defect, monkeypatch):
    name, plant, want = GPU_DEFECTS[defect]
    x0, kw = inputs(name)
    res = {}
    with torch.no_grad():
        for planted in (False, True):
            mod = make(name)
            if planted:
                plant(monkeypatch)
            x = x0.clone()
            launches = traced(mod, x, kw, "fold")
            eng = mod.engine()
            out = x.clone()
            if eng.norm is not None:
                out = torch.empty_like(x)
                eng.final_norm(x, out_f32=out)
            want_out = _eager(mod, x0, kw)
            res[planted] = ((out - want_out).abs().max().item(), want_out.abs().max().item())
            if planted:
                with pytest.raises(AssertionError) as e:
                    LT.check_provenance(mod, x0, kw, launches, "fold", name)
                assert all(w in str(e.value) for w in want), str(e.value)
                monkeypatch.undo()
    (clean, scale), (bad, _) = res[False], res[True]
    print(f"\n{defect} ({name}): max |fused - eager fp32| over the encoder output {clean:.3e} without the defect, "
          f"{bad:.3e} with it (max |eager| {scale:.3e}); a 3e-2 max-abs criterion would "
          f"{'miss' if bad < 3e-2 else 'catch'} it, 2e-2 would {'miss' if bad < 2e-2 else 'catch'} it")
