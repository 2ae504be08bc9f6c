"""NesT (vit_pytorch_b200.nest) without a GPU: the module surface and that the eager graph raises where the reference
does, the block-major row map against the reference's '(b b1 b2)(h w)' token order, a pure-torch fp64 emulation of
the fused dataflow (block-major rows, the level entry's LayerNorm -> max-pool -> position order, the im2col column
order of Aggregate's convolution, the head's LayerNorm before the mean) against the reference's logits on every parity
case, the fallback rules, the argument checks of the new entry points, and the launch sequence of the whole fused
forward (tests/golden/nest_schedule.json, made by make_nest_schedule.py).  The reference-parity tests are in
test_nest_parity.py."""
import ctypes
import importlib
import json
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN_DIR, ROOT, import_reference, load_golden, reference_available
from vit_pytorch_b200 import _lib, build, nest as nt
from vit_pytorch_b200.engine import attention_kernel
from vit_pytorch_b200.nest import NesT

sys.path.insert(0, GOLDEN_DIR)
import make_engine_schedule as S  # noqa: E402
import make_nest_schedule as NS  # noqa: E402
from nest_spec import FAMILY  # noqa: E402

README = dict(image_size=224, patch_size=4, dim=96, heads=3, num_hierarchies=3, block_repeats=(2, 2, 8),
              num_classes=1000)


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def small(**kw):
    torch.manual_seed(0)
    return NesT(**dict(dict(image_size=64, patch_size=4, dim=32, heads=1, num_hierarchies=3, block_repeats=1,
                            num_classes=5), **kw)).eval()


# ------------------------------------------------------------------------------------------------ surface
def test_module_surface():
    assert set(nt.__all__) >= {"Aggregate", "Attention", "FeedForward", "LayerNorm", "NesT", "Transformer",
                               "cast_tuple"}
    m = small()
    assert [n for n, _ in m.layers[0][0].named_parameters()][:5] == [
        "pos_emb", "layers.0.0.norm.g", "layers.0.0.norm.b", "layers.0.0.to_qkv.weight", "layers.0.0.to_out.0.weight"]
    assert isinstance(m.layers[-1][1], torch.nn.Identity)
    assert m.level_maps(64, 64) == [(16, 16, 4), (8, 8, 2), (4, 4, 1)]
    assert m.level_maps(224, 112) == [(56, 28, 4), (28, 14, 2), (14, 7, 1)]


def test_eager_graph_raises_where_the_reference_does():
    m = small()
    bad = {"patch": torch.randn(1, 3, 66, 64), "blocks": torch.randn(1, 3, 72, 72),
           "seq_len": torch.randn(1, 3, 128, 128)}
    with torch.no_grad():
        assert m(torch.randn(1, 3, 32, 64)).shape == (1, 5)
        with pytest.raises(RuntimeError, match="4 x 4 patches"):
            m(bad["patch"])
        with pytest.raises(RuntimeError, match="4 x 4 blocks"):
            m(bad["blocks"])
        with pytest.raises(RuntimeError, match="needs 64 positions"):
            m(bad["seq_len"])
    with pytest.raises(AssertionError, match="divisible by the patch size"):
        NesT(image_size=66, patch_size=4, dim=32, heads=1, num_hierarchies=3, block_repeats=1, num_classes=5)
    if not reference_available():
        return
    ref = import_reference()
    RefNesT = importlib.import_module(f"{ref.__name__}.nest").NesT
    torch.manual_seed(0)
    r = RefNesT(image_size=64, patch_size=4, dim=32, heads=1, num_hierarchies=3, block_repeats=1, num_classes=5)
    with torch.no_grad():
        for x in bad.values():
            with pytest.raises(Exception):
                r(x)


# ------------------------------------------------------------------------------------------------ block-major rows
def block_rows(B: int, H: int, W: int, nb: int) -> torch.Tensor:
    """Per map-order row (b*H + y)*W + x, its row in the block-major stream of nb x nb blocks (the kernels' map)."""
    sh, sw = H // nb, W // nb
    b, y, x = torch.meshgrid(torch.arange(B), torch.arange(H), torch.arange(W), indexing="ij")
    return (((b * nb + y // sh) * nb + x // sw) * (sh * sw) + (y % sh) * sw + x % sw).reshape(-1)


@pytest.mark.parametrize("B,H,W,nb", [(2, 56, 56, 4), (1, 56, 28, 4), (3, 8, 8, 4), (2, 14, 14, 2), (2, 7, 7, 1)])
def test_block_major_rows_are_the_reference_token_order(B, H, W, nb):
    """Token t of block s after the reference's 'b c (b1 h) (b2 w) -> (b b1 b2) c h w' and Attention's '(x y)'
    flattening is row s*(sh*sw) + t of the stream."""
    ids = torch.arange(B * H * W).view(B, H, W, 1).permute(0, 3, 1, 2)        # (b, c=1, H, W): the map-order row
    blocks = nt.to_blocks(ids, nb)                                            # ((b b1 b2), 1, sh, sw)
    order = blocks.reshape(blocks.shape[0], -1).reshape(-1)                    # stream row -> map-order row
    rows = block_rows(B, H, W, nb)
    assert torch.equal(order[rows], torch.arange(B * H * W))
    assert torch.equal(nt.from_blocks(blocks, nb), ids)
    try:
        from einops import rearrange
    except ImportError:
        return
    ref = rearrange(ids, 'b c (b1 h) (b2 w) -> (b b1 b2) c h w', b1=nb, b2=nb)
    assert torch.equal(rearrange(ref, 'b c x y -> b (c x y)').reshape(-1), order)


# ------------------------------------------------------------------------------------------------ fp64 dataflow
def _ln(x: torch.Tensor, ln) -> torch.Tensor:
    g, b = ln.g.reshape(-1), ln.b.reshape(-1)
    return (x - x.mean(1, keepdim=True)) / (x.var(1, unbiased=False, keepdim=True) + ln.eps).sqrt() * g + b


def level_entry(y: torch.Tensor, ln, pos: torch.Tensor, B: int, H: int, W: int, k: int, s: int, p: int,
                nb: int) -> torch.Tensor:
    """b200vit_nest_level_entry: y [B*H*W, D] map order -> LN per pixel -> max over the (k, s, p) window, padding
    -inf -> + pos[(r % sh)*sw + q % sw] -> block-major rows."""
    D = y.shape[1]
    z = _ln(y, ln).view(B, H, W, D).permute(0, 3, 1, 2)
    z = F.pad(z, (p, p, p, p), value=float("-inf")).unfold(2, k, s).unfold(3, k, s).amax(dim=(-1, -2))
    oh, ow = z.shape[2], z.shape[3]
    sh, sw = oh // nb, ow // nb
    r, q = torch.meshgrid(torch.arange(oh), torch.arange(ow), indexing="ij")
    z = z + pos[(r % sh) * sw + q % sw]
    out = torch.empty(B * oh * ow, D, dtype=y.dtype)
    out[block_rows(B, oh, ow, nb)] = z.permute(0, 2, 3, 1).reshape(-1, D)
    return out


def im2col(x: torch.Tensor, B: int, H: int, W: int, nb: int) -> torch.Tensor:
    """b200vit_nest_im2col: block-major x [B*H*W, D] -> map-order rows, column (i*3 + j)*D + c = pixel
    (y - 1 + i, x - 1 + j), zero outside the map."""
    D = x.shape[1]
    m = torch.zeros(B, H + 2, W + 2, D, dtype=x.dtype)
    m[:, 1:-1, 1:-1] = x[block_rows(B, H, W, nb)].view(B, H, W, D)
    taps = [m[:, i:i + H, j:j + W] for i in range(3) for j in range(3)]
    return torch.cat(taps, dim=-1).reshape(B * H * W, 9 * D)


def encoder(tr, x: torch.Tensor, S: int, n: int) -> torch.Tensor:
    """The engine's pre-LN layers over S sequences of n consecutive rows."""
    for attn, ff in tr.layers:
        D, Hh = x.shape[1], attn.heads
        I = attn.to_qkv.weight.shape[0] // 3
        qkv = (_ln(x, attn.norm) @ attn.to_qkv.weight.reshape(3 * I, D).t()).view(S, n, 3, Hh, I // Hh)
        q, k, v = (qkv[:, :, j].transpose(1, 2) for j in range(3))
        o = (torch.softmax(q @ k.transpose(-1, -2) * attn.scale, -1) @ v).transpose(1, 2).reshape(S * n, I)
        x = x + o @ attn.to_out[0].weight.reshape(D, I).t() + attn.to_out[0].bias
        f = ff.net
        h = F.gelu(_ln(x, f[0]) @ f[1].weight.reshape(-1, D).t() + f[1].bias)
        x = x + h @ f[4].weight.reshape(D, -1).t() + f[4].bias
    return x


def fused_dataflow(m: NesT, img: torch.Tensor) -> torch.Tensor:
    """NesT.forward_fused's dataflow in the dtype of m and img."""
    pe = m.to_patch_embedding
    B, C, Hi, Wi = img.shape
    p = pe[0].p
    maps = m.level_maps(Hi, Wi)
    h, w, _ = maps[0]
    # (p1 p2 c) patch rows in map order, as b200vit_patchify_ln writes them
    a = img.reshape(B, C, h, p, w, p).permute(0, 2, 4, 3, 5, 1).reshape(B * h * w, p * p * C)
    y = _ln(a, pe[1]) @ pe[2].weight.reshape(pe[2].out_channels, -1).t() + pe[2].bias
    ln, pool, ph, pw = pe[3], (1, 1, 0), h, w
    for i, ((tr, agg), (h, w, nb)) in enumerate(zip(m.layers, maps)):
        x = level_entry(y, ln, tr.pos_emb, B, ph, pw, *pool, nb)
        x = encoder(tr, x, B * nb * nb, (h // nb) * (w // nb))
        if i + 1 < len(m.layers):
            c = agg[0]
            y = im2col(x, B, h, w, nb) @ c.weight.permute(0, 2, 3, 1).reshape(c.out_channels, -1).t() + c.bias
            ln, pool, ph, pw = agg[1], (3, 2, 1), h, w
    pooled = _ln(x, m.mlp_head[0]).view(B, h * w, -1).mean(1)
    return pooled @ m.mlp_head[2].weight.t() + m.mlp_head[2].bias


@pytest.mark.parametrize("name", sorted(FAMILY.cases))
def test_fused_dataflow_matches_the_reference_in_fp64(name):
    spec = FAMILY.cases[name]
    m = FAMILY.build(spec).double()
    with torch.no_grad():
        got = fused_dataflow(m, FAMILY.input(spec).double())
    want = load_golden("nest")["cases"][name]["logits_fp32"]
    torch.testing.assert_close(got.float(), want, rtol=1e-4, atol=1e-4)


# ------------------------------------------------------------------------------------------------ fallback rules
def test_fused_reason_rules(monkeypatch):
    x = torch.zeros(2, 3, 64, 64, dtype=torch.bfloat16)
    m = small().bfloat16()
    assert m.fused_reason(x) == "input is not on a CUDA device"
    monkeypatch.setattr(nt, "common_reason", lambda *a, **k: None)
    assert m.fused_reason(x) is None
    assert m.fused_reason(torch.zeros(2, 3, 32, 96)) is None                   # non-square, pos_emb prefix
    assert "channels" in m.fused_reason(torch.zeros(2, 1, 64, 64))
    assert "(B, C, H, W)" in m.fused_reason(torch.zeros(3, 64, 64))
    assert "not divisible by patch_size=4" in m.fused_reason(torch.zeros(1, 3, 66, 64))
    assert "level 1: the 18 x 18 map does not split into 4 x 4 blocks" in m.fused_reason(torch.zeros(1, 3, 72, 72))
    assert "blocks of 64 tokens, more than seq_len=16" in m.fused_reason(torch.zeros(1, 3, 128, 128))
    assert "multiples of 8" in small(dim=97, heads=3).fused_reason(x)          # heads 32 wide over 97 channels
    assert small(dim=160, heads=2).fused_reason(x) is None                     # heads 80 wide
    assert "dim_head=48" in small(dim=48, heads=1).fused_reason(x)
    assert "dim_head=16" in small(dim=32, heads=2).fused_reason(x)
    assert "sequence length 65536 > 16384" in small(image_size=512, patch_size=2, num_hierarchies=1).fused_reason(
        torch.zeros(1, 3, 512, 512))
    m.train()
    assert "training" in m.fused_reason(x)


def test_fused_reason_names_dtype_device_depth_and_hooks(monkeypatch):
    m = small().bfloat16()
    assert "CUDA" in m.fused_reason(torch.zeros(1, 3, 64, 64, dtype=torch.bfloat16))
    import vit_pytorch_b200.engine as E
    monkeypatch.setattr(E, "why_not_fused", lambda *a, **k: None)
    h = m.layers[1][0].layers[0][0].to_qkv.register_forward_hook(lambda *a: None)
    assert "hooks" in m.fused_reason(torch.zeros(2, 3, 64, 64))
    h.remove()
    assert m.fused_reason(torch.zeros(2, 3, 64, 64)) is None
    assert small(block_repeats=(1, 0, 1)).fused_reason(torch.zeros(2, 3, 64, 64)) == "depth == 0"
    monkeypatch.undo()
    m32 = small()
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    assert "dtype" in m32.fused_reason(torch.zeros(1, 3, 64, 64))


def test_encoder_layers_of_the_readme_config():
    torch.manual_seed(0)
    m = NesT(**README).eval()
    assert m.level_maps(224, 224) == [(56, 56, 4), (28, 28, 2), (14, 14, 1)]
    for (tr, _), depth, heads, dim in zip(m.layers, (2, 2, 8), (3, 6, 12), (96, 192, 384)):
        layers, norm = tr.encoder_layers()
        assert len(layers) == depth and norm is None and tr.pos_emb.numel() == 196
        for L in layers:
            assert (L.heads, L.dim_head, L.scale) == (heads, 32, 32 ** -0.5) and L.attention is None
            assert L.qkv_w.shape == (3 * dim, dim) and L.fc1_w.shape == (4 * dim, dim)
            assert attention_kernel(L) == "plain"
        assert tr.engine().unsupported_reason(196) is None
        assert tr.engine().prepared()["c_layers"] is not None                  # the one-call C layer loop


# ------------------------------------------------------------------------------------------------ argument checks
def test_nest_level_entry_rejects_bad_arguments(lib):
    p, q, r = ctypes.c_void_p(256), ctypes.c_void_p(1 << 30), ctypes.c_void_p(1 << 31)

    def call(*, y=p, M=2 * 8 * 8, g=p, b=p, pos=p, n_pos=16, x=q, xb=None, st=None, B=2, H=8, W=8, D=32, pk=3, ps=2,
             pp=1, nb=1):
        rc = lib.b200vit_nest_level_entry(y, M, g, b, 1e-5, pos, n_pos, x, xb, st, B, H, W, D, pk, ps, pp, nb, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(y=None), dict(g=None), dict(b=None), dict(pos=None), dict(x=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw, what in ((dict(xb=r), b"both or neither"), (dict(st=r), b"both or neither"), (dict(B=0), b"bad shape"),
                     (dict(D=0), b"bad shape"), (dict(pk=4), b"bad shape"), (dict(pk=3, pp=2), b"bad shape"),
                     (dict(ps=0), b"bad shape"), (dict(H=1, W=1, pk=3, pp=0), b"bad shape"),
                     (dict(M=2 * 8 * 8 - 1), b"127 rows"), (dict(nb=3), b"into 3 x 3 blocks"),
                     (dict(n_pos=15), b"15 positions for blocks of 16 tokens"),
                     (dict(y=ctypes.c_void_p(260)), b"16-byte aligned"), (dict(g=ctypes.c_void_p(264)), b"aligned"),
                     (dict(xb=ctypes.c_void_p(r.value + 8), st=r), b"aligned"),
                     (dict(xb=r, st=ctypes.c_void_p(r.value + 4)), b"8-byte aligned"),
                     (dict(x=ctypes.c_void_p(256 + 4096)), b"overlap"), (dict(xb=p, st=r), b"overlap")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)


def test_nest_im2col_rejects_bad_arguments(lib):
    p, q = ctypes.c_void_p(256), ctypes.c_void_p(1 << 30)

    def call(*, x=p, M=2 * 8 * 8, out=q, ldo=9 * 32, B=2, H=8, W=8, D=32, nb=2):
        rc = lib.b200vit_nest_im2col(x, M, out, ldo, B, H, W, D, nb, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(x=None), dict(out=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw, what in ((dict(B=0), b"bad shape"), (dict(D=12, ldo=9 * 16), b"bad shape"), (dict(H=0), b"bad shape"),
                     (dict(M=100), b"100 rows"), (dict(nb=3), b"into 3 x 3 blocks"), (dict(ldo=280), b"ldo=280"),
                     (dict(ldo=9 * 32 + 4), b"ldo=292"), (dict(x=ctypes.c_void_p(272 + 4)), b"16-byte aligned"),
                     (dict(out=ctypes.c_void_p(256 + 4096)), b"overlaps")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)


NEW = ("nest_level_entry", "nest_im2col")


def test_header_declares_the_new_entry_points():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    for name in NEW:
        assert f"int b200vit_{name}(" in h and f"b200vit_{name}" in _lib.SYMBOLS
    assert f"#define B200VIT_NEST_POOL_MAX_KERNEL {_lib.NEST_POOL_MAX_KERNEL}" in h


def test_library_exports_the_new_entry_points(lib):
    for name in NEW:
        assert hasattr(lib, f"b200vit_{name}")


# ------------------------------------------------------------------------------------------------ launch sequence
@pytest.fixture(scope="module")
def schedule():
    with open(NS.FIXTURE) as f:
        return json.load(f)


def test_schedule_fixture_lists_every_run(schedule):
    assert list(schedule) == [NS.run_name(m, h) for m, h in NS.RUNS]


@pytest.mark.parametrize("ln_mode,host_loop", NS.RUNS)
def test_fused_forward_schedule_matches_fixture(lib, schedule, ln_mode, host_loop):
    name = NS.run_name(ln_mode, host_loop)
    got, want = NS.record(ln_mode, host_loop), schedule[name]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: call {i} differs"
    assert len(got) == len(want), f"{name}: {len(got)} calls, {len(want)} expected"


@pytest.mark.parametrize("ln_mode,host_loop", NS.RUNS)
def test_level_launches_run_the_persistent_attention_lengths(schedule, ln_mode, host_loop):
    """Every level attends over blocks of 196 tokens with heads 32 wide: the persistent attention kernel's range
    (128 < N <= 256, dim_head 32 or 64; b200vit_attention chooses it by length), whether the layers run in the one-call
    C loop (encoder_blocks) or launch by launch (attention)."""
    calls = schedule[NS.run_name(ln_mode, host_loop)]
    names = [c["call"] for c in calls]
    assert names[:3] == ["patchify_ln", "gemm", "nest_level_entry"]
    assert names[-4:] == ["layernorm", "mean_pool", "cast_f32_bf16", "gemm"]
    entries = [c for c in calls if c["call"] == "nest_level_entry"]
    assert [(c["H"], c["W"], c["pk"], c["ps"], c["pp"], c["nb"]) for c in entries] == [
        (56, 56, 1, 1, 0, 4), (56, 56, 3, 2, 1, 2), (28, 28, 3, 2, 1, 1)]
    assert all((c["xb"] is not None) == (ln_mode == "fold") for c in entries)
    assert [(c["H"], c["W"], c["nb"]) for c in calls if c["call"] == "nest_im2col"] == [(56, 56, 4), (28, 28, 2)]
    fused = ln_mode == "fold" and host_loop == "c"
    att = [c for c in calls if c["call"] == ("encoder_blocks" if fused else "attention")]
    assert [(c["B"], c["N"], c["dh"]) for c in att] == (
        [(32, 196, 32), (8, 196, 32), (2, 196, 32)] if fused else
        [(32, 196, 32), (8, 196, 32), (2, 196, 32), (2, 196, 32)])
    assert all(128 < c["N"] <= 256 and c["dh"] in (32, 64) for c in att)


def test_other_families_schedule_fixtures_are_unchanged(lib):
    """Every other family's pinned launch sequence, regenerated, is byte-identical to its fixture."""
    for mod in ("make_engine_schedule", "make_cct_schedule", "make_pit_schedule", "make_levit_schedule",
                "make_twins_svt_schedule", "make_max_vit_schedule", "make_cvt_schedule",
                "make_crossformer_schedule", "make_mobile_vit_schedule", "make_sep_vit_schedule",
                "make_regionvit_schedule"):
        g = importlib.import_module(mod)
        with open(g.FIXTURE) as f:
            assert S.dumps(g.generate()) == f.read(), mod
