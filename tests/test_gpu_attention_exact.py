"""-m gpu: which keys every attention kernel reads, checked exactly.

Random-data tolerance tests cannot see a key read from the wrong sequence (its probability is 0, and 0 x finite = 0)
nor a dropped key at long lengths (one key of 4096 moves an output by ~2e-4).  So:
  A. isolation: one sequence poisoned with NaN / Inf (or NaN only in allocation rows past the view passed in) must
     leave every other sequence's output bit-identical to the clean run -- each image of a batch is computed on its own;
  B. inputs whose answers are known exactly: q = 0 with indicator values (every included key gives 1/len, every
     excluded key exactly 0), values that are the one-hot sequence id, and dominant keys (out_i = v_i to the bit);
  C. head routing of the head-mixing kernels: permutation mixes and random mixes at every head count, each output
     element within the bound of the fp64 references of oracle/headmix_bounds.py and oracle/attention_fp32_bounds.py;
  D. the GEMM's operand margins: NaN beyond K, past M and past N must not reach the output.
plus model-level batches with one NaN image.
"""
import contextlib
import math

import pytest
import torch

from oracle import attention_fp32_bounds as FB
from oracle import bounds as Bd
from oracle import headmix_bounds as HB
from vit_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN, INF = float("nan"), float("inf")
BF16_REL = 2.0 ** -7          # one bf16 ulp, relative


@contextlib.contextmanager
def hooks(**kv):
    """Test hooks of include/b200vit.h (key -> value), reset to 0 afterwards: k15 = the tiled kernel at every length."""
    L = _lib.lib()
    try:
        for k, v in kv.items():
            assert L.b200vit_debug_set(int(k[1:]), v) == 0
        yield
    finally:
        for k in kv:
            L.b200vit_debug_set(int(k[1:]), 0)


def poison(qkv, r0, r1, I, how):
    """NaN in q, k and v ('nan') or +Inf in v only ('inf_v') of rows [r0, r1) of a packed q | k | v buffer."""
    if how == "nan":
        qkv[r0:r1] = NAN
    else:
        qkv[r0:r1, 2 * I:] = INF


def assert_rows_equal(got, want, keep, what):
    """Rows where keep is True must be bit-identical."""
    keep = keep.to(got.device)
    g, w = got[keep], want[keep]
    bad = ~((g == w) | (torch.isnan(g) & torch.isnan(w))).all(1)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {int(keep.sum())} protected rows changed"


# ====================================================================================================== A. isolation
# (test hook 15, MASK_SELF): the kernel each length runs by default, the tiled kernel at 128 < N <= 256 as well, and
# the self-masked instance
PLAIN_CONFIGS = {"default": (0, False), "tiled": (1, False), "mask_self": (0, True)}


def run_plain(qkv, B, N, H, dh, cfg):
    k15, ms = PLAIN_CONFIGS[cfg]
    out = torch.full((B * N, H * dh), 5.0, device=DEV, dtype=torch.bfloat16)
    with hooks(k15=k15):
        _lib.attention(qkv, out, B, N, H, dh, dh ** -0.5, mask_self=ms)
        torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("N", [64, 65, 127, 128, 129, 197, 255])      # len % 64 in {0, 1, 63}
@pytest.mark.parametrize("cfg", sorted(PLAIN_CONFIGS))
@pytest.mark.parametrize("dh", [32, 64, 80, 128])
def test_attention_isolation_under_poisoning(dh, cfg, N):
    B, H = 3, 2
    I = H * dh
    g = torch.Generator(device=DEV).manual_seed(dh * 1000 + N)
    qkv = torch.randn(B * N, 3 * I, device=DEV, generator=g).bfloat16()
    clean = run_plain(qkv, B, N, H, dh, cfg)
    assert torch.isfinite(clean.float()).all()
    seq = torch.arange(B * N, device=DEV) // N
    for s in (1, 0, 2):                  # the sequence after the probe and the one before it
        for how in ("nan", "inf_v"):
            bad = qkv.clone()
            poison(bad, s * N, (s + 1) * N, I, how)
            assert_rows_equal(run_plain(bad, B, N, H, dh, cfg), clean, seq != s, f"poisoned {s} {how}")
    # NaN only in allocation rows past the view passed in
    buf = torch.full((B * N + 2 * N + 7, 3 * I), NAN, device=DEV, dtype=torch.bfloat16)
    buf[:B * N] = qkv
    assert torch.equal(run_plain(buf[:B * N], B, N, H, dh, cfg), clean)


VARLEN_CONFIGS = {"kb64": False, "mask_self": True}                      # MASK_SELF
# length-1 sequences, lengths on and around 64 / 128 boundaries, sequences crossing 128-row tiles of the pack
VARLEN_PACK = [1, 130, 64, 1, 63, 257, 128, 65, 1, 200, 127, 129, 2]


def run_varlen(qkv, lengths, H, dh, cfg):
    cu, tp, tiles = _lib.varlen_index(lengths, DEV)
    out = torch.full((qkv.shape[0], H * dh), 5.0, device=DEV, dtype=torch.bfloat16)
    _lib.attention_varlen(qkv, out, cu, tp, tiles, H, dh, dh ** -0.5, mask_self=VARLEN_CONFIGS[cfg])
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("cfg", sorted(VARLEN_CONFIGS))
@pytest.mark.parametrize("dh", [32, 64, 80, 128])
def test_attention_varlen_isolation_under_poisoning(dh, cfg):
    H, lengths = 2, VARLEN_PACK
    I, T = H * dh, sum(VARLEN_PACK)
    g = torch.Generator(device=DEV).manual_seed(dh)
    qkv = torch.randn(T, 3 * I, device=DEV, generator=g).bfloat16()
    clean = run_varlen(qkv, lengths, H, dh, cfg)
    assert torch.isfinite(clean.float()).all()
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    seq = torch.repeat_interleave(torch.arange(len(lengths)), torch.tensor(lengths)).to(DEV)
    for s in range(len(lengths)):        # every sequence in turn: each one is both before and after another
        for how in ("nan", "inf_v"):
            bad = qkv.clone()
            poison(bad, cu[s], cu[s + 1], I, how)
            assert_rows_equal(run_varlen(bad, lengths, H, dh, cfg), clean, seq != s, f"poisoned {s} {how}")
    buf = torch.full((T + 300, 3 * I), NAN, device=DEV, dtype=torch.bfloat16)
    buf[:T] = qkv
    assert torch.equal(run_varlen(buf[:T], lengths, H, dh, cfg), clean)


def run_headmix(qkv, B, N, H, dh, pre, post, ln):
    out = torch.full((B * N, H * dh), 5.0, device=DEV, dtype=torch.bfloat16)
    _lib.attention_headmix(qkv, out, B, N, H, dh, dh ** -0.5, post, ln, pre=pre)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("N", [16, 17, 31, 197])                      # len % 16 in {0, 1, 15, 5}
@pytest.mark.parametrize("H,dh", [(6, 48), (3, 64), (9, 32), (2, 128), (5, 80)])
@pytest.mark.parametrize("pre_on,ln_on", [(False, False), (False, True), (True, False), (True, True)])
def test_attention_headmix_isolation_under_poisoning(pre_on, ln_on, H, dh, N):
    B, I = 3, H * dh
    g = torch.Generator(device=DEV).manual_seed(H * 100 + dh + N)
    qkv = torch.randn(B * N, 3 * I, device=DEV, generator=g).bfloat16()
    pre = torch.randn(H, H, device=DEV, generator=g) if pre_on else None
    post = torch.randn(H, H, device=DEV, generator=g)
    ln = (1 + 0.2 * torch.randn(H, device=DEV, generator=g), 0.1 * torch.randn(H, device=DEV, generator=g),
          1e-5) if ln_on else None
    clean = run_headmix(qkv, B, N, H, dh, pre, post, ln)
    assert torch.isfinite(clean.float()).all()
    seq = torch.arange(B * N, device=DEV) // N
    for s in (1, 0, 2):
        for how in ("nan", "inf_v"):
            bad = qkv.clone()
            poison(bad, s * N, (s + 1) * N, I, how)
            assert_rows_equal(run_headmix(bad, B, N, H, dh, pre, post, ln), clean, seq != s, f"poisoned {s} {how}")
    buf = torch.full((B * N + 40, 3 * I), NAN, device=DEV, dtype=torch.bfloat16)
    buf[:B * N] = qkv
    assert torch.equal(run_headmix(buf[:B * N], B, N, H, dh, pre, post, ln), clean)


def axial_masks(B, L, g):
    partial = torch.rand(B, L, device=DEV, generator=g) > 0.4
    partial[:, 0] = True
    partial[1] = False                   # batch element 1: every key masked
    return {"none": None, "partial": partial.to(torch.uint8).contiguous()}


def run_axial(qkv, km, B, L, G, H, dh, zero):
    out = torch.full((B * L * G, H * dh), 5.0, device=DEV, dtype=torch.bfloat16)
    _lib.attention_axial(qkv, out, km, B, L, G, H, dh, dh ** -0.5, zero)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("L,G", [(1, 1), (5, 1), (8, 1), (17, 1), (5, 3), (8, 3)])
@pytest.mark.parametrize("dh", [32, 64, 80, 128])
def test_attention_axial_isolation_under_poisoning(dh, L, G):
    """Several short sequences share a 64-row tile; a batch element's NaN must stay within it."""
    B, H = 9, 2
    I, T = H * dh, B * L * G
    g = torch.Generator(device=DEV).manual_seed(dh * 100 + L * 10 + G)
    qkv = torch.randn(T, 3 * I, device=DEV, generator=g).bfloat16()
    b_of_row = torch.arange(T, device=DEV) // (L * G)
    for name, km in axial_masks(B, L, g).items():
        for zero in ((True,) if km is None else (True, False)):
            clean = run_axial(qkv, km, B, L, G, H, dh, zero)
            assert torch.isfinite(clean.float()).all()
            for b in (0, 4, 8):
                for how in ("nan", "inf_v"):
                    bad = qkv.clone()
                    poison(bad, b * L * G, (b + 1) * L * G, I, how)
                    assert_rows_equal(run_axial(bad, km, B, L, G, H, dh, zero), clean, b_of_row != b,
                                      f"{name} zero={zero}: poisoned b={b} {how}")
            buf = torch.full((T + 64, 3 * I), NAN, device=DEV, dtype=torch.bfloat16)
            buf[:T] = qkv
            assert torch.equal(run_axial(buf[:T], km, B, L, G, H, dh, zero), clean)


def assert_nan_query_row(run, qkv, row, dh, what):
    """A NaN query in one row: every score of that row is NaN, so the row is NaN (the reference's softmax); every
    other row, and the row's other heads, are bit-identical to the clean run."""
    clean = run(qkv)
    assert torch.isfinite(clean.float()).all()
    bad = qkv.clone()
    bad[row, :dh] = NAN                  # head 0's query
    got = run(bad)
    assert torch.isnan(got[row, :dh].float()).all(), f"{what}: the NaN query row is not NaN"
    keep = torch.ones(got.shape[0], dtype=torch.bool, device=DEV)
    keep[row] = False
    assert_rows_equal(got, clean, keep, what)
    assert torch.equal(got[row, dh:], clean[row, dh:]), f"{what}: the other heads of the NaN query row changed"


@pytest.mark.parametrize("dh", [32, 64, 80, 128])
def test_attention_axial_nan_query_row(dh):
    B, L, G, H = 3, 8, 3, 2
    g = torch.Generator(device=DEV).manual_seed(dh)
    qkv = torch.randn(B * L * G, 3 * H * dh, device=DEV, generator=g).bfloat16()
    for name, km in axial_masks(B, L, g).items():
        for zero in (True, False):
            assert_nan_query_row(lambda x: run_axial(x, km, B, L, G, H, dh, zero), qkv, 2 * L * G + 5, dh,
                                 f"{name} zero={zero}")


@pytest.mark.parametrize("dh", [32, 64, 80, 128])
@pytest.mark.parametrize("p", [2, 7])                 # several windows per tile, one window per tile
def test_attention_window_nan_query_row(dh, p):
    B, H, gh, gw = 2, 2, 2 * p, 3 * p
    g = torch.Generator(device=DEV).manual_seed(dh * 10 + p)
    qkv = torch.randn(B * gh * gw, 3 * H * dh, device=DEV, generator=g).bfloat16()

    def run(x):
        out = torch.full((B * gh * gw, H * dh), 5.0, device=DEV, dtype=torch.bfloat16)
        _lib.attention_window(x, out, B, gh, gw, p, H, dh, dh ** -0.5)
        torch.cuda.synchronize()
        return out
    assert_nan_query_row(run, qkv, gh * gw + gw + 1, dh, f"p={p}")


@pytest.mark.parametrize("dh", [32, 64, 80, 128])
@pytest.mark.parametrize("grid", [False, True])
def test_attention_window_relpos_nan_query_row(dh, grid):
    B, H, w = 2, 2, 7
    gh = gw = 2 * w
    g = torch.Generator(device=DEV).manual_seed(dh * 10 + grid)
    qkv = torch.randn(B * gh * gw, 3 * H * dh, device=DEV, generator=g).bfloat16()
    table = torch.randn(H, (2 * w - 1) ** 2, device=DEV, generator=g)

    def run(x):
        out = torch.full((B * gh * gw, H * dh), 5.0, device=DEV, dtype=torch.bfloat16)
        _lib.attention_window_relpos(x, out, table, B, gh, gw, w, grid, H, dh, dh ** -0.5)
        torch.cuda.synchronize()
        return out
    assert_nan_query_row(run, qkv, gh * gw + gw + 1, dh, f"grid={grid}")


def cls_inputs(B, n, first, H, dh, g):
    I = H * dh
    rows = n + first + 2                  # every image: `first` skipped rows, n context rows, 2 unused rows
    qkv_self = torch.randn(B, 3 * I, device=DEV, generator=g).bfloat16()
    ctx = torch.randn(B * rows, 2 * I + 8, device=DEV, generator=g).bfloat16()
    return qkv_self, ctx, rows


def run_cls(kind, qkv_self, ctx, rows, first, n, H, dh, pre=None, post=None):
    B, I = qkv_self.shape[0], H * dh
    out = torch.full((B, I), 5.0, device=DEV, dtype=torch.bfloat16)
    if kind == "cls":
        _lib.attention_cls(qkv_self, ctx, out, rows, first, n, H, dh, dh ** -0.5)
    else:
        _lib.attention_cls_headmix(qkv_self, ctx, out, rows, first, n, H, dh, dh ** -0.5, pre, post)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("kind", ["cls", "cls_headmix"])
@pytest.mark.parametrize("n,first", [(0, 0), (1, 1), (17, 0), (300, 1)])
def test_attention_cls_isolation_under_poisoning(kind, n, first):
    B, H, dh = 4, 6, 48 if kind == "cls_headmix" else 64
    I = H * dh
    g = torch.Generator(device=DEV).manual_seed(n * 10 + first)
    qkv_self, ctx, rows = cls_inputs(B, n, first, H, dh, g)
    pre, post = torch.randn(H, H, device=DEV, generator=g), torch.randn(H, H, device=DEV, generator=g)
    clean = run_cls(kind, qkv_self, ctx, rows, first, n, H, dh, pre, post)
    assert torch.isfinite(clean.float()).all()
    img = torch.arange(B, device=DEV)
    for b in (1, 0, 3):
        for how in ("nan", "inf_v"):
            s, c = qkv_self.clone(), ctx.clone()
            poison(s, b, b + 1, I, how)
            if how == "nan":
                c[b * rows:(b + 1) * rows] = NAN
            else:
                c[b * rows:(b + 1) * rows, I:2 * I] = INF
            assert_rows_equal(run_cls(kind, s, c, rows, first, n, H, dh, pre, post), clean, img != b,
                              f"poisoned {b} {how}")
    # rows no image reads: the skipped `first` rows, the unused tail rows and columns past 2 I
    c = ctx.clone()
    for b in range(B):
        c[b * rows:b * rows + first] = NAN
        c[b * rows + first + n:(b + 1) * rows] = NAN
    c[:, 2 * I:] = NAN
    assert torch.equal(run_cls(kind, qkv_self, c, rows, first, n, H, dh, pre, post), clean)


def test_attn_pool_isolation_under_poisoning():
    H, dh, lengths = 4, 64, VARLEN_PACK
    I, T, S = H * dh, sum(VARLEN_PACK), len(VARLEN_PACK)
    g = torch.Generator(device=DEV).manual_seed(3)
    kv = torch.randn(T, 2 * I, device=DEV, generator=g).bfloat16()
    qn = torch.randn(I, device=DEV, generator=g)
    cu, _, _ = _lib.varlen_index(lengths, DEV)

    def run(kvx):
        out = torch.full((S, I), 5.0, device=DEV, dtype=torch.bfloat16)
        _lib.attn_pool(kvx, qn, cu, out, H, dh)
        torch.cuda.synchronize()
        return out

    clean = run(kv)
    assert torch.isfinite(clean.float()).all()
    cuh = cu.tolist()
    for s in range(S):
        for how in ("nan", "inf_v"):
            bad = kv.clone()
            if how == "nan":
                bad[cuh[s]:cuh[s + 1]] = NAN
            else:
                bad[cuh[s]:cuh[s + 1], I:] = INF
            assert_rows_equal(run(bad), clean, torch.arange(S) != s, f"poisoned {s} {how}")
    buf = torch.full((T + 50, 2 * I), NAN, device=DEV, dtype=torch.bfloat16)
    buf[:T] = kv
    assert torch.equal(run(buf[:T]), clean)


# ================================================================================================ B. exact key sets
LENGTHS = [1, 2, 15, 16, 17, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512]


def indicator_v(T, local, H, dh, windows):
    """V[t, h*dh + d] = 1 iff local[t] == windows[h] * dh + d: head h probes keys [w dh, w dh + dh) of every
    sequence."""
    j = (torch.as_tensor(windows, device=DEV)[:, None] * dh + torch.arange(dh, device=DEV)[None]).reshape(-1)
    return (local[:, None] == j[None]).to(torch.bfloat16), j


def uniform_expect(local, length, j, mask_self):
    """q = 0: every included key has probability 1/len (1/(len - 1) without the self key), so output column j is
    that for an included key j and exactly 0 for an excluded one."""
    L = length[:, None].double()
    inc = j[None] < length[:, None]
    if mask_self:
        selfk = (j[None] == local[:, None]) & (length[:, None] > 1)
        inc = inc & ~selfk
        L = torch.where(length[:, None] > 1, L - 1, L)
    return torch.where(inc, 1.0 / L, torch.zeros_like(L))


def assert_exact_keys(out, want, what):
    got = out.double()
    zero = want == 0
    assert (got[zero] == 0).all(), f"{what}: {int((got[zero] != 0).sum())} excluded keys contribute"
    rel = ((got[~zero] - want[~zero]).abs() / want[~zero])
    assert rel.max().item() <= BF16_REL, f"{what}: included key off by {rel.max().item():.3g} relative"


def probe_windows(max_len, H, dh):
    """Window lists of H heads per launch covering keys [0, max_len)."""
    nw = (max_len + dh - 1) // dh
    ws = list(range(nw))
    ws += [ws[-1]] * (-len(ws) % H)
    return [ws[i:i + H] for i in range(0, len(ws), H)]


@pytest.mark.parametrize("cfg", sorted(PLAIN_CONFIGS))
@pytest.mark.parametrize("dh", [32, 64, 80, 128])
def test_attention_uniform_exact_key_sets(dh, cfg):
    H, B = 4, 2
    for N in LENGTHS:
        local = torch.arange(B * N, device=DEV) % N
        length = torch.full_like(local, N)
        for wins in probe_windows(N, H, dh):
            qkv = torch.zeros(B * N, 3 * H * dh, device=DEV, dtype=torch.bfloat16)
            qkv[:, H * dh:2 * H * dh] = torch.randn(B * N, H * dh, device=DEV).bfloat16()     # any keys: q = 0
            v, j = indicator_v(B * N, local, H, dh, wins)
            qkv[:, 2 * H * dh:] = v
            out = run_plain(qkv, B, N, H, dh, cfg)
            assert_exact_keys(out, uniform_expect(local, length, j, PLAIN_CONFIGS[cfg][1]), f"N={N} windows {wins}")


def pack_index(lengths):
    lens = torch.tensor(lengths, device=DEV)
    seq = torch.repeat_interleave(torch.arange(len(lengths), device=DEV), lens)
    start = torch.cumsum(lens, 0) - lens
    return seq, torch.arange(int(lens.sum()), device=DEV) - start[seq], lens[seq]


@pytest.mark.parametrize("cfg", sorted(VARLEN_CONFIGS))
@pytest.mark.parametrize("dh", [32, 64, 80, 128])
def test_attention_varlen_uniform_exact_key_sets(dh, cfg):
    """Every boundary length and the long ones (4097, 16384) in one pack of about 24k tokens."""
    H = 1024 // dh if dh != 80 else 12
    lengths = LENGTHS + [4097, 16384, 3, 1]
    _, local, length = pack_index(lengths)
    T = len(local)
    for wins in probe_windows(max(lengths), H, dh):
        qkv = torch.zeros(T, 3 * H * dh, device=DEV, dtype=torch.bfloat16)
        qkv[:, H * dh:2 * H * dh] = 1.0
        v, j = indicator_v(T, local, H, dh, wins)
        qkv[:, 2 * H * dh:] = v
        out = run_varlen(qkv, lengths, H, dh, cfg)
        assert_exact_keys(out, uniform_expect(local, length, j, VARLEN_CONFIGS[cfg]), f"windows {wins}")


def test_attention_varlen_sequence_id_values():
    """V = one-hot(sequence id mod dh), random q / k, several hundred sequences of about 20k tokens: each query gives
    1 in its own sequence's column and exactly 0 in every other."""
    H, dh = 2, 64
    g = torch.Generator(device="cpu").manual_seed(5)
    lengths = torch.randint(1, 140, (300,), generator=g).tolist()
    lengths[7], lengths[100] = 1, 1
    seq, _, _ = pack_index(lengths)
    T = len(seq)
    for cfg in sorted(VARLEN_CONFIGS):
        qkv = torch.randn(T, 3 * H * dh, device=DEV).bfloat16()
        onehot = (seq[:, None] % dh == torch.arange(dh, device=DEV)[None]).to(torch.bfloat16)
        qkv[:, 2 * H * dh:] = onehot.repeat(1, H)
        out = run_varlen(qkv, lengths, H, dh, cfg).double().view(T, H, dh)
        want = onehot.double()[:, None].expand(T, H, dh)
        assert (out[want == 0] == 0).all(), cfg
        assert ((out[want == 1] - 1).abs() <= BF16_REL).all(), cfg


def test_attention_sequence_id_values():
    B, H, dh = 300, 2, 64
    for cfg in sorted(PLAIN_CONFIGS):
        for N in (17, 65, 197):
            seq = torch.arange(B * N, device=DEV) // N
            qkv = torch.randn(B * N, 3 * H * dh, device=DEV).bfloat16()
            onehot = (seq[:, None] % dh == torch.arange(dh, device=DEV)[None]).to(torch.bfloat16)
            qkv[:, 2 * H * dh:] = onehot.repeat(1, H)
            out = run_plain(qkv, B, N, H, dh, cfg).double().view(B * N, H, dh)
            want = onehot.double()[:, None].expand(B * N, H, dh)
            assert (out[want == 0] == 0).all(), (cfg, N)
            assert ((out[want == 1] - 1).abs() <= BF16_REL).all(), (cfg, N)


def dominant_qkv(T, H, dh, alpha, g):
    """q_i = alpha k_i with random +-1 keys: the own key dominates every other by >= e^16, so out_i = v_i (values of
    magnitude 0.5 .. 2.5, so that the other keys' share stays below half an ulp)."""
    k = (torch.randint(0, 2, (T, H * dh), device=DEV, generator=g) * 2 - 1).float()
    sign = torch.randint(0, 2, (T, H * dh), device=DEV, generator=g) * 2 - 1
    v = (sign * (0.5 + 2 * torch.rand(T, H * dh, device=DEV, generator=g))).bfloat16()
    return torch.cat([alpha * k, k, v.float()], 1).bfloat16(), v


@pytest.mark.parametrize("dh", [64, 128])
def test_attention_dominant_key_lands_in_its_own_row(dh):
    H, alpha = 2, 16.0 if dh == 64 else 24.0
    g = torch.Generator(device=DEV).manual_seed(dh)
    for cfg in ("default", "tiled"):
        for N in (1, 2, 17, 65, 128, 129, 197, 257, 512):
            B = 3
            qkv, v = dominant_qkv(B * N, H, dh, alpha, g)
            assert torch.equal(run_plain(qkv, B, N, H, dh, cfg), v), (cfg, N)
    lengths = [1, 2, 65, 129, 511, 4097, 16384, 3]
    qkv, v = dominant_qkv(sum(lengths), H, dh, alpha, g)
    assert torch.equal(run_varlen(qkv, lengths, H, dh, "kb64"), v)


@pytest.mark.parametrize("dh", [32, 48, 64, 80, 128])
def test_attention_headmix_uniform_exact_key_sets(dh):
    """q = 0, post = identity: p = 1/len for every key of the sequence, 0 beyond it."""
    H = 4
    eye = torch.eye(H, device=DEV)
    for N in LENGTHS + [1025, 16384]:
        local = torch.arange(N, device=DEV)
        length = torch.full_like(local, N)
        for wins in probe_windows(N, H, dh):
            qkv = torch.zeros(N, 3 * H * dh, device=DEV, dtype=torch.bfloat16)
            qkv[:, H * dh:2 * H * dh] = torch.randn(N, H * dh, device=DEV).bfloat16()
            v, j = indicator_v(N, local, H, dh, wins)
            qkv[:, 2 * H * dh:] = v
            out = run_headmix(qkv, 1, N, H, dh, None, eye, None)
            assert_exact_keys(out, uniform_expect(local, length, j, False), f"N={N} windows {wins}")


@pytest.mark.parametrize("dh", [32, 64, 80])
@pytest.mark.parametrize("L", [1, 2, 5, 8, 17, 33, 64])
@pytest.mark.parametrize("G", [1, 3])
def test_attention_axial_uniform_exact_key_sets(dh, L, G):
    """q = 0: each kept key of the sequence gets 1/kept; a row with no kept key gets 0 (zero_masked_rows) or 1/L for
    every key of its sequence."""
    if L > 32 and dh == 32 and G == 3:
        pytest.skip("covered by G = 1")
    B, H = 5, 2
    T = B * L * G
    g = torch.Generator(device=DEV).manual_seed(L * 10 + G)
    km = torch.rand(B, L, device=DEV, generator=g) > 0.5
    km[0] = True
    km[2] = False
    km8 = km.to(torch.uint8).contiguous()
    local = (torch.arange(T, device=DEV) // G) % L
    b_of = torch.arange(T, device=DEV) // (L * G)
    for wins in probe_windows(L, H, dh):
        qkv = torch.zeros(T, 3 * H * dh, device=DEV, dtype=torch.bfloat16)
        qkv[:, H * dh:2 * H * dh] = torch.randn(T, H * dh, device=DEV, generator=g).bfloat16()
        v, j = indicator_v(T, local, H, dh, wins)
        qkv[:, 2 * H * dh:] = v
        valid = (j < L)[None].expand(T, -1)
        for mask in (None, km8):
            if mask is None:
                kept, nk = valid, torch.full((T, 1), float(L), device=DEV, dtype=torch.float64)
            else:
                kept = valid & km[b_of][:, j.clamp(max=L - 1)]
                nk = km[b_of].sum(1, keepdim=True).double()
            for zero in (True, False):
                out = run_axial(qkv, mask, B, L, G, H, dh, zero)
                want = torch.where(kept, 1.0 / nk.clamp(min=1), torch.zeros_like(nk))
                if not zero:                 # no kept key: the mean of the sequence's L values
                    want = torch.where((nk == 0) & valid, torch.full_like(want, 1.0 / L), want)
                assert_exact_keys(out, want, f"mask={mask is not None} zero={zero} windows {wins}")


@pytest.mark.parametrize("kind", ["cls", "cls_headmix"])
@pytest.mark.parametrize("first", [0, 1, 3])
def test_attention_cls_uniform_exact_key_sets(kind, first):
    """q = 0: the self key and the n context rows of the image, rows first .. first + n - 1, get 1/(n + 1) each;
    the skipped rows, the unused ones and other images' rows nothing."""
    B, H, dh = 3, 16, 64
    I = H * dh
    for n in (0, 1, 2, 15, 16, 17, 255, 256, 257, 4096, 16384):
        rows = n + first + 2
        for wins in probe_windows(n + 1, H, dh):
            qkv_self = torch.zeros(B, 3 * I, device=DEV, dtype=torch.bfloat16)
            qkv_self[:, I:2 * I] = torch.randn(B, I, device=DEV).bfloat16()
            ctx = torch.zeros(B * rows, 2 * I, device=DEV, dtype=torch.bfloat16)
            ctx[:, :I] = torch.randn(B * rows, I, device=DEV).bfloat16()
            # key index: 0 = self, 1 + r - first for context row r of the image; rows outside the image's context get
            # indices past n, whose output columns must stay 0
            r = torch.arange(B * rows, device=DEV) % rows
            kidx = torch.where((r >= first) & (r < first + n), 1 + r - first, (n + 1) + r)
            v, j = indicator_v(B * rows, kidx, H, dh, wins)
            ctx[:, I:] = v
            vs, _ = indicator_v(B, torch.zeros(B, dtype=torch.long, device=DEV), H, dh, wins)
            qkv_self[:, 2 * I:] = vs
            eye = torch.eye(H, device=DEV)
            out = run_cls(kind, qkv_self, ctx, rows, first, n, H, dh, eye, eye)
            want = torch.where(j[None] < n + 1, 1.0 / (n + 1), 0.0).double().expand(B, -1)
            assert_exact_keys(out, want, f"n={n} windows {wins}")


# ================================================================================================ C. head routing
HEAD_COUNTS = [(H, dh) for dh in (32, 48, 64, 80, 128) for H in range(1, 17) if H * dh <= 1024]


def perm_mixes(H, seed):
    """pre = sigma and post = pi permutation matrices ([input head, output head]): s'_f = s_sigma(f), p'_f = p_pi(f)."""
    pi = torch.randperm(H, generator=torch.Generator().manual_seed(H)).tolist()
    sg = torch.randperm(H, generator=torch.Generator().manual_seed(H + seed)).tolist()
    post, pre = torch.zeros(H, H, device=DEV), torch.zeros(H, H, device=DEV)
    for f in range(H):
        post[pi[f], f] = 1.0
        pre[sg[f], f] = 1.0
    return pi, sg, pre, post


@pytest.mark.parametrize("H,dh", HEAD_COUNTS)
def test_attention_headmix_permutation_routes_heads(H, dh):
    """pre = sigma and post = pi permutation matrices, no LayerNorm: output head f is plain attention with the scores
    of head sigma(pi(f)) and the values of head f -- within the bound of oracle/headmix_bounds.py, whose fp64
    reference routes the heads by the matrices alone."""
    B, N = 2, 77
    g = torch.Generator(device=DEV).manual_seed(H * 1000 + dh)
    qkv = torch.randn(B * N, 3 * H * dh, device=DEV, generator=g).bfloat16()
    _, _, pre, post = perm_mixes(H, 99)
    for use_pre in (False, True):
        p_ = pre if use_pre else None
        out = run_headmix(qkv, B, N, H, dh, p_, post, None)
        Bd.check(out, *HB.headmix_reference(qkv, B, N, H, dh, dh ** -0.5, p_, post), f"permutation pre={use_pre}")


@pytest.mark.parametrize("H,dh", HEAD_COUNTS)
def test_attention_headmix_random_mix_every_head_count(H, dh):
    B, N = 2, 100
    g = torch.Generator(device=DEV).manual_seed(H * 7 + dh)
    qkv = torch.randn(B * N, 3 * H * dh, device=DEV, generator=g).bfloat16()
    pre, post = torch.randn(H, H, device=DEV, generator=g), torch.randn(H, H, device=DEV, generator=g)
    ln = (1 + 0.2 * torch.randn(H, device=DEV, generator=g), 0.1 * torch.randn(H, device=DEV, generator=g), 1e-5)
    for p_, l_ in ((None, None), (pre, None), (None, ln), (pre, ln)):
        out = run_headmix(qkv, B, N, H, dh, p_, post, l_)
        Bd.check(out, *HB.headmix_reference(qkv, B, N, H, dh, dh ** -0.5, p_, post, l_),
                 f"random mix pre={p_ is not None} ln={l_ is not None}")


@pytest.mark.parametrize("H,dh", [(6, 48), (16, 64), (5, 80)])
def test_attention_headmix_random_mix_16384(H, dh):
    N = 16384
    g = torch.Generator(device=DEV).manual_seed(H + dh)
    qkv = torch.randn(N, 3 * H * dh, device=DEV, generator=g).bfloat16()
    pre, post = torch.randn(H, H, device=DEV, generator=g), torch.randn(H, H, device=DEV, generator=g)
    out = run_headmix(qkv, 1, N, H, dh, pre, post, None)
    Bd.check(out, *HB.headmix_reference(qkv, 1, N, H, dh, dh ** -0.5, pre, post), "16384")


@pytest.mark.parametrize("H,dh", HEAD_COUNTS)
def test_attention_cls_headmix_every_head_count(H, dh):
    B, n, first = 3, 197, 1
    g = torch.Generator(device=DEV).manual_seed(H * 31 + dh)
    qkv_self, ctx, rows = cls_inputs(B, n, first, H, dh, g)
    pre, post = torch.randn(H, H, device=DEV, generator=g), torch.randn(H, H, device=DEV, generator=g)
    out = run_cls("cls_headmix", qkv_self, ctx, rows, first, n, H, dh, pre, post)
    Bd.check(out, *FB.cls_headmix_reference(qkv_self, ctx, rows, first, n, H, dh, dh ** -0.5, pre, post), "random")
    # permutations: output head f = plain class attention of scores sigma(pi(f)), values f
    _, _, S, P = perm_mixes(H, 5)
    out = run_cls("cls_headmix", qkv_self, ctx, rows, first, n, H, dh, S, P)
    Bd.check(out, *FB.cls_headmix_reference(qkv_self, ctx, rows, first, n, H, dh, dh ** -0.5, S, P), "permutation")


# ================================================================================================ D. GEMM margins
@pytest.mark.parametrize("M,N,K", [(256, 192, 48), (130, 264, 72), (1, 768, 776), (591, 1000, 200)])
def test_gemm_operand_margins_are_not_read(M, N, K):
    """A[M, K] and W[N, K] views into larger NaN-filled allocations: NaN beyond K (same row stride), in rows of A
    past M and rows of W past N must not change a bit of the output."""
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    ld = K + 24
    a0 = torch.randn(M, K, device=DEV, generator=g).bfloat16()
    w0 = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=DEV, generator=g)

    def run(fill):
        a = torch.full((M + 130, ld), fill, device=DEV, dtype=torch.bfloat16)
        w = torch.full((N + 260, ld), fill, device=DEV, dtype=torch.bfloat16)
        a[:M, :K], w[:N, :K] = a0, w0
        of = torch.zeros(M, N, device=DEV)
        ob = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
        _lib.gemm(a[:M], w[:N], out_f32=of, bias=bias, k=K)
        _lib.gemm(a[:M], w[:N], out_bf16=ob, bias=bias, gelu=True, k=K)
        torch.cuda.synchronize()
        return of, ob

    clean_f, clean_b = run(0.0)
    bad_f, bad_b = run(NAN)
    assert torch.isfinite(clean_f).all()
    assert torch.equal(bad_f, clean_f) and torch.equal(bad_b, clean_b)
    ref = a0.double() @ w0.double().t() + bias.double()
    assert (clean_f.double() - ref).abs().max().item() < 1e-3 * ref.abs().max().item() + 1e-4


# ================================================================================================ models
def one_nan_batch(model, x, bad=1):
    """Logits of the clean batch and of the batch with image `bad` all NaN: every other image bit-identical."""
    xb = x.clone()
    xb[bad] = NAN
    with torch.inference_mode():
        if hasattr(model, "fused_reason"):
            assert model.fused_reason(x) is None
        _lib.reset_launch_count()
        clean = model(x)
        dirty = model(xb)
        torch.cuda.synchronize()
        assert _lib.launch_count() > 0
    keep = torch.arange(x.shape[0], device=DEV) != bad
    assert torch.isfinite(clean.float()).all()
    assert torch.equal(dirty[keep], clean[keep])


def test_vit_batch_with_one_nan_image():
    from vit_pytorch_b200 import ViT
    torch.manual_seed(0)
    m = ViT(image_size=224, patch_size=16, num_classes=10, dim=192, depth=2, heads=3, mlp_dim=384).eval()
    m = m.to(DEV, torch.bfloat16)
    x = torch.randn(4, 3, 224, 224, device=DEV).bfloat16()          # N = 197: 59 rows of the next image in a block
    one_nan_batch(m, x, bad=1)
    one_nan_batch(m, x, bad=3)


def test_vit_long_sequence_batch_with_one_nan_image():
    from vit_pytorch_b200 import ViT
    torch.manual_seed(1)
    m = ViT(image_size=384, patch_size=16, num_classes=10, dim=128, depth=2, heads=2, mlp_dim=256).eval()
    m = m.to(DEV, torch.bfloat16)
    x = torch.randn(3, 3, 384, 384, device=DEV).bfloat16()          # N = 577 > 512: the varlen path
    one_nan_batch(m, x, bad=1)


def test_deepvit_batch_with_one_nan_image():
    from vit_pytorch_b200.deepvit import DeepViT
    torch.manual_seed(2)
    m = DeepViT(image_size=64, patch_size=8, num_classes=10, dim=128, depth=2, heads=4, dim_head=32,
                mlp_dim=256).eval().to(DEV, torch.bfloat16)
    x = torch.randn(4, 3, 64, 64, device=DEV).bfloat16()            # N = 65
    one_nan_batch(m, x, bad=1)


def test_cait_batch_with_one_nan_image():
    from vit_pytorch_b200.cait import CaiT
    torch.manual_seed(3)
    m = CaiT(image_size=64, patch_size=8, num_classes=10, dim=144, depth=2, cls_depth=1, heads=3, dim_head=48,
             mlp_dim=256).eval().to(DEV, torch.bfloat16)
    x = torch.randn(4, 3, 64, 64, device=DEV).bfloat16()
    one_nan_batch(m, x, bad=1)


def test_vivit_factorized_encoder_batch_with_one_nan_video():
    from vit_pytorch_b200.vivit import ViViT
    torch.manual_seed(4)
    m = ViViT(image_size=32, image_patch_size=8, frames=16, frame_patch_size=2, num_classes=10, dim=128,
              spatial_depth=1, temporal_depth=2, heads=2, dim_head=64, mlp_dim=256).eval().to(DEV, torch.bfloat16)
    x = torch.randn(5, 3, 16, 32, 32, device=DEV).bfloat16()        # temporal sequences of 9 tokens, G = 1
    one_nan_batch(m, x, bad=1)
