"""Drop-in `RegionViT` for lucidrains/vit-pytorch's `vit_pytorch.regionvit.RegionViT` (regional and local tokens: the
region tokens attend to each other, then every window of local tokens attends together with its region token), with
`ChanLayerNorm`, `Downsample`, `PEG`, `FeedForward`, `Attention` and `R2LTransformer` of the same file, and a fused
sm_90a forward.

Same constructor keywords and defaults, parameter names / shapes / registration order (=> identical `state_dict` and
identical random init under the same seed).  As in the reference (regionvit.py:255), every R2LTransformer is built
without `heads` or `dim_head`: 4 heads of 32 at every stage width.  The PyTorch graph mirrors the reference without
einops (the Rearrange / Reduce layers as parameter-free modules at the same indices) and raises where it raises: an
AssertionError on an image that the region or local patch does not divide, and an error from the window split when
the local map is not a multiple of the region map's windows.

Fused forward, one fp32 stream per stage: the B local maps channels-last, token (b, y, x) of the lh x lw map at row
(b*lh + y)*lw + x, followed by the B region maps, token (b, i, j) of the rh x rw map at row B*lh*lw + (b*rh + i)*rw + j.
  * stage 1: the local encoder as b200vit_conv_im2col_nchw (8 x 8, stride 4, padding 3) + GEMM with bias into the
    local rows (tokenize_local_3_conv: three im2col + GEMMs, the first two followed by b200vit_head_layernorm_gelu as
    ChanLayerNorm + GELU over one head of width dim[0]); the region encoder as b200vit_patchify_nd (the (p1 p2 c)
    patches of region_patch_size) + GEMM with bias (weight columns permuted from the reference's (c p1 p2)) into the
    region rows; in fold mode b200vit_rowstats_cast primes the LN-folded chain;
  * stages 2 to 4: the shared Downsample (3 x 3, stride 2) as b200vit_conv_im2col_nhwc of both maps' bf16 copies and
    one GEMM with bias into the next stage's stream; with use_peg the local rows' GEMM goes to a scratch map and
    b200vit_peg writes them into the stream, the region rows' GEMM straight into it;
  * R2LTransformer: TransformerEngine.run_blocks with `grid` the local map and `regions` the region map: per layer the
    regional attention (QKV GEMM, b200vit_attention, out-projection residual on the region rows), the QKV GEMM over all
    rows, b200vit_attention_region_local, the out-projection residual and the GELU feed-forward (engine.py);
  * head: b200vit_mean_pool over the region rows, b200vit_layernorm on the B pooled rows, the classifier GEMM.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
from torch import nn

from . import _lib
from .engine import (HEAD_WIDTHS, PEG_KERNEL_SIZES, EncoderLayer, FusedEncoder, FusedWeightsMixin, Norm,
                     RegionLocalBlock, _bf16_rows, _f32, cached, common_reason, head_engine, head_ln_pool, on_device,
                     why_not_fused)
from .sep_vit import conv_weights, peg_weights

__all__ = ["Attention", "ChanLayerNorm", "Downsample", "FeedForward", "PEG", "R2LTransformer", "RegionViT",
           "cast_tuple", "default", "divisible_by", "exists"]


def exists(val):
    return val is not None


def default(val, d):
    return val if exists(val) else d


def cast_tuple(val, length=1):
    return val if isinstance(val, tuple) else ((val,) * length)


def divisible_by(val, d):
    return (val % d) == 0


class ChanLayerNorm(nn.Module):
    def __init__(self, dim, eps=1e-5):
        super().__init__()
        self.eps = eps
        self.g = nn.Parameter(torch.ones(1, dim, 1, 1))
        self.b = nn.Parameter(torch.zeros(1, dim, 1, 1))

    def forward(self, x):
        var = torch.var(x, dim=1, unbiased=False, keepdim=True)
        mean = torch.mean(x, dim=1, keepdim=True)
        return (x - mean) / (var + self.eps).sqrt() * self.g + self.b


class Downsample(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.conv = nn.Conv2d(dim_in, dim_out, 3, stride=2, padding=1)

    def forward(self, x):
        return self.conv(x)


class PEG(nn.Module):
    def __init__(self, dim, kernel_size=3):
        super().__init__()
        self.proj = nn.Conv2d(dim, dim, kernel_size=kernel_size, padding=kernel_size // 2, groups=dim, stride=1)

    def forward(self, x):
        return self.proj(x) + x


def FeedForward(dim, mult=4, dropout=0.):
    return nn.Sequential(
        nn.LayerNorm(dim),
        nn.Linear(dim, dim * mult, 1),
        nn.GELU(),
        nn.Dropout(dropout),
        nn.Linear(dim * mult, dim, 1)
    )


class Attention(nn.Module):
    def __init__(
        self,
        dim,
        heads=4,
        dim_head=32,
        dropout=0.
    ):
        super().__init__()
        self.heads = heads
        self.scale = dim_head ** -0.5
        inner_dim = dim_head * heads
        self.dim_head = dim_head

        self.norm = nn.LayerNorm(dim)
        self.dropout = nn.Dropout(dropout)
        self.to_qkv = nn.Linear(dim, inner_dim * 3, bias=False)

        self.to_out = nn.Sequential(
            nn.Linear(inner_dim, dim),
            nn.Dropout(dropout)
        )

    def forward(self, x, rel_pos_bias=None):
        h = self.heads

        # prenorm

        x = self.norm(x)

        q, k, v = self.to_qkv(x).chunk(3, dim=-1)

        # 'b n (h d) -> b h n d'
        q, k, v = (t.reshape(t.shape[0], t.shape[1], h, -1).transpose(1, 2) for t in (q, k, v))
        q = q * self.scale

        sim = torch.matmul(q, k.transpose(-1, -2))

        # add relative positional bias for local tokens

        if exists(rel_pos_bias):
            sim = sim + rel_pos_bias

        attn = sim.softmax(dim=-1)
        attn = self.dropout(attn)

        # merge heads: 'b h n d -> b n (h d)'
        out = torch.matmul(attn, v)
        out = out.transpose(1, 2).reshape(out.shape[0], out.shape[2], -1)
        return self.to_out(out)


def _windows(t, lh, wh, ww):
    """'b (h w) d -> b h w d', then 'b (h p1) (w p2) d -> (b h w) (p1 p2) d' with p1 = wh, p2 = ww
    (regionvit.py:169-170); raises, as einops does, when the map does not split into whole windows."""
    b, n, d = t.shape
    if n % lh:
        raise RuntimeError(f"'b (h w) d -> b h w d': {n} tokens do not split into {lh} rows")
    lw = n // lh
    if wh == 0 or ww == 0 or lh % wh or lw % ww:
        raise RuntimeError(f"'b (h p1) (w p2) d -> (b h w) (p1 p2) d': a {lh} x {lw} map does not split into "
                           f"{wh} x {ww} windows")
    t = t.reshape(b, lh // wh, wh, lw // ww, ww, d).permute(0, 1, 3, 2, 4, 5)
    return t.reshape(-1, wh * ww, d)


class R2LTransformer(FusedEncoder, nn.Module):
    """depth x (regional attention, region-to-local attention, FeedForward) (reference regionvit.py:114-190).  A direct
    call on (b, c, h, w) bf16 CUDA maps runs fused through engine() and returns both maps as the reference does."""

    def __init__(
        self,
        dim,
        *,
        window_size,
        depth=4,
        heads=4,
        dim_head=32,
        attn_dropout=0.,
        ff_dropout=0.,
    ):
        super().__init__()
        self.layers = nn.ModuleList([])

        self.window_size = window_size
        rel_positions = 2 * window_size - 1
        self.local_rel_pos_bias = nn.Embedding(rel_positions ** 2, heads)

        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, heads=heads, dim_head=dim_head, dropout=attn_dropout),
                FeedForward(dim, dropout=ff_dropout)
            ]))
        self._dropout_p = float(max(attn_dropout, ff_dropout))

    def encoder_layers(self) -> Tuple[List[EncoderLayer], Optional[Norm]]:
        layers = []
        block = RegionLocalBlock(bias=self.local_rel_pos_bias.weight, window=self.window_size)
        for attn, ff in self.layers:
            layers.append(EncoderLayer(
                ln1=Norm.of(attn.norm), qkv_w=attn.to_qkv.weight, out_w=attn.to_out[0].weight,
                out_b=attn.to_out[0].bias, ln2=Norm.of(ff[0]), fc1_w=ff[1].weight, fc1_b=ff[1].bias,
                fc2_w=ff[4].weight, fc2_b=ff[4].bias, heads=attn.heads, dim_head=attn.dim_head, scale=attn.scale,
                attention=block))
        return layers, None

    def map_reason(self, lh: int, lw: int, rh: int, rw: int) -> Optional[str]:
        """Why an lh x lw local map with an rh x rw region map cannot run fused, or None."""
        return self.engine().unsupported_reason(lh * lw, grid=(lh, lw), regions=(rh, rw))

    def fused_reason(self, local_tokens: torch.Tensor, region_tokens: torch.Tensor) -> Optional[str]:
        if local_tokens.dim() != 4 or region_tokens.dim() != 4:
            return "inputs are not (b, c, h, w) maps"
        if local_tokens.shape[:2] != region_tokens.shape[:2]:
            return "the local and region maps differ in batch or channels"
        r = common_reason(self, local_tokens, encoders=(self,), dropout_p=self._dropout_p, inside="transformer")
        if r is None:
            r = why_not_fused([], region_tokens, training=self.training, dropout_p=self._dropout_p)
        if r is not None:
            return r
        if region_tokens.device != local_tokens.device:
            return "the local and region maps are on different devices"
        if self.training:
            return "training mode (the fused path is inference only)"
        if local_tokens.shape[1] % 8:
            return f"dim={local_tokens.shape[1]} (the GEMMs need multiples of 8)"
        return self.map_reason(*local_tokens.shape[2:], *region_tokens.shape[2:])

    def forward(self, local_tokens, region_tokens):
        if self.fused_reason(local_tokens, region_tokens) is None:
            return self.forward_fused(local_tokens, region_tokens)
        return self.forward_eager(local_tokens, region_tokens)

    def forward_fused(self, local_tokens, region_tokens):
        b, c, lh, lw = local_tokens.shape
        rh, rw = region_tokens.shape[2:]
        Ml = b * lh * lw
        with on_device(local_tokens):
            x = torch.cat((local_tokens.permute(0, 2, 3, 1).reshape(Ml, c),
                           region_tokens.permute(0, 2, 3, 1).reshape(-1, c))).float()
            self.engine().run_blocks(x, b, lh * lw, grid=(lh, lw), regions=(rh, rw))
            out = x.to(torch.bfloat16)
        local = out[:Ml].view(b, lh, lw, c).permute(0, 3, 1, 2).contiguous()
        region = out[Ml:].view(b, rh, rw, c).permute(0, 3, 1, 2).contiguous()
        return local, region

    def forward_eager(self, local_tokens, region_tokens):
        device = local_tokens.device
        lh, lw = local_tokens.shape[-2:]
        rh, rw = region_tokens.shape[-2:]
        window_size_h, window_size_w = lh // rh, lw // rw

        # 'b c h w -> b (h w) c'
        local_tokens = local_tokens.flatten(2).transpose(1, 2)
        region_tokens = region_tokens.flatten(2).transpose(1, 2)

        # calculate local relative positional bias

        h_range = torch.arange(window_size_h, device=device)
        w_range = torch.arange(window_size_w, device=device)

        grid_x, grid_y = torch.meshgrid(h_range, w_range, indexing='ij')
        grid = torch.stack((grid_x, grid_y))
        grid = grid.reshape(2, -1)
        grid = (grid[:, :, None] - grid[:, None, :]) + (self.window_size - 1)
        bias_indices = (grid * torch.tensor([1, self.window_size * 2 - 1], device=device)[:, None, None]).sum(dim=0)
        rel_pos_bias = self.local_rel_pos_bias(bias_indices)
        rel_pos_bias = rel_pos_bias.permute(2, 0, 1)[None]                   # 'i j h -> () h i j'
        rel_pos_bias = nn.functional.pad(rel_pos_bias, (1, 0, 1, 0), value=0)

        # go through r2l transformer layers

        for attn, ff in self.layers:
            region_tokens = attn(region_tokens) + region_tokens

            # concat region tokens to local tokens

            local_tokens = _windows(local_tokens, lh, window_size_h, window_size_w)
            region_tokens = region_tokens.reshape(-1, 1, region_tokens.shape[-1])   # 'b n d -> (b n) () d'

            # do self attention on local tokens, along with its regional token

            region_and_local_tokens = torch.cat((region_tokens, local_tokens), dim=1)
            region_and_local_tokens = attn(region_and_local_tokens, rel_pos_bias=rel_pos_bias) + region_and_local_tokens

            # feedforward

            region_and_local_tokens = ff(region_and_local_tokens) + region_and_local_tokens

            # split back local and regional tokens

            region_tokens, local_tokens = region_and_local_tokens[:, :1], region_and_local_tokens[:, 1:]
            # '(b h w) (p1 p2) d -> b (h p1 w p2) d'
            nh, nw, d = lh // window_size_h, lw // window_size_w, local_tokens.shape[-1]
            local_tokens = local_tokens.reshape(-1, nh, nw, window_size_h, window_size_w, d)
            local_tokens = local_tokens.permute(0, 1, 3, 2, 4, 5).reshape(-1, lh * lw, d)
            region_tokens = region_tokens.reshape(-1, rh * rw, d)             # '(b n) () d -> b n d'

        # 'b (h w) c -> b c h w'
        local_tokens = local_tokens.transpose(1, 2).reshape(local_tokens.shape[0], -1, lh, lw)
        region_tokens = region_tokens.transpose(1, 2).reshape(region_tokens.shape[0], -1, rh, rw)
        return local_tokens, region_tokens


class _RegionPatches(nn.Module):
    """Rearrange('b c (h p1) (w p2) -> b (c p1 p2) h w', p1 = p2 = patch) (reference regionvit.py:238), without
    einops."""

    def __init__(self, patch):
        super().__init__()
        self.patch = patch

    def forward(self, x):
        b, c, H, W = x.shape
        p = self.patch
        if H % p or W % p:
            raise RuntimeError(f"'b c (h p1) (w p2) -> b (c p1 p2) h w': a {H} x {W} image does not split into "
                               f"{p} x {p} patches")
        x = x.reshape(b, c, H // p, p, W // p, p).permute(0, 1, 3, 5, 2, 4)
        return x.reshape(b, c * p * p, H // p, W // p)


class _MeanHW(nn.Module):
    """Reduce('b c h w -> b c', 'mean') (reference regionvit.py:263), without einops."""

    def forward(self, x):
        if x.dim() != 4:
            raise RuntimeError(f"Reduce('b c h w -> b c'): expected 4 dims, got {x.dim()}")
        return x.mean(dim=(2, 3))


def region_weights(conv: nn.Conv2d, channels: int, p: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """(bf16 [out, p*p*C] GEMM weight, fp32 bias) of the region encoder's 1 x 1 convolution over the (c p1 p2) patches,
    columns permuted to the (p1 p2 c) order of b200vit_patchify_nd."""
    w = conv.weight.detach().reshape(conv.out_channels, channels, p, p).permute(0, 2, 3, 1)
    return _bf16_rows(w.reshape(conv.out_channels, -1).to(torch.bfloat16), None), _f32(conv.bias)


class RegionViT(FusedWeightsMixin, nn.Module):
    def __init__(
        self,
        *,
        dim=(64, 128, 256, 512),
        depth=(2, 2, 8, 2),
        window_size=7,
        num_classes=1000,
        tokenize_local_3_conv=False,
        local_patch_size=4,
        use_peg=False,
        attn_dropout=0.,
        ff_dropout=0.,
        channels=3,
    ):
        super().__init__()
        dim = cast_tuple(dim, 4)
        depth = cast_tuple(depth, 4)
        assert len(dim) == 4, 'dim needs to be a single value or a tuple of length 4'
        assert len(depth) == 4, 'depth needs to be a single value or a tuple of length 4'

        self.local_patch_size = local_patch_size

        region_patch_size = local_patch_size * window_size
        self.region_patch_size = local_patch_size * window_size

        init_dim, *_, last_dim = dim

        # local and region encoders

        if tokenize_local_3_conv:
            self.local_encoder = nn.Sequential(
                nn.Conv2d(3, init_dim, 3, 2, 1),
                ChanLayerNorm(init_dim),
                nn.GELU(),
                nn.Conv2d(init_dim, init_dim, 3, 2, 1),
                ChanLayerNorm(init_dim),
                nn.GELU(),
                nn.Conv2d(init_dim, init_dim, 3, 1, 1)
            )
        else:
            self.local_encoder = nn.Conv2d(3, init_dim, 8, 4, 3)

        self.region_encoder = nn.Sequential(
            _RegionPatches(region_patch_size),
            nn.Conv2d((region_patch_size ** 2) * channels, init_dim, 1)
        )

        # layers

        current_dim = init_dim
        self.layers = nn.ModuleList([])

        for ind, dim, num_layers in zip(range(4), dim, depth):
            not_first = ind != 0
            need_downsample = not_first
            need_peg = not_first and use_peg

            self.layers.append(nn.ModuleList([
                Downsample(current_dim, dim) if need_downsample else nn.Identity(),
                PEG(dim) if need_peg else nn.Identity(),
                R2LTransformer(dim, depth=num_layers, window_size=window_size, attn_dropout=attn_dropout,
                               ff_dropout=ff_dropout)
            ]))

            current_dim = dim

        # final logits

        self.to_logits = nn.Sequential(
            _MeanHW(),
            nn.LayerNorm(last_dim),
            nn.Linear(last_dim, num_classes)
        )
        self._channels = channels
        self._three_conv = bool(tokenize_local_3_conv)
        self._dropout_p = float(max(attn_dropout, ff_dropout))

    # ---------------------------------------------------------------------------------------------- dispatch
    def stage_maps(self, H: int, W: int) -> List[Tuple[int, int, int, int]]:
        """(lh, lw, rh, rw), the local and region maps of every stage, for an H x W image."""
        enc = self.local_encoder
        convs = [c for c in enc if isinstance(c, nn.Conv2d)] if self._three_conv else [enc]
        lh, lw = H, W
        for c in convs:
            lh = _lib.conv_out_size(lh, c.kernel_size[0], c.stride[0], c.padding[0])
            lw = _lib.conv_out_size(lw, c.kernel_size[1], c.stride[1], c.padding[1])
        rh, rw = H // self.region_patch_size, W // self.region_patch_size
        maps = []
        for i in range(len(self.layers)):
            if i > 0:
                lh, lw, rh, rw = (_lib.conv_out_size(n, 3, 2, 1) for n in (lh, lw, rh, rw))
            maps.append((lh, lw, rh, rw))
        return maps

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4:
            return "input is not (B, C, H, W)"
        if img.shape[1] != 3 or self._channels != 3:
            return (f"an input of {img.shape[1]} channels for a model of channels={self._channels} (the local encoder "
                    f"takes 3 and the region encoder `channels`; the reference raises otherwise)")
        H, W = img.shape[2:]
        if H % self.region_patch_size or W % self.region_patch_size or H % self.local_patch_size \
                or W % self.local_patch_size:
            return (f"a {H} x {W} image is not divisible by the region patch size {self.region_patch_size} and the "
                    f"local patch size {self.local_patch_size} (the reference raises)")
        r = common_reason(self, img, encoders=[t for _, _, t in self.layers], dropout_p=self._dropout_p)
        if r is not None:
            return r
        if self.training:
            return "training mode (the fused path is inference only)"
        d0 = self.region_encoder[1].out_channels
        if self._three_conv and d0 not in HEAD_WIDTHS:
            return (f"tokenize_local_3_conv with dim[0]={d0} (the channel LayerNorm + GELU kernel takes 32, 64, 80 "
                    f"and 128)")
        for i, ((_, peg, tr), maps) in enumerate(zip(self.layers, self.stage_maps(H, W))):
            D = tr.layers[0][0].norm.normalized_shape[0] if len(tr.layers) else d0
            if D % 8:
                return f"stage {i + 1}: width {D} (the GEMMs need multiples of 8)"
            if isinstance(peg, PEG) and peg.proj.kernel_size[0] not in PEG_KERNEL_SIZES:
                return (f"PEG kernel_size={peg.proj.kernel_size[0]} (the positional-encoding kernel is built for 1, 3, "
                        f"5 and 7)")
            if min(maps) < 1:
                return f"stage {i + 1}: an empty map"
            r = tr.map_reason(*maps)
            if r is not None:
                return f"stage {i + 1}: {r} (the PyTorch graph raises where the maps do not split)"
        return None

    def forward(self, x):
        if self.fused_reason(x) is None:
            with on_device(x):
                return self.forward_fused(x)
        return self.forward_eager(x)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, x):
        *_, h, w = x.shape
        assert divisible_by(h, self.region_patch_size) and divisible_by(w, self.region_patch_size), \
            'height and width must be divisible by region patch size'
        assert divisible_by(h, self.local_patch_size) and divisible_by(w, self.local_patch_size), \
            'height and width must be divisible by local patch size'

        local_tokens = self.local_encoder(x)
        region_tokens = self.region_encoder(x)

        for down, peg, transformer in self.layers:
            local_tokens, region_tokens = down(local_tokens), down(region_tokens)
            local_tokens = peg(local_tokens)
            local_tokens, region_tokens = transformer(local_tokens, region_tokens)

        return self.to_logits(region_tokens)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def prepared(self) -> dict:
        """'local<j>.w' / '.b' (the local encoder's convolutions as GEMMs, 'local<j>.g' / '.beta' its ChanLayerNorms),
        'region.w' / '.b', and 'down<i>.w' / '.b', 'peg<i>.w' / '.b' of every stage after the first."""
        params = list(self.local_encoder.parameters()) + list(self.region_encoder.parameters())
        params += [p for down, peg, _ in self.layers for p in (*down.parameters(), *peg.parameters())]
        return cached(self, "_prepared", params, self._build)

    def _build(self) -> dict:
        t = {}
        if self._three_conv:
            for j in (0, 3, 6):
                t[f"local{j}.w"], t[f"local{j}.b"] = conv_weights(self.local_encoder[j], channels_last=j > 0)
            for j in (1, 4):
                ln = self.local_encoder[j]
                t[f"local{j}.g"], t[f"local{j}.beta"] = _f32(ln.g.reshape(-1)), _f32(ln.b.reshape(-1))
        else:
            t["local0.w"], t["local0.b"] = conv_weights(self.local_encoder, channels_last=False)
        t["region.w"], t["region.b"] = region_weights(self.region_encoder[1], self._channels, self.region_patch_size)
        for i, (down, peg, _) in enumerate(self.layers):
            if isinstance(down, Downsample):
                t[f"down{i}.w"], t[f"down{i}.b"] = conv_weights(down.conv, channels_last=True)
            if isinstance(peg, PEG):
                t[f"peg{i}.w"], t[f"peg{i}.b"] = peg_weights(peg)
        return t

    def _local_tokens(self, img: torch.Tensor, t: dict, x: torch.Tensor) -> None:
        """The local encoder into x [B*lh*lw, d0] fp32."""
        dev, B = img.device, img.shape[0]
        bf = dict(device=dev, dtype=torch.bfloat16)
        if not self._three_conv:
            c = self.local_encoder
            col = torch.empty(x.shape[0], t["local0.w"].shape[1], **bf)
            _lib.conv_im2col_nchw(img, col, c.kernel_size[0], c.stride[0], c.padding[0])
            _lib.gemm(col, t["local0.w"], out_f32=x, bias=t["local0.b"])
            return
        h, w, y = img.shape[2], img.shape[3], None
        for j in (0, 3, 6):
            c = self.local_encoder[j]
            k, s, p = c.kernel_size[0], c.stride[0], c.padding[0]
            oh, ow = _lib.conv_out_size(h, k, s, p), _lib.conv_out_size(w, k, s, p)
            col = torch.empty(B * oh * ow, t[f"local{j}.w"].shape[1], **bf)
            if j == 0:
                _lib.conv_im2col_nchw(img, col, k, s, p)
            else:
                _lib.conv_im2col_nhwc(y, col, B, h, w, k, s, p)
            h, w = oh, ow
            if j == 6:
                _lib.gemm(col, t[f"local{j}.w"], out_f32=x, bias=t[f"local{j}.b"])
                return
            y = torch.empty(B * h * w, c.out_channels, **bf)
            _lib.gemm(col, t[f"local{j}.w"], out_bf16=y, bias=t[f"local{j}.b"])
            # ChanLayerNorm + GELU: one head as wide as the channels
            ln = self.local_encoder[j + 1]
            _lib.head_layernorm_gelu(y, t[f"local{j + 1}.g"], t[f"local{j + 1}.beta"], 1, c.out_channels, eps=ln.eps)

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        dev = img.device
        bf, f32 = dict(device=dev, dtype=torch.bfloat16), dict(device=dev, dtype=torch.float32)
        t = self.prepared()
        img = img.contiguous()
        B = img.shape[0]
        x, prev, maps_prev = None, None, None
        for i, ((down, peg, tr), maps) in enumerate(zip(self.layers, self.stage_maps(img.shape[2], img.shape[3]))):
            lh, lw, rh, rw = maps
            Ml, Mr = B * lh * lw, B * rh * rw
            if i == 0:
                D = self.region_encoder[1].out_channels
                x = torch.empty(Ml + Mr, D, **f32)
                self._local_tokens(img, t, x[:Ml])
                P = self.region_patch_size
                col = torch.empty(Mr, t["region.w"].shape[1], **bf)
                _lib.patchify_nd(img, col, (P, P))
                _lib.gemm(col, t["region.w"], out_f32=x[Ml:], bias=t["region.b"])
            else:
                # the shared Downsample on both maps' bf16 copies: one im2col buffer, local rows then region rows
                plh, plw, prh, prw = maps_prev
                pMl = B * plh * plw
                xb = prev.engine().stream_bf16(x)
                c = down.conv
                D = c.out_channels
                col = torch.empty(Ml + Mr, t[f"down{i}.w"].shape[1], **bf)
                _lib.conv_im2col_nhwc(xb[:pMl], col[:Ml], B, plh, plw, 3, 2, 1)
                _lib.conv_im2col_nhwc(xb[pMl:], col[Ml:], B, prh, prw, 3, 2, 1)
                x = torch.empty(Ml + Mr, D, **f32)
                if isinstance(peg, PEG):
                    # the PEG writes out of place: the local rows' GEMM into a scratch map, the region rows' into x
                    y = torch.empty(Ml, D, **f32)
                    _lib.gemm(col[:Ml], t[f"down{i}.w"], out_f32=y, bias=t[f"down{i}.b"])
                    _lib.gemm(col[Ml:], t[f"down{i}.w"], out_f32=x[Ml:], bias=t[f"down{i}.b"])
                    _lib.peg(y, t[f"peg{i}.w"], t[f"peg{i}.b"], x[:Ml], B, lh, lw, peg.proj.kernel_size[0])
                else:
                    _lib.gemm(col, t[f"down{i}.w"], out_f32=x, bias=t[f"down{i}.b"])
            eng = tr.engine()
            xb, stats = eng.entry_buffers(Ml + Mr, dev)
            if xb is not None:
                _lib.rowstats_cast(x, xb, stats)
            eng.run_blocks(x, B, lh * lw, primed=xb is not None, grid=(lh, lw), regions=(rh, rw))
            prev, maps_prev = tr, maps
        # head: mean over the region tokens, LayerNorm of the B pooled rows, the classifier
        lh, lw, rh, rw = maps_prev
        pooled = head_ln_pool(self, self.to_logits[1], x[B * lh * lw:], B, rh * rw, mean=True)
        return head_engine(self, self.to_logits[2]).run(pooled)
