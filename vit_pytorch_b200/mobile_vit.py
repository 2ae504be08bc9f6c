"""Drop-in `MobileViT` for lucidrains/vit-pytorch's `vit_pytorch.mobile_vit.MobileViT` (MobileNetV2 blocks and
MobileViT blocks: local 3 x 3 convolutions, a transformer over strided patch groups, fusion), with `conv_1x1_bn`,
`conv_nxn_bn`, `FeedForward`, `Attention`, `Transformer`, `MV2Block` and `MobileViTBlock` of the same file, and a fused
sm_90a forward.

Same constructor keywords, parameter and buffer names / shapes / registration order (=> identical `state_dict` and
identical random init under the same seed), `stem.3`'s input width `channels[2]` included (reference
mobile_vit.py:203-206).  The PyTorch graph mirrors the reference without einops and raises where it raises: a block
map that (ph, pw) does not divide, `kernel_size != 3` (padding 1 changes the map and torch.cat fails) and
`channels[2] != channels[3]`.

Fused forward, channels-last throughout: token (b, y, x) of an h x w map is row (b*h + y)*w + x.
  * conv1: b200vit_conv_im2col_nchw (k 3, s 2, p 1), then a GEMM with the BatchNorm folded and SiLU;
  * MV2Block: the 1 x 1 GEMM with its BatchNorm folded and SiLU (none when expansion == 1), b200vit_mbconv_dwconv_ex
    (stride 1 or 2, BatchNorm folded, SiLU, no channel sums), the 1 x 1 GEMM with its BatchNorm folded, adding the
    fp32 input when use_res_connect;
  * MobileViTBlock: conv1 as b200vit_conv_im2col_nhwc + GEMM (BatchNorm folded, SiLU); conv2 as a GEMM (BatchNorm
    folded, SiLU) into the fp32 stream; the transformer layers through TransformerEngine.run_blocks with the map as
    `grid` and the patch as `groups` (b200vit_attention_groups, SiLU feed-forward); conv3 as a GEMM (BatchNorm folded,
    SiLU) writing columns [0, C) of the [M, 2C] concatenation, whose columns [C, 2C) the block's input MV2Block wrote
    (conv1's im2col reads that column slice in place, b200vit_conv_im2col_nhwc_ex);
    conv4 as b200vit_conv_im2col_nhwc over the 2C channels + GEMM (BatchNorm folded, SiLU);
  * to_logits: GEMM (BatchNorm folded, SiLU), b200vit_mean_pool, the bias-free classifier GEMM.
BatchNorm runs on its running statistics: a BatchNorm2d in training mode sends the call to the PyTorch graph.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
from torch import nn

from . import _lib
from .engine import (EncoderLayer, FusedEncoder, FusedWeightsMixin, Norm, PatchGroups, _bf16_rows, cached,
                     common_reason, head_engine, on_device)
from .levit import fold_bn
from .xcit import batchnorm_reason

__all__ = ["Attention", "FeedForward", "MV2Block", "MobileViT", "MobileViTBlock", "Transformer", "conv_1x1_bn",
           "conv_nxn_bn"]


def conv_1x1_bn(inp, oup):
    return nn.Sequential(
        nn.Conv2d(inp, oup, 1, 1, 0, bias=False),
        nn.BatchNorm2d(oup),
        nn.SiLU()
    )


def conv_nxn_bn(inp, oup, kernel_size=3, stride=1):
    return nn.Sequential(
        nn.Conv2d(inp, oup, kernel_size, stride, 1, bias=False),
        nn.BatchNorm2d(oup),
        nn.SiLU()
    )


class FeedForward(nn.Module):
    def __init__(self, dim, hidden_dim, dropout=0.):
        super().__init__()
        self.net = nn.Sequential(
            nn.LayerNorm(dim),
            nn.Linear(dim, hidden_dim),
            nn.SiLU(),
            nn.Dropout(dropout),
            nn.Linear(hidden_dim, dim),
            nn.Dropout(dropout)
        )

    def forward(self, x):
        return self.net(x)


class Attention(nn.Module):
    def __init__(self, dim, heads=8, dim_head=64, dropout=0.):
        super().__init__()
        inner_dim = dim_head * heads
        self.heads = heads
        self.scale = dim_head ** -0.5

        self.norm = nn.LayerNorm(dim)
        self.attend = nn.Softmax(dim=-1)
        self.dropout = nn.Dropout(dropout)

        self.to_qkv = nn.Linear(dim, inner_dim * 3, bias=False)

        self.to_out = nn.Sequential(
            nn.Linear(inner_dim, dim),
            nn.Dropout(dropout)
        )
        self.dim_head = dim_head

    def forward(self, x):
        x = self.norm(x)
        qkv = self.to_qkv(x).chunk(3, dim=-1)

        # 'b p n (h d) -> b p h n d'
        q, k, v = (t.reshape(*t.shape[:3], self.heads, -1).transpose(2, 3) for t in qkv)

        dots = torch.matmul(q, k.transpose(-1, -2)) * self.scale

        attn = self.attend(dots)
        attn = self.dropout(attn)

        out = torch.matmul(attn, v)
        # 'b p h n d -> b p n (h d)'
        out = out.transpose(2, 3).reshape(*out.shape[:2], out.shape[3], -1)
        return self.to_out(out)


class Transformer(FusedEncoder, nn.Module):
    """Transformer block described in ViT.  A direct call on (b, p, n, d) bf16 CUDA tokens runs fused, one group of n
    tokens per (b, p) (b200vit_attention_groups with ph = pw = gw = 1)."""

    def __init__(self, dim, depth, heads, dim_head, mlp_dim, dropout=0.):
        super().__init__()
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, heads, dim_head, dropout),
                FeedForward(dim, mlp_dim, dropout)
            ]))
        self._dropout_p = float(dropout)

    def encoder_layers(self) -> Tuple[List[EncoderLayer], None]:
        layers = []
        for attn, ff in self.layers:
            f = ff.net
            layers.append(EncoderLayer(
                ln1=Norm.of(attn.norm), qkv_w=attn.to_qkv.weight, out_w=attn.to_out[0].weight,
                out_b=attn.to_out[0].bias, ln2=Norm.of(f[0]), fc1_w=f[1].weight, fc1_b=f[1].bias, fc2_w=f[4].weight,
                fc2_b=f[4].bias, heads=attn.heads, dim_head=attn.dim_head, scale=attn.scale, ff_act="silu",
                attention=PatchGroups()))
        return layers, None

    def fused_reason(self, x: torch.Tensor) -> Optional[str]:
        if x.dim() != 4:
            return "tokens are not (b, p, n, d)"
        r = common_reason(self, x, encoders=(self,), dropout_p=self._dropout_p, inside="transformer")
        if r is not None:
            return r
        if x.shape[-1] % 8:
            return f"dim={x.shape[-1]} (the GEMMs need multiples of 8)"
        return self.engine().unsupported_reason(x.shape[2], grid=(x.shape[2], 1), groups=(1, 1))

    def forward(self, x):
        if self.fused_reason(x) is None:
            b, p, n, d = x.shape
            out = self.engine().forward_tokens(x.reshape(b * p, n, d), grid=(n, 1), groups=(1, 1))
            return out.view(b, p, n, d)
        return self.forward_eager(x)

    def forward_eager(self, x):
        for attn, ff in self.layers:
            x = attn(x) + x
            x = ff(x) + x
        return x


class MV2Block(nn.Module):
    """MV2 block described in MobileNetV2."""

    def __init__(self, inp, oup, stride=1, expansion=4):
        super().__init__()
        self.stride = stride
        assert stride in [1, 2]

        hidden_dim = int(inp * expansion)
        self.use_res_connect = self.stride == 1 and inp == oup

        if expansion == 1:
            self.conv = nn.Sequential(
                # dw
                nn.Conv2d(hidden_dim, hidden_dim, 3, stride,
                          1, groups=hidden_dim, bias=False),
                nn.BatchNorm2d(hidden_dim),
                nn.SiLU(),
                # pw-linear
                nn.Conv2d(hidden_dim, oup, 1, 1, 0, bias=False),
                nn.BatchNorm2d(oup),
            )
        else:
            self.conv = nn.Sequential(
                # pw
                nn.Conv2d(inp, hidden_dim, 1, 1, 0, bias=False),
                nn.BatchNorm2d(hidden_dim),
                nn.SiLU(),
                # dw
                nn.Conv2d(hidden_dim, hidden_dim, 3, stride,
                          1, groups=hidden_dim, bias=False),
                nn.BatchNorm2d(hidden_dim),
                nn.SiLU(),
                # pw-linear
                nn.Conv2d(hidden_dim, oup, 1, 1, 0, bias=False),
                nn.BatchNorm2d(oup),
            )

    def forward(self, x):
        out = self.conv(x)
        if self.use_res_connect:
            out = out + x
        return out


def to_groups(x: torch.Tensor, ph: int, pw: int) -> torch.Tensor:
    """rearrange('b d (h ph) (w pw) -> b (ph pw) (h w) d') (reference mobile_vit.py:150), without einops; raises
    where einops does."""
    b, d, H, W = x.shape
    if H % ph or W % pw:
        raise RuntimeError(f"Rearrange: a {H} x {W} map is not divisible into {ph} x {pw} patches")
    h, w = H // ph, W // pw
    return x.reshape(b, d, h, ph, w, pw).permute(0, 3, 5, 2, 4, 1).reshape(b, ph * pw, h * w, d)


def from_groups(x: torch.Tensor, h: int, w: int, ph: int, pw: int) -> torch.Tensor:
    """rearrange('b (ph pw) (h w) d -> b d (h ph) (w pw)') (reference mobile_vit.py:152), without einops."""
    b, _, _, d = x.shape
    return x.reshape(b, ph, pw, h, w, d).permute(0, 5, 3, 1, 4, 2).reshape(b, d, h * ph, w * pw)


class MobileViTBlock(nn.Module):
    def __init__(self, dim, depth, channel, kernel_size, patch_size, mlp_dim, dropout=0.):
        super().__init__()
        self.ph, self.pw = patch_size

        self.conv1 = conv_nxn_bn(channel, channel, kernel_size)
        self.conv2 = conv_1x1_bn(channel, dim)

        self.transformer = Transformer(dim, depth, 4, 8, mlp_dim, dropout)

        self.conv3 = conv_1x1_bn(dim, channel)
        self.conv4 = conv_nxn_bn(2 * channel, channel, kernel_size)

    def forward(self, x):
        y = x.clone()

        # Local representations
        x = self.conv1(x)
        x = self.conv2(x)

        # Global representations
        _, _, h, w = x.shape
        x = to_groups(x, self.ph, self.pw)
        x = self.transformer(x)
        x = from_groups(x, h // self.ph, w // self.pw, self.ph, self.pw)

        # Fusion
        x = self.conv3(x)
        x = torch.cat((x, y), 1)
        x = self.conv4(x)
        return x


class _MeanHW(nn.Module):
    """Reduce('b c h w -> b c', 'mean') (reference mobile_vit.py:230), without einops."""

    def forward(self, x):
        if x.dim() != 4:
            raise RuntimeError(f"Reduce('b c h w -> b c'): expected 4 dims, got {x.dim()}")
        return x.mean(dim=(2, 3))


# -------------------------------------------------------------------------------------------------- prepared weights
def conv_bn_weights(conv: nn.Conv2d, bn: nn.BatchNorm2d, channels_last: bool = True
                    ) -> Tuple[torch.Tensor, torch.Tensor]:
    """(bf16 [out, K] GEMM weight, fp32 bias) of a bias-free Conv2d followed by BatchNorm2d (eval): the BatchNorm folded
    in fp32, then rounded; columns (cin, ky, kx) for the NCHW image (b200vit_conv_im2col_nchw), (ky, kx, cin) for a
    channels-last input (b200vit_conv_im2col_nhwc, or a 1 x 1 GEMM), K zero-padded to a multiple of 8."""
    w, b = fold_bn(conv.weight, conv.bias, bn)
    w = w.reshape(conv.weight.shape)
    if channels_last:
        w = w.permute(0, 2, 3, 1)
    w = w.reshape(w.shape[0], -1)
    return _bf16_rows(w.to(torch.bfloat16), (w.shape[1] + 7) // 8 * 8), b.contiguous()


def mv2_weights(blk: MV2Block) -> dict:
    """'w1' / 'b1' (the expansion 1 x 1 with its BatchNorm folded; absent when expansion == 1), 'w9' fp32 [9, hidden]
    tap-major / 'b9' (the depthwise 3 x 3 with its BatchNorm folded), 'w3' / 'b3' (the projection 1 x 1)."""
    c = blk.conv
    t = {}
    if len(c) == 8:
        t["w1"], t["b1"] = conv_bn_weights(c[0], c[1])
        dw, bn2, pw, bn3 = c[3], c[4], c[6], c[7]
    else:
        dw, bn2, pw, bn3 = c[0], c[1], c[3], c[4]
    w9, b9 = fold_bn(dw.weight, dw.bias, bn2)
    t["w9"], t["b9"] = w9.t().contiguous(), b9.contiguous()
    t["w3"], t["b3"] = conv_bn_weights(pw, bn3)
    return t


class MobileViT(FusedWeightsMixin, nn.Module):
    """MobileViT.
    Paper: https://arxiv.org/abs/2110.02178
    """

    def __init__(
        self,
        image_size,
        dims,
        channels,
        num_classes,
        expansion=4,
        kernel_size=3,
        patch_size=(2, 2),
        depths=(2, 4, 3)
    ):
        super().__init__()
        assert len(dims) == 3, 'dims must be a tuple of 3'
        assert len(depths) == 3, 'depths must be a tuple of 3'

        ih, iw = image_size
        ph, pw = patch_size
        assert ih % ph == 0 and iw % pw == 0

        init_dim, *_, last_dim = channels

        self.conv1 = conv_nxn_bn(3, init_dim, stride=2)

        self.stem = nn.ModuleList([])
        self.stem.append(MV2Block(channels[0], channels[1], 1, expansion))
        self.stem.append(MV2Block(channels[1], channels[2], 2, expansion))
        self.stem.append(MV2Block(channels[2], channels[3], 1, expansion))
        self.stem.append(MV2Block(channels[2], channels[3], 1, expansion))

        self.trunk = nn.ModuleList([])
        self.trunk.append(nn.ModuleList([
            MV2Block(channels[3], channels[4], 2, expansion),
            MobileViTBlock(dims[0], depths[0], channels[5],
                           kernel_size, patch_size, int(dims[0] * 2))
        ]))

        self.trunk.append(nn.ModuleList([
            MV2Block(channels[5], channels[6], 2, expansion),
            MobileViTBlock(dims[1], depths[1], channels[7],
                           kernel_size, patch_size, int(dims[1] * 4))
        ]))

        self.trunk.append(nn.ModuleList([
            MV2Block(channels[7], channels[8], 2, expansion),
            MobileViTBlock(dims[2], depths[2], channels[9],
                           kernel_size, patch_size, int(dims[2] * 4))
        ]))

        self.to_logits = nn.Sequential(
            conv_1x1_bn(channels[-2], last_dim),
            _MeanHW(),
            nn.Linear(channels[-1], num_classes, bias=False)
        )

        self.kernel_size = kernel_size
        self.patch_size = (ph, pw)

    # ---------------------------------------------------------------------------------------------- dispatch
    def block_maps(self, H: int, W: int) -> List[Tuple[int, int]]:
        """The (h, w) map of every MobileViTBlock for an H x W image: conv1 and stem.1 halve it (rounding up), every
        trunk MV2Block halves it again."""
        h, w = _lib.conv_out_size(H, 3, 2, 1), _lib.conv_out_size(W, 3, 2, 1)
        h, w = -(-h // 2), -(-w // 2)
        maps = []
        for _ in self.trunk:
            h, w = -(-h // 2), -(-w // 2)
            maps.append((h, w))
        return maps

    def _mv2s(self) -> List[MV2Block]:
        return list(self.stem) + [mv2 for mv2, _ in self.trunk]

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4 or img.shape[1] != 3:
            return "input is not (B, 3, H, W)"
        r = common_reason(self, img, encoders=[blk.transformer for _, blk in self.trunk])
        if r is not None:
            return r
        r = batchnorm_reason(self)
        if r is not None:
            return r
        if self.kernel_size != 3:
            return f"kernel_size={self.kernel_size} (padding 1 changes the map; the reference raises in torch.cat)"
        if self.stem[2].conv[-1].num_features != self.stem[3].conv[0].in_channels:
            return "channels[2] != channels[3] (stem.3 takes channels[2]; the reference raises)"
        for mv2 in self._mv2s():
            c = mv2.conv
            widths = (c[0].in_channels, c[0].out_channels, c[-1].num_features)
            if any(v % 8 for v in widths):
                return f"MV2Block widths {widths} (the GEMMs and the depthwise kernel need multiples of 8)"
        head = self.to_logits[0][0]
        if head.in_channels % 8 or head.out_channels % 8:
            return (f"to_logits widths {head.in_channels} -> {head.out_channels} (channels[-2] and channels[-1]; the "
                    f"GEMMs need multiples of 8)")
        ph, pw = self.patch_size
        for i, ((mv2, blk), (h, w)) in enumerate(zip(self.trunk, self.block_maps(img.shape[2], img.shape[3]))):
            C, D = blk.conv1[0].in_channels, blk.conv2[0].out_channels
            if mv2.conv[-1].num_features != C:
                return f"trunk {i}: the MV2Block writes {mv2.conv[-1].num_features} channels, the block takes {C}"
            if C % 8 or D % 8:
                return f"trunk {i}: channel={C}, dim={D} (the GEMMs need multiples of 8)"
            if h % ph or w % pw:
                return f"trunk {i}: the {h} x {w} map is not divisible into {ph} x {pw} patches (the reference raises)"
            r = blk.transformer.engine().unsupported_reason(h * w, grid=(h, w), groups=(ph, pw))
            if r is not None:
                return r
        return None

    def forward(self, x):
        if self.fused_reason(x) is None:
            with on_device(x):
                return self.forward_fused(x)
        return self.forward_eager(x)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, x):
        x = self.conv1(x)

        for conv in self.stem:
            x = conv(x)

        for conv, attn in self.trunk:
            x = conv(x)
            x = attn(x)

        return self.to_logits(x)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def prepared_buffers(self) -> List[torch.Tensor]:
        """Every BatchNorm's running statistics, which the folded weights are made of, and its batch counter (as
        levit.LeViT.prepared_buffers)."""
        return [b for m in self.modules() if isinstance(m, nn.BatchNorm2d)
                for b in (m.running_mean, m.running_var, m.num_batches_tracked) if b is not None]

    def prepared(self) -> dict:
        """The convolutions' prepared weights: 'conv1.*', 'stem<i>.*' / 'trunk<i>.*' (mv2_weights), 'block<i>.c1' ..
        '.c4' ('.w' / '.b') and 'head.*'."""
        params = [p for n, p in self.named_parameters() if ".transformer." not in n and not n.startswith("to_logits.2")]
        return cached(self, "_prepared", params + self.prepared_buffers(), self._build)

    def _build(self) -> dict:
        t = {}
        t["conv1.w"], t["conv1.b"] = conv_bn_weights(self.conv1[0], self.conv1[1], channels_last=False)
        for i, mv2 in enumerate(self.stem):
            t.update({f"stem{i}.{k}": v for k, v in mv2_weights(mv2).items()})
        for i, (mv2, blk) in enumerate(self.trunk):
            t.update({f"trunk{i}.{k}": v for k, v in mv2_weights(mv2).items()})
            for j, conv in enumerate((blk.conv1, blk.conv2, blk.conv3, blk.conv4), 1):
                t[f"block{i}.c{j}.w"], t[f"block{i}.c{j}.b"] = conv_bn_weights(conv[0], conv[1])
        t["head.w"], t["head.b"] = conv_bn_weights(self.to_logits[0][0], self.to_logits[0][1])
        return t

    def _mv2_fused(self, t: dict, p: str, mv2: MV2Block, xb: torch.Tensor, x32: Optional[torch.Tensor], B: int,
                   h: int, w: int, want_f32: bool, out_bf16: Optional[torch.Tensor] = None
                   ) -> Tuple[torch.Tensor, Optional[torch.Tensor], int, int]:
        """One MV2Block on the bf16 map xb (x32 its fp32 values, needed when use_res_connect) -> (bf16, fp32 or None,
        oh, ow).  `out_bf16` given, the bf16 output goes there: the right half of a MobileViTBlock's concatenation, a
        column slice that the block's conv1 and conv4 both read in place."""
        dev = xb.device
        bf = dict(device=dev, dtype=torch.bfloat16)
        s = mv2.stride
        if p + "w1" in t:
            hid = torch.empty(B * h * w, t[p + "w1"].shape[0], **bf)
            _lib.gemm_act(xb, t[p + "w1"], out_bf16=hid, bias=t[p + "b1"], act="silu")
        else:
            hid = xb
        oh, ow = -(-h // s), -(-w // s)
        hid2 = torch.empty(B * oh * ow, hid.shape[1], **bf)
        _lib.mbconv_dwconv_ex(hid, t[p + "w9"], t[p + "b9"], hid2, None, B, h, w, s, act="silu")
        C = t[p + "w3"].shape[0]
        yb = torch.empty(B * oh * ow, C, **bf) if out_bf16 is None else out_bf16
        if mv2.use_res_connect:
            # in place on the fp32 input: the residual GEMM reads each element before it writes it
            _lib.gemm(hid2, t[p + "w3"], out_bf16=yb, out_f32=x32, bias=t[p + "b3"], resid=x32)
            return yb, x32, oh, ow
        y32 = torch.empty(B * oh * ow, C, device=dev, dtype=torch.float32) if want_f32 else None
        _lib.gemm(hid2, t[p + "w3"], out_bf16=yb, out_f32=y32, bias=t[p + "b3"])
        return yb, y32, oh, ow

    def _block_fused(self, t: dict, p: str, blk: MobileViTBlock, cat: torch.Tensor, B: int, h: int, w: int
                     ) -> torch.Tensor:
        """One MobileViTBlock on the bf16 map in cat[:, C:] (cat [B*h*w, 2C]) -> its bf16 output [B*h*w, C]."""
        dev = cat.device
        bf = dict(device=dev, dtype=torch.bfloat16)
        M, C = cat.shape[0], cat.shape[1] // 2
        xb = cat[:, C:]
        # local representations: 3 x 3 (im2col + GEMM), 1 x 1 into the fp32 stream, both BatchNorm-folded with SiLU
        col = torch.empty(M, t[p + "c1.w"].shape[1], **bf)
        _lib.conv_im2col_nhwc(xb, col, B, h, w, 3, 1, 1)
        loc = torch.empty(M, C, **bf)
        _lib.gemm_act(col, t[p + "c1.w"], out_bf16=loc, bias=t[p + "c1.b"], act="silu")
        x = torch.empty(M, t[p + "c2.w"].shape[0], device=dev, dtype=torch.float32)
        _lib.gemm_act(loc, t[p + "c2.w"], out_f32=x, bias=t[p + "c2.b"], act="silu")
        # global representations: the transformer over the strided patch groups of the map
        eng = blk.transformer.engine()
        eng.run_blocks(x, B, h * w, grid=(h, w), groups=(blk.ph, blk.pw))
        # fusion: conv3 into the left half of the concatenation, conv4 over both halves
        _lib.gemm_act(eng.stream_bf16(x), t[p + "c3.w"], out_bf16=cat[:, :C], bias=t[p + "c3.b"], act="silu")
        col = torch.empty(M, t[p + "c4.w"].shape[1], **bf)
        _lib.conv_im2col_nhwc(cat, col, B, h, w, 3, 1, 1)
        out = torch.empty(M, C, **bf)
        _lib.gemm_act(col, t[p + "c4.w"], out_bf16=out, bias=t[p + "c4.b"], act="silu")
        return out

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        dev = img.device
        bf, f32 = dict(device=dev, dtype=torch.bfloat16), dict(device=dev, dtype=torch.float32)
        t = self.prepared()
        B, _, H, W = img.shape
        # conv1: im2col + GEMM (BatchNorm folded, SiLU); fp32 too when stem.0 adds its input
        h, w = _lib.conv_out_size(H, 3, 2, 1), _lib.conv_out_size(W, 3, 2, 1)
        a = torch.empty(B * h * w, t["conv1.w"].shape[1], **bf)
        _lib.conv_im2col_nchw(img.contiguous(), a, 3, 2, 1)
        xb = torch.empty(B * h * w, t["conv1.w"].shape[0], **bf)
        x32 = torch.empty(B * h * w, xb.shape[1], **f32) if self.stem[0].use_res_connect else None
        _lib.gemm_act(a, t["conv1.w"], out_bf16=xb, out_f32=x32, bias=t["conv1.b"], act="silu")
        nxt = list(self.stem)[1:] + [self.trunk[0][0]]
        for i, mv2 in enumerate(self.stem):
            xb, x32, h, w = self._mv2_fused(t, f"stem{i}.", mv2, xb, x32, B, h, w, nxt[i].use_res_connect)
        for i, (mv2, blk) in enumerate(self.trunk):
            C = t[f"block{i}.c1.w"].shape[0]
            oh, ow = -(-h // mv2.stride), -(-w // mv2.stride)
            cat = torch.empty(B * oh * ow, 2 * C, **bf)
            _, _, h, w = self._mv2_fused(t, f"trunk{i}.", mv2, xb, x32, B, h, w, False, out_bf16=cat[:, C:])
            x32 = None
            xb = self._block_fused(t, f"block{i}.", blk, cat, B, h, w)
        # to_logits: 1 x 1 GEMM (BatchNorm folded, SiLU) in fp32, the mean over the map, the classifier
        Cl = t["head.w"].shape[0]
        y = torch.empty(B * h * w, Cl, **f32)
        _lib.gemm_act(xb, t["head.w"], out_f32=y, bias=t["head.b"], act="silu")
        pm = torch.empty(B, Cl, **f32)
        _lib.mean_pool(y, pm, B, h * w, Cl)
        pooled = torch.empty(B, Cl, **bf)
        _lib.cast_f32_bf16(pm, pooled)
        return head_engine(self, self.to_logits[2]).run(pooled)
