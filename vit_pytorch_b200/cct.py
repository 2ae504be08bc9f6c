"""Drop-in `CCT` for lucidrains/vit-pytorch's `vit_pytorch.cct.CCT` (Compact Convolutional Transformer), with the presets
`cct_2` ... `cct_16`, `Tokenizer`, `TransformerClassifier`, `TransformerEncoderLayer`, `Attention`, `DropPath` and
`sinusoidal_embedding` of the same file, and a fused sm_90a forward.

Same constructor keywords (the `*args, **kwargs` passthrough to TransformerClassifier and the presets' defaults
included), parameter names / shapes / registration order (=> identical `state_dict` and identical random init under
the same seed): `tokenizer.conv_layers.i.0` the Conv2d of conv block i (no bias), `classifier.positional_emb` (1, n, D)
-- a fixed sin-cos table for 'sine', learnable for 'learnable', absent for 'none' --, `classifier.attention_pool`,
`classifier.blocks.i.{pre_norm, self_attn.qkv, self_attn.proj, linear1, norm1, linear2}`, `classifier.norm`,
`classifier.fc` (reference cct.py:75-353).  The PyTorch graph below mirrors the reference module for module, so hooks on
any submodule keep working there.

Fused forward:
  * per tokenizer block (cct.py:181-201): b200vit_conv_im2col_nchw (the image, columns (cin, ky, kx)) or
    b200vit_conv_im2col_nhwc (the previous block's channels-last output, columns (ky, kx, cin), the weight permuted to
    match), the convolution as one GEMM with a bf16 channels-last output, then b200vit_relu_maxpool -- into the next
    block's bf16 input, or after the last block into the fp32 tokens [B*n, D];
  * b200vit_embed_tokens without a cls row or LayerNorm: the positional table if there is one, and in fold mode the
    first layer's bf16 copy and row statistics (cct.py:276-277);
  * TransformerClassifier.engine().run_blocks: post-norm layers (EncoderLayer.post_norm, cct.py:137-142) in the
    per-kernel loop;
  * b200vit_seq_pool: the final LayerNorm, attention_pool, the softmax over each image's tokens and the weighted sum
    (cct.py:284-288), then the `fc` GEMM.
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib
from .engine import (EncoderLayer, FusedEncoder, FusedWeightsMixin, Norm, _bf16_rows, _f32, cached, common_reason,
                     head_engine, head_width_reason, on_device)

__all__ = ["Attention", "CCT", "DropPath", "Tokenizer", "TransformerClassifier", "TransformerEncoderLayer", "cct_2",
           "cct_4", "cct_6", "cct_7", "cct_8", "cct_14", "cct_16", "conv_weights", "sinusoidal_embedding"]

CONV_MAX_KERNEL = 16        # B200VIT_CONV_MAX_KERNEL
POOL_MAX_KERNEL = 16        # B200VIT_POOL_MAX_KERNEL
SEQ_POOL_MAX_DIM = 1024     # B200VIT_SEQ_POOL_MAX_DIM
MAX_TOKENS = 16384


def exists(val):
    return val is not None


def default(val, d):
    return val if exists(val) else d


def pair(t):
    return t if isinstance(t, tuple) else (t, t)


# ---------------------------------------------------------------------------------------------------------- presets
def _cct(num_layers, num_heads, mlp_ratio, embedding_dim, kernel_size=3, stride=None, padding=None, *args, **kwargs):
    """A CCT whose stride and padding default from the kernel size (cct.py:58-71)."""
    stride = default(stride, max(1, (kernel_size // 2) - 1))
    padding = default(padding, max(1, (kernel_size // 2)))
    return CCT(num_layers=num_layers, num_heads=num_heads, mlp_ratio=mlp_ratio, embedding_dim=embedding_dim,
               kernel_size=kernel_size, stride=stride, padding=padding, *args, **kwargs)


def cct_2(*args, **kwargs):
    return _cct(num_layers=2, num_heads=2, mlp_ratio=1, embedding_dim=128, *args, **kwargs)


def cct_4(*args, **kwargs):
    return _cct(num_layers=4, num_heads=2, mlp_ratio=1, embedding_dim=128, *args, **kwargs)


def cct_6(*args, **kwargs):
    return _cct(num_layers=6, num_heads=4, mlp_ratio=2, embedding_dim=256, *args, **kwargs)


def cct_7(*args, **kwargs):
    return _cct(num_layers=7, num_heads=4, mlp_ratio=2, embedding_dim=256, *args, **kwargs)


def cct_8(*args, **kwargs):
    return _cct(num_layers=8, num_heads=4, mlp_ratio=2, embedding_dim=256, *args, **kwargs)


def cct_14(*args, **kwargs):
    return _cct(num_layers=14, num_heads=6, mlp_ratio=3, embedding_dim=384, *args, **kwargs)


def cct_16(*args, **kwargs):
    return _cct(num_layers=16, num_heads=6, mlp_ratio=3, embedding_dim=384, *args, **kwargs)


# ---------------------------------------------------------------------------------------------------------- modules
def sinusoidal_embedding(n_channels, dim):
    """(1, n_channels, dim) fixed table: position t, channel i -> t / 10000^(2 (i // 2) / dim), sine on the even
    channels and cosine on the odd ones (cct.py:75-80).  The angles are formed in Python floats and rounded to fp32
    once, then sin / cos run in fp32, so the table has the reference's bits."""
    freq = [10000 ** (2 * (i // 2) / dim) for i in range(dim)]
    pe = torch.tensor([[t / f for f in freq] for t in range(n_channels)], dtype=torch.float32)
    pe[:, 0::2] = torch.sin(pe[:, 0::2])
    pe[:, 1::2] = torch.cos(pe[:, 1::2])
    return pe.unsqueeze(0)


class Attention(nn.Module):
    """Multi-head self-attention, qkv without bias, proj with bias, heads dim // num_heads wide (cct.py:84-111)."""

    def __init__(self, dim, num_heads=8, attention_dropout=0.1, projection_dropout=0.1):
        super().__init__()
        self.heads = num_heads
        head_dim = dim // self.heads
        self.scale = head_dim ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=False)
        self.attn_drop = nn.Dropout(attention_dropout)
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(projection_dropout)

    def forward(self, x):
        b, n, _ = x.shape
        h = self.heads
        q, k, v = self.qkv(x).chunk(3, dim=-1)
        if q.shape[-1] % h:
            # what einops raises for 'b n (h d) -> b h n d' with h not dividing the width
            raise RuntimeError(f"Attention: {q.shape[-1]} channels cannot be split into {h} heads (cct.py:100)")
        q, k, v = (t.reshape(b, n, h, -1).transpose(1, 2) for t in (q, k, v))
        attn = torch.einsum('b h i d, b h j d -> b h i j', q * self.scale, k).softmax(dim=-1)
        attn = self.attn_drop(attn)
        out = torch.einsum('b h i j, b h j d -> b h i d', attn, v).transpose(1, 2).reshape(b, n, -1)
        return self.proj_drop(self.proj(out))


class DropPath(nn.Module):
    """Stochastic depth: in training, each sample's branch is zeroed with probability drop_prob and the survivors are
    scaled by 1 / (1 - drop_prob) (cct.py:144-160)."""

    def __init__(self, drop_prob=None):
        super().__init__()
        self.drop_prob = float(drop_prob)

    def forward(self, x):
        if self.drop_prob <= 0. or not self.training:
            return x
        keep = 1 - self.drop_prob
        mask = torch.zeros((x.shape[0],) + (1,) * (x.ndim - 1), device=x.device).float().uniform_(0, 1) < keep
        return x.div(keep) * mask.float()


class TransformerEncoderLayer(nn.Module):
    """x += proj(attn(pre_norm(x)));  x = norm1(x);  x += linear2(GELU(linear1(x)))  (cct.py:114-142)."""

    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, attention_dropout=0.1, drop_path_rate=0.1):
        super().__init__()
        self.pre_norm = nn.LayerNorm(d_model)
        self.self_attn = Attention(dim=d_model, num_heads=nhead, attention_dropout=attention_dropout,
                                   projection_dropout=dropout)
        self.linear1 = nn.Linear(d_model, dim_feedforward)
        self.dropout1 = nn.Dropout(dropout)
        self.norm1 = nn.LayerNorm(d_model)
        self.linear2 = nn.Linear(dim_feedforward, d_model)
        self.dropout2 = nn.Dropout(dropout)
        self.drop_path = DropPath(drop_path_rate)
        self.activation = F.gelu

    def forward(self, src, *args, **kwargs):
        src = src + self.drop_path(self.self_attn(self.pre_norm(src)))
        src = self.norm1(src)
        src2 = self.linear2(self.dropout1(self.activation(self.linear1(src))))
        return src + self.drop_path(self.dropout2(src2))


class Tokenizer(nn.Module):
    """n_conv_layers x (Conv2d(k, s, p), activation, MaxPool2d(pk, ps, pp)), channels n_input_channels -> in_planes ...
    -> n_output_channels, then 'b c h w -> b (h w) c' (cct.py:162-201)."""

    def __init__(self, kernel_size, stride, padding, pooling_kernel_size=3, pooling_stride=2, pooling_padding=1,
                 n_conv_layers=1, n_input_channels=3, n_output_channels=64, in_planes=64, activation=None,
                 max_pool=True, conv_bias=False):
        super().__init__()
        chans = [n_input_channels] + [in_planes] * (n_conv_layers - 1) + [n_output_channels]
        self.conv_layers = nn.Sequential(*[
            nn.Sequential(
                nn.Conv2d(cin, cout, kernel_size=(kernel_size, kernel_size), stride=(stride, stride),
                          padding=(padding, padding), bias=conv_bias),
                nn.Identity() if not exists(activation) else activation(),
                nn.MaxPool2d(kernel_size=pooling_kernel_size, stride=pooling_stride, padding=pooling_padding)
                if max_pool else nn.Identity(),
            )
            for cin, cout in zip(chans[:-1], chans[1:])
        ])
        self.apply(self.init_weight)

    def sequence_length(self, n_channels=3, height=224, width=224):
        return self.forward(torch.zeros((1, n_channels, height, width))).shape[1]

    def forward(self, x):
        return self.conv_layers(x).flatten(2).transpose(1, 2)

    @staticmethod
    def init_weight(m):
        if isinstance(m, nn.Conv2d):
            nn.init.kaiming_normal_(m.weight)


class TransformerClassifier(FusedEncoder, nn.Module):
    """Positional table, post-norm encoder layers, final LayerNorm, sequence pooling (or a cls token) and `fc`
    (cct.py:209-292).  Describes its blocks to the engine as EncoderLayers with post_norm=True."""

    def __init__(self, seq_pool=True, embedding_dim=768, num_layers=12, num_heads=12, mlp_ratio=4.0, num_classes=1000,
                 dropout_rate=0.1, attention_dropout=0.1, stochastic_depth_rate=0.1, positional_embedding='sine',
                 sequence_length=None, *args, **kwargs):
        super().__init__()
        assert positional_embedding in {'sine', 'learnable', 'none'}
        dim_feedforward = int(embedding_dim * mlp_ratio)
        self.embedding_dim = embedding_dim
        self.sequence_length = sequence_length
        self.seq_pool = seq_pool
        assert exists(sequence_length) or positional_embedding == 'none', \
            f"Positional embedding is set to {positional_embedding} and the sequence length was not specified."
        if not seq_pool:
            sequence_length += 1
            self.class_emb = nn.Parameter(torch.zeros(1, 1, self.embedding_dim), requires_grad=True)
        else:
            self.attention_pool = nn.Linear(self.embedding_dim, 1)
        if positional_embedding == 'none':
            self.positional_emb = None
        elif positional_embedding == 'learnable':
            self.positional_emb = nn.Parameter(torch.zeros(1, sequence_length, embedding_dim), requires_grad=True)
            nn.init.trunc_normal_(self.positional_emb, std=0.2)
        else:
            self.positional_emb = nn.Parameter(sinusoidal_embedding(sequence_length, embedding_dim),
                                               requires_grad=False)
        self.dropout = nn.Dropout(p=dropout_rate)
        rates = [r.item() for r in torch.linspace(0, stochastic_depth_rate, num_layers)]
        self.blocks = nn.ModuleList([
            TransformerEncoderLayer(d_model=embedding_dim, nhead=num_heads, dim_feedforward=dim_feedforward,
                                    dropout=dropout_rate, attention_dropout=attention_dropout, drop_path_rate=r)
            for r in rates])
        self.norm = nn.LayerNorm(embedding_dim)
        self.fc = nn.Linear(embedding_dim, num_classes)
        self.apply(self.init_weight)
        self.dropout_p = max(float(dropout_rate), float(attention_dropout), float(stochastic_depth_rate))

    def forward(self, x):
        b = x.shape[0]
        if not exists(self.positional_emb) and x.size(1) < self.sequence_length:
            # the reference pads to `self.n_channels`, an attribute it never sets: the call raises AttributeError
            x = F.pad(x, (0, 0, 0, self.n_channels - x.size(1)), mode='constant', value=0)
        if not self.seq_pool:
            x = torch.cat((self.class_emb.expand(b, -1, -1), x), dim=1)
        if exists(self.positional_emb):
            x += self.positional_emb
        x = self.dropout(x)
        for blk in self.blocks:
            x = blk(x)
        x = self.norm(x)
        if self.seq_pool:
            weights = self.attention_pool(x).squeeze(-1).softmax(dim=1)
            x = torch.einsum('b n, b n d -> b d', weights, x)
        else:
            x = x[:, 0]
        return self.fc(x)

    @staticmethod
    def init_weight(m):
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=.02)
            if isinstance(m, nn.Linear) and exists(m.bias):
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def encoder_layers(self) -> Tuple[List[EncoderLayer], Optional[Norm]]:
        layers = []
        for blk in self.blocks:
            attn = blk.self_attn
            D = attn.qkv.in_features
            layers.append(EncoderLayer(
                ln1=Norm.of(blk.pre_norm), qkv_w=attn.qkv.weight, out_w=attn.proj.weight, out_b=attn.proj.bias,
                ln2=Norm.of(blk.norm1), fc1_w=blk.linear1.weight, fc1_b=blk.linear1.bias, fc2_w=blk.linear2.weight,
                fc2_b=blk.linear2.bias, heads=attn.heads, dim_head=D // attn.heads, scale=float(attn.scale),
                post_norm=True))
        return layers, Norm.of(self.norm)


def conv_weights(conv: nn.Conv2d, channels_last_input: bool) -> torch.Tensor:
    """The convolution's GEMM weight, bf16 [Cout, K] with K padded to a multiple of 8 by zeros: columns (cin, ky, kx)
    -- the weight's own layout, b200vit_conv_im2col_nchw's order -- or, for a channels-last input, (ky, kx, cin) as
    b200vit_conv_im2col_nhwc writes them."""
    w = conv.weight.detach()
    if channels_last_input:
        w = w.permute(0, 2, 3, 1)
    w = w.reshape(w.shape[0], -1)
    return _bf16_rows(w, (w.shape[1] + 7) // 8 * 8)


class CCT(FusedWeightsMixin, nn.Module):
    def __init__(self, img_size=224, embedding_dim=768, n_input_channels=3, n_conv_layers=1, kernel_size=7, stride=2,
                 padding=3, pooling_kernel_size=3, pooling_stride=2, pooling_padding=1, dropout_rate=0.,
                 attention_dropout=0.1, stochastic_depth_rate=0.1, *args, **kwargs):
        super().__init__()
        img_height, img_width = pair(img_size)
        self.tokenizer = Tokenizer(n_input_channels=n_input_channels, n_output_channels=embedding_dim,
                                   kernel_size=kernel_size, stride=stride, padding=padding,
                                   pooling_kernel_size=pooling_kernel_size, pooling_stride=pooling_stride,
                                   pooling_padding=pooling_padding, max_pool=True, activation=nn.ReLU,
                                   n_conv_layers=n_conv_layers, conv_bias=False)
        self.classifier = TransformerClassifier(
            sequence_length=self.tokenizer.sequence_length(n_channels=n_input_channels, height=img_height,
                                                           width=img_width),
            embedding_dim=embedding_dim, seq_pool=True, dropout_rate=dropout_rate,
            attention_dropout=attention_dropout, stochastic_depth_rate=stochastic_depth_rate, *args, **kwargs)

    # ---------------------------------------------------------------------------------------------- dispatch
    def token_grid(self, H: int, W: int) -> Optional[List[Tuple[int, int, int, int]]]:
        """Per conv block, (conv output h, w, pool output h, w) for an H x W image; None where a block has no output
        (the reference's Conv2d or MaxPool2d raises)."""
        out = []
        for blk in self.tokenizer.conv_layers:
            conv, pool = blk[0], blk[2]
            (k, _), (s, _), (p, _) = conv.kernel_size, conv.stride, conv.padding
            H, W = _lib.conv_out_size(H, k, s, p), _lib.conv_out_size(W, k, s, p)
            if H < 1 or W < 1:
                return None
            pk, ps, pp = (pool.kernel_size, pool.stride, pool.padding)
            if H + 2 * pp < pk or W + 2 * pp < pk:
                return None
            out.append((H, W, _lib.conv_out_size(H, pk, ps, pp), _lib.conv_out_size(W, pk, ps, pp)))
            H, W = out[-1][2], out[-1][3]
        return out

    def _kernel_reason(self) -> Optional[str]:
        """The conv, pool and pooling-width limits of the tokenizer and sequence-pooling kernels."""
        for i, blk in enumerate(self.tokenizer.conv_layers):
            conv, act, pool = blk
            if not isinstance(act, nn.ReLU) or not isinstance(pool, nn.MaxPool2d):
                return f"conv block {i} is not Conv2d, ReLU, MaxPool2d"
            ks, st, pd = conv.kernel_size, conv.stride, conv.padding
            if (conv.bias is not None or conv.groups != 1 or conv.dilation != (1, 1) or ks[0] != ks[1]
                    or st[0] != st[1] or not isinstance(pd, tuple) or pd[0] != pd[1] or conv.padding_mode != "zeros"):
                return f"conv block {i}: a convolution the tokenizer kernels are not built for"
            k, s, p = ks[0], st[0], pd[0]
            if not (1 <= k <= CONV_MAX_KERNEL and 0 <= p < k):
                return f"conv block {i}: kernel {k}, padding {p} (the im2col kernels take 1 <= k <= " \
                       f"{CONV_MAX_KERNEL} and padding < k)"
            if i > 0 and conv.in_channels % 8:
                return f"conv block {i}: {conv.in_channels} input channels, not a multiple of 8"
            if conv.out_channels % 8:
                return f"conv block {i}: {conv.out_channels} output channels, not a multiple of 8"
            pk, ps, pp = pool.kernel_size, pool.stride, pool.padding
            if (not all(isinstance(v, int) for v in (pk, ps, pp)) or pool.dilation != 1 or pool.ceil_mode
                    or not 1 <= pk <= POOL_MAX_KERNEL or ps < 1 or pp > pk // 2):
                return f"conv block {i}: a MaxPool2d the pooling kernel is not built for"
        D = self.classifier.embedding_dim
        if D > SEQ_POOL_MAX_DIM:
            return f"embedding_dim={D} (the sequence-pooling kernel takes at most {SEQ_POOL_MAX_DIM})"
        return None

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4:
            return "input is not (B, C, H, W)"
        if img.shape[1] != self.tokenizer.conv_layers[0][0].in_channels:
            return "channel count differs from the constructor's (the reference's Conv2d raises)"
        cl = self.classifier
        if len(cl.blocks) == 0:
            return "num_layers == 0"
        if not cl.seq_pool:
            return "seq_pool=False (a cls token)"
        r = common_reason(self, img, dropout_p=cl.dropout_p)
        if r is not None:
            return r
        attn = cl.blocks[0].self_attn
        D = cl.embedding_dim
        if D % attn.heads:
            return f"embedding_dim={D} not divisible by num_heads={attn.heads} (the reference's rearrange raises)"
        r = head_width_reason(D // attn.heads) or self._kernel_reason()
        if r is not None:
            return r
        grid = self.token_grid(img.shape[2], img.shape[3])
        if grid is None:
            return "a conv block has no output for this image (the reference raises)"
        n = grid[-1][2] * grid[-1][3]
        L = cl.sequence_length
        if exists(cl.positional_emb) and n != L:
            return f"{n} tokens against a positional table of {L} (the reference's add raises)"
        if not exists(cl.positional_emb) and n < L:
            return f"{n} tokens, fewer than sequence_length={L} (the reference's padding raises)"
        return cl.engine().unsupported_reason(n)

    def forward(self, x):
        if self.fused_reason(x) is None:
            with on_device(x):
                return self.forward_fused(x)
        return self.forward_eager(x)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, x):
        x = self.tokenizer(x)
        return self.classifier(x)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def _conv_weights(self, i: int, conv: nn.Conv2d) -> torch.Tensor:
        return cached(self, f"_conv{i}", [conv.weight], lambda: conv_weights(conv, i > 0))

    def _pool_weights(self) -> dict:
        cl = self.classifier
        params = [cl.norm.weight, cl.norm.bias, cl.attention_pool.weight, cl.attention_pool.bias]
        if exists(cl.positional_emb):
            params.append(cl.positional_emb)

        def build():
            D = cl.embedding_dim
            pos = cl.positional_emb
            return {"norm.w": _f32(cl.norm.weight), "norm.b": _f32(cl.norm.bias),
                    "pool.w": _f32(cl.attention_pool.weight).reshape(D), "pool.b": _f32(cl.attention_pool.bias),
                    "pos": None if pos is None else pos.detach().float().reshape(-1, D).contiguous()}
        return cached(self, "_seq_pool", params, build)

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        dev, bf = img.device, dict(device=img.device, dtype=torch.bfloat16)
        B, _, H, W = img.shape
        cl = self.classifier
        D = cl.embedding_dim
        blocks = list(self.tokenizer.conv_layers)
        src = img.contiguous()
        y = None
        for i, ((oh, ow, ph, pw), blk) in enumerate(zip(self.token_grid(H, W), blocks)):
            conv, pool = blk[0], blk[2]
            k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
            w = self._conv_weights(i, conv)
            a = torch.empty(B * oh * ow, w.shape[1], **bf)
            if i == 0:
                _lib.conv_im2col_nchw(src, a, k, s, p)
            else:
                _lib.conv_im2col_nhwc(src, a, B, H, W, k, s, p)
            c = torch.empty(B * oh * ow, conv.out_channels, **bf)
            _lib.gemm(a, w, out_bf16=c)
            if i + 1 < len(blocks):
                src = torch.empty(B * ph * pw, conv.out_channels, **bf)
                _lib.relu_maxpool(c, B, oh, ow, pool.kernel_size, pool.stride, pool.padding, out_bf16=src)
            else:
                y = torch.empty(B * ph * pw, D, device=dev, dtype=torch.float32)
                _lib.relu_maxpool(c, B, oh, ow, pool.kernel_size, pool.stride, pool.padding, out_f32=y)
            H, W = ph, pw
        n = H * W
        t = self._pool_weights()
        eng = cl.engine()
        xb, stats = eng.entry_buffers(B * n, dev)
        x = torch.empty(B * n, D, device=dev, dtype=torch.float32)
        _lib.embed_tokens(y, None, None, None, t["pos"], x, B, n, 0, xb=xb, stats=stats)
        eng.run_blocks(x, B, n, primed=xb is not None)
        pooled = torch.empty(B, D, **bf)
        _lib.seq_pool(x, B, n, t["norm.w"], t["norm.b"], t["pool.w"], t["pool.b"], pooled, eps=cl.norm.eps)
        return head_engine(self, cl.fc).run(pooled)
