"""Stock-PyTorch multi-scale ViT harness around the fused attention operator.

Per the north star the MsViT block structure, patch embedding, LayerNorm, MLP and
the dense attention of the low-resolution stages stay ordinary PyTorch; only the
stages whose arch field is `s1` use the B200 attention module.  This file is the
host-side mirror of `MsViT` (src/models/msvit.py:343-547) needed to run the
BASELINE configs (ViL-Tiny/Small/Medium-Deep/Base-Deep) end to end on a box where
the reference tree does not exist; module / parameter names follow the reference
so its checkpoints load unchanged (pinned by tests/test_msvit_harness.py against
golden vectors generated from the reference).

With dense_impl="vil" and the longformer stages on the fused operator, the attention backward is deterministic, rpe
on or off (include/vil_attn.h), so a training step repeats bit for bit under torch.use_deterministic_algorithms(True).

Arch string grammar (msvit.py:402-410): stages separated by `_`, fields by `,`:
  l<stage id> h<heads> d<dim> n<blocks> s<1: longformer attention, 0: dense>
  g<global tokens> p<patch size> f<window w> a<1: absolute pos-embed, 0: relative bias>
"""
from __future__ import annotations

from functools import partial
from typing import Callable, Optional

import torch
import torch.nn.functional as F
from torch import nn

from .attention import B200Long2DSCSelfAttention
from . import epilogue
from .layernorm import B200LayerNorm

ARCHS = {   # README.md:210-239 of the reference
    "vil_tiny": "l1,h1,d48,n1,s1,g1,p4,f7_l2,h3,d96,n1,s1,g1,p2,f7_l3,h3,d192,n9,s0,g1,p2,f7_l4,h6,d384,n1,s0,g0,p2,f7",
    "vil_small": "l1,h3,d96,n1,s1,g1,p4,f7_l2,h3,d192,n2,s1,g1,p2,f7_l3,h6,d384,n8,s0,g1,p2,f7_l4,h12,d768,n1,s0,g0,p2,f7",
    "vil_medium_deep": "l1,h3,d96,n1,s1,g1,p4,f7_l2,h3,d192,n4,s1,g1,p2,f7_l3,h6,d384,n16,s0,g1,p2,f7_l4,h12,d768,n1,s0,g0,p2,f7",
    # README.md:300 of the reference: the 384x384 fine-tuning variant (w = 8 on 96x96 tokens, w = 12 on 48x48)
    "vil_medium_deep_384": "l1,h3,d96,n1,s1,g1,p4,f8_l2,h3,d192,n4,s1,g1,p2,f12_l3,h6,d384,n16,s0,g1,p2,f7_l4,h12,d768,n1,s0,g0,p2,f7",
    "vil_medium_wide": "l1,h3,d192,n1,s1,g1,p4,f7_l2,h6,d384,n2,s1,g1,p2,f7_l3,h8,d512,n8,s0,g1,p2,f7_l4,h12,d768,n1,s0,g0,p2,f7",
    "vil_medium_wide_384": "l1,h3,d192,n1,s1,g1,p4,f8_l2,h6,d384,n2,s1,g1,p2,f12_l3,h8,d512,n8,s0,g1,p2,f7_l4,h12,d768,n1,s0,g0,p2,f7",
    "vil_base_deep": "l1,h3,d96,n1,s1,g1,p4,f6_l2,h3,d192,n8,s1,g1,p2,f8_l3,h6,d384,n24,s0,g1,p2,f7_l4,h12,d768,n1,s0,g0,p2,f7",
    "vil_base_wide": "l1,h3,d192,n1,s1,g1,p4,f8_l2,h6,d384,n2,s1,g1,p2,f8_l3,h12,d768,n8,s0,g1,p2,f7_l4,h16,d1024,n1,s0,g0,p2,f7",
}

_STAGE_DEFAULTS = dict(l=1, h=3, d=192, n=1, s=1, g=1, p=2, f=7, a=1)


def parse_arch(arch: str):
    stages = []
    for spec in arch.split("_"):
        cfg = dict(_STAGE_DEFAULTS)
        for field in spec.split(","):
            cfg[field[0]] = int(field[1:])
        stages.append(cfg)
    return stages


class DropPath(nn.Module):
    """Stochastic depth per sample."""

    def __init__(self, p: float = 0.):
        super().__init__()
        self.drop_prob = p

    def forward(self, x):
        scale = self.sample_scale(x.shape[0], x.device)
        if scale is None:
            return x
        return x * scale.view((x.shape[0],) + (1,) * (x.dim() - 1)).to(x.dtype)

    def sample_scale(self, batch, device):
        """The same per-sample factor (0 or 1 / keep) as a (B,) fp32 vector, or None when DropPath is the identity: consumed
        by the fused residual-add kernel (epilogue.add_norm) instead of a multiply pass over the branch."""
        if self.drop_prob == 0. or not self.training:
            return None
        keep = 1.0 - self.drop_prob
        return torch.empty(batch, dtype=torch.float32, device=device).bernoulli_(keep).div_(keep)


class Mlp(nn.Module):
    def __init__(self, in_features, hidden_features, out_features=None, drop=0.):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = nn.GELU()
        self.fc2 = nn.Linear(hidden_features, out_features or in_features)
        self.drop = nn.Dropout(drop)

    def forward(self, x):
        return self.drop(self.fc2(self.drop(self.act(self.fc1(x)))))

    def forward_deferred(self, x):
        """(fc2 output WITHOUT its bias, fc2.bias): the caller's residual-add kernel applies the bias (and its backward yields
        the bias gradient); fc1's bias is applied together with the GELU (one pass forward, one backward incl. d_bias)."""
        if (self.training and self.drop.p > 0) or not epilogue.bias_act_applies(x) or self.fc1.bias is None or self.fc2.bias is None:
            return self.forward(x), None
        z = F.linear(x, self.fc1.weight)
        if not epilogue.bias_act_applies(z):
            return self.forward(x), None
        return F.linear(epilogue.bias_gelu(z, self.fc1.bias), self.fc2.weight), self.fc2.bias


class _SplitQKV(torch.autograd.Function):
    """(B, N, 3·H·D) -> q, k, v as (B, H, N, D) views.  The backward assembles the packed gradient with ONE strided
    copy; stock `unbind` + `permute` autograd does a `stack` and then a second layout copy (≈ 2.4 ms of the ViL-Small
    step)."""

    @staticmethod
    def forward(ctx, qkv, num_heads):
        B, N, C3 = qkv.shape
        t = qkv.view(B, N, 3, num_heads, C3 // (3 * num_heads))
        ctx.shape = (B, N, C3)
        return t[:, :, 0].transpose(1, 2), t[:, :, 1].transpose(1, 2), t[:, :, 2].transpose(1, 2)

    @staticmethod
    def backward(ctx, dq, dk, dv):
        g = torch.stack((dq.transpose(1, 2), dk.transpose(1, 2), dv.transpose(1, 2)), dim=2)     # (B, N, 3, H, D)
        return g.view(ctx.shape), None


class DenseAttention(nn.Module):
    """Full multi-head attention of the `s0` stages with optional Swin-style relative bias and global-token biases
    (reference `Attention`, msvit.py:37-120).

    impl = "vil"  : the vil_attn sm_90a kernels - dense attention over nglo + w*w tokens is the SINGLE-CHUNK case of the
                    sliding-chunk operator (nx = ny = w, every local query sees every local key, global tokens as usual),
                    so the same tensor-core kernels serve it when w in {7, 14} (7x7 and 14x14 stages of the 224 nets),
                    head dim <= 128 (a multiple of 8), bf16/fp16 on CUDA; no (H,N,N) bias tensor is materialised: the Swin-style
                    (2wx-1)(2wy-1) table is embedded in the operator's (4w-1)^2 index space (same Delta-row / Delta-col).
    impl = "sdpa" : stock F.scaled_dot_product_attention (cuDNN) with the bias as attn_mask.
    impl = "auto" : "sdpa": at 50..197 tokens the chunk-tiled kernels (64-row tiles, one global-token side kernel, two
                    backward passes) are not expected to beat a dedicated dense flash kernel (tools/time_dense.py times both),
                    so the library path stays the default and "vil" is opt-in (parity-tested in
                    tests/test_gpu_parity.py::test_dense_attention_on_the_operator_kernels)."""

    supports_deferred_bias = True       # forward(..., defer_proj_bias=True) -> (projection without bias, bias)

    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_scale=None, attn_drop=0., proj_drop=0.,
                 rpe=False, wx=14, wy=14, nglo=1, impl="auto"):
        super().__init__()
        self.impl = impl
        self.wx, self.wy, self.nglo = wx, wy, nglo
        self.num_heads = num_heads
        self.scale = qk_scale or (dim // num_heads) ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.attn_drop = nn.Dropout(attn_drop)
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(proj_drop)
        self.rpe = rpe
        if rpe:
            self.local_relative_position_bias_table = nn.Parameter(torch.zeros((2 * wx - 1) * (2 * wy - 1), num_heads))
            nn.init.trunc_normal_(self.local_relative_position_bias_table, std=.02)
            if nglo >= 1:
                self.g2l_relative_position_bias = nn.Parameter(torch.zeros(2, num_heads, nglo))
                self.g2g_relative_position_bias = nn.Parameter(torch.zeros(num_heads, nglo, nglo))
                nn.init.trunc_normal_(self.g2l_relative_position_bias, std=.02)
                nn.init.trunc_normal_(self.g2g_relative_position_bias, std=.02)
            ys, xs = torch.meshgrid(torch.arange(wx), torch.arange(wy), indexing="ij")
            pos = torch.stack([ys.flatten(), xs.flatten()])                      # (2, wx*wy)
            rel = pos[:, :, None] - pos[:, None, :]
            idx = (rel[0] + wx - 1) * (2 * wy - 1) + (rel[1] + wy - 1)
            self.register_buffer("relative_position_index", idx)

    def _bias(self, N):
        n = self.wx * self.wy
        assert N == self.nglo + n, "For relative position, N != self.nglo + self.wx*self.wy!"
        H = self.num_heads
        loc = self.local_relative_position_bias_table[self.relative_position_index.reshape(-1)]
        loc = loc.view(n, n, H).permute(2, 0, 1)
        if self.nglo == 0:
            return loc
        top = torch.cat([self.g2g_relative_position_bias,
                         self.g2l_relative_position_bias[0].unsqueeze(-1).expand(-1, -1, n)], dim=-1)
        bot = torch.cat([self.g2l_relative_position_bias[1].unsqueeze(1).expand(-1, n, -1), loc], dim=-1)
        return torch.cat([top, bot], dim=1)                                       # (H, N, N)

    def _vil_applies(self, x):
        w = self.wx
        return (self.impl == "vil" and x.is_cuda and self.wx == self.wy and w in (7, 14)
                and x.shape[1] == self.nglo + w * w and (x.shape[2] // self.num_heads) <= 128
                and (x.shape[2] // self.num_heads) % 8 == 0 and self.nglo <= 8
                and (torch.is_autocast_enabled("cuda") or x.dtype in (torch.bfloat16, torch.float16)))

    def _vil_table(self):
        """(2w-1)^2 Swin table -> the operator's (4w-1)^2 layout (index (dr + 2w-1)(4w-1) + dc + 2w-1); differentiable."""
        w = self.wx
        d = torch.arange(-(w - 1), w, device=self.local_relative_position_bias_table.device)
        idx = ((d[:, None] + 2 * w - 1) * (4 * w - 1) + (d[None, :] + 2 * w - 1)).reshape(-1)
        big = self.local_relative_position_bias_table.new_zeros((4 * w - 1) ** 2, self.num_heads)
        return big.index_put((idx,), self.local_relative_position_bias_table)

    def forward(self, x, nx=None, ny=None, defer_proj_bias: bool = False):
        if defer_proj_bias:
            if (self.training and self.proj_drop.p > 0) or self.proj.bias is None:
                return self.forward(x, nx, ny), None
            proj = lambda t: (F.linear(t, self.proj.weight), self.proj.bias)
        else:
            proj = lambda t: self.proj_drop(self.proj(t))
        B, N, C = x.shape
        if self._vil_applies(x):
            from .ops import vil_dense_attention
            table = g2l = g2g = None
            if self.rpe:
                table = self._vil_table()
                if self.nglo >= 1:
                    g2l, g2g = self.g2l_relative_position_bias, self.g2g_relative_position_bias
            drop = self.attn_drop.p if self.training else 0.0
            if drop >= 1.0:         # nn.Dropout(1): the attention output is exactly 0
                return proj(x.new_zeros(B, N, C))
            out = vil_dense_attention(self.qkv(x), table, g2l, g2g, num_heads=self.num_heads, nx=self.wx, ny=self.wy,
                                      nglo=self.nglo, scale=self.scale, dropout_p=drop)
            return proj(out)
        if self.impl == "vil":
            raise NotImplementedError("DenseAttention(impl='vil') needs a 7x7 or 14x14 token grid, head dim <= 128 and bf16/fp16 on CUDA")
        q, k, v = _SplitQKV.apply(epilogue.linear_colsum_bias(x, self.qkv.weight, self.qkv.bias), self.num_heads)
        mask = self._bias(N).unsqueeze(0).to(q.dtype) if self.rpe else None
        out = F.scaled_dot_product_attention(q, k, v, attn_mask=mask,
                                             dropout_p=self.attn_drop.p if self.training else 0., scale=self.scale)
        return proj(out.transpose(1, 2).reshape(B, N, C))


class PatchEmbed(nn.Module):
    """Conv patchify (+LN) + global (cls) tokens + separable absolute position embedding (msvit.py:159-224)."""

    def __init__(self, patch_size, nx, ny, in_chans=3, embed_dim=768, nglo=1, norm_layer=nn.LayerNorm,
                 norm_embed=True, drop_rate=0.0, ape=True):
        super().__init__()
        self.patch_size = (patch_size, patch_size)
        self.channels_last = True       # CUDA only; CPU keeps the reference's NCHW path bit for bit
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)
        self.norm_embed = norm_layer(embed_dim) if norm_embed else None
        self.nx, self.ny, self.Nglo, self.ape = nx, ny, nglo, ape
        if nglo >= 1:
            self.cls_token = nn.Parameter(torch.zeros(1, nglo, embed_dim))
            nn.init.trunc_normal_(self.cls_token, std=.02)
            # the gradient of `expand` comes back with the batch stride on its size-1 dim; DDP then warns ("grad strides do
            # not match bucket view strides") and takes a copy path for this parameter: hand it canonical strides (no copy)
            self.cls_token.register_hook(lambda g: g.reshape(-1).view(g.shape))
        else:
            self.cls_token = None
        if ape:
            self.cls_pos_embed = nn.Parameter(torch.zeros(1, nglo, embed_dim))
            self.x_pos_embed = nn.Parameter(torch.zeros(1, nx, embed_dim // 2))
            self.y_pos_embed = nn.Parameter(torch.zeros(1, ny, embed_dim // 2))
            for p in (self.cls_pos_embed, self.x_pos_embed, self.y_pos_embed):
                nn.init.trunc_normal_(p, std=.02)
            # the gradient of the `cat` slice keeps the batch stride of the summed stream on its size-1 dim (same DDP
            # "grad strides do not match bucket view strides" copy path as cls_token above)
            self.cls_pos_embed.register_hook(lambda g: g.reshape(-1).view(g.shape))
        self.pos_drop = nn.Dropout(p=drop_rate)

    def forward(self, xtuple):
        x = xtuple[0]
        if x.is_cuda and self.channels_last:
            # NHWC convolution: the (B, tokens, C) streams on both sides of the patch merge ARE NHWC images, so the patchify conv
            # consumes / produces them without the NCHW <-> token transposing copies (and cuDNN drops its own nchwToNhwc pass);
            # under autocast the cast and the layout change of the input are one pass
            dt = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else x.dtype
            x = x.to(dtype=dt, memory_format=torch.channels_last)
            x = F.conv2d(x, self.proj.weight.to(dtype=dt, memory_format=torch.channels_last),
                         None if self.proj.bias is None else self.proj.bias.to(dt), stride=self.proj.stride)
        else:
            x = self.proj(x)
        B, _, nx, ny = x.shape
        assert nx == self.nx and ny == self.ny, "Fix input size!"
        x = x.flatten(2).transpose(1, 2)         # a view for an NHWC conv output (already (B, tokens, C) in memory)
        if self.norm_embed is not None:
            x = self.norm_embed(x)
        if self.cls_token is not None:
            x = torch.cat((self.cls_token.expand(B, -1, -1), x), dim=1)
        if self.ape:
            grid = torch.cat([self.x_pos_embed.unsqueeze(2).expand(-1, -1, ny, -1),
                              self.y_pos_embed.unsqueeze(1).expand(-1, nx, -1, -1)], dim=-1).flatten(1, 2)
            x = x + torch.cat([self.cls_pos_embed, grid], dim=1)
        return self.pos_drop(x), nx, ny


def _unpack(xtuple):
    """(x, nx, ny) or (x, nx, ny, pending) with pending = (branch output, deferred bias or None, per-sample scale or None)."""
    if len(xtuple) == 4:
        return xtuple
    x, nx, ny = xtuple
    return x, nx, ny, None


def _flush(x, pend):
    """Join a pending branch into the residual stream with stock ops (stage ends, unfused blocks, CPU)."""
    if pend is None:
        return x
    br, bias, scale = pend
    if bias is not None:
        br = br + bias
    if scale is not None:
        br = br * scale.view(-1, *([1] * (br.dim() - 1))).to(br.dtype)
    return x + br


def _join_and_norm(x, pend, norm):
    """x <- x + scale * (branch + bias);  h = norm(x)  - one kernel when a branch is pending (epilogue.add_norm)."""
    if pend is None:
        return x, norm(x)
    br, bias, scale = pend
    if not epilogue.addnorm_applies(x, br, x.shape[-1]):
        x = _flush(x, pend)
        return x, norm(x)
    return epilogue.add_norm(x, br, bias, scale, norm)


class AttnBlock(nn.Module):
    """x + drop_path(attn(norm(x), nx, ny))  (msvit.py:245-316).  `attn_type` dispatch: 'full' -> dense,
    'longformerhand' / 'longformer_b200' -> the fused B200 module (or `attn_cls` when given)."""

    def __init__(self, dim, num_heads, qkv_bias=False, qk_scale=None, drop=0., attn_drop=0., drop_path=0.,
                 norm_layer=nn.LayerNorm, attn_type="full", w=7, d=1, sharew=False, nglo=1, only_glo=False,
                 sw_exact=0, rpe=False, wx=14, wy=14, mode=0, attn_cls: Optional[Callable] = None, dense_impl="auto",
                 fused_residual=False):
        super().__init__()
        self.fused_residual = fused_residual
        self.norm = norm_layer(dim)
        if attn_type == "full":
            self.attn = DenseAttention(dim, num_heads=num_heads, qkv_bias=qkv_bias, qk_scale=qk_scale,
                                       attn_drop=attn_drop, proj_drop=drop, rpe=rpe, wx=wx, wy=wy, nglo=nglo, impl=dense_impl)
        elif attn_type in ("longformerhand", "longformerauto", "longformer_b200"):
            cls = attn_cls or B200Long2DSCSelfAttention
            self.attn = cls(dim, exact=sw_exact, num_heads=num_heads, qkv_bias=qkv_bias, qk_scale=qk_scale,
                            attn_drop=attn_drop, proj_drop=drop, w=w, d=d, sharew=sharew, nglo=nglo,
                            only_glo=only_glo, autograd=(attn_type == "longformerauto"), rpe=rpe, mode=mode)
        else:
            raise ValueError("Not supported attention type {}".format(attn_type))
        self.drop_path = DropPath(drop_path) if drop_path > 0. else nn.Identity()

    def forward(self, xtuple):
        x, nx, ny, pend = _unpack(xtuple)
        if (self.fused_residual and getattr(self.attn, "supports_deferred_bias", False) and isinstance(self.norm, B200LayerNorm)
                and epilogue.addnorm_applies(x, None, x.shape[-1])):
            # fused epilogue: the previous block's branch joins the residual stream inside this block's norm kernel, and this
            # block hands its own branch (projection output without bias, the bias, the DropPath scale) to the next one
            x, h = _join_and_norm(x, pend, self.norm)
            br, bias = self.attn(h, nx, ny, defer_proj_bias=True)
            return x, nx, ny, (br, bias, self.drop_path.sample_scale(x.shape[0], x.device) if isinstance(self.drop_path, DropPath) else None)
        x = _flush(x, pend)
        return x + self.drop_path(self.attn(self.norm(x), nx, ny)), nx, ny


class MlpBlock(nn.Module):
    def __init__(self, dim, out_dim=None, mlp_ratio=4., drop=0., drop_path=0., norm_layer=nn.LayerNorm, fused_residual=False):
        super().__init__()
        self.fused_residual = fused_residual
        self.drop_path = DropPath(drop_path) if drop_path > 0. else nn.Identity()
        self.norm = norm_layer(dim)
        self.mlp = Mlp(dim, int(dim * mlp_ratio), out_dim, drop=drop)
        self.shortcut = nn.Identity()
        if out_dim is not None and out_dim != dim:
            self.shortcut = nn.Sequential(nn.Linear(dim, out_dim), nn.Dropout(drop))

    def forward(self, xtuple):
        x, nx, ny, pend = _unpack(xtuple)
        if (self.fused_residual and isinstance(self.shortcut, nn.Identity) and epilogue.addnorm_applies(x, None, x.shape[-1])
                and isinstance(self.norm, B200LayerNorm)):
            x, h = _join_and_norm(x, pend, self.norm)
            br, bias = self.mlp.forward_deferred(h)
            return x, nx, ny, (br, bias, self.drop_path.sample_scale(x.shape[0], x.device) if isinstance(self.drop_path, DropPath) else None)
        x = _flush(x, pend)
        return self.shortcut(x) + self.drop_path(self.mlp(self.norm(x))), nx, ny


class MsViT(nn.Module):
    def __init__(self, arch, img_size=512, in_chans=3, num_classes=1000, qkv_bias=True, qk_scale=None,
                 drop_rate=0., attn_drop_rate=0., drop_path_rate=0., norm_embed=False, w=7, d=1, sharew=False,
                 only_glo=False, attn_type="longformerhand", sw_exact=0, mode=0, ln_eps=1e-6, avg_pool=False,
                 attn_cls: Optional[Callable] = None, fused_norm: bool = True, dense_impl: str = "auto",
                 fused_residual: bool = True, **unused):
        super().__init__()
        self.num_classes, self.attn_type, self.avg_pool = num_classes, attn_type, avg_pool
        # NB: the reference stores partial(LayerNorm, eps=ln_eps) in self.norm_layer but never uses it - every
        # LayerNorm it builds comes from the `norm_layer` ARGUMENT, whose default eps is 1e-6 (msvit.py:350,
        # 356-361, 378-390, 436).  LN_EPS therefore has no effect there; mirrored here for parity.
        del ln_eps
        # fused_norm: nn.LayerNorm subclass backed by the sm_90a LayerNorm kernels (SURVEY.md section 8 (f) row 4);
        # same parameters / state_dict, falls back to nn.LayerNorm on CPU.  The patch-embedding norm keeps its
        # input dtype because its output becomes the fp32 residual stream.
        # fused_residual: residual add + DropPath scale + deferred Linear bias + LayerNorm in one kernel per block boundary,
        # bias + GELU in one, bias gradients from those passes (epilogue.py; needs fused_norm).  Same parameters / state_dict.
        fused_residual = fused_residual and fused_norm
        self.fused_residual = fused_residual
        norm_layer = partial(B200LayerNorm, eps=1e-6) if fused_norm else partial(nn.LayerNorm, eps=1e-6)
        embed_norm = partial(B200LayerNorm, eps=1e-6, keep_dtype=True) if fused_norm else norm_layer
        self.layer_cfgs = parse_arch(arch)
        if len(self.layer_cfgs) not in (3, 4):
            raise ValueError("Numer of layers {} not implemented yet!".format(len(self.layer_cfgs)))
        self.depth = sum(c["n"] for c in self.layer_cfgs)
        self.Nglos = [c["g"] for c in self.layer_cfgs]
        self.out_planes = self.layer_cfgs[-1]["d"]
        rates = torch.linspace(0, drop_path_rate, self.depth).split([c["n"] for c in self.layer_cfgs])
        common = dict(qkv_bias=qkv_bias, qk_scale=qk_scale, drop=drop_rate, attn_drop=attn_drop_rate, d=d,
                      sharew=sharew, only_glo=only_glo, sw_exact=sw_exact, mode=mode, norm_layer=norm_layer,
                      attn_cls=attn_cls, dense_impl=dense_impl)
        res, in_dim = img_size, in_chans
        stages = []
        sticky_full = False     # msvit.py:460-461 mutates the shared attn_args: after the first s0 stage every
                                # later stage is dense too
        for i, cfg in enumerate(self.layer_cfgs):
            sticky_full = sticky_full or not cfg["s"]
            assert cfg["l"] == i + 1, "Error in _make_layer: layerid {} does not equal to layer_id {}".format(i + 1, cfg["l"])
            res = res // cfg["p"]
            ape = bool(cfg["a"])
            blocks = [PatchEmbed(cfg["p"], res, res, in_chans=in_dim, embed_dim=cfg["d"], nglo=cfg["g"],
                                 norm_layer=embed_norm, norm_embed=norm_embed, drop_rate=drop_rate, ape=ape)]
            for dpr in rates[i]:
                blocks.append(AttnBlock(cfg["d"], cfg["h"], drop_path=float(dpr),
                                        attn_type="full" if sticky_full else attn_type, w=cfg["f"], nglo=cfg["g"],
                                        rpe=not ape, wx=res, wy=res, fused_residual=fused_residual, **common))
                blocks.append(MlpBlock(cfg["d"], drop_path=float(dpr), mlp_ratio=4.0, drop=drop_rate,
                                       norm_layer=norm_layer, fused_residual=fused_residual))
            stages.append(nn.Sequential(*blocks))
            in_dim = cfg["d"]
        self.layer1, self.layer2, self.layer3 = stages[:3]
        self.layer4 = stages[3] if len(stages) == 4 else None
        self.norm = norm_layer(self.out_planes)
        self.head = nn.Linear(self.out_planes, num_classes) if num_classes > 0 else nn.Identity()
        self.apply(self._init_weights)

    @staticmethod
    def _init_weights(m):
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def no_weight_decay(self):
        return {"pos_embed", "cls_token", "norm.weight", "norm.bias", "norm_embed", "head.bias", "relative_position"}

    def forward_features(self, x):
        B = x.shape[0]
        stages = [s for s in (self.layer1, self.layer2, self.layer3, self.layer4) if s is not None]
        nx = ny = None
        for i, stage in enumerate(stages):
            if i > 0:   # drop the previous stage's global tokens, back to an image for the next patch merge
                if x.is_cuda and getattr(stage[0], "channels_last", False):
                    # the local tokens (B, nx*ny, C) are an NHWC image: one dense copy (with the autocast cast folded in), then a
                    # channels_last VIEW - instead of a transposing fp32 copy + cast + cuDNN's own NCHW -> NHWC pass
                    t = x[:, self.Nglos[i - 1]:]
                    t = t.to(torch.get_autocast_dtype("cuda")) if torch.is_autocast_enabled("cuda") else t.contiguous()
                    x = t.view(B, nx, ny, -1).permute(0, 3, 1, 2)
                else:
                    x = x[:, self.Nglos[i - 1]:].transpose(-2, -1).reshape(B, -1, nx, ny)
            x, nx, ny, pend = _unpack(stage((x, nx, ny)))
            if i + 1 < len(stages):
                x = _flush(x, pend)       # stage boundary: the last branch joins the stream with stock ops
        # the last block's branch joins inside the final norm's kernel
        if pend is not None and isinstance(self.norm, B200LayerNorm) and epilogue.addnorm_applies(x, pend[0], x.shape[-1]):
            x = epilogue.add_norm(x, pend[0], pend[1], pend[2], self.norm)[1]
        else:
            x = self.norm(_flush(x, pend))
        if self.Nglos[-1] > 0 and not self.avg_pool:
            return x[:, 0]
        return x.mean(dim=1)

    def reset_vil_mode(self, mode):
        """Switch the random-shift training mode of every longformer attention (msvit.py:532-541)."""
        for m in self.modules():
            if hasattr(m, "attention_window") and hasattr(m, "mode"):
                m.mode = mode

    def forward(self, x):
        return self.head(self.forward_features(x))


def build_vil(name: str = "vil_small", img_size: int = 224, **overrides) -> MsViT:
    """The kwargs `build_model` passes for the published ViL configs (models/__init__.py:37-54 with the
    defaults of config/defaults.py:131-161 / msvit.yaml)."""
    kw = dict(arch=ARCHS.get(name, name), img_size=img_size, drop_rate=0.0, drop_path_rate=0.1, norm_embed=True,
              avg_pool=False, sharew=True, attn_type="longformerhand", only_glo=False, sw_exact=0, ln_eps=1e-6,
              mode=0)
    kw.update(overrides)
    return MsViT(**kw)
