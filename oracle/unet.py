"""ORACLE (test infrastructure only — never imported by the product path).

Plain-torch fp32 restatement of diffusers' `UNet2DConditionModel` in the Stable-Diffusion-2
configuration Marigold uses (reference call site: marigold/marigold_depth_pipeline.py:461-463;
`in_channels=8` pinned by src/trainer/marigold_depth_trainer.py:189-204).

PARITY UNPINNED: `diffusers` (requirements.txt:2, `>=0.25.0`, no lockfile) is neither vendored in
the reference repository nor installed, and no checkpoint is on disk, so this restatement follows the
published architecture (SURVEY.md App. A.1) and is cross-checked only by its parameter count
(865.9 M for the SD-2 config, tests/test_oracle.py). Module/parameter names are diffusers'
state-dict names so that a real checkpoint would load unchanged.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List

import torch
import torch.nn as nn
import torch.nn.functional as F


@dataclass
class UNetConfig:
    in_channels: int = 8
    out_channels: int = 4
    block_out_channels: List[int] = field(default_factory=lambda: [320, 640, 1280, 1280])
    layers_per_block: int = 2
    cross_attention_dim: int = 1024
    head_dim: int = 64            # diffusers' "attention_head_dim" [5,10,20,20] are head COUNTS = C/64
    norm_num_groups: int = 32
    norm_eps: float = 1e-5

    @staticmethod
    def tiny():
        return UNetConfig(block_out_channels=[64, 128, 256, 256], cross_attention_dim=128)


def timestep_embedding(t: torch.Tensor, dim: int) -> torch.Tensor:
    """get_timestep_embedding(flip_sin_to_cos=True, downscale_freq_shift=0), fp32. App. A.1 step 1."""
    half = dim // 2
    exponent = -math.log(10000.0) * torch.arange(half, dtype=torch.float32, device=t.device) / half
    ang = t.float()[:, None] * torch.exp(exponent)[None, :]
    return torch.cat([torch.cos(ang), torch.sin(ang)], dim=-1)


class TimestepEmbedding(nn.Module):
    def __init__(self, cin, dim):
        super().__init__()
        self.linear_1 = nn.Linear(cin, dim)
        self.linear_2 = nn.Linear(dim, dim)

    def forward(self, x):
        return self.linear_2(F.silu(self.linear_1(x)))


class ResnetBlock2D(nn.Module):
    def __init__(self, cin, cout, temb_dim, groups, eps):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin, eps=eps)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb_dim, cout) if temb_dim else None
        self.norm2 = nn.GroupNorm(groups, cout, eps=eps)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None

    def forward(self, x, temb=None):
        h = self.conv1(F.silu(self.norm1(x)))
        if self.time_emb_proj is not None:
            h = h + self.time_emb_proj(F.silu(temb))[:, :, None, None]
        h = self.conv2(F.silu(self.norm2(h)))
        if self.conv_shortcut is not None:
            x = self.conv_shortcut(x)
        return x + h


class Attention(nn.Module):
    """diffusers Attention: to_q/to_k/to_v without bias, to_out.0 with bias; heads of `head_dim`."""

    def __init__(self, dim, ctx_dim, head_dim):
        super().__init__()
        self.heads = dim // head_dim
        self.head_dim = head_dim
        self.to_q = nn.Linear(dim, dim, bias=False)
        self.to_k = nn.Linear(ctx_dim, dim, bias=False)
        self.to_v = nn.Linear(ctx_dim, dim, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(dim, dim)])

    def forward(self, x, ctx=None):
        ctx = x if ctx is None else ctx
        B, T, _ = x.shape
        q = self.to_q(x).reshape(B, T, self.heads, self.head_dim).transpose(1, 2)
        k = self.to_k(ctx).reshape(B, -1, self.heads, self.head_dim).transpose(1, 2)
        v = self.to_v(ctx).reshape(B, -1, self.heads, self.head_dim).transpose(1, 2)
        o = F.scaled_dot_product_attention(q, k, v)  # scale 1/sqrt(head_dim)
        return self.to_out[0](o.transpose(1, 2).reshape(B, T, -1))


class GEGLU(nn.Module):
    def __init__(self, dim, inner):
        super().__init__()
        self.proj = nn.Linear(dim, inner * 2)

    def forward(self, x):
        u, g = self.proj(x).chunk(2, dim=-1)   # first half value, second half gate
        return u * F.gelu(g)                   # exact erf GELU


class FeedForward(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, 4 * dim), nn.Identity(), nn.Linear(4 * dim, dim)])

    def forward(self, x):
        return self.net[2](self.net[0](x))


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim, ctx_dim, head_dim):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim)
        self.attn1 = Attention(dim, dim, head_dim)
        self.norm2 = nn.LayerNorm(dim)
        self.attn2 = Attention(dim, ctx_dim, head_dim)
        self.norm3 = nn.LayerNorm(dim)
        self.ff = FeedForward(dim)

    def forward(self, x, ctx):
        x = x + self.attn1(self.norm1(x))
        x = x + self.attn2(self.norm2(x), ctx)
        x = x + self.ff(self.norm3(x))
        return x


class Transformer2DModel(nn.Module):
    """use_linear_projection=True, one BasicTransformerBlock, GroupNorm eps 1e-6."""

    def __init__(self, dim, ctx_dim, head_dim, groups):
        super().__init__()
        self.norm = nn.GroupNorm(groups, dim, eps=1e-6)
        self.proj_in = nn.Linear(dim, dim)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(dim, ctx_dim, head_dim)])
        self.proj_out = nn.Linear(dim, dim)

    def forward(self, x, ctx):
        B, C, H, W = x.shape
        res = x
        h = self.norm(x).permute(0, 2, 3, 1).reshape(B, H * W, C)
        h = self.proj_in(h)
        for blk in self.transformer_blocks:
            h = blk(h, ctx)
        h = self.proj_out(h)
        return h.reshape(B, H, W, C).permute(0, 3, 1, 2) + res


class Downsample2D(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=2, padding=1)

    def forward(self, x):
        return self.conv(x)


class Upsample2D(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, padding=1)

    def forward(self, x, output_size=None):
        # diffusers Upsample2D.forward: scale_factor=2 by default; when the UNet forwards `upsample_size` (latent sizes
        # that are not a multiple of 2**num_upsamplers) the target is the skip connection's size: interpolate(size=...)
        if output_size is None:
            return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))
        return self.conv(F.interpolate(x, size=output_size, mode="nearest"))


class DownBlock(nn.Module):
    def __init__(self, cin, cout, temb, cfg: UNetConfig, attn: bool, down: bool):
        super().__init__()
        g, e = cfg.norm_num_groups, cfg.norm_eps
        self.resnets = nn.ModuleList(
            [ResnetBlock2D(cin if i == 0 else cout, cout, temb, g, e) for i in range(cfg.layers_per_block)])
        self.attentions = nn.ModuleList(
            [Transformer2DModel(cout, cfg.cross_attention_dim, cfg.head_dim, g)
             for _ in range(cfg.layers_per_block)]) if attn else None
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if down else None

    def forward(self, x, temb, ctx):
        outs = []
        for i, r in enumerate(self.resnets):
            x = r(x, temb)
            if self.attentions is not None:
                x = self.attentions[i](x, ctx)
            outs.append(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
            outs.append(x)
        return x, outs


class MidBlock(nn.Module):
    def __init__(self, c, temb, cfg: UNetConfig):
        super().__init__()
        g, e = cfg.norm_num_groups, cfg.norm_eps
        self.resnets = nn.ModuleList([ResnetBlock2D(c, c, temb, g, e), ResnetBlock2D(c, c, temb, g, e)])
        self.attentions = nn.ModuleList([Transformer2DModel(c, cfg.cross_attention_dim, cfg.head_dim, g)])

    def forward(self, x, temb, ctx):
        x = self.resnets[0](x, temb)
        x = self.attentions[0](x, ctx)
        return self.resnets[1](x, temb)


class UpBlock(nn.Module):
    def __init__(self, skip_channels: List[int], prev, cout, temb, cfg: UNetConfig, attn: bool, up: bool):
        super().__init__()
        g, e = cfg.norm_num_groups, cfg.norm_eps
        res = []
        cin = prev
        for sc in skip_channels:
            res.append(ResnetBlock2D(cin + sc, cout, temb, g, e))
            cin = cout
        self.resnets = nn.ModuleList(res)
        self.attentions = nn.ModuleList(
            [Transformer2DModel(cout, cfg.cross_attention_dim, cfg.head_dim, g) for _ in skip_channels]) if attn else None
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if up else None

    def forward(self, x, skips, temb, ctx, forward_upsample_size=False):
        for i, r in enumerate(self.resnets):
            x = torch.cat([x, skips.pop()], dim=1)
            x = r(x, temb)
            if self.attentions is not None:
                x = self.attentions[i](x, ctx)
        if self.upsamplers is not None:
            # UNet2DConditionModel.forward: `upsample_size = down_block_res_samples[-1].shape[2:]` (the next skip) when
            # any latent dim % 2**num_upsamplers != 0; this is how odd sizes such as 54 -> 27 -> 14 -> 7 come back up
            size = tuple(skips[-1].shape[2:]) if forward_upsample_size else None
            x = self.upsamplers[0](x, size)
        return x


class UNet2DConditionOracle(nn.Module):
    def __init__(self, cfg: UNetConfig = UNetConfig()):
        super().__init__()
        self.cfg = cfg
        ch = cfg.block_out_channels
        temb = ch[0] * 4
        self.conv_in = nn.Conv2d(cfg.in_channels, ch[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(ch[0], temb)
        n = len(ch)
        self.down_blocks = nn.ModuleList()
        skip_ch = [ch[0]]
        prev = ch[0]
        for i, c in enumerate(ch):
            last = i == n - 1
            self.down_blocks.append(DownBlock(prev, c, temb, cfg, attn=not last, down=not last))
            skip_ch += [c] * cfg.layers_per_block + ([c] if not last else [])
            prev = c
        self.mid_block = MidBlock(ch[-1], temb, cfg)
        self.up_blocks = nn.ModuleList()
        rev = list(reversed(ch))
        prev = ch[-1]
        for i, c in enumerate(rev):
            skips = [skip_ch.pop() for _ in range(cfg.layers_per_block + 1)]
            self.up_blocks.append(UpBlock(skips, prev, c, temb, cfg, attn=i > 0, up=i < n - 1))
            prev = c
        self.conv_norm_out = nn.GroupNorm(cfg.norm_num_groups, ch[0], eps=cfg.norm_eps)
        self.conv_out = nn.Conv2d(ch[0], cfg.out_channels, 3, padding=1)

    def forward(self, x, t, encoder_hidden_states):
        B = x.shape[0]
        t = torch.as_tensor(t, device=x.device).reshape(-1).expand(B)
        temb = self.time_embedding(timestep_embedding(t, self.cfg.block_out_channels[0]).to(x.dtype))
        h = self.conv_in(x)
        skips = [h]
        for blk in self.down_blocks:
            h, outs = blk(h, temb, encoder_hidden_states)
            skips += outs
        h = self.mid_block(h, temb, encoder_hidden_states)
        up_factor = 2 ** (len(self.up_blocks) - 1)
        fwd_size = any(d % up_factor != 0 for d in x.shape[-2:])
        for blk in self.up_blocks:
            h = blk(h, skips, temb, encoder_hidden_states, fwd_size)
        return self.conv_out(F.silu(self.conv_norm_out(h)))
