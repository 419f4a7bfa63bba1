"""SD1.5- and SD2.x-shaped UNet *host model* (plain PyTorch; stands in for diffusers' UNet2DConditionModel).

diffusers is not installed in this image and no SD weights exist offline, so the caller side of
the LoRA hot path is restated here: an architecture with the SD1.5 hyper-parameters
(block_out_channels (320,640,1280,1280), 2 layers per block, 8 heads, cross-attention dim 768,
GroupNorm-32), random-initialised. It is NOT part of the accelerated path: everything in this
file is ordinary torch.nn and runs through ATen/cuDNN. Its only contract with the LoRA code is
the one the reference relies on (lora_diffusion/lora.py:159-165, 208-212):

  * class NAMES: CrossAttention, GEGLU, ResnetBlock2D are what the target sets match on;
  * REGISTRATION ORDER: down_blocks -> up_blocks -> mid_block at the top level, `attentions`
    before `resnets` inside a block, attn1 -> ff -> attn2 inside a BasicTransformerBlock and
    conv1 -> time_emb_proj -> conv2 -> conv_shortcut inside a ResnetBlock2D. This reproduces the
    site order of the reference's fixture files (example_loras/*.safetensors: 144 UNet sites,
    per-block channel sequence [320,320,640,640,1280,1280 | 1280x3,640x3,320x3 | 1280];
    checked in tests/test_site_census.py).

SD 2.x (`UNetConfig.sd21()`, the topology of both stable-diffusion-2-1 768-v and 2-1-base) differs in
three hyper-parameters only: per-block head counts (5, 10, 20, 20) -- head dim 64 everywhere --,
cross-attention dim 1024 (OpenCLIP-H text encoder, host/clip.py) and `nn.Linear` proj_in / proj_out
(`use_linear_projection`). proj_in / proj_out sit in Transformer2DModel, outside every target set, so
the SD2 UNet has the same 144 default sites. diffusers' `upcast_attention` (softmax in fp32 for the
768-v model) is not restated: F.scaled_dot_product_attention already keeps its softmax in fp32 under
bf16 / fp16, and attention scores are not a LoRA site.
"""
import math
from dataclasses import dataclass, field
from typing import Optional, Tuple, Union

import torch
import torch.nn as nn
import torch.nn.functional as F


@dataclass
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    layers_per_block: int = 2
    # diffusers' meaning: the NUMBER of heads (dim_head = channels // heads); one int for every block
    # (SD1.5: 8) or one per down block (SD2.x: (5, 10, 20, 20)) -- up blocks take the tuple reversed,
    # the mid block its last entry
    attention_head_dim: Union[int, Tuple[int, ...]] = 8
    cross_attention_dim: int = 768
    norm_num_groups: int = 32
    # which down blocks carry cross-attention (SD1.5: first three)
    down_has_attn: Tuple[bool, ...] = (True, True, True, False)
    # Transformer2DModel proj_in / proj_out as nn.Linear on NHWC tokens (SD2.x) instead of 1x1 convs
    use_linear_projection: bool = False

    @staticmethod
    def sd15() -> "UNetConfig":
        return UNetConfig()

    @staticmethod
    def sd21() -> "UNetConfig":
        """stable-diffusion-2-1 (768-v, 96x96 latents) and 2-1-base (512, 64x64): same topology."""
        return UNetConfig(attention_head_dim=(5, 10, 20, 20), cross_attention_dim=1024,
                          use_linear_projection=True)

    @staticmethod
    def sd2_tiny() -> "UNetConfig":
        """SD2 features at toy widths (CPU tests): per-block heads, linear projection, and a
        cross-attention width (64, host/clip.py's tiny SD2 encoder) unlike the UNet's."""
        return UNetConfig(block_out_channels=(32, 64, 64), attention_head_dim=(2, 4, 4),
                          cross_attention_dim=64, norm_num_groups=8,
                          down_has_attn=(True, True, False), layers_per_block=1,
                          use_linear_projection=True)

    @staticmethod
    def tiny() -> "UNetConfig":
        """Same topology, toy widths (CPU tests)."""
        return UNetConfig(block_out_channels=(32, 64, 64), attention_head_dim=2,
                          cross_attention_dim=48, norm_num_groups=8,
                          down_has_attn=(True, True, False), layers_per_block=1)


class CrossAttention(nn.Module):
    def __init__(self, query_dim: int, cross_attention_dim: Optional[int], heads: int, dim_head: int):
        super().__init__()
        inner = heads * dim_head
        ctx_dim = cross_attention_dim if cross_attention_dim is not None else query_dim
        self.heads = heads
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(ctx_dim, inner, bias=False)
        self.to_v = nn.Linear(ctx_dim, inner, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(inner, query_dim), nn.Dropout(0.0)])

    def forward(self, hidden_states, encoder_hidden_states=None):
        ctx = hidden_states if encoder_hidden_states is None else encoder_hidden_states
        B, L, _ = hidden_states.shape
        q = self.to_q(hidden_states)
        k = self.to_k(ctx)
        v = self.to_v(ctx)
        h = self.heads
        q = q.view(B, L, h, -1).transpose(1, 2)
        k = k.view(B, ctx.shape[1], h, -1).transpose(1, 2)
        v = v.view(B, ctx.shape[1], h, -1).transpose(1, 2)
        o = F.scaled_dot_product_attention(q, k.to(q.dtype), v.to(q.dtype))
        o = o.transpose(1, 2).reshape(B, L, -1)
        o = self.to_out[0](o)
        return self.to_out[1](o)


class GEGLU(nn.Module):
    def __init__(self, dim_in: int, dim_out: int):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)

    def forward(self, x):
        h, gate = self.proj(x).chunk(2, dim=-1)
        return h * F.gelu(gate)


class FeedForward(nn.Module):
    def __init__(self, dim: int, mult: int = 4):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, dim * mult), nn.Dropout(0.0), nn.Linear(dim * mult, dim)])

    def forward(self, x):
        for m in self.net:
            x = m(x)
        return x


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim: int, heads: int, dim_head: int, cross_attention_dim: int):
        super().__init__()
        self.attn1 = CrossAttention(dim, None, heads, dim_head)
        self.ff = FeedForward(dim)
        self.attn2 = CrossAttention(dim, cross_attention_dim, heads, dim_head)
        self.norm1 = nn.LayerNorm(dim)
        self.norm2 = nn.LayerNorm(dim)
        self.norm3 = nn.LayerNorm(dim)

    def forward(self, x, context):
        x = self.attn1(self.norm1(x)) + x
        x = self.attn2(self.norm2(x), context) + x
        x = self.ff(self.norm3(x)) + x
        return x


class Transformer2DModel(nn.Module):
    def __init__(self, channels: int, heads: int, cross_attention_dim: int, groups: int, linear: bool = False):
        super().__init__()
        self.linear = linear
        proj = (lambda: nn.Linear(channels, channels)) if linear else (lambda: nn.Conv2d(channels, channels, 1))
        self.norm = nn.GroupNorm(groups, channels, eps=1e-6)
        self.proj_in = proj()
        self.transformer_blocks = nn.ModuleList(
            [BasicTransformerBlock(channels, heads, channels // heads, cross_attention_dim)])
        self.proj_out = proj()

    def forward(self, x, context):
        B, C, H, W = x.shape
        res = x
        h = self.norm(x)
        if not self.linear:
            h = self.proj_in(h)
        h = h.permute(0, 2, 3, 1).reshape(B, H * W, C)
        if self.linear:                      # diffusers' order: reshape to tokens, then proj_in
            h = self.proj_in(h)
        for blk in self.transformer_blocks:
            h = blk(h, context)
        if self.linear:
            h = self.proj_out(h)
        h = h.reshape(B, H, W, C).permute(0, 3, 1, 2)
        if not self.linear:
            h = self.proj_out(h)
        return h + res


class ResnetBlock2D(nn.Module):
    def __init__(self, in_channels: int, out_channels: int, temb_channels: int, groups: int):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=1e-5)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb_channels, out_channels)
        self.norm2 = nn.GroupNorm(groups, out_channels, eps=1e-5)
        self.dropout = nn.Dropout(0.0)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(in_channels, out_channels, 1) if in_channels != out_channels else None

    def forward(self, x, temb):
        h = self.conv1(F.silu(self.norm1(x)))
        t = self.time_emb_proj(F.silu(temb))
        h = h + t[:, :, None, None].to(h.dtype)
        h = self.conv2(self.dropout(F.silu(self.norm2(h))))
        if self.conv_shortcut is not None:
            x = self.conv_shortcut(x)
        return x + h


class Downsample2D(nn.Module):
    def __init__(self, channels: int):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, stride=2, padding=1)

    def forward(self, x):
        return self.conv(x)


class Upsample2D(nn.Module):
    def __init__(self, channels: int):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, padding=1)

    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))


class DownBlock(nn.Module):
    """CrossAttnDownBlock2D / DownBlock2D."""

    def __init__(self, cin, cout, temb, layers, has_attn, heads, ctx_dim, groups, add_down, linear=False):
        super().__init__()
        if has_attn:
            self.attentions = nn.ModuleList(
                [Transformer2DModel(cout, heads, ctx_dim, groups, linear) for _ in range(layers)])
        self.resnets = nn.ModuleList(
            [ResnetBlock2D(cin if i == 0 else cout, cout, temb, groups) for i in range(layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if add_down else None
        self.has_attn = has_attn

    def forward(self, x, temb, context):
        outs = []
        for i, res in enumerate(self.resnets):
            x = res(x, temb)
            if self.has_attn:
                x = self.attentions[i](x, context)
            outs.append(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
            outs.append(x)
        return x, outs


class UpBlock(nn.Module):
    """CrossAttnUpBlock2D / UpBlock2D."""

    def __init__(self, cin, cout, cprev, temb, layers, has_attn, heads, ctx_dim, groups, add_up, linear=False):
        super().__init__()
        if has_attn:
            self.attentions = nn.ModuleList(
                [Transformer2DModel(cout, heads, ctx_dim, groups, linear) for _ in range(layers)])
        resnets = []
        for i in range(layers):
            skip = cin if i == layers - 1 else cout
            inp = cprev if i == 0 else cout
            resnets.append(ResnetBlock2D(inp + skip, cout, temb, groups))
        self.resnets = nn.ModuleList(resnets)
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_up else None
        self.has_attn = has_attn

    def forward(self, x, skips, temb, context):
        for i, res in enumerate(self.resnets):
            x = torch.cat([x, skips.pop()], dim=1)
            x = res(x, temb)
            if self.has_attn:
                x = self.attentions[i](x, context)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x)
        return x


class MidBlock(nn.Module):
    """UNetMidBlock2DCrossAttn: resnet, attention, resnet."""

    def __init__(self, ch, temb, heads, ctx_dim, groups, linear=False):
        super().__init__()
        self.attentions = nn.ModuleList([Transformer2DModel(ch, heads, ctx_dim, groups, linear)])
        self.resnets = nn.ModuleList([ResnetBlock2D(ch, ch, temb, groups) for _ in range(2)])

    def forward(self, x, temb, context):
        x = self.resnets[0](x, temb)
        x = self.attentions[0](x, context)
        return self.resnets[1](x, temb)


class TimestepEmbedding(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.linear_1 = nn.Linear(cin, cout)
        self.linear_2 = nn.Linear(cout, cout)

    def forward(self, x):
        return self.linear_2(F.silu(self.linear_1(x)))


def sinusoidal_embedding(timesteps: torch.Tensor, dim: int) -> torch.Tensor:
    """flip_sin_to_cos = True, freq_shift = 0 (SD1.5)."""
    half = dim // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32, device=timesteps.device) / half)
    args = timesteps.float()[:, None] * freqs[None, :]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


class UNetOutput:
    __slots__ = ("sample",)

    def __init__(self, sample):
        self.sample = sample


class UNet2DConditionModel(nn.Module):
    def __init__(self, cfg: UNetConfig = UNetConfig()):
        super().__init__()
        self.cfg = cfg
        ch = cfg.block_out_channels
        temb = ch[0] * 4
        g = cfg.norm_num_groups
        heads = cfg.attention_head_dim
        if isinstance(heads, int):
            heads = (heads,) * len(ch)
        if len(heads) != len(ch):
            raise ValueError(f"attention_head_dim {heads}: one head count per block {ch}")
        lin = cfg.use_linear_projection
        self.conv_in = nn.Conv2d(cfg.in_channels, ch[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(ch[0], temb)
        self.down_blocks = nn.ModuleList()
        self.mid_block = None            # plain attribute for now; registered after up_blocks
        self.up_blocks = nn.ModuleList()
        cout = ch[0]
        for i, c in enumerate(ch):
            cin, cout = cout, c
            last = i == len(ch) - 1
            self.down_blocks.append(DownBlock(cin, cout, temb, cfg.layers_per_block,
                                              cfg.down_has_attn[i], heads[i], cfg.cross_attention_dim,
                                              g, add_down=not last, linear=lin))
        rev = list(reversed(ch))
        rev_attn = list(reversed(cfg.down_has_attn))
        rev_heads = list(reversed(heads))
        cout = rev[0]
        for i, c in enumerate(rev):
            cprev, cout = cout, c
            cin = rev[min(i + 1, len(ch) - 1)]
            last = i == len(ch) - 1
            self.up_blocks.append(UpBlock(cin, cout, cprev, temb, cfg.layers_per_block + 1,
                                          rev_attn[i], rev_heads[i], cfg.cross_attention_dim, g,
                                          add_up=not last, linear=lin))
        self.mid_block = MidBlock(ch[-1], temb, heads[-1], cfg.cross_attention_dim, g, linear=lin)
        self.conv_norm_out = nn.GroupNorm(g, ch[0], eps=1e-5)
        self.conv_out = nn.Conv2d(ch[0], cfg.out_channels, 3, padding=1)

    @property
    def device(self):
        return self.conv_in.weight.device

    @property
    def dtype(self):
        return self.conv_in.weight.dtype

    def forward(self, sample, timesteps, encoder_hidden_states):
        if not torch.is_tensor(timesteps):
            timesteps = torch.tensor([timesteps], device=sample.device)
        if timesteps.dim() == 0:
            timesteps = timesteps[None]
        timesteps = timesteps.expand(sample.shape[0])
        t_emb = sinusoidal_embedding(timesteps, self.cfg.block_out_channels[0]).to(sample.dtype)
        temb = self.time_embedding(t_emb)
        ctx = encoder_hidden_states
        x = self.conv_in(sample)
        skips = [x]
        for blk in self.down_blocks:
            x, outs = blk(x, temb, ctx)
            skips.extend(outs)
        x = self.mid_block(x, temb, ctx)
        for blk in self.up_blocks:
            x = blk(x, skips, temb, ctx)
        x = self.conv_out(F.silu(self.conv_norm_out(x)))
        return UNetOutput(x)
