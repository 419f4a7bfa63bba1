"""SD 1.x / 2.x VAE *host model* (plain PyTorch; stands in for diffusers' AutoencoderKL): the encoder
half always, the decoder half on request.

diffusers is not installed here, so the frozen encoder the reference's trainers call every step
(`vae.encode(pixel_values).latent_dist.sample()`, train_lora_dreambooth.py:818-821,
cli_lora_pti.py:273-290) is restated, as host/unet_sd15.py restates the UNet: AutoencoderKL's
`encoder` plus `quant_conv` -- conv_in, four DownEncoderBlock2D (128, 256, 512, 512; two
ResnetBlock2D each, GroupNorm-32 with eps 1e-6, SiLU; a Downsample2D that pads (0, 1, 0, 1) and runs
a stride-2 conv after all but the last), the mid block (resnet, single-head attention, resnet),
GroupNorm + SiLU + conv_out to 2 x 4 channels (`double_z`), then the 1x1 quant_conv. It is frozen
and runs through ATen / cuDNN; nothing here is a LoRA site.

State-dict keys are diffusers' (`encoder.down_blocks.0.resnets.0.norm1.weight`, ...). The mid-block
attention is named as in diffusers releases before 0.14 (`group_norm`, `query`, `key`, `value`,
`proj_attn`), the names `lora_b200.to_ckpt.convert_vae_state_dict` maps to the original SD
checkpoint; state dicts with the later names (`to_q`, `to_k`, `to_v`, `to_out.0`) load too.

`encode(x).latent_dist` is a DiagonalGaussianDistribution with diffusers' attributes, so a diffusers
AutoencoderKL and this encoder fill the same slot of the step engine (which reads only
`.latent_dist.parameters`).

`AutoencoderKL(cfg, with_decoder=True)` adds diffusers' `post_quant_conv` (1x1) and `Decoder`: conv_in
from the latents to the widest channel count, the mid block, four UpDecoderBlock2D (the encoder's
widths reversed, three ResnetBlock2D each, nearest x2 upsampling + 3x3 conv after all but the last),
GroupNorm + SiLU + conv_out to 3 channels. `decode(z).sample` is the image in [-1, 1] (before
clamping). The decoder is built after the encoder and quant_conv, so those draw the same random
numbers, and have the same keys, with or without it.
"""
from dataclasses import dataclass
from typing import Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F


@dataclass
class VAEConfig:
    in_channels: int = 3
    latent_channels: int = 4
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    norm_num_groups: int = 32

    @staticmethod
    def sd() -> "VAEConfig":
        """The VAE of SD 1.x and SD 2.x (both use the same autoencoder topology)."""
        return VAEConfig()

    @staticmethod
    def tiny() -> "VAEConfig":
        """Same topology (four blocks, 8x downsampling, two resnets per block), toy widths (CPU tests)."""
        return VAEConfig(block_out_channels=(8, 16, 16, 16), norm_num_groups=4)


class DiagonalGaussianDistribution:
    """diffusers' posterior: parameters [B, 2C, h, w] = (mean ; logvar), logvar clamped to [-30, 20].
    logvar / std / var are evaluated when read (the same ops as diffusers), so an encode whose caller
    reads only `parameters` launches nothing for them."""

    def __init__(self, parameters: torch.Tensor):
        self.parameters = parameters
        self.mean = torch.chunk(parameters, 2, dim=1)[0]

    @property
    def logvar(self) -> torch.Tensor:
        return torch.clamp(torch.chunk(self.parameters, 2, dim=1)[1], -30.0, 20.0)

    @property
    def std(self) -> torch.Tensor:
        return torch.exp(0.5 * self.logvar)

    @property
    def var(self) -> torch.Tensor:
        return torch.exp(self.logvar)

    def sample(self, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        """mean + std * eps, eps drawn in the parameters' dtype (current diffusers' randn_tensor)."""
        eps = torch.randn(self.mean.shape, generator=generator, device=self.parameters.device,
                          dtype=self.parameters.dtype)
        return self.mean + self.std * eps

    def mode(self) -> torch.Tensor:
        return self.mean


class AutoencoderKLOutput:
    __slots__ = ("latent_dist",)

    def __init__(self, latent_dist):
        self.latent_dist = latent_dist


class ResnetBlock2D(nn.Module):
    def __init__(self, cin: int, cout: int, groups: int):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin, eps=1e-6)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.norm2 = nn.GroupNorm(groups, cout, eps=1e-6)
        self.dropout = nn.Dropout(0.0)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None

    def forward(self, x):
        h = self.conv1(F.silu(self.norm1(x)))
        h = self.conv2(self.dropout(F.silu(self.norm2(h))))
        if self.conv_shortcut is not None:
            x = self.conv_shortcut(x)
        return x + h


class Downsample2D(nn.Module):
    def __init__(self, channels: int):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, stride=2, padding=0)

    def forward(self, x):
        return self.conv(F.pad(x, (0, 1, 0, 1), mode="constant", value=0))


class DownEncoderBlock2D(nn.Module):
    def __init__(self, cin: int, cout: int, layers: int, groups: int, add_down: bool):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, groups) for i in range(layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if add_down else None

    def forward(self, x):
        for res in self.resnets:
            x = res(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
        return x


# diffusers >= 0.14 names of the mid-block attention -> the names this module (and to_ckpt) uses
_NEW_ATTN_NAMES = {"to_q.": "query.", "to_k.": "key.", "to_v.": "value.", "to_out.0.": "proj_attn."}


class AttentionBlock(nn.Module):
    """Single-head self-attention over the h*w positions, with the residual (the VAE mid block)."""

    def __init__(self, channels: int, groups: int):
        super().__init__()
        self.group_norm = nn.GroupNorm(groups, channels, eps=1e-6)
        self.query = nn.Linear(channels, channels)
        self.key = nn.Linear(channels, channels)
        self.value = nn.Linear(channels, channels)
        self.proj_attn = nn.Linear(channels, channels)
        self._register_load_state_dict_pre_hook(self._rename_new_keys)

    @staticmethod
    def _rename_new_keys(state_dict, prefix, *args):
        for new, old in _NEW_ATTN_NAMES.items():
            for leaf in ("weight", "bias"):
                k = prefix + new + leaf
                if k in state_dict:
                    state_dict[prefix + old + leaf] = state_dict.pop(k)

    def forward(self, x):
        B, C, H, W = x.shape
        h = self.group_norm(x).reshape(B, C, H * W).transpose(1, 2)
        q, k, v = self.query(h), self.key(h), self.value(h)
        o = F.scaled_dot_product_attention(q[:, None], k[:, None], v[:, None])[:, 0]
        o = self.proj_attn(o)
        return o.transpose(1, 2).reshape(B, C, H, W) + x


class UNetMidBlock2D(nn.Module):
    def __init__(self, channels: int, groups: int):
        super().__init__()
        self.attentions = nn.ModuleList([AttentionBlock(channels, groups)])
        self.resnets = nn.ModuleList([ResnetBlock2D(channels, channels, groups) for _ in range(2)])

    def forward(self, x):
        x = self.resnets[0](x)
        x = self.attentions[0](x)
        return self.resnets[1](x)


class Encoder(nn.Module):
    def __init__(self, cfg: VAEConfig):
        super().__init__()
        ch, g = cfg.block_out_channels, cfg.norm_num_groups
        self.conv_in = nn.Conv2d(cfg.in_channels, ch[0], 3, padding=1)
        self.down_blocks = nn.ModuleList()
        cout = ch[0]
        for i, c in enumerate(ch):
            cin, cout = cout, c
            self.down_blocks.append(DownEncoderBlock2D(cin, cout, cfg.layers_per_block, g,
                                                       add_down=i < len(ch) - 1))
        self.mid_block = UNetMidBlock2D(ch[-1], g)
        self.conv_norm_out = nn.GroupNorm(g, ch[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(ch[-1], 2 * cfg.latent_channels, 3, padding=1)

    def forward(self, x):
        x = self.conv_in(x)
        for blk in self.down_blocks:
            x = blk(x)
        x = self.mid_block(x)
        return self.conv_out(F.silu(self.conv_norm_out(x)))


class Upsample2D(nn.Module):
    def __init__(self, channels: int):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, padding=1)

    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))


class UpDecoderBlock2D(nn.Module):
    def __init__(self, cin: int, cout: int, layers: int, groups: int, add_up: bool):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, groups) for i in range(layers)])
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_up else None

    def forward(self, x):
        for res in self.resnets:
            x = res(x)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x)
        return x


class Decoder(nn.Module):
    def __init__(self, cfg: VAEConfig):
        super().__init__()
        ch, g = tuple(reversed(cfg.block_out_channels)), cfg.norm_num_groups
        self.conv_in = nn.Conv2d(cfg.latent_channels, ch[0], 3, padding=1)
        self.mid_block = UNetMidBlock2D(ch[0], g)
        self.up_blocks = nn.ModuleList()
        cout = ch[0]
        for i, c in enumerate(ch):
            cin, cout = cout, c
            self.up_blocks.append(UpDecoderBlock2D(cin, cout, cfg.layers_per_block + 1, g,
                                                   add_up=i < len(ch) - 1))
        self.conv_norm_out = nn.GroupNorm(g, ch[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(ch[-1], cfg.in_channels, 3, padding=1)

    def forward(self, z):
        x = self.mid_block(self.conv_in(z))
        for blk in self.up_blocks:
            x = blk(x)
        return self.conv_out(F.silu(self.conv_norm_out(x)))


class DecoderOutput:
    __slots__ = ("sample",)

    def __init__(self, sample):
        self.sample = sample


class AutoencoderKL(nn.Module):
    """diffusers' AutoencoderKL: `encode(x)` of [B, 3, H, W] images in [-1, 1] gives the posterior over
    [B, 4, H/8, W/8] latents; with `with_decoder=True`, `decode(z).sample` maps latents back to images.
    Runs in whatever dtype / memory format the module is given (the step engine uses the VAE's dtype
    and channels_last); no host sync and no data-dependent allocation, so it runs inside a captured
    CUDA graph."""

    def __init__(self, cfg: VAEConfig = VAEConfig(), with_decoder: bool = False):
        super().__init__()
        self.cfg = cfg
        self.encoder = Encoder(cfg)
        self.quant_conv = nn.Conv2d(2 * cfg.latent_channels, 2 * cfg.latent_channels, 1)
        self.has_decoder = with_decoder
        if with_decoder:
            self.decoder = Decoder(cfg)
            self.post_quant_conv = nn.Conv2d(cfg.latent_channels, cfg.latent_channels, 1)

    @property
    def dtype(self):
        return self.quant_conv.weight.dtype

    @property
    def device(self):
        return self.quant_conv.weight.device

    def encode(self, x: torch.Tensor) -> AutoencoderKLOutput:
        return AutoencoderKLOutput(DiagonalGaussianDistribution(self.quant_conv(self.encoder(x))))

    def decode(self, z: torch.Tensor) -> DecoderOutput:
        if not self.has_decoder:
            raise ValueError("this AutoencoderKL was built without its decoder: AutoencoderKL(cfg, with_decoder=True)")
        return DecoderOutput(self.decoder(self.post_quant_conv(z)))
