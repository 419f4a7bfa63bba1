"""ORACLE (test infrastructure only): the reference's training steps that start from images, in plain
PyTorch eager, float64 when the models are.

  train_lora_dreambooth.py:818-821   latents = vae.encode(batch["pixel_values"].to(weight_dtype))
                                     .latent_dist.sample() * 0.18215, every step
  cli_lora_pti.py:273-290            loss_step(cached_latents=False): the same, and with
                                     train_inpainting the masked image encoded and sampled too and
                                     mask = F.interpolate(mask_values, scale_factor=1/8)
  dataset.py:108-116, 240-252        pixel_values = Normalize([0.5], [0.5])(ToTensor()(image));
                                     masked_image = image * (mask < 0.5)

The posterior is diffusers' DiagonalGaussianDistribution: mean, logvar = chunk(moments, 2, dim=1),
logvar.clamp(-30, 20), std = exp(0.5 * logvar), sample = mean + std * eps. The posterior noise eps
is passed in (the reference draws it inside `sample()`, before the step's noise and timesteps). The
latents are widened to at least fp32 before noising, as the step engine does (float64 stays float64).
Everything after the latents is oracle/ref_step_v.py's loss, unchanged. Imports nothing from the
product package.
"""
import torch
import torch.nn.functional as F

from .ref_step_v import RefDreamboothStepV

SCALING = 0.18215


def to_vae_input(pixels: torch.Tensor) -> torch.Tensor:
    """uint8 [B, H, W, 3] -> ToTensor + Normalize([0.5], [0.5]) -> fp32 [B, 3, H, W]; fp32 [B, 3, H, W]
    pixels are already normalised and pass unchanged."""
    if pixels.dtype == torch.uint8:
        return (pixels.permute(0, 3, 1, 2).float() / 255 - 0.5) / 0.5
    return pixels


def masked_image(image: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    return image * (mask < 0.5)


def posterior_sample(moments: torch.Tensor, eps: torch.Tensor, scaling: float = SCALING) -> torch.Tensor:
    mean, logvar = torch.chunk(moments, 2, dim=1)
    logvar = torch.clamp(logvar, -30.0, 20.0)
    std = torch.exp(0.5 * logvar)
    return (mean + std * eps) * scaling


def latent_mask(mask: torch.Tensor) -> torch.Tensor:
    """cli_lora_pti.py:286-289: the image-resolution mask on the latent grid (nearest, pixel (8i, 8j))."""
    return F.interpolate(mask, scale_factor=1 / 8)


@torch.no_grad()
def encode(vae, pixels, posterior_noise, mask=None, masked_posterior_noise=None, scaling: float = SCALING):
    """(latents, inpaint) from a batch of images through the frozen `vae`, in its dtype: latents
    [B, C, h, w]; inpaint None, or (latent-grid mask, masked-image latents) when `mask` ([B, 1, H, W],
    image resolution) is given -- the `inpaint=` argument of RefDreamboothStep.forward_loss."""
    vdt = next(vae.parameters()).dtype
    dev = next(vae.parameters()).device
    image = to_vae_input(pixels.cpu()).to(dev)          # the data loader's ToTensor runs on the CPU

    def encode_one(x, eps):
        moments = vae.encode(x.to(vdt)).latent_dist.parameters
        lat = posterior_sample(moments, eps.to(dev), scaling)
        return lat.to(torch.promote_types(lat.dtype, torch.float32))

    latents = encode_one(image, posterior_noise)
    if mask is None:
        return latents, None
    mask = mask.to(dev).float()
    masked = encode_one(masked_image(image, mask), masked_posterior_noise)
    return latents, (latent_mask(mask).to(latents.dtype), masked)


class RefImageStep(RefDreamboothStepV):
    """RefDreamboothStep (with the prediction type) fed from images through a frozen VAE."""

    def __init__(self, vae, *args, scaling: float = SCALING, **kw):
        super().__init__(*args, **kw)
        self.vae, self.scaling = vae, scaling
        vae.requires_grad_(False)

    def encode(self, pixels, posterior_noise, mask=None, masked_posterior_noise=None):
        return encode(self.vae, pixels, posterior_noise, mask, masked_posterior_noise, self.scaling)

    def forward_loss_from_pixels(self, pixels, input_ids, posterior_noise, noise, timesteps, mask=None,
                                 masked_posterior_noise=None, **loss_kw):
        latents, inpaint = self.encode(pixels, posterior_noise, mask, masked_posterior_noise)
        if inpaint is not None:
            loss_kw["inpaint"] = inpaint
        return self.forward_loss(latents, input_ids, noise.to(latents.dtype), timesteps, **loss_kw)

    def step_from_pixels(self, pixels, input_ids, posterior_noise, noise, timesteps, mask=None,
                         masked_posterior_noise=None, **loss_kw):
        """One optimizer step (RefDreamboothStep.step's clip + AdamW) from images."""
        latents, inpaint = self.encode(pixels, posterior_noise, mask, masked_posterior_noise)
        if inpaint is not None:
            loss_kw["inpaint"] = inpaint
        return self.step(latents, input_ids, noise=noise.to(latents.dtype), timesteps=timesteps, **loss_kw)
