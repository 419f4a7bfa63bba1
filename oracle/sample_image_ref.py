"""ORACLE (test infrastructure only -- never imported by the product path).

diffusers' StableDiffusionImg2ImgPipeline and StableDiffusionInpaintPipeline (releases 0.11-0.14, the
releases oracle/sample_ref.py pins) written eagerly, op by op, as the pipelines write them, on top of
sample_ref's schedulers and loop:

  img2img   preprocess: 2.0 * (uint8 / 255.0) - 1.0 (float32, NCHW);
            init_latents = 0.18215 * vae.encode(image).latent_dist.sample();
            get_timesteps (0.11-0.14): init_timestep = min(int(n * strength), n),
            t_start = max(n - init_timestep, 0), timesteps = scheduler.timesteps[t_start:];
            latents = scheduler.add_noise(init_latents, z_0, timesteps[:1]); then the txt2img loop over
            the kept timesteps (the schedulers look their sigma / alpha up by timestep: index t_start + j).
  inpaint   prepare_mask_and_masked_image: image = uint8 / 127.5 - 1.0, mask = L-mode uint8 / 255.0
            binarised at 0.5, masked_image = image * (mask < 0.5); prepare_mask_latents: the mask
            F.interpolate'd (nearest) to the latent grid, masked_image_latents = 0.18215 *
            vae.encode(masked_image).latent_dist.sample(); latents = randn * init_noise_sigma; each step
            cat([scale_model_input(cat([latents] * 2), t), mask, masked_image_latents], dim=1).

The noise is pre-drawn as the engine's sampler reads it: noise [k + 1, B, C, h, w] (z_0, then step j's
z) and the posterior eps [B, C, h, w] of the one encoded image. Run it on deep copies of the models
carrying the reference's LoRA modules, in float64 or in the run's dtype.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import sample_ref as R


class RefEulerAncestral(R.RefEulerAncestral):
    def add_noise(self, original_samples, noise, timesteps):
        """original + noise * sigma[index of t], the sigmas cast to the samples' dtype."""
        sigmas = self.sigmas.to(device=original_samples.device, dtype=original_samples.dtype)
        schedule_timesteps = self.timesteps.to(original_samples.device)
        timesteps = timesteps.to(original_samples.device)
        step_indices = [(schedule_timesteps == t).nonzero().item() for t in timesteps]
        sigma = sigmas[step_indices].flatten()
        while len(sigma.shape) < len(original_samples.shape):
            sigma = sigma.unsqueeze(-1)
        return original_samples + noise * sigma


class RefDDIM(R.RefDDIM):
    def add_noise(self, original_samples, noise, timesteps):
        """sqrt(acp[t]) * original + sqrt(1 - acp[t]) * noise, acp cast to the samples' dtype."""
        alphas_cumprod = self.alphas_cumprod.to(device=original_samples.device, dtype=original_samples.dtype)
        timesteps = timesteps.to(original_samples.device)
        sqrt_alpha_prod = (alphas_cumprod[timesteps] ** 0.5).flatten()
        while len(sqrt_alpha_prod.shape) < len(original_samples.shape):
            sqrt_alpha_prod = sqrt_alpha_prod.unsqueeze(-1)
        sqrt_one_minus_alpha_prod = ((1 - alphas_cumprod[timesteps]) ** 0.5).flatten()
        while len(sqrt_one_minus_alpha_prod.shape) < len(original_samples.shape):
            sqrt_one_minus_alpha_prod = sqrt_one_minus_alpha_prod.unsqueeze(-1)
        return sqrt_alpha_prod * original_samples + sqrt_one_minus_alpha_prod * noise


def make_scheduler(name, prediction_type):
    return {"euler_ancestral": RefEulerAncestral, "ddim": RefDDIM}[name](prediction_type)


def get_timesteps(scheduler, num_inference_steps, strength):
    """(timesteps[t_start:], num_inference_steps - t_start), after scheduler.set_timesteps(n)."""
    init_timestep = min(int(num_inference_steps * strength), num_inference_steps)
    t_start = max(num_inference_steps - init_timestep, 0)
    timesteps = scheduler.timesteps[t_start:]
    return timesteps, num_inference_steps - t_start


def preprocess(image_u8):
    """The img2img pipeline's preprocess of uint8 [B, H, W, 3] images: float32 [B, 3, H, W]."""
    image = image_u8.cpu().numpy().astype(np.float32) / 255.0
    image = image.transpose(0, 3, 1, 2)
    image = 2.0 * image - 1.0
    return torch.from_numpy(np.ascontiguousarray(image))


def prepare_mask_and_masked_image(image_u8, mask_u8):
    """(mask float32 [B, 1, H, W] of 0 / 1, masked_image float32 [B, 3, H, W]) from uint8 [B, H, W, 3]
    images and uint8 [B, H, W] L-mode masks."""
    image = image_u8.cpu().numpy().transpose(0, 3, 1, 2)
    image = torch.from_numpy(np.ascontiguousarray(image)).to(dtype=torch.float32) / 127.5 - 1.0
    mask = mask_u8.cpu().numpy().astype(np.float32) / 255.0
    mask = mask[:, None]
    mask[mask < 0.5] = 0
    mask[mask >= 0.5] = 1
    mask = torch.from_numpy(mask)
    masked_image = image * (mask < 0.5)
    return mask, masked_image


def _posterior_sample(vae, x, eps, scaling):
    """scaling * vae.encode(x).latent_dist.sample() with the sample's eps given (in the VAE's dtype)."""
    dist = vae.encode(x).latent_dist
    return scaling * (dist.mean + dist.std * eps.to(dist.mean.dtype))


def _text(text_encoder, input_ids, negative_input_ids, cfg, ac):
    with ac:
        ehs = text_encoder(input_ids)[0]
        if cfg:
            ehs = torch.cat([text_encoder(negative_input_ids)[0], ehs])
    return ehs


def _autocast(autocast_dtype):
    return (torch.autocast("cuda", dtype=autocast_dtype) if autocast_dtype is not None
            else torch.autocast("cuda", enabled=False))


@torch.no_grad()
def sample_img2img(unet, text_encoder, vae, scheduler, n, strength, input_ids, negative_input_ids, image_u8, noise,
                   posterior_eps, guidance_scale, scaling=0.18215, dtype=torch.float64, autocast_dtype=None):
    """(uint8 images, final latents) of the img2img pipeline. noise: [k + 1, B, C, h, w] (z_0 for
    add_noise, then step j's z); posterior_eps [B, C, h, w]."""
    dev = noise.device
    scheduler.set_timesteps(n, device=dev)
    timesteps, k = get_timesteps(scheduler, n, strength)
    t_start = n - k
    cfg = guidance_scale > 1.0
    ac = _autocast(autocast_dtype)
    ehs = _text(text_encoder, input_ids, negative_input_ids, cfg, ac)
    vae_dtype = next(vae.parameters()).dtype
    image = preprocess(image_u8).to(device=dev, dtype=vae_dtype)
    init_latents = _posterior_sample(vae, image, posterior_eps, scaling).to(dtype)
    latents = scheduler.add_noise(init_latents, noise[0].to(dtype), timesteps[:1])
    for j, t in enumerate(timesteps):
        i = t_start + j
        inp = torch.cat([latents] * 2) if cfg else latents
        inp = scheduler.scale_model_input(inp, i)
        with ac:
            out = unet(inp.to(dtype), t.to(dev), ehs).sample
        if cfg:
            out_u, out_c = out.chunk(2)
            out = out_u + guidance_scale * (out_c - out_u)
        latents = scheduler.step(out.to(dtype), i, latents, noise[j + 1].to(dtype))
    image = vae.decode((1 / scaling * latents).to(vae_dtype)).sample
    return R.postprocess(image), latents


@torch.no_grad()
def sample_inpaint(unet, text_encoder, vae, scheduler, n, input_ids, negative_input_ids, image_u8, mask_u8, noise,
                   posterior_eps, guidance_scale, scaling=0.18215, dtype=torch.float64, autocast_dtype=None):
    """(uint8 images, final latents) of the inpainting pipeline on a UNet of 2C + 1 input channels.
    noise: [n + 1, B, C, h, w]; posterior_eps [B, C, h, w] of the masked image's encode."""
    dev = noise.device
    scheduler.set_timesteps(n, device=dev)
    cfg = guidance_scale > 1.0
    ac = _autocast(autocast_dtype)
    ehs = _text(text_encoder, input_ids, negative_input_ids, cfg, ac)
    vae_dtype = next(vae.parameters()).dtype
    mask, masked_image = prepare_mask_and_masked_image(image_u8, mask_u8)
    h, w = noise.shape[-2:]
    mask = F.interpolate(mask, size=(h, w)).to(device=dev, dtype=dtype)
    masked_image_latents = _posterior_sample(vae, masked_image.to(device=dev, dtype=vae_dtype), posterior_eps,
                                             scaling).to(dtype)
    if cfg:
        mask = torch.cat([mask] * 2)
        masked_image_latents = torch.cat([masked_image_latents] * 2)
    latents = noise[0].to(dtype) * scheduler.init_noise_sigma
    for i, t in enumerate(scheduler.timesteps):
        inp = torch.cat([latents] * 2) if cfg else latents
        inp = scheduler.scale_model_input(inp, i)
        inp = torch.cat([inp, mask, masked_image_latents], dim=1)
        with ac:
            out = unet(inp.to(dtype), t.to(dev), ehs).sample
        if cfg:
            out_u, out_c = out.chunk(2)
            out = out_u + guidance_scale * (out_c - out_u)
        latents = scheduler.step(out.to(dtype), i, latents, noise[i + 1].to(dtype))
    image = vae.decode((1 / scaling * latents).to(vae_dtype)).sample
    return R.postprocess(image), latents
