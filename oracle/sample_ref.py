"""ORACLE (test infrastructure only -- never imported by the product path).

The sampling loop of diffusers' StableDiffusionPipeline (releases 0.11-0.14) written eagerly, op by op,
as the pipeline and its schedulers write it: randn * init_noise_sigma, then per step
scale_model_input, the UNet on cat([latents] * 2), chunk(2), the guidance sum and scheduler.step (not
folded coefficients); then 1 / scaling * latents, vae.decode and the post-processing. The noise is taken
pre-drawn ([N + 1, B, C, h, w]: z_0, then each step's z_i), the same draws the engine's sampler reads.
Run it on deep copies of the models carrying the reference's LoRA modules (oracle/ref_modules.py), in
float64 or in the run's dtype.
"""
import numpy as np
import torch


def _alphas_cumprod():
    betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


class RefEulerAncestral:
    """EulerAncestralDiscreteScheduler (scaled_linear, 1000 steps)."""

    def __init__(self, prediction_type="epsilon"):
        self.prediction_type = prediction_type
        self.alphas_cumprod = _alphas_cumprod()

    def set_timesteps(self, n, device="cpu"):
        ts = np.linspace(0, 999, n, dtype=float)[::-1].copy()
        sigmas = np.array(((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5)
        sigmas = np.interp(ts, np.arange(0, len(sigmas)), sigmas)
        sigmas = np.concatenate([sigmas, [0.0]]).astype(np.float32)
        self.sigmas = torch.from_numpy(sigmas).to(device=device)
        self.timesteps = torch.from_numpy(ts).to(device=device)
        self.init_noise_sigma = self.sigmas.max()

    def scale_model_input(self, sample, i):
        sigma = self.sigmas[i]
        return sample / ((sigma ** 2 + 1) ** 0.5)

    def step(self, model_output, i, sample, noise):
        sigma = self.sigmas[i]
        if self.prediction_type == "epsilon":
            x0 = sample - sigma * model_output
        else:
            x0 = model_output * (-sigma / (sigma ** 2 + 1) ** 0.5) + (sample / (sigma ** 2 + 1))
        sigma_from, sigma_to = self.sigmas[i], self.sigmas[i + 1]
        sigma_up = (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5
        sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
        derivative = (sample - x0) / sigma
        dt = sigma_down - sigma
        prev = sample + derivative * dt
        return prev + noise * sigma_up


class RefDDIM:
    """DDIMScheduler with Stable Diffusion's config (steps_offset=1, set_alpha_to_one=False,
    clip_sample=False), eta = 0."""

    def __init__(self, prediction_type="epsilon"):
        self.prediction_type = prediction_type
        self.alphas_cumprod = _alphas_cumprod()
        self.final_alpha_cumprod = self.alphas_cumprod[0]
        self.init_noise_sigma = 1.0

    def set_timesteps(self, n, device="cpu"):
        self.n = n
        ratio = 1000 // n
        ts = (np.arange(0, n) * ratio).round()[::-1].copy().astype(np.int64) + 1
        self.timesteps = torch.from_numpy(ts).to(device)

    def scale_model_input(self, sample, i):
        return sample

    def step(self, model_output, i, sample, noise=None):
        t = int(self.timesteps[i])
        prev_t = t - 1000 // self.n
        a = self.alphas_cumprod[t]
        a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        b = 1 - a
        if self.prediction_type == "epsilon":
            x0 = (sample - b ** 0.5 * model_output) / a ** 0.5
            eps = model_output
        else:
            x0 = (a ** 0.5) * sample - (b ** 0.5) * model_output
            eps = (a ** 0.5) * model_output + (b ** 0.5) * sample
        direction = (1 - a_prev) ** 0.5 * eps
        return a_prev ** 0.5 * x0 + direction


def make_scheduler(name, prediction_type):
    return {"euler_ancestral": RefEulerAncestral, "ddim": RefDDIM}[name](prediction_type)


def postprocess(image):
    """(image / 2 + 0.5).clamp(0, 1), then numpy_to_pil's (x.float() * 255).round() as uint8 [B, H, W, 3]."""
    image = (image / 2 + 0.5).clamp(0, 1)
    return (image.float() * 255).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous()


@torch.no_grad()
def sample(unet, text_encoder, vae, scheduler, n, input_ids, negative_input_ids, noise, guidance_scale,
           scaling=0.18215, dtype=torch.float64, autocast_dtype=None):
    """(uint8 images, final latents). dtype: the latents' / models' dtype (float64 for the exact run);
    autocast_dtype: run the text encoder and UNet under torch.autocast (the engine's bf16 runs)."""
    dev = noise.device
    scheduler.set_timesteps(n, device=dev)
    cfg = guidance_scale > 1.0
    ac = (torch.autocast("cuda", dtype=autocast_dtype) if autocast_dtype is not None
          else torch.autocast("cuda", enabled=False))
    with ac:
        ehs = text_encoder(input_ids)[0]
        if cfg:
            ehs = torch.cat([text_encoder(negative_input_ids)[0], ehs])
    latents = noise[0].to(dtype) * scheduler.init_noise_sigma
    for i, t in enumerate(scheduler.timesteps):
        inp = torch.cat([latents] * 2) if cfg else latents
        inp = scheduler.scale_model_input(inp, i)
        with ac:
            out = unet(inp.to(dtype), t.to(dev), ehs).sample
        if cfg:
            out_u, out_c = out.chunk(2)
            out = out_u + guidance_scale * (out_c - out_u)
        latents = scheduler.step(out.to(dtype), i, latents, noise[i + 1].to(dtype))
    vae_dtype = next(vae.parameters()).dtype
    image = vae.decode((1 / scaling * latents).to(vae_dtype)).sample
    return postprocess(image), latents
