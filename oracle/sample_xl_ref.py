"""ORACLE (test infrastructure only -- never imported by the product path).

diffusers' StableDiffusionXLPipeline and StableDiffusionXLImg2ImgPipeline (requires_aesthetics_score=False,
SDXL base's setting) written eagerly, op by op, as the pipelines write them, never folded:

  RefEulerDiscrete   EulerDiscreteScheduler with the scheduler config SDXL base ships (scaled_linear,
                     timestep_spacing="leading", steps_offset=1, linear interpolation, s_churn = 0)
  encode_prompt_xl   both encoders' hidden_states[-2] concatenated, encoder 2's text_embeds pooled, and
                     with force_zeros_for_empty_prompt zeroed negatives when no negative prompt is given
  rescale_noise_cfg  the guidance rescale of "Common Diffusion Noise Schedules are Flawed", as diffusers
                     writes it
  sample             the txt2img / img2img loop: an encode function, added_cond_kwargs, any of the four
                     schedulers (sample_ref, sample_image_ref, sample_dpm_ref and RefEulerDiscrete) and
                     guidance_rescale, so it runs SD 1.x / 2.x with rescale as well as SDXL.

No copy of diffusers is installed to run against: this restates the pipelines' source. The noise is
pre-drawn as the engine's sampler reads it ([k + 1, B, C, h, w]: z_0, then step j's z; the posterior eps
[B, C, h, w] of an img2img encode). Run it on deep copies of the models carrying the reference's LoRA
modules, in float64 or in the run's dtype.
"""
import numpy as np
import torch

from . import sample_image_ref as RI
from . import sample_ref as R


class RefEulerDiscrete:
    """EulerDiscreteScheduler (SDXL base's config). `step` takes the step's index, as sample_ref's
    schedulers do."""

    def __init__(self, prediction_type="epsilon"):
        self.prediction_type = prediction_type
        self.alphas_cumprod = R._alphas_cumprod()

    def set_timesteps(self, n, device="cpu"):
        step_ratio = 1000 // n
        ts = (np.arange(0, n) * step_ratio).round()[::-1].copy().astype(np.float32)
        ts += 1                                                   # steps_offset
        sigmas = np.array(((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5)
        sigmas = np.interp(ts, np.arange(0, len(sigmas)), sigmas)
        sigmas = np.concatenate([sigmas, [0.0]]).astype(np.float32)
        self.sigmas = torch.from_numpy(sigmas).to(device=device)
        self.timesteps = torch.from_numpy(ts).to(device=device)
        self.init_noise_sigma = (self.sigmas.max() ** 2 + 1) ** 0.5     # "leading" spacing

    def scale_model_input(self, sample, i):
        sigma = self.sigmas[i]
        return sample / ((sigma ** 2 + 1) ** 0.5)

    def step(self, model_output, i, sample, noise=None):
        sigma = self.sigmas[i]
        gamma = 0.0                                              # s_churn = 0
        sigma_hat = sigma * (gamma + 1)
        if self.prediction_type == "epsilon":
            x0 = sample - sigma_hat * model_output
        else:
            x0 = model_output * (-sigma / (sigma ** 2 + 1) ** 0.5) + (sample / (sigma ** 2 + 1))
        derivative = (sample - x0) / sigma_hat
        dt = self.sigmas[i + 1] - sigma_hat
        return sample + derivative * dt

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


def make_scheduler(name, prediction_type):
    """The oracle scheduler of each engine scheduler name, with add_noise."""
    from .sample_dpm_ref import RefDPMSolverMultistep
    return {"euler_ancestral": RI.RefEulerAncestral, "ddim": RI.RefDDIM, "dpmsolver_multistep": RefDPMSolverMultistep,
            "euler": RefEulerDiscrete}[name](prediction_type)


def rescale_noise_cfg(noise_cfg, noise_pred_text, guidance_rescale=0.0):
    """Rescale `noise_cfg` according to `guidance_rescale` (section 3.4 of "Common Diffusion Noise
    Schedules are Flawed"), as diffusers writes it."""
    std_text = noise_pred_text.std(dim=list(range(1, noise_pred_text.ndim)), keepdim=True)
    std_cfg = noise_cfg.std(dim=list(range(1, noise_cfg.ndim)), keepdim=True)
    noise_pred_rescaled = noise_cfg * (std_text / std_cfg)
    noise_cfg = guidance_rescale * noise_pred_rescaled + (1 - guidance_rescale) * noise_cfg
    return noise_cfg


def encode_prompt_xl(text_encoder, text_encoder_2, input_ids, input_ids_2, negative_input_ids=None,
                     negative_input_ids_2=None, do_classifier_free_guidance=True, force_zeros_for_empty_prompt=True):
    """(prompt_embeds, pooled_prompt_embeds), [negative ; prompt] under guidance."""
    def enc(ids1, ids2):
        prompt_embeds_list = []
        pooled_prompt_embeds = None
        for ids, te in ((ids1, text_encoder), (ids2, text_encoder_2)):
            out = te(ids, output_hidden_states=True)
            if pooled_prompt_embeds is None and out[0].ndim == 2:
                pooled_prompt_embeds = out[0]
            prompt_embeds_list.append(out.hidden_states[-2])
        return torch.concat(prompt_embeds_list, dim=-1), pooled_prompt_embeds

    prompt_embeds, pooled_prompt_embeds = enc(input_ids, input_ids_2)
    if not do_classifier_free_guidance:
        return prompt_embeds, pooled_prompt_embeds
    zero_out_negative_prompt = negative_input_ids is None and force_zeros_for_empty_prompt
    if zero_out_negative_prompt:
        negative_prompt_embeds = torch.zeros_like(prompt_embeds)
        negative_pooled_prompt_embeds = torch.zeros_like(pooled_prompt_embeds)
    else:
        negative_prompt_embeds, negative_pooled_prompt_embeds = enc(negative_input_ids, negative_input_ids_2)
    return (torch.cat([negative_prompt_embeds, prompt_embeds], dim=0),
            torch.cat([negative_pooled_prompt_embeds, pooled_prompt_embeds], dim=0))


def add_time_ids(original_size, crops_coords_top_left, target_size, batch, cfg, dtype, device):
    """_get_add_time_ids, then cat([negative, positive]) under guidance and repeat over the batch."""
    ids = torch.tensor([list(original_size + crops_coords_top_left + target_size)], dtype=dtype)
    if cfg:
        ids = torch.cat([ids, ids], dim=0)
    return ids.to(device).repeat(batch, 1)


@torch.no_grad()
def sample(unet, vae, scheduler, n, encode, noise, guidance_scale, guidance_rescale=0.0, added_cond_kwargs=None,
           image_u8=None, strength=None, posterior_eps=None, scaling=0.13025, dtype=torch.float64,
           autocast_dtype=None, divide_by_scaling=True):
    """(uint8 images, final latents).

    encode() -> (encoder_hidden_states [G*B, ...], pooled or None) runs the text side under the loop's
    autocast, which it must not enter again (re-entering an active torch.autocast object leaves autocast
    on after the loop); pooled is None for SD, encode_prompt_xl's pooled embeddings for SDXL, passed to
    the UNet as added_cond_kwargs' text_embeds together with `added_cond_kwargs` -- SDXL's
    {"time_ids": ...}. img2img with image_u8,
    strength and posterior_eps. divide_by_scaling: the SDXL pipelines decode `latents / scaling`; the SD
    pipelines `1 / scaling * latents` (False)."""
    dev = noise.device
    scheduler.set_timesteps(n, device=dev)
    cfg = guidance_scale > 1.0
    ac = RI._autocast(autocast_dtype)
    with ac:
        ehs, pooled = encode()
    added = None
    if pooled is not None or added_cond_kwargs is not None:
        added = dict(added_cond_kwargs or {})
        if pooled is not None:
            added["text_embeds"] = pooled
    vae_dtype = next(vae.parameters()).dtype
    if image_u8 is None:
        timesteps, t_start = scheduler.timesteps, 0
        latents = noise[0].to(dtype) * scheduler.init_noise_sigma
    else:
        timesteps, k = RI.get_timesteps(scheduler, n, strength)
        t_start = n - k
        image = RI.preprocess(image_u8).to(device=dev, dtype=vae_dtype)
        init_latents = RI._posterior_sample(vae, image, posterior_eps, scaling).to(dtype)
        latents = scheduler.add_noise(init_latents, noise[0].to(dtype), timesteps[:1])
    for j, t in enumerate(timesteps):
        i = t_start + j
        inp = torch.cat([latents] * 2) if cfg else latents
        inp = scheduler.scale_model_input(inp, i)
        kw = {} if added is None else {"added_cond_kwargs": added}
        with ac:
            out = unet(inp.to(dtype), t.to(dev), ehs, **kw).sample
        if cfg:
            out_u, out_c = out.chunk(2)
            out = out_u + guidance_scale * (out_c - out_u)
            if guidance_rescale > 0.0:
                out = rescale_noise_cfg(out, out_c, guidance_rescale=guidance_rescale)
        latents = scheduler.step(out.to(dtype), i, latents, noise[j + 1].to(dtype))
    z = latents / scaling if divide_by_scaling else 1 / scaling * latents
    image = vae.decode(z.to(vae_dtype)).sample
    return R.postprocess(image), latents
