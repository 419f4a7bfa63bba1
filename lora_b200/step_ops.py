"""The two ends of a training step as single kernels (csrc/step_glue.cu):

  pixels_ingest     uint8 HWC images -> ToTensor + Normalize([0.5], [0.5]) -> the VAE's dtype,
                    channels_last (+ the inpainting masked image)   dataset.py:108-116
  step_prologue     scheduler.add_noise + cast to the model dtype + NCHW -> channels_last
                    (+ the 9-channel inpainting concat)   cli_lora_pti.py:295-313
                    (+ the v-prediction target scheduler.get_velocity, cli_lora_pti.py:333-338)
  step_prologue_posterior  the same with the VAE posterior sample in front
                    (latent_dist.sample() * 0.18215, train_lora_dreambooth.py:818-821,
                    cli_lora_pti.py:273-290)
  fused_masked_mse  (mask-weighted) MSE and its gradient w.r.t. the prediction in one pass
                    cli_lora_pti.py:340-370, train_lora_dreambooth.py:855-875

and the two ends of a sampling step (lora_b200/sample.py):

  sample_step       guidance sum + the scheduler's update (folded coefficients) + the next UNet input
                    and timestep (+ the decoder input on the last step); init=True: the first input
  sample_step_ch    the same into the 9-channel inpainting UNet's input (latent channels only)
  sample_step_ms    the same for a multistep scheduler (DPM-Solver++(2M)): the data prediction x0, the
                    update from it and the previous step's x0, and that history kept in a device buffer
  sample_init       the start of an img2img / inpainting loop: posterior sample, add_noise, the first
                    UNet input (+ the inpainting mask and masked-image latent channels)
  pixels_ingest_inpaint  uint8 image + 0..255 mask -> the inpainting pipeline's masked image
  pixels_emit       decoded image -> (x / 2 + 0.5).clamp(0, 1) -> uint8 HWC, diffusers' post-processing

and the latent cache of cli_lora_pti.py:141-151 (`cached_latents=True`): the VAE runs once per
image, training steps start from stored latents.
"""
from typing import List, Optional, Sequence

import torch

from . import _C, ops
from ._C import check, dtype_code, ptr, stream_ptr


def step_prologue(latents: torch.Tensor, noise: torch.Tensor, timesteps: torch.Tensor, noiser,
                  out_dtype: torch.dtype, inpaint_mask: Optional[torch.Tensor] = None,
                  masked_latents: Optional[torch.Tensor] = None, velocity: bool = False):
    """noisy (+ inpainting channels) as a channels_last [B, C', H, W] tensor of `out_dtype`.
    velocity=True: `(noisy, v)`, v = sqrt_acp[t] * noise - sqrt_one_minus_acp[t] * latents as an fp32
    NCHW tensor (the v-prediction target), written by the same launch."""
    if not latents.is_cuda:
        raise _C.LoraB200Error("step_prologue needs CUDA tensors (no CPU path)")
    B, C, H, W = latents.shape
    lat = latents.float().contiguous()
    eps = noise.float().contiguous()
    t = timesteps.to(torch.int64).contiguous()
    c_out = C if inpaint_mask is None else 2 * C + 1
    out = torch.empty((B, c_out, H, W), device=latents.device, dtype=out_dtype,
                      memory_format=torch.channels_last)
    im = None if inpaint_mask is None else inpaint_mask.float().contiguous()
    ml = None if masked_latents is None else masked_latents.float().contiguous()
    args = (ptr(lat), ptr(eps), ptr(t), ptr(noiser.sqrt_acp), ptr(noiser.sqrt_one_minus_acp),
            int(noiser.num_train_timesteps), ptr(im), ptr(ml), ptr(out), dtype_code(out_dtype))
    if velocity:
        v = torch.empty((B, C, H, W), device=latents.device, dtype=torch.float32)
        check(_C.lib.lb_step_prologue_v(*args, ptr(v), B, C, H, W, stream_ptr()), "lb_step_prologue_v")
    else:
        check(_C.lib.lb_step_prologue(*args, B, C, H, W, stream_ptr()), "lb_step_prologue")
    ops._count()
    return (out, v) if velocity else out


def _mask_arg(mask: Optional[torch.Tensor], shape):
    """(tensor, is_uint8) of a [B, 1, H, W] mask for the glue kernels: fp32 or uint8, contiguous."""
    if mask is None:
        return None, 0
    if tuple(mask.shape) != tuple(shape):
        raise _C.LoraB200Error(f"mask of shape {tuple(mask.shape)}, expected {tuple(shape)}")
    if mask.dtype == torch.uint8:
        return mask.contiguous(), 1
    return mask.float().contiguous(), 0


def pixels_ingest(pixels: torch.Tensor, out_dtype: torch.dtype, mask: Optional[torch.Tensor] = None,
                  channels_last: bool = True):
    """The VAE input from a batch of images, one launch: `(x, masked)`, [B, 3, H, W] tensors of
    `out_dtype` (channels_last or contiguous NCHW); masked is None without a mask.

    pixels: uint8 [B, H, W, 3] (decoded images, HWC) -> torchvision's ToTensor + Normalize([0.5], [0.5]),
    bit for bit; or fp32 [B, 3, H, W] already normalised (a cast). mask: fp32 or uint8 [B, 1, H, W]:
    masked = image * (mask < 0.5), the inpainting dataset's masked image (dataset.py:115)."""
    if not pixels.is_cuda:
        raise _C.LoraB200Error("pixels_ingest needs CUDA tensors (no CPU path)")
    if pixels.dtype == torch.uint8:
        if pixels.dim() != 4 or pixels.shape[3] != 3:
            raise _C.LoraB200Error(f"uint8 pixels must be [B, H, W, 3], got {tuple(pixels.shape)}")
        B, H, W, _ = pixels.shape
    elif pixels.dtype == torch.float32:
        if pixels.dim() != 4 or pixels.shape[1] != 3:
            raise _C.LoraB200Error(f"float32 pixels must be [B, 3, H, W], got {tuple(pixels.shape)}")
        B, _, H, W = pixels.shape
    else:
        raise _C.LoraB200Error(f"pixels must be uint8 or float32, got {pixels.dtype}")
    px = pixels.contiguous()
    m, m_u8 = _mask_arg(mask, (B, 1, H, W))
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    x = torch.empty((B, 3, H, W), device=pixels.device, dtype=out_dtype, memory_format=fmt)
    xm = None if m is None else torch.empty_like(x)
    check(_C.lib.lb_pixels_ingest(ptr(px), int(px.dtype == torch.uint8), ptr(m), m_u8, ptr(x), ptr(xm),
                                  dtype_code(out_dtype), int(channels_last), B, H, W, stream_ptr()),
          "lb_pixels_ingest")
    ops._count()
    return x, xm


def _moments_strides(moments: torch.Tensor):
    sb, sc, sh, sw = moments.stride()
    if sh != moments.shape[3] * sw:
        moments = moments.contiguous()
        sb, sc, sh, sw = moments.stride()
    return moments, (sb, sc, sw)


def step_prologue_posterior(moments: torch.Tensor, posterior_noise: torch.Tensor, noise: torch.Tensor,
                            timesteps: torch.Tensor, noiser, out_dtype: torch.dtype, latents: torch.Tensor,
                            scaling: float = 0.18215, masked_moments: Optional[torch.Tensor] = None,
                            masked_posterior_noise: Optional[torch.Tensor] = None,
                            mask: Optional[torch.Tensor] = None, masked_latents: Optional[torch.Tensor] = None,
                            inpaint_mask: Optional[torch.Tensor] = None, velocity: bool = False):
    """step_prologue with the VAE posterior sample in front, one launch.

    moments: `vae.encode(x).latent_dist.parameters` [B, 2C, h, w] (mean ; logvar) in the VAE's dtype;
    posterior_noise: [B, C, h, w] standard normal in that dtype or fp32. The latents
    `DiagonalGaussianDistribution(moments).sample() * scaling` (each op rounded as torch rounds it) are
    written to `latents` (fp32 [B, C, h, w], contiguous) and noised as step_prologue noises latents.
    Inpainting: mask [B, 1, 8h, 8w] (image resolution, fp32 or uint8), masked_moments and
    masked_posterior_noise give the masked-image latents; `masked_latents` ([B, C, h, w]) and
    `inpaint_mask` ([B, 1, h, w], the mask at (8i, 8j): F.interpolate(scale_factor=1/8)) are fp32
    outputs, and the UNet input is the 9-channel concat. Returns what step_prologue returns."""
    if not moments.is_cuda:
        raise _C.LoraB200Error("step_prologue_posterior needs CUDA tensors (no CPU path)")
    B, C2, H, W = moments.shape
    C = C2 // 2
    shape = (B, C, H, W)
    if C2 != 2 * C or tuple(posterior_noise.shape) != shape or tuple(latents.shape) != shape:
        raise _C.LoraB200Error(f"moments {tuple(moments.shape)}, posterior noise {tuple(posterior_noise.shape)}, "
                               f"latents {tuple(latents.shape)}: need [B, 2C, h, w] and two [B, C, h, w]")
    if latents.dtype != torch.float32 or not latents.is_contiguous():
        raise _C.LoraB200Error("latents must be a contiguous float32 tensor")
    mom, (sb, sc, sp) = _moments_strides(moments)
    pe = posterior_noise.contiguous()
    eps = noise.float().contiguous()
    t = timesteps.to(torch.int64).contiguous()
    m, m_u8 = _mask_arg(mask, (B, 1, 8 * H, 8 * W))
    mm = mpe = None
    if m is not None:
        if masked_moments is None or masked_posterior_noise is None or masked_latents is None or inpaint_mask is None:
            raise _C.LoraB200Error("inpainting needs masked_moments, masked_posterior_noise, masked_latents and "
                                   "inpaint_mask with the mask")
        if tuple(masked_moments.shape) != tuple(moments.shape) or masked_moments.dtype != moments.dtype:
            raise _C.LoraB200Error("masked_moments must have the shape and dtype of moments")
        if (tuple(masked_posterior_noise.shape) != shape or masked_posterior_noise.dtype != posterior_noise.dtype
                or tuple(masked_latents.shape) != shape or tuple(inpaint_mask.shape) != (B, 1, H, W)):
            raise _C.LoraB200Error("masked posterior noise / masked_latents [B, C, h, w], inpaint_mask [B, 1, h, w]")
        for o in (masked_latents, inpaint_mask):
            if o.dtype != torch.float32 or not o.is_contiguous():
                raise _C.LoraB200Error("masked_latents and inpaint_mask must be contiguous float32 tensors")
        mm = masked_moments
        if mm.stride() != mom.stride():          # one stride set serves both (two outputs of one VAE agree)
            mom, mm = mom.contiguous(), mm.contiguous()
            sb, sc, _, sp = mom.stride()
        mpe = masked_posterior_noise.contiguous()
    c_out = C if m is None else 2 * C + 1
    out = torch.empty((B, c_out, H, W), device=moments.device, dtype=out_dtype, memory_format=torch.channels_last)
    v = torch.empty(shape, device=moments.device, dtype=torch.float32) if velocity else None
    check(_C.lib.lb_step_prologue_posterior(
        ptr(mom), dtype_code(mom.dtype), sb, sc, sp, ptr(pe), dtype_code(pe.dtype), float(scaling), ptr(latents),
        ptr(mm), ptr(mpe), ptr(m), m_u8, ptr(masked_latents if m is not None else None),
        ptr(inpaint_mask if m is not None else None), ptr(eps), ptr(t), ptr(noiser.sqrt_acp),
        ptr(noiser.sqrt_one_minus_acp), int(noiser.num_train_timesteps), ptr(out), dtype_code(out_dtype), ptr(v),
        B, C, H, W, stream_ptr()), "lb_step_prologue_posterior")
    ops._count()
    return (out, v) if velocity else out


def _dense_hw_strides(t: torch.Tensor, what: str):
    """(stride_b, stride_c, stride_p) of a [N, C, H, W] tensor dense in (H, W) (NCHW or channels_last)."""
    sb, sc, sh, sw = t.stride()
    if sh != t.shape[3] * sw:
        raise _C.LoraB200Error(f"{what} must be dense in (H, W) (contiguous or channels_last), strides {t.stride()}")
    return sb, sc, sw


def _sample_step_args(model_out, x, noise, table, guidance, step_index, counter, unet_in, timestep, vae_in,
                      vae_scaling, init, unet_channels, what, x0_hist=None):
    """The argument tuple of lb_sample_step / lb_sample_step_ch after sample_step's checks (unet_in has
    `unet_channels` channels). With x0_hist (lb_sample_step_ms) the history takes the noise's place."""
    if not x.is_cuda:
        raise _C.LoraB200Error(f"{what} needs CUDA tensors (no CPU path)")
    if not vae_scaling > 0.0:
        raise _C.LoraB200Error(f"{what}: vae_scaling must be positive, got {vae_scaling}")
    B, C, H, W = x.shape
    Cu = C if unet_channels is None else unet_channels
    G = unet_in.shape[0] // B
    if x.dtype != torch.float32 or not x.is_contiguous():
        raise _C.LoraB200Error(f"{what}: x must be a contiguous float32 tensor")
    if (tuple(unet_in.shape) != (G * B, Cu, H, W) or unet_in.shape[0] % B
            or not unet_in.is_contiguous(memory_format=torch.channels_last)):
        raise _C.LoraB200Error(f"{what}: unet_in must be a channels_last [G*B, {Cu}, {H}, {W}] tensor, "
                               f"got {tuple(unet_in.shape)}")
    if table.dtype != torch.float32 or table.dim() != 2 or table.shape[1] != 8 or not table.is_contiguous():
        raise _C.LoraB200Error(f"{what}: table must be fp32 [rows, 8]" +
                               ("" if x0_hist is not None else " and noise fp32 [rows, B, C, H, W]"))
    if x0_hist is not None:
        if x0_hist.dtype != torch.float32 or tuple(x0_hist.shape) != (B, C, H, W) or not x0_hist.is_contiguous():
            raise _C.LoraB200Error(f"{what}: x0_hist must be a contiguous fp32 [{B}, {C}, {H}, {W}] tensor")
        noise = x0_hist
    elif noise.dtype != torch.float32 or tuple(noise.shape) != (table.shape[0], B, C, H, W) or not noise.is_contiguous():
        raise _C.LoraB200Error(f"{what}: table must be fp32 [rows, 8] and noise fp32 [rows, B, C, H, W]")
    if step_index.dtype != torch.int32 or counter.dtype != torch.int32 or timestep.dtype != torch.float32:
        raise _C.LoraB200Error(f"{what}: step_index / counter int32 [1], timestep fp32 [1]")
    sb = sc = sp = 0
    mdt = vdt = _C.LB_F32
    vcl = 0
    if not init:
        if model_out is None or tuple(model_out.shape) != (G * B, C, H, W):
            raise _C.LoraB200Error(f"{what}: model_out must be [{G * B}, {C}, {H}, {W}]")
        sb, sc, sp = _dense_hw_strides(model_out, "model_out")
        mdt = dtype_code(model_out.dtype)
        if vae_in is None or tuple(vae_in.shape) != (B, C, H, W):
            raise _C.LoraB200Error(f"{what}: vae_in must be [{B}, {C}, {H}, {W}]")
        vcl = int(not vae_in.is_contiguous())
        if vcl and not vae_in.is_contiguous(memory_format=torch.channels_last):
            raise _C.LoraB200Error(f"{what}: vae_in must be contiguous or channels_last")
        vdt = dtype_code(vae_in.dtype)
        if guidance is None or guidance.dtype != torch.float32:
            raise _C.LoraB200Error(f"{what}: guidance must be a float32 [1] tensor")
    head = (ptr(model_out), mdt, sb, sc, sp, G, ptr(x), ptr(noise), ptr(table), table.shape[0], ptr(guidance),
            ptr(step_index), ptr(counter), ptr(unet_in), dtype_code(unet_in.dtype))
    tail = (ptr(timestep), ptr(vae_in), vdt, vcl, 1.0 / float(vae_scaling), B, C, H, W, int(init), stream_ptr())
    return head, tail


def sample_step(model_out: Optional[torch.Tensor], x: torch.Tensor, noise: torch.Tensor, table: torch.Tensor,
                guidance: Optional[torch.Tensor], step_index: torch.Tensor, counter: torch.Tensor,
                unet_in: torch.Tensor, timestep: torch.Tensor, vae_in: Optional[torch.Tensor],
                vae_scaling: float, init: bool = False):
    """One launch of lb_sample_step, in place on preallocated buffers (nothing is allocated: capturable).

    model_out: the UNet output [G*B, C, H, W] (G = 2: [uncond ; cond]) in any float dtype, dense in (H, W);
    x: fp32 contiguous latents [B, C, H, W]; noise: fp32 [rows, B, C, H, W] (slice 0 is z_0); table: fp32
    [rows, 8] (host/schedulers.pack_table); guidance: fp32 [1]; step_index: int32 [1]; counter: int32 [1]
    zero-initialised; unet_in: [G*B, C, H, W] channels_last in the UNet's dtype; timestep: fp32 [1];
    vae_in: [B, C, H, W] in the VAE's dtype, contiguous or channels_last, written on the last step as
    `1 / vae_scaling * x` (the pipeline's expression, the reciprocal rounded to fp32).
    init=True: x = z_0 * init_noise_sigma and the first UNet input and timestep; the index is reset."""
    head, tail = _sample_step_args(model_out, x, noise, table, guidance, step_index, counter, unet_in, timestep,
                                   vae_in, vae_scaling, init, None, "sample_step")
    check(_C.lib.lb_sample_step(*head, *tail), "lb_sample_step")
    ops._count()


def sample_step_ch(model_out: Optional[torch.Tensor], x: torch.Tensor, noise: torch.Tensor, table: torch.Tensor,
                   guidance: Optional[torch.Tensor], step_index: torch.Tensor, counter: torch.Tensor,
                   unet_in: torch.Tensor, timestep: torch.Tensor, vae_in: Optional[torch.Tensor],
                   vae_scaling: float, init: bool = False):
    """sample_step into a UNet input of more channels than the latents (lb_sample_step_ch): unet_in is a
    channels_last [G*B, C', H, W] tensor, C' >= C (the inpainting UNet's 2C + 1), and only its channels
    [0, C) are written."""
    Cu = unet_in.shape[1] if unet_in.dim() == 4 else -1
    if Cu < x.shape[1]:
        raise _C.LoraB200Error(f"sample_step_ch: unet_in has {Cu} channels, fewer than the latents' {x.shape[1]}")
    head, tail = _sample_step_args(model_out, x, noise, table, guidance, step_index, counter, unet_in, timestep,
                                   vae_in, vae_scaling, init, Cu, "sample_step_ch")
    check(_C.lib.lb_sample_step_ch(*head, Cu, *tail), "lb_sample_step_ch")
    ops._count()


def sample_step_ms(model_out: torch.Tensor, x: torch.Tensor, x0_hist: torch.Tensor, table: torch.Tensor,
                   guidance: torch.Tensor, step_index: torch.Tensor, counter: torch.Tensor, unet_in: torch.Tensor,
                   timestep: torch.Tensor, vae_in: torch.Tensor, vae_scaling: float):
    """One launch of lb_sample_step_ms, in place on preallocated buffers (nothing is allocated: capturable).

    The arguments of sample_step_ch with x0_hist (fp32 contiguous [B, C, H, W]) in place of noise and no
    init: the loop starts with sample_step(init=True) or sample_init. table rows are
    (a, b, d, s_next, t_next, last, p, q) (host/schedulers.pack_table for a multistep scheduler):
    x0 = p x + q m_hat, x = a x + b x0 + d x0_hist (x0_hist unread when d = 0), then x0_hist = x0.
    unet_in may have more channels than the latents; only channels [0, C) are written."""
    Cu = unet_in.shape[1] if unet_in.dim() == 4 else -1
    if Cu < x.shape[1]:
        raise _C.LoraB200Error(f"sample_step_ms: unet_in has {Cu} channels, fewer than the latents' {x.shape[1]}")
    if x0_hist is None:
        raise _C.LoraB200Error("sample_step_ms needs the x0_hist buffer")
    head, tail = _sample_step_args(model_out, x, None, table, guidance, step_index, counter, unet_in, timestep,
                                   vae_in, vae_scaling, False, Cu, "sample_step_ms", x0_hist=x0_hist)
    check(_C.lib.lb_sample_step_ms(*head, Cu, *tail[:-2], tail[-1]), "lb_sample_step_ms")   # no init argument
    ops._count()


def sample_step_rescale(model_out: torch.Tensor, x: torch.Tensor, noise: Optional[torch.Tensor],
                        x0_hist: Optional[torch.Tensor], table: torch.Tensor, guidance: torch.Tensor,
                        guidance_rescale: torch.Tensor, step_index: torch.Tensor, counter: torch.Tensor,
                        unet_in: torch.Tensor, timestep: torch.Tensor, vae_in: torch.Tensor, vae_scaling: float):
    """One launch of lb_sample_step_rescale, in place on preallocated buffers (nothing is allocated:
    capturable): a classifier-free-guided step (model_out [2B, C, H, W]) with guidance rescale.

    guidance_rescale: a device fp32 [1] holding phi. x0_hist None: sample_step_ch's single-step update,
    reading `noise`; x0_hist given: sample_step_ms's multistep update (noise unused, may be None).
    Per sample, m_hat = m_u + g (m_c - m_u) is scaled by phi * std(m_c) / std(m_hat) + (1 - phi) before
    the update (diffusers' rescale_noise_cfg); at phi = 0 the result equals sample_step_ch's /
    sample_step_ms's bit for bit."""
    Cu = unet_in.shape[1] if unet_in.dim() == 4 else -1
    if Cu < x.shape[1]:
        raise _C.LoraB200Error(f"sample_step_rescale: unet_in has {Cu} channels, fewer than the latents' "
                               f"{x.shape[1]}")
    if unet_in.shape[0] != 2 * x.shape[0]:
        raise _C.LoraB200Error("sample_step_rescale: guidance rescale needs classifier-free guidance (G = 2): "
                               f"unet_in has {unet_in.shape[0]} rows for {x.shape[0]} latents")
    if (guidance_rescale is None or guidance_rescale.dtype != torch.float32 or guidance_rescale.numel() != 1
            or guidance_rescale.device != x.device):
        raise _C.LoraB200Error("sample_step_rescale: guidance_rescale must be a float32 [1] tensor on x's device")
    head, tail = _sample_step_args(model_out, x, noise, table, guidance, step_index, counter, unet_in, timestep,
                                   vae_in, vae_scaling, False, Cu, "sample_step_rescale", x0_hist=x0_hist)
    # head[7] is the noise, or x0_hist in its place: split it into the two pointers; phi follows guidance
    pair = (ptr(None), head[7]) if x0_hist is not None else (head[7], ptr(None))
    head = head[:7] + pair + head[8:11] + (ptr(guidance_rescale),) + head[11:]
    check(_C.lib.lb_sample_step_rescale(*head, Cu, *tail[:-2], tail[-1]), "lb_sample_step_rescale")
    ops._count()


def sample_init(moments: Optional[torch.Tensor], posterior_noise: Optional[torch.Tensor], x: torch.Tensor,
                noise: torch.Tensor, table: torch.Tensor, step_index: torch.Tensor, counter: torch.Tensor,
                unet_in: torch.Tensor, timestep: torch.Tensor, scaling: float = 0.18215,
                mask: Optional[torch.Tensor] = None):
    """One launch of lb_sample_init, in place on preallocated buffers (nothing is allocated: capturable).

    moments: `vae.encode(image).latent_dist.parameters` [B, 2C, h, w] in the VAE's dtype (NCHW or
    channels_last) or None; posterior_noise: [B, C, h, w] standard normal in that dtype or fp32.
    Without mask (img2img): x = add_noise(latent_dist.sample() * scaling, z_0, t_start) from row 0 of the
    table (c_noise, s_start, t_start, c_lat); without moments: x = z_0 * c_noise. mask (inpainting): uint8
    [B, 8h, 8w], 0..255, the pipeline's mask image; moments are then the masked image's, x = z_0 * c_noise,
    and unet_in ([G*B, 2C + 1, h, w]) gets the binarised latent-grid mask in channel C and the masked
    image's latents in channels C+1..2C. The first UNet input s_start * x goes to channels [0, C) of every
    half; timestep, step_index and counter are set as lb_sample_step's init sets them."""
    if not x.is_cuda:
        raise _C.LoraB200Error("sample_init needs CUDA tensors (no CPU path)")
    B, C, H, W = x.shape
    if x.dtype != torch.float32 or not x.is_contiguous():
        raise _C.LoraB200Error("sample_init: x must be a contiguous float32 tensor")
    Cu = C if mask is None else 2 * C + 1
    G = unet_in.shape[0] // B
    if (tuple(unet_in.shape) != (G * B, Cu, H, W) or G not in (1, 2)
            or not unet_in.is_contiguous(memory_format=torch.channels_last)):
        raise _C.LoraB200Error(f"sample_init: unet_in must be a channels_last [G*B, {Cu}, {H}, {W}] tensor, "
                               f"got {tuple(unet_in.shape)}")
    if (table.dtype != torch.float32 or table.dim() != 2 or table.shape[1] != 8 or not table.is_contiguous()
            or noise.dtype != torch.float32 or tuple(noise.shape) != (table.shape[0], B, C, H, W)
            or not noise.is_contiguous()):
        raise _C.LoraB200Error("sample_init: table must be fp32 [rows, 8] and noise fp32 [rows, B, C, H, W]")
    if step_index.dtype != torch.int32 or counter.dtype != torch.int32 or timestep.dtype != torch.float32:
        raise _C.LoraB200Error("sample_init: step_index / counter int32 [1], timestep fp32 [1]")
    mom, sb, sc, sp, md, pe, ed = None, 0, 0, 0, _C.LB_F32, None, _C.LB_F32
    if moments is not None:
        if tuple(moments.shape) != (B, 2 * C, H, W):
            raise _C.LoraB200Error(f"sample_init: moments must be [{B}, {2 * C}, {H}, {W}], got {tuple(moments.shape)}")
        if posterior_noise is None or tuple(posterior_noise.shape) != (B, C, H, W):
            raise _C.LoraB200Error(f"sample_init: posterior_noise must be [{B}, {C}, {H}, {W}]")
        if posterior_noise.dtype not in (moments.dtype, torch.float32) or not posterior_noise.is_contiguous():
            raise _C.LoraB200Error("sample_init: posterior_noise must be contiguous, in the moments' dtype or fp32")
        mom, (sb, sc, sp) = _moments_strides(moments)
        md, pe, ed = dtype_code(mom.dtype), posterior_noise, dtype_code(posterior_noise.dtype)
    if mask is not None:
        if moments is None:
            raise _C.LoraB200Error("sample_init: the inpainting mask needs the masked image's moments")
        if mask.dtype != torch.uint8 or tuple(mask.shape) != (B, 8 * H, 8 * W) or not mask.is_contiguous():
            raise _C.LoraB200Error(f"sample_init: mask must be a contiguous uint8 [{B}, {8 * H}, {8 * W}] tensor")
    check(_C.lib.lb_sample_init(ptr(mom), md, sb, sc, sp, ptr(pe), ed, float(scaling), ptr(mask), ptr(noise),
                                ptr(table), table.shape[0], ptr(x), ptr(step_index), ptr(counter), ptr(unet_in),
                                dtype_code(unet_in.dtype), Cu, ptr(timestep), G, B, C, H, W, stream_ptr()),
          "lb_sample_init")
    ops._count()


def pixels_ingest_inpaint(pixels: torch.Tensor, mask: torch.Tensor, out_dtype: torch.dtype,
                          channels_last: bool = True) -> torch.Tensor:
    """The inpainting pipeline's masked image, one launch (lb_pixels_ingest_inpaint): [B, 3, H, W] of
    `out_dtype`, channels_last or contiguous NCHW, = image * (mask < 0.5) with image = uint8 / 127.5 - 1
    and mask = (uint8 / 255 >= 0.5) (prepare_mask_and_masked_image). pixels: uint8 [B, H, W, 3]; mask:
    uint8 [B, H, W], 0..255 -- not pixels_ingest's 0 / 1 training mask."""
    if not pixels.is_cuda:
        raise _C.LoraB200Error("pixels_ingest_inpaint needs CUDA tensors (no CPU path)")
    if pixels.dtype != torch.uint8 or pixels.dim() != 4 or pixels.shape[3] != 3:
        raise _C.LoraB200Error(f"pixels must be uint8 [B, H, W, 3], got {pixels.dtype} {tuple(pixels.shape)}")
    B, H, W, _ = pixels.shape
    if mask.dtype != torch.uint8 or tuple(mask.shape) != (B, H, W):
        raise _C.LoraB200Error(f"mask must be uint8 [{B}, {H}, {W}], got {mask.dtype} {tuple(mask.shape)}")
    px, m = pixels.contiguous(), mask.contiguous()
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    xm = torch.empty((B, 3, H, W), device=pixels.device, dtype=out_dtype, memory_format=fmt)
    check(_C.lib.lb_pixels_ingest_inpaint(ptr(px), ptr(m), ptr(xm), dtype_code(out_dtype), int(channels_last),
                                          B, H, W, stream_ptr()), "lb_pixels_ingest_inpaint")
    ops._count()
    return xm


def pixels_emit(image: torch.Tensor, out: torch.Tensor):
    """uint8 [B, H, W, 3] images from the decoder's [B, 3, H, W] output (fp32 / bf16 / fp16, contiguous or
    channels_last), into `out`: diffusers' `(image / 2 + 0.5).clamp(0, 1)` and numpy_to_pil's
    `(x.float() * 255).round().astype(uint8)`, bit for bit, one launch."""
    if not image.is_cuda:
        raise _C.LoraB200Error("pixels_emit needs CUDA tensors (no CPU path)")
    if image.dim() != 4 or image.shape[1] != 3:
        raise _C.LoraB200Error(f"pixels_emit: image must be [B, 3, H, W], got {tuple(image.shape)}")
    B, _, H, W = image.shape
    if out.dtype != torch.uint8 or tuple(out.shape) != (B, H, W, 3) or not out.is_contiguous():
        raise _C.LoraB200Error(f"pixels_emit: out must be a contiguous uint8 [{B}, {H}, {W}, 3] tensor")
    cl = not image.is_contiguous()
    if cl and not image.is_contiguous(memory_format=torch.channels_last):
        raise _C.LoraB200Error("pixels_emit: image must be contiguous or channels_last")
    check(_C.lib.lb_pixels_emit(ptr(image), dtype_code(image.dtype), int(cl), ptr(out), B, H, W, stream_ptr()),
          "lb_pixels_emit")
    ops._count()
    return out


class _MaskedMSE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target, mask, weights, scratch, grad_scale):
        B, C, H, W = pred.shape
        if not pred.is_cuda:
            raise _C.LoraB200Error("fused_masked_mse needs CUDA tensors (no CPU path)")
        if not (pred.is_contiguous() or pred.is_contiguous(memory_format=torch.channels_last)):
            pred = pred.contiguous()
        grad = torch.empty_like(pred)          # same strides (contiguous or channels_last)
        sb, sc, sh, sw = pred.stride()
        assert sh == W * sw, "prediction must be dense in (H, W)"
        loss = torch.empty((), device=pred.device, dtype=torch.float32)
        tgt = target.float().contiguous()
        m = None if mask is None else mask.float().contiguous()
        w = None if weights is None else weights.float().contiguous()
        partials, counter = scratch
        check(_C.lib.lb_masked_mse_fwd_bwd(ptr(pred), dtype_code(pred.dtype), sb, sc, sw, ptr(tgt), ptr(m), ptr(w),
                                           ptr(grad), ptr(loss), ptr(partials), ptr(counter), B, C, H, W,
                                           ptr(grad_scale), stream_ptr()), "lb_masked_mse_fwd_bwd")
        ops._count()
        ctx.save_for_backward(grad)
        return loss

    @staticmethod
    def backward(ctx, gl):
        (grad,) = ctx.saved_tensors
        return grad * gl.to(grad.dtype), None, None, None, None, None


_SCRATCH = {}


def _scratch(device):
    s = _SCRATCH.get(device)
    if s is None:
        s = (torch.zeros(64, device=device, dtype=torch.float32), torch.zeros(1, device=device, dtype=torch.int32))
        _SCRATCH[device] = s
    return s


def fused_masked_mse(pred: torch.Tensor, target: torch.Tensor, mask: Optional[torch.Tensor] = None,
                     weights: Optional[torch.Tensor] = None, grad_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """sum_b weights[b] * mean_{c,h,w}((mask (pred - target))^2)  (weights None: 1/B), differentiable
    w.r.t. pred; mask [B,1,H,W] is the already-normalised weighting of cli_lora_pti.py:356-364.
    grad_scale: a device fp32 [1] loss scale (LoraArena.loss_scale) or None. The returned loss is
    unscaled; its backward seeds `grad_scale * d loss / d pred` (GradScaler.scale(loss).backward())."""
    if grad_scale is not None and (grad_scale.dtype != torch.float32 or grad_scale.numel() != 1
                                   or grad_scale.device != pred.device):
        raise _C.LoraB200Error("fused_masked_mse: grad_scale must be a one-element float32 tensor on pred's device")
    return _MaskedMSE.apply(pred, target, mask, weights, _scratch(pred.device), grad_scale)


class LatentCache:
    """cli_lora_pti.py:141-151 (`cached_latents=True`): encode every training image ONCE with the
    frozen VAE (`vae.encode(x).latent_dist.sample() * 0.18215`) and train from the stored latents.
    `vae` is anything with diffusers' AutoencoderKL encode interface; latents are kept on `device`
    (SD1.5 at 512x512: 64 KB per image -- a million images fit in 64 GB of the 180 GB HBM) or, with
    pin_host=True, in pinned host memory for step_host()."""

    def __init__(self, scaling: float = 0.18215, pin_host: bool = False):
        self.scaling, self.pin_host = scaling, pin_host
        self.items: List[dict] = []

    @torch.no_grad()
    def build(self, vae, dataset: Sequence[dict], image_key: str = "instance_images"):
        dev = next(vae.parameters()).device
        dt = next(vae.parameters()).dtype
        for idx in range(len(dataset)):
            batch = dict(dataset[idx])
            x = batch[image_key].unsqueeze(0).to(device=dev, dtype=dt)
            lat = vae.encode(x).latent_dist.sample() * self.scaling
            lat = lat.squeeze(0).float()
            batch[image_key] = lat.cpu().pin_memory() if self.pin_host else lat
            self.items.append(batch)
        return self

    def __len__(self):
        return len(self.items)

    def __getitem__(self, i):
        return self.items[i]
