"""Sampling from LoRA-patched models: the denoising loop of diffusers' StableDiffusionPipeline
(classifier-free guidance, Euler-ancestral, DDIM or DPM-Solver++(2M), the VAE decode and the uint8
post-processing) over the same host models and fused LoRA kernels the training steps use.

    from lora_b200.sample import LoraSampler, SamplerConfig
    s = LoraSampler(unet, text_encoder, vae, SamplerConfig(scheduler="euler_ancestral", guidance_scale=7.0),
                    latent_shape=(B, 4, 64, 64), seq_len=77)
    s.prepare()
    img = s.sample(input_ids, negative_input_ids, seed=0)   # uint8 [B, 8h, 8w, 3] on the device

img2img (StableDiffusionImg2ImgPipeline) and inpainting (StableDiffusionInpaintPipeline on the
9-channel UNet) run through the same three graphs, with `SamplerConfig(task="img2img" | "inpaint")`:

    s = LoraSampler(unet, text_encoder, vae, SamplerConfig(task="img2img", strength=0.75), latent_shape=...)
    img = s.sample(input_ids, negative_input_ids, seed=0, image=init_u8)             # [B, 8h, 8w, 3] uint8
    s = LoraSampler(unet_9ch, text_encoder, vae, SamplerConfig(task="inpaint"), latent_shape=...)
    img = s.sample(input_ids, negative_input_ids, seed=0, image=init_u8, mask_image=mask_u8)  # [B, 8h, 8w]

Images and masks come at the sampler's resolution (8h x 8w; resizing is the caller's job) and are
copied into static buffers. The mask is the pipeline's: uint8 0..255, white (>= 128) repainted.

A `sample()` replays three CUDA graphs, with no host sync and no allocation between them:
  A  the sampled sites' down factors re-cast into the 16-bit operands graph B reads, the text encoder on
     [negative ; prompt] ids, and the init launch of lb_sample_step (x = z_0 * init_noise_sigma);
     img2img / inpaint: the image ingest (lb_pixels_ingest / lb_pixels_ingest_inpaint), the VAE encoder
     (torch, in the VAE's dtype and layout) and lb_sample_init in place of that init launch: the posterior
     sample, add_noise at the first kept timestep (img2img), the first UNet input, and for inpainting
     the mask and masked-image latent channels of the UNet input, which no later launch rewrites;
  B  one denoising step: the UNet at batch G*B, then lb_sample_step (guidance sum, the scheduler's update
     as folded coefficients, the next UNet input and timestep). Replayed N times: the step index lives
     on the device and the kernel advances it. img2img runs the last k = n - t_start steps of the
     n-step schedule (host/schedulers.t_start: int(n * strength) steps), so B is replayed k times.
     A multistep scheduler (DPM-Solver++(2M), "dpmsolver_multistep") runs lb_sample_step_ms in place of
     lb_sample_step: it also keeps the previous step's data prediction in the static `x0_hist`;
  C  the VAE decoder and lb_pixels_emit.
`use_cuda_graph=False` runs the same code eagerly. The number of steps (up to `max_steps`), the
scheduler, the guidance scale, the seed, the strength, the image and the mask may change per call:
they rewrite device tables and buffers. A guidance
scale <= 1 runs without the unconditional half (G = 1), as the pipeline does; that is a capture of its own.
So is each scheduler family (schedulers.family: "single-step" for Euler-ancestral, Euler and DDIM,
"multistep" for DPM-Solver++): switching between Euler-ancestral and DDIM costs no capture, the first call
of the other family one, and later calls none. Guidance rescale (`guidance_rescale` phi > 0 with
guidance; diffusers' rescale_noise_cfg) runs lb_sample_step_rescale in place of the step launch, in either
family: a capture of its own, while phi itself is a device scalar and changes per call. LoraXLSampler
(below) samples SDXL.
The graphs are captured again only when something baked into a launch changes: a site's scale, a
selector, the set of sites or their parameter storage, the grouping policy (`captures` counts them).

Per-image LoRA coefficients: `sample(..., lora_scale={"unet": [..B], "text_encoder": 0.5},
lora_diag={"unet": rows_BxR})` (model names as save_safeloras writes them; LoraXLSampler also takes
"text_encoder_2") runs per-sample graphs, a capture key of their own: every sampled site reads its
[B, r] coefficients (per_sample.py) from one static device table that the call rewrites before graph A,
so they depend on the sites, ranks, factor storage and grouping only -- new values, tune_lora_scale,
set_lora_diag and LoRAManager.tune between such calls cost no capture. `shared_noise=True` draws the
noise as batch 1 from `seed` and copies it to every image (a strength sweep with one seed as one call).

All noise (z_0 and each step's z_i) is one draw of [k + 1, B, C, h, w] from the sampler's own
torch.Generator seeded by `seed`, then (img2img / inpaint) the posterior noise [B, C, h, w] of the one
encoded image, in the VAE's dtype as DiagonalGaussianDistribution.sample draws it; the global CUDA RNG stream is never touched, so a training step's noise
is the same with or without sampling in between. The models run in eval() under no_grad and get their
train / eval modes back afterwards.
"""
import contextlib
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn as nn

from . import ops
from .host import schedulers
from .step_ops import (pixels_emit, pixels_ingest, pixels_ingest_inpaint, sample_init, sample_step, sample_step_ch,
                       sample_step_ms, sample_step_rescale)

_SITE_NAMES = ("LoraInjectedLinear", "LoraInjectedConv2d")


@dataclass
class SamplerConfig:
    scheduler: str = "euler_ancestral"         # "euler_ancestral" | "ddim" | "dpmsolver_multistep"
    num_inference_steps: int = 50
    guidance_scale: float = 7.5
    prediction_type: str = "epsilon"           # the UNet's: "epsilon" | "v_prediction" (SD 2.x 768-v)
    vae_scaling: float = 0.18215
    # torch.autocast dtype for the text encoder and the UNet (None: the models' own dtype); the VAE
    # always runs in its own dtype
    autocast_dtype: Optional[torch.dtype] = None
    max_steps: int = 50                        # capacity of the noise buffer and the coefficient table
    use_cuda_graph: bool = True
    # read the noise from `self.noise` ([max_steps + 1, B, C, h, w], caller-filled) instead of drawing it
    external_noise: bool = False
    graph_warmup: int = 2
    # "txt2img" | "img2img" (StableDiffusionImg2ImgPipeline) | "inpaint" (StableDiffusionInpaintPipeline,
    # a UNet of 2C + 1 input channels); with external_noise the caller fills `self.posterior_noise` too
    task: str = "txt2img"
    strength: float = 0.8                      # img2img: the part of the schedule run (the pipeline's default)
    # phi of rescale_noise_cfg ("Common Diffusion Noise Schedules are Flawed"), in [0, 1]; applied under
    # classifier-free guidance only (G = 2), by lb_sample_step_rescale; 0 runs the plain step launches
    guidance_rescale: float = 0.0


TASKS = ("txt2img", "img2img", "inpaint")


def _sites(*models):
    return [m for model in models for m in model.modules() if type(m).__name__ in _SITE_NAMES]


def _check_phi(phi: float) -> float:
    phi = float(phi)
    if not 0.0 <= phi <= 1.0:
        raise ValueError(f"guidance_rescale must be in [0, 1], got {phi}")
    return phi


class LoraSampler:
    _sdxl = False             # LoraXLSampler: the UNet takes the SDXL "text_time" conditioning

    def __init__(self, unet: nn.Module, text_encoder: nn.Module, vae: nn.Module, cfg: SamplerConfig,
                 latent_shape=(1, 4, 64, 64), seq_len: int = 77, device=None):
        schedulers.check(cfg.scheduler, cfg.prediction_type)
        ucfg = getattr(unet, "cfg", None) or getattr(unet, "config", None)
        if not self._sdxl and getattr(ucfg, "addition_embed_type", None) is not None:
            raise ValueError("LoraSampler does not sample SDXL UNets (addition_embed_type "
                             f"{ucfg.addition_embed_type!r}): sample them with LoraXLSampler")
        _check_phi(cfg.guidance_rescale)
        B, C, h, w = latent_shape
        if cfg.task not in TASKS:
            raise ValueError(f"unknown task {cfg.task!r}: one of {TASKS}")
        Cu = 2 * C + 1 if cfg.task == "inpaint" else C
        if getattr(ucfg, "in_channels", Cu) != Cu:
            if cfg.task == "inpaint":
                raise ValueError(f"task 'inpaint' needs a UNet of {Cu} input channels (latents, mask, masked-image "
                                 f"latents), this one takes {ucfg.in_channels}")
            raise ValueError(f"the UNet takes {ucfg.in_channels} input channels, the latents have {C}: inpainting "
                             "UNets are sampled with SamplerConfig(task='inpaint')")
        if cfg.task == "img2img":
            schedulers.t_start(cfg.num_inference_steps, cfg.strength)        # refuses strengths that run no step
        elif not 0.0 < cfg.strength <= 1.0:
            raise ValueError(f"strength must be in (0, 1], got {cfg.strength}")
        if not getattr(vae, "has_decoder", hasattr(vae, "decoder")):
            raise ValueError("the VAE has no decoder: build it with AutoencoderKL(cfg, with_decoder=True)")
        if cfg.num_inference_steps < 1 or cfg.max_steps < cfg.num_inference_steps:
            raise ValueError(f"need 1 <= num_inference_steps ({cfg.num_inference_steps}) <= max_steps "
                             f"({cfg.max_steps})")
        self.cfg = cfg
        self.unet, self.text_encoder, self.vae = unet, text_encoder, vae
        self.device = torch.device(device or "cuda")
        dev = self.device
        self.model_dtype = unet.dtype if hasattr(unet, "dtype") else next(unet.parameters()).dtype
        self.vae_dtype = next(vae.decoder.parameters()).dtype
        vae_cl = not vae.decoder.conv_in.weight.is_contiguous()
        rows = cfg.max_steps + 1
        # static I/O (graph-stable addresses)
        self.input_ids = torch.zeros((2 * B, seq_len), device=dev, dtype=torch.long)    # [negative ; prompt]
        self.noise = torch.zeros((rows, B, C, h, w), device=dev, dtype=torch.float32)
        self.latents = torch.zeros(latent_shape, device=dev, dtype=torch.float32)
        self.x0_hist = torch.zeros(latent_shape, device=dev, dtype=torch.float32)      # multistep: last x0
        self.table = torch.zeros((rows, schedulers.TABLE_COLS), device=dev, dtype=torch.float32)
        self.guidance = torch.zeros(1, device=dev, dtype=torch.float32)
        self.guidance_rescale = torch.zeros(1, device=dev, dtype=torch.float32)      # phi
        self.step_index = torch.zeros(1, device=dev, dtype=torch.int32)
        self._counter = torch.zeros(1, device=dev, dtype=torch.int32)
        self.timestep = torch.zeros(1, device=dev, dtype=torch.float32)
        self.unet_in = {G: torch.zeros((G * B, Cu, h, w), device=dev, dtype=self.model_dtype).contiguous(
            memory_format=torch.channels_last) for G in (1, 2)}
        self.vae_in = torch.zeros(latent_shape, device=dev, dtype=self.vae_dtype).contiguous(
            memory_format=torch.channels_last if vae_cl else torch.contiguous_format)
        self.image = torch.zeros((B, 8 * h, 8 * w, 3), device=dev, dtype=torch.uint8)
        self.generator = torch.Generator(device=dev)
        if cfg.task != "txt2img":
            self.vae_enc_cl = not vae.encoder.conv_in.weight.is_contiguous()
            self.pixels = torch.zeros((B, 8 * h, 8 * w, 3), device=dev, dtype=torch.uint8)
            self.posterior_noise = torch.zeros(latent_shape, device=dev, dtype=next(vae.encoder.parameters()).dtype)
        if cfg.task == "inpaint":
            self.mask_image = torch.zeros((B, 8 * h, 8 * w), device=dev, dtype=torch.uint8)
        self._ehs = {}
        self._table_key = None
        self._graphs = {}             # (G, scheduler family[, "rescale"]) -> (A, B, C)
        self._fingerprint = None
        self._ps_fingerprint = None   # the structural fingerprint the per-sample graphs were captured for
        self._ps_buf = None           # per-sample graphs: the static coefficient table (per_sample.py layout)
        self._factor_bufs = []
        self._conv_tables = {}        # ops.conv_tap_table's row tables of the conv sites' down factors
        self.captures = 0

    # ------------------------------------------------------------------ what a capture bakes in
    def _fingerprint_now(self, structural: bool = False):
        """Everything of the models that a captured launch holds as a constant or an address. The
        structural part (sites, ranks, factor storage, grouping) is all a per-sample graph depends on:
        it reads scales and selectors from the static coefficient table."""
        from .grouping import get_grouping
        sig = []
        for m in _sites(*self._lora_models()):
            base = m.linear if hasattr(m, "linear") else m.conv
            sel = getattr(m.selector, "weight", None)
            values = () if structural else (float(m.scale), id(sel), None if sel is None else sel.data_ptr())
            sig.append((id(m), m.r) + values + (
                id(m.lora_down.weight), m.lora_down.weight.data_ptr(), m.lora_down.weight.dtype,
                id(m.lora_up.weight), m.lora_up.weight.data_ptr(), m.lora_up.weight.dtype,
                id(base.weight), base.weight.data_ptr()))
        return get_grouping(), tuple(sig)

    def _collect_factor_buffers(self):
        """The 16-bit padded down-factor copies the sites' forward reads (modules._SiteState.down): held
        here so that the addresses graph B captured stay valid, and re-cast by `_refresh_factors`."""
        bufs = []
        for m in _sites(*self._lora_models()):
            if m.r > ops.MAX_RANK:        # rank chunks cast their factors inside every forward
                continue
            if type(m).__name__ == "LoraInjectedConv2d":      # its re-cast walks a row table: upload it now
                ops.conv_tap_table(m.lora_down.weight, self._conv_tables)
            for dt, (_, buf) in list(m._lb.down.items()):
                bufs.append((m, dt, buf))
        self._factor_bufs = bufs

    def _refresh_factors(self):
        """Re-cast every held down-factor copy from the factor's current value (an arena step, an
        in-place optimizer update and a `.data` edit all leave the fused forward's copy stale)."""
        for m, dt, buf in self._factor_bufs:
            a = m.lora_down.weight.detach()
            if type(m).__name__ == "LoraInjectedLinear":
                a = a if a.dtype == torch.float32 and a.is_contiguous() else a.float().contiguous()
                ops.cast_rows_pad16(a, a.shape[1], 1, m.r, a.shape[1], dt, out=buf)
            else:
                ops.conv_down16(a, dt, self._conv_tables, out=buf)

    def _lora_models(self):
        """The models whose LoRA sites the sampler covers (fingerprint, factor refresh, eval mode)."""
        return (self.unet, self.text_encoder)

    # ------------------------------------------------------------------ the three bodies
    def _autocast(self):
        dt = self.cfg.autocast_dtype
        return torch.autocast("cuda", dtype=dt) if dt is not None else torch.autocast("cuda", enabled=False)

    def _encode(self, G: int):
        """The conditioning of the G halves (under the autocast): [negative ; prompt] hidden states."""
        B = self.latents.shape[0]
        ids = self.input_ids if G == 2 else self.input_ids[B:]
        self._ehs[G] = self.text_encoder(ids)[0].to(self.model_dtype)

    def _unet(self, G: int):
        return self.unet(self.unet_in[G], self.timestep, self._ehs[G]).sample

    def _body_a(self, G: int):
        self._refresh_factors()
        with self._autocast():
            self._encode(G)
        task = self.cfg.task
        if task == "txt2img":
            sample_step(None, self.latents, self.noise, self.table, None, self.step_index, self._counter,
                        self.unet_in[G], self.timestep, None, self.cfg.vae_scaling, init=True)
            return
        enc_dtype = self.posterior_noise.dtype
        if task == "img2img":          # preprocess: 2 * (u8 / 255) - 1, equal to the ingest bit for bit
            x, _ = pixels_ingest(self.pixels, enc_dtype, channels_last=self.vae_enc_cl)
        else:                          # prepare_mask_and_masked_image
            x = pixels_ingest_inpaint(self.pixels, self.mask_image, enc_dtype, channels_last=self.vae_enc_cl)
        moments = self.vae.encode(x).latent_dist.parameters
        sample_init(moments, self.posterior_noise, self.latents, self.noise, self.table, self.step_index,
                    self._counter, self.unet_in[G], self.timestep, self.cfg.vae_scaling,
                    mask=self.mask_image if task == "inpaint" else None)

    def _body_b(self, G: int, family: str = "single-step", rescale: bool = False):
        with self._autocast():
            out = self._unet(G)
        if rescale:                   # G = 2, either family: lb_sample_step_rescale
            ms = family == "multistep"
            sample_step_rescale(out, self.latents, None if ms else self.noise, self.x0_hist if ms else None,
                                self.table, self.guidance, self.guidance_rescale, self.step_index, self._counter,
                                self.unet_in[G], self.timestep, self.vae_in, self.cfg.vae_scaling)
            return
        if family == "multistep":
            sample_step_ms(out, self.latents, self.x0_hist, self.table, self.guidance, self.step_index,
                           self._counter, self.unet_in[G], self.timestep, self.vae_in, self.cfg.vae_scaling)
            return
        step = sample_step_ch if self.cfg.task == "inpaint" else sample_step
        step(out, self.latents, self.noise, self.table, self.guidance, self.step_index, self._counter,
             self.unet_in[G], self.timestep, self.vae_in, self.cfg.vae_scaling)

    def _body_c(self):
        pixels_emit(self.vae.decode(self.vae_in).sample, self.image)

    def _run_eager(self, G: int, n: int, family: str = "single-step", rescale: bool = False):
        self._collect_factor_buffers()
        self._body_a(G)
        for _ in range(n):
            self._body_b(G, family, rescale)
        self._body_c()

    # ------------------------------------------------------------------ capture
    def _key(self, G: int, family: str, rescale: bool):
        """The capture key: guidance mode, scheduler family, and the rescale launch when it runs."""
        return (G, family) + (("rescale",) if rescale else ())

    def _capture(self, key):
        G, family, rescale = key[0], key[1], "rescale" in key[2:]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(max(1, self.cfg.graph_warmup)):
                self._run_eager(G, 1, family, rescale)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self._collect_factor_buffers()
        ga = torch.cuda.CUDAGraph()
        with torch.cuda.graph(ga):
            self._body_a(G)
        gb = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gb, pool=ga.pool()):
            self._body_b(G, family, rescale)
        gc = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gc, pool=ga.pool()):
            self._body_c()
        torch.cuda.synchronize()
        self._graphs[key] = (ga, gb, gc)
        self.captures += 1

    def _graphs_for(self, key):
        ps = "per_sample" in key
        fp = self._fingerprint_now(structural=ps)
        if fp != (self._ps_fingerprint if ps else self._fingerprint):
            for k in [k for k in self._graphs if ("per_sample" in k) == ps]:
                del self._graphs[k]
            if ps:
                self._ps_fingerprint = fp
            else:
                self._fingerprint = fp
        if key not in self._graphs:
            self._capture(key)
        return self._graphs[key]

    # ------------------------------------------------------------------ modes
    def _enter_eval(self):
        models = self._lora_models() + (self.vae,)
        saved = [(m, m.training) for model in models for m in model.modules()]
        for model in models:
            model.eval()
        return saved

    @staticmethod
    def _restore_modes(saved):
        for m, training in saved:
            m.training = training

    # ------------------------------------------------------------------ public API
    def _options(self, num_inference_steps, scheduler, guidance_scale, strength=None):
        """(n, scheduler, guidance, t_start) of a call."""
        cfg = self.cfg
        n = cfg.num_inference_steps if num_inference_steps is None else int(num_inference_steps)
        sched = cfg.scheduler if scheduler is None else scheduler
        g = cfg.guidance_scale if guidance_scale is None else float(guidance_scale)
        schedulers.check(sched, cfg.prediction_type)
        if not 1 <= n <= cfg.max_steps:
            raise ValueError(f"num_inference_steps {n}: need 1 <= n <= max_steps ({cfg.max_steps})")
        if strength is not None and cfg.task != "img2img":
            raise ValueError(f"strength applies to img2img only, not to task {cfg.task!r}")
        start = schedulers.t_start(n, cfg.strength if strength is None else float(strength)) \
            if cfg.task == "img2img" else 0
        return n, sched, g, start

    def _set_table(self, sched: str, n: int, start: int = 0):
        key = (sched, n, start)
        if key != self._table_key:
            self.table.copy_(schedulers.pack_table(sched, self.cfg.prediction_type, n, self.cfg.max_steps, start,
                                                   from_image=self.cfg.task == "img2img"))
            self._table_key = key

    def _set_images(self, image, mask_image):
        """Copy the call's image (and mask) into the static buffers, after checking them."""
        task = self.cfg.task
        if task == "txt2img":
            if image is not None or mask_image is not None:
                raise ValueError("task 'txt2img' takes no image or mask_image: use task 'img2img' or 'inpaint'")
            return
        if image is None or image.dtype != torch.uint8 or tuple(image.shape) != tuple(self.pixels.shape):
            raise ValueError(f"task {task!r} needs image: uint8 {tuple(self.pixels.shape)} (B, 8h, 8w, RGB) at the "
                             f"sampler's resolution, got "
                             f"{None if image is None else (image.dtype, tuple(image.shape))}")
        if task == "img2img":
            if mask_image is not None:
                raise ValueError("task 'img2img' takes no mask_image: use task 'inpaint'")
        elif (mask_image is None or mask_image.dtype != torch.uint8
              or tuple(mask_image.shape) != tuple(self.mask_image.shape)):
            raise ValueError(f"task 'inpaint' needs mask_image: uint8 {tuple(self.mask_image.shape)} (B, 8h, 8w, "
                             f"0..255), got {None if mask_image is None else (mask_image.dtype, tuple(mask_image.shape))}")
        self.pixels.copy_(image)
        if task == "inpaint":
            self.mask_image.copy_(mask_image)

    def prepare(self, guidance_scale: Optional[float] = None, guidance_rescale: Optional[float] = None):
        """Capture the graphs for the configured (or given) guidance scale and rescale ahead of the first
        sample()."""
        if not self.cfg.use_cuda_graph:
            return
        n, sched, g, start = self._options(None, None, guidance_scale)
        phi = _check_phi(self.cfg.guidance_rescale if guidance_rescale is None else guidance_rescale)
        G = 2 if g > 1.0 else 1
        saved = self._enter_eval()
        try:
            with torch.no_grad():
                self._set_table(sched, n, start)
                self._graphs_for(self._key(G, schedulers.family(sched), G == 2 and phi > 0.0))
        finally:
            self._restore_modes(saved)

    def sample(self, input_ids: torch.Tensor, negative_input_ids: Optional[torch.Tensor] = None, seed: int = 0,
               num_inference_steps: Optional[int] = None, scheduler: Optional[str] = None,
               guidance_scale: Optional[float] = None, image: Optional[torch.Tensor] = None,
               mask_image: Optional[torch.Tensor] = None, strength: Optional[float] = None,
               guidance_rescale: Optional[float] = None, lora_scale: Optional[dict] = None,
               lora_diag: Optional[dict] = None, shared_noise: bool = False) -> torch.Tensor:
        """uint8 [B, 8h, 8w, 3] images (a view of `self.image`, overwritten by the next call) for the token
        ids [B, seq_len] of the prompts and of the negative prompts (the empty prompt's ids for plain
        classifier-free guidance; unused when guidance_scale <= 1). `self.latents` holds the final latents.
        img2img: image uint8 [B, 8h, 8w, 3], strength in (0, 1] (default cfg.strength); inpaint: image and
        mask_image uint8 [B, 8h, 8w] (0..255, >= 128 repainted). guidance_rescale: phi in [0, 1] (default
        cfg.guidance_rescale), applied when guidance_scale > 1.
        lora_scale / lora_diag: per-image LoRA coefficients by model name ("unet", "text_encoder"; see
        _per_sample_plan); shared_noise: every image gets the noise of a batch-1 call with this seed."""
        plan = self._per_sample_plan(lora_scale, lora_diag)
        self._check_shared_noise(shared_noise)
        n, sched, g, start = self._options(num_inference_steps, scheduler, guidance_scale, strength)
        phi = _check_phi(self.cfg.guidance_rescale if guidance_rescale is None else guidance_rescale)
        G = 2 if g > 1.0 else 1
        B = self.latents.shape[0]
        if tuple(input_ids.shape) != tuple(self.input_ids[B:].shape):
            raise ValueError(f"input_ids of shape {tuple(input_ids.shape)}: the sampler takes "
                             f"{tuple(self.input_ids[B:].shape)}")
        if G == 2 and (negative_input_ids is None or tuple(negative_input_ids.shape) != tuple(input_ids.shape)):
            raise ValueError("guidance_scale > 1 needs negative_input_ids of the prompts' shape")
        self._set_images(image, mask_image)

        def write_ids():
            self.input_ids[B:].copy_(input_ids)
            if G == 2:
                self.input_ids[:B].copy_(negative_input_ids)

        return self._generate(n, sched, g, start, phi, seed, write_ids, plan, shared_noise)

    # ------------------------------------------------------------------ per-image LoRA coefficients
    def _model_names(self):
        """The sampled models by their save_safeloras names."""
        return {"unet": self.unet, "text_encoder": self.text_encoder}

    def _per_sample_plan(self, lora_scale, lora_diag):
        """None for a call without per-image coefficients; else {name: (scale [B] | None, diag [B, r] | None)},
        validated (ValueError): known model names, models with LoRA sites, B values per scale, diag rows
        [r] or [B, r] of the sites' one rank."""
        if lora_scale is None and lora_diag is None:
            return None
        from . import per_sample
        B = self.latents.shape[0]
        names = self._model_names()
        plan = {}
        for what, arg in (("lora_scale", lora_scale), ("lora_diag", lora_diag)):
            if arg is None:
                continue
            if not isinstance(arg, dict):
                raise ValueError(f"{what} maps model names ({', '.join(names)}) to values, got {type(arg).__name__}")
            for name in arg:
                if name not in names:
                    raise ValueError(f"{what}: unknown model {name!r}, one of {', '.join(names)}")
        for name, model in names.items():
            sc, dg = (lora_scale or {}).get(name), (lora_diag or {}).get(name)
            if sc is None and dg is None:
                continue
            sites = per_sample.sites_of(model)
            if not sites:
                raise ValueError(f"{name} has no LoRA sites to scale per image")
            try:
                plan[name] = per_sample.check_args(sites, sc, dg, B)
            except ValueError as e:
                raise ValueError(f"{name}: {e}") from None
        return plan

    def _check_shared_noise(self, shared_noise: bool):
        if shared_noise and self.cfg.external_noise:
            raise ValueError("shared_noise draws the noise from the seed: not with SamplerConfig(external_noise=True)")

    def _per_sample_tables(self, plan):
        """Write the call's coefficients into the static table (allocated for these sites on first
        use) and return (sites, per-site views): every sampled site is bound, those without
        per-image values take their current scale and selector."""
        from . import per_sample
        B = self.latents.shape[0]
        sites, parts = [], []
        for name, model in self._model_names().items():
            ms = per_sample.sites_of(model)
            sc, dg = plan.get(name, (None, None))
            sites += ms
            sel = per_sample.selector_diags(ms) if dg is None else {}     # one read of the selectors
            parts += [per_sample.site_rows(m, sc, dg, B, sel).reshape(-1) for m in ms]
        flat = torch.cat(parts) if parts else torch.zeros(0)
        if self._ps_buf is None or self._ps_buf.numel() != flat.numel():
            self._ps_buf = torch.empty(flat.numel(), device=self.device, dtype=torch.float32)
        self._ps_buf.copy_(flat)
        return sites, per_sample.table_views(self._ps_buf, sites, B)

    def _draw_noise(self, k: int, seed: int, shared: bool):
        """z_0 and the steps' noise (and the posterior noise) from the sampler's generator; shared: drawn
        once as batch 1, as a batch-1 call with this seed draws it, and copied to every image."""
        self.generator.manual_seed(int(seed))
        image_task = self.cfg.task != "txt2img"
        if not shared:
            self.noise[:k + 1].normal_(generator=self.generator)
            if image_task:
                self.posterior_noise.normal_(generator=self.generator)
            return
        one = torch.empty((k + 1, 1) + tuple(self.noise.shape[2:]), device=self.device, dtype=self.noise.dtype)
        one.normal_(generator=self.generator)
        self.noise[:k + 1].copy_(one.expand(-1, self.noise.shape[1], -1, -1, -1))
        if image_task:
            p1 = torch.empty((1,) + tuple(self.posterior_noise.shape[1:]), device=self.device,
                             dtype=self.posterior_noise.dtype)
            p1.normal_(generator=self.generator)
            self.posterior_noise.copy_(p1.expand_as(self.posterior_noise))

    def _generate(self, n: int, sched: str, g: float, start: int, phi: float, seed: int, write_inputs,
                  plan=None, shared_noise: bool = False):
        """The call's tables, scalars, inputs (write_inputs()) and noise, then the graphs (or the eager
        path): the part of sample() every sampler shares. plan (per-image LoRA coefficients): the
        per-sample graphs, with every sampled site bound to the static coefficient table."""
        from . import per_sample
        k = n - start
        G = 2 if g > 1.0 else 1
        rescale = G == 2 and phi > 0.0
        key = self._key(G, schedulers.family(sched), rescale) + (("per_sample",) if plan is not None else ())
        saved = self._enter_eval()
        try:
            with torch.no_grad():
                self._set_table(sched, n, start)
                self.guidance.fill_(g)
                if rescale:
                    self.guidance_rescale.fill_(phi)
                write_inputs()
                if not self.cfg.external_noise:
                    self._draw_noise(k, seed, shared_noise)
                binding = contextlib.nullcontext()
                if plan is not None:
                    sites, views = self._per_sample_tables(plan)
                    binding = per_sample.bound(sites, views, self.latents.shape[0])
                with binding:
                    if self.cfg.use_cuda_graph:
                        ga, gb, gc = self._graphs_for(key)
                        ga.replay()
                        for _ in range(k):
                            gb.replay()
                        gc.replay()
                    else:
                        self._run_eager(G, k, key[1], rescale)
        finally:
            self._restore_modes(saved)
        return self.image


def _int_ids(t: torch.Tensor, shape, what: str):
    if not isinstance(t, torch.Tensor) or tuple(t.shape) != tuple(shape):
        raise ValueError(f"{what} of shape {None if not isinstance(t, torch.Tensor) else tuple(t.shape)}: the "
                         f"sampler takes {tuple(shape)}")
    if t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool:
        raise ValueError(f"{what} must be integer token ids, got {t.dtype}")


def _pair(v, what: str):
    if v is None or len(v) != 2:
        raise ValueError(f"{what} must be a pair (height, width) or (top, left), got {v!r}")
    return float(v[0]), float(v[1])


class LoraXLSampler(LoraSampler):
    """Sampling from LoRA-patched SDXL models: the denoising loop of diffusers' StableDiffusionXLPipeline
    (txt2img) and StableDiffusionXLImg2ImgPipeline (img2img, requires_aesthetics_score=False) over the
    LoraSampler machinery -- the same three graphs, schedulers, step launches and per-call options.

        s = LoraXLSampler(unet, text_encoder, text_encoder_2, vae,
                          SamplerConfig(scheduler="euler", num_inference_steps=30, guidance_scale=5.0,
                                        vae_scaling=0.13025, autocast_dtype=torch.bfloat16),
                          latent_shape=(1, 4, 128, 128))
        img = s.sample(input_ids, input_ids_2, seed=0)        # uint8 [B, 1024, 1024, 3] on the device

    The conditioning is the pipeline's encode_prompt (LoraXLTrainStep._predict's): both encoders'
    penultimate hidden states concatenated ([G*B, 77, 2048]), encoder 2's text_embeds as the pooled
    conditioning, and `time_ids` [G*B, 6] fp32 (original size, crop top-left, target size) from a static
    buffer written per call, which costs no capture. With guidance and no negative ids the negative
    embeddings and pooled embeddings are zeros (force_zeros_for_empty_prompt, SDXL base's setting); with
    both negative id tensors they are encoded. Zeroed or encoded negatives is a capture key of its own, like
    the scheduler family and guidance rescale (`SamplerConfig.guidance_rescale` or sample(guidance_rescale=)).

    Refused before any CUDA call: a non-SDXL UNet, encoders that do not fit it, task "inpaint", and an
    fp16 VAE (SDXL's VAE overflows in fp16; diffusers upcasts it, this sampler asks for fp32 or bf16)."""
    _sdxl = True

    def __init__(self, unet: nn.Module, text_encoder: nn.Module, text_encoder_2: nn.Module, vae: nn.Module,
                 cfg: SamplerConfig, latent_shape=(1, 4, 128, 128), seq_len: int = 77, device=None):
        from .train import _check_xl_models
        ucfg = getattr(unet, "cfg", None) or getattr(unet, "config", None)
        if getattr(ucfg, "addition_embed_type", None) != "text_time":
            raise ValueError("LoraXLSampler samples SDXL UNets (addition_embed_type='text_time'); sample SD 1.x / "
                             "2.x UNets with LoraSampler")
        _check_xl_models(unet, text_encoder, text_encoder_2)
        if cfg.task == "inpaint":
            raise ValueError("LoraXLSampler does not inpaint: tasks 'txt2img' and 'img2img' only")
        if any(p.dtype == torch.float16 for p in vae.parameters()):
            raise ValueError("the SDXL VAE overflows in fp16 (diffusers' SDXL VAE config sets force_upcast): pass it "
                             "in fp32 or bf16")
        self.text_encoder_2 = text_encoder_2
        super().__init__(unet, text_encoder, vae, cfg, latent_shape=latent_shape, seq_len=seq_len, device=device)
        B, _, h, w = latent_shape
        dev = self.device
        self.input_ids_2 = torch.zeros((2 * B, seq_len), device=dev, dtype=torch.long)    # [negative ; prompt]
        self.time_ids = torch.tensor([[8.0 * h, 8.0 * w, 0.0, 0.0, 8.0 * h, 8.0 * w]] * (2 * B), device=dev,
                                     dtype=torch.float32)
        self._added = {}
        self._zero_negatives = True

    def _lora_models(self):
        return (self.unet, self.text_encoder, self.text_encoder_2)

    def _model_names(self):
        return {"unet": self.unet, "text_encoder": self.text_encoder, "text_encoder_2": self.text_encoder_2}

    def _key(self, G: int, family: str, rescale: bool):
        zeros = G == 2 and self._zero_negatives
        return super()._key(G, family, rescale) + (("zero_negatives",) if zeros else ())

    def _encode(self, G: int):
        B = self.latents.shape[0]
        zeros = G == 2 and self._zero_negatives
        lo = B if G == 1 or zeros else 0
        out1 = self.text_encoder(self.input_ids[lo:], output_hidden_states=True)
        out2 = self.text_encoder_2(self.input_ids_2[lo:], output_hidden_states=True)
        ehs = torch.cat([out1.hidden_states[-2], out2.hidden_states[-2]], dim=-1)
        pooled = out2.text_embeds
        if zeros:
            ehs = torch.cat([torch.zeros_like(ehs), ehs])
            pooled = torch.cat([torch.zeros_like(pooled), pooled])
        self._ehs[G] = ehs.to(self.model_dtype)
        self._added[G] = {"text_embeds": pooled, "time_ids": self.time_ids[(2 - G) * B:]}

    def _unet(self, G: int):
        return self.unet(self.unet_in[G], self.timestep, self._ehs[G], added_cond_kwargs=self._added[G]).sample

    def prepare(self, guidance_scale: Optional[float] = None, guidance_rescale: Optional[float] = None,
                encoded_negatives: bool = False):
        """LoraSampler.prepare, for zeroed (the default call's) or encoded negative prompts."""
        self._zero_negatives = not encoded_negatives
        super().prepare(guidance_scale, guidance_rescale)

    def sample(self, input_ids: torch.Tensor, input_ids_2: torch.Tensor,
               negative_input_ids: Optional[torch.Tensor] = None, negative_input_ids_2: Optional[torch.Tensor] = None,
               seed: int = 0, original_size=None, crops_coords_top_left=(0, 0), target_size=None,
               guidance_rescale: Optional[float] = None, num_inference_steps: Optional[int] = None,
               scheduler: Optional[str] = None, guidance_scale: Optional[float] = None,
               image: Optional[torch.Tensor] = None, strength: Optional[float] = None,
               lora_scale: Optional[dict] = None, lora_diag: Optional[dict] = None,
               shared_noise: bool = False) -> torch.Tensor:
        """uint8 [B, 8h, 8w, 3] images (a view of `self.image`) for the two tokenizers' ids [B, seq_len] of
        the prompts. The negative prompts' ids come as a pair or not at all (zeroed negatives).
        original_size and target_size default to (8h, 8w); with crops_coords_top_left they make each
        sample's time ids. img2img: image uint8 [B, 8h, 8w, 3] and strength, as LoraSampler.sample.
        lora_scale / lora_diag / shared_noise as LoraSampler.sample, with "text_encoder_2" a model name too."""
        plan = self._per_sample_plan(lora_scale, lora_diag)
        self._check_shared_noise(shared_noise)
        n, sched, g, start = self._options(num_inference_steps, scheduler, guidance_scale, strength)
        phi = _check_phi(self.cfg.guidance_rescale if guidance_rescale is None else guidance_rescale)
        G = 2 if g > 1.0 else 1
        B = self.latents.shape[0]
        shape = tuple(self.input_ids[B:].shape)
        _int_ids(input_ids, shape, "input_ids")
        _int_ids(input_ids_2, shape, "input_ids_2")
        if (negative_input_ids is None) != (negative_input_ids_2 is None):
            raise ValueError("give both negative_input_ids and negative_input_ids_2, or neither (zeroed negatives)")
        encoded = negative_input_ids is not None
        if encoded:
            _int_ids(negative_input_ids, shape, "negative_input_ids")
            _int_ids(negative_input_ids_2, shape, "negative_input_ids_2")
        _, _, h, w = self.latents.shape
        sizes = (_pair((8 * h, 8 * w) if original_size is None else original_size, "original_size")
                 + _pair(crops_coords_top_left, "crops_coords_top_left")
                 + _pair((8 * h, 8 * w) if target_size is None else target_size, "target_size"))
        self._set_images(image, None)
        self._zero_negatives = not encoded

        def write_inputs():
            self.input_ids[B:].copy_(input_ids)
            self.input_ids_2[B:].copy_(input_ids_2)
            if G == 2 and encoded:
                self.input_ids[:B].copy_(negative_input_ids)
                self.input_ids_2[:B].copy_(negative_input_ids_2)
            self.time_ids.copy_(torch.tensor(sizes, dtype=torch.float32).expand(2 * B, 6))

        return self._generate(n, sched, g, start, phi, seed, write_inputs, plan, shared_noise)
