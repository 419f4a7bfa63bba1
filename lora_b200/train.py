"""Training-step engine: the step loop of the reference's trainers, restated around the fused
LoRA path and captured as ONE CUDA graph.

Restates (diffusers / accelerate are not installed, so the scripts themselves cannot run):
  training_scripts/train_lora_dreambooth.py:811-888  -- Dreambooth step (noise, timestep,
      add_noise, text encoder, UNet, MSE, backward, clip_grad_norm_(1.0), AdamW, zero_grad)
  lora_diffusion/cli_lora_pti.py:260-370, 585-617     -- PTI LoRA-tuning phase (same step with
      t_mutliplier and mean([1,2,3]).mean() reduction)
Differences by design: LoRA factors/grads/moments live in a LoraArena, clip + AdamW + zero_grad
are one cooperative launch that also takes in the DDP all-reduce (peer reads over NVLink; one
NCCL call before it without peer access), and steady-state steps are CUDA-graph replays (no
Python, no launch gaps, no host sync).
"""
import contextlib
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .arena import LoraArena
from .host.ddpm import DDPMNoiser


@dataclass
class StepConfig:
    # defaults = training_scripts/train_lora_dreambooth.py:364-387 and run_lora_db_w_text.sh:6-20
    learning_rate: float = 1e-4
    learning_rate_text: float = 5e-5
    adam_beta1: float = 0.9
    adam_beta2: float = 0.999
    adam_weight_decay: float = 1e-2
    adam_epsilon: float = 1e-8
    max_grad_norm: float = 1.0
    train_text_encoder: bool = True
    t_multiplier: float = 1.0          # cli_lora_pti.py:598 uses 0.8 in the tuning phase
    compute_dtype: torch.dtype = torch.bfloat16
    use_cuda_graph: bool = True
    graph_warmup: int = 3
    # EXPERIMENTAL (not yet run on hardware): capture the NCCL all-reduce INSIDE one step graph,
    # with capture_error_mode="thread_local" so that the NCCL watchdog thread's event queries do
    # not collide with the capture (the suspected cause of the round-1 dead-lock with a globally
    # scoped capture). Saves the host gap between the two replays.
    capture_collective: bool = False
    # accelerate-style mixed precision (fp32 frozen weights + torch.autocast), the reference's
    # own configuration (train_lora_dreambooth.py:489-494). None: run in the models' own dtype.
    autocast_dtype: Optional[torch.dtype] = None
    # lr_scheduler: "constant" (train_lora_dreambooth.py default; ignores lr_warmup_steps like
    # diffusers' get_scheduler), "constant_with_warmup", or "linear" decay to 0 over
    # max_train_steps after lr_warmup_steps (cli_lora_pti.py:730-741 `lr_scheduler_lora="linear"`)
    lr_scheduler: str = "constant"
    lr_warmup_steps: int = 0
    max_train_steps: int = 1000
    # The two trainers advance the schedule at different points: train_lora_dreambooth.py:886 calls
    # lr_scheduler.step() AFTER optimizer.step() (iteration k, 0-based, runs at lambda(k));
    # cli_lora_pti.py:587 (perform_tuning) and :417 (train_inversion) call it FIRST (iteration k runs
    # at lambda(k + 1)). True selects the PTI order.
    lr_step_first: bool = False
    # PTI masked loss (cli_lora_pti.py:340-368): mask (latent resolution, in `self.mask`) ->
    # (mask + 0.01)^mask_temperature / max -> pred*mask, target*mask -> mse.mean([1,2,3]).mean()
    use_mask: bool = False
    mask_temperature: float = 1.0
    # inpainting variant (cli_lora_pti.py:279-313): the UNet (in_channels = 9) sees
    # cat([noisy latents, mask, masked-image latents], dim=1); both extra inputs are per-sample
    # data at latent resolution, in `self.inpaint_mask` / `self.masked_latents`
    train_inpainting: bool = False
    # Dreambooth prior preservation (train_lora_dreambooth.py:855-873): the batch is
    # [instance images ; class images]; loss = mse(instance).mean([1,2,3]).mean()
    # + prior_loss_weight * mse(class)
    with_prior_preservation: bool = False
    prior_loss_weight: float = 1.0
    # take the step's noise / timesteps from `self.noise` / `self.timesteps` (caller-filled static
    # buffers) instead of drawing them inside the step: lets a parity test or a replayed trace feed
    # the SAME draws to this engine and to the reference step, eager or graph-replayed
    external_noise: bool = False
    # the step's prologue (add_noise + cast + channels_last [+ inpainting concat]) and loss epilogue
    # ((masked) MSE + its gradient) as one kernel each (step_ops.py) instead of ~10 small torch ops
    fused_glue: bool = True
    # data parallel: run the gradient all-reduce INSIDE the optimizer launch over NVLink peer memory
    # (arena.enable_peer_allreduce / lb_optim_step_dp) -- no NCCL call on the step path, so the whole
    # step is ONE CUDA graph at any world size. False (or IPC unavailable): one NCCL all-reduce
    # between two graphs.
    peer_allreduce: bool = True
    # queue the dA / dB reductions of all linear sites (and the conv sites' dB) during backward and
    # run them in ceil(n/24) launches at its end (ops.wgrad_flush / lb_lora_wgrad_batch)
    defer_wgrad: bool = True
    # the regression target, as the reference's trainers read it from scheduler.config.prediction_type
    # (cli_lora_pti.py:333-338, train_lora_dreambooth.py:846-853): "epsilon" (SD 1.x, SD 2.x base)
    # regresses the noise, "v_prediction" (SD 2.x 768-v) the velocity
    # sqrt_acp[t] * noise - sqrt(1 - acp[t]) * latents
    prediction_type: str = "epsilon"
    # accelerate's `--mixed_precision fp16` (train_lora_dreambooth.py:409-414,489-494): fp16 autocast
    # plus torch.amp.GradScaler, run on the device -- the backward is seeded with the loss scale, and
    # the optimizer launch unscales, skips the update on an inf / NaN gradient, updates the scale and
    # advances the LR schedule only after an applied step (accelerate's step_was_skipped). Needs
    # autocast_dtype = compute_dtype = torch.float16. The constants are torch.amp.GradScaler's.
    grad_scaler: bool = False
    init_scale: float = 65536.0
    growth_factor: float = 2.0
    backoff_factor: float = 0.5
    growth_interval: int = 2000
    # `--gradient_checkpointing` (train_lora_dreambooth.py:627-630): unet.enable_gradient_checkpointing(),
    # and text_encoder.gradient_checkpointing_enable() when the text encoder runs with gradients. Every
    # ResnetBlock2D / Transformer2DModel / CLIP encoder layer drops its activations after the forward
    # and runs again in backward: less activation memory for one more forward. Gradients equal the
    # un-checkpointed ones (non-reentrant checkpointing; dropout masks survive the recompute).
    gradient_checkpointing: bool = False
    # train from images (train_lora_dreambooth.py:818-821; cli_lora_pti.py:273-290 with cached_latents=False):
    # the step's input is a batch of images (`self.pixels`, uint8 [B, 8h, 8w, 3] by default) that the frozen
    # VAE (LoraTrainStep's `vae=`) encodes inside the step, in its own dtype, and a NEW posterior sample
    # `latent_dist.sample() * vae_scaling` is drawn every step -- the trainers' behaviour, unlike
    # step_ops.LatentCache, which freezes one sample per image. With train_inpainting the masked image is
    # encoded too and the image-resolution mask (`self.pixel_mask`) is resized to the latent grid.
    encode_images: bool = False
    # the VAE's latent scaling: 0.18215 for SD 1.x / 2.x, 0.13025 for SDXL (same VAE architecture)
    vae_scaling: float = 0.18215
    # the posterior noise's dtype: False draws it in the VAE's dtype (current diffusers' randn_tensor),
    # True in fp32 (diffusers releases of the reference's era; std * eps then promotes to fp32)
    posterior_noise_fp32: bool = False
    # the image buffer's dtype: torch.uint8 (decoded images, [B, H, W, 3]) or torch.float32 (images already
    # normalised to [-1, 1] by a float loader, [B, 3, H, W])
    pixel_dtype: torch.dtype = torch.uint8


def _check_encode_images(cfg: StepConfig, vae):
    """StepConfig.encode_images needs a VAE; refused before any CUDA call."""
    if not cfg.encode_images:
        return
    if vae is None:
        raise ValueError("StepConfig.encode_images needs the frozen VAE: pass vae= (an AutoencoderKL)")
    if cfg.pixel_dtype not in (torch.uint8, torch.float32):
        raise ValueError(f"StepConfig.pixel_dtype must be torch.uint8 or torch.float32, got {cfg.pixel_dtype}")


def _enable_gradient_checkpointing(unet: nn.Module, text_encoder: nn.Module, text_grad: bool, *more_encoders):
    """train_lora_dreambooth.py:627-630. The step draws nothing from torch's generator inside a
    checkpointed segment (LoRA dropout seeds come from dropout_path's pool), and the generator state
    cannot be read while a CUDA graph is captured: CLIP's layers skip stashing it. SDXL's second text
    encoder comes in `more_encoders` and is checkpointed like the first."""
    unet.enable_gradient_checkpointing()
    if text_grad:
        for te in (text_encoder,) + more_encoders:
            te.gradient_checkpointing_enable(
                gradient_checkpointing_kwargs={"use_reentrant": False, "preserve_rng_state": False})


PREDICTION_TYPES = ("epsilon", "v_prediction")


def _check_prediction_type(cfg: StepConfig):
    if cfg.prediction_type not in PREDICTION_TYPES:
        raise ValueError(f"Unknown prediction type {cfg.prediction_type}")


def _check_grad_scaler(cfg: StepConfig, refuse: Optional[str] = None):
    """StepConfig.grad_scaler combinations the step cannot run faithfully, refused before any CUDA
    call. refuse: the name of a step flavour that never runs with a GradScaler in the reference."""
    if not cfg.grad_scaler:
        return
    if refuse is not None:
        raise ValueError(f"{refuse} does not support StepConfig.grad_scaler: pivotal tuning never uses a GradScaler")
    if cfg.autocast_dtype != torch.float16 or cfg.compute_dtype != torch.float16:
        raise ValueError("StepConfig.grad_scaler needs autocast_dtype=torch.float16 and compute_dtype=torch.float16 "
                         f"(got {cfg.autocast_dtype} and {cfg.compute_dtype})")
    if cfg.lr_step_first:
        raise ValueError("StepConfig.grad_scaler with lr_step_first=True: no reference trainer steps its scheduler "
                         "first under a GradScaler")
    if not (cfg.growth_factor > 1.0 and 0.0 < cfg.backoff_factor < 1.0 and cfg.growth_interval >= 1
            and cfg.init_scale > 0.0):
        raise ValueError("StepConfig.grad_scaler: need init_scale > 0, growth_factor > 1, 0 < backoff_factor < 1, "
                         "growth_interval >= 1")


def _check_ranks_agree(what: str, **fields):
    """Collective: raise ValueError on every rank unless every rank passed the same fields."""
    import torch.distributed as dist
    everyone = [None] * dist.get_world_size()
    dist.all_gather_object(everyone, fields)
    bad = sorted(k for k in fields if any(e[k] != everyone[0][k] for e in everyone))
    if bad:
        raise ValueError(f"{what}: the data-parallel ranks disagree on " +
                         ", ".join(f"{k} ({[e[k] for e in everyone]})" for k in bad))


class LoraTrainStep:
    """One data-parallel replica of the LoRA fine-tuning step (bs = latents.shape[0] per GPU)."""

    # run the text encoder with gradients even when it has no trained LoRA factors
    _text_encoder_grad = False
    # LoraArena's rows= argument (capacity, D, lr) of a step that trains embedding rows too
    _arena_rows = None

    def __init__(self, unet: nn.Module, text_encoder: nn.Module, cfg: StepConfig,
                 latent_shape=(1, 4, 64, 64), seq_len: int = 77, device=None, vae: Optional[nn.Module] = None):
        _check_prediction_type(cfg)
        _check_grad_scaler(cfg)
        _check_encode_images(cfg, vae)
        self.cfg = cfg
        self.unet, self.text_encoder = unet, text_encoder
        self.device = torch.device(device or "cuda")
        from .grouping import link_sites
        encoders = self._text_encoders()
        link_sites(unet, *encoders)          # a copied / unpickled model has lost its back-references
        self.arena = LoraArena(self._arena_groups(), compute_dtype=cfg.compute_dtype, device=self.device,
                               rows=self._arena_rows)
        if cfg.grad_scaler:
            self.arena.enable_loss_scaling(cfg.init_scale, cfg.growth_factor, cfg.backoff_factor, cfg.growth_interval)
        self.noiser = DDPMNoiser(device=self.device)
        self.model_dtype = next(unet.parameters()).dtype
        # static step I/O (graph-stable addresses)
        self.latents = torch.zeros(latent_shape, device=self.device, dtype=torch.float32)
        self.input_ids = torch.zeros((latent_shape[0], seq_len), device=self.device, dtype=torch.long)
        self.loss = torch.zeros((), device=self.device, dtype=torch.float32)
        if cfg.external_noise:
            self.noise = torch.zeros(latent_shape, device=self.device, dtype=torch.float32)
            self.timesteps = torch.zeros((latent_shape[0],), device=self.device, dtype=torch.long)
        self.mask = torch.ones((latent_shape[0], 1, latent_shape[2], latent_shape[3]), device=self.device)
        if cfg.train_inpainting:
            self.inpaint_mask = torch.zeros((latent_shape[0], 1, latent_shape[2], latent_shape[3]), device=self.device)
            self.masked_latents = torch.zeros(latent_shape, device=self.device, dtype=torch.float32)
        self._init_image_inputs(vae, latent_shape)
        self.global_step = 0
        # pinned host mirrors for the end-to-end path
        self.h_latents = torch.zeros(latent_shape, dtype=torch.float32).pin_memory()
        self.h_input_ids = torch.zeros((latent_shape[0], seq_len), dtype=torch.long).pin_memory()
        self.h_loss = torch.zeros((), dtype=torch.float32).pin_memory()
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.graph_update: Optional[torch.cuda.CUDAGraph] = None
        self.graph_error: Optional[str] = None
        self._world = 1
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            self._world = dist.get_world_size()
        self.peer_allreduce = False
        if self._world > 1 and cfg.peer_allreduce:
            try:
                self.peer_allreduce = bool(self.arena.enable_peer_allreduce())
            except Exception as e:        # e.g. ranks on different nodes: keep the NCCL all-reduce
                self.peer_allreduce = False
                self.peer_allreduce_error = f"{type(e).__name__}: {e}"
            # a rank whose mapping failed must not leave the others waiting on its flags
            ok = torch.tensor([1.0 if self.peer_allreduce else 0.0], device=self.device)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN)
            if float(ok) == 0.0 and self.peer_allreduce:
                self.peer_allreduce = False
                self.arena._dp = None
        self.unet.train()
        for te in encoders:
            te.train()
        if cfg.gradient_checkpointing:
            _enable_gradient_checkpointing(unet, text_encoder, cfg.train_text_encoder or self._text_encoder_grad,
                                           *encoders[1:])

    def _text_encoders(self):
        """The step's text encoders, in arena-group order."""
        return (self.text_encoder,)

    def _arena_groups(self):
        """(model or site list, lr) per optimizer param-group: the UNet, then each text encoder when trained."""
        cfg = self.cfg
        groups = [(self.unet, cfg.learning_rate)]
        if cfg.train_text_encoder:
            groups += [(te, cfg.learning_rate_text) for te in self._text_encoders()]
        return groups

    def _init_image_inputs(self, vae, latent_shape):
        """Static inputs of a StepConfig.encode_images step (graph-stable addresses): the images at 8x the
        latent grid (+ the image-resolution inpainting mask) with pinned host mirrors, and with
        external_noise the posterior noise beside `self.noise`. The latents buffers then hold what the
        step samples: `self.latents` (and `self.masked_latents` / `self.inpaint_mask`) are outputs."""
        self.vae = vae
        cfg = self.cfg
        if not cfg.encode_images:
            return
        B, _, h, w = latent_shape
        self.vae_dtype = next(vae.parameters()).dtype
        self.posterior_noise_dtype = torch.float32 if cfg.posterior_noise_fp32 else self.vae_dtype
        shape = (B, 8 * h, 8 * w, 3) if cfg.pixel_dtype == torch.uint8 else (B, 3, 8 * h, 8 * w)
        self.pixels = torch.zeros(shape, device=self.device, dtype=cfg.pixel_dtype)
        self.h_pixels = torch.zeros(shape, dtype=cfg.pixel_dtype).pin_memory()
        if cfg.train_inpainting:
            self.pixel_mask = torch.zeros((B, 1, 8 * h, 8 * w), device=self.device, dtype=torch.float32)
            self.h_pixel_mask = torch.zeros((B, 1, 8 * h, 8 * w), dtype=torch.float32).pin_memory()
        if cfg.external_noise:
            self.posterior_noise = torch.zeros(latent_shape, device=self.device, dtype=self.posterior_noise_dtype)
            if cfg.train_inpainting:
                self.masked_posterior_noise = torch.zeros_like(self.posterior_noise)

    def _encode_images(self, fused: bool):
        """train_lora_dreambooth.py:818-821 / cli_lora_pti.py:273-290: images -> VAE input -> the frozen
        VAE (no_grad, its own dtype) -> posterior moments, then the posterior noise (image first, then
        the masked image: the reference's draw order, before the step's noise and timesteps).
        Returns (moments, posterior noise, masked moments, masked posterior noise) for the fused
        prologue; the unfused path samples here, into self.latents (+ masked_latents, inpaint_mask)."""
        cfg = self.cfg
        inpaint = cfg.train_inpainting
        with torch.no_grad():
            if fused:
                from .step_ops import pixels_ingest
                x, xm = pixels_ingest(self.pixels, self.vae_dtype, self.pixel_mask if inpaint else None)
            else:
                x = self.pixels
                if x.dtype == torch.uint8:           # torchvision's ToTensor + Normalize([0.5], [0.5])
                    x = x.permute(0, 3, 1, 2).float().div(255).sub(0.5).div(0.5)
                xm = x * (self.pixel_mask < 0.5) if inpaint else None        # dataset.py:115
                x = x.to(self.vae_dtype).contiguous(memory_format=torch.channels_last)
                if inpaint:
                    xm = xm.to(self.vae_dtype).contiguous(memory_format=torch.channels_last)
            moments = self.vae.encode(x).latent_dist.parameters
            masked_moments = self.vae.encode(xm).latent_dist.parameters if inpaint else None
        if cfg.external_noise:
            pe = self.posterior_noise
            mpe = self.masked_posterior_noise if inpaint else None
        else:
            pe = torch.randn(self.latents.shape, device=self.latents.device, dtype=self.posterior_noise_dtype)
            mpe = torch.randn_like(pe) if inpaint else None
        if not fused:
            from .host.vae import DiagonalGaussianDistribution

            def sample(m, e):                        # latent_dist.sample() * 0.18215
                post = DiagonalGaussianDistribution(m)
                return (post.mean + post.std * e) * cfg.vae_scaling

            with torch.no_grad():
                self.latents.copy_(sample(moments, pe))
                if inpaint:
                    self.masked_latents.copy_(sample(masked_moments, mpe))
                    self.inpaint_mask.copy_(F.interpolate(self.pixel_mask, scale_factor=1 / 8))
        return moments, pe, masked_moments, mpe

    # ------------------------------------------------------------------ the step body
    def _fwd_bwd(self):
        """noise -> text encoder -> UNet -> MSE -> backward; dA/dB land in the arena's g buffer."""
        cfg = self.cfg
        lat = self.latents
        bsz = lat.shape[0]
        from . import dropout_path
        if lat.is_cuda and getattr(self, "_has_dropout", None) is None:
            self._has_dropout = any(
                type(m).__name__ in ("LoraInjectedLinear", "LoraInjectedConv2d") and m.dropout.p > 0.0
                for mod in (self.unet,) + self._text_encoders() for m in mod.modules())
        if lat.is_cuda and self._has_dropout:
            dropout_path.begin_step(lat.device)      # one RNG launch for all dropout sites of the step
        fused = cfg.fused_glue and lat.is_cuda
        if cfg.encode_images:
            moments, post_eps, masked_moments, masked_post_eps = self._encode_images(fused)
        if cfg.external_noise:
            noise, timesteps = self.noise, self.timesteps
        else:
            noise = torch.randn_like(lat)
            t_max = int(self.noiser.num_train_timesteps * cfg.t_multiplier)
            timesteps = torch.randint(0, t_max, (bsz,), device=lat.device).long()
        v_pred = cfg.prediction_type == "v_prediction"
        target = noise
        if fused and cfg.encode_images:
            from .step_ops import step_prologue_posterior
            inp = cfg.train_inpainting
            noisy = step_prologue_posterior(moments, post_eps, noise, timesteps, self.noiser, self.model_dtype, lat,
                                            cfg.vae_scaling, masked_moments, masked_post_eps,
                                            self.pixel_mask if inp else None, self.masked_latents if inp else None,
                                            self.inpaint_mask if inp else None, velocity=v_pred)
            if v_pred:
                noisy, target = noisy
        elif fused:
            from .step_ops import step_prologue
            noisy = step_prologue(lat, noise, timesteps, self.noiser, self.model_dtype,
                                  self.inpaint_mask if cfg.train_inpainting else None,
                                  self.masked_latents if cfg.train_inpainting else None, velocity=v_pred)
            if v_pred:
                noisy, target = noisy
        else:
            noisy = self.noiser.add_noise(lat, noise, timesteps)
            if v_pred:
                target = self.noiser.get_velocity(lat, noise, timesteps)
            if cfg.train_inpainting:
                noisy = torch.cat([noisy, self.inpaint_mask.to(noisy.dtype), self.masked_latents.to(noisy.dtype)], dim=1)
        ac = (torch.autocast("cuda", dtype=cfg.autocast_dtype) if cfg.autocast_dtype is not None
              else torch.autocast("cuda", enabled=False))
        with ac:
            pred = self._predict(noisy, timesteps)
        m = None
        if cfg.use_mask:
            m = (self.mask.float() + 0.01).pow(cfg.mask_temperature)
            m = m / m.max()
        if fused:
            from .step_ops import fused_masked_mse
            w = None
            if cfg.with_prior_preservation:      # [instance ; class] halves: mean + prior_loss_weight * mean
                half = bsz // 2
                w = torch.cat([torch.full((half,), 1.0 / half, device=lat.device),
                               torch.full((bsz - half,), cfg.prior_loss_weight / (bsz - half), device=lat.device)])
            loss = fused_masked_mse(pred, target, m, w, grad_scale=self.arena.loss_scale if cfg.grad_scaler else None)
        else:
            if cfg.use_mask:
                pred, target = pred * m, target * m
            if cfg.with_prior_preservation:
                pred, pred_prior = torch.chunk(pred, 2, dim=0)
                target, target_prior = torch.chunk(target, 2, dim=0)
                loss = (F.mse_loss(pred.float(), target.float(), reduction="none").mean([1, 2, 3]).mean()
                        + cfg.prior_loss_weight * F.mse_loss(pred_prior.float(), target_prior.float(), reduction="mean"))
            elif cfg.use_mask:
                loss = F.mse_loss(pred.float(), target.float(), reduction="none").mean([1, 2, 3]).mean()
            else:
                loss = F.mse_loss(pred.float(), target.float(), reduction="mean")
        from . import ops
        defer = cfg.defer_wgrad and lat.is_cuda and hasattr(self, "arena")
        if defer:
            ops.wgrad_defer_begin()
        try:
            if cfg.grad_scaler and not fused:
                (loss * self.arena.loss_scale).backward()      # GradScaler.scale(loss).backward()
            else:
                loss.backward()
            if defer:
                ops.wgrad_flush()
        finally:
            ops.wgrad_defer_cancel()
        dropout_path.end_step()
        self.loss.copy_(loss.detach())

    def _text_grad(self):
        """The text encoders run with gradients, or under no_grad when nothing of theirs is trained."""
        if self.cfg.train_text_encoder or self._text_encoder_grad:
            return contextlib.nullcontext()
        return torch.no_grad()

    def _unet_input(self, noisy):
        """The fused prologue already wrote the model's dtype in channels_last; the torch path casts here."""
        if self.cfg.fused_glue and noisy.is_cuda:
            return noisy
        return noisy.to(self.model_dtype).contiguous(memory_format=torch.channels_last)

    def _predict(self, noisy, timesteps):
        """Conditioning and the UNet, under the step's autocast: text encoder -> UNet -> prediction."""
        with self._text_grad():
            ehs = self.text_encoder(self.input_ids)[0]
        return self.unet(self._unet_input(noisy), timesteps, ehs.to(self.model_dtype)).sample

    def set_loss_mask(self, mask_image_res: torch.Tensor):
        """`batch["mask"]` of the PTI dataset (image resolution, [B,1,8h,8w] or anything that
        reshapes to it) -> nearest-neighbour resize to the latent grid, as cli_lora_pti.py:342-354
        does every step; stored in `self.mask` for `use_mask` steps."""
        b, _, h, w = self.mask.shape
        m = mask_image_res.to(self.device, torch.float32).reshape(b, 1, h * 8, w * 8)
        self.mask.copy_(F.interpolate(m, size=(h, w), mode="nearest"))

    def _update(self):
        cfg = self.cfg
        schedule = None
        if cfg.grad_scaler:       # the schedule follows the applied-step count on the device
            from .arena import LrSchedule
            schedule = LrSchedule(cfg.lr_scheduler, cfg.lr_warmup_steps, cfg.max_train_steps,
                                  self._scheduled_groups())
        self.arena.step(cfg.adam_beta1, cfg.adam_beta2, cfg.adam_epsilon, cfg.adam_weight_decay,
                        cfg.max_grad_norm, world_size=self._world, schedule=schedule)

    def _scheduled_groups(self):
        """Parameter groups whose lr follows the LR schedule (loss-scaled steps): all of them."""
        return tuple(range(len(self.arena.base_lr)))

    def _body(self):
        """One eager step: forward/backward, the one collective, fused clip+AdamW."""
        self._fwd_bwd()
        self.arena.allreduce_grads()
        self._update()

    def _capture(self):
        """Two graphs around the collective: [forward+backward] - NCCL all-reduce - [clip+AdamW].
        The all-reduce stays an ordinary stream-ordered NCCL call between the two replays (a
        collective inside a captured graph would tie every rank's capture to its peers')."""
        # Warm-up runs real step bodies (cuDNN/cuBLAS autotuning, allocator pools, grouping
        # families) but must not TRAIN: the arena (p, m, v, Adam's t), the loss buffer and the CUDA
        # RNG stream are snapshotted here and restored after capture, so the first replay starts
        # from exactly the state prepare() was called in and optimizer t stays in step with the
        # lr schedule. (The reference has no warm-up; round 1 let these steps count.)
        snap = self._snapshot()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        try:
            with torch.cuda.stream(side):
                for _ in range(self.cfg.graph_warmup):
                    self._body()
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            self._capture_graphs()
        finally:
            torch.cuda.synchronize()
            self._restore(snap)

    def _snapshot(self):
        a = self.arena
        snap = {"p": a.p.clone(), "m": a.m.clone(), "v": a.v.clone(), "step": a.step_dev.clone(),
                "loss": self.loss.clone(), "rng": torch.cuda.get_rng_state(self.device)}
        if a.loss_scaling:
            snap["scaler"] = [t.clone() for t in (a.loss_scale, a._growth_tracker, a._found_inf, a.applied_steps)]
        return snap

    def _restore(self, snap):
        a = self.arena
        a.p.copy_(snap["p"]); a.m.copy_(snap["m"]); a.v.copy_(snap["v"]); a.step_dev.copy_(snap["step"])
        if a.loss_scaling:
            for t, saved in zip((a.loss_scale, a._growth_tracker, a._found_inf, a.applied_steps), snap["scaler"]):
                t.copy_(saved)
        a.g.zero_()
        self.loss.copy_(snap["loss"])
        a.refresh_shadows()
        a._publish_shadows()
        torch.cuda.set_rng_state(snap["rng"], self.device)
        torch.cuda.synchronize()

    def _capture_graphs(self):
        if self._world == 1 or self.peer_allreduce:
            # no library collective on the step path (single rank, or the all-reduce lives inside
            # lb_optim_step_dp): the WHOLE step is one graph
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._body()
            self.graph, self.graph_update = g, None
            return
        if self.cfg.capture_collective and self._world > 1:
            import torch.distributed as dist
            dist.barrier()                      # every rank enters its capture at the same time
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                self._body()
            self.graph, self.graph_update = g, None
            return
        g1 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g1):
            self._fwd_bwd()
        g2 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g2, pool=g1.pool()):
            self._update()
        self.graph, self.graph_update = g1, g2

    # ------------------------------------------------------------------ public API
    def prepare(self):
        """Warm up and (optionally) capture. Leaves parameters, optimizer state and the RNG stream
        exactly as it found them (the warm-up steps are rolled back)."""
        if self.cfg.use_cuda_graph and self.graph is None and self.graph_error is None:
            try:
                self._capture()
            except Exception as e:  # capture refused (e.g. a host sync inside the host model)
                self.graph_error = f"{type(e).__name__}: {e}"
                self.graph = self.graph_update = None
                torch.cuda.synchronize()
                self.arena.zero_grad()

    def lr_multiplier(self, step: int) -> float:
        """diffusers `get_scheduler` semantics: "constant" IGNORES num_warmup_steps (so the
        reference's defaults, constant + 500 warm-up steps at train_lora_dreambooth.py:345-356, mean
        no warm-up at all); "constant_with_warmup" and "linear" ramp 0 -> 1 over lr_warmup_steps,
        "linear" then decays to 0 at max_train_steps."""
        cfg = self.cfg
        if cfg.lr_scheduler == "constant":
            return 1.0
        if cfg.lr_scheduler not in ("linear", "constant_with_warmup"):
            raise ValueError(f"lr_scheduler {cfg.lr_scheduler!r}: constant | constant_with_warmup | linear")
        if cfg.lr_warmup_steps > 0 and step < cfg.lr_warmup_steps:
            return float(step) / float(max(1, cfg.lr_warmup_steps))
        if cfg.lr_scheduler == "linear":
            return max(0.0, float(cfg.max_train_steps - step) /
                       float(max(1, cfg.max_train_steps - cfg.lr_warmup_steps)))
        return 1.0

    def _set_step_lr(self):
        """Per-group learning rates of the step about to run (iteration self.global_step). Loss-scaled
        steps schedule every group on the device, from the applied-step count (a skipped step does
        not advance the schedule): the arena keeps the base lrs."""
        if self.cfg.grad_scaler:
            return
        if self.cfg.lr_scheduler != "constant":
            k = self.global_step + (1 if self.cfg.lr_step_first else 0)
            mult = self.lr_multiplier(k)                     # host-side schedule, tiny async H2D copy
            self.arena.set_lr([b * mult for b in self.arena.base_lr])

    def step_device(self) -> torch.Tensor:
        """One step on inputs already resident in self.latents / self.input_ids."""
        self._set_step_lr()
        self.global_step += 1
        if self.graph is not None:
            self.graph.replay()
            if self.graph_update is not None:   # two graphs around an eager collective (default)
                self.arena.allreduce_grads()
                self.graph_update.replay()
        else:
            self._body()
        return self.loss

    def step_host(self, latents_cpu: torch.Tensor, input_ids_cpu: torch.Tensor,
                  mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """End-to-end step from pinned host memory: H2D inputs, step, D2H loss (async, returns the
        pinned loss buffer; synchronise the stream before reading it).
        With StepConfig.encode_images the first argument is the batch of images instead, shaped and
        typed like `self.pixels` (uint8 [B, 8h, 8w, 3], or fp32 [B, 3, 8h, 8w] with pixel_dtype
        float32), and `mask` the image-resolution inpainting mask [B, 1, 8h, 8w] (train_inpainting)."""
        if self.cfg.encode_images:
            self._check_pixels(latents_cpu, mask)
            self.h_pixels.copy_(latents_cpu)
            self.pixels.copy_(self.h_pixels, non_blocking=True)
            if mask is not None:
                self.h_pixel_mask.copy_(mask.reshape(self.h_pixel_mask.shape))
                self.pixel_mask.copy_(self.h_pixel_mask, non_blocking=True)
            self.h_input_ids.copy_(input_ids_cpu)
        else:
            self.h_latents.copy_(latents_cpu)
            self.h_input_ids.copy_(input_ids_cpu)
            self.latents.copy_(self.h_latents, non_blocking=True)
        self.input_ids.copy_(self.h_input_ids, non_blocking=True)
        self.step_device()
        self.h_loss.copy_(self.loss, non_blocking=True)
        return self.h_loss

    def _check_pixels(self, pixels: torch.Tensor, mask: Optional[torch.Tensor]):
        """Refuse, before any copy, images the encode_images step cannot take."""
        cfg = self.cfg
        if pixels.dtype not in (torch.uint8, torch.float32):
            raise ValueError(f"pixels must be uint8 or float32, got {pixels.dtype}")
        if pixels.dtype != self.pixels.dtype:
            raise ValueError(f"pixels are {pixels.dtype} but the step was built for StepConfig.pixel_dtype="
                             f"{self.pixels.dtype}")
        if tuple(pixels.shape) != tuple(self.pixels.shape):
            raise ValueError(f"pixels of shape {tuple(pixels.shape)}: the step takes {tuple(self.pixels.shape)}, "
                             f"8x the latent grid {tuple(self.latents.shape[2:])}")
        if cfg.train_inpainting:
            if mask is None:
                raise ValueError("train_inpainting from images needs the image-resolution mask: step_host(..., mask=)")
            if mask.numel() != self.pixel_mask.numel():
                raise ValueError(f"mask of shape {tuple(mask.shape)}: the step takes {tuple(self.pixel_mask.shape)}")
        elif mask is not None:
            raise ValueError("a mask is the inpainting input: StepConfig.train_inpainting is off")

    def h2d_bytes(self) -> int:
        if self.cfg.encode_images:
            n = self.h_pixels.numel() * self.h_pixels.element_size() + self.h_input_ids.numel() * 8
            return n + (self.h_pixel_mask.numel() * 4 if self.cfg.train_inpainting else 0)
        return self.h_latents.numel() * 4 + self.h_input_ids.numel() * 8

    def d2h_bytes(self) -> int:
        return 4


def _check_xl_models(unet: nn.Module, text_encoder: nn.Module, text_encoder_2: nn.Module):
    """The SDXL pair of encoders must fit the UNet: refused before any CUDA call."""
    ucfg = getattr(unet, "cfg", None) or getattr(unet, "config", None)
    if getattr(ucfg, "addition_embed_type", None) != "text_time":
        raise ValueError("LoraXLTrainStep needs an SDXL UNet (addition_embed_type='text_time')")
    c1, c2 = text_encoder.config, text_encoder_2.config
    if not hasattr(text_encoder_2, "text_projection"):
        raise ValueError("text_encoder_2 must be a CLIPTextModelWithProjection: its text_embeds are the pooled "
                         "conditioning")
    ctx = c1.hidden_size + c2.hidden_size
    if ctx != ucfg.cross_attention_dim:
        raise ValueError(f"the text encoders' widths {c1.hidden_size} + {c2.hidden_size} = {ctx} do not match the "
                         f"UNet's cross_attention_dim {ucfg.cross_attention_dim}")
    add_in = c2.projection_dim + 6 * ucfg.addition_time_embed_dim
    if add_in != ucfg.projection_class_embeddings_input_dim:
        raise ValueError(f"text_encoder_2's projection_dim {c2.projection_dim} + 6 x {ucfg.addition_time_embed_dim} "
                         f"= {add_in} does not match the UNet's projection_class_embeddings_input_dim "
                         f"{ucfg.projection_class_embeddings_input_dim}")


class LoraXLTrainStep(LoraTrainStep):
    """The LoRA step on SDXL: two text encoders and the "text_time" conditioning, the conditioning of
    diffusers' train_dreambooth_lora_sdxl.py (`encode_prompt`, `compute_time_ids`, the UNet call with
    added_cond_kwargs). Per step:

        h1 = text_encoder(input_ids, output_hidden_states=True).hidden_states[-2]
        out2 = text_encoder_2(input_ids_2, output_hidden_states=True)
        encoder_hidden_states = cat([h1, out2.hidden_states[-2]], -1)      # [B, 77, 768 + 1280]
        unet(noisy, t, encoder_hidden_states,
             added_cond_kwargs={"text_embeds": out2.text_embeds, "time_ids": time_ids})

    Everything else -- noise, timesteps, the latents or the image encode (StepConfig.vae_scaling = 0.13025
    for the SDXL VAE), the loss and its options, clip + AdamW -- is LoraTrainStep's. The arena has up to
    three groups: (unet, learning_rate), then (text_encoder, learning_rate_text) and (text_encoder_2,
    learning_rate_text) with train_text_encoder; one global clip and one optimizer launch cover all three.
    The sites of the first encoder's last layer are not trained (see _arena_groups).

    Static inputs besides LoraTrainStep's: `input_ids_2` [B, seq_len] (the second tokenizer's ids) and
    `time_ids` [B, 6] fp32 (original size, crop top-left, target size), which starts at (8h, 8w, 0, 0, 8h,
    8w) for every sample -- the Dreambooth script's default -- and keeps what is written into it."""

    def __init__(self, unet: nn.Module, text_encoder: nn.Module, text_encoder_2: nn.Module, cfg: StepConfig,
                 latent_shape=(1, 4, 128, 128), seq_len: int = 77, device=None, vae: Optional[nn.Module] = None):
        _check_xl_models(unet, text_encoder, text_encoder_2)
        self.text_encoder_2 = text_encoder_2
        super().__init__(unet, text_encoder, cfg, latent_shape=latent_shape, seq_len=seq_len, device=device,
                         vae=vae)
        B, _, h, w = latent_shape
        self.input_ids_2 = torch.zeros((B, seq_len), device=self.device, dtype=torch.long)
        size = [8.0 * h, 8.0 * w, 0.0, 0.0, 8.0 * h, 8.0 * w]
        self.time_ids = torch.tensor([size] * B, device=self.device, dtype=torch.float32)
        self.h_input_ids_2 = torch.zeros((B, seq_len), dtype=torch.long).pin_memory()
        self.h_time_ids = self.time_ids.cpu().pin_memory()

    def _text_encoders(self):
        return (self.text_encoder, self.text_encoder_2)

    def _arena_groups(self):
        """The first encoder's last layer only feeds hidden_states[-1], which the conditioning never reads:
        its LoRA factors get no gradient, and torch's AdamW leaves a parameter without a gradient as it is
        (no weight decay either). They stay out of the arena, so they are never updated either."""
        groups = super()._arena_groups()
        if self.cfg.train_text_encoder:
            from .arena import lora_sites
            dead = {id(m) for m in lora_sites(self.text_encoder.text_model.encoder.layers[-1])}
            groups[1] = ([m for m in lora_sites(self.text_encoder) if id(m) not in dead], groups[1][1])
        return groups

    def _predict(self, noisy, timesteps):
        """diffusers' SDXL encode_prompt: both encoders' penultimate hidden states, concatenated; encoder 2's
        projected pooled output and the time ids as the UNet's added conditioning."""
        with self._text_grad():
            out1 = self.text_encoder(self.input_ids, output_hidden_states=True)
            out2 = self.text_encoder_2(self.input_ids_2, output_hidden_states=True)
            ehs = torch.cat([out1.hidden_states[-2], out2.hidden_states[-2]], dim=-1)
            added = {"text_embeds": out2.text_embeds, "time_ids": self.time_ids}
        return self.unet(self._unet_input(noisy), timesteps, ehs.to(self.model_dtype), added_cond_kwargs=added).sample

    def _check_xl_inputs(self, input_ids_2: torch.Tensor, time_ids: Optional[torch.Tensor]):
        if tuple(input_ids_2.shape) != tuple(self.input_ids_2.shape):
            raise ValueError(f"input_ids_2 of shape {tuple(input_ids_2.shape)}: the step takes "
                             f"{tuple(self.input_ids_2.shape)}")
        if input_ids_2.dtype.is_floating_point or input_ids_2.dtype.is_complex:
            raise ValueError(f"input_ids_2 must be integer token ids, got {input_ids_2.dtype}")
        if time_ids is not None and tuple(time_ids.shape) != tuple(self.time_ids.shape):
            raise ValueError(f"time_ids of shape {tuple(time_ids.shape)}: the step takes {tuple(self.time_ids.shape)} "
                             "(original size, crop top-left, target size per sample)")

    def step_host(self, latents_cpu: torch.Tensor, input_ids_cpu: torch.Tensor, input_ids_2_cpu: torch.Tensor,
                  time_ids: Optional[torch.Tensor] = None, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """LoraTrainStep.step_host with the second encoder's ids and, optionally, new time ids [B, 6]
        (None keeps the buffer's current contents)."""
        self._check_xl_inputs(input_ids_2_cpu, time_ids)
        if self.cfg.encode_images:
            self._check_pixels(latents_cpu, mask)
        self.h_input_ids_2.copy_(input_ids_2_cpu)
        self.input_ids_2.copy_(self.h_input_ids_2, non_blocking=True)
        if time_ids is not None:
            self.h_time_ids.copy_(time_ids)
            self.time_ids.copy_(self.h_time_ids, non_blocking=True)
        return super().step_host(latents_cpu, input_ids_cpu, mask)

    def h2d_bytes(self) -> int:
        """Per step_host call, with new time ids."""
        return super().h2d_bytes() + self.h_input_ids_2.numel() * 8 + self.h_time_ids.numel() * 4


class TextualInversionStep(LoraTrainStep):
    """Phase 1 of pivotal tuning as a runnable loop: `train_inversion`, cli_lora_pti.py:373-542.

    Per iteration (the reference's order): lr_scheduler.step() FIRST (:417) -> loss_step (:420-431,
    the same noise / add_noise / text encoder / UNet / (masked) MSE body as the tuning phase, UNet in
    eval mode, text encoder in train mode) -> backward -> optimizer.step + zero_grad (:447-448) ->
    norm decay of the placeholder rows (:451-468) -> every other row restored (:477-479).
    Here only the placeholder rows are trainable (`TextualInversionRows`: a forward hook substitutes
    them into the embedding lookup, `lb_ti_embed_step` does AdamW + decay + write-back in one
    kernel), so the 49408 x 768 table is never touched. LoRA factors, if already injected, are
    frozen for the duration (the reference leaves them requires_grad=True and lets unused gradients
    pile up; with lora_up = 0 the forward is identical) -- `release()` restores their flags."""

    def __init__(self, unet: nn.Module, text_encoder: nn.Module, placeholder_token_ids, cfg: StepConfig,
                 lr: float = 5e-4, weight_decay: float = 0.0, clip_ti_decay: bool = True,
                 latent_shape=(1, 4, 64, 64), seq_len: int = 77, device=None, vae: Optional[nn.Module] = None):
        from .ti import TextualInversionRows
        _check_prediction_type(cfg)
        _check_grad_scaler(cfg, refuse="TextualInversionStep")
        _check_encode_images(cfg, vae)
        self.cfg = cfg
        self.unet, self.text_encoder = unet, text_encoder
        self.device = torch.device(device or "cuda")
        self.noiser = DDPMNoiser(device=self.device)
        self.model_dtype = next(unet.parameters()).dtype
        self.latents = torch.zeros(latent_shape, device=self.device, dtype=torch.float32)
        self.input_ids = torch.zeros((latent_shape[0], seq_len), device=self.device, dtype=torch.long)
        self.loss = torch.zeros((), device=self.device, dtype=torch.float32)
        if cfg.external_noise:
            self.noise = torch.zeros(latent_shape, device=self.device, dtype=torch.float32)
            self.timesteps = torch.zeros((latent_shape[0],), device=self.device, dtype=torch.long)
        self.mask = torch.ones((latent_shape[0], 1, latent_shape[2], latent_shape[3]), device=self.device)
        if cfg.train_inpainting:
            self.inpaint_mask = torch.zeros((latent_shape[0], 1, latent_shape[2], latent_shape[3]), device=self.device)
            self.masked_latents = torch.zeros(latent_shape, device=self.device, dtype=torch.float32)
        self._init_image_inputs(vae, latent_shape)
        from .dist import world_info
        _, self._world = world_info()
        if self._world > 1:
            _check_ranks_agree("TextualInversionStep", placeholder_token_ids=[int(t) for t in placeholder_token_ids],
                               table=tuple(text_encoder.get_input_embeddings().weight.shape),
                               latent_shape=tuple(int(s) for s in latent_shape), seq_len=int(seq_len))
        self.global_step = 0
        self.graph = self.graph_update = None
        self.graph_error = None
        self.base_lr = float(lr)
        self.ti = TextualInversionRows(text_encoder, placeholder_token_ids, lr=lr, weight_decay=weight_decay,
                                       clip_ti_decay=clip_ti_decay)
        if self._world > 1:
            self.ti.sync_replicas()        # rank 0's placeholder rows, in the rows and in the table
        self._frozen = []
        for m in list(unet.modules()) + list(text_encoder.modules()):
            if type(m).__name__ in ("LoraInjectedLinear", "LoraInjectedConv2d"):
                for prm in (m.lora_up.weight, m.lora_down.weight):
                    if prm.requires_grad:
                        prm.requires_grad_(False)
                        self._frozen.append(prm)
        self.unet.eval()               # cli_lora_pti.py:411-412
        self.text_encoder.train()
        if cfg.gradient_checkpointing:  # the UNet runs in eval mode here: only the text encoder recomputes
            _enable_gradient_checkpointing(unet, text_encoder, cfg.train_text_encoder)

    def prepare(self):
        return None                    # eager loop (phase 1 is not the timed path)

    def step_device(self) -> torch.Tensor:
        cfg = self.cfg
        k = self.global_step + 1       # the scheduler is stepped before the update (:417)
        self.ti.set_lr(self.base_lr * (self.lr_multiplier(k) if cfg.lr_scheduler != "constant" else 1.0))
        self.global_step += 1
        if not cfg.train_text_encoder:
            raise ValueError("TextualInversionStep needs StepConfig.train_text_encoder=True")
        self._fwd_bwd()                # rows.grad <- d loss / d placeholder rows
        if self._world > 1:            # DDP's mean over the ranks: pre-divide, one all-reduce(sum)
            import torch.distributed as dist
            g = self.ti.rows.grad
            g.mul_(1.0 / self._world)
            dist.all_reduce(g, op=dist.ReduceOp.SUM)
        self.ti.step()                 # AdamW + norm decay + write-back + zero_grad, one kernel
        return self.loss

    def release(self):
        """End of phase 1: drop the lookup hook, give the LoRA factors their requires_grad back."""
        self.ti.remove()
        for prm in self._frozen:
            prm.requires_grad_(True)
        self._frozen = []


class LoraEmbeddingStep(LoraTrainStep):
    """The LoRA step with the CLIP token-embedding table trained by the same AdamW and clipped by the
    same clip_grad_norm_ as the factors -- the reference's two joint configurations:

      mode="table"         cli_lora_pti.py phase 2 with `--continue_inversion` (:958-997 optimizer,
                           :545-620 loop): lr_scheduler.step() first, loss_step(t_mutliplier=0.8),
                           backward, clip over UNet + text encoder, AdamW(weight_decay_lora) over
                           [unet LoRA, table (+ text LoRA)]; every row decays every step, nothing
                           is restored.
          LoraEmbeddingStep(unet, text_encoder, placeholder_ids,
                            StepConfig(learning_rate=unet_lr, learning_rate_text=text_encoder_lr,
                                       train_text_encoder=train_text_encoder,
                                       adam_weight_decay=weight_decay_lora, t_multiplier=0.8,
                                       lr_step_first=True, lr_scheduler="linear", ...),
                            lr_embedding=continue_inversion_lr or ti_lr, mode="table")

      mode="placeholders"  train_lora_w_ti.py (:830-853 optimizer, :986-1075 loop): before
                           iteration k < unfreeze_lora_step the LoRA groups get lr 0 (moments still
                           move, gradients still enter the norm) and the table runs at
                           lr_ti * lambda(k); from then on the LoRA groups run at their base lr
                           (unscheduled) and the table at 0. clip, AdamW, lr_scheduler.step(); every
                           row except the placeholders is restored.
          LoraEmbeddingStep(unet, text_encoder, [placeholder_token_id],
                            StepConfig(learning_rate=learning_rate, learning_rate_text=learning_rate_text,
                                       train_text_encoder=True, adam_weight_decay=adam_weight_decay,
                                       lr_scheduler=lr_scheduler, lr_warmup_steps=..., max_train_steps=...),
                            lr_embedding=learning_rate_ti, mode="placeholders",
                            unfreeze_lora_step=unfreeze_lora_step)

    The table keeps requires_grad=False; the rows that get a gradient are claimed into
    `row_capacity` slots of the arena (lora_b200/embed_rows.py). Per step this adds two launches
    to the plain step: the gradient scatter (in backward) and the write-back (after the optimizer).
    Mode "table" leaves the decay of unseen rows pending: call `flush()` before reading the table
    outside the step (validation, saving a full text encoder); `release()` flushes too.

    Data parallel (torch.distributed, one process per GPU of one node): the scatter claims slots over
    the union of every rank's input_ids in rank order -- the slots one process would claim for the
    concatenated batch -- so the rows group is summed, clipped and updated by the arena's all-reduce
    and optimizer launch like the factors. The peers' ids are read inside the scatter launch over
    CUDA IPC (peer_allreduce, the whole step stays one graph) or all-gathered by NCCL before the
    backward. world * B * seq_len must not exceed 2048; ranks must agree on the placeholders,
    row_capacity, mode and shapes (checked at construction); rank 0's table is broadcast."""

    _text_encoder_grad = True

    def __init__(self, unet: nn.Module, text_encoder: nn.Module, placeholder_token_ids, cfg: StepConfig,
                 lr_embedding: float, mode: str = "table", unfreeze_lora_step: Optional[int] = None,
                 row_capacity: int = 1024, latent_shape=(1, 4, 64, 64), seq_len: int = 77, device=None,
                 vae: Optional[nn.Module] = None):
        from ._C import LoraB200Error
        from .embed_rows import MAX_SCATTER_TOKENS, MODES, EmbeddingRows
        from .dist import world_info
        if mode not in MODES:
            raise ValueError(f"mode {mode!r}: one of {MODES}")
        _check_grad_scaler(cfg, refuse="LoraEmbeddingStep(mode='table')" if mode == "table" else None)
        if mode == "placeholders" and not cfg.train_text_encoder:
            raise ValueError("mode='placeholders' (train_lora_w_ti.py) needs StepConfig.train_text_encoder=True: "
                             "without it the script clips the UNet factors only but updates the table too")
        if mode == "table" and unfreeze_lora_step is not None:
            raise ValueError("unfreeze_lora_step belongs to mode='placeholders'")
        self.mode = mode
        self.unfreeze_lora_step = (500 if unfreeze_lora_step is None else int(unfreeze_lora_step)) \
            if mode == "placeholders" else None        # train_lora_w_ti.py:570-574 default
        table = text_encoder.get_input_embeddings().weight
        D = table.shape[1]
        _, world = world_info()
        n_tok = world * int(latent_shape[0]) * int(seq_len)
        if n_tok > MAX_SCATTER_TOKENS:
            raise LoraB200Error(f"LoraEmbeddingStep: {world} rank(s) x batch {latent_shape[0]} x {seq_len} tokens = "
                                f"{n_tok} exceed the gradient scatter's limit of {MAX_SCATTER_TOKENS} tokens per step")
        if world > 1:
            if cfg.capture_collective:
                raise ValueError("LoraEmbeddingStep: capture_collective is not supported with data parallelism")
            # ranks that disagree would enter incompatible graphs: refuse on every rank, before anything runs
            _check_ranks_agree("LoraEmbeddingStep", placeholder_token_ids=[int(t) for t in placeholder_token_ids],
                               row_capacity=int(row_capacity), D=int(D), vocab=int(table.shape[0]), mode=mode,
                               latent_shape=tuple(int(s) for s in latent_shape), seq_len=int(seq_len))
        self._arena_rows = (int(row_capacity), int(D), float(lr_embedding))
        super().__init__(unet, text_encoder, cfg, latent_shape=latent_shape, seq_len=seq_len, device=device, vae=vae)
        self.rows = EmbeddingRows(text_encoder, self.arena, placeholder_token_ids, mode=mode,
                                  weight_decay=cfg.adam_weight_decay)
        if self._world > 1:
            self.rows.sync_replicas()            # rank 0's table and row state everywhere
            if not self.rows.enable_data_parallel(self.input_ids, peer=self.peer_allreduce) and self.peer_allreduce:
                # a rank could not map the peers' ids: the whole step takes the NCCL path
                self.peer_allreduce = False
                self.arena._dp = None
        # overflow flag of the last two step_host calls (pinned, copied without a synchronise)
        self._h_flags = [torch.zeros(1, dtype=torch.int32).pin_memory() for _ in range(2)]
        self._flag_events = [None, None]
        self._host_calls = 0

    def _set_step_lr(self):
        if self.mode == "table":
            return super()._set_step_lr()
        cfg = self.cfg
        k = self.global_step
        mult = 1.0
        if cfg.lr_scheduler != "constant":
            mult = self.lr_multiplier(k + (1 if cfg.lr_step_first else 0))
        if cfg.grad_scaler:                      # the rows' schedule runs on the device (applied steps)
            mult = 1.0
        base, rg = self.arena.base_lr, self.arena.rows_group
        if k < self.unfreeze_lora_step:          # train_lora_w_ti.py:988-991
            lrs = [0.0] * len(base)
            lrs[rg] = base[rg] * mult
        else:                                    # :992-995: LoRA at its base lr, table frozen
            lrs = list(base)
            lrs[rg] = 0.0
        self.arena.set_lr(lrs)

    def _scheduled_groups(self):
        if self.mode == "table":
            return super()._scheduled_groups()
        # train_lora_w_ti.py sets the LoRA groups by hand every iteration; only the table follows the
        # LambdaLR (its lr is 0 after unfreeze_lora_step, so lambda * 0 stays 0)
        return (self.arena.rows_group,)

    def _body(self):
        if self.rows.gathers_ids:                # NCCL path: every rank's ids before the backward
            self.rows.gather_ids()
        super()._body()

    def step_device(self) -> torch.Tensor:
        if self.graph is not None and self.graph_update is not None and self.rows.gathers_ids:
            self.rows.gather_ids()               # outside graph 1, like the gradient all-reduce
        return super().step_device()

    def _update(self):
        super()._update()
        self.rows.write_back()

    def _snapshot(self):
        snap = super()._snapshot()
        snap["rows"] = self.rows.snapshot()
        return snap

    def _restore(self, snap):
        self.rows.restore(snap["rows"])
        super()._restore(snap)

    def step_host(self, latents_cpu: torch.Tensor, input_ids_cpu: torch.Tensor,
                  mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """LoraTrainStep.step_host; an overflow of the row slots in this step raises no later than the
        next call (the flag is copied to pinned memory behind the step and read one call later)."""
        out = super().step_host(latents_cpu, input_ids_cpu, mask)
        i = self._host_calls % 2
        self._h_flags[i].copy_(self.rows.state[3:4], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._flag_events[i] = ev
        self._host_calls += 1
        prev = self._flag_events[1 - i]
        if prev is not None:                     # the previous step: finished or about to (this one is queued)
            prev.synchronize()
            self.rows.raise_for_flags(int(self._h_flags[1 - i][0]))
        return out

    def flush(self):
        """Apply the pending decay to the rows no gradient has touched yet (mode "table") and check
        for an overflow of the row slots: the table then holds what dense AdamW would."""
        self.rows.flush()

    def release(self):
        """End of training: flush, then drop the lookup hook."""
        try:
            self.flush()
        finally:
            self.rows.remove()
