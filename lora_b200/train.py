"""Training-step engine: the step loop of the reference's trainers, restated around the fused
LoRA path and captured as ONE CUDA graph.

Restates (diffusers / accelerate are not installed, so the scripts themselves cannot run):
  training_scripts/train_lora_dreambooth.py:811-888  -- Dreambooth step (noise, timestep,
      add_noise, text encoder, UNet, MSE, backward, clip_grad_norm_(1.0), AdamW, zero_grad)
  lora_diffusion/cli_lora_pti.py:260-370, 585-617     -- PTI LoRA-tuning phase (same step with
      t_mutliplier and mean([1,2,3]).mean() reduction)
Differences by design: LoRA factors/grads/moments live in a LoraArena, the
DDP all-reduce + clip + AdamW + zero_grad are one NCCL call and two kernels, and steady-state
steps are CUDA-graph replays (no Python, no launch gaps, no host sync).
"""
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


PREDICTION_TYPES = ("epsilon", "v_prediction")


def _check_prediction_type(cfg: StepConfig):
    if cfg.prediction_type not in PREDICTION_TYPES:
        raise ValueError(f"Unknown prediction type {cfg.prediction_type}")


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
                 latent_shape=(1, 4, 64, 64), seq_len: int = 77, device=None):
        _check_prediction_type(cfg)
        self.cfg = cfg
        self.unet, self.text_encoder = unet, text_encoder
        self.device = torch.device(device or "cuda")
        from .grouping import link_sites
        link_sites(unet, text_encoder)       # a copied / unpickled model has lost its back-references
        groups = [(unet, cfg.learning_rate)]
        if cfg.train_text_encoder:
            groups.append((text_encoder, cfg.learning_rate_text))
        self.arena = LoraArena(groups, compute_dtype=cfg.compute_dtype, device=self.device,
                               rows=self._arena_rows)
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
        self.text_encoder.train()

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
                for mod in (self.unet, self.text_encoder) for m in mod.modules())
        if lat.is_cuda and self._has_dropout:
            dropout_path.begin_step(lat.device)      # one RNG launch for all dropout sites of the step
        if cfg.external_noise:
            noise, timesteps = self.noise, self.timesteps
        else:
            noise = torch.randn_like(lat)
            t_max = int(self.noiser.num_train_timesteps * cfg.t_multiplier)
            timesteps = torch.randint(0, t_max, (bsz,), device=lat.device).long()
        fused = cfg.fused_glue and lat.is_cuda
        v_pred = cfg.prediction_type == "v_prediction"
        target = noise
        if fused:
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
            if cfg.train_text_encoder or self._text_encoder_grad:
                ehs = self.text_encoder(self.input_ids)[0]
            else:
                with torch.no_grad():
                    ehs = self.text_encoder(self.input_ids)[0]
            if not fused:
                noisy = noisy.to(self.model_dtype).contiguous(memory_format=torch.channels_last)
            pred = self.unet(noisy, timesteps, ehs.to(self.model_dtype)).sample
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
            loss = fused_masked_mse(pred, target, m, w)
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
            loss.backward()
            if defer:
                ops.wgrad_flush()
        finally:
            ops.wgrad_defer_cancel()
        dropout_path.end_step()
        self.loss.copy_(loss.detach())

    def set_loss_mask(self, mask_image_res: torch.Tensor):
        """`batch["mask"]` of the PTI dataset (image resolution, [B,1,8h,8w] or anything that
        reshapes to it) -> nearest-neighbour resize to the latent grid, as cli_lora_pti.py:342-354
        does every step; stored in `self.mask` for `use_mask` steps."""
        b, _, h, w = self.mask.shape
        m = mask_image_res.to(self.device, torch.float32).reshape(b, 1, h * 8, w * 8)
        self.mask.copy_(F.interpolate(m, size=(h, w), mode="nearest"))

    def _update(self):
        cfg = self.cfg
        self.arena.step(cfg.adam_beta1, cfg.adam_beta2, cfg.adam_epsilon, cfg.adam_weight_decay,
                        cfg.max_grad_norm, world_size=self._world)

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
        return {"p": a.p.clone(), "m": a.m.clone(), "v": a.v.clone(), "step": a.step_dev.clone(),
                "loss": self.loss.clone(), "rng": torch.cuda.get_rng_state(self.device)}

    def _restore(self, snap):
        a = self.arena
        a.p.copy_(snap["p"]); a.m.copy_(snap["m"]); a.v.copy_(snap["v"]); a.step_dev.copy_(snap["step"])
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
        """Per-group learning rates of the step about to run (iteration self.global_step)."""
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

    def step_host(self, latents_cpu: torch.Tensor, input_ids_cpu: torch.Tensor) -> torch.Tensor:
        """End-to-end step from pinned host memory: H2D inputs, step, D2H loss (async, returns the
        pinned loss buffer; synchronise the stream before reading it)."""
        self.h_latents.copy_(latents_cpu)
        self.h_input_ids.copy_(input_ids_cpu)
        self.latents.copy_(self.h_latents, non_blocking=True)
        self.input_ids.copy_(self.h_input_ids, non_blocking=True)
        self.step_device()
        self.h_loss.copy_(self.loss, non_blocking=True)
        return self.h_loss

    def h2d_bytes(self) -> int:
        return self.h_latents.numel() * 4 + self.h_input_ids.numel() * 8

    def d2h_bytes(self) -> int:
        return 4


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
                 latent_shape=(1, 4, 64, 64), seq_len: int = 77, device=None):
        from .ti import TextualInversionRows
        _check_prediction_type(cfg)
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
                 row_capacity: int = 1024, latent_shape=(1, 4, 64, 64), seq_len: int = 77, device=None):
        from ._C import LoraB200Error
        from .embed_rows import MAX_SCATTER_TOKENS, MODES, EmbeddingRows
        from .dist import world_info
        if mode not in MODES:
            raise ValueError(f"mode {mode!r}: one of {MODES}")
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
        super().__init__(unet, text_encoder, cfg, latent_shape=latent_shape, seq_len=seq_len, device=device)
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
        base, rg = self.arena.base_lr, self.arena.rows_group
        if k < self.unfreeze_lora_step:          # train_lora_w_ti.py:988-991
            lrs = [0.0] * len(base)
            lrs[rg] = base[rg] * mult
        else:                                    # :992-995: LoRA at its base lr, table frozen
            lrs = list(base)
            lrs[rg] = 0.0
        self.arena.set_lr(lrs)

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

    def step_host(self, latents_cpu: torch.Tensor, input_ids_cpu: torch.Tensor) -> torch.Tensor:
        """LoraTrainStep.step_host; an overflow of the row slots in this step raises no later than the
        next call (the flag is copied to pinned memory behind the step and read one call later)."""
        out = super().step_host(latents_cpu, input_ids_cpu)
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
