"""Sampling from LoRA-patched models: the denoising loop of diffusers' StableDiffusionPipeline
(classifier-free guidance, Euler-ancestral or DDIM, the VAE decode and the uint8 post-processing) over
the same host models and fused LoRA kernels the training steps use.

    from lora_b200.sample import LoraSampler, SamplerConfig
    s = LoraSampler(unet, text_encoder, vae, SamplerConfig(scheduler="euler_ancestral", guidance_scale=7.0),
                    latent_shape=(B, 4, 64, 64), seq_len=77)
    s.prepare()
    img = s.sample(input_ids, negative_input_ids, seed=0)   # uint8 [B, 8h, 8w, 3] on the device

A `sample()` replays three CUDA graphs, with no host sync and no allocation between them:
  A  the sampled sites' down factors re-cast into the 16-bit operands graph B reads, the text encoder on
     [negative ; prompt] ids, and the init launch of lb_sample_step (x = z_0 * init_noise_sigma);
  B  one denoising step: the UNet at batch G*B, then lb_sample_step (guidance sum, the scheduler's update
     as folded coefficients, the next UNet input and timestep). Replayed N times: the step index lives
     on the device and the kernel advances it;
  C  the VAE decoder and lb_pixels_emit.
`use_cuda_graph=False` runs the same code eagerly. The number of steps (up to `max_steps`), the
scheduler, the guidance scale and the seed may change per call: they rewrite device tables. A guidance
scale <= 1 runs without the unconditional half (G = 1), as the pipeline does; that is a capture of its own.
The graphs are captured again only when something baked into a launch changes: a site's scale, a
selector, the set of sites or their parameter storage, the grouping policy (`captures` counts them).

All noise (z_0 and each step's z_i) is one draw of [N + 1, B, C, h, w] from the sampler's own
torch.Generator seeded by `seed`; the global CUDA RNG stream is never touched, so a training step's noise
is the same with or without sampling in between. The models run in eval() under no_grad and get their
train / eval modes back afterwards.
"""
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn as nn

from . import _C, ops
from .host import schedulers
from .step_ops import pixels_emit, sample_step

_SITE_NAMES = ("LoraInjectedLinear", "LoraInjectedConv2d")


@dataclass
class SamplerConfig:
    scheduler: str = "euler_ancestral"         # "euler_ancestral" | "ddim"
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


def _sites(*models):
    return [m for model in models for m in model.modules() if type(m).__name__ in _SITE_NAMES]


class LoraSampler:
    def __init__(self, unet: nn.Module, text_encoder: nn.Module, vae: nn.Module, cfg: SamplerConfig,
                 latent_shape=(1, 4, 64, 64), seq_len: int = 77, device=None):
        schedulers.check(cfg.scheduler, cfg.prediction_type)
        ucfg = getattr(unet, "cfg", None) or getattr(unet, "config", None)
        if getattr(ucfg, "addition_embed_type", None) is not None:
            raise ValueError("LoraSampler does not sample SDXL UNets (addition_embed_type "
                             f"{ucfg.addition_embed_type!r}): their pooled and time-id conditioning is not supported")
        B, C, h, w = latent_shape
        if getattr(ucfg, "in_channels", C) != C:
            raise ValueError(f"the UNet takes {ucfg.in_channels} input channels, the latents have {C}: inpainting "
                             "UNets are not sampled")
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
        self.table = torch.zeros((rows, schedulers.TABLE_COLS), device=dev, dtype=torch.float32)
        self.guidance = torch.zeros(1, device=dev, dtype=torch.float32)
        self.step_index = torch.zeros(1, device=dev, dtype=torch.int32)
        self._counter = torch.zeros(1, device=dev, dtype=torch.int32)
        self.timestep = torch.zeros(1, device=dev, dtype=torch.float32)
        self.unet_in = {G: torch.zeros((G * B, C, h, w), device=dev, dtype=self.model_dtype).contiguous(
            memory_format=torch.channels_last) for G in (1, 2)}
        self.vae_in = torch.zeros(latent_shape, device=dev, dtype=self.vae_dtype).contiguous(
            memory_format=torch.channels_last if vae_cl else torch.contiguous_format)
        self.image = torch.zeros((B, 8 * h, 8 * w, 3), device=dev, dtype=torch.uint8)
        self.generator = torch.Generator(device=dev)
        self._ehs = {}
        self._table_key = None
        self._graphs = {}             # G -> (A, B, C)
        self._fingerprint = None
        self._factor_bufs = []
        self.captures = 0

    # ------------------------------------------------------------------ what a capture bakes in
    def _fingerprint_now(self):
        """Everything of the models that a captured launch holds as a constant or an address."""
        from .grouping import get_grouping
        sig = []
        for m in _sites(self.unet, self.text_encoder):
            base = m.linear if hasattr(m, "linear") else m.conv
            sel = getattr(m.selector, "weight", None)
            sig.append((id(m), float(m.scale), m.r, id(sel), None if sel is None else sel.data_ptr(),
                        id(m.lora_down.weight), m.lora_down.weight.data_ptr(), m.lora_down.weight.dtype,
                        id(m.lora_up.weight), m.lora_up.weight.data_ptr(), m.lora_up.weight.dtype,
                        id(base.weight), base.weight.data_ptr()))
        return get_grouping(), tuple(sig)

    def _collect_factor_buffers(self):
        """The 16-bit padded down-factor copies the sites' forward reads (modules._SiteState.down): held
        here so that the addresses graph B captured stay valid, and re-cast by `_refresh_factors`."""
        bufs = []
        for m in _sites(self.unet, self.text_encoder):
            if m.r > ops.MAX_RANK:        # rank chunks cast their factors inside every forward
                continue
            tab = None
            if type(m).__name__ == "LoraInjectedConv2d":      # the tap-major row table of ops.conv_down16
                r, cin, kh, kw = m.lora_down.weight.shape
                taps, rp = kh * kw, ops.rank_pad(r)
                tab = torch.tensor([(t, cin * taps, taps, r, cin, t * cin, taps * cin, rp) for t in range(taps)],
                                   device=self.device, dtype=torch.int64)
            for dt, (_, buf) in list(m._lb.down.items()):
                bufs.append((m, dt, buf, tab))
        self._factor_bufs = bufs

    def _refresh_factors(self):
        """Re-cast every held down-factor copy from the factor's current value (an arena step, an
        in-place optimizer update and a `.data` edit all leave the fused forward's copy stale)."""
        for m, dt, buf, tab in self._factor_bufs:
            a = m.lora_down.weight.detach()
            if a.dtype != torch.float32 or not a.is_contiguous():
                a = a.float().contiguous()
            r = m.r
            if type(m).__name__ == "LoraInjectedLinear":
                K = a.shape[1]
                _C.check(_C.lib.lb_cast_rows_pad(_C.ptr(a), K, 1, _C.ptr(buf), r, buf.shape[0], K, _C.dtype_code(dt),
                                                 _C.stream_ptr()), "lb_cast_rows_pad")
            else:
                _, cin, kh, kw = a.shape
                _C.check(_C.lib.lb_refresh_shadows(_C.ptr(a), _C.ptr(tab), kh * kw, cin, _C.ptr(buf),
                                                   _C.dtype_code(dt), _C.stream_ptr()), "lb_refresh_shadows")
            ops._count()

    # ------------------------------------------------------------------ the three bodies
    def _autocast(self):
        dt = self.cfg.autocast_dtype
        return torch.autocast("cuda", dtype=dt) if dt is not None else torch.autocast("cuda", enabled=False)

    def _body_a(self, G: int):
        self._refresh_factors()
        B = self.latents.shape[0]
        ids = self.input_ids if G == 2 else self.input_ids[B:]
        with self._autocast():
            self._ehs[G] = self.text_encoder(ids)[0].to(self.model_dtype)
        sample_step(None, self.latents, self.noise, self.table, None, self.step_index, self._counter,
                    self.unet_in[G], self.timestep, None, self.cfg.vae_scaling, init=True)

    def _body_b(self, G: int):
        with self._autocast():
            out = self.unet(self.unet_in[G], self.timestep, self._ehs[G]).sample
        sample_step(out, self.latents, self.noise, self.table, self.guidance, self.step_index, self._counter,
                    self.unet_in[G], self.timestep, self.vae_in, self.cfg.vae_scaling)

    def _body_c(self):
        pixels_emit(self.vae.decode(self.vae_in).sample, self.image)

    def _run_eager(self, G: int, n: int):
        self._collect_factor_buffers()
        self._body_a(G)
        for _ in range(n):
            self._body_b(G)
        self._body_c()

    # ------------------------------------------------------------------ capture
    def _capture(self, G: int):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(max(1, self.cfg.graph_warmup)):
                self._run_eager(G, 1)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self._collect_factor_buffers()
        ga = torch.cuda.CUDAGraph()
        with torch.cuda.graph(ga):
            self._body_a(G)
        gb = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gb, pool=ga.pool()):
            self._body_b(G)
        gc = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gc, pool=ga.pool()):
            self._body_c()
        torch.cuda.synchronize()
        self._graphs[G] = (ga, gb, gc)
        self.captures += 1

    def _graphs_for(self, G: int):
        fp = self._fingerprint_now()
        if fp != self._fingerprint:
            self._graphs.clear()
            self._fingerprint = fp
        if G not in self._graphs:
            self._capture(G)
        return self._graphs[G]

    # ------------------------------------------------------------------ modes
    def _enter_eval(self):
        saved = [(m, m.training) for model in (self.unet, self.text_encoder, self.vae) for m in model.modules()]
        for model in (self.unet, self.text_encoder, self.vae):
            model.eval()
        return saved

    @staticmethod
    def _restore_modes(saved):
        for m, training in saved:
            m.training = training

    # ------------------------------------------------------------------ public API
    def _options(self, num_inference_steps, scheduler, guidance_scale):
        cfg = self.cfg
        n = cfg.num_inference_steps if num_inference_steps is None else int(num_inference_steps)
        sched = cfg.scheduler if scheduler is None else scheduler
        g = cfg.guidance_scale if guidance_scale is None else float(guidance_scale)
        schedulers.check(sched, cfg.prediction_type)
        if not 1 <= n <= cfg.max_steps:
            raise ValueError(f"num_inference_steps {n}: need 1 <= n <= max_steps ({cfg.max_steps})")
        return n, sched, g

    def _set_table(self, sched: str, n: int):
        key = (sched, n)
        if key != self._table_key:
            self.table.copy_(schedulers.pack_table(sched, self.cfg.prediction_type, n, self.cfg.max_steps))
            self._table_key = key

    def prepare(self, guidance_scale: Optional[float] = None):
        """Capture the graphs for the configured (or given) guidance scale ahead of the first sample()."""
        if not self.cfg.use_cuda_graph:
            return
        _, _, g = self._options(None, None, guidance_scale)
        saved = self._enter_eval()
        try:
            with torch.no_grad():
                self._set_table(self.cfg.scheduler, self.cfg.num_inference_steps)
                self._graphs_for(2 if g > 1.0 else 1)
        finally:
            self._restore_modes(saved)

    def sample(self, input_ids: torch.Tensor, negative_input_ids: Optional[torch.Tensor] = None, seed: int = 0,
               num_inference_steps: Optional[int] = None, scheduler: Optional[str] = None,
               guidance_scale: Optional[float] = None) -> torch.Tensor:
        """uint8 [B, 8h, 8w, 3] images (a view of `self.image`, overwritten by the next call) for the token
        ids [B, seq_len] of the prompts and of the negative prompts (the empty prompt's ids for plain
        classifier-free guidance; unused when guidance_scale <= 1). `self.latents` holds the final latents."""
        n, sched, g = self._options(num_inference_steps, scheduler, guidance_scale)
        G = 2 if g > 1.0 else 1
        B = self.latents.shape[0]
        if tuple(input_ids.shape) != tuple(self.input_ids[B:].shape):
            raise ValueError(f"input_ids of shape {tuple(input_ids.shape)}: the sampler takes "
                             f"{tuple(self.input_ids[B:].shape)}")
        if G == 2 and (negative_input_ids is None or tuple(negative_input_ids.shape) != tuple(input_ids.shape)):
            raise ValueError("guidance_scale > 1 needs negative_input_ids of the prompts' shape")
        saved = self._enter_eval()
        try:
            with torch.no_grad():
                self._set_table(sched, n)
                self.guidance.fill_(g)
                self.input_ids[B:].copy_(input_ids)
                if G == 2:
                    self.input_ids[:B].copy_(negative_input_ids)
                if not self.cfg.external_noise:
                    self.generator.manual_seed(int(seed))
                    self.noise[:n + 1].normal_(generator=self.generator)
                if self.cfg.use_cuda_graph:
                    ga, gb, gc = self._graphs_for(G)
                    ga.replay()
                    for _ in range(n):
                        gb.replay()
                    gc.replay()
                else:
                    self._run_eager(G, n)
        finally:
            self._restore_modes(saved)
        return self.image
