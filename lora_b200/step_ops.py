"""The two ends of a training step as single kernels (csrc/step_glue.cu):

  step_prologue     scheduler.add_noise + cast to the model dtype + NCHW -> channels_last
                    (+ the 9-channel inpainting concat)   cli_lora_pti.py:295-313
                    (+ the v-prediction target scheduler.get_velocity, cli_lora_pti.py:333-338)
  fused_masked_mse  (mask-weighted) MSE and its gradient w.r.t. the prediction in one pass
                    cli_lora_pti.py:340-370, train_lora_dreambooth.py:855-875

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


class _MaskedMSE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target, mask, weights, scratch):
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
                                           stream_ptr()), "lb_masked_mse_fwd_bwd")
        ops._count()
        ctx.save_for_backward(grad)
        return loss

    @staticmethod
    def backward(ctx, gl):
        (grad,) = ctx.saved_tensors
        return grad * gl.to(grad.dtype), None, None, None, None


_SCRATCH = {}


def _scratch(device):
    s = _SCRATCH.get(device)
    if s is None:
        s = (torch.zeros(64, device=device, dtype=torch.float32), torch.zeros(1, device=device, dtype=torch.int32))
        _SCRATCH[device] = s
    return s


def fused_masked_mse(pred: torch.Tensor, target: torch.Tensor, mask: Optional[torch.Tensor] = None,
                     weights: Optional[torch.Tensor] = None) -> torch.Tensor:
    """sum_b weights[b] * mean_{c,h,w}((mask (pred - target))^2)  (weights None: 1/B), differentiable
    w.r.t. pred; mask [B,1,H,W] is the already-normalised weighting of cli_lora_pti.py:356-364."""
    return _MaskedMSE.apply(pred, target, mask, weights, _scratch(pred.device))


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
