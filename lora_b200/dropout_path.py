"""Keep-mask seeds of the LoRA sites with an ACTIVE nn.Dropout on the branch (module.training and
p > 0): the default state of every operator built by inject_trainable_lora_extended and by the
monkeypatch_* loaders (class default dropout_p = 0.1, fresh modules are in training mode;
lora.py:34,84,334-356,689-694). The sites' own autograd functions (modules._FusedLoraLinearFn,
conv_path._FusedLoraConv2dFn) run the masked forms described here; this module hands out the seeds.

    y = base(x) + mask o (up(sel(down(x)))) / (1-p) * scale            (lora.py:53-58, 130-135)

The mask sits between the up-projection and the sum, so the branch cannot be accumulated into the
base accumulator -- but it still never leaves the SM: the fused kernel gives the LoRA product
T'.U^T its own accumulator and applies keep(m,n)/(1-p) while the tile is drained
(lb_lora_linear_fwd_dropout / lb_lora_conv2d_fwd_dropout; csrc/fused_core.cuh, DROP): ONE launch,
no extra pass over Y. Backward recomputes the same counter-based mask: one masked pass over gY gives
dTs = (mask o gY / (1-p)) . B (lb_lora_dropout_dt), and the plain dX kernel takes its rank-r
activations from dTs (T_in) instead of computing gY . B; dA reduces X against dTs, and dB uses the
masked reduction (lb_lora_wgrad_masked).

The keep-mask is a hash of (per-call device seed, element index; csrc/dropmask.cuh) -- NOT ATen's Philox stream, so
parity with the reference under dropout is distributional (keep probability, 1/(1-p) scaling,
forward/backward mask consistency; tests/test_dropout_gpu.py), not bitwise.
"""
from collections import deque

import torch


class _SeedPool:
    """One device-side draw of mask seeds per training step instead of one tiny RNG launch per
    dropout site (224 sites in the extended SD1.5 set): the step engine calls `begin_step`, every
    dropout forward takes the next int64 slot (a 1-element view: the kernels read the seed through
    a device pointer, so a captured graph re-reads freshly drawn values on every replay).

    Gradient checkpointing runs a site's forward a second time inside the backward pass. That
    recompute must draw the keep-mask its first forward drew -- the rest of the network consumed
    that output -- so every forward records the slot it took (`taken`, per site, in call order) and
    a forward that runs inside the backward pass takes the site's oldest recorded slot instead of a
    new one. This holds whoever called torch.utils.checkpoint (the host UNet, transformers' CLIP, a
    caller's own model). Without a step engine the seeds come from torch's CUDA generator, whose
    state torch.utils.checkpoint restores before a recompute (preserve_rng_state, its default)."""
    pool = None
    used = 0
    taken = {}        # id(site module) -> deque of the slots its forwards took this step


def begin_step(device, n_slots: int = 1024):
    """Draw this step's mask seeds (graph-capturable: torch's CUDA generator, new values per replay)."""
    _SeedPool.pool = torch.randint(0, 2 ** 62, (n_slots,), device=device, dtype=torch.int64)
    _SeedPool.used = 0
    _SeedPool.taken = {}


def end_step():
    _SeedPool.pool = None
    _SeedPool.used = 0
    _SeedPool.taken = {}


def _in_backward() -> bool:
    """True while the autograd engine runs a backward pass on this thread: a forward called now is a
    gradient-checkpointing recompute."""
    return torch._C._current_graph_task_id() != -1


def _fresh_seed(mod, device) -> torch.Tensor:
    pool = _SeedPool.pool
    if pool is not None and pool.device == device:
        recompute = _in_backward()
        if recompute:
            slots = _SeedPool.taken.get(id(mod))
            if slots:
                i = slots.popleft()
                return pool[i:i + 1]
        if _SeedPool.used < pool.numel():
            i = _SeedPool.used
            _SeedPool.used = i + 1
            if not recompute:
                _SeedPool.taken.setdefault(id(mod), deque()).append(i)
            return pool[i:i + 1]
    # no step engine around this call: drawn on the device from torch's CUDA generator
    return torch.randint(0, 2 ** 62, (1,), device=device, dtype=torch.int64)
