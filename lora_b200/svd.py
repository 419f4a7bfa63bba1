"""SVD distillation of a fine-tune into LoRA factors, batched on the GPU.

Contract = /root/reference/lora_diffusion/cli_svd.py:24-142 (`overwrite_base`, `svd_distill`):
per LoRA site, dW = (W_tuned - W_base) (conv: flattened to [Cout, Cin*kh*kw]), keep the top `rank`
singular triplets, up = U_r diag(S_r), down = Vh_r, clamp both symmetrically at the
`clamp_quantile` quantile of their joint values, write them into lora_up / lora_down.

The reference loops over sites calling a full `torch.linalg.svd`. Here ALL sites of a model,
whatever their shapes, go through ONE C call (csrc/svd_batched.cu: lb_svd_truncated_batched --
randomized range finder, 32 probes, q power iterations re-orthonormalised through a 32x32 Jacobi
eigen-solve, exact quantile clamp): the only passes over the weights are 2(q+1) streaming reads of
(W_tuned, W_base), q = 1 by default (4 passes), with the contraction on the tensor cores
(3-term split-bf16, fp32-faithful).

Singular vectors are unique up to a per-component sign, and the reference's clamp threshold is a
quantile over SIGNED values, so elementwise equality with LAPACK is not defined;
parity is stated on singular values, on the rank-r product before clamping and on the clamp rule
(tests/test_svd_gpu.py).
"""
import ctypes
from collections import defaultdict
from typing import List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from . import _C, ops
from ._C import check, dtype_code, ptr, stream_ptr

L = 32


def svd_lowrank_ragged(W_tuned: Sequence[torch.Tensor], W_base: Sequence[torch.Tensor], rank: int,
                       power_iters: int = 1, clamp_quantile: Optional[float] = None, seed: int = 0):
    """ONE C call (lb_svd_truncated_batched) for any mix of 2-D weight shapes of one dtype
    (fp32 / bf16 / fp16): returns ([up_b [N_b, rank] = U_r diag(S_r)], [down_b [rank, K_b] = Vh_r],
    sigma [batch, 32] descending, hi [batch] or None). With clamp_quantile the reference's clamp
    (cli_svd.py:43-47) is applied in the same call (exact radix-select quantile per matrix)."""
    if not 1 <= rank <= 16:
        raise _C.LoraB200Error("svd_lowrank: rank must be in [1,16]")
    batch = len(W_tuned)
    if batch == 0:
        return [], [], None, None
    w0 = W_tuned[0]
    if not w0.is_cuda:
        raise _C.LoraB200Error("svd_lowrank needs CUDA tensors (no CPU path)")
    dev = w0.device
    keep_t = [t.detach().contiguous() for t in W_tuned]
    keep_b = [t.detach().contiguous() for t in W_base]
    for t, bt in zip(keep_t, keep_b):
        assert t.dim() == 2 and t.shape == bt.shape and t.dtype == w0.dtype and bt.dtype == w0.dtype
    Ns = [int(t.shape[0]) for t in keep_t]
    Ks = [int(t.shape[1]) for t in keep_t]
    IA = ctypes.c_int * batch
    VP = ctypes.c_void_p * batch
    n_arr, k_arr = IA(*Ns), IA(*Ks)
    wt_arr = VP(*[t.data_ptr() for t in keep_t])
    wb_arr = VP(*[t.data_ptr() for t in keep_b])
    wdt = dtype_code(w0.dtype)
    lib = _C.lib
    ws_bytes = int(lib.lb_svd_workspace_bytes(n_arr, k_arr, batch, wdt))
    if ws_bytes <= 0:
        raise _C.LoraB200Error(f"lb_svd_workspace_bytes failed: {ws_bytes}")
    ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
    offs, total = [], 0
    for n, k in zip(Ns, Ks):
        offs.append(total)
        total += rank * (n + k)
    out = torch.empty(total, device=dev, dtype=torch.float32)
    sigma = torch.empty((batch, L), device=dev, dtype=torch.float32)
    do_clamp = clamp_quantile is not None and clamp_quantile > 0.0
    hi = torch.empty(batch, device=dev, dtype=torch.float32) if do_clamp else None
    check(lib.lb_svd_truncated_batched(wt_arr, wb_arr, n_arr, k_arr, batch, wdt, rank, int(power_iters),
                                       float(clamp_quantile) if do_clamp else -1.0,
                                       ctypes.c_ulonglong(seed * 2654435761 + 12345), ptr(out), ptr(sigma),
                                       ptr(hi), ptr(ws), ws_bytes, stream_ptr()),
          "lb_svd_truncated_batched")
    # launches: probes + (2q+2) passes + Gram/Jacobi/transform stages + factors x2 (+ clamp)
    ops._count(1 + (2 * power_iters + 2) + 6 * power_iters + 7 + 2 + (1 if do_clamp else 0))
    ups = [out[o:o + rank * n].view(n, rank) for o, n in zip(offs, Ns)]
    downs = [out[o + rank * n:o + rank * (n + k)].view(rank, k) for o, n, k in zip(offs, Ns, Ks)]
    return ups, downs, sigma, hi


def svd_lowrank_batched(W_tuned: Sequence[torch.Tensor], W_base: Sequence[torch.Tensor], rank: int,
                        power_iters: int = 1, seed: int = 0, jacobi_sweeps: int = 10
                        ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Same-shape 2-D weight pairs -> (up [b,N,rank] = U_r diag(S_r), down [b,rank,K] = Vh_r,
    sigma [b,32] descending). Weights may be fp32 / bf16 / fp16 (all the same dtype)."""
    ups, downs, sigma, _ = svd_lowrank_ragged(W_tuned, W_base, rank, power_iters=power_iters, seed=seed)
    return torch.stack(ups), torch.stack(downs), sigma


def _clamp_pair_(up: torch.Tensor, down: torch.Tensor, q: float):
    """cli_svd.py:42-47: hi = quantile(cat(U, Vh), q); clamp both to [-hi, hi] (in place)."""
    hi = torch.quantile(torch.cat([up.flatten(), down.flatten()]), q)
    up.clamp_(-hi, hi)
    down.clamp_(-hi, hi)
    return hi


def _iter_lora(model):
    for m in model.modules():
        if type(m).__name__ in ("LoraInjectedLinear", "LoraInjectedConv2d"):
            yield m


def overwrite_base(base_model: nn.Module, tuned_model: nn.Module, rank: int, clamp_quantile: float,
                   power_iters: int = 1, shard: Optional[Tuple[int, int]] = None):
    """cli_svd.py:24-92 on two LoRA-injected models with identical site structure: the factors of
    `base_model`'s sites are overwritten with the rank-`rank` distillation of (tuned - base).

    shard=(rank, world) (svd distillation on several GPUs): the weight deltas are
    independent, so this process distils only sites i = rank (mod world) in traversal order -- no
    collective on the compute path -- and the factors are then exchanged with ONE SUM all-reduce
    over a zero-initialised flat fp32 buffer in which every rank has filled only its own slots
    (exact: each slot receives one value plus zeros). Every rank ends with all sites overwritten."""
    sites = list(zip(_iter_lora(base_model), _iter_lora(tuned_model)))
    me, world = shard if shard is not None else (0, 1)
    groups = defaultdict(list)
    for i, (sb, st_) in enumerate(sites):
        if i % world != me:
            continue
        hb = sb.linear if hasattr(sb, "linear") else sb.conv
        ht = st_.linear if hasattr(st_, "linear") else st_.conv
        wb, wt = hb.weight.data, ht.weight.data
        groups[wb.dtype].append((sb, wb.flatten(start_dim=1), wt.flatten(start_dim=1)))
    for _, items in groups.items():
        # every site of this dtype -- whatever its shape -- in ONE call, clamp included
        ups, downs, _, _ = svd_lowrank_ragged([x[2] for x in items], [x[1] for x in items], rank,
                                              power_iters=power_iters, clamp_quantile=clamp_quantile)
        for (site, _, _), u, d in zip(items, ups, downs):
            dev, dt = site.lora_up.weight.device, site.lora_up.weight.dtype
            assert site.lora_up.weight.flatten(1).shape == u.shape
            assert site.lora_down.weight.flatten(1).shape == d.shape
            site.lora_up.weight.data = u.reshape(site.lora_up.weight.shape).to(device=dev, dtype=dt)
            site.lora_down.weight.data = d.reshape(site.lora_down.weight.shape).to(device=dev, dtype=dt)
    if world > 1:
        _exchange_factors([sb for sb, _ in sites], me, world)


def _exchange_factors(sites, me: int, world: int):
    """Every rank holds valid factors for sites i = me (mod world); after this every rank holds all."""
    from .dist import allreduce_sum_
    tensors = [t for s in sites for t in (s.lora_up.weight, s.lora_down.weight)]
    owners = [i % world for i in range(len(sites)) for _ in range(2)]
    flat = torch.zeros(sum(t.numel() for t in tensors), dtype=torch.float32, device=tensors[0].device)
    off = 0
    for t, owner in zip(tensors, owners):
        if owner == me:
            flat[off:off + t.numel()] = t.data.flatten().float()
        off += t.numel()
    allreduce_sum_(flat)
    off = 0
    for t in tensors:
        t.data = flat[off:off + t.numel()].reshape(t.shape).to(t.dtype)
        off += t.numel()


def svd_distill(unet_base: nn.Module, unet_tuned: nn.Module, text_base: nn.Module, text_tuned: nn.Module,
                rank: int = 4, clamp_quantile: float = 0.99, save_path: str = "svd_distill.safetensors",
                shard: Optional[Tuple[int, int]] = None):
    """cli_svd.py:95-142 with module arguments instead of hub ids (diffusers pipelines cannot be
    loaded offline): inject (extended for the UNet, CLIPAttention for the text encoder), distill,
    save with save_all (which, like the reference, writes only the default-target UNet sites)."""
    from .inject import inject_trainable_lora, inject_trainable_lora_extended
    from .persist import save_all
    inject_trainable_lora_extended(unet_base, r=rank)
    inject_trainable_lora_extended(unet_tuned, r=rank)
    overwrite_base(unet_base, unet_tuned, rank=rank, clamp_quantile=clamp_quantile, shard=shard)
    inject_trainable_lora(text_base, r=rank, target_replace_module={"CLIPAttention"})
    inject_trainable_lora(text_tuned, r=rank, target_replace_module={"CLIPAttention"})
    overwrite_base(text_base, text_tuned, rank=rank, clamp_quantile=clamp_quantile, shard=shard)
    if shard is not None and shard[0] != 0:
        return                              # sharded run: every rank holds all factors, rank 0 writes
    save_all(unet=unet_base, text_encoder=text_base, placeholder_token_ids=None, placeholder_tokens=None,
             save_path=save_path, save_lora=True, save_ti=False)
