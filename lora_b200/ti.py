"""Pivotal-tuning phase 1: textual inversion of a few placeholder tokens.

Restates what `train_inversion` does to the embedding table each step
(lora_diffusion/cli_lora_pti.py:373-542: AdamW over the input-embedding table, the norm "decay" of
the new rows :451-468, then `weight[index_no_updates] = orig[index_no_updates]` :477-479) without
touching the other 49 k rows: the trained rows live in a small fp32 Parameter `rows [n, D]`, a
forward hook on the embedding module substitutes them into the lookup (so autograd produces an
[n, D] gradient instead of a dense 49408 x 768 one), and one kernel (`lb_ti_embed_step`) does
AdamW + norm decay + write-back into the table (which stays what `save_all` reads).
"""
from typing import List, Sequence

import torch
import torch.nn as nn

from . import _C, ops
from ._C import check, dtype_code, ptr, stream_ptr


class TextualInversionRows(nn.Module):
    def __init__(self, text_encoder: nn.Module, token_ids: Sequence[int], lr: float = 5e-4,
                 betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0,
                 clip_ti_decay: bool = True, target_norm: float = 0.4):
        super().__init__()
        emb = text_encoder.get_input_embeddings()
        table = emb.weight
        if not table.is_cuda:
            raise _C.LoraB200Error("TextualInversionRows needs the text encoder on a CUDA device")
        self.emb = [emb]                     # not a registered submodule (owned by the text encoder)
        self.token_ids = torch.tensor(list(token_ids), device=table.device, dtype=torch.int64)
        self.rows = nn.Parameter(table.detach()[self.token_ids].float().clone())
        self.rows.grad = torch.zeros_like(self.rows)
        self.m = torch.zeros_like(self.rows.data)
        self.v = torch.zeros_like(self.rows.data)
        self.lr = torch.tensor([float(lr)], device=table.device, dtype=torch.float32)
        self.step_dev = torch.zeros(1, device=table.device, dtype=torch.int32)
        self.betas, self.eps, self.wd = betas, eps, weight_decay
        self.clip_ti_decay, self.target_norm = clip_ti_decay, target_norm
        self._hook = emb.register_forward_hook(self._substitute)

    def _substitute(self, module, inputs, out):
        ids = inputs[0]
        for j in range(self.token_ids.numel()):
            hit = (ids == self.token_ids[j]).unsqueeze(-1)
            out = torch.where(hit, self.rows[j].to(out.dtype), out)
        return out

    @torch.no_grad()
    def sync_replicas(self, src: int = 0):
        """Broadcast rank `src`'s trained rows, and the table rows they were taken from, to every
        rank (DDP's parameter broadcast). A no-op outside torch.distributed."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
            return
        table = self.emb[0].weight
        src_rows = table.detach()[self.token_ids].contiguous()
        dist.broadcast(src_rows, src=src)
        table.data[self.token_ids] = src_rows
        dist.broadcast(self.rows.data, src=src)

    def set_lr(self, lr: float):
        self.lr.fill_(float(lr))

    @torch.no_grad()
    def step(self):
        """AdamW + norm decay on the trained rows, written back into the embedding table; zero_grad."""
        table = self.emb[0].weight
        n, D = self.rows.shape
        check(_C.lib.lb_ti_embed_step(ptr(self.rows.data), ptr(self.rows.grad), ptr(self.m), ptr(self.v),
                                      ptr(self.token_ids), ptr(table.data), dtype_code(table.dtype), n, D,
                                      ptr(self.lr), self.betas[0], self.betas[1], self.eps, self.wd,
                                      ptr(self.step_dev), 1 if self.clip_ti_decay else 0,
                                      float(self.target_norm), stream_ptr()), "lb_ti_embed_step")
        ops._count(2)

    def remove(self):
        self._hook.remove()
