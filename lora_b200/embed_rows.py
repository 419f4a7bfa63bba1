"""Token-embedding rows trained together with the LoRA factors: sparse, exact AdamW over the table.

The reference trains the whole CLIP token-embedding table (49408 x 768 fp32) in the same AdamW as
the LoRA factors, with one clip_grad_norm_ over both:
  lora_diffusion/cli_lora_pti.py:958-997, 545-620   `continue_inversion` (mode "table": every row
      decays by fl32(1 - lr*wd) each step, every row that ever had a gradient keeps moving)
  training_scripts/train_lora_w_ti.py:830-853, 986-1075   (mode "placeholders": every row except
      the placeholders is restored from the original table after each update)
Only the few hundred rows of tokens that occur in the batches ever get a gradient. Here those rows
are *claimed* into fixed slots that form one more param-group of the LoraArena (fp32 master, m, v,
gradient), so the arena's single optimizer launch clips and updates them with the factors:

  forward   a hook on the embedding module wraps its output in an autograd Function; the table
            itself keeps requires_grad=False
  backward  lb_embed_rows_scatter sums each distinct token's gradient rows into its slot and claims
            slots for tokens seen for the first time (master = stored row * pending decay)
  update    the arena's optimizer launch (unchanged)
  after     lb_embed_rows_write_back copies the claimed masters (mode "placeholders": the
            placeholder slots only) into the table and advances the pending decay
  flush     lb_embed_rows_flush applies the pending decay to every unclaimed row (mode "table";
            call it before reading the table outside the step)

An unclaimed row has zero gradient and zero moments, so dense AdamW only scales it by the step's
decay factor; its stored value times the pending decay is exactly what dense AdamW holds. In the
step where a token is seen for the first time, the forward reads its stored row, which still lacks
the pending decay (a relative difference of 1 - decay, about steps * lr * wd); its master, and so
every later step, starts from the decayed value.
"""
from typing import Sequence

import torch
import torch.nn as nn

from . import _C, ops
from ._C import check, dtype_code, ptr, stream_ptr

MODES = ("table", "placeholders")


class _Lookup(torch.autograd.Function):
    """Identity on the lookup output; its backward is the sparse embedding backward."""

    @staticmethod
    def forward(ctx, anchor, out, ids, rows):
        ctx.ids, ctx.rows = ids, rows
        return out.view_as(out)

    @staticmethod
    def backward(ctx, grad_out):
        ctx.rows._scatter(ctx.ids, grad_out)
        return None, None, None, None


class EmbeddingRows:
    """Row state of the jointly trained embedding table: slot map (token -> slot, int32 [V]), slot
    list (slot -> token), pending decay (fp64), overflow flag, placeholder ids. `arena` must have been
    built with rows=(capacity, D, lr); the placeholder rows take the first slots at construction."""

    def __init__(self, text_encoder: nn.Module, arena, placeholder_token_ids: Sequence[int],
                 mode: str = "table", weight_decay: float = 1e-2):
        if mode not in MODES:
            raise ValueError(f"mode {mode!r}: one of {MODES}")
        if arena.rows_group is None:
            raise _C.LoraB200Error("EmbeddingRows needs a LoraArena built with rows=(capacity, D, lr)")
        emb = text_encoder.get_input_embeddings()
        table = emb.weight
        if not table.is_cuda:
            raise _C.LoraB200Error("EmbeddingRows needs the text encoder on a CUDA device")
        V, D = table.shape
        cap, width = arena.rows_shape
        if width != D:
            raise _C.LoraB200Error(f"EmbeddingRows: arena rows are {width} wide, the table is {D}")
        ph = [int(t) for t in placeholder_token_ids]
        if len(set(ph)) != len(ph) or any(t < 0 or t >= V for t in ph):
            raise ValueError(f"placeholder ids {ph} must be distinct ids in [0, {V})")
        if len(ph) > cap:
            raise _C.LoraB200Error(f"EmbeddingRows: {len(ph)} placeholders exceed the capacity {cap}")
        self.emb = [emb]                     # owned by the text encoder, not a submodule here
        self.arena, self.mode, self.weight_decay = arena, mode, float(weight_decay)
        self.V, self.D, self.capacity = V, D, cap
        self.placeholder_ids = ph
        dev = table.device
        table.requires_grad_(False)
        self.slot_of = torch.full((V,), -1, device=dev, dtype=torch.int32)
        self.slot_tok = torch.full((cap,), -1, device=dev, dtype=torch.int32)
        self.state = torch.zeros(4, device=dev, dtype=torch.int32)
        self.decay = torch.ones(1, device=dev, dtype=torch.float64)
        if ph:                               # the reference moves them every step, seen or not
            idx = torch.tensor(ph, device=dev, dtype=torch.long)
            self.slot_of[idx] = torch.arange(len(ph), device=dev, dtype=torch.int32)
            self.slot_tok[: len(ph)] = idx.to(torch.int32)
            arena.rows_view(arena.p)[: len(ph)] = table.detach()[idx].float()
            self.state[:2] = len(ph)
        self._anchor = torch.zeros((), device=dev, requires_grad=True)
        self._hook = emb.register_forward_hook(self._wrap)

    # ------------------------------------------------------------------ step pieces
    def _wrap(self, module, inputs, out):
        if not torch.is_grad_enabled():
            return out
        return _Lookup.apply(self._anchor, out, inputs[0], self)

    def _scatter(self, ids: torch.Tensor, grad_out: torch.Tensor):
        a = self.arena
        ids = ids.reshape(-1)
        if ids.dtype != torch.int64:
            ids = ids.long()
        g = grad_out.reshape(-1, self.D).contiguous()
        table = self.emb[0].weight
        check(_C.lib.lb_embed_rows_scatter(ptr(ids.contiguous()), ptr(g), dtype_code(g.dtype), ids.numel(), self.D,
                                           self.V, ptr(self.slot_of), ptr(self.slot_tok), self.capacity,
                                           ptr(self.state), ptr(table.data), dtype_code(table.dtype),
                                           ptr(self.decay), ptr(a.rows_view(a.p)), ptr(a.rows_view(a.g)),
                                           stream_ptr()), "lb_embed_rows_scatter")
        ops._count(1)

    def write_back(self):
        """After the optimizer launch: updated masters into the table, pending decay advanced."""
        a = self.arena
        table = self.emb[0].weight
        decays = self.mode == "table"
        check(_C.lib.lb_embed_rows_write_back(ptr(a.rows_view(a.p)), ptr(self.slot_tok), self.capacity,
                                              ptr(self.state), -1 if decays else len(self.placeholder_ids),
                                              ptr(table.data), dtype_code(table.dtype), self.D, self.V,
                                              ptr(self.decay) if decays else None,
                                              ptr(a.lr) if decays else None, a.rows_group,
                                              self.weight_decay, stream_ptr()), "lb_embed_rows_write_back")
        ops._count(1)

    def flush(self):
        """Apply the pending decay to every unclaimed row (the table then equals dense AdamW's), then
        check the overflow flag. Mode "placeholders" never decays unclaimed rows: only the check."""
        if self.mode == "table":
            table = self.emb[0].weight
            check(_C.lib.lb_embed_rows_flush(ptr(table.data), dtype_code(table.dtype), self.V, self.D,
                                             ptr(self.slot_of), ptr(self.decay), ptr(self.state), stream_ptr()),
                  "lb_embed_rows_flush")
            ops._count(1)
        self.check()

    def check(self):
        """Raise if a token found no free slot (synchronises the stream)."""
        self.raise_for_flags(int(self.state[3].item()))

    def raise_for_flags(self, flags: int):
        if flags & 1:
            raise _C.LoraB200Error(
                f"EmbeddingRows: more than {self.capacity} distinct tokens were seen; the gradient of the "
                "tokens past the capacity was dropped (raise row_capacity)")
        if flags & 2:
            raise _C.LoraB200Error(f"EmbeddingRows: a token id outside [0, {self.V}) reached the embedding")

    def claimed(self) -> int:
        return int(self.state[0].item())

    def slot_tokens(self) -> torch.Tensor:
        """Claimed tokens in slot order (synchronises)."""
        return self.slot_tok[: self.claimed()].long()

    # ------------------------------------------------------------------ snapshot (CUDA-graph warm-up)
    def snapshot(self):
        return {"table": self.emb[0].weight.detach().clone(), "slot_of": self.slot_of.clone(),
                "slot_tok": self.slot_tok.clone(), "state": self.state.clone(), "decay": self.decay.clone()}

    def restore(self, snap):
        with torch.no_grad():
            self.emb[0].weight.copy_(snap["table"])
        self.slot_of.copy_(snap["slot_of"]); self.slot_tok.copy_(snap["slot_tok"])
        self.state.copy_(snap["state"]); self.decay.copy_(snap["decay"])

    def remove(self):
        self._hook.remove()
