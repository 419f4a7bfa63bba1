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
            (data parallel: lb_embed_rows_scatter_dp claims over the union of every rank's ids, in
            rank order, so that every rank's slots hold the same tokens; see enable_data_parallel)
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
import ctypes
from typing import Sequence

import torch
import torch.nn as nn

from . import _C, ops
from ._C import check, dtype_code, ptr, stream_ptr

MODES = ("table", "placeholders")
# tokens one scatter launch can take: B * S, times the world size under data parallelism
MAX_SCATTER_TOKENS = 2048


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

    # ------------------------------------------------------------------ data parallel
    def sync_replicas(self, src: int = 0):
        """Broadcast rank `src`'s table and row state (slot map, slot list, counters, pending decay,
        the rows' masters) to every rank: the common starting point DDP's parameter broadcast gives
        the reference. A no-op outside torch.distributed."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
            return
        a = self.arena
        for buf in (self.emb[0].weight.data, self.slot_of, self.slot_tok, self.state, self.decay, a.rows_view(a.p)):
            dist.broadcast(buf, src=src)

    def enable_data_parallel(self, ids: torch.Tensor, peer: bool) -> bool:
        """Collective: from now on the scatter claims slots over the union of every rank's `ids`
        (the step's static [B, S] input buffer; the embedding must see exactly that buffer), in rank
        order, so every rank's rows group holds the same tokens in the same slots.
        peer=True: the peers' id buffers and a one-word flag per rank are mapped over CUDA IPC
        (arena.map_peer_tensors) and read inside the scatter launch, after a flag handshake.
        Otherwise, or when a mapping fails on any rank: `gather_ids()` (one NCCL all-gather into a
        static [world * B, S] buffer) must run before each step's backward. Returns whether the peer
        path is in use (the same on every rank)."""
        import torch.distributed as dist
        world, rank = dist.get_world_size(), dist.get_rank()
        n = ids.numel()
        if ids.dtype != torch.int64 or not ids.is_contiguous():
            raise _C.LoraB200Error("EmbeddingRows.enable_data_parallel: ids must be a contiguous int64 buffer")
        if world * n > MAX_SCATTER_TOKENS:
            raise _C.LoraB200Error(f"EmbeddingRows: {world} ranks x {n} tokens exceed the scatter's limit of "
                                   f"{MAX_SCATTER_TOKENS} tokens per step")
        dev = ids.device
        VP = ctypes.c_void_p * world
        self._gathered = None
        ok = False
        if peer:
            self._flag = torch.zeros(1, device=dev, dtype=torch.int32)
            self._epoch = torch.zeros(2, device=dev, dtype=torch.int32)
            try:
                id_ptrs, flag_ptrs = self.arena.map_peer_tensors([ids, self._flag])
                ok = True
            except Exception as e:           # e.g. ranks on different nodes: all-gather the ids instead
                self.peer_error = f"{type(e).__name__}: {e}"
            agree = torch.tensor([1.0 if ok else 0.0], device=dev)
            dist.all_reduce(agree, op=dist.ReduceOp.MIN)
            ok = float(agree) == 1.0
        if ok:
            self._dp_ids, self._dp_flags = VP(*id_ptrs), VP(*flag_ptrs)
        else:
            self._flag = self._epoch = self._dp_flags = None
            self._gathered = torch.zeros((world,) + tuple(ids.shape), device=dev, dtype=torch.int64)
            base, nbytes = self._gathered.data_ptr(), n * self._gathered.element_size()
            self._dp_ids = VP(*[base + r * nbytes for r in range(world)])
        self._dp_local = ids
        self._dp = (world, rank, n)
        return ok

    @property
    def gathers_ids(self) -> bool:
        """True on the NCCL path: gather_ids() must run before each backward."""
        return getattr(self, "_gathered", None) is not None

    def gather_ids(self):
        import torch.distributed as dist
        dist.all_gather_into_tensor(self._gathered, self._dp_local)

    def _scatter(self, ids: torch.Tensor, grad_out: torch.Tensor):
        if getattr(self, "_dp", None) is not None:
            return self._scatter_dp(ids, grad_out)
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

    def _scatter_dp(self, ids: torch.Tensor, grad_out: torch.Tensor):
        a = self.arena
        world, rank, n = self._dp
        local = self._dp_local
        if ids.data_ptr() != local.data_ptr() or ids.numel() != n:
            raise _C.LoraB200Error("EmbeddingRows: under data parallelism the embedding must look up the step's "
                                   "input_ids buffer (the peers read it)")
        g = grad_out.reshape(-1, self.D).contiguous()
        table = self.emb[0].weight
        check(_C.lib.lb_embed_rows_scatter_dp(self._dp_ids, world, rank, n, ptr(g), dtype_code(g.dtype), self.D,
                                              self.V, ptr(self.slot_of), ptr(self.slot_tok), self.capacity,
                                              ptr(self.state), ptr(table.data), dtype_code(table.dtype),
                                              ptr(self.decay), ptr(a.rows_view(a.p)), ptr(a.rows_view(a.g)),
                                              self._dp_flags, ptr(self._epoch), stream_ptr()),
              "lb_embed_rows_scatter_dp")
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
