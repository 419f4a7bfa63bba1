"""Flat LoRA-parameter arena + fused clip/AdamW step + data-parallel gradient exchange.

GPU-first replacement for what the reference gets from torch.optim.AdamW over 288-448 tiny
tensors, clip_grad_norm_ and DDP's bucketed allreduce
(training_scripts/train_lora_dreambooth.py:651-676, 744-757, 877-888;
lora_diffusion/cli_lora_pti.py:997, 606-609):

  * every LoRA factor of every model lives in ONE contiguous fp32 buffer `p` (the module
    Parameters become views; Parameter object identity is preserved so the generators returned
    by inject_trainable_lora stay valid) with sibling buffers g, m, v;
  * backward kernels accumulate dA/dB straight into `g` (no autograd accumulation kernels);
  * one cooperative launch per step (lb_optim_step_fused) computes the global-norm clip
    coefficient, runs AdamW, zeroes the gradients and refreshes the 16-bit operand copies the
    wgmma kernels read (with fp16 loss scaling: also unscale, skip and the scale update);
  * data parallel: with enable_peer_allreduce() the gradient sum over the ranks happens inside
    that launch by peer reads over NVLink (lb_optim_step_dp, no NCCL call); otherwise ONE NCCL
    all-reduce(sum) over `g` precedes it and the launch folds in the 1/world average;
  * nothing here synchronises the host, so a whole training step can be captured in a CUDA graph
    (learning rates and the step counter live in device memory).
"""
import ctypes
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from . import _C, ops
from ._C import check, dtype_code, ptr, stream_ptr

_ALIGN = 8  # elements; keeps every factor 32-byte aligned inside the arena
_LORA_CLASS_NAMES = ("LoraInjectedLinear", "LoraInjectedConv2d")
# peer memory blocks this process has opened over CUDA IPC: handle -> base address
_IPC_OPENED: Dict[bytes, int] = {}


class LrSchedule(NamedTuple):
    """The LR schedule the loss-scaled optimizer launch applies on the device (diffusers'
    get_scheduler lambdas, LoraTrainStep.lr_multiplier): group i in `groups` runs at
    base_lr[i] * lambda(applied steps), the others at the lr last given to set_lr."""
    kind: str = "constant"                 # "constant" | "constant_with_warmup" | "linear"
    warmup_steps: int = 0
    max_train_steps: int = 0
    groups: Tuple[int, ...] = ()


_SCHED_KINDS = {"constant": _C.LB_SCHED_CONSTANT, "constant_with_warmup": _C.LB_SCHED_CONSTANT_WITH_WARMUP,
                "linear": _C.LB_SCHED_LINEAR}


def lora_sites(model: nn.Module) -> List[nn.Module]:
    return [m for m in model.modules() if type(m).__name__ in _LORA_CLASS_NAMES]


def _round_up(x: int, a: int) -> int:
    return (x + a - 1) // a * a


class LoraArena:
    """groups: [(model_or_list_of_sites, lr)] -- one optimizer param-group per entry, in the order
    the reference builds them (unet first, then text encoder: train_lora_dreambooth.py:659-669)."""

    def __init__(self, groups: Sequence[Tuple[object, float]], compute_dtype=torch.bfloat16,
                 device: Optional[torch.device] = None, rows: Optional[Tuple[int, int, float]] = None):
        """rows: (capacity, D, lr) appends one more param-group of `capacity` fp32 rows of width D
        after the LoRA groups -- the claimed token-embedding rows of lora_b200.embed_rows, clipped
        and updated by the same optimizer launch (`rows_group`, `rows_master`, `rows_grad`)."""
        self.compute_dtype = compute_dtype
        site_groups: List[List[nn.Module]] = []
        for model, _ in groups:
            sites = lora_sites(model) if isinstance(model, nn.Module) else list(model)
            site_groups.append(sites)
        if not any(site_groups):
            raise _C.LoraB200Error("LoraArena: no LoRA sites found (inject_trainable_lora first)")
        first = next(s for sg in site_groups for s in sg)
        self.device = device or first.lora_up.weight.device
        if self.device.type != "cuda":
            raise _C.LoraB200Error("LoraArena needs the LoRA modules on a CUDA device")

        # ---- layout: [group0: up0, down0, up1, down1, ... | group1: ...]
        off = 0
        self.group_off = [0]
        self.entries = []  # (site, which, param, off, numel)
        for sites in site_groups:
            for s in sites:
                for which, holder in (("up", s.lora_up), ("down", s.lora_down)):
                    w = holder.weight
                    self.entries.append((s, which, holder, off, w.numel()))
                    off = _round_up(off + w.numel(), _ALIGN)
            self.group_off.append(off)
        lrs = [float(lr) for _, lr in groups]
        self.rows_group = None
        if rows is not None:
            cap, width, rows_lr = int(rows[0]), int(rows[1]), float(rows[2])
            if cap <= 0 or width <= 0:
                raise _C.LoraB200Error(f"LoraArena: rows=(capacity={cap}, D={width}) must be positive")
            self.rows_group, self.rows_shape = len(lrs), (cap, width)
            off = _round_up(off + cap * width, _ALIGN)
            self.group_off.append(off)
            lrs.append(rows_lr)
        self.n = off
        self.n_params = sum(e[4] for e in self.entries)
        dev = self.device
        self.p = torch.zeros(self.n, device=dev, dtype=torch.float32)
        self.g = torch.zeros_like(self.p)
        self.m = torch.zeros_like(self.p)
        self.v = torch.zeros_like(self.p)
        self.lr = torch.tensor(lrs, device=dev, dtype=torch.float32)
        self.base_lr = lrs
        self.step_dev = torch.zeros(1, device=dev, dtype=torch.int32)
        self.partials = torch.zeros(1024, device=dev, dtype=torch.float32)
        self.gnorm = torch.zeros(1, device=dev, dtype=torch.float32)
        self._grid_bar = torch.zeros(2, device=dev, dtype=torch.int32)   # the optimizer launch's grid barrier
        self._group_off_c = (ctypes.c_longlong * len(self.group_off))(*self.group_off)

        # ---- adopt: Parameters become views of p; .grad views of g
        for s, which, holder, o, n in self.entries:
            w = holder.weight
            view = self.p[o:o + n].view(w.shape)
            view.copy_(w.detach().to(torch.float32))
            if w.dtype == torch.float32:
                w.data = view
            else:  # 16-bit host model: the trainable master copy is still fp32
                holder.weight = nn.Parameter(view, requires_grad=True)
                w = holder.weight
            w.requires_grad_(True)
            w.grad = self.g[o:o + n].view(w.shape)

        # ---- data-parallel replicas start identical: what accelerate/DDP's wrap does for the
        # reference (rank 0's parameters are broadcast, train_lora_dreambooth.py:744-757). Without
        # it per-rank seeding, `loras=` resumes or a checkpoint patched on one rank would diverge
        # silently, because only gradients are exchanged afterwards.
        self.sync_replicas()

        # ---- 16-bit operand copies ("shadows") + the table the refresh kernel walks
        # (each site's slots hold rank_pad(r) rows, the table's last column)
        rows, sh_off, max_c = [], 0, 1
        self._shadow_slots = []  # (site, kind, off, C, rows)
        for s in (s for sg in site_groups for s in sg):
            o_up = self._off_of(s, "up")
            o_dn = self._off_of(s, "down")
            r = s.r
            rp = ops.rank_pad(r)
            if type(s).__name__ == "LoraInjectedLinear":
                N, K = s.linear.out_features, s.linear.in_features
                # down16 [RP,K] <- A[r,K]
                rows.append((o_dn, K, 1, r, K, sh_off, K, rp))
                self._shadow_slots.append((s, "down", sh_off, K, rp)); sh_off += rp * K
                # upT16 [RP,N] <- B[N,r]^T
                rows.append((o_up, 1, r, r, N, sh_off, N, rp))
                self._shadow_slots.append((s, "upT", sh_off, N, rp)); sh_off += rp * N
                max_c = max(max_c, K, N)
            else:
                conv = s.conv
                cin, cout = conv.in_channels, conv.out_channels
                kh, kw = conv.kernel_size
                taps = kh * kw
                ktot = taps * cin
                # down16 [RP, taps*Cin], K index = tap*Cin + c  <- A[r,Cin,kh,kw]
                rows += ops.conv_tap_rows(o_dn, sh_off, r, cin, taps, rp)
                self._shadow_slots.append((s, "down", sh_off, ktot, rp)); sh_off += rp * ktot
                rows.append((o_up, 1, r, r, cout, sh_off, cout, rp))
                self._shadow_slots.append((s, "upT", sh_off, cout, rp)); sh_off += rp * cout
                max_c = max(max_c, cin, cout)
            sh_off = _round_up(sh_off, 64)
        self.shadow = torch.zeros(max(sh_off, 64), device=dev, dtype=compute_dtype)
        self.table = torch.tensor(rows, device=dev, dtype=torch.int64).contiguous()
        self.table_max_c = max_c
        self.refresh_shadows()
        self._publish_shadows()
        for s in (s for sg in site_groups for s in sg):
            s._lb.grad_sink = (self._gview(s, "down"), self._gview(s, "up"))

    # ------------------------------------------------------------------ NVLink peer all-reduce
    def enable_peer_allreduce(self) -> bool:
        """Map every rank's flat gradient buffer (and a small flag array) into this process over
        CUDA IPC so that `step()` can run lb_optim_step_dp: the gradient all-reduce happens INSIDE the
        optimizer launch by direct peer reads over NVLink/NVSwitch -- no NCCL call on the step path,
        the whole step is capturable as ONE CUDA graph at any world size. All ranks must call this
        (collectively) and must be on one node. Returns False (and leaves NCCL in place) when the
        process group is absent / single-rank."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
            return False
        world, rank = dist.get_world_size(), dist.get_rank()
        if world > 16:
            raise _C.LoraB200Error("enable_peer_allreduce: at most 16 ranks (one NVSwitch node)")
        if any(rp > 16 for *_, rp in self._shadow_slots):
            raise _C.LoraB200Error("enable_peer_allreduce: LoRA ranks above 16 are not supported by the "
                                   "peer all-reduce step (use the NCCL all-reduce path)")
        dev = self.device
        self._dp_flags = torch.zeros(2 * world, device=dev, dtype=torch.int32)
        self._dp_epoch = torch.zeros(1, device=dev, dtype=torch.int32)
        self.gsum = torch.zeros_like(self.g)
        g_ptrs, f_ptrs = self.map_peer_tensors([self.g, self._dp_flags])
        VP = ctypes.c_void_p * world
        self._dp = (VP(*g_ptrs), VP(*f_ptrs), world, rank)
        return True

    def map_peer_tensors(self, tensors: Sequence[torch.Tensor]) -> List[List[int]]:
        """Collective over the process group (every rank passes its own tensors of the same list):
        exports each device tensor over CUDA IPC, all-gathers the handles and opens the peers' ones.
        Returns, per tensor, the `world` device addresses of every rank's copy in rank order (this
        rank's own included), usable by kernels of this process. All ranks must be on one node; the
        tensors must outlive every launch that reads them. Ends in a barrier: on return every rank
        has mapped every tensor."""
        import torch.distributed as dist
        world, rank = dist.get_world_size(), dist.get_rank()
        torch.cuda.synchronize(self.device)

        def export(t):
            h = ctypes.create_string_buffer(64)
            off = ctypes.c_longlong(0)
            check(_C.lib.lb_ipc_export(ptr(t), h, ctypes.byref(off)), "lb_ipc_export")
            return bytes(h.raw), int(off.value)

        mine = [export(t) for t in tensors]
        everyone = [None] * world
        dist.all_gather_object(everyone, mine)

        def open_(handle, off):
            if handle not in _IPC_OPENED:     # a block is opened once per process
                base = ctypes.c_void_p()
                check(_C.lib.lb_ipc_open(ctypes.create_string_buffer(handle, 64), ctypes.byref(base)), "lb_ipc_open")
                _IPC_OPENED[handle] = int(base.value)
            return _IPC_OPENED[handle] + off

        out = []
        for i, t in enumerate(tensors):
            out.append([t.data_ptr() if r == rank else open_(*everyone[r][i]) for r in range(world)])
        dist.barrier()            # every rank has mapped every buffer before anybody launches
        return out

    def sync_replicas(self, src: int = 0):
        """Broadcast rank `src`'s LoRA factors and optimizer state (p, m, v, Adam's t) to every
        rank, and with loss scaling the whole scaler state (scale, growth tracker, applied-step count
        and the growth / backoff / interval constants); a no-op outside torch.distributed. Called at
        construction; call it again after loading a checkpoint (or a scaler.pt) on one rank, before
        prepare() captures the step."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
            return
        bufs = [self.p, self.m, self.v, self.step_dev]
        if self.loss_scaling:
            bufs += [self.loss_scale, self._growth_tracker, self.applied_steps]
            consts = [self._scaler_consts]
            dist.broadcast_object_list(consts, src=src,
                                       device=self.device if dist.get_backend() == "nccl" else None)
            self._set_scaler_consts(*consts[0])
        for buf in bufs:
            dist.broadcast(buf, src=src)
        if hasattr(self, "shadow"):
            self.refresh_shadows()
            self._publish_shadows()

    # ------------------------------------------------------------------ helpers
    def _off_of(self, site, which):
        for s, w, _, o, _n in self.entries:
            if s is site and w == which:
                return o
        raise KeyError

    def rows_view(self, buf: torch.Tensor) -> torch.Tensor:
        """[capacity, D] view of the rows group inside one of the flat buffers (p, g, m or v)."""
        if self.rows_group is None:
            raise _C.LoraB200Error("LoraArena was built without rows=")
        o = self.group_off[self.rows_group]
        cap, width = self.rows_shape
        return buf[o:o + cap * width].view(cap, width)

    def _gview(self, site, which):
        for s, w, holder, o, n in self.entries:
            if s is site and w == which:
                shape = holder.weight.shape
                return self.g[o:o + n].view(shape[0], -1)
        raise KeyError

    def _publish_shadows(self):
        """Pre-populate every site's operand cache with views into the shadow buffer. The cache
        key is the Parameter's (id, version, data_ptr): torch-side in-place edits bump the version
        and fall back to a private re-cast; our own kernels edit p in place without touching the
        version counter and refresh the shadows themselves."""
        from .modules import _key
        dt = self.compute_dtype
        for s, kind, o, C, rp in self._shadow_slots:
            view = self.shadow[o:o + rp * C].view(rp, C)
            if kind == "down":
                s._lb.down[dt] = (_key(s.lora_down.weight), view)
            else:
                s._lb.upT[dt] = (_key(s.lora_up.weight), view)

    def refresh_shadows(self):
        check(_C.lib.lb_refresh_shadows(ptr(self.p), ptr(self.table), self.table.shape[0],
                                        self.table_max_c, ptr(self.shadow),
                                        dtype_code(self.compute_dtype), stream_ptr()),
              "lb_refresh_shadows")
        ops._count(1)

    # ------------------------------------------------------------------ fp16 dynamic loss scaling
    loss_scaling = False

    def enable_loss_scaling(self, init_scale: float = 65536.0, growth_factor: float = 2.0,
                            backoff_factor: float = 0.5, growth_interval: int = 2000):
        """torch.amp.GradScaler on the device (accelerate's `--mixed_precision fp16`). Allocates the
        scaler state; from then on `step()` takes the scaled launch: it unscales the gradients, skips
        the update when any of them is inf / NaN, and updates the scale by GradScaler's rule, without
        a host round trip. The caller's backward must be seeded with `loss_scale` (the device
        tensor below) times the loss gradient, e.g. `(loss * arena.loss_scale).backward()` or
        step_ops.fused_masked_mse(..., grad_scale=arena.loss_scale)."""
        if not init_scale > 0.0:
            raise ValueError("enable_loss_scaling: need init_scale > 0")
        self._set_scaler_consts(growth_factor, backoff_factor, growth_interval)
        dev = self.device
        self.loss_scale = torch.full((1,), float(init_scale), device=dev, dtype=torch.float32)
        self._growth_tracker = torch.zeros(1, device=dev, dtype=torch.int32)
        self._found_inf = torch.zeros(1, device=dev, dtype=torch.int32)
        self.applied_steps = torch.zeros(1, device=dev, dtype=torch.int32)   # the LR schedule's step count
        self._base_lr64 = torch.tensor(self.base_lr, device=dev, dtype=torch.float64)
        self.loss_scaling = True

    def _set_scaler_consts(self, growth_factor, backoff_factor, growth_interval):
        if not (growth_factor > 1.0 and 0.0 < backoff_factor < 1.0 and int(growth_interval) >= 1):
            raise ValueError("loss scaling: need growth_factor > 1, 0 < backoff_factor < 1, growth_interval >= 1")
        self._scaler_consts = (float(growth_factor), float(backoff_factor), int(growth_interval))
        self._scaler_args = {}        # launch arguments are rebuilt with the new constants

    def _require_loss_scaling(self, what: str):
        if not self.loss_scaling:
            raise _C.LoraB200Error(f"{what} needs enable_loss_scaling() first")

    def _scaler(self, schedule: Optional[LrSchedule]):
        schedule = schedule or LrSchedule()
        a = self._scaler_args.get(schedule)
        if a is None:
            if schedule.kind not in _SCHED_KINDS:
                raise ValueError(f"lr schedule {schedule.kind!r}: one of {tuple(_SCHED_KINDS)}")
            mask = 0
            for gi in schedule.groups:
                if not 0 <= gi < len(self.base_lr):
                    raise ValueError(f"lr schedule: no parameter group {gi}")
                mask |= 1 << gi
            gf, bf, gi_ = self._scaler_consts
            a = _C.GradScalerArgs(gf, bf, gi_, _SCHED_KINDS[schedule.kind], int(schedule.warmup_steps),
                                  int(schedule.max_train_steps), mask, self._base_lr64.data_ptr(),
                                  self.loss_scale.data_ptr(), self._growth_tracker.data_ptr(),
                                  self._found_inf.data_ptr(), self.applied_steps.data_ptr())
            self._scaler_args[schedule] = a
        return ctypes.byref(a)

    def step_was_skipped(self) -> bool:
        """Whether the last step() found an inf / NaN gradient and skipped the update (host read:
        synchronises the stream)."""
        self._require_loss_scaling("step_was_skipped()")
        return bool(self._found_inf.item())

    def scaler_state_dict(self) -> dict:
        """torch.amp.GradScaler.state_dict()'s keys and values (accelerate's scaler.pt). Host read."""
        self._require_loss_scaling("scaler_state_dict()")
        gf, bf, gi = self._scaler_consts
        return {"scale": float(self.loss_scale.item()), "growth_factor": gf, "backoff_factor": bf,
                "growth_interval": gi, "_growth_tracker": int(self._growth_tracker.item())}

    def load_scaler_state_dict(self, state: dict):
        """Inverse of scaler_state_dict (also takes a GradScaler.state_dict()). Outside any graph: a
        captured step keeps the constants it was captured with, so load before prepare(). Under
        torch.distributed, load on every rank, or on one and call sync_replicas()."""
        self._require_loss_scaling("load_scaler_state_dict()")
        if not state:
            raise ValueError("load_scaler_state_dict: empty state (a disabled GradScaler's)")
        self._set_scaler_consts(state["growth_factor"], state["backoff_factor"], state["growth_interval"])
        self.loss_scale.fill_(float(state["scale"]))
        self._growth_tracker.fill_(int(state["_growth_tracker"]))

    # ------------------------------------------------------------------ step
    def set_lr(self, lrs: Sequence[float]):
        """Scheduler hook: host->device copy of per-group learning rates (outside any graph). With
        loss scaling these are also the base lrs of the groups the device schedule scales."""
        self.lr.copy_(torch.tensor([float(x) for x in lrs], dtype=torch.float32), non_blocking=True)
        if self.loss_scaling:
            self._base_lr64.copy_(torch.tensor([float(x) for x in lrs], dtype=torch.float64), non_blocking=True)

    def allreduce_grads(self):
        """The one data-path collective: sum of the flat gradient buffer over NVLink/NVSwitch. With
        enable_peer_allreduce() it is folded into step() (lb_optim_step_dp) and this is a no-op."""
        if getattr(self, "_dp", None) is not None:
            return self._dp[2]
        from .dist import allreduce_sum_
        return allreduce_sum_(self.g)

    def step(self, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-2, max_norm=1.0,
             world_size: int = 1, schedule: Optional[LrSchedule] = None):
        """clip_grad_norm_(max_norm) + AdamW + zero_grad on the (already summed) gradients, then the
        16-bit operand shadows -- one cooperative launch (lb_optim_step_fused; lb_optim_step_dp, which
        also sums the ranks' gradients, after enable_peer_allreduce()). After enable_loss_scaling():
        unscale, skip on inf / NaN, scale update and `schedule` in the same launch."""
        scaler = None
        if self.loss_scaling:
            scaler = self._scaler(schedule)
        elif schedule is not None:
            raise _C.LoraB200Error("step(schedule=...) needs enable_loss_scaling(); otherwise use set_lr")
        dp = getattr(self, "_dp", None)
        if dp is not None:       # all-reduce over NVLink peer memory inside the optimizer launch
            assert world_size == dp[2], "world size changed after enable_peer_allreduce()"
            check(_C.lib.lb_optim_step_dp(ptr(self.p), ptr(self.g), ptr(self.gsum), ptr(self.m), ptr(self.v),
                                          self.n, self._group_off_c, len(self.group_off) - 1, ptr(self.lr),
                                          beta1, beta2, eps, weight_decay, float(max_norm if max_norm else 0.0),
                                          ptr(self.step_dev), ptr(self.partials), ptr(self.gnorm),
                                          ptr(self.table), self.table.shape[0], self.table_max_c,
                                          ptr(self.shadow), dtype_code(self.compute_dtype), ptr(self._grid_bar),
                                          dp[0], dp[1], dp[2], dp[3], ptr(self._dp_epoch), scaler, stream_ptr()),
                  "lb_optim_step_dp")
        else:
            check(_C.lib.lb_optim_step_fused(ptr(self.p), ptr(self.g), ptr(self.m), ptr(self.v), self.n,
                                             self._group_off_c, len(self.group_off) - 1, ptr(self.lr),
                                             beta1, beta2, eps, weight_decay,
                                             float(max_norm if max_norm else 0.0), 1.0 / world_size,
                                             ptr(self.step_dev), ptr(self.partials), ptr(self.gnorm),
                                             ptr(self.table), self.table.shape[0], self.table_max_c,
                                             ptr(self.shadow), dtype_code(self.compute_dtype),
                                             ptr(self._grid_bar), scaler, stream_ptr()), "lb_optim_step_fused")
        ops._count(1)
        # re-validate the per-site operand caches: if torch-side code edited a factor in place since
        # the last step (version bump -> the site fell back to a private re-cast), point it back at
        # the arena's shadow buffer, which the launch above has just refreshed
        self._publish_shadows()

    def zero_grad(self):
        self.g.zero_()

    def parameters(self):
        return [holder.weight for _, _, holder, _, _ in self.entries]
