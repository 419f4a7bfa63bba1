"""LoRA sites with an ACTIVE nn.Dropout on the branch (module.training and p > 0): the default
state of every operator built by inject_trainable_lora_extended and by the monkeypatch_* loaders
(class default dropout_p = 0.1, fresh modules are in training mode; lora.py:34,84,334-356,689-694).

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

from . import ops
from ._C import LoraB200Error
from .modules import _LOW, _SiteState, _compute_dtype, _fp32_master, _out_dtype


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


class _LoraLinearDropoutFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, A, B, mod):
        if not x.is_cuda:
            raise LoraB200Error("LoraInjectedLinear.forward: lora_b200 runs on CUDA tensors only")
        st: _SiteState = mod._lb
        lin = mod.linear
        cdt = _compute_dtype(x)
        odt = _out_dtype(x, cdt)
        K, N, r = lin.in_features, lin.out_features, mod.r
        x2d = x.reshape(-1, K)
        if x2d.dtype != cdt or not x2d.is_contiguous():
            x2d = x2d.to(cdt).contiguous()
        w16, _ = st.frozen(lin.weight, cdt, need_t=False)
        b32 = st.bias32(lin.bias)
        down16 = st.down16(A, cdt)
        B32 = _fp32_master(B)
        diag = mod._selector_diag()
        scale, p = float(mod.scale), float(mod.dropout.p)
        seed = _fresh_seed(mod, x.device)
        y, T = ops.fused_linear(x2d, w16, b32, down16, B32, r, 1, diag, scale, r, odt, True,
                                drop_p=p, seed=seed)
        ctx.mod, ctx.cdt, ctx.scale, ctx.p, ctx.diag = mod, cdt, scale, p, diag
        ctx.x_shape, ctx.x_dtype = x.shape, x.dtype
        ctx.save_for_backward(x2d, T, A, B, seed)
        return y.view(*x.shape[:-1], N)

    @staticmethod
    def backward(ctx, gy):
        mod = ctx.mod
        st: _SiteState = mod._lb
        x2d, T, A, B, seed = ctx.saved_tensors
        lin = mod.linear
        K, N, r = lin.in_features, lin.out_features, mod.r
        cdt = ctx.cdt
        gy2d = gy.reshape(-1, N)
        if gy2d.dtype != cdt or not gy2d.is_contiguous():
            gy2d = gy2d.to(cdt).contiguous()
        _, wt16 = st.frozen(lin.weight, cdt, need_t=True)
        upT16 = st.upT16(B, cdt)
        A32, B32 = _fp32_master(A), _fp32_master(B)
        dx_dtype = ctx.x_dtype if ctx.x_dtype in _LOW else torch.float32
        # a masked pass over gY, then the dX kernel takes the rank-r activations from it (T_in)
        dTs = ops.dropout_dt(gy2d, B32, r, 1, ctx.p, seed, r)          # (mask o gY / (1-p)) . B
        dX, _ = ops.fused_linear(gy2d, wt16, None, upT16, A32, 1, K, ctx.diag, ctx.scale, r,
                                 dx_dtype, False, t_in=dTs)
        need_x, need_a, need_b = ctx.needs_input_grad[:3]
        sink = st.grad_sink
        dA = dB = None
        tA = tB = None
        if need_a:
            tA = sink[0] if sink is not None else torch.zeros((r, K), device=gy.device, dtype=torch.float32)
        if need_b:
            tB = sink[1] if sink is not None else torch.zeros((N, r), device=gy.device, dtype=torch.float32)
        if need_a:
            ops.wgrad(x2d, dTs, ctx.diag, ctx.scale, tA, K, 1, r, deferrable=sink is not None)
        if need_b:
            ops.wgrad_masked(gy2d, T, ctx.diag, ctx.scale, tB, 1, r, r, ctx.p, seed, deferrable=sink is not None)
        if sink is None:
            dA = tA.to(A.dtype).view_as(A) if need_a else None
            dB = tB.to(B.dtype).view_as(B) if need_b else None
        dx = dX.view(ctx.x_shape).to(ctx.x_dtype) if need_x else None
        return dx, dA, dB, None


def lora_linear_dropout(mod, x):
    return _LoraLinearDropoutFn.apply(x, mod.lora_down.weight, mod.lora_up.weight, mod)


class _LoraConv2dDropoutFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, A, B, mod):
        from .conv_path import _down16, _frozen_conv, _geometry, _nhwc16
        if not x.is_cuda:
            raise LoraB200Error("LoraInjectedConv2d.forward: lora_b200 runs on CUDA tensors only")
        conv = mod.conv
        kh, kw, ph, pw = _geometry(conv)
        st: _SiteState = mod._lb
        cdt = _compute_dtype(x)
        odt = _out_dtype(x, cdt)
        r = mod.r
        x16 = _nhwc16(x, cdt)
        w_f, _ = _frozen_conv(st, conv.weight, cdt, False)
        b32 = st.bias32(conv.bias)
        down16 = _down16(st, A, cdt)
        B32 = _fp32_master(B)
        diag = mod._selector_diag()
        scale, p = float(mod.scale), float(mod.dropout.p)
        seed = _fresh_seed(mod, x.device)
        cout = conv.out_channels
        y, T = ops.fused_conv2d(x16, w_f, b32, down16, B32, 0, r, 1, 0, diag, scale, r, cout, kh, kw,
                                ph, pw, False, odt, True, drop_p=p, seed=seed)
        ctx.mod, ctx.cdt, ctx.scale, ctx.p, ctx.diag = mod, cdt, scale, p, diag
        ctx.geom, ctx.x_dtype = (kh, kw, ph, pw), x.dtype
        ctx.save_for_backward(x16, T, A, B, seed)
        return y

    @staticmethod
    def backward(ctx, gy):
        from .conv_path import _frozen_conv, _nhwc16, _upT16
        mod = ctx.mod
        st: _SiteState = mod._lb
        x16, T, A, B, seed = ctx.saved_tensors
        conv = mod.conv
        kh, kw, ph, pw = ctx.geom
        taps = kh * kw
        cin, cout, r = conv.in_channels, conv.out_channels, mod.r
        cdt = ctx.cdt
        gy16 = _nhwc16(gy, cdt)
        n, _, h, w = gy16.shape
        gy2d = gy16.permute(0, 2, 3, 1).reshape(n * h * w, cout)
        _, w_b = _frozen_conv(st, conv.weight, cdt, True)
        upT16 = _upT16(st, B, cdt)
        A32, B32 = _fp32_master(A), _fp32_master(B)
        dx_dtype = ctx.x_dtype if ctx.x_dtype in _LOW else torch.float32
        dTs = ops.dropout_dt(gy2d, B32, r, 1, ctx.p, seed, r)
        dX, _ = ops.fused_conv2d(gy16, w_b, None, upT16, A32, taps - 1, taps, cin * taps, -1,
                                 ctx.diag, ctx.scale, r, cin, kh, kw, kh - 1 - ph, kw - 1 - pw,
                                 True, dx_dtype, False, t_in=dTs)
        need_x, need_a, need_b = ctx.needs_input_grad[:3]
        sink = st.grad_sink
        dA = dB = None
        if need_a:
            tgt = sink[0] if sink is not None else torch.zeros((r, cin * taps), device=gy.device, dtype=torch.float32)
            ops.wgrad_conv(x16, dTs, ctx.diag, ctx.scale, tgt, r, cin, h, w, kh, kw, ph, pw, deferrable=sink is not None)
            if sink is None:
                dA = tgt.view_as(A).to(A.dtype)
        if need_b:
            tgt = sink[1] if sink is not None else torch.zeros((cout, r), device=gy.device, dtype=torch.float32)
            ops.wgrad_masked(gy2d, T, ctx.diag, ctx.scale, tgt, 1, r, r, ctx.p, seed, deferrable=sink is not None)
            if sink is None:
                dB = tgt.view_as(B).to(B.dtype)
        dx = dX.to(ctx.x_dtype) if need_x else None
        return dx, dA, dB, None


def lora_conv2d_dropout(mod, x):
    return _LoraConv2dDropoutFn.apply(x, mod.lora_down.weight, mod.lora_up.weight, mod)
