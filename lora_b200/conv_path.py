"""autograd glue for LoraInjectedConv2d on the fused NHWC implicit-GEMM kernel
(lb_lora_conv2d_fwd / lb_lora_wgrad_conv). Replaces lora_diffusion/lora.py:130-135 + autograd.

Supported geometry = the reference's conv LoRA sites in SD1.5 (`ResnetBlock2D.conv1/conv2`
3x3 pad 1, `conv_shortcut` 1x1): stride 1, dilation 1, groups 1, "same" padding. Anything else
raises LoraB200Error (there is no eager fallback).
"""
import torch

from . import dropout_path, ops
from ._C import LoraB200Error
from .modules import (_SiteState, _active_dropout, _compute_dtype, _dx_dtype, _factor_grads, _fp32_master,
                      _grad_targets, _out_dtype)


def _geometry(conv):
    kh, kw = conv.kernel_size
    ph, pw = conv.padding if isinstance(conv.padding, tuple) else (conv.padding, conv.padding)
    ok = (tuple(conv.stride) == (1, 1) and tuple(conv.dilation) == (1, 1) and conv.groups == 1
          and (kh, kw) in ((1, 1), (3, 3)) and 2 * ph == kh - 1 and 2 * pw == kw - 1
          and conv.padding_mode == "zeros")
    if not ok:
        raise LoraB200Error(
            f"LoraInjectedConv2d: unsupported geometry kernel={conv.kernel_size} stride={conv.stride} "
            f"padding={conv.padding} dilation={conv.dilation} groups={conv.groups}; the sm_90a "
            "kernel covers stride-1 'same' 1x1/3x3 convs (the SD1.5 ResnetBlock2D sites)")
    return kh, kw, ph, pw


def _nhwc16(x, dtype):
    if x.dtype != dtype:
        x = x.to(dtype)
    return x.contiguous(memory_format=torch.channels_last)


class _FusedLoraConv2dFn(torch.autograd.Function):
    """autograd node for one LoRA conv site; with an active nn.Dropout the branch is masked in the
    forward's drain and the backward recomputes the mask from the saved seed (dropout_path.py)."""

    @staticmethod
    def forward(ctx, x, A, B, mod):
        if not x.is_cuda:
            raise LoraB200Error("LoraInjectedConv2d.forward: lora_b200 runs on CUDA tensors only")
        if x.dim() != 4:
            raise LoraB200Error("LoraInjectedConv2d expects a 4-D NCHW input")
        conv = mod.conv
        kh, kw, ph, pw = _geometry(conv)
        st: _SiteState = mod._lb
        cdt = _compute_dtype(x)
        odt = _out_dtype(x, cdt)
        r = mod.r
        x16 = _nhwc16(x, cdt)
        w_f, _ = st.frozen_conv(conv.weight, cdt, False)
        b32 = st.bias32(conv.bias)
        down16 = st.conv_down16(A, cdt)
        diag = mod._selector_diag()
        scale = float(mod.scale)
        p = _active_dropout(mod)
        seed = dropout_path._fresh_seed(mod, x.device) if p > 0.0 else None
        want_t = p > 0.0 or any(ctx.needs_input_grad[:3])
        y, T = ops.fused_conv2d(x16, w_f, b32, down16, _fp32_master(B), 0, r, 1, 0, diag, scale, r,
                                conv.out_channels, kh, kw, ph, pw, False, odt, want_t, drop_p=p, seed=seed)
        ctx.mod, ctx.cdt, ctx.scale, ctx.p, ctx.diag = mod, cdt, scale, p, diag
        ctx.geom, ctx.x_dtype = (kh, kw, ph, pw), x.dtype
        ctx.save_for_backward(x16, T, A, B, *([] if seed is None else [seed]))
        return y

    @staticmethod
    def backward(ctx, gy):
        mod = ctx.mod
        st: _SiteState = mod._lb
        x16, T, A, B, *seed = ctx.saved_tensors
        conv = mod.conv
        kh, kw, ph, pw = ctx.geom
        taps = kh * kw
        cin, cout, r, p = conv.in_channels, conv.out_channels, mod.r, ctx.p
        cdt = ctx.cdt
        gy16 = _nhwc16(gy, cdt)
        n, _, h, w = gy16.shape
        gy2d = gy16.permute(0, 2, 3, 1).reshape(n * h * w, cout)       # NHWC bytes as [pixels, Cout]
        _, w_b = st.frozen_conv(conv.weight, cdt, True)
        upT16 = st.upT16(B, cdt)
        A32 = _fp32_master(A)
        # dX = conv_T(gY, W) + conv_T((gY.B)*s*d, A); "up" = A read flipped: element (c, tap g, j)
        # at A[j, c, taps-1-g]  ->  base offset taps-1, up_rs = taps, up_cs = cin*taps, up_gs = -1
        # (rank pads 32 / 64: the entry computes dTs = gY.B first and runs the taps through it);
        # with dropout one masked pass gives dTs = (mask o gY / (1-p)) . B first and dX takes it (T_in)
        t_in = ops.dropout_dt(gy2d, _fp32_master(B), r, 1, p, seed[0], r) if p > 0.0 else None
        dX, dTs = ops.fused_conv2d(gy16, w_b, None, upT16, A32, taps - 1, taps, cin * taps, -1,
                                   ctx.diag, ctx.scale, r, cin, kh, kw, kh - 1 - ph, kw - 1 - pw,
                                   True, _dx_dtype(ctx.x_dtype), t_in is None, t_in=t_in)
        dTs = dTs if t_in is None else t_in
        need_x, need_a, need_b = ctx.needs_input_grad[:3]
        tA, tB, deferrable = _grad_targets(st, need_a, need_b, (r, cin * taps), (cout, r), gy.device)
        if need_a:
            ops.wgrad_conv(x16, dTs, ctx.diag, ctx.scale, tA, r, cin, h, w, kh, kw, ph, pw, deferrable=deferrable)
        if need_b and p > 0.0:      # dB reduces the masked gY
            ops.wgrad_masked(gy2d, T, ctx.diag, ctx.scale, tB, 1, r, r, p, seed[0], deferrable=deferrable)
        elif need_b:
            ops.wgrad(gy2d, T, ctx.diag, ctx.scale, tB, 1, r, r, deferrable=deferrable)
        dA, dB = _factor_grads(tA, tB, deferrable, A, B)
        dx = dX.to(ctx.x_dtype) if need_x else None
        return dx, dA, dB, None


def lora_conv2d(mod, x):
    if mod.r > ops.MAX_RANK:
        raise LoraB200Error(f"LoraInjectedConv2d: LoRA rank {mod.r} > {ops.MAX_RANK} is not supported by the "
                            "fused conv kernel (linear sites run as rank chunks, rank_chunks.py)")
    return _FusedLoraConv2dFn.apply(x, mod.lora_down.weight, mod.lora_up.weight, mod)
