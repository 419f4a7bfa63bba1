"""autograd glue for LoraInjectedConv2d on the fused NHWC implicit-GEMM kernel
(lb_lora_conv2d_fwd / lb_lora_wgrad_conv). Replaces lora_diffusion/lora.py:130-135 + autograd.

Supported geometry = the reference's conv LoRA sites in SD1.5 (`ResnetBlock2D.conv1/conv2`
3x3 pad 1, `conv_shortcut` 1x1): stride 1, dilation 1, groups 1, "same" padding. Anything else
raises LoraB200Error (there is no eager fallback).
"""
import torch

from . import ops
from ._C import LoraB200Error
from .modules import _LOW, _SiteState, _compute_dtype, _fp32_master, _key, _out_dtype


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


def _frozen_conv(st: _SiteState, weight, dtype, need_bwd: bool):
    k = _key(weight, tag="conv")
    ent = st.w.get(dtype)
    if ent is not None and ent[0] != k:
        ent = None
    have_f = ent is not None
    have_b = ent is not None and ent[2] is not None
    if not have_f or (need_bwd and not have_b):
        f, b = ops.cast_conv_weight(weight, dtype, not have_f, need_bwd)
        ent = (k, ent[1] if have_f else f, b if need_bwd else None)
        st.w[dtype] = ent
    return ent[1], ent[2]


def _down16(st: _SiteState, A, dtype):
    k = _key(A)
    ent = st.down.get(dtype)
    if ent is None or ent[0] != k:
        if not hasattr(st, "conv_tables"):
            st.conv_tables = {}
        ent = (k, ops.conv_down16(A, dtype, st.conv_tables))
        st.down[dtype] = ent
    return ent[1]


def _upT16(st: _SiteState, B, dtype):
    k = _key(B)
    ent = st.upT.get(dtype)
    if ent is None or ent[0] != k:
        cout, r = B.shape[0], B.shape[1]
        src = _fp32_master(B)
        ent = (k, ops.cast_rows_pad16(src, 1, r, r, cout, dtype))
        st.upT[dtype] = ent
    return ent[1]


def _nhwc16(x, dtype):
    if x.dtype != dtype:
        x = x.to(dtype)
    return x.contiguous(memory_format=torch.channels_last)


class _FusedLoraConv2dFn(torch.autograd.Function):
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
        need_bwd = any(ctx.needs_input_grad[:3])
        x16 = _nhwc16(x, cdt)
        w_f, _ = _frozen_conv(st, conv.weight, cdt, False)
        b32 = st.bias32(conv.bias)
        down16 = _down16(st, A, cdt)
        B32 = _fp32_master(B)
        diag = mod._selector_diag()
        scale = float(mod.scale)
        y, T = ops.fused_conv2d(x16, w_f, b32, down16, B32, 0, r, 1, 0, diag, scale, r,
                                conv.out_channels, kh, kw, ph, pw, False, odt, need_bwd)
        ctx.mod, ctx.cdt, ctx.scale, ctx.diag = mod, cdt, scale, diag
        ctx.geom = (kh, kw, ph, pw)
        ctx.x_dtype = x.dtype
        ctx.save_for_backward(x16, T, A, B)
        return y

    @staticmethod
    def backward(ctx, gy):
        mod = ctx.mod
        st: _SiteState = mod._lb
        x16, T, A, B = ctx.saved_tensors
        conv = mod.conv
        kh, kw, ph, pw = ctx.geom
        taps = kh * kw
        cin, cout, r = conv.in_channels, conv.out_channels, mod.r
        cdt = ctx.cdt
        gy16 = _nhwc16(gy, cdt)
        n, _, h, w = gy16.shape
        _, w_b = _frozen_conv(st, conv.weight, cdt, True)
        upT16 = _upT16(st, B, cdt)
        A32 = _fp32_master(A)
        dx_dtype = ctx.x_dtype if ctx.x_dtype in _LOW else torch.float32
        # dX = conv_T(gY, W) + conv_T((gY.B)*s*d, A); "up" = A read flipped: element (c, tap g, j)
        # at A[j, c, taps-1-g]  ->  base offset taps-1, up_rs = taps, up_cs = cin*taps, up_gs = -1
        # (rank pads 32 / 64: the entry computes dTs = gY.B first and runs the taps through it)
        dX, dTs = ops.fused_conv2d(gy16, w_b, None, upT16, A32, taps - 1, taps, cin * taps, -1,
                                   ctx.diag, ctx.scale, r, cin, kh, kw, kh - 1 - ph, kw - 1 - pw,
                                   True, dx_dtype, True)
        need_x, need_a, need_b = ctx.needs_input_grad[:3]
        sink = st.grad_sink
        dA = dB = None
        if need_a:
            tgt = sink[0] if sink is not None else torch.zeros((r, cin * taps), device=gy.device,
                                                               dtype=torch.float32)
            ops.wgrad_conv(x16, dTs, ctx.diag, ctx.scale, tgt, r, cin, h, w, kh, kw, ph, pw, deferrable=sink is not None)
            if sink is None:
                dA = tgt.view_as(A).to(A.dtype)
        if need_b:
            tgt = sink[1] if sink is not None else torch.zeros((cout, r), device=gy.device,
                                                               dtype=torch.float32)
            gy2d = gy16.permute(0, 2, 3, 1).reshape(n * h * w, cout)       # NHWC bytes as [pixels, Cout]
            ops.wgrad(gy2d, T, ctx.diag, ctx.scale, tgt, 1, r, r, deferrable=sink is not None)
            if sink is None:
                dB = tgt.view_as(B).to(B.dtype)
        dx = dX.to(ctx.x_dtype) if need_x else None
        return dx, dA, dB, None


def lora_conv2d(mod, x):
    if mod.r > ops.MAX_RANK:
        raise LoraB200Error(f"LoraInjectedConv2d: LoRA rank {mod.r} > {ops.MAX_RANK} is not supported by the "
                            "fused conv kernel (linear sites run as rank chunks, rank_chunks.py)")
    if mod.training and mod.dropout.p > 0.0:
        from .dropout_path import lora_conv2d_dropout
        return lora_conv2d_dropout(mod, x)
    return _FusedLoraConv2dFn.apply(x, mod.lora_down.weight, mod.lora_up.weight, mod)
