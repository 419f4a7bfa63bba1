"""fp32-faithful mode of the LoRA linear ("split-bf16" operands).

The tensor cores take 16-bit operands. For fp32 activations OUTSIDE autocast the default policy
computes with bf16 operands (fp32 accumulate/output). `lora_b200.set_fp32_mode("split")` instead
represents every fp32 operand as hi + lo with hi = bf16(x), lo = bf16(x - hi) and lays the terms
side by side along K (activations [hi|lo|hi], weights/factors [hi|hi|lo]): the SAME fused kernel,
called with K := 3K, evaluates hi*hi + lo*hi + hi*lo in fp32 -- relative error 2^-16 per product
instead of 2^-8, at 3x the tensor-core work. X and gY stay fp32 for the factor gradients
(lb_lora_wgrad* read fp32 rows). Remaining 16-bit roundings: the scaled rank-r activations T' and
the up-factor tile inside the kernel (relative to the LoRA branch only).

This is the path behind the north star's "FP32 loss within 1e-4 of the reference for the same
seed" (tests/test_precise_gpu.py); it targets the reference's fp32 configuration
(BASELINE.json configs[0], mixed_precision = "no").
"""
import torch

from . import _C, ops
from ._C import LoraB200Error, check, ptr, stream_ptr
from .modules import _SiteState, _factor_grads, _fp32_master, _grad_targets, _key, _rows


def _split(src2d: torch.Tensor, pattern: int, rows_pad: int = 0) -> torch.Tensor:
    """fp32 [R,C] -> bf16 [max(R, rows_pad), 3C] (extra rows zero)."""
    R, C = src2d.shape
    src = src2d.detach()
    if src.dtype != torch.float32 or not src.is_contiguous():
        src = src.float().contiguous()
    rows = max(R, rows_pad)
    out = (torch.zeros if rows > R else torch.empty)((rows, 3 * C), device=src.device, dtype=torch.bfloat16)
    check(_C.lib.lb_split_bf16x3(ptr(src), C, ptr(out), R, C, pattern, stream_ptr()), "lb_split_bf16x3")
    ops._count()
    return out


def _frozen3(st: _SiteState, weight: torch.Tensor, need_t: bool):
    k = _key(weight)
    ent = st.w3
    if ent is None or ent[0] != k:
        ent = (k, _split(weight, 1), None)
    if need_t and ent[2] is None:
        ent = (k, ent[1], _split(weight.detach().t().contiguous(), 1))
    st.w3 = ent
    return ent[1], ent[2]


class _PreciseLoraLinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, A, B, mod):
        if not x.is_cuda:
            raise LoraB200Error("LoraInjectedLinear.forward: lora_b200 runs on CUDA tensors only")
        st: _SiteState = mod._lb
        lin = mod.linear
        K, N, r = lin.in_features, lin.out_features, mod.r
        x2d = _rows(x, K, torch.float32)
        need_bwd = any(ctx.needs_input_grad[:3])
        w3, _ = _frozen3(st, lin.weight, False)
        b32 = st.bias32(lin.bias)
        down3 = _split(A, 1, rows_pad=ops.rank_pad(r))
        diag = mod._selector_diag()
        scale = float(mod.scale)
        y, T = ops.fused_linear(_split(x2d, 0), w3, b32, down3, _fp32_master(B), r, 1, diag, scale, r,
                                torch.float32, need_bwd)
        ctx.mod, ctx.scale, ctx.diag, ctx.x_shape = mod, scale, diag, x.shape
        ctx.save_for_backward(x2d, T, A, B)
        return y.view(*x.shape[:-1], N)

    @staticmethod
    def backward(ctx, gy):
        mod = ctx.mod
        st: _SiteState = mod._lb
        x2d, T, A, B = ctx.saved_tensors
        lin = mod.linear
        K, N, r = lin.in_features, lin.out_features, mod.r
        gy2d = _rows(gy, N, torch.float32)
        _, wt3 = _frozen3(st, lin.weight, True)
        upT3 = _split(_fp32_master(B).t().contiguous(), 1, rows_pad=ops.rank_pad(r))   # B^T [r,N] -> [RP,3N]
        dX, dTs = ops.fused_linear(_split(gy2d, 0), wt3, None, upT3, _fp32_master(A), 1, K, ctx.diag,
                                   ctx.scale, r, torch.float32, True)
        need_x, need_a, need_b = ctx.needs_input_grad[:3]
        tA, tB, sunk = _grad_targets(st, need_a, need_b, (r, K), (N, r), gy.device)
        # launched at once, never queued: `sunk` only decides what autograd gets back
        if need_a and need_b:
            ops.wgrad_pair(x2d, dTs, tA, gy2d, T, tB, ctx.diag, ctx.scale, r)
        elif need_a:
            ops.wgrad(x2d, dTs, ctx.diag, ctx.scale, tA, K, 1, r)
        elif need_b:
            ops.wgrad(gy2d, T, ctx.diag, ctx.scale, tB, 1, r, r)
        dA, dB = _factor_grads(tA, tB, sunk, A, B)
        return (dX.view(ctx.x_shape) if need_x else None), dA, dB, None


def lora_linear_precise(mod, x):
    return _PreciseLoraLinearFn.apply(x, mod.lora_down.weight, mod.lora_up.weight, mod)
