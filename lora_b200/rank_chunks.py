"""LoRA ranks above 64 on a linear site (a `lora_join` of wide files adds their ranks,
lora_diffusion/lora_manager.py:13-71): the fused kernel carries at most 64 ranks per launch
(the rank axis rides the K loop as up to 64 extra operand rows), so wider ranks run as rank chunks:

    chunk 0     the ordinary fused launch  y = x W^T + b + s (x A_0^T d_0) B_0^T
    chunk c>0   T_c = x A_c^T from the same kernel on an 8-row slice of the frozen weight (its output is
                discarded: the launch exists for its T side output), then  y += s (T_c d_c) B_c^T  in
                place (lb_lora_up_dropout with p = 0)

and the mirror image in backward (dX chunks accumulate in place; dA_c / dB_c through lb_lora_wgrad on
views of the gradient tensors). Every extra chunk re-reads x once: correct, not fast -- ranks above
64 are an inference-time artefact of joined files.
"""
import torch

from . import ops
from ._C import LoraB200Error
from .modules import _LOW, _SiteState, _compute_dtype, _fp32_master, _out_dtype

CH = 64


def _chunks(r):
    return [(j0, min(j0 + CH, r)) for j0 in range(0, r, CH)]


class _ChunkedLoraLinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, A, B, mod):
        if not x.is_cuda:
            raise LoraB200Error("LoraInjectedLinear.forward: lora_b200 runs on CUDA tensors only")
        if mod.training and mod.dropout.p > 0.0:
            raise LoraB200Error("LoRA rank > 64 with active dropout is not supported (train with r <= 64, "
                                "or call .eval() / set dropout.p = 0 on joined LoRAs)")
        st: _SiteState = mod._lb
        lin = mod.linear
        cdt, K, N, r = _compute_dtype(x), lin.in_features, lin.out_features, mod.r
        odt = _out_dtype(x, cdt)
        x2d = x.reshape(-1, K)
        if x2d.dtype != cdt or not x2d.is_contiguous():
            x2d = x2d.to(cdt).contiguous()
        w16, _ = st.frozen(lin.weight, cdt, need_t=False, tiled=False)
        b32 = st.bias32(lin.bias)
        A32, B32 = _fp32_master(A), _fp32_master(B)
        diag = mod._selector_diag()
        scale = float(mod.scale)
        need_bwd = any(ctx.needs_input_grad[:3])
        seed0 = torch.zeros(1, device=x.device, dtype=torch.int64)
        y, Ts = None, []
        for c, (j0, j1) in enumerate(_chunks(r)):
            rc = j1 - j0
            d16 = ops.cast_rows_pad16(A32[j0:j1].contiguous(), K, 1, rc, K, cdt)
            dg = None if diag is None else diag[j0:j1].contiguous()
            if c == 0:
                y, T = ops.fused_linear(x2d, w16, b32, d16, B32[:, j0:], r, 1, dg, scale, rc, odt, True)
            else:
                _, T = ops.fused_linear(x2d, w16[:8], None, d16, B32[:, j0:], r, 1, dg, 0.0, rc, odt, True)
                ops.up_dropout_(y, T, B32[:, j0:], r, 1, dg, scale, 0.0, seed0, rc)
            Ts.append(T if need_bwd else None)
        ctx.mod, ctx.cdt, ctx.scale, ctx.diag = mod, cdt, scale, diag
        ctx.x_shape, ctx.x_dtype = x.shape, x.dtype
        ctx.save_for_backward(x2d, A, B, *[t for t in Ts if t is not None])
        return y.view(*x.shape[:-1], N)

    @staticmethod
    def backward(ctx, gy):
        mod = ctx.mod
        st: _SiteState = mod._lb
        x2d, A, B, *Ts = ctx.saved_tensors
        lin = mod.linear
        K, N, r, cdt = lin.in_features, lin.out_features, mod.r, ctx.cdt
        gy2d = gy.reshape(-1, N)
        if gy2d.dtype != cdt or not gy2d.is_contiguous():
            gy2d = gy2d.to(cdt).contiguous()
        _, wt16 = st.frozen(lin.weight, cdt, need_t=True, tiled=False)
        A32, B32 = _fp32_master(A), _fp32_master(B)
        dx_dtype = ctx.x_dtype if ctx.x_dtype in _LOW else torch.float32
        need_x, need_a, need_b = ctx.needs_input_grad[:3]
        sink = st.grad_sink
        tA = tB = None
        if need_a:
            tA = sink[0] if sink is not None else torch.zeros((r, K), device=gy.device, dtype=torch.float32)
        if need_b:
            tB = sink[1] if sink is not None else torch.zeros((N, r), device=gy.device, dtype=torch.float32)
        seed0 = torch.zeros(1, device=gy.device, dtype=torch.int64)
        dX = None
        for c, (j0, j1) in enumerate(_chunks(r)):
            rc = j1 - j0
            bt16 = ops.cast_rows_pad16(B32[:, j0:], 1, r, rc, N, cdt)          # B_c^T padded [RP, N]
            dg = None if ctx.diag is None else ctx.diag[j0:j1].contiguous()
            if c == 0:
                dX, dT = ops.fused_linear(gy2d, wt16, None, bt16, A32[j0:], 1, K, dg, ctx.scale, rc, dx_dtype, True)
            else:
                _, dT = ops.fused_linear(gy2d, wt16[:8], None, bt16, A32[j0:], 1, K, dg, 0.0, rc, dx_dtype, True)
                ops.up_dropout_(dX, dT, A32[j0:], 1, K, dg, ctx.scale, 0.0, seed0, rc)
            if need_a:
                ops.wgrad(x2d, dT, dg, ctx.scale, tA[j0:], K, 1, rc)
            if need_b:
                ops.wgrad(gy2d, Ts[c], dg, ctx.scale, tB[:, j0:], 1, r, rc)
        dA = dB = None
        if sink is None:
            dA = tA.to(A.dtype).view_as(A) if need_a else None
            dB = tB.to(B.dtype).view_as(B) if need_b else None
        dx = dX.view(ctx.x_shape).to(ctx.x_dtype) if need_x else None
        return dx, dA, dB, None


def lora_linear_chunked(mod, x):
    return _ChunkedLoraLinearFn.apply(x, mod.lora_down.weight, mod.lora_up.weight, mod)
