"""ORACLE (test infrastructure only -- never imported by the product path).

CPU restatement of the arithmetic of the reference's LoRA hot path, written as explicit matrix
formulas in float64 (torch CPU tensors used as plain ndarrays; no autograd, no nn.Module). The
forward / backward restatements take `device=`: the same float64 formulas on another device, for the
kernel tests at full SD1.5 conv sizes, where CPU float64 convolutions would dominate the run time.
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this package.

Pinned against the real reference: tests/golden/*.pt were produced by running
/root/reference/lora_diffusion/lora.py itself (scripts/make_golden.py, committed) and
tests/test_oracle_golden.py checks every function below against them.

Each function cites the reference lines it restates (paths relative to /root/reference).
"""
from typing import Optional, Tuple

import torch

F64 = torch.float64


def _f(x, device="cpu"):
    return None if x is None else x.detach().to(device, F64)


def selector_matrix(diag: Optional[torch.Tensor], r: int, device="cpu") -> torch.Tensor:
    """lora_diffusion/lora.py:63-70 -- selector is Identity or a Linear whose weight is diag(d)."""
    if diag is None:
        return torch.eye(r, dtype=F64, device=device)
    return torch.diag(_f(diag, device))


def lora_linear_forward(x, W, bias, A, B, scale: float, diag=None, keep_mask=None,
                        dropout_p: float = 0.0, device="cpu"):
    """lora_diffusion/lora.py:53-58.

        y = x W^T (+ b) + dropout( ((x A^T) S^T) B^T ) * scale

    x: [M,K]; W: [N,K]; A = lora_down.weight [r,K]; B = lora_up.weight [N,r]; S = selector weight.
    dropout (lora.py:45,56): keep_mask in {0,1}^[M,N] applied to the LoRA branch and rescaled by
    1/(1-p); None means eval mode or p == 0.
    device: where the float64 arithmetic runs (the result lives there too).
    """
    x, W, A, B, bias = (_f(t, device) for t in (x, W, A, B, bias))
    r = A.shape[0]
    S = selector_matrix(diag, r, device)
    base = x @ W.T
    if bias is not None:
        base = base + bias
    t = x @ A.T                      # lora_down
    t = t @ S.T                      # selector (nn.Linear: y = t S^T)
    u = t @ B.T                      # lora_up
    if keep_mask is not None:
        u = u * _f(keep_mask, device) / (1.0 - dropout_p)
    return base + u * scale


def lora_linear_backward(gy, x, W, A, B, scale: float, diag=None, keep_mask=None,
                         dropout_p: float = 0.0, device="cpu") -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Autograd of lora.py:53-58 with W, b frozen (train_lora_dreambooth.py:595): returns
    (dX, dA, dB). No dW.

        gU = scale * gY (* mask/(1-p))      dB = gU^T (x A^T S^T)
        dT = gU B S                         dA = dT^T x
        dX = gY W + dT A
    """
    gy, x, W, A, B = (_f(t, device) for t in (gy, x, W, A, B))
    r = A.shape[0]
    S = selector_matrix(diag, r, device)
    gu = gy * scale
    if keep_mask is not None:
        gu = gu * _f(keep_mask, device) / (1.0 - dropout_p)
    t_sel = (x @ A.T) @ S.T
    dB = gu.T @ t_sel
    dT = (gu @ B) @ S
    dA = dT.T @ x
    dX = gy @ W + dT @ A
    return dX, dA, dB


def _conv2d_naive(x, w, stride, padding, dilation):
    """Direct convolution, float64, NCHW, groups = 1 (what F.conv2d computes; lora.py:132-133)."""
    import torch.nn.functional as F
    return F.conv2d(x, w, None, stride, padding, dilation, 1)


def lora_conv2d_forward(x, W, bias, A, B, scale: float, stride=1, padding=0, dilation=1,
                        diag=None, keep_mask=None, dropout_p: float = 0.0, device="cpu"):
    """lora_diffusion/lora.py:130-135.

    x: [N,Cin,H,W]; W: [Cout,Cin,kh,kw]; A = lora_down.weight [r,Cin,kh,kw] (same stride/padding/
    dilation as the base conv, lora.py:105-114); B = lora_up.weight [Cout,r,1,1] (1x1, lora.py:116-123).
    The selector, when set, is a 1x1 conv with weight diag(d) (lora.py:140-156).
    device: where the float64 arithmetic runs (the result lives there too).
    """
    x, W, A, B, bias = (_f(t, device) for t in (x, W, A, B, bias))
    r = A.shape[0]
    base = _conv2d_naive(x, W, stride, padding, dilation)
    if bias is not None:
        base = base + bias.view(1, -1, 1, 1)
    t = _conv2d_naive(x, A, stride, padding, dilation)           # [N,r,Ho,Wo]
    S = selector_matrix(diag, r, device)
    t = torch.einsum("nchw,dc->ndhw", t, S)
    u = torch.einsum("nrhw,or->nohw", t, B.reshape(B.shape[0], r))
    if keep_mask is not None:
        u = u * _f(keep_mask, device) / (1.0 - dropout_p)
    return base + u * scale


def clip_adamw_step(p, g, m, v, step: int, lr, beta1=0.9, beta2=0.999, eps=1e-8,
                    weight_decay=1e-2, max_norm=1.0, inv_world=1.0):
    """clip_grad_norm_ + torch.optim.AdamW.step as used at
    training_scripts/train_lora_dreambooth.py:878-885 (defaults :364-387) and
    lora_diffusion/cli_lora_pti.py:606-609, restated per element in float64.

    p, g, m, v: lists of tensors (one per parameter); lr: one float per tensor.
    step: the 1-based step index of THIS update. Returns (new_p, new_m, new_v, total_norm).

        total = || concat(g) * inv_world ||_2 ; coef = min(1, max_norm/(total + 1e-6))
        g' = g * inv_world * coef
        p  = p * (1 - lr*wd)
        m  = b1 m + (1-b1) g' ;  v = b2 v + (1-b2) g'^2
        p  = p - (lr / (1-b1^t)) * m / ( sqrt(v)/sqrt(1-b2^t) + eps )
    """
    g64 = [_f(x) * inv_world for x in g]
    total = torch.sqrt(sum((x * x).sum() for x in g64))
    coef = 1.0
    if max_norm is not None and max_norm > 0:
        coef = min(1.0, float(max_norm / (total + 1e-6)))
    bc1 = 1.0 - beta1 ** step
    bc2 = 1.0 - beta2 ** step
    out_p, out_m, out_v = [], [], []
    for pi, gi, mi, vi, lri in zip(p, g64, m, v, lr):
        pi, mi, vi = _f(pi), _f(mi), _f(vi)
        gi = gi * coef
        pi = pi * (1.0 - lri * weight_decay)
        mi = beta1 * mi + (1.0 - beta1) * gi
        vi = beta2 * vi + (1.0 - beta2) * gi * gi
        denom = vi.sqrt() / (bc2 ** 0.5) + eps
        pi = pi - (lri / bc1) * (mi / denom)
        out_p.append(pi)
        out_m.append(mi)
        out_v.append(vi)
    return out_p, out_m, out_v, float(total)


def collapse_delta(A, B, alpha: float = 1.0):
    """lora_diffusion/lora.py:646-669: W += alpha * (up @ down) (conv: flattened)."""
    A, B = _f(A), _f(B)
    return alpha * (B.flatten(1) @ A.flatten(1))


def lora_conv2d_backward(gy, x, W, A, B, scale: float, stride=1, padding=0, dilation=1, diag=None,
                         keep_mask=None, dropout_p: float = 0.0, device="cpu"):
    """Autograd of lora.py:130-135 with the base conv frozen: returns (dX, dA, dB), written with
    the explicit transposed-convolution / weight-gradient operators (float64, no autograd graph).

        gU = scale * gY ;  dB[o,j] = sum_{n,h,w} gU[n,o,h,w] * (S t)[n,j,h,w]   (t = conv(x, A))
        dT = S^T (B^T gU)                      (1x1 up-projection transposed, then the selector)
        dA = conv_weight_grad(x, dT) ;  dX = conv_input_grad(gY, W) + conv_input_grad(dT, A)
    """
    from torch.nn import grad as G
    gy, x, W, A, B = (_f(t, device) for t in (gy, x, W, A, B))
    r = A.shape[0]
    S = selector_matrix(diag, r, device)
    t = _conv2d_naive(x, A, stride, padding, dilation)
    t_sel = torch.einsum("nchw,dc->ndhw", t, S)
    gu = gy * scale
    if keep_mask is not None:                 # nn.Dropout on the branch (lora.py:115,133): same mask
        gu = gu * _f(keep_mask, device) / (1.0 - dropout_p)
    B2 = B.reshape(B.shape[0], r)
    dB = torch.einsum("nohw,njhw->oj", gu, t_sel).reshape(B.shape)
    dT = torch.einsum("nohw,oj->njhw", gu, B2)
    dT = torch.einsum("njhw,jc->nchw", dT, S)
    dA = G.conv2d_weight(x, A.shape, dT, stride, padding, dilation, 1)
    dX = G.conv2d_input(x.shape, W, gy, stride, padding, dilation, 1) + \
        G.conv2d_input(x.shape, A, dT, stride, padding, dilation, 1)
    return dX, dA, dB
