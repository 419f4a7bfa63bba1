"""GPU parity of the fused LoRA Conv2d path (NHWC implicit GEMM on wgmma) against the oracle
(oracle/lora_ops.py: lora_conv2d_forward / lora_conv2d_backward, float64), through the module API.

Tolerances: 16-bit operands, fp32 accumulate. Outputs are compared with the oracle evaluated on the
same 16-bit-rounded x / W; the LoRA branch additionally carries one 16-bit rounding of the rank-r
activations (like the reference under autocast) => relative Frobenius error < 2^-7 of bf16 outputs,
gradients of the factors < 1e-2 (they are linear in 16-bit-rounded factor copies)."""
import pytest
import torch
import torch.nn as nn

from oracle import lora_ops as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


CASES = [
    # n, cin, cout, k, H, W, r
    (1, 320, 320, 3, 64, 64, 4),      # down0 resnet conv
    (1, 640, 1280, 3, 16, 16, 8),     # down2 conv1
    (1, 960, 640, 1, 32, 32, 8),      # up2 conv_shortcut (1x1)
    (1, 1280, 1280, 3, 8, 8, 16),     # mid block (8x8: half-empty 128-row tile)
    (2, 24, 40, 3, 12, 12, 3),        # ragged: C < 64, W not a multiple of the tile, 2 images
    (3, 64, 64, 1, 5, 7, 4),
]


@pytest.mark.parametrize("n,cin,cout,k,H,W,r", CASES)
def test_conv_module_fwd_bwd_vs_oracle(n, cin, cout, k, H, W, r):
    import lora_b200 as L
    torch.manual_seed(n + cin + cout + H)
    pad = k // 2
    m = L.LoraInjectedConv2d(cin, cout, k, 1, pad, r=r, dropout_p=0.0, scale=0.8).to(DEV)
    m.conv.weight.data.mul_(0.5)
    m.conv.requires_grad_(False)
    m.lora_up.weight.data.normal_(0, 0.05)
    dt = torch.bfloat16
    x = torch.randn(n, cin, H, W, device=DEV).to(dt).requires_grad_(True)
    y = m(x)
    assert y.shape == (n, cout, H, W) and y.dtype == dt
    gy = torch.randn(n, cout, H, W, device=DEV).to(dt)
    y.backward(gy)
    torch.cuda.synchronize()
    W16 = m.conv.weight.detach().to(dt)
    A, B = m.lora_down.weight.detach(), m.lora_up.weight.detach()
    ref = O.lora_conv2d_forward(x, W16, m.conv.bias, A, B, 0.8, padding=pad)
    assert rel(y, ref) < 2 ** -7
    dX, dA, dB = O.lora_conv2d_backward(gy, x, W16, A, B, 0.8, padding=pad)
    assert rel(x.grad, dX) < 2 ** -7
    assert rel(m.lora_down.weight.grad, dA) < 1e-2
    assert rel(m.lora_up.weight.grad, dB) < 1e-2
    assert m.conv.weight.grad is None


def test_conv_kernel_fp32_out_tight():
    """fp32 output, scale = 0: pure frozen conv, only accumulation order differs (1e-5);
    T side output = conv(x, A16) to 1e-5."""
    from lora_b200 import ops
    torch.manual_seed(0)
    n, cin, cout, H, W, r = 2, 96, 72, 20, 20, 5
    dt = torch.bfloat16
    x = torch.randn(n, cin, H, W, device=DEV).to(dt).contiguous(memory_format=torch.channels_last)
    Wt = (torch.randn(cout, cin, 3, 3, device=DEV) * 0.05).to(dt)
    A = torch.randn(r, cin, 3, 3, device=DEV) / r
    B = torch.randn(cout, r, device=DEV) * 0.05
    bias = torch.randn(cout, device=DEV)
    wf, wb = ops.cast_conv_weight(Wt, dt, True, True)
    assert torch.equal(wf.view(cout, 9, cin), Wt.permute(0, 2, 3, 1).reshape(cout, 9, cin))
    assert torch.equal(wb.view(cin, 9, cout), Wt.flip(2, 3).permute(1, 2, 3, 0).reshape(cin, 9, cout))
    d16 = ops.conv_down16(A, dt, {})
    assert torch.equal(d16[:r].view(r, 9, cin), A.permute(0, 2, 3, 1).reshape(r, 9, cin).to(dt))
    y, T = ops.fused_conv2d(x, wf, bias, d16, B, 0, r, 1, 0, None, 0.0, r, cout, 3, 3, 1, 1, False,
                            torch.float32, True)
    torch.cuda.synchronize()
    ref = O.lora_conv2d_forward(x, Wt, bias, A, torch.zeros(cout, r, 1, 1), 0.0, padding=1)
    assert rel(y, ref) < 1e-5
    A16 = d16[:r].view(r, 3, 3, cin).permute(0, 3, 1, 2).float()
    t_ref = torch.nn.functional.conv2d(x.double().cpu(), A16.double().cpu(), padding=1)
    t_ref = t_ref.permute(0, 2, 3, 1).reshape(-1, r)
    assert rel(T[:, :r], t_ref) < 1e-5
    assert torch.count_nonzero(T[:, r:]) == 0


def test_conv_unsupported_geometry_raises():
    import lora_b200 as L
    from lora_b200._C import LoraB200Error
    m = L.LoraInjectedConv2d(16, 16, 3, 2, 1, r=4, dropout_p=0.0).to(DEV)
    with pytest.raises(LoraB200Error):
        m(torch.randn(1, 16, 8, 8, device=DEV, dtype=torch.bfloat16))
