"""LoRA sites with active dropout on the branch (training mode, p > 0), GPU.

The keep-mask comes from a counter-based hash, not ATen's Philox stream, so these are the
distribution-level checks the reference semantics allow (nn.Dropout: keep prob 1-p, survivors
scaled by 1/(1-p), the SAME mask in forward and backward), plus exactness in the degenerate
cases (eval mode == no dropout)."""
import pytest
import torch
import torch.nn as nn

from oracle import lora_ops as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _mod(K=320, N=640, r=4, p=0.25, bias=True):
    import lora_b200 as L
    torch.manual_seed(0)
    m = L.LoraInjectedLinear(K, N, bias=bias, r=r, dropout_p=p, scale=1.5).to(DEV)
    m.linear.requires_grad_(False)
    m.lora_up.weight.data.normal_(0, 0.2)
    return m


def test_mask_recovered_from_forward_is_consistent_with_backward():
    """Recover the realised mask from y (branch/clean-branch ratio), then check dX, dA, dB equal
    the oracle's backward evaluated WITH THAT MASK."""
    p = 0.25
    m = _mod(p=p)
    M, K, N, r = 512, 320, 640, 4
    x = torch.randn(M, K, device=DEV).to(torch.bfloat16).float().requires_grad_(True)
    m.train()
    y = m(x)                                    # fp32 in, fp32 out (bf16 operands)
    gy = torch.randn(M, N, device=DEV).to(torch.bfloat16).float()
    y.backward(gy)
    W16 = m.linear.weight.detach().to(torch.bfloat16)
    A, B = m.lora_down.weight.detach(), m.lora_up.weight.detach()
    base = O.lora_linear_forward(x, W16, m.linear.bias, A, torch.zeros_like(B), 0.0)
    clean = O.lora_linear_forward(x, W16, m.linear.bias, A, B, 1.5) - base      # un-dropped branch
    branch = y.detach().double().cpu() - base
    ratio = branch / clean
    big = clean.abs() > 0.05 * clean.abs().mean()
    kept = (ratio.abs() > 0.5)
    keep_rate = float(kept[big].double().mean())
    assert abs(keep_rate - (1 - p)) < 0.01, keep_rate
    # survivors are scaled by 1/(1-p) (up to bf16 rounding of the rank-r activations)
    surv = ratio[big & kept]
    assert abs(float(surv.median()) - 1 / (1 - p)) < 0.02
    mask = kept.double()
    dX, dA, dB = O.lora_linear_backward(gy, x.detach(), W16, A, B, 1.5, keep_mask=mask, dropout_p=p)
    # elements with tiny |clean| are classified unreliably: compare with a tolerance that absorbs them
    assert rel(x.grad, dX) < 3e-2
    assert rel(m.lora_down.weight.grad, dA) < 3e-2
    assert rel(m.lora_up.weight.grad, dB) < 3e-2


def test_eval_mode_and_p0_are_exactly_the_no_dropout_path():
    m = _mod(p=0.3)
    x = torch.randn(2, 77, 320, device=DEV, dtype=torch.bfloat16)
    m.eval()
    y_eval = m(x)
    m.dropout.p = 0.0
    m.train()
    y_p0 = m(x)
    assert torch.equal(y_eval, y_p0)
    ref = O.lora_linear_forward(x.reshape(-1, 320), m.linear.weight.to(torch.bfloat16), m.linear.bias,
                                m.lora_down.weight, m.lora_up.weight, 1.5)
    assert rel(y_eval.reshape(-1, 640), ref) < 2 ** -7


def test_masks_differ_between_calls_and_expectation_matches():
    m = _mod(p=0.5)
    m.train()
    x = torch.randn(256, 320, device=DEV, dtype=torch.bfloat16)
    ys = torch.stack([m(x).float() for _ in range(64)])
    assert not torch.equal(ys[0], ys[1])
    m.eval()
    y_clean = m(x).float()
    # E[dropout(u)] = u: the mean over n = 64 calls approaches the eval output with relative
    # error sqrt(p/(1-p)/n) = 0.125 OF THE BRANCH (p = 0.5); bounds: random masks, unbiased scaling
    m.dropout.p = 0.0
    from oracle import lora_ops as O
    base = O.lora_linear_forward(x, m.linear.weight.to(torch.bfloat16), m.linear.bias, m.lora_down.weight,
                                 torch.zeros_like(m.lora_up.weight), 0.0)
    br_mean = ys.mean(0).double().cpu() - base
    br_clean = y_clean.double().cpu() - base
    err = float((br_mean - br_clean).norm() / br_clean.norm())
    assert 0.06 < err < 0.2, err


def test_conv_dropout_statistics_and_grads_finite():
    import lora_b200 as L
    torch.manual_seed(1)
    m = L.LoraInjectedConv2d(64, 64, 3, 1, 1, r=8, dropout_p=0.1, scale=1.0).to(DEV)
    m.conv.requires_grad_(False)
    m.lora_up.weight.data.normal_(0, 0.2)
    x = torch.randn(2, 64, 16, 16, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    m.train()
    y = m(x)
    y.float().square().mean().backward()
    m.eval()
    y_clean = m(x.detach())
    W16 = m.conv.weight.detach().to(torch.bfloat16)
    base = O.lora_conv2d_forward(x, W16, m.conv.bias, m.lora_down.weight, torch.zeros_like(m.lora_up.weight), 0.0, padding=1)
    branch = y.detach().double().cpu() - base
    clean = y_clean.double().cpu() - base
    big = clean.abs() > 0.2 * clean.abs().mean()
    keep_rate = float(((branch / clean).abs() > 0.5)[big].double().mean())
    assert abs(keep_rate - 0.9) < 0.02, keep_rate
    for g in (x.grad, m.lora_down.weight.grad, m.lora_up.weight.grad):
        assert g is not None and torch.isfinite(g).all() and float(g.abs().sum()) > 0


def test_conv_dropout_backward_matches_oracle_with_recovered_mask():
    """Conv site with active dropout: recover the realised keep-mask from the forward output
    (branch / clean-branch ratio, as for the linear site above), then dX, dA, dB must equal the
    oracle's backward (oracle/lora_ops.py::lora_conv2d_backward, autograd of lora.py:130-135)
    evaluated WITH THAT MASK. The up factor is given a floor away from zero so that almost every
    branch element is classifiable; the tolerance absorbs the few that are not."""
    import lora_b200 as L
    torch.manual_seed(2)
    p, r, cin, cout, H = 0.2, 8, 64, 128, 16
    m = L.LoraInjectedConv2d(cin, cout, 3, 1, 1, r=r, dropout_p=p, scale=1.25).to(DEV)
    m.conv.requires_grad_(False)
    m.lora_up.weight.data.normal_(0, 0.3)
    x = (torch.randn(2, cin, H, H, device=DEV).to(torch.bfloat16)
         .contiguous(memory_format=torch.channels_last).requires_grad_(True))
    m.train()
    y = m(x)
    gy = torch.randn_like(y)
    y.backward(gy)
    W16 = m.conv.weight.detach().to(torch.bfloat16)
    A, B = m.lora_down.weight.detach(), m.lora_up.weight.detach()
    base = O.lora_conv2d_forward(x.detach(), W16, m.conv.bias, A, torch.zeros_like(B), 0.0, padding=1)
    clean = O.lora_conv2d_forward(x.detach(), W16, m.conv.bias, A, B, 1.25, padding=1) - base
    branch = y.detach().double().cpu() - base
    ratio = branch / clean
    kept = ratio.abs() > 0.5
    big = clean.abs() > 0.05 * clean.abs().mean()
    assert abs(float(kept[big].double().mean()) - (1 - p)) < 0.02
    dX, dA, dB = O.lora_conv2d_backward(gy, x.detach(), W16, A, B, 1.25, padding=1,
                                        keep_mask=kept.double(), dropout_p=p)
    assert rel(x.grad, dX) < 3e-2
    assert rel(m.lora_down.weight.grad, dA) < 3e-2
    assert rel(m.lora_up.weight.grad, dB) < 3e-2
