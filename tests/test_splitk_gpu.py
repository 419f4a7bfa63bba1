"""Split-K plans of the fused kernels (csrc/fused_core.cuh, SPLITK; planners in fused_linear.cu /
fused_conv.cu): sites with few output tiles and a long reduction (the dX of the GEGLU projections,
the 8x8 / 16x16 ResnetBlock2D convs) are split over gridDim.z CTAs per tile, every CTA adds its
partial accumulator into an L2-resident fp32 buffer (vector reductions) and the last CTA to arrive
reads the reduced tile back and finishes it. Parity
against the float64 oracle on exactly the shapes where `auto` picks a split, repeated launches (the
election counters must reset themselves), CUDA-graph replay, and the dropout drain on a split tile."""
import pytest
import torch

from oracle import lora_ops as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


# (M, K, N, r): shapes for which plan_split() chooses split > 1 on a 132-SM H100
LONG_K = [(256, 10240, 1280, 4), (1024, 5120, 640, 8), (64, 10240, 1280, 16), (256, 5120, 1280, 4),
          (77, 2560, 768, 12), (1, 5120, 320, 8), (200, 2560, 136, 3)]


@pytest.mark.parametrize("M,K,N,r", LONG_K)
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
def test_split_plans_match_oracle_and_reset_their_counters(M, K, N, r, out_dtype):
    from test_kernels_gpu import make_case, run_fused
    x, W, A, B, b, d = make_case(M, K, N, r, torch.bfloat16, seed=M + K + N + r, diag=True)
    ref = O.lora_linear_forward(x, W, b, A, B, 0.9, diag=d)
    base = O.lora_linear_forward(x, W, b, A, torch.zeros_like(B), 0.0)
    branch = float((ref - base).norm())
    t_ref = None
    for rep in range(3):                     # same workspace ring / counters re-used
        y, t, down16 = run_fused(x, W, A, B, b, d, 0.9, out_dtype)
        if t_ref is None:
            t_ref = x.double() @ down16.cpu().double().T
        assert rel(t, t_ref) < 1e-5
        tol = 2.0 ** -7 * branch + (1e-5 if out_dtype == torch.float32 else 2.0 ** -8) * float(ref.norm())
        assert float((y.double().cpu() - ref).norm()) <= tol, rep


def test_split_plan_equals_unsplit_schedule_bitwise_close():
    """Same site through a forced un-split schedule (one tile per CTA, BLOCK_N 64) and through auto."""
    from lora_b200 import _C
    from test_kernels_gpu import make_case, run_fused
    x, W, A, B, b, d = make_case(256, 10240, 1280, 4, torch.bfloat16, seed=1, diag=False)
    y_auto, t_auto, _ = run_fused(x, W, A, B, b, d, 1.0, torch.float32)
    try:
        _C.lib.lb_debug_set_linear_mode(1 + 4)
        y_one, t_one, _ = run_fused(x, W, A, B, b, d, 1.0, torch.float32)
    finally:
        _C.lib.lb_debug_set_linear_mode(0)
    # fp32 summation order over K = 10240 differs (7 partials reduced at L2 vs one serial chain)
    assert rel(t_auto, t_one) < 3e-5 and rel(y_auto, y_one) < 3e-4


def test_split_plan_inside_a_cuda_graph():
    from lora_b200 import ops
    from test_kernels_gpu import make_case
    x, W, A, B, b, d = make_case(256, 10240, 1280, 4, torch.bfloat16, seed=2)
    xd, Wd, Ad, Bd, bd = (t.to(DEV) for t in (x, W, A, B, b))
    d16 = ops.cast_rows_pad16(Ad, 10240, 1, 4, 10240, torch.bfloat16)
    y0, _ = ops.fused_linear(xd, Wd, bd, d16, Bd, 4, 1, None, 1.0, 4, torch.bfloat16, True)   # allocates the workspace
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.fused_linear(xd, Wd, bd, d16, Bd, 4, 1, None, 1.0, 4, torch.bfloat16, True)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y, t = ops.fused_linear(xd, Wd, bd, d16, Bd, 4, 1, None, 1.0, 4, torch.bfloat16, True)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, y0) or rel(y, y0) < 2 ** -8


def test_conv_dropout_forward_on_a_split_tile():
    """8x8 mid-block conv (1 row tile, K = 9 x 1280): split-K AND the masked drain in one kernel."""
    import lora_b200 as L
    torch.manual_seed(3)
    p = 0.25
    m = L.LoraInjectedConv2d(1280, 1280, 3, 1, 1, r=8, dropout_p=p, scale=1.0).to(DEV)
    m.conv.requires_grad_(False)
    m.conv.weight.data.mul_(0.3)
    m.lora_up.weight.data.normal_(0, 0.3)
    x = torch.randn(1, 1280, 8, 8, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    m.train()
    y = m(x)
    m.eval()
    y_clean = m(x)
    W16 = m.conv.weight.detach().to(torch.bfloat16)
    base = O.lora_conv2d_forward(x, W16, m.conv.bias, m.lora_down.weight, torch.zeros_like(m.lora_up.weight), 0.0, padding=1)
    clean = O.lora_conv2d_forward(x, W16, m.conv.bias, m.lora_down.weight, m.lora_up.weight, 1.0, padding=1) - base
    assert rel(y_clean, base + clean) < 2 ** -7
    branch = y.detach().double().cpu() - base
    big = clean.abs() > 0.5 * clean.abs().mean()
    ratio = (branch / clean)[big]
    kept = ratio.abs() > 0.5
    assert abs(float(kept.double().mean()) - (1 - p)) < 0.02
    assert abs(float(ratio[kept].median()) - 1 / (1 - p)) < 0.05
