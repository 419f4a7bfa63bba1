"""GPU parity of the raw C-ABI kernels against the oracle (oracle/lora_ops.py), through ctypes.

Tolerances (stated per test):
  * base GEMM / T, fp32 output: 16-bit inputs are exact in fp32 products, only the fp32
    accumulation order differs from the float64 oracle -> rel Frobenius error < 2e-6 ... 1e-5.
  * full fused output: the kernel rounds the scaled rank-r activations T' to the 16-bit operand
    type before the up-projection (like the reference under autocast, which rounds lora_down's
    output). Against the oracle fed the same rounding: < 1e-5 (fp32 out) / one 16-bit ulp (bf16 out).
    Against the unrounded oracle: error bounded by 2^-8 of the LoRA-branch magnitude.
"""
import pytest
import torch

from oracle import lora_ops as O

pytestmark = pytest.mark.gpu


def _ops():
    from lora_b200 import ops
    return ops


def rel_err(a, b):
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def make_case(M, K, N, r, dtype, seed, bias=True, diag=False):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(M, K, generator=g).to(dtype)
    W = (torch.randn(N, K, generator=g) * 0.05).to(dtype)
    A = torch.randn(r, K, generator=g) / r
    B = torch.randn(N, r, generator=g) * 0.05
    b = torch.randn(N, generator=g) * 0.1 if bias else None
    d = (torch.rand(r, generator=g) + 0.5) if diag else None
    return x, W, A, B, b, d


def run_fused(x, W, A, B, b, d, scale, out_dtype, want_t=True):
    ops = _ops()
    dev = "cuda"
    r, K = A.shape
    N = W.shape[0]
    xd, Wd = x.to(dev), W.to(dev)
    Ad, Bd = A.to(dev), B.to(dev)
    down16 = ops.cast_rows_pad16(Ad, K, 1, r, K, x.dtype)
    y, t = ops.fused_linear(xd, Wd, None if b is None else b.to(dev), down16, Bd, r, 1,
                            None if d is None else d.to(dev), scale, r, out_dtype, want_t)
    torch.cuda.synchronize()
    return y, t, down16


SHAPES = [
    # (M, K, N, r)  -- SD1.5 site census + ragged edges
    (4096, 320, 320, 4),
    (4096, 320, 2560, 4),
    (1024, 640, 640, 4),
    (1024, 640, 5120, 8),
    (256, 1280, 1280, 4),
    (256, 1280, 10240, 16),
    (64, 1280, 1280, 4),
    (77, 768, 320, 4),
    (77, 768, 768, 1),
    (77, 768, 1280, 12),
    (1, 1280, 320, 8),        # time_emb_proj site of the extended set (M = 1)
    (130, 72, 88, 3),         # ragged everything: partial M, K and N tiles
    (128, 64, 64, 16),
    (300, 200, 136, 5),
]


@pytest.mark.parametrize("M,K,N,r", SHAPES)
def test_base_gemm_and_T_fp32_out(M, K, N, r):
    """scale = 0 isolates the frozen GEMM (+bias); T_out = X.A16^T. fp32 accumulate => tight."""
    x, W, A, B, b, d = make_case(M, K, N, r, torch.bfloat16, seed=M + K + N + r)
    y, t, down16 = run_fused(x, W, A, B, b, d, 0.0, torch.float32)
    ref = O.lora_linear_forward(x, W, b, A, torch.zeros_like(B), 0.0)
    assert rel_err(y, ref) < 1e-5
    t_ref = x.double() @ down16.cpu().double().T
    assert rel_err(t, t_ref) < 1e-5
    assert torch.count_nonzero(t[:, r:]) == 0


@pytest.mark.parametrize("M,K,N,r", SHAPES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_fused_forward_matches_oracle(M, K, N, r, dtype):
    scale = 0.7
    x, W, A, B, b, d = make_case(M, K, N, r, dtype, seed=7 * M + K + N + r, diag=(r % 2 == 0))
    y32, t, down16 = run_fused(x, W, A, B, b, d, scale, torch.float32)
    y16, _, _ = run_fused(x, W, A, B, b, d, scale, dtype, want_t=False)

    # (1) oracle with the kernel's declared roundings (A, B and T' rounded to the operand type)
    A16 = down16[:r].cpu().float()
    dd = torch.ones(r) if d is None else d
    tprime = ((x.double() @ A16.double().T) * (scale * dd.double())).float().to(dtype)
    ref_model = O.lora_linear_forward(x, W, b, A16, torch.zeros_like(B), 0.0) + \
        tprime.double() @ B.to(dtype).double().T
    # not 1e-5: the kernel forms T' from an fp32 accumulation, the model from float64, so a few
    # T' entries sitting on a 16-bit rounding boundary land one 16-bit ulp apart (measured 6e-5)
    assert rel_err(y32, ref_model) < 3e-4
    ulp = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11
    assert rel_err(y16, ref_model) < ulp

    # (2) the plain oracle (reference semantics, fp64, unrounded LoRA factors)
    ref = O.lora_linear_forward(x, W, b, A, B, scale, diag=d)
    branch = (ref - O.lora_linear_forward(x, W, b, A, torch.zeros_like(B), 0.0)).norm()
    err = (y32.double().cpu() - ref).norm()
    assert float(err) <= 2.0 ** -7 * float(branch) + 1e-5 * float(ref.norm())


@pytest.mark.parametrize("M,K,N,r", [(4096, 320, 320, 4), (1024, 640, 5120, 8), (77, 768, 1280, 12),
                                     (130, 72, 88, 3), (256, 1280, 1280, 16)])
def test_backward_kernels_match_oracle(M, K, N, r):
    """dX through the same fused kernel on W^T; dA/dB through the skinny wgrad reduction."""
    ops = _ops()
    dtype = torch.bfloat16
    scale = 1.3
    x, W, A, B, b, d = make_case(M, K, N, r, dtype, seed=11 * M + N, diag=True)
    g = torch.Generator().manual_seed(5)
    gy = torch.randn(M, N, generator=g).to(dtype)
    dev = "cuda"
    xd, Wd, Ad, Bd, dd, gyd = (t.to(dev) for t in (x, W, A, B, d, gy))
    _, Wt = ops.cast_weight(Wd, dtype, False, True)
    assert torch.equal(Wt, Wd.t().contiguous())
    down16 = ops.cast_rows_pad16(Ad, K, 1, r, K, dtype)
    bt16 = ops.cast_rows_pad16(Bd, 1, r, r, N, dtype)
    assert torch.equal(bt16[:r], Bd.t().to(dtype))
    # forward (for T)
    _, T = ops.fused_linear(xd, Wd, None, down16, Bd, r, 1, dd, scale, r, dtype, True)
    # dX = gY.W + ((gY.B)*s*d).A   and  dTs = gY.B16
    dX, dTs = ops.fused_linear(gyd, Wt, None, bt16, Ad, 1, K, dd, scale, r, torch.float32, True)
    dA = torch.zeros(r, K, device=dev)
    dB = torch.zeros(N, r, device=dev)
    ops.wgrad(xd, dTs, dd, scale, dA, K, 1, r)
    ops.wgrad(gyd, T, dd, scale, dB, 1, r, r)
    torch.cuda.synchronize()

    A16 = down16[:r].cpu().float()
    B16 = bt16[:r].cpu().float().t().contiguous()
    # oracle with 16-bit-rounded factors where the kernels consume 16-bit copies
    rdX, _, _ = O.lora_linear_backward(gy, x, W, A, B16, scale, diag=d)
    _, rdA, _ = O.lora_linear_backward(gy, x, W, A, B16, scale, diag=d)
    _, _, rdB = O.lora_linear_backward(gy, x, W, A16, B, scale, diag=d)
    assert rel_err(dA, rdA) < 2e-5
    assert rel_err(dB, rdB) < 2e-5
    # dX: T' is rounded to bf16 before the A-projection
    base = gy.double() @ W.double()
    branch = (rdX - base).norm()
    assert float((dX.double().cpu() - rdX).norm()) <= 2.0 ** -7 * float(branch) + 1e-5 * float(rdX.norm())
    # and against the unrounded oracle, loosely
    fdX, fdA, fdB = O.lora_linear_backward(gy, x, W, A, B, scale, diag=d)
    assert rel_err(dX, fdX) < 1e-2 and rel_err(dA, fdA) < 1e-2 and rel_err(dB, fdB) < 1e-2


@pytest.mark.parametrize("M,K,N,r", [(256, 1280, 2304, 4), (64, 640, 1000, 8), (300, 320, 192, 4)])
def test_block_n_192_schedule_matches_default(M, K, N, r):
    """The 192-wide tile (208-column accumulator incl. T, 3 store boxes; 16-bit outputs) is the same math."""
    from lora_b200 import _C
    x, W, A, B, b, d = make_case(M, K, N, r, torch.bfloat16, seed=M + N + r, diag=True)
    try:
        assert _C.lib.lb_debug_set_linear_mode(1 + 4 * 3) == 0
        y, t, _ = run_fused(x, W, A, B, b, d, 0.9, torch.bfloat16)
    finally:
        _C.lib.lb_debug_set_linear_mode(0)
    y0, t0, _ = run_fused(x, W, A, B, b, d, 0.9, torch.bfloat16)
    assert rel_err(t, t0) < 3e-6
    assert rel_err(y, y0) < 3e-3          # both rounded to bf16 once


@pytest.mark.parametrize("mode", [1 + 4, 1 + 8, 2 + 4, 2 + 8])
@pytest.mark.parametrize("M,K,N,r", SHAPES)
def test_every_tile_schedule_gives_the_same_result(M, K, N, r, mode):
    """Forced schedules 1 (one tile per CTA; 2 CTAs per SM on crowded sites) and 2 (one CTA per SM)
    at BLOCK_N 64 and 128 vs the auto schedule: same math, results equal to fp32-accumulation noise
    (1e-5) between schedules and vs the oracle. The cluster split-K schedule is
    tests/test_zz_splitk_experimental_gpu.py."""
    from lora_b200 import _C
    x, W, A, B, b, d = make_case(M, K, N, r, torch.bfloat16, seed=M * 3 + N + r, diag=True)
    try:
        _C.lib.lb_debug_set_linear_mode(mode)
        y, t, down16 = run_fused(x, W, A, B, b, d, 0.9, torch.float32)
    finally:
        _C.lib.lb_debug_set_linear_mode(0)
    y0, t0, _ = run_fused(x, W, A, B, b, d, 0.9, torch.float32)
    assert rel_err(t, t0) < 3e-6       # fp32 summation order only (auto may pick a split-K plan)
    assert rel_err(y, y0) < 3e-4
    ref = O.lora_linear_forward(x, W, b, A, B, 0.9, diag=d)
    branch = (ref - O.lora_linear_forward(x, W, b, A, torch.zeros_like(B), 0.0)).norm()
    assert float((y.double().cpu() - ref).norm()) <= 2.0 ** -7 * float(branch) + 1e-5 * float(ref.norm())


def test_linearity_full_size():
    """Size-independent property at the largest SD1.5 site: f(x1 + x2) - f(0) = f(x1) + f(x2) - 2 f(0)."""
    M, K, N, r = 4096, 320, 2560, 4
    x, W, A, B, b, d = make_case(M, K, N, r, torch.bfloat16, seed=3)
    x1 = (x.float() * 0.5).to(torch.bfloat16)
    y1, _, _ = run_fused(x1, W, A, B, b, d, 1.0, torch.float32, want_t=False)
    y2, _, _ = run_fused((x1.float() * 2).to(torch.bfloat16), W, A, B, b, d, 1.0, torch.float32, want_t=False)
    y0, _, _ = run_fused(torch.zeros_like(x1), W, A, B, b, d, 1.0, torch.float32, want_t=False)
    assert rel_err(y2 - y0, 2 * (y1 - y0)) < 2e-3  # only T' bf16 rounding differs between the two


def test_rejects_bad_arguments():
    ops = _ops()
    from lora_b200._C import LoraB200Error
    x, W, A, B, b, d = make_case(64, 64, 64, 4, torch.bfloat16, seed=1)
    dev = "cuda"
    down16 = ops.cast_rows_pad16(A.to(dev), 64, 1, 4, 64, torch.bfloat16)
    with pytest.raises(LoraB200Error):
        ops.fused_linear(x.to(dev), W.to(dev), None, down16, B.to(dev), 4, 1, None, 1.0, 17,
                         torch.bfloat16, False)
    with pytest.raises(LoraB200Error):
        ops.fused_linear(x, W, None, down16.cpu(), B, 4, 1, None, 1.0, 4, torch.bfloat16, False)
