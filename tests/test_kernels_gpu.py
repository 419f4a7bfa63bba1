"""GPU parity of the single-problem fused LoRA-linear launches (lb_lora_linear_fwd and
lb_lora_linear_fwd_dropout, csrc/fused_linear.cu; kernel fused_lora_kernel, csrc/fused_core.cuh) and
of the factor-gradient reductions against float64: oracle/lora_ops.py and plain float64 matrix
products, evaluated on the GPU, through ctypes.

The first tests (the SHAPES census, the backward chain, the forced schedules) are also run by
test_sd2_gpu.py / test_sdxl_gpu.py / test_sample_xl_gpu.py at their own site shapes, with whole-tensor
bounds. The kernel-level census below them is driven by `linear_plan`, a restatement of the launch
planner: an unmarked CPU test checks that the census, the T_in cases and the dropout cases together
reach all 40 launch branches at 132 SMs (H100 SXM), and a GPU test checks the same at the device's
own SM count. The census holds the single-site linear shapes of SD1.5 at 512 px (batch 1 and 2),
SD2.1 at 768 px, SDXL at 1024 px and the CLIP-L / OpenCLIP-H / OpenCLIP-bigG attention and MLP sites,
each forward problem and its transposed input-gradient problem, minus the levels above 4096 rows
(they reach no branch a smaller shape does not), plus ragged synthetic shapes. Every launch of the
census writes into NaN-filled outputs with 256-byte guards: every element of Y and of T must be
written, no guard byte touched.

Every bound of the census is checked on the whole tensor AND separately on the last 128-row tile and
on the last BLOCK_N-column tile of the plan the launch takes (192 for the 192-wide plan), so that an
error in a ragged tile cannot hide in a Frobenius norm over the whole output.

Tolerances (those of test_conv_kernels_gpu.py and test_grouped_kernels_gpu.py):
  * frozen GEMM (scale = 0, fp32 output) and the T side output: 16-bit operands are exact in fp32
    products, only the fp32 accumulation differs from float64 -> rel < max(1e-5, K/16 * 2^-24); the
    second term allows half an fp32 ulp per 16-deep K-step (the tensor core truncates when it adds a
    K-step into the fp32 accumulator; test_conv_kernels_gpu.py). T's padded columns [r, r_pad) are
    zero. The older SHAPES tests keep their flat 1e-5 (their K stays below 2684, where both agree).
  * full output against a model with the kernel's declared roundings (A and B as 16-bit copies, the
    scaled rank-r activations T' = 16-bit(fp32(T * scale * diag)) formed from the kernel's own fp32 T,
    or from T_in): fp32 output < 3e-4 (a few T' entries on a 16-bit rounding boundary land one ulp
    apart, measured 6e-5), 16-bit output < one 16-bit ulp (2^-8 bf16, 2^-11 fp16).
  * fp32 output against the unrounded oracle: err <= 2^-7 * ||LoRA branch|| + 1e-5 * ||ref||.
  * dropout: the exact keep-mask (oracle/dropmask.py) goes into the model and the oracle; the bounds
    above apply unchanged.
  * factor gradients fed the kernels' own T and dTs: rel < 2e-5; against the fully unrounded oracle
    1e-2 (test_backward_kernels_match_oracle).
"""
import math
from collections import namedtuple
from functools import partial

import pytest
import torch

from oracle import dropmask as DM
from oracle import lora_ops as O
from test_conv_kernels_gpu import Guarded

DEV = "cuda"
F64, F32 = torch.float64, torch.float32
BF, FP = torch.bfloat16, torch.float16
gpu = pytest.mark.gpu


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


@gpu
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


@gpu
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


@gpu
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


@gpu
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


@gpu
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


@gpu
def test_linearity_full_size():
    """Size-independent property at the largest SD1.5 site: f(x1 + x2) - f(0) = f(x1) + f(x2) - 2 f(0)."""
    M, K, N, r = 4096, 320, 2560, 4
    x, W, A, B, b, d = make_case(M, K, N, r, torch.bfloat16, seed=3)
    x1 = (x.float() * 0.5).to(torch.bfloat16)
    y1, _, _ = run_fused(x1, W, A, B, b, d, 1.0, torch.float32, want_t=False)
    y2, _, _ = run_fused((x1.float() * 2).to(torch.bfloat16), W, A, B, b, d, 1.0, torch.float32, want_t=False)
    y0, _, _ = run_fused(torch.zeros_like(x1), W, A, B, b, d, 1.0, torch.float32, want_t=False)
    assert rel_err(y2 - y0, 2 * (y1 - y0)) < 2e-3  # only T' bf16 rounding differs between the two


@gpu
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


# ==================================================================================== launch plan
Plan = namedtuple("Plan", "rp form bn stages out min_ctas split inline_tma")


def rank_pad(r):
    return 16 if r <= 16 else (32 if r <= 32 else 64)


def plan_split(M, K, N, n_sms):
    """Split factor of the L2 split-K plan (1: none); restates plan_split, csrc/fused_linear.cu:56-78."""
    num_kb, m_tiles, bn = -(-K // 64), -(-M // 128), 64
    tiles = m_tiles * -(-N // bn)
    per_kb = (128.0 + bn + 16.0) * 128.0 / 92e3
    base_t = -(-tiles // n_sms) * (2.0 + num_kb * per_kb)
    best, best_t = 1, 1e30
    for sp in range(2, 9):
        if tiles * sp > n_sms or num_kb // sp < 4:
            break
        t = 2.0 + -(-num_kb // sp) * per_kb + 3.0
        if t < best_t:
            best_t, best = t, sp
    return best if best > 1 and best_t < 0.75 * base_t else 1


def linear_plan(M, K, N, r_pad, out, drop, t_in, n_sms):
    """Which kernel lb_lora_linear_fwd / _dropout launch in the auto schedule (lb_debug_set_linear_mode(0)):
    linear_fwd_impl, csrc/fused_linear.cu:189-285, with launch_linear_wide (108-128) and plan_split (56-78).
    out: "f32" or "16". Returns Plan(rank pad, form, BLOCK_N, stages, output, CTAs per SM, split, inline
    TMA); split is the split-K factor ("splitk" forms), the cluster size ("cluster") or 1. Forms:
    "plain", "t_in" (rank activations read from T_in: no cluster or 192-wide plan), "drop" (masked drain),
    "splitk" / "t_in splitk" / "drop splitk" (L2 split-K), "cluster" (cluster split-K), "192" (192-wide).
    At rank pads 32 and 64 the planner does not look at T_in: those launches are "plain"."""
    m_tiles = -(-M // 128)
    t128, t64 = m_tiles * -(-N // 128), m_tiles * -(-N // 64)
    f32 = out == "f32"
    if r_pad > 16:
        narrow = t64 <= n_sms
        bn = 64 if narrow or (drop and f32 and r_pad == 64) else 128
        return Plan(r_pad, "drop" if drop else "plain", bn, 4, out, 1, 1, False)
    if drop:
        sp = plan_split(M, K, N, n_sms)
        if sp > 1:
            return Plan(16, "drop splitk", 64, 4 if f32 else 5, out, 1, sp, False)
        nar = t128 < 120 and not (K >= 2048 and t128 >= 64)
        return Plan(16, "drop", 64, 3, out, 2, 1, False) if nar else Plan(16, "drop", 128, 4, out, 1, 1, False)
    sp = plan_split(M, K, N, n_sms)
    if sp > 1:
        return Plan(16, "t_in splitk" if t_in else "splitk", 64, 5 if f32 else 6, out, 1, sp, False)
    if not t_in:
        if K >= 640 and t64 * 2 <= n_sms:
            return Plan(16, "cluster", 64, 4 if f32 else 6, out, 1, 2, False)
        if not f32 and t128 > n_sms and m_tiles * -(-N // 192) <= n_sms and K >= 640:
            return Plan(16, "192", 192, 4, out, 1, 1, False)
    narrow = t64 <= n_sms or (t64 <= 2 * n_sms and K < 2048 and m_tiles >= 8)
    if K >= 2048 and t128 >= 64:
        narrow = False
    crowded = (t64 if narrow else t128) > n_sms
    form = "t_in" if t_in else "plain"
    if f32:
        return Plan(16, form, 64, 3, out, 2, 1, False) if narrow else Plan(16, form, 128, 4, out, 1, 1, False)
    if narrow:
        return Plan(16, form, 64, 2, out, 2, 1, False) if crowded else Plan(16, form, 64, 7, out, 1, 1, False)
    return Plan(16, form, 128, 2, out, 2, 1, True) if crowded else Plan(16, form, 128, 4, out, 1, 1, False)


def branch(p):
    """A launch branch: the plan with the split-K factor reduced to split or not."""
    return p._replace(split=p.split > 1)


def _all_branches():
    req = set()
    for out in ("f32", "16"):
        f32 = out == "f32"
        for form in ("plain", "t_in"):
            req |= {Plan(16, form, 64, 3 if f32 else 2, out, 2, False, False),
                    Plan(16, form, 128, 4 if f32 else 2, out, 1 if f32 else 2, False, not f32),
                    Plan(16, form + " splitk" if form == "t_in" else "splitk", 64, 5 if f32 else 6, out, 1, True,
                         False)}
            if not f32:
                req |= {Plan(16, form, 64, 7, out, 1, False, False), Plan(16, form, 128, 4, out, 1, False, False)}
        req |= {Plan(16, "cluster", 64, 4 if f32 else 6, out, 1, True, False),
                Plan(16, "drop splitk", 64, 4 if f32 else 5, out, 1, True, False),
                Plan(16, "drop", 64, 3, out, 2, False, False), Plan(16, "drop", 128, 4, out, 1, False, False)}
        for rp in (32, 64):
            for bn in (64, 128):
                req.add(Plan(rp, "plain", bn, 4, out, 1, False, False))
                if not (rp == 64 and f32 and bn == 128):      # does not fit shared memory: runs 64 wide
                    req.add(Plan(rp, "drop", bn, 4, out, 1, False, False))
    req.add(Plan(16, "192", 192, 4, "16", 1, False, False))
    return req


ALL_BRANCHES = _all_branches()
OUTS = ("f32", "16")

# (id, M, K, N, r, bias, diag, scale): the single-site problems. "_dx" is the input gradient of the
# site of the same name: [M, N] x W [N, K], i.e. the site's K and N swapped.
CENSUS = [
    # SD1.5, 512 px, batch 1 (64 x 64 .. 8 x 8 latents, 77-token context of 768)
    ("sd15_64_qkv", 4096, 320, 320, 4, False, False, 0.7),
    ("sd15_64_geglu", 4096, 320, 2560, 16, True, True, -1.3),
    ("sd15_64_geglu_dx", 4096, 2560, 320, 1, False, False, 1.9),
    ("sd15_64_ffout", 4096, 1280, 320, 32, True, True, 0.45),
    ("sd15_kv320", 77, 768, 320, 3, False, True, 0.0),
    ("sd15_kv320_dx", 77, 320, 768, 64, False, True, -0.6),
    ("sd15_32_qkv", 1024, 640, 640, 17, False, True, 1.1),
    ("sd15_32_geglu", 1024, 640, 5120, 24, True, False, -0.8),
    ("sd15_16_geglu", 256, 1280, 10240, 8, True, True, 0.9),
    ("sd15_16_geglu_dx", 256, 10240, 1280, 4, False, True, -1.2),
    ("sd15_16_ffout", 256, 5120, 1280, 64, True, False, 0.7),
    ("sd15_8_qkv", 64, 1280, 1280, 33, False, True, 1.3),
    ("sd15_time_emb", 1, 1280, 320, 16, True, True, 0.8),
    # batch 2
    ("sd15_b2_32_qkv", 2048, 640, 640, 4, False, True, -0.9),
    ("sd15_b2_kv640", 154, 768, 640, 16, False, False, 0.0),
    ("sd15_b2_16_ffout_dx", 512, 1280, 5120, 3, False, True, 1.4),
    # SD2.1, 768 px (96 x 96 latents; the 9216-row level left out), 77-token context of 1024
    ("sd21_48_qkv", 2304, 640, 640, 64, True, True, 0.6),
    ("sd21_24_geglu_dx", 576, 10240, 1280, 4, False, False, 1.0),
    ("sd21_kv1280", 77, 1024, 1280, 32, False, True, -1.1),
    ("sd21_12_qkv", 144, 1280, 1280, 1, True, False, 0.5),
    # SDXL, 1024 px (128 x 128 latents), 77-token context of 2048
    ("sdxl_64_qkv", 4096, 640, 640, 16, False, True, 0.75),
    ("sdxl_32_geglu", 1024, 1280, 10240, 4, True, False, -0.7),
    ("sdxl_kv1280", 77, 2048, 1280, 3, False, True, 1.2),
    ("sdxl_32_ffout", 1024, 5120, 1280, 24, True, True, 0.65),
    # text encoders (77 tokens): attention and MLP sites, with bias
    ("clip_l_qkv", 77, 768, 768, 4, True, False, 0.9),
    ("clip_l_fc1", 77, 768, 3072, 17, True, True, -0.5),
    ("clip_l_fc2", 77, 3072, 768, 16, True, True, 1.1),
    ("openclip_h_qkv", 77, 1024, 1024, 33, True, False, 0.8),
    ("openclip_h_fc1", 77, 1024, 4096, 8, True, True, -1.5),
    ("openclip_h_fc2", 77, 4096, 1024, 64, True, True, 0.7),
    ("bigg_qkv", 77, 1280, 1280, 16, True, False, 1.6),
    ("bigg_fc1", 77, 1280, 5120, 3, True, True, 0.4),
    ("bigg_fc2", 77, 5120, 1280, 32, True, False, -0.9),
    # synthetic, ragged: M % 128, K % 64 and N % BLOCK_N != 0, M = 1; one per plan family
    ("ragged_mkn", 130, 72, 88, 3, True, True, 0.8),
    ("ragged_m1", 1, 200, 328, 1, True, False, -1.4),
    ("ragged_splitk", 200, 2560, 136, 5, True, True, 0.9),
    ("ragged_cluster", 130, 776, 88, 12, False, True, -1.0),
    ("ragged_192", 200, 1280, 10240, 16, True, True, 0.6),
    ("ragged_inline", 4000, 328, 2552, 4, True, False, 1.2),
    ("ragged_rp32", 300, 200, 136, 24, True, True, 0.0),
    ("ragged_rp64", 3000, 136, 1000, 40, False, True, -0.7),
]

# (id, M, K, N, r): the site whose input gradient runs from T_in ([M, N] x W [N, K] -> [M, K])
TIN_CASES = [
    ("sd15_16_geglu", 256, 1280, 10240, 4),        # L2 split-K
    ("sd15_64_qkv", 4096, 320, 320, 16),           # 64 wide, 2 CTAs per SM
    ("sd15_64_geglu", 4096, 320, 2560, 3),         # 128 wide, one CTA per SM (16-bit)
    ("sd15_64_ffout", 4096, 1280, 320, 8),         # 128 wide, inline TMA (16-bit)
    ("sd15_kv320", 77, 768, 320, 1),               # 64 wide, deep ring (16-bit)
    ("ragged", 300, 200, 136, 5),
    ("ragged_splitk", 200, 136, 2560, 12),
    ("sd15_32_qkv", 1024, 640, 640, 24),           # rank pad 32
    ("clip_l_fc1", 77, 768, 3072, 40),             # rank pad 64
    ("ragged_rp64", 130, 72, 88, 64),
]

# (id, M, K, N, r, p, backward chain): dropout on the branch, forward (and, once per rank pad, backward)
DROP_CASES = [
    ("sd15_16_ffout", 256, 5120, 1280, 8, 0.25, False),     # L2 split-K with the masked drain
    ("sd15_64_qkv", 4096, 320, 320, 4, 0.1, False),         # 64 wide
    ("sd15_64_geglu", 4096, 320, 2560, 16, 0.25, False),    # 128 wide
    ("ragged", 333, 200, 648, 3, 0.5, True),
    ("ragged_splitk", 200, 2560, 136, 5, 0.2, False),
    ("sd15_32_qkv", 1024, 640, 640, 24, 0.1, True),         # rank pad 32, 64 wide
    ("sd15_64_qkv_r32", 4096, 320, 320, 32, 0.25, False),   # rank pad 32, 128 wide
    ("ragged_rp32", 130, 72, 88, 17, 0.3, False),
    ("sd15_kv320", 77, 768, 320, 64, 0.25, True),           # rank pad 64, 64 wide
    ("sd15_64_qkv_r40", 4096, 320, 320, 40, 0.1, False),    # rank pad 64: fp32 forced 64 wide, 16-bit 128
]


def census_branches(n_sms):
    seen = set()
    for out in OUTS:
        for (_, M, K, N, r, *_) in CENSUS:
            seen.add(branch(linear_plan(M, K, N, rank_pad(r), out, False, False, n_sms)))
        for (_, M, K, N, r) in TIN_CASES:
            seen.add(branch(linear_plan(M, N, K, rank_pad(r), out, False, True, n_sms)))
        for (_, M, K, N, r, _, _) in DROP_CASES:
            seen.add(branch(linear_plan(M, K, N, rank_pad(r), out, True, False, n_sms)))
    return seen


def test_census_reaches_every_linear_launch_branch():
    """CPU: at 132 SMs (H100 SXM) the census, T_in and dropout cases reach all 40 launch branches."""
    assert len(ALL_BRANCHES) == 40
    missing = ALL_BRANCHES - census_branches(132)
    assert not missing, sorted(map(str, missing))


@gpu
def test_census_reaches_every_linear_launch_branch_on_this_device():
    missing = ALL_BRANCHES - census_branches(n_sms())
    assert not missing, (n_sms(), sorted(map(str, missing)))


def test_linear_plan_moves_with_the_sm_count():
    """The OpenCLIP-H fc1 site fits one cluster wave on 132 SMs (2 x 64 CTAs), not on 114; the
    16 x 16 GEGLU input gradient splits 3 ways on 132 SMs, 2 ways on 114."""
    assert linear_plan(77, 1024, 4096, 16, "16", False, False, 132) == Plan(16, "cluster", 64, 6, "16", 1, 2, False)
    assert linear_plan(77, 1024, 4096, 16, "16", False, False, 114) == Plan(16, "plain", 64, 7, "16", 1, 1, False)
    assert linear_plan(77, 1024, 4096, 16, "f32", False, False, 114) == Plan(16, "plain", 64, 3, "f32", 2, 1, False)
    for form, t_in, drop in (("splitk", False, False), ("t_in splitk", True, False), ("drop splitk", False, True)):
        assert linear_plan(256, 10240, 1280, 16, "f32", drop, t_in, 132).split == 3
        p = linear_plan(256, 10240, 1280, 16, "f32", drop, t_in, 114)
        assert (p.form, p.split) == (form, 2)


def test_ragged_cases_cover_every_plan_family():
    """A case whose last row tile or last BLOCK_N-column tile is partial reaches each plan family."""
    fams = set()

    def add(M, N, p):
        if M % 128 or N % p.bn:
            fams.add(p.form.split()[-1] if p.rp == 16 else f"rp{p.rp}")
            fams.update({"inline"} if p.inline_tma else set())
            fams.update({"drop"} if "drop" in p.form else set())
    for out in OUTS:
        for (_, M, K, N, r, *_) in CENSUS:
            add(M, N, linear_plan(M, K, N, rank_pad(r), out, False, False, 132))
        for (_, M, K, N, r) in TIN_CASES:
            add(M, K, linear_plan(M, N, K, rank_pad(r), out, False, True, 132))
        for (_, M, K, N, r, _, _) in DROP_CASES:
            add(M, N, linear_plan(M, K, N, rank_pad(r), out, True, False, 132))
    assert {"splitk", "cluster", "192", "inline", "drop", "t_in", "plain", "rp32", "rp64"} <= fams, fams


# ==================================================================================== helpers
def n_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def acc_tol(K):
    """Bound for a tensor-core reduction over K (module docstring)."""
    return max(1e-5, K / 16 * 2.0 ** -24)


def ulp16(dt):
    return 2.0 ** -8 if dt == BF else 2.0 ** -11


def regions(M, N, bn):
    """(name, rows, cols): the whole tensor, the last 128-row tile, the last bn-column tile."""
    return [("all", slice(None), slice(None)), ("last row tile", slice((M - 1) // 128 * 128, None), slice(None)),
            ("last column tile", slice(None), slice((N - 1) // bn * bn, None))]


def check_rel(got, ref, tol, bn, what):
    got, ref = got.detach().to(DEV, F64), ref.detach().to(DEV, F64)
    for name, rs, cs in regions(*ref.shape, bn):
        g, r_ = got[rs, cs], ref[rs, cs]
        e = float((g - r_).norm() / (r_.norm() + 1e-30))
        assert e < tol, f"{what} [{name}]: rel {e:.3e} >= {tol:.1e}"


def check_branch(got, ref, base, bn, what):
    """err <= 2^-7 ||ref - base|| + 1e-5 ||ref|| on every region (base: the frozen GEMM + bias)."""
    got, ref, base = (t.detach().to(DEV, F64) for t in (got, ref, base))
    for name, rs, cs in regions(*ref.shape, bn):
        g, r_, b_ = got[rs, cs], ref[rs, cs], base[rs, cs]
        err, bound = float((g - r_).norm()), 2.0 ** -7 * float((r_ - b_).norm()) + 1e-5 * float(r_.norm())
        assert err <= bound, f"{what} [{name}]: err {err:.3e} > {bound:.3e}"


def check_t(T, t_ref, r, K, what):
    """T side output: rel < acc_tol(K) on the whole tensor and the last row tile, padded columns zero."""
    check_rel(T[:, :r], t_ref, acc_tol(K), r, what)
    assert torch.count_nonzero(T[:, r:]) == 0, f"{what}: padded rank columns written"


def tprime(T, r, scale, diag, dt):
    """T' as the drain forms it: fp32 T * fp32(scale * diag), rounded to the 16-bit operand type."""
    coef = torch.full((r,), scale, dtype=F32, device=DEV)
    if diag is not None:
        coef = coef * diag.float()
    return (T[:, :r] * coef).to(dt).to(F64)


def device_case(M, K, N, r, dt, seed, bias, diag):
    return tuple(None if t is None else t.to(DEV) for t in make_case(M, K, N, r, dt, seed, bias=bias, diag=diag))


def launch(x, w, bias, d16, up, up_rs, up_cs, diag, scale, r, out_dt, want_t=True, t_in=None, drop_p=0.0,
           seed=None, out=None):
    """lb_lora_linear_fwd (drop_p = 0) or lb_lora_linear_fwd_dropout, straight into NaN-filled Y and T
    with 256-byte guards (out=None), or into the given (Y, T). Returns (Y, T or None, [Guarded])."""
    from lora_b200 import _C
    from lora_b200._C import check, dtype_code, ptr, stream_ptr
    M, K = x.shape
    N, rp = w.shape[0], d16.shape[0]
    if out is None:
        gs = [Guarded((M, N), out_dt)] + ([Guarded((M, rp), F32)] if want_t else [])
        y, t = gs[0].t, gs[1].t if want_t else None
    else:
        gs, (y, t) = [], out
    head = (ptr(x), ptr(w), ptr(bias), ptr(d16), ptr(up), up_rs, up_cs, ptr(diag), float(scale), ptr(y), ptr(t))
    codes = (dtype_code(x.dtype), dtype_code(out_dt))
    if drop_p > 0.0:
        check(_C.lib.lb_lora_linear_fwd_dropout(*head, M, K, N, r, rp, *codes, float(drop_p), ptr(seed),
                                                stream_ptr()), "lb_lora_linear_fwd_dropout")
    else:
        check(_C.lib.lb_lora_linear_fwd(*head, ptr(t_in), M, K, N, r, rp, *codes, stream_ptr()),
              "lb_lora_linear_fwd")
    return y, t, gs


def check_guards(gs, what):
    torch.cuda.synchronize()
    for g in gs:
        g.check(what)


DTS = [pytest.param(BF, id="bf16"), pytest.param(FP, id="fp16")]


# ==================================================================================== census
@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", CENSUS, ids=lambda c: c[0])
def test_linear_launch_matches_float64(case, dt):
    """Frozen GEMM and T at scale 0, T of both launches, fp32 and 16-bit output against the rounded-T'
    model, fp32 output against the unrounded oracle; every output written, no guard byte touched."""
    ops = _ops()
    name, M, K, N, r, bias, diag, scale = case
    x, W, A, B, b, d = device_case(M, K, N, r, dt, M + K + N + r, bias, diag)
    rp = rank_pad(r)
    bn = {out: linear_plan(M, K, N, rp, out, False, False, n_sms()).bn for out in OUTS}
    d16 = ops.cast_rows_pad16(A, K, 1, r, K, dt)
    y0, T0, g0 = launch(x, W, b, d16, B, r, 1, d, 0.0, r, F32)
    y32, T32, g32 = launch(x, W, b, d16, B, r, 1, d, scale, r, F32)
    y16, T16, g16 = launch(x, W, b, d16, B, r, 1, d, scale, r, dt)
    check_guards(g0 + g32 + g16, name)
    x64, W64 = x.to(F64), W.to(F64)
    base = x64 @ W64.T + (0.0 if b is None else b.to(F64))
    t_ref = x64 @ d16[:r].to(F64).T
    check_rel(y0, base, acc_tol(K), bn["f32"], f"{name}: frozen GEMM (scale 0)")
    for T, what in ((T0, "T (scale 0)"), (T32, "T (fp32 out)"), (T16, "T (16-bit out)")):
        check_t(T, t_ref, r, K, f"{name}: {what}")
    B16 = B.to(dt).to(F64)
    check_rel(y32, base + tprime(T32, r, scale, d, dt) @ B16.T, 3e-4, bn["f32"], f"{name}: fp32 out vs rounded model")
    check_rel(y16, base + tprime(T16, r, scale, d, dt) @ B16.T, ulp16(dt), bn["16"],
              f"{name}: 16-bit out vs rounded model")
    ref = O.lora_linear_forward(x, W, b, A, B, scale, diag=d, device=DEV)
    check_branch(y32, ref, base, bn["f32"], f"{name}: fp32 out vs oracle")


# ==================================================================================== T_in
def tin_operands(M, K, N, r, dt, seed):
    """The dX launch of a dropout site's backward (modules._FusedLoraLinearFn): gY [M, N] on W^T (wt16)
    and B^T (upT16), up = A read transposed, and a dTs that is NOT gY . B16: independent values, padded
    columns included (the kernel must ignore columns >= r)."""
    ops = _ops()
    x, W, A, B, _, d = device_case(M, K, N, r, dt, seed, False, True)
    g = torch.Generator().manual_seed(seed)
    gy = torch.randn(M, N, generator=g).to(dt).to(DEV)
    dts = (torch.randn(M, rank_pad(r), generator=g) * 3).to(DEV)
    _, wt16 = ops.cast_weight(W, dt, False, True)
    upT16 = ops.cast_rows_pad16(B, 1, r, r, N, dt)
    return x, W, A, B, d, gy, dts, wt16, upT16


@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", TIN_CASES, ids=lambda c: c[0])
def test_input_gradient_from_t_in_matches_float64(case, dt):
    """dX = gY.W + (dTs' * scale * diag).A16 with fp32 and 16-bit dX; T_out, when requested, is T_in."""
    name, M, K, N, r = case
    scale = -0.8
    x, W, A, B, d, gy, dts, wt16, upT16 = tin_operands(M, K, N, r, dt, M + K + N + r)
    base = gy.to(F64) @ W.to(F64)
    model = base + tprime(dts, r, scale, d, dt) @ A.to(dt).to(F64)
    exact = base + (dts[:, :r].to(F64) * (scale * d.to(F64))) @ A.to(F64)
    for out in OUTS:
        bn = linear_plan(M, N, K, rank_pad(r), out, False, True, n_sms()).bn
        odt = F32 if out == "f32" else dt
        what = f"{name} dX {out}"
        dx, tout, gs = launch(gy, wt16, None, upT16, A, 1, K, d, scale, r, odt, want_t=(out == "f32"), t_in=dts)
        check_guards(gs, what)
        if tout is not None:
            assert torch.equal(tout, dts), f"{what}: T_out differs from T_in"
        check_rel(dx, model, 3e-4 if out == "f32" else ulp16(dt), bn, what + " vs rounded model")
        if out == "f32":
            check_branch(dx, exact, base, bn, what + " vs float64")


# ==================================================================================== dropout, exact
_MASKS = {}


def linear_mask(seed, p, M, N):
    key = (seed, p, M, N)
    if key not in _MASKS:
        _MASKS[key] = torch.from_numpy(DM.linear_mask(seed, p, M, N)).to(DEV, F64)
    return _MASKS[key]


@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", DROP_CASES, ids=lambda c: c[0])
def test_dropout_launch_matches_oracle_with_the_exact_mask(case, dt):
    """Forward (masked drain) with fp32 and 16-bit output against the model and the oracle fed the
    mask of oracle/dropmask.py; with `chain`, the backward of modules._FusedLoraLinearFn with p > 0:
    masked dT pass, dX from T_in, dA, masked dB."""
    ops = _ops()
    name, M, K, N, r, p, chain = case
    scale = 1.25
    x, W, A, B, b, d = device_case(M, K, N, r, dt, M + K + N + r + 1, True, True)
    seed = 0x5DEECE66D1234567 + M + r
    seed_t = torch.tensor([seed], dtype=torch.int64, device=DEV)
    mask = linear_mask(seed, p, M, N)
    d16 = ops.cast_rows_pad16(A, K, 1, r, K, dt)
    x64, W64 = x.to(F64), W.to(F64)
    base = x64 @ W64.T + b.to(F64)
    t_ref = x64 @ d16[:r].to(F64).T
    ref = O.lora_linear_forward(x, W, b, A, B, scale, diag=d, keep_mask=mask, dropout_p=p, device=DEV)
    T = None
    for out in OUTS:
        bn = linear_plan(M, K, N, rank_pad(r), out, True, False, n_sms()).bn
        odt = F32 if out == "f32" else dt
        what = f"{name} dropout {out}"
        y, t, gs = launch(x, W, b, d16, B, r, 1, d, scale, r, odt, drop_p=p, seed=seed_t)
        check_guards(gs, what)
        check_t(t, t_ref, r, K, what + ": T")
        model = base + mask * (tprime(t, r, scale, d, dt) @ B.to(dt).to(F64).T) / (1.0 - p)
        check_rel(y, model, 3e-4 if out == "f32" else ulp16(dt), bn, what + " vs rounded model")
        if out == "f32":
            check_branch(y, ref, base, bn, what + " vs oracle")
            T = t
    if not chain:
        return
    g = torch.Generator().manual_seed(M + r)
    gy = torch.randn(M, N, generator=g).to(dt).to(DEV)
    dTs = ops.dropout_dt(gy, B, r, 1, p, seed_t, r)
    check_t(dTs, (gy.to(F64) * mask / (1.0 - p)) @ B.to(F64), r, N, "masked dT")
    _, wt16 = ops.cast_weight(W, dt, False, True)
    upT16 = ops.cast_rows_pad16(B, 1, r, r, N, dt)
    dX, _, gs = launch(gy, wt16, None, upT16, A, 1, K, d, scale, r, F32, want_t=False, t_in=dTs)
    dA = torch.zeros(r, K, device=DEV)
    dB = torch.zeros(N, r, device=DEV)
    ops.wgrad(x, dTs, d, scale, dA, K, 1, r)
    ops.wgrad_masked(gy, T, d, scale, dB, 1, r, r, p, seed_t)
    check_guards(gs, "dropout dX")
    rdX, rdA, _ = O.lora_linear_backward(gy, x, W, A, B, scale, diag=d, keep_mask=mask, dropout_p=p, device=DEV)
    _, _, rdB = O.lora_linear_backward(gy, x, W, d16[:r].float(), B, scale, diag=d, keep_mask=mask, dropout_p=p,
                                       device=DEV)
    dx_base = gy.to(F64) @ W64
    bn = linear_plan(M, N, K, rank_pad(r), "f32", False, True, n_sms()).bn
    check_rel(dX, dx_base + tprime(dTs, r, scale, d, dt) @ A.to(dt).to(F64), 3e-4, bn, "dropout dX vs rounded model")
    check_branch(dX, rdX, dx_base, bn, "dropout dX vs oracle")
    assert rel_err(dA, rdA) < 2e-5, "dA"
    assert rel_err(dB, rdB) < 2e-5, "dB"


# ==================================================================================== split-K state
RING_BYTES, RING_COUNTERS = 96 << 20, 1 << 16        # the split workspace, lora_b200/csrc/tmap.h:106-107


def _split_footprint(M, N):
    """(bytes, counters) one linear split launch takes from the ring: tiles * 128 * (64 + 16) * 4 bytes
    (rounded up to 256, tmap.h split_ws_reserve) and one counter per tile (fused_linear.cu:26-31)."""
    tiles = -(-M // 128) * -(-N // 64)
    return (tiles * 128 * 80 * 4 + 255) // 256 * 256, tiles


def _split_runs(dt, scale):
    """Three L2 split-K launches (plain, T_in, dropout), each with fp32 output, its float64 reference
    and its oracle bound; each launch's arguments are bound when the run is made (partial)."""
    ops = _ops()
    runs = []
    # plain: the OpenCLIP-bigG fc2 site
    M, K, N, r = 77, 5120, 1280, 8
    x, W, A, B, b, d = device_case(M, K, N, r, dt, 11, True, True)
    d16 = ops.cast_rows_pad16(A, K, 1, r, K, dt)
    ref = O.lora_linear_forward(x, W, b, A, B, scale, diag=d, device=DEV)
    base = x.to(F64) @ W.to(F64).T + b.to(F64)
    runs.append(("plain", (M, K, N, False, False), ref, base,
                 partial(launch, x, W, b, d16, B, r, 1, d, scale, r, F32)))
    # T_in: the input gradient of the 16 x 16 GEGLU site
    M, K, N, r = 256, 1280, 10240, 4
    _, W2, A2, _, d2, gy, dts, wt16, upT16 = tin_operands(M, K, N, r, dt, 12)
    base2 = gy.to(F64) @ W2.to(F64)
    ref2 = base2 + (dts[:, :r].to(F64) * (scale * d2.to(F64))) @ A2.to(F64)
    runs.append(("T_in", (M, N, K, True, False), ref2, base2,
                 partial(launch, gy, wt16, None, upT16, A2, 1, K, d2, scale, r, F32, t_in=dts)))
    # dropout: the 16 x 16 feed-forward output site
    M, K, N, r, p = 256, 5120, 1280, 16, 0.25
    x3, W3, A3, B3, b3, d3 = device_case(M, K, N, r, dt, 13, True, True)
    d163 = ops.cast_rows_pad16(A3, K, 1, r, K, dt)
    seed = 0x1234567890ABCDEF
    seed_t = torch.tensor([seed], dtype=torch.int64, device=DEV)
    ref3 = O.lora_linear_forward(x3, W3, b3, A3, B3, scale, diag=d3, keep_mask=linear_mask(seed, p, M, N),
                                 dropout_p=p, device=DEV)
    base3 = x3.to(F64) @ W3.to(F64).T + b3.to(F64)
    runs.append(("dropout", (M, K, N, False, True), ref3, base3,
                 partial(launch, x3, W3, b3, d163, B3, r, 1, d3, scale, r, F32, drop_p=p, seed=seed_t)))
    for (what, (M, K, N, t_in, drop), *_rest) in runs:
        assert linear_plan(M, K, N, 16, "f32", drop, t_in, n_sms()).split > 1, f"{what}: not a split plan here"
    return [(what, prob, ref, 2.0 ** -7 * float((ref - base).norm()) + 1e-5 * float(ref.norm()), call)
            for (what, prob, ref, base, call) in runs]


@gpu
def test_split_workspace_ring_wraps_twice_without_stale_partials():
    """Plain, T_in and dropout split launches interleaved for as many launches as make the workspace
    ring (bytes and counters) wrap twice: a partial or an election counter left behind by an earlier
    launch only shows once a launch is handed a region an earlier one used. Every output starts as NaN."""
    runs = _split_runs(BF, 0.9)
    feet = [_split_footprint(M, N) for (_, (M, K, N, _, _), *_r) in runs]
    rounds = math.ceil(2 * max(RING_BYTES / sum(f[0] for f in feet), RING_COUNTERS / sum(f[1] for f in feet))) + 1
    ys = [torch.empty(ref.shape, dtype=F32, device=DEV) for (_, _, ref, _, _) in runs]
    errs = torch.empty(rounds, len(runs), dtype=F64, device=DEV)
    for i in range(rounds):
        for j, (_, _, ref, _, call) in enumerate(runs):
            ys[j].fill_(float("nan"))
            call(out=(ys[j], None))
            errs[i, j] = (ys[j].to(F64) - ref).norm()
    torch.cuda.synchronize()
    for j, (what, _, _, bound, _) in enumerate(runs):
        bad = (~(errs[:, j] <= bound)).nonzero().flatten()
        assert bad.numel() == 0, \
            f"{what}: launches {bad[:8].tolist()} of {rounds} off ({errs[bad[0], j]:.3e} > {bound:.3e})"


@gpu
def test_t_in_and_dropout_split_launches_inside_a_cuda_graph():
    """One T_in and one dropout split launch captured once, replayed 3 times into NaN-refilled outputs."""
    runs = [r for r in _split_runs(FP, -1.1) if r[0] != "plain"]
    ys = [torch.empty(ref.shape, dtype=F32, device=DEV) for (_, _, ref, _, _) in runs]
    for (_, _, _, _, call), y in zip(runs, ys):
        call(out=(y, None))                    # allocates the split workspace outside the capture
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for (_, _, _, _, call), y in zip(runs, ys):
            call(out=(y, None))
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for (_, _, _, _, call), y in zip(runs, ys):
            call(out=(y, None))
    for rep in range(3):
        for y in ys:
            y.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        for (what, _, ref, bound, _), y in zip(runs, ys):
            err = float((y.to(F64) - ref).norm())
            assert err <= bound, f"{what} replay {rep}: err {err:.3e} > {bound:.3e}"
