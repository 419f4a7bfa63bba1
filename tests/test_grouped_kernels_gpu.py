"""Kernel-level parity of the grouped fused LoRA-linear launch (lb_lora_linear_fwd_grouped,
csrc/fused_linear.cu; kernel fused_lora_grouped_kernel, csrc/fused_core.cuh) against float64:
oracle/lora_ops.py and plain float64 matrix products, evaluated on the GPU.

The launch is called as the autograd glue calls it (grouping.py: the forward of a family of sites that
share an input, and the family's input gradient on the transposed weights, whose dTs then feed
lb_lora_wgrad_multi). The forward census holds the families of SD1.5 at 512 px (batch 1 and 2), SD2.1
at 768 px, SDXL at 1024 px and the q/k/v of the CLIP-L / OpenCLIP text encoders (with bias), minus the
levels above 4096 rows (the 9216 / 8192-token self-attentions): the kernel sees only tiles, and those
levels reach no launch plan that a smaller family of the census does not. Every member of a family has
its own rank, scale and selector diagonal, so a member that reads another member's parameters is off.
`grouped_plan` restates the planner; an unmarked CPU test checks that the census reaches all six launch
plans at 132 SMs (H100 SXM), and a GPU test checks the same at the device's own SM count.

Every bound is checked on the whole tensor AND separately on the last 128-row tile and on the last
BLOCK_N-column tile of the plan the launch takes, so that an error in a ragged tile cannot hide in a
Frobenius norm over the whole output.

Tolerances (those of test_kernels_gpu.py and test_conv_kernels_gpu.py):
  * frozen GEMM (scale = 0, fp32 output) and the T side output: 16-bit operands are exact in fp32
    products, only the fp32 accumulation differs from float64 -> rel < max(1e-5, K/16 * 2^-24); the
    second term is the conv suite's allowance of half an fp32 ulp per 16-deep K-step (the tensor core
    truncates when it adds a K-step into the fp32 accumulator). T's padded columns [r, 16) are zero.
  * full output against a model with the kernel's declared roundings (A and B as 16-bit copies, the
    scaled rank-r activations T' = 16-bit(fp32(T * scale * diag)) formed from the kernel's own T):
    fp32 output < 3e-4, 16-bit output < one 16-bit ulp (2^-8 bf16, 2^-11 fp16).
  * fp32 output against the unrounded oracle: err <= 2^-7 * ||LoRA branch|| + 1e-5 * ||ref||.
  * input gradient: the same three bounds with the roles of W / W^T and A / B swapped; the factor
    gradients fed the kernels' own T and dTs: rel < 2e-5; against the fully unrounded oracle 1e-2
    (test_backward_kernels_match_oracle).
  * module level under autocast: the output is 16-bit, so its rounding (at most half a 16-bit ulp per
    element) replaces the 1e-5 * ||ref|| term of the oracle bound by one 16-bit ulp * ||ref||.
"""
import ctypes
from collections import namedtuple

import pytest
import torch
import torch.nn as nn

import test_kernels_gpu as KG
from test_kernels_gpu import acc_tol, check_branch, check_rel, check_t, n_sms, tprime, ulp16
from oracle import lora_ops as O

DEV = "cuda"
F64, F32 = torch.float64, torch.float32
BF, FP = torch.bfloat16, torch.float16
gpu = pytest.mark.gpu


# ------------------------------------------------------------------------------------ launch plan
Plan = namedtuple("Plan", "bn stages out min_ctas inline_tma")


def grouped_plan(problems, out_dtype, n_sms):
    """Which kernel lb_lora_linear_fwd_grouped launches (lora_b200/csrc/fused_linear.cu:322-350).
    problems: [(M, K, N)]; out_dtype: "f32" or "16"."""
    tiles128 = sum(-(-M // 128) * -(-N // 128) for (M, _, N) in problems)
    tiles64 = sum(-(-M // 128) * -(-N // 64) for (M, _, N) in problems)
    narrow = tiles128 < 120
    crowded = (tiles64 if narrow else tiles128) > n_sms
    if out_dtype == "f32":
        return Plan(64, 3, "f32", 2, False) if narrow else Plan(128, 4, "f32", 1, False)
    if narrow:
        return Plan(64, 2, "16", 2, False) if crowded else Plan(64, 7, "16", 1, False)
    return Plan(128, 2, "16", 2, True) if crowded else Plan(128, 4, "16", 1, False)


ALL_PLANS = {Plan(64, 3, "f32", 2, False), Plan(128, 4, "f32", 1, False), Plan(64, 2, "16", 2, False),
             Plan(64, 7, "16", 1, False), Plan(128, 2, "16", 2, True), Plan(128, 4, "16", 1, False)}

# (id, M, K, Ns, bias): the families grouping.py forms (sites fed one tensor)
FAMILIES = [
    # SD1.5, 512 px, batch 1: self-attention q/k/v per level, cross-attention k/v on the 77-token context
    ("sd15_b1_64x64_qkv", 4096, 320, (320,) * 3, False),
    ("sd15_b1_32x32_qkv", 1024, 640, (640,) * 3, False),
    ("sd15_b1_16x16_qkv", 256, 1280, (1280,) * 3, False),
    ("sd15_b1_8x8_qkv", 64, 1280, (1280,) * 3, False),
    ("sd15_b1_kv320", 77, 768, (320,) * 2, False),
    ("sd15_b1_kv640", 77, 768, (640,) * 2, False),
    ("sd15_b1_kv1280", 77, 768, (1280,) * 2, False),
    # batch 2
    ("sd15_b2_32x32_qkv", 2048, 640, (640,) * 3, False),
    ("sd15_b2_16x16_qkv", 512, 1280, (1280,) * 3, False),
    ("sd15_b2_8x8_qkv", 128, 1280, (1280,) * 3, False),
    ("sd15_b2_kv320", 154, 768, (320,) * 2, False),
    ("sd15_b2_kv1280", 154, 768, (1280,) * 2, False),
    # SD2.1, 768 px (96 x 96 latents), 1024-wide context
    ("sd21_48x48_qkv", 2304, 640, (640,) * 3, False),
    ("sd21_24x24_qkv", 576, 1280, (1280,) * 3, False),
    ("sd21_12x12_qkv", 144, 1280, (1280,) * 3, False),
    ("sd21_kv320", 77, 1024, (320,) * 2, False),
    ("sd21_kv640", 77, 1024, (640,) * 2, False),
    ("sd21_kv1280", 77, 1024, (1280,) * 2, False),
    # SDXL, 1024 px (128 x 128 latents), 2048-wide context
    ("sdxl_64x64_qkv", 4096, 640, (640,) * 3, False),
    ("sdxl_32x32_qkv", 1024, 1280, (1280,) * 3, False),
    ("sdxl_kv640", 77, 2048, (640,) * 2, False),
    ("sdxl_kv1280", 77, 2048, (1280,) * 2, False),
    # text encoders: q/k/v with bias
    ("clip_l_qkv", 77, 768, (768,) * 3, True),
    ("openclip_h_qkv", 77, 1024, (1024,) * 3, True),
    ("openclip_bigg_qkv", 77, 1280, (1280,) * 3, True),
    # synthetic: the narrow, crowded 16-bit plan, which no real site reaches at batch 1
    ("narrow_crowded_640", 640, 640, (640,) * 3, False),
]
# per member of a family: rank, scale, selector diagonal
RANKS, SCALES, DIAGS = (4, 16, 3, 8), (0.7, -1.3, 1.9, 0.45), (False, True, True, True)


def census_plans(n_sms):
    return {grouped_plan([(M, K, N) for N in Ns], out, n_sms) for (_, M, K, Ns, _) in FAMILIES
            for out in ("f32", "16")}


def test_census_reaches_every_grouped_launch_plan():
    """CPU: at 132 SMs (H100 SXM) the forward census reaches all six plans."""
    assert census_plans(132) == ALL_PLANS


def test_grouped_plan_moves_with_the_sm_count():
    """(256, 1280, [1280] x 3): 120 64-wide tiles, a single wave on 132 SMs, crowded on 114."""
    fam = [(256, 1280, 1280)] * 3
    assert grouped_plan(fam, "16", 132) == Plan(64, 7, "16", 1, False)
    assert grouped_plan(fam, "16", 114) == Plan(64, 2, "16", 2, False)
    assert grouped_plan([(4096, 320, 320)] * 3, "16", 132).inline_tma
    assert grouped_plan([(1024, 640, 640)] * 3, "16", 132) == Plan(128, 4, "16", 1, False)


@gpu
def test_census_reaches_every_grouped_launch_plan_on_this_device():
    missing = ALL_PLANS - census_plans(n_sms())
    assert not missing, (n_sms(), sorted(missing))


# ------------------------------------------------------------------------------------ helpers
Member = namedtuple("Member", "x W A B bias diag scale r")


def _ops():
    from lora_b200 import ops
    return ops


def make_member(M, K, N, r, dt, seed, scale, bias=False, diag=False, x=None):
    """KG.make_case's operands on the device; x: the family's shared input (None: the member's own)."""
    x_, W, A, B, b, d = KG.make_case(M, K, N, r, dt, seed, bias=bias, diag=diag)
    dev = lambda t: None if t is None else t.to(DEV)
    return Member(dev(x_) if x is None else x, dev(W), dev(A), dev(B), dev(b), dev(d), float(scale), r)


def make_family(M, K, Ns, dt, seed, bias):
    mems = []
    for i, N in enumerate(Ns):
        mems.append(make_member(M, K, N, RANKS[i], dt, seed + 17 * i, SCALES[i], bias=bias, diag=DIAGS[i],
                                x=mems[0].x if mems else None))
    return mems


def shapes(mems):
    return [(m.x.shape[0], m.x.shape[1], m.W.shape[0]) for m in mems]


def problems(mems, dt, tiled=False, scale0=False):
    """The per-site tuples of grouping.py:112-113."""
    ops = _ops()
    out = []
    for m in mems:
        K = m.x.shape[1]
        d16 = ops.cast_rows_pad16(m.A, K, 1, m.r, K, dt)
        w = ops.tile_weight(m.W, dt) if tiled else m.W
        out.append((m.x, w, m.bias, d16, m.B, m.r, 1, m.diag, 0.0 if scale0 else m.scale, m.r))
    return out


def run_family(mems, dt, tiled=False):
    """Three grouped launches: scale 0 (fp32 out, T), the family (fp32 out, T), the family (16-bit out)."""
    ops = _ops()
    y0s, t0s = ops.fused_linear_grouped(problems(mems, dt, tiled, scale0=True), F32, True)
    probs = problems(mems, dt, tiled)
    y32s, ts = ops.fused_linear_grouped(probs, F32, True)
    y16s, none = ops.fused_linear_grouped(probs, dt, False)
    torch.cuda.synchronize()
    assert all(t is None for t in none)
    return [p[3] for p in probs], y0s, t0s, y32s, ts, y16s


def check_member(m, i, d16, y0, t0, y32, T, y16, dt, bn32, bn16, what):
    M, K = m.x.shape
    N, r = m.W.shape[0], m.r
    tag = f"{what} member {i} ({M}x{K}->{N} r{r} scale {m.scale})"
    x64, W64 = m.x.to(F64), m.W.to(F64)
    base = x64 @ W64.T + (0.0 if m.bias is None else m.bias.to(F64))
    t_ref = x64 @ d16[:r].to(F64).T
    if y0 is not None:
        check_rel(y0, base, acc_tol(K), bn32, tag + ": frozen GEMM (scale 0)")
        check_t(t0, t_ref, r, K, tag + ": T (scale 0)")
    if m.scale == 0.0 and y32 is not None:
        check_rel(y32, base, acc_tol(K), bn32, tag + ": scale-0 member vs frozen GEMM")
    check_t(T, t_ref, r, K, tag + ": T")
    y_model = base + tprime(T, r, m.scale, m.diag, dt) @ m.B.to(dt).to(F64).T
    if y32 is not None:
        check_rel(y32, y_model, 3e-4, bn32, tag + ": fp32 out vs rounded model")
        ref = O.lora_linear_forward(m.x, m.W, m.bias, m.A, m.B, m.scale, diag=m.diag, device=DEV)
        check_branch(y32, ref, base, bn32, tag + ": fp32 out vs oracle")
    if y16 is not None:
        check_rel(y16, y_model, ulp16(dt), bn16, tag + ": 16-bit out vs rounded model")


def check_family(mems, res, dt, what):
    d16s, y0s, t0s, y32s, ts, y16s = res
    bn32 = grouped_plan(shapes(mems), "f32", n_sms()).bn
    bn16 = grouped_plan(shapes(mems), "16", n_sms()).bn
    for i, m in enumerate(mems):
        check_member(m, i, d16s[i], y0s[i], t0s[i], y32s[i], ts[i], y16s[i], dt, bn32, bn16, what)


DTS = [pytest.param(BF, id="bf16"), pytest.param(FP, id="fp16")]


# ------------------------------------------------------------------------------------ forward census
@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("fam", FAMILIES, ids=lambda f: f[0])
def test_grouped_forward_matches_float64(fam, dt):
    name, M, K, Ns, bias = fam
    mems = make_family(M, K, Ns, dt, seed=M + K + sum(Ns), bias=bias)
    check_family(mems, run_family(mems, dt), dt, name)


# ------------------------------------------------------------------------------------ mixed members
# members that differ in M, K, N, rank, bias, selector and scale (0 and negative among them); the
# scale-0 member carries a bias, so its frozen GEMM shows whether a member past the first reads its own
HETERO = [(130, 72, 88, 3, True, False, 0.8), (77, 768, 320, 16, False, True, 1.1),
          (300, 200, 136, 1, True, False, 0.0), (4096, 320, 320, 4, False, False, -1.3)]


def hetero_members(dt):
    return [make_member(M, K, N, r, dt, seed=M + K + N + r, scale=s, bias=b, diag=d)
            for (M, K, N, r, b, d, s) in HETERO]


@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("n", [1, 4])
def test_grouped_members_of_different_shapes_match_float64(n, dt):
    """n = 1: each member launched alone; n = 4: all four in one launch (tile_start routes 4 problems)."""
    mems = hetero_members(dt)
    fams = [[m] for m in mems] if n == 1 else [mems]
    for fam in fams:
        check_family(fam, run_family(fam, dt), dt, f"n={n}")


def _arr(ty, vals):
    return (ty * len(vals))(*vals)


def columns(probs, ys, ts):
    """Per-problem argument columns of lb_lora_linear_fwd_grouped (as ops.fused_linear_grouped builds them)."""
    dp = lambda t: None if t is None else t.data_ptr()
    return dict(X=[p[0].data_ptr() for p in probs], W=[p[1].data_ptr() for p in probs], B=[dp(p[2]) for p in probs],
                D=[p[3].data_ptr() for p in probs], U=[p[4].data_ptr() for p in probs], RS=[p[5] for p in probs],
                CS=[p[6] for p in probs], DG=[dp(p[7]) for p in probs], SC=[float(p[8]) for p in probs],
                Y=[dp(y) for y in ys], T=[dp(t) for t in ts], M=[p[0].shape[0] for p in probs],
                K=[p[0].shape[1] for p in probs], N=[p[1].shape[0] for p in probs], R=[p[9] for p in probs])


def call_grouped(c, in_code, out_code, n=None):
    from lora_b200 import _C
    from lora_b200._C import check, stream_ptr
    VP, LL, I, F = ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_float
    n = len(c["X"]) if n is None else n
    check(_C.lib.lb_lora_linear_fwd_grouped(
        n, _arr(VP, c["X"]), _arr(VP, c["W"]), _arr(VP, c["B"]), _arr(VP, c["D"]), _arr(VP, c["U"]),
        _arr(LL, c["RS"]), _arr(LL, c["CS"]), _arr(VP, c["DG"]), _arr(F, c["SC"]), _arr(VP, c["Y"]),
        _arr(VP, c["T"]), _arr(I, c["M"]), _arr(I, c["K"]), _arr(I, c["N"]), _arr(I, c["R"]), in_code, out_code,
        stream_ptr()), "lb_lora_linear_fwd_grouped")


@gpu
@pytest.mark.parametrize("out", ["f32", "16"])
@pytest.mark.parametrize("dt", DTS)
def test_grouped_outputs_stay_inside_their_own_buffers(dt, out):
    """The four mixed members' Y and T carved from ONE buffer of 0xFF bytes (NaN in fp32, bf16 and
    fp16), separated by 16-byte-aligned gaps: no gap byte may change, every output element is written
    and each member matches its own float64 model."""
    from lora_b200._C import dtype_code
    mems = hetero_members(dt)
    probs = problems(mems, dt)
    odt = F32 if out == "f32" else dt
    esz = torch.empty((), dtype=odt).element_size()
    GAP = 272                          # a multiple of 16 bytes, of no TMA box or tile
    sizes = [(m.x.shape[0], m.W.shape[0], odt, esz) for m in mems] + [(m.x.shape[0], 16, F32, 4) for m in mems]
    offs, pos = [], GAP
    for (rows, cols, _, e) in sizes:
        offs.append(pos)
        pos += (rows * cols * e + 15) // 16 * 16 + GAP
    buf = torch.full((pos,), 0xFF, dtype=torch.uint8, device=DEV)
    views = [buf[o:o + rows * cols * e].view(t).view(rows, cols) for o, (rows, cols, t, e) in zip(offs, sizes)]
    ys, ts = views[:4], views[4:]
    call_grouped(columns(probs, ys, ts), dtype_code(dt), dtype_code(odt))
    torch.cuda.synchronize()
    gap = torch.ones(pos, dtype=torch.bool, device=DEV)
    for o, v in zip(offs, views):
        gap[o:o + v.numel() * v.element_size()] = False
    assert bool((buf[gap] == 0xFF).all()), "a gap byte between two members' outputs was written"
    for i, v in enumerate(views):
        assert not bool(torch.isnan(v.float()).any()), f"output {i}: elements left unwritten"
    plan = grouped_plan(shapes(mems), out, n_sms())
    for i, m in enumerate(mems):
        y32, y16 = (ys[i], None) if out == "f32" else (None, ys[i])
        check_member(m, i, probs[i][3], None, None, y32, ts[i], y16, dt, plan.bn, plan.bn, f"canary {out}")


# ------------------------------------------------------------------------------------ input gradient
# (M, K, Ns): the family's shared input is [M, K]; member i has N_i outputs
DX_FAMILIES = [(4096, 320, (320,) * 3), (1024, 640, (640,) * 4), (77, 768, (768,) * 3),
               (300, 320, (320, 640, 1280, 88))]


@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("M,K,Ns", DX_FAMILIES)
def test_grouped_input_gradient_and_factor_gradients_match_float64(M, K, Ns, dt):
    """The family's dX launch as grouping.py:133-148 builds it, fp32 and 16-bit dX; its dTs and the
    forward's T into ops.wgrad_multi; against O.lora_linear_backward with the bounds of
    test_backward_kernels_match_oracle."""
    ops = _ops()
    mems = make_family(M, K, Ns, dt, seed=M + K + len(Ns), bias=False)
    _, Ts = ops.fused_linear_grouped(problems(mems, dt), dt, True)
    g = torch.Generator().manual_seed(M + len(Ns))
    gys = [torch.randn(M, N, generator=g).to(dt).to(DEV) for N in Ns]
    dprobs = []
    for m, gy in zip(mems, gys):
        N = m.W.shape[0]
        _, wt16 = ops.cast_weight(m.W, dt, False, True)
        dprobs.append((gy, wt16, None, ops.cast_rows_pad16(m.B, 1, m.r, m.r, N, dt), m.A, 1, K, m.diag, m.scale,
                       m.r))
    for out in ("f32", "16"):
        dXs, dTs = ops.fused_linear_grouped(dprobs, F32 if out == "f32" else dt, True)
        torch.cuda.synchronize()
        bn = grouped_plan([(M, N, K) for N in Ns], out, n_sms()).bn
        sum_got = sum_ref = sum_base = sum_model = 0.0
        for i, (m, gy) in enumerate(zip(mems, gys)):
            N, r = m.W.shape[0], m.r
            tag = f"dX {out} member {i} ({M}x{N}->{K} r{r})"
            gy64, W64 = gy.to(F64), m.W.to(F64)
            B16 = dprobs[i][3][:r].to(F64).t()
            check_t(dTs[i], gy64 @ B16, r, N, tag + ": dTs")
            base = gy64 @ W64
            model = base + tprime(dTs[i], r, m.scale, m.diag, dt) @ m.A.to(dt).to(F64)
            check_rel(dXs[i], model, 3e-4 if out == "f32" else ulp16(dt), bn, tag + " vs rounded model")
            rdX = O.lora_linear_backward(gy, m.x, m.W, m.A, B16, m.scale, diag=m.diag, device=DEV)[0]
            if out == "f32":
                check_branch(dXs[i], rdX, base, bn, tag + " vs oracle")
                fdX = O.lora_linear_backward(gy, m.x, m.W, m.A, m.B, m.scale, diag=m.diag, device=DEV)[0]
                assert KG.rel_err(dXs[i], fdX) < 1e-2, tag
            sum_got, sum_ref = sum_got + dXs[i].to(F64), sum_ref + rdX
            sum_base, sum_model = sum_base + base, sum_model + model
        check_rel(sum_got, sum_model, 3e-4 if out == "f32" else ulp16(dt), bn, f"sum of dX {out} vs rounded model")
        if out == "f32":
            check_branch(sum_got, sum_ref, sum_base, bn, "sum of dX vs oracle")
            dAs = [torch.zeros(m.r, K, device=DEV) for m in mems]
            dBs = [torch.zeros(m.W.shape[0], m.r, device=DEV) for m in mems]
            ops.wgrad_multi(mems[0].x, [(dTs[i], dAs[i], gys[i], Ts[i], dBs[i], m.diag, m.scale, m.r)
                                        for i, m in enumerate(mems)])
            torch.cuda.synchronize()
            for i, (m, gy) in enumerate(zip(mems, gys)):
                r = m.r
                B16 = dprobs[i][3][:r].to(F64).t()
                A16 = ops.cast_rows_pad16(m.A, K, 1, r, K, dt)[:r].to(F64)
                _, rdA, _ = O.lora_linear_backward(gy, m.x, m.W, m.A, B16, m.scale, diag=m.diag, device=DEV)
                _, _, rdB = O.lora_linear_backward(gy, m.x, m.W, A16, m.B, m.scale, diag=m.diag, device=DEV)
                assert KG.rel_err(dAs[i], rdA) < 2e-5, f"dA member {i}"
                assert KG.rel_err(dBs[i], rdB) < 2e-5, f"dB member {i}"
                _, fdA, fdB = O.lora_linear_backward(gy, m.x, m.W, m.A, m.B, m.scale, diag=m.diag, device=DEV)
                assert KG.rel_err(dAs[i], fdA) < 1e-2 and KG.rel_err(dBs[i], fdB) < 1e-2, f"member {i}"


# ------------------------------------------------------------------------------------ layouts, fallback
# one family per 16-bit plan at 132 SMs; each also takes one of the two fp32 plans
PLAN_FAMILIES = ["sd15_b1_64x64_qkv", "sd15_b1_32x32_qkv", "sd15_b1_16x16_qkv", "narrow_crowded_640"]


@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("name", PLAN_FAMILIES)
def test_grouped_forward_with_tiled_weights_matches_float64(name, dt):
    """The frozen weights in the 64 x 64-block layout (ops.tile_weight, LB_W_TILED)."""
    _, M, K, Ns, bias = next(f for f in FAMILIES if f[0] == name)
    mems = make_family(M, K, Ns, dt, seed=M + K + sum(Ns) + 1, bias=bias)
    check_family(mems, run_family(mems, dt, tiled=True), dt, name + " tiled")


def test_grouped_plans_of_the_tiled_families_cover_every_plan():
    fams = [f for f in FAMILIES if f[0] in PLAN_FAMILIES]
    assert {grouped_plan([(M, K, N) for N in Ns], out, 132) for (_, M, K, Ns, _) in fams
            for out in ("f32", "16")} == ALL_PLANS


@gpu
@pytest.mark.parametrize("dt", DTS)
def test_grouped_family_with_a_wide_rank_member_launches_per_problem(dt):
    """A rank-24 member (rank pad 32) makes ops.fused_linear_grouped launch each problem on its own."""
    ops = _ops()
    mems = [make_member(256, 1280, 1280, 4, dt, seed=1, scale=0.9, diag=True),
            make_member(256, 1280, 1280, 24, dt, seed=2, scale=-1.4, diag=True)]
    mems[1] = mems[1]._replace(x=mems[0].x)
    probs = problems(mems, dt)
    before = ops.LAUNCH_COUNT
    ops.fused_linear_grouped(probs, F32, True)
    assert ops.LAUNCH_COUNT - before == 2                     # one launch per problem
    res = run_family(mems, dt)
    assert res[2][1].shape == (256, 32)
    d16s, y0s, t0s, y32s, ts, y16s = res
    for i, m in enumerate(mems):
        check_member(m, i, d16s[i], y0s[i], t0s[i], y32s[i], ts[i], y16s[i], dt, 64, 64, "rank 24 fallback")


@gpu
def test_grouped_entry_rejects_bad_arguments():
    """Refused with a status before any launch: n outside 1..4, K % 8, N % 8 with 16-bit output,
    N % 4 with fp32 output, r > 16, a misaligned pointer, an output type that is neither fp32 nor
    the operand type."""
    from lora_b200._C import LB_BF16, LB_F16, LB_F32, LoraB200Error
    dt = BF
    mems = [make_member(128, 64, 96, 4, dt, seed=3, scale=1.0) for _ in range(2)]
    probs = problems(mems, dt)
    ys = [torch.zeros(128, 96, dtype=F32, device=DEV) for _ in mems]
    up17 = torch.zeros(96, 17, device=DEV)

    def call(status, out_code=LB_BF16, in_code=LB_BF16, n=None, **edit):
        c = columns(probs, ys, [None] * len(probs))
        for key, (i, v) in edit.items():
            c[key][i] = v
        if n == 5:
            c = {k: v + [v[0]] * 3 for k, v in c.items()}
        with pytest.raises(LoraB200Error, match=status):
            call_grouped(c, in_code, out_code, n=n)

    call_grouped(columns(probs, ys, [None, None]), LB_BF16, LB_F32)     # the unedited call is accepted
    call("LB_ERR_SHAPE", n=0)
    call("LB_ERR_SHAPE", n=5)
    call("LB_ERR_SHAPE", K=(1, 60))
    call("LB_ERR_SHAPE", N=(1, 92))                           # 16-bit output: N % 8
    call("LB_ERR_SHAPE", out_code=LB_F32, N=(1, 90))          # fp32 output: N % 4
    call("LB_ERR_RANK", R=(1, 17), U=(1, up17.data_ptr()), RS=(1, 17))
    call("LB_ERR_ALIGN", X=(1, mems[1].x.data_ptr() + 2))
    call("LB_ERR_ALIGN", Y=(0, ys[0].data_ptr() + 8))
    call("LB_ERR_DTYPE", out_code=LB_F16)                     # bf16 operands, fp16 output
    call("LB_ERR_DTYPE", in_code=LB_F32, out_code=LB_F32)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------ module level
@gpu
@pytest.mark.parametrize("dt", DTS)
def test_grouped_module_family_with_mixed_rank_scale_and_selector(dt, monkeypatch):
    """q/k/v of one attention patched with ranks 4 / 16 / 1 (monkeypatch_or_replace_lora), each with
    its own scale and selector, run grouped under autocast: forward, input gradient and factor
    gradients against the float64 oracle."""
    import lora_b200 as L
    from lora_b200 import ops

    class Attention(nn.Module):
        def __init__(self):
            super().__init__()
            self.to_q = nn.Linear(640, 640, bias=True)
            self.to_k = nn.Linear(640, 640, bias=False)
            self.to_v = nn.Linear(640, 640, bias=True)

    torch.manual_seed(0)
    att = Attention().to(DEV)
    ranks = [4, 16, 1]
    g = torch.Generator().manual_seed(4)
    loras = []
    for r in ranks:
        # small up factors: the branch stays below the frozen output, so that a lost bias (0.02 RMS per
        # element) stands far above the branch term of the bound
        loras += [torch.randn(640, r, generator=g) * 0.005, torch.randn(r, 640, generator=g) / r]
    L.monkeypatch_or_replace_lora(att, loras, target_replace_module={"Attention"}, r=list(ranks))
    sites = [att.to_q, att.to_k, att.to_v]
    assert [type(m).__name__ for m in sites] == ["LoraInjectedLinear"] * 3 and [m.r for m in sites] == ranks
    att.requires_grad_(False)
    for m in sites:
        m.lora_down.weight.requires_grad_(True)
        m.lora_up.weight.requires_grad_(True)
    for m, s in zip(sites, (0.6, -1.2, 1.7)):
        m.scale = s
    att.to_k.set_selector_from_diag(torch.rand(16, generator=g) + 0.5)
    att.to_v.set_selector_from_diag(torch.tensor([1.3]))
    att.eval()                                          # dropout sites are never grouped
    launched = []
    real = ops.fused_linear_grouped

    def spy(probs, out_dtype, want_t):
        launched.append(len(probs))
        return real(probs, out_dtype, want_t)

    monkeypatch.setattr(ops, "fused_linear_grouped", spy)
    x = torch.randn(2, 300, 640, device=DEV, requires_grad=True)
    gys = [torch.randn(2, 300, 640, device=DEV).to(dt) for _ in sites]
    L.set_grouping(True)
    try:
        with torch.autocast("cuda", dtype=dt):
            for m in sites:                             # learning pass: the three sites share x
                m(x)
            assert launched == []
            ys = [m(x) for m in sites]
        torch.autograd.backward(ys, gys)
        torch.cuda.synchronize()
    finally:
        L.set_grouping(False)
    assert launched == [3, 3], launched                 # one forward and one dX launch for the family
    x16 = x.detach().reshape(600, 640).to(dt)
    dx_ref = dx_base = 0.0
    for i, (m, y, gy) in enumerate(zip(sites, ys, gys)):
        assert y.dtype == dt
        W16 = m.linear.weight.detach().to(dt)
        diag = m._selector_diag()
        A, B = m.lora_down.weight.detach(), m.lora_up.weight.detach()
        base = O.lora_linear_forward(x16, W16, m.linear.bias, A, torch.zeros_like(B), 0.0, device=DEV)
        ref = O.lora_linear_forward(x16, W16, m.linear.bias, A, B, m.scale, diag=diag, device=DEV)
        err = float((y.detach().reshape(600, 640).to(F64) - ref).norm())
        bound = 2.0 ** -7 * float((ref - base).norm()) + ulp16(dt) * float(ref.norm())
        assert err <= bound, f"site {i} forward: err {err:.3e} > {bound:.3e}"
        gy2 = gy.reshape(600, 640)
        A16, B16 = A.to(dt).float(), B.to(dt).float()
        rdX, rdA, _ = O.lora_linear_backward(gy2, x16, W16, A, B16, m.scale, diag=diag, device=DEV)
        _, _, rdB = O.lora_linear_backward(gy2, x16, W16, A16, B, m.scale, diag=diag, device=DEV)
        assert KG.rel_err(m.lora_down.weight.grad, rdA) < 2e-5, f"site {i} dA"
        assert KG.rel_err(m.lora_up.weight.grad, rdB) < 2e-5, f"site {i} dB"
        dx_ref, dx_base = dx_ref + rdX, dx_base + gy2.to(F64) @ W16.to(F64)
    bn = grouped_plan([(600, 640, 640)] * 3, "f32", n_sms()).bn
    check_branch(x.grad.reshape(600, 640), dx_ref, dx_base, bn, "summed input gradient")
