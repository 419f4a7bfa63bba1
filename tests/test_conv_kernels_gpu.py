"""Kernel-level parity of the fused LoRA conv (lb_lora_conv2d_fwd / _dropout, csrc/fused_core.cuh CONV)
and of its factor-gradient reductions (lb_lora_wgrad_conv, lb_lora_wgrad) against float64 references:
oracle/lora_ops.py and plain float64 F.conv2d / conv2d_input / conv2d_weight, evaluated on the GPU.

The kernels are called as the autograd glue calls them (conv_path.py forward and backward, with and
without dropout), at every SD1.5 512-px conv site and at ragged shapes. The census is chosen so that
it reaches every launch branch of conv2d_fwd_impl; `conv_plan` restates that selection and an
unmarked CPU test checks the coverage.

Every bound is checked on the whole tensor AND separately on two pixel regions -- the border ring
(pixels within 1 of an image edge: the TMA zero-fill halo) and the last tile row and column (the
ragged tiles) -- so that a local error cannot hide in a Frobenius norm over the whole image.

Tolerances:
  * frozen conv (scale = 0, fp32 output), the T side output, the input gradient of the frozen conv:
    16-bit operands are exact in fp32 products, only the fp32 accumulation differs from float64 ->
    rel < max(1e-5, K/16 * 2^-24), K = taps * channels reduced. The second term: the H100 tensor
    core adds each 16-deep K-step into the fp32 accumulator with truncation rather than
    round-to-nearest, so the error is a bias that grows linearly with the number of K-steps instead
    of cancelling (measured on H100 SXM at 700 W: rel ~1.1e-9 * K, 1.9e-5 at K = 9 * 1920); the bound
    allows half an fp32 ulp per K-step and is 1e-5 up to K = 2684.
  * full output against a model with the kernel's declared roundings (A and B as 16-bit copies, the
    scaled rank-r activations T' = 16-bit(fp32(T * scale * diag)) formed from the kernel's own fp32 T,
    as the drain forms them): fp32 output < 3e-4 (test_kernels_gpu.py's bound for the same model),
    16-bit output < one 16-bit ulp (2^-8 bf16, 2^-11 fp16).
  * against the unrounded oracle: err <= 2^-7 * ||LoRA branch|| + 1e-5 * ||ref|| (the linear
    suite's rule, test_kernels_gpu.py).
  * factor gradients fed the kernels' own T: S is 16-bit data and V fp32, so only the fp32
    accumulation order differs -> rel < 2e-5.
  * dropout: the exact keep-mask (oracle/dropmask.py) goes into the oracle; the bounds above apply.
"""
import ctypes
import math
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F
from torch.nn import grad as G

from oracle import dropmask as DM
from oracle import lora_ops as O

DEV = "cuda"
F64 = torch.float64
gpu = pytest.mark.gpu


def rank_pad(r):
    return 16 if r <= 16 else (32 if r <= 32 else 64)


# ------------------------------------------------------------------------------------ launch plan
Plan = namedtuple("Plan", "bn split G form narrow")


def plan_conv_split(m_tiles, num_kb, N, g, n_sms):
    """Restates plan_conv_split, lora_b200/csrc/fused_conv.cu:47-66."""
    bn = 64
    tiles = m_tiles * ((N + bn - 1) // bn)
    per_kb = (128.0 + bn + 16.0) * 128.0 / 92e3
    base_t = ((tiles + n_sms - 1) // n_sms) * (2.0 + num_kb * per_kb)
    best, best_t = 1, 1e30
    for sp in range(2, 9):
        if tiles * sp > n_sms or num_kb // sp < 4:
            break
        t = 2.0 + ((num_kb + sp - 1) // sp) * per_kb + 3.0 + (2.0 if g > 1 else 0.0)
        if t < best_t:
            best_t, best = t, sp
    return best if best > 1 and best_t < 0.75 * base_t else 1


def conv_plan(n_img, H, W, Cin, Cout, k, r_pad, per_tap, drop, n_sms, t_in=False):
    """Which kernel conv2d_fwd_impl launches (lora_b200/csrc/fused_conv.cu:68-91 and 141-188):
    tile width bn (64 / 128), split-K factor, T groups G (9 = per-tap T of the 3x3 input gradient) and
    form: "fwd" (T rides the main loop), "drop" (masked drain), "tap_in" (rank pad > 16 tap loop reading
    T_in), "tap_pre" (tap loop after the T pre-pass, launch_t_from16)."""
    taps = k * k
    TW = 16 if W >= 16 else 8
    TH = 128 // TW
    m_tiles = n_img * (-(-H // TH)) * (-(-W // TW))
    groups = per_tap and taps > 1
    narrow = m_tiles * (-(-Cout // 64)) <= n_sms
    bn = 64 if narrow else 128
    if r_pad > 16:
        if drop:
            return Plan(64 if narrow or r_pad == 64 else 128, 1, 1, "drop", narrow)
        if groups:
            return Plan(bn, 1, taps, "tap_in" if t_in else "tap_pre", narrow)
        return Plan(bn, 1, 1, "fwd", narrow)
    split = plan_conv_split(m_tiles, taps * (-(-Cin // 64)), Cout, taps if groups else 1, n_sms)
    return Plan(64 if split > 1 else bn, split, 1 if drop or not groups else taps, "drop" if drop else "fwd",
                narrow)


BF, FP = torch.bfloat16, torch.float16
# (n_img, H, W, Cin, Cout, k, r, dtype)
SD15 = [
    (1, 64, 64, 320, 320, 3, 4, BF), (1, 64, 64, 960, 320, 3, 8, FP), (1, 64, 64, 640, 320, 3, 16, BF),
    (1, 32, 32, 320, 640, 3, 4, FP), (1, 32, 32, 640, 640, 3, 1, BF), (1, 32, 32, 1920, 640, 3, 8, BF),
    (1, 32, 32, 1280, 640, 3, 3, FP), (1, 32, 32, 960, 640, 3, 16, FP),
    (1, 16, 16, 640, 1280, 3, 4, BF), (1, 16, 16, 1280, 1280, 3, 8, FP), (1, 16, 16, 2560, 1280, 3, 16, BF),
    (1, 16, 16, 1920, 1280, 3, 3, BF), (1, 8, 8, 1280, 1280, 3, 4, FP), (1, 8, 8, 2560, 1280, 3, 8, BF),
    (1, 64, 64, 960, 320, 1, 4, BF), (1, 64, 64, 640, 320, 1, 8, FP), (1, 32, 32, 320, 640, 1, 4, BF),
    (1, 32, 32, 1920, 640, 1, 16, FP), (1, 16, 16, 2560, 1280, 1, 4, FP), (1, 8, 8, 2560, 1280, 1, 8, BF),
    # wide ranks at SD1.5 sites: 128-wide (64 x 64 pixels) and 64-wide tiles at pads 32 and 64
    (1, 64, 64, 320, 320, 3, 32, BF), (1, 32, 32, 640, 640, 3, 17, FP),
    (1, 64, 64, 320, 320, 3, 64, FP), (1, 16, 16, 1280, 1280, 3, 33, BF),
]
# ragged: W in {3, 7, 9, 15, 17, 33} (TW 8 and 16, partial last tiles), H not a multiple of TH,
# Cin / Cout not multiples of BLOCK_K / the store box
RAGGED = [
    (2, 12, 7, 24, 40, 3, 3, BF), (3, 5, 3, 8, 8, 3, 1, FP), (1, 9, 9, 72, 88, 3, 16, BF),
    (2, 15, 15, 136, 200, 3, 17, FP), (1, 17, 17, 24, 88, 3, 32, BF), (3, 33, 33, 72, 200, 3, 33, FP),
    (2, 7, 9, 136, 40, 1, 64, BF), (1, 13, 33, 136, 8, 3, 64, BF), (3, 5, 17, 72, 8, 1, 16, FP),
    (2, 11, 3, 8, 200, 3, 16, BF),
]
CENSUS = SD15 + RAGGED
# (n_img, H, W, Cin, Cout, k, r, dtype, p): dropout on the branch, forward and backward
DROP_CASES = [
    (1, 64, 64, 320, 320, 3, 4, BF, 0.25),     # 128-wide masked drain
    (1, 32, 32, 640, 640, 3, 8, FP, 0.1),      # 64-wide
    (1, 8, 8, 1280, 1280, 3, 16, BF, 0.25),    # split-K with the masked drain
    (3, 33, 33, 72, 200, 3, 64, BF, 0.25),     # rank pad 64, fp32 output: forced 64 wide
    (2, 12, 7, 24, 40, 3, 24, FP, 0.5),        # rank pad 32, ragged
    (1, 9, 15, 136, 88, 1, 3, FP, 0.2),        # 1x1, ragged
]
OUTS = ("f32", "16")


def census_plans(n_sms):
    """Launch branches the census reaches: {(rank pad, bn, split > 1, G, form, output)}."""
    seen = set()
    for (n, H, W, cin, cout, k, r, _) in CENSUS:
        rp = rank_pad(r)
        for out in OUTS:
            p = conv_plan(n, H, W, cin, cout, k, rp, False, False, n_sms)
            seen.add((rp, p.bn, p.split > 1, p.G, p.form, out))
            for t_in in ((False, True) if rp > 16 and k == 3 else (False,)):
                p = conv_plan(n, H, W, cout, cin, k, rp, True, False, n_sms, t_in=t_in)
                seen.add((rp, p.bn, p.split > 1, p.G, p.form, out))
    for (n, H, W, cin, cout, k, r, _, _) in DROP_CASES:
        rp = rank_pad(r)
        for out in OUTS:
            p = conv_plan(n, H, W, cin, cout, k, rp, False, True, n_sms)
            seen.add((rp, p.bn, p.split > 1, p.G, p.form, out))
            if rp == 64 and out == "f32" and not p.narrow:
                seen.add("rp64 drop fp32 forced 64")
        p = conv_plan(n, H, W, cout, cin, k, rp, True, False, n_sms, t_in=True)
        seen.add((rp, p.bn, p.split > 1, p.G, p.form, "f32"))
    return seen


def required_plans():
    req = set()
    for out in OUTS:
        for G_ in (1, 9):
            req |= {(16, 64, False, G_, "fwd", out), (16, 128, False, G_, "fwd", out), (16, 64, True, G_, "fwd", out)}
        req |= {(16, 64, False, 1, "drop", out), (16, 128, False, 1, "drop", out), (16, 64, True, 1, "drop", out)}
        for rp in (32, 64):
            for bn in (64, 128):
                req |= {(rp, bn, False, 1, "fwd", out), (rp, bn, False, 9, "tap_in", out),
                        (rp, bn, False, 9, "tap_pre", out)}
    req.add((64, 64, False, 1, "drop", "f32"))
    req.add("rp64 drop fp32 forced 64")
    return req


def test_census_reaches_every_conv_launch_branch():
    """CPU: at 132 SMs (H100 SXM) the census reaches every launch branch of conv2d_fwd_impl."""
    missing = required_plans() - census_plans(132)
    assert not missing, sorted(map(str, missing))


@gpu
def test_census_reaches_every_conv_launch_branch_on_this_device():
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    missing = required_plans() - census_plans(n_sms)
    assert not missing, (n_sms, sorted(map(str, missing)))


# ------------------------------------------------------------------------------------ helpers
def _ops():
    from lora_b200 import ops
    return ops


def rel(a, b):
    a, b = a.detach().to(DEV, F64), b.detach().to(DEV, F64)
    return float((a - b).norm() / (b.norm() + 1e-30))


def regions(H, W):
    """(name, [H, W] bool mask): whole image, border ring, last tile row + column (TW/TH as the kernel)."""
    TW = 16 if W >= 16 else 8
    TH = 128 // TW
    h = torch.arange(H, device=DEV).view(H, 1)
    w = torch.arange(W, device=DEV).view(1, W)
    ring = (h <= 0) | (h >= H - 1) | (w <= 0) | (w >= W - 1)
    last = (h >= ((H - 1) // TH) * TH) | (w >= ((W - 1) // TW) * TW)
    return [("all", torch.ones(H, W, dtype=torch.bool, device=DEV)), ("ring", ring), ("last tile", last)]


def check_rel(got, ref, tol, what):
    """got / ref: [n, C, H, W]; rel error below tol on every region."""
    got, ref = got.detach().to(DEV, F64), ref.detach().to(DEV, F64)
    for name, m in regions(ref.shape[2], ref.shape[3]):
        e = rel(got[..., m], ref[..., m])
        assert e < tol, f"{what} [{name}]: rel {e:.3e} >= {tol:.1e}"


def check_branch(got, ref, base, what):
    """err <= 2^-7 ||ref - base|| + 1e-5 ||ref|| on every region (base: the frozen conv + bias)."""
    got, ref, base = (t.detach().to(DEV, F64) for t in (got, ref, base))
    for name, m in regions(ref.shape[2], ref.shape[3]):
        g, r_, b_ = got[..., m], ref[..., m], base[..., m]
        err, bound = float((g - r_).norm()), 2.0 ** -7 * float((r_ - b_).norm()) + 1e-5 * float(r_.norm())
        assert err <= bound, f"{what} [{name}]: err {err:.3e} > {bound:.3e}"


def rows_to_nchw(t, n, H, W):
    """[n*H*W, c] pixel rows (NHWC order) -> [n, c, H, W]."""
    return t.reshape(n, H, W, -1).permute(0, 3, 1, 2)


def nchw_to_rows(t):
    n, c, H, W = t.shape
    return t.permute(0, 2, 3, 1).reshape(n * H * W, c)


def acc_tol(K):
    """Bound for a tensor-core reduction over K (module docstring)."""
    return max(1e-5, K / 16 * 2.0 ** -24)


def tprime(T, r, scale, diag, dt, n, H, W):
    """T' as the drain forms it: fp32 T * fp32(scale * diag), rounded to the 16-bit operand type."""
    coef = torch.full((r,), scale, dtype=torch.float32, device=DEV)
    if diag is not None:
        coef = coef * diag.float()
    return rows_to_nchw((T[:, :r] * coef).to(dt).to(F64), n, H, W)


def ulp16(dt):
    return 2.0 ** -8 if dt == BF else 2.0 ** -11


def make_conv(n, H, W, cin, cout, k, r, dt, seed):
    g = torch.Generator().manual_seed(seed)
    fan = cin * k * k
    x = torch.randn(n, cin, H, W, generator=g).to(dt)
    Wt = (torch.randn(cout, cin, k, k, generator=g) / math.sqrt(fan)).to(dt)
    A = torch.randn(r, cin, k, k, generator=g) / math.sqrt(fan)
    B = torch.randn(cout, r, generator=g) / math.sqrt(r)
    bias = torch.randn(cout, generator=g) * 0.1
    diag = torch.rand(r, generator=g) + 0.5 if r % 2 == 0 else None
    gy = torch.randn(n, cout, H, W, generator=g).to(dt)
    cl = torch.channels_last
    return (x.to(DEV).contiguous(memory_format=cl), Wt.to(DEV), A.to(DEV), B.to(DEV), bias.to(DEV),
            None if diag is None else diag.to(DEV), gy.to(DEV).contiguous(memory_format=cl))


class Guarded:
    """A tensor view placed inside a larger buffer of 0xFF bytes (NaN in fp32, bf16 and fp16) with
    256-byte guards on both sides: every in-bounds element must be written, no guard byte touched."""
    GUARD = 256

    def __init__(self, shape, dtype):
        esz = torch.empty((), dtype=dtype).element_size()
        self.nbytes = math.prod(shape) * esz
        self.buf = torch.full((self.nbytes + 2 * self.GUARD,), 0xFF, dtype=torch.uint8, device=DEV)
        self.t = self.buf[self.GUARD:self.GUARD + self.nbytes].view(dtype).view(shape)

    def check(self, what):
        g = self.GUARD
        assert bool((self.buf[:g] == 0xFF).all()) and bool((self.buf[g + self.nbytes:] == 0xFF).all()), \
            f"{what}: a guard byte was written"
        assert not bool(torch.isnan(self.t.float()).any()), f"{what}: in-bounds elements left unwritten"


def conv_call(x, w16, bias, down16, up, up_off, up_rs, up_cs, up_gs, diag, scale, r, cout, k, per_tap,
              out_dtype, want_t, t_in=None, guarded=False):
    """ops.fused_conv2d, or (guarded) lb_lora_conv2d_fwd straight into guarded Y / T_out buffers.
    Returns (Y [n, cout, H, W], T rows or None, list of Guarded)."""
    ops = _ops()
    pad = k // 2
    if not guarded:
        y, t = ops.fused_conv2d(x, w16, bias, down16, up, up_off, up_rs, up_cs, up_gs, diag, scale, r, cout, k, k,
                                pad, pad, per_tap, out_dtype, want_t, t_in=t_in)
        return y, t, []
    from lora_b200 import _C
    from lora_b200._C import check, dtype_code, ptr, stream_ptr
    n, cin, H, W = x.shape
    rp = down16.shape[0]
    gy_ = Guarded((n, H, W, cout), out_dtype)
    gt = Guarded((n * H * W, rp), torch.float32) if want_t else None
    check(_C.lib.lb_lora_conv2d_fwd(ptr(x), ptr(w16), ptr(bias), ptr(down16),
                                    ctypes.c_void_p(up.data_ptr() + 4 * up_off), up_rs, up_cs, up_gs, ptr(diag),
                                    float(scale), ptr(gy_.t), None if gt is None else ptr(gt.t), ptr(t_in), n, H, W,
                                    cin, cout, k, k, pad, pad, r, rp, 1 if per_tap else 0, dtype_code(x.dtype),
                                    dtype_code(out_dtype), stream_ptr()), "lb_lora_conv2d_fwd")
    return gy_.t.permute(0, 3, 1, 2), None if gt is None else gt.t, [gy_] + ([gt] if gt else [])


def check_t_rows(t, t_ref, r, tol, what):
    """T side output: rel < tol on every region, each element close (a row written by an out-of-image
    tile pixel would be off by O(1)), padded rank columns exactly zero."""
    n, c, H, W = t_ref.shape
    check_rel(rows_to_nchw(t[:, :r], n, H, W), t_ref, tol, what)
    tr = nchw_to_rows(t_ref)
    assert bool((t[:, :r].double() - tr).abs().le(1e-3 * float(tr.abs().max())).all()), f"{what}: element off"
    assert torch.count_nonzero(t[:, r:]) == 0, f"{what}: padded rank columns written"


# ------------------------------------------------------------------------------------ census
@gpu
@pytest.mark.parametrize("case", CENSUS, ids=lambda c: "n{}_{}x{}_{}to{}_k{}_r{}_{}".format(*c[:7], str(c[7])[6:]))
def test_conv_kernels_match_float64(case):
    ops = _ops()
    n, H, W, cin, cout, k, r, dt = case
    ragged = case in RAGGED
    pad, taps, rp = k // 2, k * k, rank_pad(r)
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    scale = 0.7
    x, Wt, A, B, bias, diag, gy = make_conv(n, H, W, cin, cout, k, r, dt, seed=sum(case[:7]))
    x64, W64, gy64 = x.to(F64), Wt.to(F64), gy.to(F64)
    dd = (torch.ones(r, device=DEV) if diag is None else diag).to(F64)
    wf, wb = ops.cast_conv_weight(Wt, dt, True, True)
    d16 = ops.conv_down16(A, dt, {})
    A16 = d16[:r].view(r, k, k, cin).permute(0, 3, 1, 2).to(F64)
    upT16 = ops.cast_rows_pad16(B, 1, r, r, cout, dt)          # B^T, 16-bit [rp, cout]
    B16 = upT16[:r].t().to(F64)
    odts = {"f32": torch.float32, "16": dt}

    base = F.conv2d(x64, W64, bias.to(F64), padding=pad)
    t_ref = F.conv2d(x64, A16, padding=pad)                   # conv(x, A16): the kernel's T
    ref = O.lora_conv2d_forward(x, Wt, bias, A, B, scale, padding=pad, diag=diag, device=DEV)
    ref_base = O.lora_conv2d_forward(x, Wt, bias, A, torch.zeros_like(B), 0.0, padding=pad, device=DEV)

    def fwd(scale_, out, want_t):
        return conv_call(x, wf, bias, d16, B, 0, r, 1, 0, diag, scale_, r, cout, k, False, odts[out], want_t,
                         guarded=ragged)

    reps = 3 if conv_plan(n, H, W, cin, cout, k, rp, False, False, n_sms).split > 1 else 1
    # (a) frozen conv
    y0, _, gs = fwd(0.0, "f32", False)
    check_rel(y0, base, acc_tol(taps * cin), "frozen conv")
    for rep in range(reps):                                    # split-K: the same ring / counters again
        # (b) T side output, (c) full output
        y32, T, gs32 = fwd(scale, "f32", True)
        y16, _, gs16 = fwd(scale, "16", False)
        torch.cuda.synchronize()
        for gd in gs + gs32 + gs16:
            gd.check(f"forward rep {rep}")
        check_t_rows(T, t_ref, r, acc_tol(taps * cin), f"forward T rep {rep}")
        y_model = base + torch.einsum("njhw,oj->nohw", tprime(T, r, scale, diag, dt, n, H, W), B16)
        check_rel(y32, y_model, 3e-4, f"forward fp32 vs rounded model rep {rep}")
        check_rel(y16, y_model, ulp16(dt), f"forward 16-bit vs rounded model rep {rep}")
        check_branch(y32, ref, ref_base, f"forward vs oracle rep {rep}")

    # (d) input gradient: conv_T(gY, W) + conv_T((gY.B16) s d, A16) on the flipped weight, A read flipped
    dx_base = G.conv2d_input(x.shape, W64, gy64, padding=pad)
    dts_ref = torch.einsum("nohw,oj->njhw", gy64, B16)        # gY . B16, per pixel
    dx_ref = O.lora_conv2d_backward(gy, x, Wt, A, B16, scale, padding=pad, diag=diag, device=DEV)[0]

    def dgrad(scale_, out, want_t, t_in=None):
        return conv_call(gy, wb, None, upT16, A, taps - 1, taps, cin * taps, -1, diag, scale_, r, cin, k, True,
                         odts[out], want_t, t_in=t_in, guarded=ragged)

    tap_loop = rp > 16 and k == 3
    dreps = 3 if conv_plan(n, H, W, cout, cin, k, rp, True, False, n_sms).split > 1 else 1
    d0, _, gs = dgrad(0.0, "f32", False, t_in=torch.zeros(n * H * W, rp, device=DEV) if tap_loop else None)
    torch.cuda.synchronize()
    for gd in gs:
        gd.check("frozen input gradient")
    check_rel(d0, dx_base, acc_tol(taps * cout), "frozen input gradient")
    dTs = None
    for rep in range(dreps):
        for out in OUTS:
            dx, dT, gs = dgrad(scale, out, True)
            torch.cuda.synchronize()
            for gd in gs:
                gd.check(f"input gradient {out} rep {rep}")
            check_t_rows(dT, dts_ref, r, acc_tol(cout), f"input-gradient T ({out}) rep {rep}")
            # the per-tap T are the same reduction as T_out at the tap-shifted pixel
            dx_model = dx_base + G.conv2d_input(x.shape, A16, tprime(dT, r, scale, diag, dt, n, H, W), padding=pad)
            forms = [(dx, "T pre-pass" if tap_loop else "")]
            if tap_loop:          # the tap loop reading T_in (the dropout backward's form)
                forms.append((dgrad(scale, out, False, t_in=dT)[0], "T_in"))
            for d, form in forms:
                what = f"input gradient {form} {out} rep {rep}"
                check_rel(d, dx_model, 3e-4 if out == "f32" else ulp16(dt), what + " vs rounded model")
                if out == "f32":
                    check_branch(d, dx_ref, dx_base, what + " vs oracle")
            if out == "f32":
                dTs = dT

    # (e) factor gradients, fed the kernels' own T
    dA = torch.zeros(r, cin * taps, device=DEV)
    ops.wgrad_conv(x, dTs, diag, scale, dA, r, cin, H, W, k, k, pad, pad)
    dB = torch.zeros(cout, r, device=DEV)
    ops.wgrad(nchw_to_rows(gy), T, diag, scale, dB, 1, r, r)
    torch.cuda.synchronize()
    sd = (scale * dd).view(1, r, 1, 1)
    dA_ref = G.conv2d_weight(x64, (r, cin, k, k), rows_to_nchw(dTs[:, :r].to(F64), n, H, W) * sd, padding=pad)
    assert rel(dA.view(r, cin, k, k), dA_ref) < 2e-5
    dB_ref = torch.einsum("nohw,njhw->oj", gy64, rows_to_nchw(T[:, :r].to(F64), n, H, W) * sd)
    assert rel(dB, dB_ref) < 2e-5


# ------------------------------------------------------------------------------------ split-K ring
RING_BYTES, RING_COUNTERS = 96 << 20, 1 << 16        # the split workspace, lora_b200/csrc/tmap.h:106-107


def _split_launch_footprint(n, H, W, cin, cout, k, per_tap, n_sms):
    """(bytes, counters) one split launch takes from the ring: tiles * 128 * (64 + 16 G) * 4 bytes
    (rounded up to 256, tmap.h split_ws_reserve) and one counter per tile (fused_conv.cu:23-26)."""
    N_, K_ = (cin, cout) if per_tap else (cout, cin)
    p = conv_plan(n, H, W, K_, N_, k, 16, per_tap, False, n_sms)
    assert p.split > 1, "not a split plan on this device"
    TW = 16 if W >= 16 else 8
    tiles = n * (-(-H // (128 // TW))) * (-(-W // TW)) * (-(-N_ // 64))
    return (tiles * 128 * (64 + 16 * p.G) * 4 + 255) // 256 * 256, tiles


@gpu
def test_split_workspace_ring_wraps_twice_without_stale_partials():
    """A G = 9 input-gradient split on a ragged 12 x 12 image interleaved with a forward split of
    another shape, for as many launches as make the workspace ring (bytes and counters) wrap twice:
    a partial or counter left behind by an earlier launch only shows once a launch is handed a region
    that an earlier one used."""
    ops = _ops()
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    dt, scale = BF, 0.9
    shapes = [(1, 12, 12, 1280, 1280, 3, True), (1, 8, 8, 1280, 1280, 3, False)]
    runs = []
    for (n, H, W, cin, cout, k, per_tap) in shapes:
        r = 8
        x, Wt, A, B, bias, diag, gy = make_conv(n, H, W, cin, cout, k, r, dt, seed=H + cin)
        wf, wb = ops.cast_conv_weight(Wt, dt, True, True)
        if per_tap:         # input gradient: gY [n, cout, H, W] -> dX [n, cin, H, W]
            upT16 = ops.cast_rows_pad16(B, 1, r, r, cout, dt)
            B16 = upT16[:r].t().to(F64)
            dd = diag.to(F64)
            dts = torch.einsum("nohw,oj->njhw", gy.to(F64), B16) * (scale * dd).view(1, r, 1, 1)
            base = G.conv2d_input(x.shape, Wt.to(F64), gy.to(F64), padding=1)
            ref = base + G.conv2d_input(x.shape, A.to(F64), dts, padding=1)
            call = (lambda gy=gy, wb=wb, upT16=upT16, A=A, diag=diag, cin=cin:
                    ops.fused_conv2d(gy, wb, None, upT16, A, 8, 9, cin * 9, -1, diag, scale, 8, cin, 3, 3, 1, 1,
                                     True, torch.float32, False)[0])
        else:
            d16 = ops.conv_down16(A, dt, {})
            ref = O.lora_conv2d_forward(x, Wt, bias, A, B, scale, padding=1, diag=diag, device=DEV)
            base = O.lora_conv2d_forward(x, Wt, bias, A, torch.zeros_like(B), 0.0, padding=1, device=DEV)
            call = (lambda x=x, wf=wf, bias=bias, d16=d16, B=B, diag=diag, cout=cout:
                    ops.fused_conv2d(x, wf, bias, d16, B, 0, 8, 1, 0, diag, scale, 8, cout, 3, 3, 1, 1, False,
                                     torch.float32, False)[0])
        bound = 2.0 ** -7 * float((ref - base).norm()) + 1e-5 * float(ref.norm())
        runs.append((call, ref, bound, _split_launch_footprint(n, H, W, cin, cout, k, per_tap, n_sms)))
    pair_bytes = sum(f[0] for (_, _, _, f) in runs)
    pair_counters = sum(f[1] for (_, _, _, f) in runs)
    pairs = math.ceil(2 * max(RING_BYTES / pair_bytes, RING_COUNTERS / pair_counters)) + 1
    errs = torch.empty(pairs, len(runs), dtype=F64, device=DEV)
    for i in range(pairs):
        for j, (call, ref, _, _) in enumerate(runs):
            errs[i, j] = (call().to(F64) - ref).norm()
    torch.cuda.synchronize()
    for j, (_, _, bound, _) in enumerate(runs):
        bad = (errs[:, j] > bound).nonzero().flatten()
        assert bad.numel() == 0, f"shape {shapes[j]}: launches {bad[:8].tolist()} of {pairs} off ({errs[bad[0], j]:.3e} > {bound:.3e})"


@gpu
def test_conv_split_plan_inside_a_cuda_graph():
    """8 x 8 mid-block conv (split-K on 132 SMs), captured once and replayed 3 times."""
    ops = _ops()
    dt, r, scale = BF, 4, 1.1
    x, Wt, A, B, bias, diag, _ = make_conv(1, 8, 8, 1280, 1280, 3, r, dt, seed=5)
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert conv_plan(1, 8, 8, 1280, 1280, 3, 16, False, False, n_sms).split > 1
    wf, _ = ops.cast_conv_weight(Wt, dt, True, False)
    d16 = ops.conv_down16(A, dt, {})
    ref = O.lora_conv2d_forward(x, Wt, bias, A, B, scale, padding=1, diag=diag, device=DEV)
    base = O.lora_conv2d_forward(x, Wt, bias, A, torch.zeros_like(B), 0.0, padding=1, device=DEV)

    def call():
        return ops.fused_conv2d(x, wf, bias, d16, B, 0, r, 1, 0, diag, scale, r, 1280, 3, 3, 1, 1, False,
                                torch.float32, True)

    call()                                     # allocates the split workspace outside the capture
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y, T = call()
    for rep in range(3):
        y.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        check_branch(y, ref, base, f"graph replay {rep}")


# ------------------------------------------------------------------------------------ dropout, exact
@gpu
@pytest.mark.parametrize("case", DROP_CASES, ids=lambda c: "n{}_{}x{}_{}to{}_k{}_r{}_{}_p{}".format(
    *c[:7], str(c[7])[6:], c[8]))
def test_conv_dropout_matches_oracle_with_the_exact_mask(case):
    """Forward (masked drain) and backward (conv_path.py with p > 0: masked dT pass, dX from T_in, dA, masked
    dB) against the oracle fed the mask of oracle/dropmask.py."""
    ops = _ops()
    n, H, W, cin, cout, k, r, dt, p = case
    pad, taps = k // 2, k * k
    scale = 1.25
    x, Wt, A, B, bias, diag, gy = make_conv(n, H, W, cin, cout, k, r, dt, seed=sum(case[:7]) + 1)
    seed = 0x5DEECE66D1234567 + H
    seed_t = torch.tensor([seed], dtype=torch.int64, device=DEV)
    mask = torch.from_numpy(DM.conv_mask(seed, p, n, H, W, cout)).to(DEV, F64)
    wf, wb = ops.cast_conv_weight(Wt, dt, True, True)
    d16 = ops.conv_down16(A, dt, {})
    A16 = d16[:r].view(r, k, k, cin).permute(0, 3, 1, 2).to(F64)
    upT16 = ops.cast_rows_pad16(B, 1, r, r, cout, dt)
    B16 = upT16[:r].t().to(F64)

    # forward
    ref = O.lora_conv2d_forward(x, Wt, bias, A, B, scale, padding=pad, diag=diag, keep_mask=mask, dropout_p=p,
                                device=DEV)
    base = O.lora_conv2d_forward(x, Wt, bias, A, torch.zeros_like(B), 0.0, padding=pad, device=DEV)
    T = None
    for out in (torch.float32, dt):
        y, t = ops.fused_conv2d(x, wf, bias, d16, B, 0, r, 1, 0, diag, scale, r, cout, k, k, pad, pad, False, out,
                                True, drop_p=p, seed=seed_t)
        tq = tprime(t, r, scale, diag, dt, n, H, W)
        model = base + mask * torch.einsum("njhw,oj->nohw", tq, B16) / (1.0 - p)
        check_rel(y, model, 3e-4 if out == torch.float32 else ulp16(dt), f"dropout forward {out} vs rounded model")
        if out == torch.float32:
            check_branch(y, ref, base, "dropout forward vs oracle")
            T = t

    # backward, as conv_path._FusedLoraConv2dFn.backward with p > 0
    gy2d = nchw_to_rows(gy)
    dTs = ops.dropout_dt(gy2d, B, r, 1, p, seed_t, r)
    dts_ref = torch.einsum("nohw,oj->njhw", gy.to(F64) * mask / (1.0 - p), B.to(F64))
    check_rel(rows_to_nchw(dTs[:, :r], n, H, W), dts_ref, 1e-5, "masked dT")
    dX, _ = ops.fused_conv2d(gy, wb, None, upT16, A, taps - 1, taps, cin * taps, -1, diag, scale, r, cin, k, k,
                             pad, pad, True, torch.float32, False, t_in=dTs)
    dA = torch.zeros(r, cin * taps, device=DEV)
    ops.wgrad_conv(x, dTs, diag, scale, dA, r, cin, H, W, k, k, pad, pad)
    dB = torch.zeros(cout, r, device=DEV)
    ops.wgrad_masked(gy2d, T, diag, scale, dB, 1, r, r, p, seed_t)
    torch.cuda.synchronize()
    rdX, rdA, _ = O.lora_conv2d_backward(gy, x, Wt, A, B, scale, padding=pad, diag=diag, keep_mask=mask,
                                         dropout_p=p, device=DEV)
    _, _, rdB = O.lora_conv2d_backward(gy, x, Wt, d16[:r].view(r, k, k, cin).permute(0, 3, 1, 2).float(), B,
                                       scale, padding=pad, diag=diag, keep_mask=mask, dropout_p=p, device=DEV)
    dx_base = G.conv2d_input(x.shape, Wt.to(F64), gy.to(F64), padding=pad)
    dtq = tprime(dTs, r, scale, diag, dt, n, H, W)
    check_rel(dX, dx_base + G.conv2d_input(x.shape, A16, dtq, padding=pad), 3e-4, "dropout dX vs rounded model")
    check_branch(dX, rdX, dx_base, "dropout dX vs oracle")
    assert rel(dA.view(r, cin, k, k), rdA) < 2e-5
    assert rel(dB, rdB.view(cout, r)) < 2e-5


@gpu
@pytest.mark.parametrize("r", [4, 40])
def test_linear_dropout_matches_oracle_with_the_exact_mask(r):
    """The same for a linear site (fused_linear with drop_p; modules._FusedLoraLinearFn with p > 0)."""
    ops = _ops()
    M, K, N, p, scale, dt = 333, 320, 640, 0.25, 1.5, BF
    g = torch.Generator().manual_seed(r)
    x = torch.randn(M, K, generator=g).to(dt).to(DEV)
    Wt = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dt).to(DEV)
    A = (torch.randn(r, K, generator=g) / math.sqrt(K)).to(DEV)
    B = (torch.randn(N, r, generator=g) / math.sqrt(r)).to(DEV)
    bias = (torch.randn(N, generator=g) * 0.1).to(DEV)
    diag = (torch.rand(r, generator=g) + 0.5).to(DEV)
    gy = torch.randn(M, N, generator=g).to(dt).to(DEV)
    seed = 987654321987 + r
    seed_t = torch.tensor([seed], dtype=torch.int64, device=DEV)
    mask = torch.from_numpy(DM.linear_mask(seed, p, M, N)).to(DEV, F64)
    rp = rank_pad(r)
    down16 = ops.cast_rows_pad16(A, K, 1, r, K, dt)
    upT16 = ops.cast_rows_pad16(B, 1, r, r, N, dt)
    _, wt16 = ops.cast_weight(Wt, dt, False, True)
    y, T = ops.fused_linear(x, Wt, bias, down16, B, r, 1, diag, scale, r, torch.float32, True, drop_p=p,
                            seed=seed_t)
    ref = O.lora_linear_forward(x, Wt, bias, A, B, scale, diag=diag, keep_mask=mask, dropout_p=p, device=DEV)
    base = O.lora_linear_forward(x, Wt, bias, A, torch.zeros_like(B), 0.0, device=DEV)
    as4 = lambda t: t.reshape(1, 1, *t.shape)        # [M, N] as a one-pixel-row "image" for the checkers
    check_branch(as4(y), as4(ref), as4(base), "linear dropout forward vs oracle")
    dTs = ops.dropout_dt(gy, B, r, 1, p, seed_t, r)
    assert dTs.shape == (M, rp)
    dX, _ = ops.fused_linear(gy, wt16, None, upT16, A, 1, K, diag, scale, r, torch.float32, False, t_in=dTs)
    dA = torch.zeros(r, K, device=DEV)
    dB = torch.zeros(N, r, device=DEV)
    ops.wgrad(x, dTs, diag, scale, dA, K, 1, r)
    ops.wgrad_masked(gy, T, diag, scale, dB, 1, r, r, p, seed_t)
    torch.cuda.synchronize()
    rdX, rdA, _ = O.lora_linear_backward(gy, x, Wt, A, B, scale, diag=diag, keep_mask=mask, dropout_p=p,
                                         device=DEV)
    _, _, rdB = O.lora_linear_backward(gy, x, Wt, down16[:r].float(), B, scale, diag=diag, keep_mask=mask,
                                       dropout_p=p, device=DEV)
    dx_base = gy.to(F64) @ Wt.to(F64)
    check_branch(as4(dX), as4(rdX), as4(dx_base), "linear dropout dX vs oracle")
    assert rel(dA, rdA) < 2e-5
    assert rel(dB, rdB) < 2e-5
