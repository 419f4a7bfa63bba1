"""The factor-gradient reductions behind every LoRA site's dA / dB (csrc/lora_aux.cu wgrad_kernel) against
float64: lb_lora_wgrad_batch (the captured training step queues every site's dA / dB and flushes them in
ceil(n / 24) launches), lb_lora_wgrad_pair and lb_lora_wgrad_multi.

    out[j * js + c * cs] += scale * diag[j] * sum_m V[m, j] * S'[m, c]
    S' = S (plain rows), S o keep / (1 - p) (masked dB of a dropout site, oracle/dropmask.py),
    conv dA: conv2d_weight of the NHWC rows S against V as the output gradient (all taps, one problem).

One batched launch mixes linear dA and dB, 3x3 and 1x1 conv dA on ragged images, masked dB with
different per-problem seeds, ranks 1 ... 64 at rank pads 16 / 32 / 64 (any pad other than 16 switches
the whole launch to the rank-group kernel), problems whose M differs by more than one 64-row slab (one
with M = 1), C not a multiple of the 128-column block, and a selector diagonal on some problems only.
`out` starts non-zero, so the += semantics is checked; V's padded rank columns hold large values that
must never reach `out`.

Tolerance: S is 16-bit data (or fp32 holding 16-bit data: the fp32-faithful path's fmt = 2) and V is
fp32, so only the fp32 accumulation order differs from float64 -> rel < 1e-5 per problem, on the
increment out - out_before.
"""
import math

import pytest
import torch
from torch.nn import grad as G

from oracle import dropmask as DM

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64


def rank_pad(r):
    return 16 if r <= 16 else (32 if r <= 32 else 64)


def rel(a, b):
    a, b = a.detach().to(DEV, F64), b.detach().to(DEV, F64)
    return float((a - b).norm() / (b.norm() + 1e-30))


# kind, r, geometry, diag, p:
#   ("dA", M, C)            linear lora_down gradient: out [r, C], js = C, cs = 1
#   ("dB", M, C)            linear lora_up gradient:   out [C, r], js = 1, cs = r   (p > 0: masked)
#   ("conv", n, H, W, C, k) conv lora_down gradient:   out [r, C*k*k] = [r, C, k, k]
SPECS = [
    (("dA", 700, 328), 4, True, 0.0),
    (("dB", 700, 136), 4, False, 0.0),
    (("conv", 2, 7, 9, 24, 3), 16, True, 0.0),
    (("conv", 3, 5, 3, 72, 1), 17, False, 0.0),
    (("dB", 1, 40), 1, False, 0.25),            # M = 1, masked
    (("dB", 260, 200), 40, True, 0.1),          # masked, another seed
    (("dA", 64, 1288), 64, False, 0.0),         # one slab, C = 10 * 128 + 8
    (("dB", 129, 88), 16, True, 0.0),
    (("conv", 1, 13, 5, 8, 3), 64, True, 0.0),
    (("dA", 333, 200), 32, False, 0.0),
    (("dB", 515, 48), 17, True, 0.5),
]


def make_problem(spec, idx, s_dtype):
    geom, r, has_diag, p = spec
    rp = rank_pad(r)
    g = torch.Generator().manual_seed(1000 + idx)
    data16 = torch.float16 if s_dtype == torch.float16 else torch.bfloat16
    if geom[0] == "conv":
        _, n, H, W, C, k = geom
        M = n * H * W
    else:
        _, M, C = geom
    S = torch.randn(M, C, generator=g).to(data16).to(s_dtype)     # 16-bit data (fp32: holding 16-bit data)
    V = torch.randn(M, rp, generator=g)
    V[:, r:] = 100.0 * torch.randn(M, rp - r, generator=g)        # padded ranks: must not reach `out`
    diag = torch.rand(r, generator=g) + 0.5 if has_diag else None
    scale = 0.5 + idx * 0.01
    seed = 0x2545F4914F6CDD1D * (idx + 1) % (1 << 62)
    coef = scale * (diag.double() if has_diag else torch.ones(r, dtype=F64))
    Sx = S.double()
    if p > 0:
        Sx = Sx * torch.from_numpy(DM.linear_mask(seed, p, M, C)).double() / (1.0 - p)
    if geom[0] == "conv":
        x = Sx.reshape(n, H, W, C).permute(0, 3, 1, 2)
        gt = V[:, :r].double().reshape(n, H, W, r).permute(0, 3, 1, 2) * coef.view(1, r, 1, 1)
        ref = G.conv2d_weight(x, (r, C, k, k), gt, padding=k // 2).reshape(r, C * k * k)
        out_shape = (r, C * k * k)
    elif geom[0] == "dA":
        ref = coef.view(r, 1) * (V[:, :r].double().T @ Sx)
        out_shape = (r, C)
    else:
        ref = (Sx.T @ V[:, :r].double()) * coef.view(1, r)
        out_shape = (C, r)
    out0 = torch.randn(out_shape, generator=g) * float(ref.std())
    d = dict(geom=geom, r=r, p=p, scale=scale, S=S.to(DEV), V=V.to(DEV), out=out0.to(DEV), out0=out0.clone(),
             diag=None if diag is None else diag.to(DEV), seed=torch.tensor([seed], dtype=torch.int64, device=DEV),
             ref=ref)
    return d


def enqueue(ops, q):
    geom, r = q["geom"], q["r"]
    if geom[0] == "conv":
        _, n, H, W, C, k = geom
        ops.wgrad_conv(q["S"], q["V"], q["diag"], q["scale"], q["out"], r, C, H, W, k, k, k // 2, k // 2,
                       deferrable=True)
    elif geom[0] == "dA":
        ops.wgrad(q["S"], q["V"], q["diag"], q["scale"], q["out"], geom[2], 1, r, deferrable=True)
    elif q["p"] > 0:
        ops.wgrad_masked(q["S"], q["V"], q["diag"], q["scale"], q["out"], 1, r, r, q["p"], q["seed"],
                         deferrable=True)
    else:
        ops.wgrad(q["S"], q["V"], q["diag"], q["scale"], q["out"], 1, r, r, deferrable=True)


@pytest.mark.parametrize("s_dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("n", [1, 24, 25, 49])
def test_wgrad_batch_matches_float64(n, s_dtype):
    from lora_b200 import ops
    probs = [make_problem(SPECS[i % len(SPECS)], i, s_dtype) for i in range(n)]
    ops.wgrad_defer_begin()
    try:
        for q in probs:
            enqueue(ops, q)
    finally:
        launches = ops.wgrad_flush()
    assert launches == math.ceil(n / ops.WG_BATCH)
    torch.cuda.synchronize()
    for i, q in enumerate(probs):
        e = rel(q["out"].double() - q["out0"].to(DEV, F64), q["ref"])
        assert e < 1e-5, f"problem {i} {q['geom']} r={q['r']} p={q['p']}: rel {e:.3e}"


def _pair_case(M, K, N, r, p, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    rp = rank_pad(r)
    x = torch.randn(M, K, generator=g).to(dtype)
    gy = torch.randn(M, N, generator=g).to(dtype)
    dTs = torch.randn(M, rp, generator=g)
    T = torch.randn(M, rp, generator=g)
    dTs[:, r:] = 0.0
    T[:, r:] = 0.0
    diag = torch.rand(r, generator=g) + 0.5
    scale = 0.8
    sd = 0x9E3779B97F4A7C15 % (1 << 62) + seed
    coef = scale * diag.double()
    gyx = gy.double()
    if p > 0:
        gyx = gyx * torch.from_numpy(DM.linear_mask(sd, p, M, N)).double() / (1.0 - p)
    dA_ref = coef.view(r, 1) * (dTs[:, :r].double().T @ x.double())
    dB_ref = (gyx.T @ T[:, :r].double()) * coef.view(1, r)
    dA0 = torch.randn(r, K, generator=g)
    dB0 = torch.randn(N, r, generator=g)
    to = lambda t: t.to(DEV)
    return dict(x=to(x), gy=to(gy), dTs=to(dTs), T=to(T), diag=to(diag), scale=scale, r=r, p=p,
                seed=torch.tensor([sd], dtype=torch.int64, device=DEV), dA=to(dA0.clone()), dB=to(dB0.clone()),
                dA0=dA0, dB0=dB0, dA_ref=dA_ref, dB_ref=dB_ref)


@pytest.mark.parametrize("r,p,dtype", [(4, 0.0, torch.bfloat16), (16, 0.25, torch.float16),
                                       (40, 0.1, torch.bfloat16), (64, 0.0, torch.float16)])
def test_wgrad_pair_matches_float64(r, p, dtype):
    from lora_b200 import ops
    c = _pair_case(300, 200, 88, r, p, dtype, seed=r)
    ops.wgrad_pair(c["x"], c["dTs"], c["dA"], c["gy"], c["T"], c["dB"], c["diag"], c["scale"], r, p,
                   c["seed"] if p > 0 else None)
    torch.cuda.synchronize()
    assert rel(c["dA"].double() - c["dA0"].to(DEV, F64), c["dA_ref"]) < 1e-5
    assert rel(c["dB"].double() - c["dB0"].to(DEV, F64), c["dB_ref"]) < 1e-5


@pytest.mark.parametrize("rs", [(4,), (1, 16, 8, 3)])
def test_wgrad_multi_matches_float64(rs):
    from lora_b200 import ops
    M, K = 333, 136
    cases = [_pair_case(M, K, 40 + 48 * i, r, 0.0, torch.bfloat16, seed=10 + i) for i, r in enumerate(rs)]
    x = cases[0]["x"]
    for c in cases:
        c["dA_ref"] = c["diag"].double().cpu().view(-1, 1) * c["scale"] * (
            c["dTs"][:, :c["r"]].double().cpu().T @ x.double().cpu())
    items = [(c["dTs"], c["dA"], c["gy"], c["T"], c["dB"], c["diag"], c["scale"], c["r"]) for c in cases]
    ops.wgrad_multi(x, items)
    torch.cuda.synchronize()
    for i, c in enumerate(cases):
        assert rel(c["dA"].double() - c["dA0"].to(DEV, F64), c["dA_ref"]) < 1e-5, i
        assert rel(c["dB"].double() - c["dB0"].to(DEV, F64), c["dB_ref"]) < 1e-5, i
