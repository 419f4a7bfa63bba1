"""The step's prologue / loss-epilogue kernels (csrc/step_glue.cu) against the plain torch
formulation the reference uses (scheduler.add_noise, cat, F.mse_loss: cli_lora_pti.py:295-370,
train_lora_dreambooth.py:822-875), and the one-launch optimizer step against the float64 oracle and
lb_refresh_shadows."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("inpaint", [False, True])
def test_step_prologue_equals_add_noise_cast_cat(out_dtype, inpaint):
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.step_ops import step_prologue
    torch.manual_seed(0)
    noiser = DDPMNoiser(device=DEV)
    lat = torch.randn(3, 4, 24, 16, device=DEV) * 0.18215
    eps = torch.randn_like(lat)
    t = torch.tensor([0, 517, 999], device=DEV)
    mask = (torch.rand(3, 1, 24, 16, device=DEV) > 0.5).float() if inpaint else None
    ml = torch.randn_like(lat) if inpaint else None
    out = step_prologue(lat, eps, t, noiser, out_dtype, mask, ml)
    want = noiser.add_noise(lat, eps, t)
    if inpaint:
        want = torch.cat([want, mask, ml], dim=1)
    assert out.shape == want.shape and out.dtype == out_dtype
    assert out.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(out, want.to(out_dtype)) or torch.allclose(out.float(), want.to(out_dtype).float(), atol=0, rtol=2e-7)


@pytest.mark.parametrize("fmt", ["nchw", "nhwc"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("variant", ["plain", "mask", "prior"])
def test_masked_mse_and_its_gradient(fmt, dtype, variant):
    from lora_b200.step_ops import fused_masked_mse
    torch.manual_seed(1)
    B, C, H, W = 4, 4, 16, 24
    pred0 = torch.randn(B, C, H, W, device=DEV).to(dtype)
    if fmt == "nhwc":
        pred0 = pred0.contiguous(memory_format=torch.channels_last)
    target = torch.randn(B, C, H, W, device=DEV)
    m = None
    if variant == "mask":
        m = (torch.rand(B, 1, H, W, device=DEV) + 0.01)
        m = m / m.max()
    w = None
    if variant == "prior":
        w = torch.cat([torch.full((2,), 1.0 / 2), torch.full((2,), 0.7 / 2)]).to(DEV)
    p1 = pred0.clone().requires_grad_(True)
    loss = fused_masked_mse(p1, target, m, w)
    (loss * 1.5).backward()
    p2 = pred0.clone().float().requires_grad_(True)      # torch reference on the same rounded inputs
    pm, tm = (p2 * m, target * m) if m is not None else (p2, target)
    if variant == "prior":
        a, b = torch.chunk(pm, 2), torch.chunk(tm, 2)
        ref = F.mse_loss(a[0], b[0], reduction="none").mean([1, 2, 3]).mean() + 0.7 * F.mse_loss(a[1], b[1])
    else:
        ref = F.mse_loss(pm, tm, reduction="none").mean([1, 2, 3]).mean()
    (ref * 1.5).backward()
    assert abs(float(loss) - float(ref)) <= 2e-6 * abs(float(ref))
    tol = 2 ** -8 if dtype == torch.bfloat16 else 1e-6
    err = float((p1.grad.float() - p2.grad).norm() / p2.grad.norm())
    assert err < tol, err
    assert p1.grad.stride() == p1.stride()


def _optimizer_run(sites_spec, mode):
    """Three optimizer steps of a LoraArena over seeded gradients (the second one large enough to
    clip). sites_spec: [("linear" | "conv", r)]; mode: "fused" (lb_optim_step_fused) or "dp"
    (lb_optim_step_dp at world = 1, with the arena's own gradient buffer and a zeroed flag array as
    the only peer). Returns the arena, its start point and the three gradients."""
    import ctypes
    import torch.nn as nn
    import lora_b200 as L
    from lora_b200.arena import LoraArena
    torch.manual_seed(0)
    sites = nn.ModuleList([L.LoraInjectedLinear(320, 640, r=r, dropout_p=0.0) if kind == "linear" else
                           L.LoraInjectedConv2d(64, 96, 3, 1, 1, r=r, dropout_p=0.0)
                           for kind, r in sites_spec]).to(DEV)
    for s in sites:
        s.lora_up.weight.data.normal_(0, 0.1)
    arena = LoraArena([(sites, 1e-3)])
    if mode == "dp":
        arena._dp_flags = torch.zeros(2, device=DEV, dtype=torch.int32)
        arena._dp_epoch = torch.zeros(1, device=DEV, dtype=torch.int32)
        arena.gsum = torch.zeros_like(arena.g)
        one = ctypes.c_void_p * 1
        arena._dp = (one(arena.g.data_ptr()), one(arena._dp_flags.data_ptr()), 1, 0)
    p0, grads = arena.p.clone(), []
    g = torch.Generator(device=DEV).manual_seed(5)
    for step in range(3):
        grads.append(torch.randn(arena.n, device=DEV, generator=g) * (2.0 if step == 1 else 0.01))
        arena.g.copy_(grads[-1])
        arena.step(0.9, 0.999, 1e-8, 1e-2, 1.0, world_size=1)
    torch.cuda.synchronize()
    assert float(arena.g.abs().max()) == 0.0 and int(arena.step_dev) == 3
    return arena, p0, grads


def _final_state(arena):
    return arena.p.clone(), arena.m.clone(), arena.v.clone(), arena.shadow.clone(), float(arena.gnorm)


def _assert_same_step(got, want):
    # same arithmetic; only the block partition of the sum of squares differs (fp32 order noise in
    # the clip coefficient), so parameters agree to ~1e-7 and the 16-bit shadows to one ulp
    for a, b in zip(got[:3], want[:3]):
        assert float((a - b).norm() / (b.norm() + 1e-30)) < 2e-6
    sa, sb = got[3].float(), want[3].float()
    assert float((sa - sb).abs().max()) <= 2.0 ** -7 * float(sb.abs().max())
    assert float((sa != sb).float().mean()) < 1e-3
    assert abs(got[4] - want[4]) <= 1e-6 * abs(want[4])


def test_one_launch_optimizer_matches_oracle_and_shadow_refresh():
    """lb_optim_step_fused / lb_optim_step_dp at world 1 (cooperative: norm, grid barrier, AdamW +
    zero_grad, grid barrier, shadows), with 16-row shadow slots only and with 32-row ones (r = 32
    linear and conv sites): the shadows are bit for bit a fresh lb_refresh_shadows of the final
    parameters, and p, m, v and the norm follow the float64 clip + AdamW of oracle.lora_ops (run
    with the fp32-rounded hyper-parameters the launch receives)."""
    from lora_b200 import _C
    from lora_b200._C import check, dtype_code, ptr, stream_ptr
    from oracle import lora_ops as O

    def f32(x):
        return float(torch.tensor(x, dtype=torch.float32))

    specs = ([("linear", 4)] * 5 + [("conv", 8)], [("linear", 4)] * 4 + [("linear", 32), ("conv", 32)])
    for mode, spec in ((mode, spec) for mode in ("fused", "dp") for spec in specs):
        arena, p0, grads = _optimizer_run(spec, mode)
        fresh = torch.zeros_like(arena.shadow)
        check(_C.lib.lb_refresh_shadows(ptr(arena.p), ptr(arena.table), arena.table.shape[0], arena.table_max_c,
                                        ptr(fresh), dtype_code(arena.compute_dtype), stream_ptr()),
              "lb_refresh_shadows")
        torch.cuda.synchronize()
        assert torch.equal(arena.shadow.view(torch.int16), fresh.view(torch.int16)), (mode, spec)
        p, m, v = [p0], [torch.zeros_like(p0)], [torch.zeros_like(p0)]
        for step, g in enumerate(grads, 1):
            p, m, v, total = O.clip_adamw_step(p, [g], m, v, step, [f32(1e-3)], beta1=f32(0.9), beta2=f32(0.999),
                                               eps=f32(1e-8), weight_decay=f32(1e-2), max_norm=1.0)
        for name, got, want in (("p", arena.p, p[0]), ("m", arena.m, m[0]), ("v", arena.v, v[0])):
            err = float((got.double().cpu() - want).norm() / want.norm())
            assert err < 2e-6, (mode, spec, name, err)
        assert abs(float(arena.gnorm) - total) <= 1e-5 * total, (mode, spec)


def test_data_parallel_optimizer_at_world_one_equals_one_launch():
    """lb_optim_step_dp with a single rank (its all-reduce reads only its own gradients) against
    lb_optim_step_fused on an identical arena with an r = 4 and an r = 32 site: the same parameters,
    moments and shadows."""
    spec = [("linear", 4), ("conv", 32)]
    _assert_same_step(_final_state(_optimizer_run(spec, "dp")[0]), _final_state(_optimizer_run(spec, "fused")[0]))
