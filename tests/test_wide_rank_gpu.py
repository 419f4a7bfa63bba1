"""LoRA ranks 17..64 on the fused kernels (rank pads 32 and 64), GPU, against the oracle at the bounds
the rank <= 16 tests use; ranks above 64 on linear sites run as rank chunks of 64."""
import copy

import pytest
import torch
import torch.nn as nn

from oracle import lora_ops as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _pair(K, N, r, bias, scale, dtype=torch.float32, seed=0):
    import lora_b200 as L
    from oracle.ref_modules import RefLoraSite
    torch.manual_seed(seed)
    base = nn.Linear(K, N, bias=bias).to(DEV).to(dtype)
    base.requires_grad_(False)
    ours = L.LoraInjectedLinear(K, N, bias=bias, r=r, dropout_p=0.0, scale=scale)
    ours.linear.weight = base.weight
    if bias:
        ours.linear.bias = base.bias
    ours = ours.to(DEV).to(dtype)
    ours.lora_up.weight.data.normal_(0, 0.05)
    ref = RefLoraSite(base, r=r, dropout_p=0.0, scale=scale)
    ref.down.data.copy_(ours.lora_down.weight.data)
    ref.up.data.copy_(ours.lora_up.weight.data)
    return ours, ref


@pytest.fixture
def linear_mode():
    from lora_b200 import _C
    yield lambda m: _C.lib.lb_debug_set_linear_mode(m)
    _C.lib.lb_debug_set_linear_mode(0)


@pytest.mark.parametrize("r", [17, 24, 32, 40, 64])
@pytest.mark.parametrize("K,N,M,bias,bn", [(72, 88, 77, True, 0), (640, 1280, 301, False, 1), (640, 1280, 301, True, 2)])
def test_linear_autocast_fwd_bwd(r, K, N, M, bias, bn, linear_mode):
    """Autocast bf16 (fp32 frozen weights), odd M; bn forces the 64- (1) or 128-wide (2) plan."""
    linear_mode(4 * bn)
    ours, ref = _pair(K, N, r, bias, 0.9)
    x1 = torch.randn(M, K, device=DEV, requires_grad=True)
    x2 = x1.detach().clone().requires_grad_(True)
    gy = torch.randn(M, N, device=DEV)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y1 = ours(x1)
        y2 = ref(x2)
    assert y1.dtype == y2.dtype == torch.bfloat16
    y1.backward(gy.to(y1.dtype))
    y2.backward(gy.to(y2.dtype))
    assert rel(y1, y2) < 2 ** -7
    assert rel(x1.grad, x2.grad) < 2 ** -6
    assert rel(ours.lora_down.weight.grad, ref.down.grad) < 2 ** -6
    assert rel(ours.lora_up.weight.grad, ref.up.grad) < 2 ** -6


@pytest.mark.parametrize("r", [24, 64])
@pytest.mark.parametrize("bn", [1, 2])
def test_linear_fp16_model_selector_and_fp32_output(r, bn, linear_mode):
    """fp16 host model with a selector diagonal; fp32 activations outside autocast (fp32 output)."""
    import lora_b200 as L
    linear_mode(4 * bn)
    ours, _ = _pair(640, 320, r, True, 1.0, dtype=torch.float16)
    x = torch.randn(257, 640, device=DEV, dtype=torch.float16)
    diag = torch.rand(r, device=DEV) + 0.25
    holder = nn.Sequential(ours)
    L.set_lora_diag(holder, diag)
    y = holder(x)
    want = O.lora_linear_forward(x, ours.linear.weight, ours.linear.bias, ours.lora_down.weight,
                                 ours.lora_up.weight, 1.0, diag=diag)
    assert y.dtype == torch.float16 and rel(y, want) < 2 ** -7
    o32, _ = _pair(320, 88, r, True, 0.7)
    x32 = torch.randn(129, 320, device=DEV)
    y32 = o32(x32)
    want32 = O.lora_linear_forward(x32.to(torch.bfloat16), o32.linear.weight.to(torch.bfloat16), o32.linear.bias,
                                   o32.lora_down.weight, o32.lora_up.weight, 0.7)
    assert y32.dtype == torch.float32 and rel(y32, want32) < 2 ** -7


@pytest.mark.parametrize("r", [24, 64])
@pytest.mark.parametrize("n,cin,cout,k,H,W", [(2, 64, 96, 3, 13, 19), (1, 320, 320, 3, 32, 32),
                                              (2, 96, 64, 1, 11, 9), (1, 640, 320, 1, 16, 16)])
def test_conv_fwd_bwd(r, n, cin, cout, k, H, W):
    import lora_b200 as L
    torch.manual_seed(n + cin + cout + H + r)
    pad = k // 2
    m = L.LoraInjectedConv2d(cin, cout, k, 1, pad, r=r, dropout_p=0.0, scale=0.8).to(DEV)
    m.conv.weight.data.mul_(0.5)
    m.conv.requires_grad_(False)
    m.lora_up.weight.data.normal_(0, 0.05)
    dt = torch.bfloat16
    x = torch.randn(n, cin, H, W, device=DEV).to(dt).requires_grad_(True)
    y = m(x)
    gy = torch.randn(n, cout, H, W, device=DEV).to(dt)
    y.backward(gy)
    W16 = m.conv.weight.detach().to(dt)
    A, B = m.lora_down.weight.detach(), m.lora_up.weight.detach()
    assert rel(y, O.lora_conv2d_forward(x, W16, m.conv.bias, A, B, 0.8, padding=pad)) < 2 ** -7
    dX, dA, dB = O.lora_conv2d_backward(gy, x, W16, A, B, 0.8, padding=pad)
    assert rel(x.grad, dX) < 2 ** -7
    assert rel(m.lora_down.weight.grad, dA) < 1e-2
    assert rel(m.lora_up.weight.grad, dB) < 1e-2


def test_linear_dropout_backward_r32():
    """Mask recovered from the forward; dX, dA, dB against the oracle with that mask."""
    import lora_b200 as L
    p, M, K, N, r = 0.25, 512, 320, 640, 32
    torch.manual_seed(0)
    m = L.LoraInjectedLinear(K, N, bias=True, r=r, dropout_p=p, scale=1.5).to(DEV)
    m.linear.requires_grad_(False)
    m.lora_up.weight.data.normal_(0, 0.2)
    x = torch.randn(M, K, device=DEV).to(torch.bfloat16).float().requires_grad_(True)
    m.train()
    y = m(x)
    gy = torch.randn(M, N, device=DEV).to(torch.bfloat16).float()
    y.backward(gy)
    W16 = m.linear.weight.detach().to(torch.bfloat16)
    A, B = m.lora_down.weight.detach(), m.lora_up.weight.detach()
    base = O.lora_linear_forward(x, W16, m.linear.bias, A, torch.zeros_like(B), 0.0)
    clean = O.lora_linear_forward(x, W16, m.linear.bias, A, B, 1.5) - base
    ratio = (y.detach().double().cpu() - base) / clean
    big = clean.abs() > 0.05 * clean.abs().mean()
    kept = ratio.abs() > 0.5
    assert abs(float(kept[big].double().mean()) - (1 - p)) < 0.01
    dX, dA, dB = O.lora_linear_backward(gy, x.detach(), W16, A, B, 1.5, keep_mask=kept.double(), dropout_p=p)
    assert rel(x.grad, dX) < 3e-2
    assert rel(m.lora_down.weight.grad, dA) < 3e-2
    assert rel(m.lora_up.weight.grad, dB) < 3e-2


@pytest.mark.parametrize("k", [1, 3])
def test_conv_dropout_backward_r32(k):
    """Conv site with active dropout at r = 32, checked like the rank-8 conv test of
    test_dropout_gpu.py: the realised keep-mask is recovered from the forward output, then dX, dA, dB
    must equal the oracle's backward evaluated with that mask. x, the down factor and the up factor
    (with a floor of 0.1) are non-negative, so every clean branch element is a sum of r positive
    terms, far from zero: each element's keep/drop is read unambiguously from the output."""
    import lora_b200 as L
    torch.manual_seed(2)
    p, r, cin, cout, H = 0.2, 32, 64, 128, 16
    pad = k // 2
    m = L.LoraInjectedConv2d(cin, cout, k, 1, pad, r=r, dropout_p=p, scale=1.25).to(DEV)
    m.conv.requires_grad_(False)
    m.lora_down.weight.data.abs_()
    up = m.lora_up.weight.data
    up.normal_(0, 0.3)
    up.copy_(up.abs() + 0.1)
    x = (torch.randn(2, cin, H, H, device=DEV).abs().to(torch.bfloat16)
         .contiguous(memory_format=torch.channels_last).requires_grad_(True))
    m.train()
    y = m(x)
    gy = torch.randn_like(y)
    y.backward(gy)
    W16 = m.conv.weight.detach().to(torch.bfloat16)
    A, B = m.lora_down.weight.detach(), m.lora_up.weight.detach()
    base = O.lora_conv2d_forward(x.detach(), W16, m.conv.bias, A, torch.zeros_like(B), 0.0, padding=pad)
    clean = O.lora_conv2d_forward(x.detach(), W16, m.conv.bias, A, B, 1.25, padding=pad) - base
    ratio = (y.detach().double().cpu() - base) / clean
    kept = ratio.abs() > 0.5
    big = clean.abs() > 0.05 * clean.abs().mean()
    assert abs(float(kept[big].double().mean()) - (1 - p)) < 0.02
    dX, dA, dB = O.lora_conv2d_backward(gy, x.detach(), W16, A, B, 1.25, padding=pad,
                                        keep_mask=kept.double(), dropout_p=p)
    assert rel(x.grad, dX) < 3e-2
    assert rel(m.lora_down.weight.grad, dA) < 3e-2
    assert rel(m.lora_up.weight.grad, dB) < 3e-2


@pytest.mark.parametrize("M,K,N,r,bias", [(512, 320, 320, 24, False), (130, 72, 88, 40, True)])
def test_split_mode_linear_wide_rank(M, K, N, r, bias):
    """fp32-faithful mode (set_fp32_mode("split")) at ranks whose pad is 32 / 64, forward and backward
    against the float64 oracle, bounds of tests/test_precise_gpu.py."""
    import lora_b200 as L
    L.set_fp32_mode("split")
    try:
        torch.manual_seed(M + N)
        m = L.LoraInjectedLinear(K, N, bias=bias, r=r, dropout_p=0.0, scale=0.7).to(DEV)
        m.linear.requires_grad_(False)
        m.lora_up.weight.data.normal_(0, 0.02)
        x = torch.randn(M, K, device=DEV, requires_grad=True)
        y = m(x)
        assert y.dtype == torch.float32
        gy = torch.randn(M, N, device=DEV)
        y.backward(gy)
    finally:
        L.set_fp32_mode("bf16")
    W, b = m.linear.weight.detach(), (m.linear.bias.detach() if bias else None)
    A, B = m.lora_down.weight.detach(), m.lora_up.weight.detach()
    ref = O.lora_linear_forward(x, W, b, A, B, 0.7)
    base = O.lora_linear_forward(x, W, b, A, torch.zeros_like(B), 0.0)
    branch = float((ref - base).norm())
    assert float((y.double().cpu() - ref).norm()) <= 2 ** -7 * branch + 1e-4 * float(ref.norm())
    dX, dA, dB = O.lora_linear_backward(gy, x, W, A, B, 0.7)
    assert rel(x.grad, dX) < 2e-3
    assert rel(m.lora_down.weight.grad, dA) < 2e-3
    assert rel(m.lora_up.weight.grad, dB) < 1e-4


def test_rank8_through_pad32_equals_pad16():
    """The same rank-8 operands run through r_pad = 32 and r_pad = 16: fp32 reordering only."""
    from lora_b200 import _C, ops
    torch.manual_seed(0)
    M, K, N, r = 300, 320, 640, 8
    dt = torch.bfloat16
    x = torch.randn(M, K, device=DEV, dtype=dt)
    W = (torch.randn(N, K, device=DEV) * 0.05).to(dt)
    A = torch.randn(r, K, device=DEV) / r
    B = torch.randn(N, r, device=DEV) * 0.1
    d16 = ops.cast_rows_pad16(A, K, 1, r, K, dt)
    d32 = torch.zeros(32, K, device=DEV, dtype=dt)
    d32[:16] = d16
    y16, t16 = ops.fused_linear(x, W, None, d16, B, r, 1, None, 0.9, r, torch.float32, True)
    y32, t32 = ops.fused_linear(x, W, None, d32, B, r, 1, None, 0.9, r, torch.float32, True)
    assert t32.shape == (M, 32) and torch.count_nonzero(t32[:, 16:]) == 0
    assert rel(t32[:, :16], t16) < 1e-6 and rel(y32, y16) < 1e-6
    # the aux kernels agree as well: dA through the pad-32 V
    out16 = torch.zeros(r, K, device=DEV)
    out32 = torch.zeros(r, K, device=DEV)
    ops.wgrad(x, t16, None, 0.5, out16, K, 1, r)
    ops.wgrad(x, t32, None, 0.5, out32, K, 1, r)
    assert rel(out32, out16) < 1e-6


@pytest.mark.parametrize("r", [65, 128])
def test_linear_above_64_runs_as_chunks(r):
    ours, ref = _pair(320, 640, r, True, 0.5)
    ours.eval()
    x1 = torch.randn(2, 77, 320, device=DEV, requires_grad=True)
    x2 = x1.detach().clone().requires_grad_(True)
    gy = torch.randn(2, 77, 640, device=DEV)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y1 = ours(x1)
        y2 = ref(x2)
    y1.backward(gy.to(y1.dtype))
    y2.backward(gy.to(y2.dtype))
    assert rel(y1, y2) < 2 ** -7
    assert rel(x1.grad, x2.grad) < 2 ** -6
    assert rel(ours.lora_down.weight.grad, ref.down.grad) < 2 ** -6
    assert rel(ours.lora_up.weight.grad, ref.up.grad) < 2 ** -6


def test_conv_above_64_raises():
    import lora_b200 as L
    from lora_b200._C import LoraB200Error
    m = L.LoraInjectedConv2d(96, 96, 3, 1, 1, r=65, dropout_p=0.0).to(DEV)
    with pytest.raises(LoraB200Error):
        m(torch.randn(1, 96, 8, 8, device=DEV, dtype=torch.bfloat16))


def test_collapse_lora_r32():
    import lora_b200 as L

    class Attention(nn.Module):
        def __init__(self):
            super().__init__()
            self.to_q = nn.Linear(320, 640, bias=False)

    class ResnetBlock2D(nn.Module):
        def __init__(self):
            super().__init__()
            self.conv1 = nn.Conv2d(64, 96, 3, padding=1)

    torch.manual_seed(0)
    for dt in (torch.float32, torch.bfloat16):
        model = nn.Sequential(Attention(), ResnetBlock2D()).to(DEV).to(dt)
        L.inject_trainable_lora_extended(model, r=32)
        lin, conv = [m for m in model.modules() if type(m).__name__.startswith("LoraInjected")]
        lin.lora_up.weight.data.normal_(0, 0.1); conv.lora_up.weight.data.normal_(0, 0.1)
        w_lin, w_conv = lin.linear.weight.data.clone(), conv.conv.weight.data.clone()
        L.collapse_lora(model, alpha=0.7)
        want_lin = w_lin.double().cpu() + O.collapse_delta(lin.lora_down.weight, lin.lora_up.weight, 0.7)
        want_conv = w_conv.double().cpu() + O.collapse_delta(conv.lora_down.weight, conv.lora_up.weight, 0.7).reshape(w_conv.shape)
        tol = 1e-6 if dt == torch.float32 else 2 ** -8
        assert rel(lin.linear.weight, want_lin) < tol
        assert rel(conv.conv.weight, want_conv) < tol


def _tiny_models(seed=0):
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    torch.manual_seed(seed)
    unet = UNet2DConditionModel(UNetConfig.tiny()).to(DEV)
    text = build_text_encoder(tiny=True).to(DEV)
    unet.requires_grad_(False)
    text.requires_grad_(False)
    return unet, text


def test_extended_training_step_r32_padded_shadow_table_matches_reference_step_tiny():
    """--use_extended_lora shape of the step at r = 32 (Linear + ResnetBlock2D Conv2d sites, rank pad
    32, 32-row shadow slots) vs the oracle's reference step, as the r = 4 test in
    test_modules_gpu.py. The first-step factor gradients go through the deferred reduction queue
    (lb_lora_wgrad_batch) that LoraTrainStep runs; then two optimizer steps: losses, and every LoRA
    factor afterwards. Dropout is 0 on both sides (mask streams differ by design)."""
    import lora_b200 as L
    from lora_b200 import ops
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.train import LoraTrainStep, StepConfig
    from oracle.ref_modules import ref_inject
    from oracle.ref_step import RefDreamboothStep

    r = 32
    unet, text = _tiny_models(seed=2)
    unet = unet.to(memory_format=torch.channels_last)
    unet_r, text_r = copy.deepcopy(unet), copy.deepcopy(text)
    L.inject_trainable_lora_extended(unet, r=r)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=r)
    us = ref_inject(unet_r, {"ResnetBlock2D", "CrossAttention", "Attention", "GEGLU"}, r=r, extended=True)
    ts = ref_inject(text_r, {"CLIPAttention"}, r=r)
    ours = [m for m in list(unet.modules()) + list(text.modules()) if type(m).__name__.startswith("LoraInjected")]
    assert len(ours) == len(us) + len(ts)
    assert any(type(m).__name__ == "LoraInjectedConv2d" for m in ours)
    g = torch.Generator(device=DEV).manual_seed(4)
    for o, rs in zip(ours, us + ts):
        o.dropout.p = 0.0
        rs.p = 0.0
        o.lora_up.weight.data.normal_(0, 0.05, generator=g)
        rs.up.data.copy_(o.lora_up.weight.data)
        rs.down.data.copy_(o.lora_down.weight.data)
    cfg = StepConfig(use_cuda_graph=False, autocast_dtype=torch.bfloat16)
    tr = LoraTrainStep(unet, text, cfg, latent_shape=(1, 4, 16, 16), seq_len=77, device=DEV)
    assert int(tr.arena.table[:, 7].max()) == 32
    ref = RefDreamboothStep(unet_r, text_r, DDPMNoiser(device=DEV), us, ts, autocast_dtype=torch.bfloat16)
    lat = torch.randn(1, 4, 16, 16, device=DEV) * 0.18215
    ids = torch.randint(0, 1000, (1, 77), device=DEV)
    tr.latents.copy_(lat)
    tr.input_ids.copy_(ids)
    torch.manual_seed(21)
    noise = torch.randn_like(lat)
    t = torch.randint(0, 1000, (1,), device=DEV).long()
    ref.forward_loss(lat, ids, noise, t).backward()
    g_ref = torch.cat([p.grad.flatten() for p in ref.unet_params + ref.text_params])
    ref.opt.zero_grad()
    tr.arena.zero_grad()
    noisy = tr.noiser.add_noise(lat, noise, t).contiguous(memory_format=torch.channels_last)
    ops.wgrad_defer_begin()
    try:
        with torch.autocast("cuda", dtype=torch.bfloat16):
            pred = unet(noisy, t, text(ids)[0]).sample
        torch.nn.functional.mse_loss(pred.float(), noise.float()).backward()
    except BaseException:
        ops.wgrad_defer_cancel()
        raise
    assert ops.wgrad_flush() >= 1
    g_ours = torch.cat([p.grad.flatten() for p in tr.arena.parameters()])
    assert g_ours.numel() == g_ref.numel()
    assert rel(g_ours, g_ref) < 3e-2
    tr.arena.zero_grad()
    p0 = torch.cat([p.detach().flatten() for p in tr.arena.parameters()]).clone()
    for step in range(2):
        torch.manual_seed(300 + step)
        l_ref = float(ref.step(lat, ids))
        torch.manual_seed(300 + step)
        l_ours = float(tr.step_device())
        assert abs(l_ours - l_ref) < 1e-2 * abs(l_ref), (step, l_ours, l_ref)
    p_ours = torch.cat([p.detach().flatten() for p in tr.arena.parameters()])
    p_ref = torch.cat([p.detach().flatten() for p in ref.unet_params + ref.text_params])
    # two AdamW steps move each factor by ~2 lr (4e-4 of factors of rms ~0.04): the factors agree far
    # inside that, and the two updates point the same way
    assert rel(p_ours, p_ref) < 2e-3
    d_ours, d_ref = (p_ours - p0).double().cpu(), (p_ref - p0).double().cpu()
    assert float(torch.nn.functional.cosine_similarity(d_ours, d_ref, dim=0)) > 0.8


def test_extended_training_step_r32_cuda_graph_equals_eager():
    """Extended (Linear + Conv2d) sites at r = 32: the captured step against the eager step, as the
    r = 4 test in test_modules_gpu.py (losses to 2e-3, factors to 1e-4: fp32 atomics are unordered)."""
    import lora_b200 as L
    from lora_b200.train import LoraTrainStep, StepConfig
    losses, finals = [], []
    for use_graph in (False, True):
        unet, text = _tiny_models(seed=5)
        unet = unet.to(torch.bfloat16).to(memory_format=torch.channels_last)
        text = text.to(torch.bfloat16)
        L.inject_trainable_lora_extended(unet, r=32)
        L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=32)
        g = torch.Generator(device=DEV).manual_seed(3)
        for m in list(unet.modules()) + list(text.modules()):
            if type(m).__name__.startswith("LoraInjected"):
                m.lora_up.weight.data.normal_(0, 0.05, generator=g)
        cfg = StepConfig(use_cuda_graph=use_graph, graph_warmup=2, external_noise=True)
        tr = LoraTrainStep(unet, text, cfg, latent_shape=(1, 4, 16, 16), device=DEV)
        torch.manual_seed(9)
        tr.latents.copy_(torch.randn(1, 4, 16, 16, device=DEV) * 0.18215)
        tr.input_ids.copy_(torch.randint(0, 1000, (1, 77), device=DEV))
        tr.prepare()
        if use_graph:
            assert tr.graph is not None, tr.graph_error
        out = []
        for i in range(3):
            gen = torch.Generator(device=DEV).manual_seed(50 + i)
            tr.noise.copy_(torch.randn(1, 4, 16, 16, device=DEV, generator=gen))
            tr.timesteps.copy_(torch.randint(0, 1000, (1,), device=DEV, generator=gen))
            out.append(float(tr.step_device()))
        torch.cuda.synchronize()
        assert int(tr.arena.step_dev) == 3
        losses.append(out)
        finals.append(tr.arena.p.clone())
    for a, b in zip(*losses):
        assert a == a and a > 0 and abs(a - b) < 2e-3 * abs(a), losses
    assert rel(finals[1], finals[0]) < 1e-4
