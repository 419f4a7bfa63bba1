"""GPU parity at the module / optimizer / training-step level (through the public Python API,
which reaches the kernels only via the C-ABI). Oracle side: oracle/ref_modules.py, oracle/ref_step.py,
oracle/lora_ops.py -- torch eager restatements of the reference, run on the same device."""
import copy

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu

DEV = "cuda"


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _pair(K, N, r, bias, scale, dtype=torch.float32, seed=0):
    """(our module, oracle site) sharing one frozen nn.Linear and identical LoRA factors."""
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


@pytest.mark.parametrize("K,N,r,bias", [(320, 320, 4, False), (640, 5120, 8, True), (768, 320, 4, False),
                                        (1280, 1280, 16, True), (72, 88, 3, True)])
def test_module_autocast_fwd_bwd_vs_oracle(K, N, r, bias):
    """fp32 frozen weights + torch.autocast(bf16): the reference's training configuration.
    The oracle rounds lora_down/lora_up outputs to bf16 (autocast), the fused kernel keeps them
    in fp32 up to one bf16 rounding of T': agreement to bf16 resolution (2^-8) of the outputs."""
    ours, ref = _pair(K, N, r, bias, 0.9)
    x1 = torch.randn(2, 77, K, device=DEV, requires_grad=True)
    x2 = x1.detach().clone().requires_grad_(True)
    gy = torch.randn(2, 77, N, device=DEV)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y1 = ours(x1)
        y2 = ref(x2)
    assert y1.dtype == y2.dtype == torch.bfloat16 and y1.shape == y2.shape
    y1.backward(gy.to(y1.dtype))
    y2.backward(gy.to(y2.dtype))
    assert rel(y1, y2) < 2 ** -7
    assert rel(x1.grad, x2.grad) < 2 ** -6
    assert rel(ours.lora_down.weight.grad, ref.down.grad) < 2 ** -6
    assert rel(ours.lora_up.weight.grad, ref.up.grad) < 2 ** -6
    assert ours.linear.weight.grad is None


def test_module_bf16_model_and_selector_and_scale():
    """16-bit host model; set_selector_from_diag + tune_lora_scale take effect on the next call."""
    import lora_b200 as L
    from oracle import lora_ops as O
    ours, _ = _pair(640, 640, 8, True, 1.0, dtype=torch.bfloat16)
    x = torch.randn(300, 640, device=DEV, dtype=torch.bfloat16)
    diag = torch.rand(8, device=DEV) + 0.25
    holder = nn.Sequential(ours)
    L.set_lora_diag(holder, diag)
    L.tune_lora_scale(holder, 0.35)
    y = holder(x)
    want = O.lora_linear_forward(x, ours.linear.weight, ours.linear.bias, ours.lora_down.weight,
                                 ours.lora_up.weight, 0.35, diag=diag)
    assert y.dtype == torch.bfloat16 and rel(y, want) < 2 ** -7
    L.tune_lora_scale(holder, 0.0)
    y0 = holder(x)
    want0 = O.lora_linear_forward(x, ours.linear.weight, ours.linear.bias, ours.lora_down.weight,
                                  torch.zeros_like(ours.lora_up.weight), 0.0)
    assert rel(y0, want0) < 2 ** -8


def test_external_weight_reassignment_is_seen():
    """The reference's API re-assigns .weight from outside (lora.py:302-303,706-711)."""
    from oracle import lora_ops as O
    ours, _ = _pair(320, 320, 4, False, 1.0)
    x = torch.randn(64, 320, device=DEV, dtype=torch.bfloat16)
    _ = ours(x)
    ours.lora_up.weight = nn.Parameter(torch.randn(320, 4, device=DEV) * 0.1)
    ours.lora_down.weight = nn.Parameter(torch.randn(4, 320, device=DEV) * 0.1)
    ours.linear.weight = nn.Parameter(torch.randn(320, 320, device=DEV) * 0.05, requires_grad=False)
    y = ours(x)
    want = O.lora_linear_forward(x, ours.linear.weight.to(torch.bfloat16), None,
                                 ours.lora_down.weight, ours.lora_up.weight, 1.0)
    assert rel(y, want) < 2 ** -7
    with torch.no_grad():
        ours.lora_up.weight.mul_(2.0)          # in-place edit bumps the version counter
    y2 = ours(x)
    want2 = O.lora_linear_forward(x, ours.linear.weight.to(torch.bfloat16), None,
                                  ours.lora_down.weight, ours.lora_up.weight, 1.0)
    assert rel(y2, want2) < 2 ** -7


def test_cpu_tensor_raises():
    import lora_b200 as L
    from lora_b200._C import LoraB200Error
    m = L.LoraInjectedLinear(32, 32, r=4, dropout_p=0.0)
    with pytest.raises(LoraB200Error):
        m(torch.randn(4, 32))


def test_arena_clip_adamw_matches_torch_and_oracle():
    """The optimizer launch (lb_optim_step_fused) vs torch.optim.AdamW + clip_grad_norm_ (what the
    reference calls) and vs the float64 oracle, 4 steps, two param groups, with and without the clip
    being active.
    Tolerance 2e-6 relative on the parameters (fp32 op-order differences only)."""
    import lora_b200 as L
    from lora_b200.arena import LoraArena
    from oracle import lora_ops as O
    torch.manual_seed(0)
    sites_a = nn.ModuleList([L.LoraInjectedLinear(64, 96, r=4, dropout_p=0.0) for _ in range(3)]).to(DEV)
    sites_b = nn.ModuleList([L.LoraInjectedLinear(48, 48, r=8, dropout_p=0.0) for _ in range(2)]).to(DEV)
    for s in list(sites_a) + list(sites_b):
        s.lora_up.weight.data.normal_(0, 0.1)
    arena = LoraArena([(sites_a, 1e-3), (sites_b, 5e-4)])
    params = arena.parameters()
    lrs = [1e-3] * 6 + [5e-4] * 4
    twins = [p.detach().clone().requires_grad_(True) for p in params]
    opt = torch.optim.AdamW([{"params": twins[:6], "lr": 1e-3}, {"params": twins[6:], "lr": 5e-4}],
                            betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    o_p = [p.detach().clone() for p in params]
    o_m = [torch.zeros_like(p) for p in params]
    o_v = [torch.zeros_like(p) for p in params]
    for step in range(1, 5):
        gs = [torch.randn_like(p) * (3.0 if step % 2 else 0.01) for p in params]
        for p, t, g in zip(params, twins, gs):
            p.grad.copy_(g)          # .grad is a view of the arena's g buffer
            t.grad = g.clone()
        total = torch.nn.utils.clip_grad_norm_(twins, 1.0)
        opt.step()
        o_p, o_m, o_v, o_total = O.clip_adamw_step(o_p, gs, o_m, o_v, step, lrs)
        arena.step(0.9, 0.999, 1e-8, 1e-2, 1.0, world_size=1)
        torch.cuda.synchronize()
        assert abs(float(arena.gnorm) - float(total)) <= 1e-5 * float(total)
        assert abs(float(arena.gnorm) - o_total) <= 1e-5 * o_total
        for p, t, op in zip(params, twins, o_p):
            assert rel(p, t) < 2e-6
            assert rel(p, op) < 2e-6
        assert float(arena.g.abs().max()) == 0.0    # zero_grad folded into the step
    # the 16-bit operand copies were refreshed by the step
    s = sites_a[0]
    d16 = s._lb.down[torch.bfloat16][1]
    assert torch.equal(d16[:4], s.lora_down.weight.detach().to(torch.bfloat16))
    assert int(arena.step_dev) == 4


def _tiny_models(seed=0):
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    torch.manual_seed(seed)
    unet = UNet2DConditionModel(UNetConfig.tiny()).to(DEV)
    text = build_text_encoder(tiny=True).to(DEV)
    unet.requires_grad_(False)
    text.requires_grad_(False)
    return unet, text


def test_training_step_matches_reference_step_tiny():
    """Whole Dreambooth step (text encoder + UNet, autocast bf16, clip, AdamW) on the tiny host
    models: lora_b200.train.LoraTrainStep vs the oracle's restated reference step with
    torch.optim.AdamW, same seeds => same noise / timesteps. Loss within 1e-2 relative per step
    (bf16 host-model arithmetic on both sides; the LoRA branch differs only in where 16-bit
    roundings sit), first-step gradients within 3e-2 relative."""
    import lora_b200 as L
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.train import LoraTrainStep, StepConfig
    from oracle.ref_modules import ref_inject
    from oracle.ref_step import RefDreamboothStep

    unet, text = _tiny_models()
    unet_r, text_r = copy.deepcopy(unet), copy.deepcopy(text)
    L.inject_trainable_lora(unet, r=4)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=4)
    us = ref_inject(unet_r, {"CrossAttention", "Attention", "GEGLU"}, r=4)
    ts = ref_inject(text_r, {"CLIPAttention"}, r=4)
    ours_sites = [m for m in list(unet.modules()) + list(text.modules()) if type(m).__name__ == "LoraInjectedLinear"]
    assert len(ours_sites) == len(us) + len(ts)
    g = torch.Generator(device=DEV).manual_seed(3)
    for o, r in zip(ours_sites, us + ts):
        o.lora_up.weight.data.normal_(0, 0.05, generator=g)
        r.up.data.copy_(o.lora_up.weight.data)
        r.down.data.copy_(o.lora_down.weight.data)

    cfg = StepConfig(use_cuda_graph=False, autocast_dtype=torch.bfloat16)
    tr = LoraTrainStep(unet, text, cfg, latent_shape=(1, 4, 16, 16), seq_len=77, device=DEV)
    ref = RefDreamboothStep(unet_r, text_r, DDPMNoiser(device=DEV), us, ts, autocast_dtype=torch.bfloat16)
    lat = torch.randn(1, 4, 16, 16, device=DEV) * 0.18215
    ids = torch.randint(0, 1000, (1, 77), device=DEV)
    tr.latents.copy_(lat)
    tr.input_ids.copy_(ids)

    # first-step gradients (before any optimizer step), same RNG stream
    torch.manual_seed(11)
    noise = torch.randn_like(lat)
    t = torch.randint(0, 1000, (1,), device=DEV).long()
    loss_r = ref.forward_loss(lat, ids, noise, t)
    loss_r.backward()
    g_ref = torch.cat([p.grad.flatten() for p in ref.unet_params + ref.text_params])
    ref.opt.zero_grad()
    torch.manual_seed(11)
    # run our body without the optimizer: forward/backward only
    tr.arena.zero_grad()
    noisy = tr.noiser.add_noise(lat, noise, t)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        ehs = text(ids)[0]
        pred = unet(noisy, t, ehs).sample
    loss_o = torch.nn.functional.mse_loss(pred.float(), noise.float())
    loss_o.backward()
    g_ours = torch.cat([p.grad.flatten() for p in tr.arena.parameters()])
    assert abs(float(loss_o) - float(loss_r)) < 1e-2 * abs(float(loss_r))
    assert rel(g_ours, g_ref) < 3e-2
    tr.arena.zero_grad()

    for step in range(3):
        torch.manual_seed(100 + step)
        l_ref = float(ref.step(lat, ids))
        torch.manual_seed(100 + step)
        l_ours = float(tr.step_device())
        assert abs(l_ours - l_ref) < 1e-2 * abs(l_ref), (step, l_ours, l_ref)


def test_training_step_cuda_graph_equals_eager():
    """The graph path (the one bench.py times) against the eager path, same models, same inputs,
    same noise/timesteps (external_noise): the per-step LOSSES must agree to 2e-3 relative over
    5 steps (not bit-for-bit: fp32 atomics in the dA/dB reductions are unordered) and the LoRA
    factors afterwards to 1e-4. prepare() rolls its warm-up steps back, so both paths take exactly
    5 optimizer steps from the same start."""
    import lora_b200 as L
    from lora_b200.train import LoraTrainStep, StepConfig
    losses, finals = [], []
    for use_graph in (False, True):
        unet, text = _tiny_models(seed=5)
        unet, text = unet.to(torch.bfloat16), text.to(torch.bfloat16)
        L.inject_trainable_lora(unet, r=4)
        L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=4)
        g = torch.Generator(device=DEV).manual_seed(3)
        for m in list(unet.modules()) + list(text.modules()):
            if type(m).__name__ == "LoraInjectedLinear":
                m.lora_up.weight.data.normal_(0, 0.05, generator=g)
        cfg = StepConfig(use_cuda_graph=use_graph, graph_warmup=2, external_noise=True)
        tr = LoraTrainStep(unet, text, cfg, latent_shape=(1, 4, 16, 16), device=DEV)
        torch.manual_seed(9)
        tr.latents.copy_(torch.randn(1, 4, 16, 16, device=DEV) * 0.18215)
        tr.input_ids.copy_(torch.randint(0, 1000, (1, 77), device=DEV))
        p_start = tr.arena.p.clone()
        tr.prepare()
        if use_graph:
            assert tr.graph is not None, tr.graph_error
        assert int(tr.arena.step_dev) == 0 and torch.equal(tr.arena.p, p_start)   # warm-up rolled back
        assert float(tr.arena.m.abs().max()) == 0.0 and float(tr.arena.g.abs().max()) == 0.0
        out = []
        for i in range(5):
            gen = torch.Generator(device=DEV).manual_seed(50 + i)
            tr.noise.copy_(torch.randn(1, 4, 16, 16, device=DEV, generator=gen))
            tr.timesteps.copy_(torch.randint(0, 1000, (1,), device=DEV, generator=gen))
            out.append(float(tr.step_device()))
        torch.cuda.synchronize()
        assert int(tr.arena.step_dev) == 5
        losses.append(out)
        finals.append(tr.arena.p.clone())
    for a, b in zip(*losses):
        assert a == a and a > 0 and abs(a - b) < 2e-3 * abs(a), losses
    assert rel(finals[1], finals[0]) < 1e-4


def test_extended_training_step_matches_reference_step_tiny():
    """--use_extended_lora shape of the step (Linear + ResnetBlock2D Conv2d sites through the arena:
    conv dA/dB land in the flat gradient buffer) vs the oracle's reference step. Dropout is set
    to 0 on both sides here (mask streams differ by design; tests/test_dropout_gpu.py)."""
    import lora_b200 as L
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.train import LoraTrainStep, StepConfig
    from oracle.ref_modules import ref_inject
    from oracle.ref_step import RefDreamboothStep

    unet, text = _tiny_models(seed=2)
    unet = unet.to(memory_format=torch.channels_last)
    unet_r, text_r = copy.deepcopy(unet), copy.deepcopy(text)
    L.inject_trainable_lora_extended(unet, r=4)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=4)
    us = ref_inject(unet_r, {"ResnetBlock2D", "CrossAttention", "Attention", "GEGLU"}, r=4, extended=True)
    ts = ref_inject(text_r, {"CLIPAttention"}, r=4)
    ours = [m for m in list(unet.modules()) + list(text.modules()) if type(m).__name__.startswith("LoraInjected")]
    assert len(ours) == len(us) + len(ts)
    assert any(type(m).__name__ == "LoraInjectedConv2d" for m in ours)
    g = torch.Generator(device=DEV).manual_seed(4)
    for o, r in zip(ours, us + ts):
        o.dropout.p = 0.0
        r.p = 0.0
        o.lora_up.weight.data.normal_(0, 0.05, generator=g)
        r.up.data.copy_(o.lora_up.weight.data)
        r.down.data.copy_(o.lora_down.weight.data)
    cfg = StepConfig(use_cuda_graph=False, autocast_dtype=torch.bfloat16)
    tr = LoraTrainStep(unet, text, cfg, latent_shape=(1, 4, 16, 16), seq_len=77, device=DEV)
    ref = RefDreamboothStep(unet_r, text_r, DDPMNoiser(device=DEV), us, ts, autocast_dtype=torch.bfloat16)
    lat = torch.randn(1, 4, 16, 16, device=DEV) * 0.18215
    ids = torch.randint(0, 1000, (1, 77), device=DEV)
    tr.latents.copy_(lat)
    tr.input_ids.copy_(ids)
    # gradients of the first step, identical noise / timestep
    torch.manual_seed(21)
    noise = torch.randn_like(lat)
    t = torch.randint(0, 1000, (1,), device=DEV).long()
    ref.forward_loss(lat, ids, noise, t).backward()
    g_ref = torch.cat([p.grad.flatten() for p in ref.unet_params + ref.text_params])
    ref.opt.zero_grad()
    noisy = tr.noiser.add_noise(lat, noise, t).contiguous(memory_format=torch.channels_last)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        pred = unet(noisy, t, text(ids)[0]).sample
    torch.nn.functional.mse_loss(pred.float(), noise.float()).backward()
    g_ours = torch.cat([p.grad.flatten() for p in tr.arena.parameters()])
    assert g_ours.numel() == g_ref.numel()
    assert rel(g_ours, g_ref) < 3e-2
    tr.arena.zero_grad()
    for step in range(2):
        torch.manual_seed(300 + step)
        l_ref = float(ref.step(lat, ids))
        torch.manual_seed(300 + step)
        l_ours = float(tr.step_device())
        assert abs(l_ours - l_ref) < 1e-2 * abs(l_ref), (step, l_ours, l_ref)


def test_collapse_lora_on_gpu_matches_oracle():
    """collapse_lora on CUDA models runs lb_lora_merge (one pass over W): W + alpha*up@down."""
    import lora_b200 as L
    from oracle import lora_ops as O
    torch.manual_seed(0)

    class Attention(nn.Module):
        def __init__(self):
            super().__init__()
            self.to_q = nn.Linear(320, 640, bias=False)

    class ResnetBlock2D(nn.Module):
        def __init__(self):
            super().__init__()
            self.conv1 = nn.Conv2d(64, 96, 3, padding=1)

    for dt in (torch.float32, torch.bfloat16):
        model = nn.Sequential(Attention(), ResnetBlock2D()).to(DEV).to(dt)
        L.inject_trainable_lora_extended(model, r=8)
        lin, conv = [m for m in model.modules() if type(m).__name__.startswith("LoraInjected")]
        lin.lora_up.weight.data.normal_(0, 0.1); conv.lora_up.weight.data.normal_(0, 0.1)
        w_lin, w_conv = lin.linear.weight.data.clone(), conv.conv.weight.data.clone()
        L.collapse_lora(model, alpha=0.7)
        want_lin = w_lin.double().cpu() + O.collapse_delta(lin.lora_down.weight, lin.lora_up.weight, 0.7)
        want_conv = w_conv.double().cpu() + O.collapse_delta(conv.lora_down.weight, conv.lora_up.weight, 0.7).reshape(w_conv.shape)
        tol = 1e-6 if dt == torch.float32 else 2 ** -8
        assert lin.linear.weight.dtype == dt and rel(lin.linear.weight, want_lin) < tol
        assert conv.conv.weight.shape == w_conv.shape and rel(conv.conv.weight, want_conv) < tol


def test_module_under_gradient_checkpointing():
    """The reference's trainers enable gradient checkpointing (train_lora_dreambooth.py:627-630):
    the site is re-run in backward. Gradients must equal the non-checkpointed ones."""
    from torch.utils.checkpoint import checkpoint
    ours, _ = _pair(640, 640, 4, True, 1.0, dtype=torch.bfloat16)
    x = torch.randn(3, 100, 640, device=DEV, dtype=torch.bfloat16)
    gy = torch.randn(3, 100, 640, device=DEV, dtype=torch.bfloat16)
    grads = []
    for use_ckpt in (False, True):
        xi = x.clone().requires_grad_(True)
        for p in (ours.lora_down.weight, ours.lora_up.weight):
            p.grad = None
        y = checkpoint(ours, xi, use_reentrant=False) if use_ckpt else ours(xi)
        y.backward(gy)
        grads.append((xi.grad.clone(), ours.lora_down.weight.grad.clone(), ours.lora_up.weight.grad.clone()))
    assert torch.equal(grads[0][0], grads[1][0])
    assert rel(grads[1][1], grads[0][1]) < 1e-5 and rel(grads[1][2], grads[0][2]) < 1e-5   # atomics order


def test_fp16_autocast_like_the_pti_trainer():
    """cli_lora_pti.py:315-316 runs torch.cuda.amp.autocast() = fp16, no GradScaler."""
    from oracle import lora_ops as O
    ours, ref = _pair(768, 1280, 16, True, 0.5)
    x = torch.randn(2, 77, 768, device=DEV, requires_grad=True)
    with torch.autocast("cuda", dtype=torch.float16):
        y = ours(x)
        y_ref = ref(x.detach())
    assert y.dtype == torch.float16
    assert rel(y, y_ref) < 2 ** -9
    y.float().sum().backward()
    dX, dA, dB = O.lora_linear_backward(torch.ones(154, 1280), x.detach().reshape(154, 768).half(),
                                        ours.linear.weight.half(), ours.lora_down.weight, ours.lora_up.weight, 0.5)
    assert rel(x.grad.reshape(154, 768), dX) < 2e-3
    assert rel(ours.lora_down.weight.grad, dA) < 2e-3 and rel(ours.lora_up.weight.grad, dB) < 2e-3


def test_batched_and_single_row_inputs():
    """Prior-preservation batches (bs 2) and the ResnetBlock2D time_emb_proj site (one row per image)."""
    from oracle import lora_ops as O
    ours, _ = _pair(1280, 320, 8, True, 1.0, dtype=torch.bfloat16)
    for shape in ((2, 1280), (1, 1280), (2, 3, 5, 1280)):
        x = torch.randn(*shape, device=DEV, dtype=torch.bfloat16)
        y = ours(x)
        assert y.shape == (*shape[:-1], 320)
        want = O.lora_linear_forward(x.reshape(-1, 1280), ours.linear.weight, ours.linear.bias,
                                     ours.lora_down.weight, ours.lora_up.weight, 1.0)
        assert rel(y.reshape(-1, 320), want) < 2 ** -7


def test_state_dict_and_device_moves():
    """Modules are built on CPU and moved (`_tmp.to(device).to(dtype)`, lora.py:295); state_dict keys
    are the reference's; loading a state_dict in place is picked up (version counter)."""
    import lora_b200 as L
    from oracle import lora_ops as O
    torch.manual_seed(0)
    m = L.LoraInjectedLinear(320, 320, bias=True, r=4, dropout_p=0.0)
    sd = {k: torch.randn_like(v) * 0.05 for k, v in m.state_dict().items()}
    m = m.to(DEV).to(torch.bfloat16)
    x = torch.randn(64, 320, device=DEV, dtype=torch.bfloat16)
    _ = m(x)
    m.load_state_dict(sd)                        # copy_ into existing Parameters: versions bump
    y = m(x)
    want = O.lora_linear_forward(x, sd["linear.weight"].to(torch.bfloat16), sd["linear.bias"].to(torch.bfloat16),
                                 sd["lora_down.weight"].to(torch.bfloat16), sd["lora_up.weight"].to(torch.bfloat16), 1.0)
    assert rel(y, want) < 2 ** -7


def test_arena_step_after_torch_side_edit_keeps_operands_fresh():
    """A factor edited in place by torch code (version bump) between two arena steps: the site
    must see the edit immediately AND the result of the following fused optimizer step."""
    import lora_b200 as L
    from lora_b200.arena import LoraArena
    from oracle import lora_ops as O
    torch.manual_seed(0)
    site = L.LoraInjectedLinear(320, 320, r=4, dropout_p=0.0).to(DEV)
    site.linear.requires_grad_(False)
    site.lora_up.weight.data.normal_(0, 0.1)
    arena = LoraArena([([site], 1e-2)])
    x = torch.randn(64, 320, device=DEV, dtype=torch.bfloat16)

    def want():
        return O.lora_linear_forward(x, site.linear.weight.to(torch.bfloat16), None, site.lora_down.weight,
                                     site.lora_up.weight, 1.0)
    assert rel(site(x), want()) < 2 ** -7
    with torch.no_grad():
        site.lora_up.weight.mul_(3.0)                 # torch-side in-place edit
    assert rel(site(x), want()) < 2 ** -7
    site.lora_up.weight.grad.normal_(0, 1.0)
    site.lora_down.weight.grad.normal_(0, 1.0)
    before = site.lora_up.weight.detach().clone()
    arena.step(max_norm=0.0)
    torch.cuda.synchronize()
    assert not torch.equal(before, site.lora_up.weight.detach())
    assert rel(site(x), want()) < 2 ** -7             # operands follow the fused step too


@pytest.mark.parametrize("r", [32, 20])
def test_rank_above_16_runs_as_rank_chunks(r):
    """A lora_join of two rank-16 files is rank 32 (lora_manager.py:13-71): the site must still run
    (rank chunks of 16, rank_chunks.py) and match the oracle forward and backward, selector included."""
    import lora_b200 as L
    from oracle import lora_ops as O
    torch.manual_seed(r)
    K, N, M = 320, 640, 300
    m = L.LoraInjectedLinear(K, N, bias=True, r=r, dropout_p=0.0, scale=0.6).to(DEV)
    m.linear.requires_grad_(False)
    m.lora_up.weight.data.normal_(0, 0.05)
    diag = torch.rand(r, device=DEV) + 0.5
    m.set_selector_from_diag(diag)
    x = torch.randn(M, K, device=DEV).to(torch.bfloat16).requires_grad_(True)
    y = m(x)
    gy = torch.randn_like(y)
    y.backward(gy)
    W16 = m.linear.weight.detach().to(torch.bfloat16)
    A, B = m.lora_down.weight.detach(), m.lora_up.weight.detach()
    ref = O.lora_linear_forward(x.detach(), W16, m.linear.bias, A, B, 0.6, diag=diag)
    base = O.lora_linear_forward(x.detach(), W16, m.linear.bias, A, torch.zeros_like(B), 0.0)
    branch = float((ref - base).norm())
    assert float((y.detach().double().cpu() - ref).norm()) <= 2 ** -6 * branch + 2 ** -8 * float(ref.norm())
    dX, dA, dB = O.lora_linear_backward(gy, x.detach(), W16, A, B, 0.6, diag=diag)
    assert rel(x.grad, dX) < 2e-2
    assert rel(m.lora_down.weight.grad, dA) < 2e-2 and rel(m.lora_up.weight.grad, dB) < 2e-2
    # eval mode / state_dict round trip keep working on the wide site
    m.eval()
    assert torch.equal(m(x.detach()), y.detach())
