"""fp16 mixed precision with dynamic loss scaling on the device, against torch.amp.GradScaler:

  * the scaled optimizer launch (lb_optim_step_fused, lb_optim_step_dp at world 1) against
    GradScaler("cuda") + clip_grad_norm_ + AdamW + LambdaLR, over clean, inf, NaN and growth steps;
    with no scaler, both launches bit-identical to the release before loss scaling
    (tests/golden/optim_null_scaler.pt); with a scaler, and unscaled at world_size 2, bit-identical
    to the release before the two launches shared one kernel (tests/golden/optim_paths.pt; both
    recorded by scripts/make_golden_optim.py);
  * the loss epilogue's grad_scale;
  * whole fp16 steps (tiny SD1.5 models) and the train_lora_w_ti.py embedding step against the oracle
    (oracle/amp_ref.py), eager and graph-replayed, with skipped steps, growth and a warm-up schedule;
  * prepare() leaving the scaler state untouched, and the launch count of the scaled step.
"""
import copy
import ctypes
import os

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _two_group_arena(seed=0):
    import lora_b200 as L
    from lora_b200.arena import LoraArena
    torch.manual_seed(seed)
    sites_a = nn.ModuleList([L.LoraInjectedLinear(64, 96, r=4, dropout_p=0.0) for _ in range(2)]).to(DEV)
    sites_b = nn.ModuleList([L.LoraInjectedLinear(48, 48, r=8, dropout_p=0.0) for _ in range(2)]).to(DEV)
    for s in list(sites_a) + list(sites_b):
        s.lora_up.weight.data.normal_(0, 0.1)
    return LoraArena([(sites_a, 1e-3), (sites_b, 5e-4)])


def _as_world_one_dp(arena):
    """lb_optim_step_dp with a single rank: its own gradient buffer and a zeroed flag array as the peer."""
    arena._dp_flags = torch.zeros(2, device=DEV, dtype=torch.int32)
    arena._dp_epoch = torch.zeros(1, device=DEV, dtype=torch.int32)
    arena.gsum = torch.zeros_like(arena.g)
    one = ctypes.c_void_p * 1
    arena._dp = (one(arena.g.data_ptr()), one(arena._dp_flags.data_ptr()), 1, 0)


def null_scaler_run(mode, inputs):
    """Three optimizer steps with no scaler from the golden's start point and gradients. Uses only
    the arena API both releases share, so the same function recorded the golden."""
    arena = _two_group_arena()
    if mode == "dp":
        _as_world_one_dp(arena)
    arena.p.copy_(inputs["p0"].to(DEV))
    arena.refresh_shadows()
    for g in inputs["grads"]:
        arena.g.copy_(g.to(DEV))
        arena.step(0.9, 0.999, 1e-8, 1e-2, 1.0, world_size=1)
    torch.cuda.synchronize()
    return {"p": arena.p.cpu(), "m": arena.m.cpu(), "v": arena.v.cpu(), "shadow": arena.shadow.cpu(),
            "gnorm": arena.gnorm.cpu(), "step": arena.step_dev.cpu()}


@pytest.mark.parametrize("mode", ["fused", "dp"])
def test_no_scaler_is_bit_identical_to_the_previous_release(mode):
    d = torch.load(os.path.join(GOLD, "optim_null_scaler.pt"))
    got = null_scaler_run(mode, d["inputs"])
    for k, want in d[mode].items():
        assert torch.equal(got[k], want), (mode, k)


def _warmup_linear(warmup, total):
    def lam(k):
        if k < warmup:
            return k / warmup
        return max(0.0, (total - k) / max(1, total - warmup))
    return lam


# step -> value written into one element of the scaled gradient
INJECT = {2: float("inf"), 4: float("nan")}


def _scaled_kernel_run(mode):
    """Eight steps of the scaled launch and of GradScaler("cuda") + clip + AdamW + LambdaLR (linear,
    2 warm-up steps) on twin parameters; init_scale 2^14, growth_interval 2."""
    from lora_b200.arena import LrSchedule
    arena = _two_group_arena()
    if mode == "dp":
        _as_world_one_dp(arena)
    arena.enable_loss_scaling(init_scale=2.0 ** 14, growth_interval=2)
    sched = LrSchedule("linear", 2, 10, (0, 1))
    params = arena.parameters()
    twins = [p.detach().clone().requires_grad_(True) for p in params]
    opt = torch.optim.AdamW([{"params": twins[:4], "lr": 1e-3}, {"params": twins[4:], "lr": 5e-4}],
                            betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    lr_sched = torch.optim.lr_scheduler.LambdaLR(opt, _warmup_linear(2, 10))
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 14, growth_interval=2)
    scaler.scale(torch.ones((), device=DEV))                   # materialises the scale tensor
    gen = torch.Generator(device=DEV).manual_seed(5)
    trace = []
    for k in range(8):
        s = scaler.get_scale()
        assert float(arena.loss_scale) == s, k
        gs = [torch.randn(p.shape, device=DEV, generator=gen) * (3.0 if k % 2 else 0.01) * s for p in params]
        if k in INJECT:
            gs[1].view(-1)[7] = INJECT[k]
        before = {"p": arena.p.clone(), "m": arena.m.clone(), "v": arena.v.clone(), "t": arena.step_dev.clone(),
                  "shadow": arena.shadow.clone(), "applied": arena.applied_steps.clone()}
        for p, t, g in zip(params, twins, gs):
            p.grad.copy_(g)
            t.grad = g.clone()
        scaler.unscale_(opt)
        total = torch.nn.utils.clip_grad_norm_(twins, 1.0)
        scaler.step(opt)
        scaler.update()
        skipped = scaler.get_scale() < s
        if not skipped:
            lr_sched.step()
        opt.zero_grad()
        arena.step(0.9, 0.999, 1e-8, 1e-2, 1.0, world_size=1, schedule=sched)
        torch.cuda.synchronize()
        assert arena.step_was_skipped() == skipped == (k in INJECT), k
        assert float(arena.loss_scale) == scaler.get_scale(), k
        assert int(arena._growth_tracker) == scaler._get_growth_tracker(), k
        assert float(arena.g.abs().max()) == 0.0, k
        if skipped:
            for name, t in (("p", arena.p), ("m", arena.m), ("v", arena.v), ("t", arena.step_dev),
                            ("shadow", arena.shadow), ("applied", arena.applied_steps)):
                assert torch.equal(t, before[name]), (k, name)
            assert not torch.isfinite(arena.gnorm).all()
        else:
            assert abs(float(arena.gnorm) - float(total)) <= 1e-5 * float(total), k
        st = opt.state[twins[0]]
        assert int(arena.step_dev) == int(st["step"]) == int(arena.applied_steps), k
        for (_, _, _, o, n), p, t in zip(arena.entries, params, twins):
            assert rel(p, t) < 2e-6, k
            assert rel(arena.m[o:o + n], opt.state[t]["exp_avg"].flatten()) < 2e-6, k
            # the kernel's (1 - beta2) comes from fp32 beta2 (0.999f): 4.7e-5 from torch's double
            assert rel(arena.v[o:o + n], opt.state[t]["exp_avg_sq"].flatten()) < 1e-4, k
        trace.append((skipped, float(arena.loss_scale)))
    # growth after two clean steps (k = 1, 6), backoff on the inf (k = 2) and the NaN (k = 4)
    assert [sc for _, sc in trace] == [2.0 ** e for e in (14, 15, 14, 14, 13, 13, 14, 14)], trace
    return arena.p.clone(), arena.m.clone(), arena.v.clone(), arena.shadow.clone(), trace


def test_scaled_fused_launch_matches_torch_grad_scaler_and_dp_at_world_one():
    fused = _scaled_kernel_run("fused")
    dp = _scaled_kernel_run("dp")
    assert fused[4] == dp[4]
    for a, b in zip(fused[:3], dp[:3]):
        assert rel(a, b) < 2e-6
    sa, sb = fused[3].float(), dp[3].float()
    assert float((sa - sb).abs().max()) <= 2.0 ** -7 * float(sb.abs().max())


# the loss scale before each of the eight scaled steps of optim_paths.pt: growth after two clean
# steps, backoff on INJECT's inf (step 2) and NaN (step 4)
PATHS_SCALES = [2.0 ** e for e in (14, 14, 15, 14, 14, 13, 13, 14)]
OPTIM_PATHS = ("fused_scaled", "dp_scaled", "fused_world2")


def optim_paths_inputs(arena, gen):
    """Host inputs of tests/golden/optim_paths.pt: the arena's start point, eight loss-scaled
    gradients (3.0 * randn on odd steps, clipped; INJECT's inf and NaN in element 7 of the second
    factor) and three unscaled ones for the world_size=2 run (the second one clipped)."""
    bad = arena.entries[1][3] + 7
    scaled = []
    for k, s in enumerate(PATHS_SCALES):
        g = torch.randn(arena.n, generator=gen) * (3.0 if k % 2 else 0.01) * s
        if k in INJECT:
            g[bad] = INJECT[k]
        scaled.append(g)
    return {"p0": arena.p.cpu().clone(), "scaled": scaled,
            "unscaled": [torch.randn(arena.n, generator=gen) * s for s in (0.01, 2.0, 0.01)]}


def optim_paths_run(run, inputs):
    """One run of optim_paths.pt: the scaled launch of lb_optim_step_fused or lb_optim_step_dp (world 1)
    with a linear warm-up schedule, or the unscaled lb_optim_step_fused at world_size 2 (inv_world
    0.5, the NCCL data-parallel path). Per step the norm and the device state, then the final arena.
    Uses only the arena API both releases share, so the same function recorded the golden."""
    from lora_b200.arena import LrSchedule
    arena = _two_group_arena()
    if run == "dp_scaled":
        _as_world_one_dp(arena)
    scaled = run != "fused_world2"
    state = {"gnorm": lambda: arena.gnorm, "step": lambda: arena.step_dev}
    if scaled:
        arena.enable_loss_scaling(init_scale=2.0 ** 14, growth_interval=2)
        state.update(loss_scale=lambda: arena.loss_scale, growth_tracker=lambda: arena._growth_tracker,
                     found_inf=lambda: arena._found_inf, applied=lambda: arena.applied_steps)
    arena.p.copy_(inputs["p0"].to(DEV))
    arena.refresh_shadows()
    trace = {k: [] for k in state}
    for k, g in enumerate(inputs["scaled" if scaled else "unscaled"]):
        arena.g.copy_(g.to(DEV))
        if scaled:
            assert float(arena.loss_scale) == PATHS_SCALES[k], (run, k)
            arena.step(0.9, 0.999, 1e-8, 1e-2, 1.0, world_size=1, schedule=LrSchedule("linear", 2, 10, (0, 1)))
        else:
            arena.step(0.9, 0.999, 1e-8, 1e-2, 1.0, world_size=2)
        for name, get in state.items():
            trace[name].append(get().clone())
    torch.cuda.synchronize()
    out = {name: torch.cat(ts).cpu() for name, ts in trace.items()}
    out.update(p=arena.p.cpu(), m=arena.m.cpu(), v=arena.v.cpu(), shadow=arena.shadow.cpu())
    return out


def _bits(t):
    return t.view({4: torch.int32, 2: torch.int16}[t.element_size()]) if t.is_floating_point() else t


def test_optimizer_paths_are_bit_identical_to_the_previous_release():
    """Both launches with loss scaling (skips, growth, the device schedule) and the unscaled launch at
    inv_world 0.5 keep the bits of the release before they shared one kernel. Bit patterns, not
    torch.equal: a skipped step's norm is NaN."""
    d = torch.load(os.path.join(GOLD, "optim_paths.pt"))
    for run in OPTIM_PATHS:
        got = optim_paths_run(run, d["inputs"])
        assert got.keys() == d[run].keys(), run
        for k, want in d[run].items():
            assert torch.equal(_bits(got[k]), _bits(want)), (run, k)


def test_scaler_state_dict_round_trips_grad_scaler_format():
    arena = _two_group_arena()
    arena.enable_loss_scaling(init_scale=1024.0, growth_interval=7)
    ts = torch.amp.GradScaler("cuda", init_scale=1024.0, growth_interval=7)
    ts.scale(torch.ones((), device=DEV))
    assert arena.scaler_state_dict() == ts.state_dict()
    ts2 = torch.amp.GradScaler("cuda")
    ts2.load_state_dict({**arena.scaler_state_dict(), "scale": 256.0, "_growth_tracker": 3})
    arena.load_scaler_state_dict(ts2.state_dict())
    assert float(arena.loss_scale) == 256.0 and int(arena._growth_tracker) == 3
    assert arena.scaler_state_dict()["growth_interval"] == 7


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_loss_epilogue_grad_scale(dtype):
    from lora_b200.step_ops import fused_masked_mse
    torch.manual_seed(1)
    B, C, H, W = 4, 4, 16, 24
    pred0 = torch.randn(B, C, H, W, device=DEV).to(dtype).contiguous(memory_format=torch.channels_last)
    target = torch.randn(B, C, H, W, device=DEV)
    w = torch.tensor([0.5, 0.5, 0.35, 0.35], device=DEV)

    def run(scale):
        p = pred0.clone().requires_grad_(True)
        loss = fused_masked_mse(p, target, None, w, grad_scale=scale)
        loss.backward()
        return loss.detach(), p.grad

    l0, g0 = run(None)
    l1, g1 = run(torch.tensor([1024.0], device=DEV))
    assert torch.equal(l0, l1)
    # exact wherever the unscaled gradient is a normal number of pred's dtype (an fp16 subnormal has
    # lost bits the scaled one keeps: that is what the scale is for)
    normal = g0.abs() >= torch.finfo(dtype).tiny
    assert normal.float().mean() > 0.5
    assert torch.equal(g1[normal], g0[normal] * 1024)
    if dtype != torch.float16:
        return
    # a scale that overflows fp16: inf exactly where torch's fp16 backward of (loss * scale) has one
    big = torch.tensor([2.0 ** 32], device=DEV)
    l2, g2 = run(big)
    p = pred0.clone().requires_grad_(True)
    a, b = p.float(), target
    ref = sum(w[i] * torch.nn.functional.mse_loss(a[i], b[i]) for i in range(B))
    (ref * big).backward()
    assert torch.equal(l2, l0)
    assert torch.isinf(p.grad).any() and not torch.isinf(p.grad).all()
    assert torch.equal(torch.isinf(g2), torch.isinf(p.grad))
    fin = torch.isfinite(p.grad)
    assert rel(g2[fin].float(), p.grad[fin].float()) < 1e-3


# ------------------------------------------------------------------------------ whole steps
def _tiny_pair(seed=0, batch=1):
    import lora_b200 as L
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from oracle.ref_modules import ref_inject
    torch.manual_seed(seed)
    unet = UNet2DConditionModel(UNetConfig.tiny()).to(DEV)
    text = build_text_encoder(tiny=True).to(DEV)
    unet.requires_grad_(False)
    text.requires_grad_(False)
    unet_r, text_r = copy.deepcopy(unet), copy.deepcopy(text)
    L.inject_trainable_lora(unet, r=4)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=4)
    us = ref_inject(unet_r, {"CrossAttention", "Attention", "GEGLU"}, r=4)
    ts = ref_inject(text_r, {"CLIPAttention"}, r=4)
    ours = [m for m in list(unet.modules()) + list(text.modules()) if type(m).__name__ == "LoraInjectedLinear"]
    g = torch.Generator(device=DEV).manual_seed(3)
    for o, r in zip(ours, us + ts):
        o.lora_up.weight.data.normal_(0, 0.05, generator=g)
        r.up.data.copy_(o.lora_up.weight.data)
        r.down.data.copy_(o.lora_down.weight.data)
    return unet, text, unet_r, text_r, us, ts


def _batches(n, batch, seed=8, ids_hi=1000, tok=None):
    gi = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for _ in range(n):
        lat = torch.randn(batch, 4, 16, 16, device=DEV, generator=gi) * 0.18215
        ids = torch.randint(0, ids_hi, (batch, 77), device=DEV, generator=gi)
        if tok is not None:
            ids[0, 2], ids[-1, 5] = tok[0], tok[1]
        noise = torch.randn(batch, 4, 16, 16, device=DEV, generator=gi)
        t = torch.randint(0, 1000, (batch,), device=DEV, generator=gi)
        out.append((lat, ids, noise, t))
    return out


# 2^50 and 2^32 overflow the fp16 backward for certain; then 2^14, growing every growth_interval = 2
# applied steps to 2^17, stays far (about 2^5) below the scale at which these steps overflow: two
# skipped steps, then growth, with no overflow decided by a rounding difference
SCALER = dict(init_scale=2.0 ** 50, backoff_factor=2.0 ** -18, growth_interval=2)
EXPECTED_SKIPS = [True, True, False, False, False, False, False, False]


def _fp16_cfg(**kw):
    from lora_b200.train import StepConfig
    return StepConfig(autocast_dtype=torch.float16, compute_dtype=torch.float16, grad_scaler=True,
                      external_noise=True, lr_scheduler="linear", lr_warmup_steps=2, max_train_steps=10,
                      **SCALER, **kw)


@pytest.mark.parametrize("variant", ["eager", "graph", "unfused", "prior"])
def test_fp16_step_matches_oracle_grad_scaler_step(variant):
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.train import LoraTrainStep
    from oracle.amp_ref import RefAmpDreamboothStep
    prior = variant == "prior"
    batch = 2 if prior else 1
    unet, text, unet_r, text_r, us, ts = _tiny_pair()
    cfg = _fp16_cfg(use_cuda_graph=variant == "graph", fused_glue=variant != "unfused",
                    with_prior_preservation=prior, prior_loss_weight=0.7)
    tr = LoraTrainStep(unet, text, cfg, latent_shape=(batch, 4, 16, 16), device=DEV)
    ref = RefAmpDreamboothStep(unet_r, text_r, DDPMNoiser(device=DEV), us, ts, _warmup_linear(2, 10), **SCALER)
    if variant == "graph":
        tr.prepare()
        assert tr.graph is not None and tr.graph_update is None, tr.graph_error
    p0 = tr.arena.p[:tr.arena.n_params].clone()
    r0 = torch.cat([p.detach().flatten() for p in ref.unet_params + ref.text_params]).clone()
    skips, scales = [], []
    for k, (lat, ids, noise, t) in enumerate(_batches(8, batch)):
        kw = {"prior_loss_weight": 0.7} if prior else {}
        l_ref = float(ref.step(lat, ids, noise, t, **kw))
        tr.latents.copy_(lat); tr.input_ids.copy_(ids); tr.noise.copy_(noise); tr.timesteps.copy_(t)
        before = tr.arena.p.clone()
        l_ours = float(tr.step_device())
        torch.cuda.synchronize()
        assert abs(l_ours - l_ref) < 1e-2 * abs(l_ref), (k, l_ours, l_ref)
        skips.append(tr.arena.step_was_skipped())
        scales.append(float(tr.arena.loss_scale))
        if skips[-1]:
            assert torch.equal(tr.arena.p, before), k
    assert skips == ref.skipped == EXPECTED_SKIPS, (skips, ref.skipped)
    assert scales == ref.scales, (scales, ref.scales)
    assert int(tr.arena.applied_steps) == int(tr.arena.step_dev) == 6
    # the factors moved the same way (Adam's first steps are ~lr * sign(g): compare the updates)
    ours = [tr.arena.p[o:o + n] for _, _, _, o, n in tr.arena.entries]
    d_ours = torch.cat([x.flatten() for x in ours]) - torch.cat(
        [p0[o:o + n] for _, _, _, o, n in tr.arena.entries])
    d_ref = torch.cat([p.detach().flatten() for p in ref.unet_params + ref.text_params]) - r0
    cos = float((d_ours.double() * d_ref.double()).sum() / (d_ours.double().norm() * d_ref.double().norm()))
    assert cos > 0.95, cos
    assert abs(float(d_ours.norm()) / float(d_ref.norm()) - 1.0) < 0.1


def test_fp16_placeholders_embedding_step_matches_oracle():
    """train_lora_w_ti.py under fp16: two skipped steps, then two table steps before unfreeze_lora_step
    = 4 and two LoRA steps after it. The table's LambdaLR follows the applied steps only (lambda(0),
    lambda(1) -- not lambda(2), lambda(3) of the iteration count: 25 % apart), the LoRA groups are
    unscheduled. Each clean step's row update and the LoRA factors' update after unfreeze match the
    oracle in direction and size. On a skipped step the placeholder rows and every other row are
    unchanged."""
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.train import LoraEmbeddingStep, StepConfig
    from oracle.amp_ref import RefAmpJointStep
    unet, text, unet_r, text_r, us, ts = _tiny_pair(seed=1)
    emb = text.get_input_embeddings()
    V = emb.weight.shape[0]
    tok = [V - 2, V - 1]
    lr, lr_text, lr_ti, wd = 1e-4, 5e-5, 5e-4, 1e-2
    cfg = StepConfig(use_cuda_graph=False, autocast_dtype=torch.float16, compute_dtype=torch.float16,
                     grad_scaler=True, lr_scheduler="linear", max_train_steps=8, learning_rate=lr,
                     learning_rate_text=lr_text, adam_weight_decay=wd, external_noise=True, **SCALER)
    eng = LoraEmbeddingStep(unet, text, tok, cfg, lr_embedding=lr_ti, mode="placeholders", unfreeze_lora_step=4,
                            latent_shape=(2, 4, 16, 16))
    ref = RefAmpJointStep(unet_r, text_r, DDPMNoiser(device=DEV), us, ts, "placeholders", lr=lr, lr_text=lr_text,
                          lr_embedding=lr_ti, lr_lambda=lambda k: max(0.0, 1.0 - k / 8), weight_decay=wd,
                          placeholder_token_ids=tok, unfreeze_lora_step=4, **SCALER)
    table0 = emb.weight.detach().clone()
    others = torch.ones(V, dtype=torch.bool, device=DEV)
    others[tok] = False
    rg = eng.arena.rows_group
    ref_factors = lambda: torch.cat([p.detach().flatten() for p in ref.unet_params + ref.text_params])  # noqa: E731
    our_factors = lambda: torch.cat([eng.arena.p[o:o + n] for *_, o, n in eng.arena.entries])         # noqa: E731

    def same_update(d_ours, d_ref, k):
        d_ours, d_ref = d_ours.double().flatten(), d_ref.double().flatten()
        cos = float((d_ours * d_ref).sum() / (d_ours.norm() * d_ref.norm()))
        ratio = float(d_ours.norm() / d_ref.norm())
        assert cos > 0.95 and abs(ratio - 1.0) < 0.1, (k, cos, ratio)

    for k, (lat, ids, noise, t) in enumerate(_batches(6, 2, seed=9, ids_hi=60, tok=tok)):
        f0 = eng.arena.p[: eng.arena.group_off[rg]].clone()
        rows0 = emb.weight.detach()[tok].clone()
        ref_rows0 = ref.table.detach()[tok].clone()
        if k == 4:
            f_unfreeze, r_unfreeze = our_factors().clone(), ref_factors().clone()
        l_ref = float(ref.step(lat, ids, noise, t))
        eng.latents.copy_(lat); eng.input_ids.copy_(ids); eng.noise.copy_(noise); eng.timesteps.copy_(t)
        l_ours = float(eng.step_device())
        torch.cuda.synchronize()
        assert abs(l_ours - l_ref) < 1e-2 * abs(l_ref), (k, l_ours, l_ref)
        skipped = eng.arena.step_was_skipped()
        assert skipped == ref.skipped[-1] == (k < 2), k
        assert float(eng.arena.loss_scale) == ref.scales[-1], k
        f1, rows1 = eng.arena.p[: eng.arena.group_off[rg]], emb.weight.detach()[tok]
        assert torch.equal(emb.weight.detach()[others], table0[others]), k
        if skipped:
            assert torch.equal(rows1, rows0) and torch.equal(f1, f0), k
        elif k < 4:
            assert torch.equal(f1, f0) and not torch.equal(rows1, rows0), k
            same_update(rows1 - rows0, ref.table.detach()[tok] - ref_rows0, k)      # this step's lr
        else:
            assert torch.equal(rows1, rows0) and not torch.equal(f1, f0), k
        want = ref.table.detach()[tok].double()
        assert float((rows1.double() - want).norm() / want.norm()) < 2e-2, k
    # the LoRA groups after unfreeze: base lrs, not scaled by the table's schedule
    same_update(our_factors() - f_unfreeze, ref_factors() - r_unfreeze, "lora")
    eng.release()


def test_prepare_leaves_scaler_state_and_launch_count_matches_bf16():
    from lora_b200 import ops
    from lora_b200.train import LoraTrainStep, StepConfig
    unet, text, *_ = _tiny_pair()
    tr = LoraTrainStep(unet, text, _fp16_cfg(), latent_shape=(1, 4, 16, 16), device=DEV)
    a = tr.arena
    state = [t.clone() for t in (a.loss_scale, a._growth_tracker, a._found_inf, a.applied_steps, a.step_dev, a.p)]
    tr.prepare()
    assert tr.graph is not None and tr.graph_update is None, tr.graph_error
    for before, now in zip(state, (a.loss_scale, a._growth_tracker, a._found_inf, a.applied_steps, a.step_dev, a.p)):
        assert torch.equal(before, now)
    counts = {}
    for name in ("fp16", "bf16"):
        u, t_, *_ = _tiny_pair()
        cfg = _fp16_cfg(use_cuda_graph=False) if name == "fp16" else \
            StepConfig(use_cuda_graph=False, autocast_dtype=torch.bfloat16, external_noise=True)
        st = LoraTrainStep(u, t_, cfg, latent_shape=(1, 4, 16, 16), device=DEV)
        st._body()
        ops.LAUNCH_COUNT = 0
        st._body()
        counts[name] = ops.LAUNCH_COUNT
    assert counts["fp16"] == counts["bf16"] > 0, counts
