"""StepConfig.gradient_checkpointing on the fused LoRA path: the same arena state, noise draws and
dropout seed pool give the same step with and without checkpointing -- default sites, extended sites
with dropout p = 0.1, grouped launches, fp16 with a GradScaler and the embedding-table step, eager and
graph-replayed. Plus: a recomputed dropout site reads the seed slot of its first forward, the
drop-in path (no step engine) gets the same gradients, and the deferred weight-gradient queue does
not hold recomputed activations past their segment (peak memory at an SD1.5-shaped step)."""
import pytest
import torch
from torch.utils.checkpoint import checkpoint

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _models(seed, extended=False, full=False, batch=1):
    import lora_b200 as L
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    torch.manual_seed(seed)
    with torch.device(DEV):
        unet = UNet2DConditionModel(UNetConfig.sd15() if full else UNetConfig.tiny())
        text = build_text_encoder(tiny=not full)
    unet.requires_grad_(False)
    text.requires_grad_(False)
    if full:
        unet, text = unet.to(torch.bfloat16).to(memory_format=torch.channels_last), text.to(torch.bfloat16)
    if extended:
        L.inject_trainable_lora_extended(unet, r=4)          # operator default dropout p = 0.1
    else:
        L.inject_trainable_lora(unet, r=4)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=4)
    g = torch.Generator(device=DEV).manual_seed(seed + 3)
    for m in list(unet.modules()) + list(text.modules()):
        if type(m).__name__ in ("LoraInjectedLinear", "LoraInjectedConv2d"):
            m.lora_up.weight.data.normal_(0, 0.05, generator=g)
    return unet, text


def _batches(n, batch, hw=16, seed=8, ids_hi=1000, tok=None):
    gi = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for _ in range(n):
        lat = torch.randn(batch, 4, hw, hw, device=DEV, generator=gi) * 0.18215
        ids = torch.randint(0, ids_hi, (batch, 77), device=DEV, generator=gi)
        if tok is not None:
            ids[0, 2] = tok[0]
        noise = torch.randn(batch, 4, hw, hw, device=DEV, generator=gi)
        t = torch.randint(0, 1000, (batch,), device=DEV, generator=gi)
        out.append((lat, ids, noise, t))
    return out


CASES = ("default", "dropout", "grouping", "grad_scaler", "embedding_table")


def _run(case, graph, ckpt, n_steps=3):
    """n_steps of one engine; returns (losses, trained parameters before and after, embedding rows or None)."""
    import lora_b200 as L
    from lora_b200.train import LoraEmbeddingStep, LoraTrainStep, StepConfig
    L.set_grouping(case == "grouping")
    try:
        unet, text = _models(0, extended=case == "dropout")
        kw = dict(use_cuda_graph=graph, external_noise=True, gradient_checkpointing=ckpt)
        if case == "grad_scaler":
            kw.update(autocast_dtype=torch.float16, compute_dtype=torch.float16, grad_scaler=True, init_scale=1024.0)
        else:
            kw.update(autocast_dtype=torch.bfloat16)
        cfg = StepConfig(**kw)
        tok = None
        if case == "embedding_table":
            V = text.get_input_embeddings().weight.shape[0]
            tok = [V - 1]
            eng = LoraEmbeddingStep(unet, text, tok, cfg, lr_embedding=5e-4, mode="table", latent_shape=(2, 4, 16, 16))
        else:
            eng = LoraTrainStep(unet, text, cfg, latent_shape=(2, 4, 16, 16), device=DEV)
        torch.cuda.manual_seed(1234)                 # the dropout seed pool's draws
        if graph:
            eng.prepare()
            assert eng.graph is not None, eng.graph_error
        assert unet.is_gradient_checkpointing == ckpt
        p_init = eng.arena.p[:eng.arena.n_params].clone()
        losses = []
        for lat, ids, noise, t in _batches(n_steps, 2, ids_hi=60 if tok else 1000, tok=tok):
            eng.latents.copy_(lat); eng.input_ids.copy_(ids); eng.noise.copy_(noise); eng.timesteps.copy_(t)
            losses.append(eng.step_device().clone())
        torch.cuda.synchronize()
        rows = None
        if case == "embedding_table":
            eng.flush()
            rows = text.get_input_embeddings().weight.detach()[tok].clone()
        return torch.stack(losses), p_init, eng.arena.p[:eng.arena.n_params].clone(), rows
    finally:
        L.set_grouping(False)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("case", CASES)
def test_checkpointed_step_matches_plain_step(case, graph):
    """The dropout case is the regression test for masks drawn anew in the recompute: without
    per-site seed slots the recompute's keep-mask differs and dA / dB drift far past 1e-5."""
    l0, init0, p0, rows0 = _run(case, graph, ckpt=False)
    l1, init1, p1, rows1 = _run(case, graph, ckpt=True)
    assert torch.equal(init0, init1) and not torch.equal(p0, init0)      # same start, and the factors moved
    assert torch.isfinite(l0).all()
    # the first step runs identical forward kernels on identical inputs; later steps see factors that
    # differ by the atomics order of the weight-gradient reductions
    assert torch.equal(l0[0], l1[0]), (l0, l1)
    assert rel(l1, l0) < 1e-5, (l0, l1)
    assert rel(p1, p0) < 1e-5
    if rows0 is not None:
        assert rel(rows1, rows0) < 1e-5


def _dropout_site(p=0.5):
    import lora_b200 as L
    torch.manual_seed(0)
    site = L.LoraInjectedLinear(320, 640, bias=True, r=4, dropout_p=p).to(DEV)
    site.linear.requires_grad_(False)
    site.lora_up.weight.data.normal_(0, 0.05)
    return site


def _grads(site, x, gy, ckpt):
    xi = x.clone().requires_grad_(True)
    for w in (site.lora_down.weight, site.lora_up.weight):
        w.grad = None
    y = checkpoint(site, xi, use_reentrant=False) if ckpt else site(xi)
    y.backward(gy)
    return y.detach(), xi.grad, site.lora_down.weight.grad.clone(), site.lora_up.weight.grad.clone()


def test_recomputed_dropout_site_reads_its_first_seed_slot(monkeypatch):
    from lora_b200 import dropout_path, ops
    site = _dropout_site()
    x = torch.randn(2, 300, 320, device=DEV, dtype=torch.bfloat16)
    gy = torch.randn(2, 300, 640, device=DEV, dtype=torch.bfloat16)
    seen = []
    real_fwd, real_dt = ops.fused_linear, ops.dropout_dt

    def fwd(*a, seed=None, **kw):
        if seed is not None:
            seen.append(("fwd", seed.data_ptr()))
        return real_fwd(*a, seed=seed, **kw)

    def dt(gy2d, up, rs, cs, p, seed, r):
        seen.append(("bwd", seed.data_ptr()))
        return real_dt(gy2d, up, rs, cs, p, seed, r)

    monkeypatch.setattr(ops, "fused_linear", fwd)
    monkeypatch.setattr(ops, "dropout_dt", dt)
    out = []
    for ckpt in (False, True):
        torch.cuda.manual_seed(7)
        dropout_path.begin_step(x.device)
        pool = dropout_path._SeedPool.pool
        seen.clear()
        out.append(_grads(site, x, gy, ckpt))
        dropout_path.end_step()
        slot0 = pool[0:1].data_ptr()
        # forward, (recompute,) backward: all on slot 0 of the step's pool
        assert [k for k, _ in seen] == (["fwd", "fwd", "bwd"] if ckpt else ["fwd", "bwd"]), seen
        assert all(ptr == slot0 for _, ptr in seen), (seen, slot0)
    (y0, dx0, da0, db0), (y1, dx1, da1, db1) = out
    assert torch.equal(y0, y1) and torch.equal(dx0, dx1)
    assert rel(da1, da0) < 1e-5 and rel(db1, db0) < 1e-5


def test_drop_in_dropout_site_without_step_engine():
    """No seed pool (a caller's own loop, as the reference scripts run): the seed comes from torch's
    CUDA generator, whose state torch.utils.checkpoint restores before the recompute."""
    site = _dropout_site()
    x = torch.randn(2, 300, 320, device=DEV, dtype=torch.bfloat16)
    gy = torch.randn(2, 300, 640, device=DEV, dtype=torch.bfloat16)
    out = []
    for ckpt in (False, True):
        torch.cuda.manual_seed(11)
        out.append(_grads(site, x, gy, ckpt))
    (y0, dx0, da0, db0), (y1, dx1, da1, db1) = out
    assert torch.equal(y0, y1) and torch.equal(dx0, dx1)
    assert rel(da1, da0) < 1e-5 and rel(db1, db0) < 1e-5


def _peak_step_bytes(ckpt, hold_queue=False, batch=4):
    """Peak allocated bytes of one eager SD1.5-shaped step (bf16, 512 px, default sites r = 4) after
    a warm-up step. hold_queue: the deferred weight-gradient queue is flushed only at the end of the
    backward, as it would be without segment flushes."""
    from lora_b200 import ops
    from lora_b200.train import LoraTrainStep, StepConfig
    unet, text = _models(0, full=True)
    cfg = StepConfig(use_cuda_graph=False, external_noise=True, train_text_encoder=False,
                     gradient_checkpointing=ckpt)
    eng = LoraTrainStep(unet, text, cfg, latent_shape=(batch, 4, 64, 64), device=DEV)
    real = ops.wgrad_segment_boundary
    if hold_queue:
        ops.wgrad_segment_boundary = lambda: 0
    try:
        lat, ids, noise, t = _batches(1, batch, hw=64)[0]
        eng.latents.copy_(lat); eng.input_ids.copy_(ids); eng.noise.copy_(noise); eng.timesteps.copy_(t)
        eng.step_device()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        eng.step_device()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
    finally:
        ops.wgrad_segment_boundary = real
    del eng, unet, text
    torch.cuda.empty_cache()
    return peak


def test_checkpointing_lowers_peak_memory_and_the_queue_does_not_retain_recomputes():
    plain = _peak_step_bytes(False)
    ckpt = _peak_step_bytes(True)
    held = _peak_step_bytes(True, hold_queue=True)
    print(f"step peak above resident state: plain {plain / 2**20:.0f} MiB, checkpointed {ckpt / 2**20:.0f} MiB, "
          f"checkpointed with the queue held to the end {held / 2**20:.0f} MiB")
    # measured on an H100 80GB HBM3 at a 700 W power limit (SD1.5, bs 4, 512 px): 3415, 696 and 1972 MiB,
    # ratios 0.20 and 0.35
    assert ckpt < 0.3 * plain, (plain, ckpt)
    assert ckpt < 0.5 * held, (ckpt, held)
