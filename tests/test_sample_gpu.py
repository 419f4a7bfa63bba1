"""Sampling on the GPU (lora_b200/sample.py): lb_sample_step against a float64 evaluation of the same
linear form, lb_pixels_emit against torch's post-processing bit for bit, and the sampler -- graph
replay against its eager path and both against the pipeline-style oracle loop (oracle/sample_ref.py)
-- on tiny and full-size models, with scale changes, re-patching and training steps in between.

Oracle bound: the sampler's error against the oracle's float64 run is at most twice the oracle's own
error in the run's dtype (bf16 autocast) against that float64 run, measured on the final latents."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _bits(t):
    t = t.detach().cpu().contiguous()
    return t.view({4: torch.int32, 2: torch.int16, 1: torch.uint8}[t.element_size()])


# ------------------------------------------------------------------------------------ kernels
def _table(rows, g):
    tab = torch.zeros(rows, 8)
    tab[0, :3] = torch.tensor([14.6, 0.068, 999.0])
    tab[1:, 0] = 1 + torch.rand(rows - 1, generator=g) * 0.1
    tab[1:, 1] = -torch.rand(rows - 1, generator=g)
    tab[1:, 2] = torch.rand(rows - 1, generator=g)
    tab[1:, 3] = torch.rand(rows - 1, generator=g)
    tab[1:, 4] = torch.arange(rows - 1, 0, -1).float() * 7.5
    tab[rows - 1, 5] = 1.0
    return tab


@pytest.mark.parametrize("mdt", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("channels_last", [True, False])
@pytest.mark.parametrize("G", [1, 2])
@pytest.mark.parametrize("with_noise", [True, False])
def test_sample_step_matches_float64(mdt, channels_last, G, with_noise):
    from lora_b200.step_ops import sample_step
    g = torch.Generator().manual_seed(G + 2 * int(channels_last))
    B, C, H, W = 3, 4, 12, 20
    rows = 4
    tab = _table(rows, g)
    if not with_noise:
        tab[1:, 2] = 0.0
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    mo = (torch.randn(G * B, C, H, W, generator=g) * 2).to(mdt).to(DEV).contiguous(memory_format=fmt)
    noise = torch.randn(rows, B, C, H, W, generator=g).to(DEV)
    x0 = (torch.randn(B, C, H, W, generator=g) * 3).to(DEV)
    x = x0.clone()
    gs = torch.tensor([7.0], device=DEV)
    idx, cnt = torch.zeros(1, device=DEV, dtype=torch.int32), torch.zeros(1, device=DEV, dtype=torch.int32)
    ts = torch.zeros(1, device=DEV)
    unet_in = torch.zeros(G * B, C, H, W, device=DEV, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    vae_in = torch.full((B, C, H, W), float("nan"), device=DEV, dtype=torch.float16)
    tab_d = tab.to(DEV)
    idx.fill_(1)                                 # step 1 of 0..2 (row 2): not the last
    sample_step(mo, x, noise, tab_d, gs, idx, cnt, unet_in, ts, vae_in, 0.18215)
    torch.cuda.synchronize()
    row = tab[2].double()
    m = mo.double().cpu()
    m_hat = m[:B] if G == 1 else m[:B] + 7.0 * (m[B:] - m[:B])
    z = noise[2].double().cpu()
    xd = x0.double().cpu()
    want = row[0] * xd + row[1] * m_hat + row[2] * z
    bound = (row[0] * xd).abs() + row[1].abs() * (m[:B].abs() + (7.0 * (m[B:] - m[:B]).abs() if G == 2 else 0)) \
        + (row[2] * z).abs()
    err = (x.double().cpu() - want).abs()
    assert bool((err <= 4 * 2 ** -23 * bound + 1e-30).all()), float((err / bound).max())
    s_next = float(tab[2, 3])
    want_in = (s_next * x).to(torch.bfloat16)
    for h in range(G):
        assert torch.equal(_bits(unet_in[h * B:(h + 1) * B]), _bits(want_in))
    assert float(ts) == float(tab[2, 4]) and int(idx) == 2 and int(cnt) == 0
    assert bool(torch.isnan(vae_in.float()).all())          # not the last step: the decoder input is untouched
    # the last step writes the pipeline's 1 / scaling * x to the decoder input
    sample_step(mo, x, noise, tab_d, gs, idx, cnt, unet_in, ts, vae_in, 0.18215)
    torch.cuda.synchronize()
    assert torch.equal(_bits(vae_in), _bits((1 / 0.18215 * x).to(torch.float16)))


def test_sample_step_replays_one_captured_launch_as_every_step():
    from lora_b200.step_ops import sample_step
    g = torch.Generator().manual_seed(0)
    B, C, H, W = 2, 4, 16, 16
    N = 6
    rows = N + 1
    tab = _table(rows, g).to(DEV)
    noise = torch.randn(rows, B, C, H, W, generator=g).to(DEV)
    mo = torch.randn(2 * B, C, H, W, generator=g).to(DEV)
    x = torch.zeros(B, C, H, W, device=DEV)
    gs = torch.tensor([3.0], device=DEV)
    idx, cnt = torch.zeros(1, device=DEV, dtype=torch.int32), torch.zeros(1, device=DEV, dtype=torch.int32)
    ts = torch.zeros(1, device=DEV)
    unet_in = torch.zeros(2 * B, C, H, W, device=DEV).contiguous(memory_format=torch.channels_last)
    vae_in = torch.zeros(B, C, H, W, device=DEV)
    args = (x, noise, tab, gs, idx, cnt, unet_in, ts, vae_in, 0.18215)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        sample_step(None, *args, init=True)
        sample_step(mo, *args)
    torch.cuda.current_stream().wait_stream(s)
    ga, gb = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.graph(ga):
        sample_step(None, *args, init=True)
    with torch.cuda.graph(gb):
        sample_step(mo, *args)
    idx.fill_(5)
    ga.replay()
    torch.cuda.synchronize()
    t = tab.double().cpu()
    xd = noise[0].double().cpu() * t[0, 0]
    assert int(idx) == 0 and float(ts) == float(t[0, 2])
    m = mo.double().cpu()
    m_hat = m[:B] + 3.0 * (m[B:] - m[:B])
    for i in range(N):
        gb.replay()
        torch.cuda.synchronize()
        r = t[1 + i]
        xd = r[0] * xd + r[1] * m_hat + r[2] * noise[1 + i].double().cpu()
        assert int(idx) == i + 1 and float(ts) == float(r[4])
        assert _rel(x, xd) < 1e-5, i
    assert torch.equal(vae_in, 1 / 0.18215 * x)


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("channels_last", [True, False])
def test_pixels_emit_is_torch_post_processing_bit_for_bit(dt, channels_last):
    from lora_b200.step_ops import pixels_emit
    from oracle.sample_ref import postprocess
    g = torch.Generator().manual_seed(1)
    img = torch.randn(2, 3, 24, 40, generator=g) * 1.2
    img[0, 0, 0, :8] = torch.tensor([-1.0, 1.0, 0.0, -1.5, 1.5, 1 / 255 - 1, 3 / 255 - 1, 5 / 255 - 1])
    img = img.to(dt).to(DEV).contiguous(memory_format=torch.channels_last if channels_last else torch.contiguous_format)
    out = torch.empty(2, 24, 40, 3, device=DEV, dtype=torch.uint8)
    pixels_emit(img, out)
    assert torch.equal(out, postprocess(img))


# ------------------------------------------------------------------------------------ tiny models
def _models(seed=0, up_std=0.05):
    """(unet, text, vae, ref unet, ref text): tiny host models with the same non-zero LoRA factors as
    engine modules and as the oracle's reference modules."""
    import lora_b200 as L
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    from oracle.ref_modules import ref_inject
    torch.manual_seed(seed)
    unet = UNet2DConditionModel(UNetConfig.tiny()).to(DEV).to(memory_format=torch.channels_last)
    text = build_text_encoder(tiny=True).to(DEV)
    vae = AutoencoderKL(VAEConfig.tiny(), with_decoder=True).to(DEV).to(memory_format=torch.channels_last)
    for m in (unet, text, vae):
        m.requires_grad_(False)
    unet_r, text_r = copy.deepcopy(unet), copy.deepcopy(text)
    L.inject_trainable_lora(unet, r=4)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=4)
    us = ref_inject(unet_r, {"CrossAttention", "Attention", "GEGLU"}, r=4)
    ts = ref_inject(text_r, {"CLIPAttention"}, r=4)
    ours = [m for m in list(unet.modules()) + list(text.modules()) if type(m).__name__ == "LoraInjectedLinear"]
    assert len(ours) == len(us) + len(ts)
    g = torch.Generator(device=DEV).manual_seed(3)
    for o, rs in zip(ours, us + ts):
        o.lora_up.weight.data.normal_(0, up_std, generator=g)
        rs.up.data.copy_(o.lora_up.weight.data)
        rs.down.data.copy_(o.lora_down.weight.data)
    return unet, text, vae, unet_r, text_r


LAT = (2, 4, 8, 8)


def _ids(text, seed=4):
    g = torch.Generator().manual_seed(seed)
    v = text.config.vocab_size
    return torch.randint(0, v, (LAT[0], 77), generator=g).to(DEV), torch.randint(0, v, (LAT[0], 77), generator=g).to(DEV)


def _sampler(unet, text, vae, graph, **kw):
    from lora_b200.sample import LoraSampler, SamplerConfig
    base = dict(num_inference_steps=10, max_steps=12, guidance_scale=7.0, autocast_dtype=torch.bfloat16,
                use_cuda_graph=graph)
    base.update(kw)
    return LoraSampler(unet, text, vae, SamplerConfig(**base), latent_shape=LAT, seq_len=77, device=DEV)


@pytest.mark.parametrize("scheduler", ["euler_ancestral", "ddim"])
@pytest.mark.parametrize("prediction_type", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("grouping", [False, True])
def test_tiny_graph_equals_eager_and_oracle(scheduler, prediction_type, grouping):
    import lora_b200 as L
    from oracle import sample_ref as R
    unet, text, vae, unet_r, text_r = _models()
    ids, neg = _ids(text)
    L.set_grouping(grouping)
    try:
        kw = dict(scheduler=scheduler, prediction_type=prediction_type, external_noise=True)
        sg, se = _sampler(unet, text, vae, True, **kw), _sampler(unet, text, vae, False, **kw)
        g = torch.Generator(device=DEV).manual_seed(11)
        noise = torch.randn(sg.noise.shape, device=DEV, generator=g)
        sg.noise.copy_(noise)
        se.noise.copy_(noise)
        sg.prepare()
        img_g = sg.sample(ids, neg).clone()
        img_e = se.sample(ids, neg).clone()
        assert sg.captures == 1
        assert torch.equal(img_g, img_e) and torch.equal(sg.latents, se.latents)
        n = 10
        args = (ids, neg, noise[:n + 1], 7.0)
        f64 = [copy.deepcopy(m).double() for m in (unet_r, text_r, vae)]
        _, lat64 = R.sample(*f64[:2], f64[2], R.make_scheduler(scheduler, prediction_type), n, *args,
                            dtype=torch.float64)
        _, lat_run = R.sample(unet_r, text_r, vae, R.make_scheduler(scheduler, prediction_type), n, *args,
                              dtype=torch.float32, autocast_dtype=torch.bfloat16)
        e_ours, e_ref = _rel(sg.latents, lat64), _rel(lat_run, lat64)
        assert e_ours <= 2 * e_ref, (e_ours, e_ref)
    finally:
        L.set_grouping(False)


def test_per_call_options_do_not_recapture_and_g1_is_its_own_capture():
    unet, text, vae, *_ = _models()
    ids, neg = _ids(text)
    s, e = _sampler(unet, text, vae, True), _sampler(unet, text, vae, False)
    for kw in (dict(seed=1), dict(seed=2, num_inference_steps=5), dict(scheduler="ddim", num_inference_steps=12),
               dict(guidance_scale=3.0, seed=3)):
        a = s.sample(ids, neg, **kw).clone()
        assert torch.equal(a, e.sample(ids, neg, **kw)), kw
    assert s.captures == 1
    a = s.sample(ids, None, guidance_scale=1.0, seed=4).clone()
    assert torch.equal(a, e.sample(ids, None, guidance_scale=1.0, seed=4))
    assert s.captures == 2
    s.sample(ids, neg, seed=5)
    assert s.captures == 2
    # the same seed gives the same image; the global CUDA RNG stream is untouched
    st = torch.cuda.get_rng_state()
    a = s.sample(ids, neg, seed=9).clone()
    assert torch.equal(a, s.sample(ids, neg, seed=9)) and torch.equal(st, torch.cuda.get_rng_state())


def test_tune_scale_recaptures_once_and_scale_zero_is_no_lora():
    import lora_b200 as L
    from oracle import sample_ref as R
    unet, text, vae, unet_r, text_r = _models()
    ids, neg = _ids(text)
    s = _sampler(unet, text, vae, True)
    s.sample(ids, neg, seed=0)
    L.tune_lora_scale(unet, 0.5)
    L.tune_lora_scale(text, 0.5)
    a = s.sample(ids, neg, seed=0).clone()
    la = s.latents.clone()
    s.sample(ids, neg, seed=0)
    assert s.captures == 2
    fresh = _sampler(unet, text, vae, True)
    assert torch.equal(a, fresh.sample(ids, neg, seed=0)) and torch.equal(la, fresh.latents)
    # scale 0 and the same models with the LoRA removed (the frozen GEMM then runs through another
    # library, so not bit for bit): both within the suite's bound of the float64 oracle without LoRA
    L.tune_lora_scale(unet, 0.0)
    L.tune_lora_scale(text, 0.0)
    s.sample(ids, neg, seed=0)
    l0 = s.latents.clone()
    assert s.captures == 3
    u2, t2 = copy.deepcopy(unet), copy.deepcopy(text)
    L.monkeypatch_remove_lora(u2)
    L.monkeypatch_remove_lora(t2)
    plain = _sampler(u2, t2, vae, True)
    plain.sample(ids, neg, seed=0)
    for m in list(unet_r.modules()) + list(text_r.modules()):
        if type(m).__name__ == "RefLoraSite":
            m.scale = 0.0
    noise = plain.noise[:11].clone()
    f64 = [copy.deepcopy(m).double() for m in (unet_r, text_r, vae)]
    _, lat64 = R.sample(*f64, R.make_scheduler("euler_ancestral", "epsilon"), 10, ids, neg, noise, 7.0)
    _, lat_run = R.sample(unet_r, text_r, vae, R.make_scheduler("euler_ancestral", "epsilon"), 10, ids, neg, noise,
                          7.0, dtype=torch.float32, autocast_dtype=torch.bfloat16)
    e_ref = _rel(lat_run, lat64)
    assert _rel(l0, lat64) <= 2 * e_ref and _rel(plain.latents, lat64) <= 2 * e_ref


def test_patching_new_factors_recaptures_and_samples_them(tmp_path):
    import lora_b200 as L
    unet, text, vae, *_ = _models()
    other, _, _, *_ = _models(seed=1, up_std=0.2)
    ids, neg = _ids(text)
    s = _sampler(unet, text, vae, True)
    s.sample(ids, neg, seed=0)
    path = str(tmp_path / "other.safetensors")
    L.save_safeloras({"unet": (other, L.DEFAULT_TARGET_REPLACE)}, path)
    from safetensors.torch import safe_open
    import types
    L.monkeypatch_or_replace_safeloras(types.SimpleNamespace(unet=unet), safe_open(path, framework="pt", device="cpu"))
    unet.to(DEV)
    s.sample(ids, neg, seed=0)
    got = s.latents.clone()
    assert s.captures == 2
    fresh = _sampler(unet, text, vae, False)
    fresh.sample(ids, neg, seed=0)
    assert torch.equal(got, fresh.latents)


# ------------------------------------------------------------------------------------ with training
def _train(unet, text, K, sampler_fn=None):
    from lora_b200.train import LoraTrainStep, StepConfig
    cfg = StepConfig(use_cuda_graph=True, graph_warmup=2, autocast_dtype=torch.bfloat16)
    tr = LoraTrainStep(unet, text, cfg, latent_shape=LAT, seq_len=77, device=DEV)
    torch.manual_seed(21)
    tr.latents.copy_(torch.randn(LAT, device=DEV) * 0.18215)
    tr.input_ids.copy_(torch.randint(0, text.config.vocab_size, (LAT[0], 77), device=DEV))
    tr.prepare()
    losses = []
    for _ in range(K):
        losses.append(tr.step_device().clone())
        if sampler_fn is not None:
            sampler_fn()
    return tr, torch.stack(losses)


def test_sampling_between_training_steps_changes_nothing():
    unet, text, vae, *_ = _models()
    u2, t2 = copy.deepcopy(unet), copy.deepcopy(text)
    ids, neg = _ids(text)
    s = _sampler(unet, text, vae, True)
    imgs = []
    tr, losses = _train(unet, text, 3, lambda: imgs.append(s.sample(ids, neg, seed=0).clone()))
    u4, t4 = copy.deepcopy(u2), copy.deepcopy(t2)
    tr2, losses2 = _train(u2, t2, 3)
    assert torch.equal(_bits(losses), _bits(losses2))
    # a second run without sampling: the factors of two plain runs are the yardstick
    tr4, _ = _train(u4, t4, 3)
    if torch.equal(tr2.arena.p, tr4.arena.p):
        assert torch.equal(tr.arena.p, tr2.arena.p)
    else:
        assert _rel(tr.arena.p, tr2.arena.p) <= 10 * _rel(tr4.arena.p, tr2.arena.p)
    assert s.captures == 1
    u3, t3 = copy.deepcopy(unet), copy.deepcopy(text)
    import lora_b200 as L
    L.link_sites(u3, t3)
    fresh = _sampler(u3, t3, vae, False)
    fresh.sample(ids, neg, seed=0)
    last = s.latents.clone()
    assert torch.equal(imgs[-1], fresh.image) and torch.equal(last, fresh.latents)
    assert unet.training and text.training          # the step's modes are restored


def test_in_place_optimizer_updates_and_data_edits_are_sampled():
    unet, text, vae, *_ = _models()
    ids, neg = _ids(text)
    s = _sampler(unet, text, vae, True)
    s.sample(ids, neg, seed=0)
    params = [p for m in (unet, text) for n, p in m.named_parameters() if "lora_" in n]
    for p in params:
        p.requires_grad_(True)
    opt = torch.optim.AdamW(params, lr=1e-2)
    for p in params:
        p.grad = torch.randn_like(p)
    opt.step()
    for m in list(unet.modules()):
        if type(m).__name__ == "LoraInjectedLinear":
            m.lora_down.weight.data.mul_(1.5)          # no version bump, no new storage
    s.sample(ids, neg, seed=0)
    got = s.latents.clone()
    assert s.captures == 1
    import lora_b200 as L
    u3, t3 = copy.deepcopy(unet), copy.deepcopy(text)
    L.link_sites(u3, t3)
    fresh = _sampler(u3, t3, vae, False)
    fresh.sample(ids, neg, seed=0)
    assert torch.equal(got, fresh.latents)


def test_launches_per_denoising_step_are_the_unet_forward_plus_one():
    from lora_b200 import ops
    unet, text, vae, *_ = _models()
    ids, neg = _ids(text)
    s = _sampler(unet, text, vae, False)
    s.sample(ids, neg, seed=0)
    unet.eval()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        c0 = ops.LAUNCH_COUNT
        unet(s.unet_in[2], s.timestep, s._ehs[2])
        fwd = ops.LAUNCH_COUNT - c0
        c0 = ops.LAUNCH_COUNT
        s._body_b(2)
        step = ops.LAUNCH_COUNT - c0
    unet.train()
    assert fwd > 0 and step == fwd + 1


# ------------------------------------------------------------------------------------ full size
def _full(unet_cfg, sd2):
    import lora_b200 as L
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    from oracle.ref_modules import ref_inject
    torch.manual_seed(0)
    with torch.device(DEV):
        unet = UNet2DConditionModel(unet_cfg)
        text = build_text_encoder(sd2=sd2)
        vae = AutoencoderKL(VAEConfig.sd(), with_decoder=True)
    for m in (unet, text, vae):
        m.requires_grad_(False)
    unet = unet.to(memory_format=torch.channels_last)
    vae = vae.to(torch.bfloat16).to(memory_format=torch.channels_last)
    unet_r, text_r = copy.deepcopy(unet), copy.deepcopy(text)
    L.inject_trainable_lora(unet, r=4)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=4)
    us = ref_inject(unet_r, {"CrossAttention", "Attention", "GEGLU"}, r=4)
    ts = ref_inject(text_r, {"CLIPAttention"}, r=4)
    ours = [m for m in list(unet.modules()) + list(text.modules()) if type(m).__name__ == "LoraInjectedLinear"]
    g = torch.Generator(device=DEV).manual_seed(3)
    for o, rs in zip(ours, us + ts):
        o.lora_up.weight.data.normal_(0, 0.02, generator=g)
        rs.up.data.copy_(o.lora_up.weight.data)
        rs.down.data.copy_(o.lora_down.weight.data)
    return unet, text, vae, unet_r, text_r


@pytest.mark.parametrize("which", ["sd15_512_euler_50", "sd21_768v_ddim_20"])
def test_full_size_graph_equals_eager_and_oracle(which):
    import lora_b200 as L
    from lora_b200.host.unet_sd15 import UNetConfig
    from lora_b200.sample import LoraSampler, SamplerConfig
    from oracle import sample_ref as R
    if which.startswith("sd15"):
        ucfg, sd2, lat, sched, pred, n = UNetConfig(), False, (1, 4, 64, 64), "euler_ancestral", "epsilon", 50
    else:
        ucfg, sd2, lat, sched, pred, n = UNetConfig.sd21(), True, (1, 4, 96, 96), "ddim", "v_prediction", 20
    unet, text, vae, unet_r, text_r = _full(ucfg, sd2)
    L.set_grouping(True)
    try:
        cfg = dict(scheduler=sched, prediction_type=pred, num_inference_steps=n, max_steps=n, guidance_scale=7.0,
                   autocast_dtype=torch.bfloat16, external_noise=True)
        sg = LoraSampler(unet, text, vae, SamplerConfig(**cfg), latent_shape=lat, device=DEV)
        se = LoraSampler(unet, text, vae, SamplerConfig(use_cuda_graph=False, **cfg), latent_shape=lat, device=DEV)
        g = torch.Generator(device=DEV).manual_seed(5)
        noise = torch.randn(sg.noise.shape, device=DEV, generator=g)
        sg.noise.copy_(noise)
        se.noise.copy_(noise)
        ids = torch.randint(0, text.config.vocab_size, (1, 77), device=DEV)
        neg = torch.randint(0, text.config.vocab_size, (1, 77), device=DEV)
        sg.prepare()
        img = sg.sample(ids, neg).clone()
        assert torch.equal(img, se.sample(ids, neg)) and torch.equal(sg.latents, se.latents)
        args = (ids, neg, noise, 7.0)
        _, lat_run = R.sample(unet_r, text_r, vae, R.make_scheduler(sched, pred), n, *args, dtype=torch.float32,
                              autocast_dtype=torch.bfloat16)
        f64 = [copy.deepcopy(m).double() for m in (unet_r, text_r)]
        vae64 = copy.deepcopy(vae).double()
        del unet_r, text_r
        _, lat64 = R.sample(f64[0], f64[1], vae64, R.make_scheduler(sched, pred), n, *args, dtype=torch.float64)
        e_ours, e_ref = _rel(sg.latents, lat64), _rel(lat_run, lat64)
        assert e_ours <= 2 * e_ref, (e_ours, e_ref)
    finally:
        L.set_grouping(False)
