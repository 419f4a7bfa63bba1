"""img2img and inpainting sampling on the GPU: lb_sample_init and lb_pixels_ingest_inpaint against torch's
op-by-op evaluation bit for bit, lb_sample_step_ch against lb_sample_step, and the img2img / inpaint
samplers -- graph replay against the eager path and both against the pipeline-style oracle loops
(oracle/sample_image_ref.py) -- on tiny and full-size models, with per-call changes and training steps
in between.

Oracle bound (as in test_sample_gpu.py): the sampler's error against the oracle's float64 run is at most
twice the oracle's own error in the run's dtype (bf16 autocast), measured on the final latents."""
import copy

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _bits(t):
    t = t.detach().cpu().contiguous()
    return t.view({4: torch.int32, 2: torch.int16, 1: torch.uint8}[t.element_size()])


def _mask_u8(B, H, W, g):
    """A random 0..255 mask with 127 and 128 at pixels the latent grid reads."""
    m = torch.randint(0, 256, (B, H, W), generator=g, dtype=torch.uint8)
    m[:, 0, 0], m[:, 0, 8], m[:, 8, 0], m[:, 8, 8] = 127, 128, 0, 255
    return m


# ------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("md", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("channels_last", [True, False])
@pytest.mark.parametrize("G", [1, 2])
@pytest.mark.parametrize("scheduler", ["euler_ancestral", "ddim"])
@pytest.mark.parametrize("inpaint", [False, True])
def test_sample_init_is_torch_op_by_op_bit_for_bit(md, channels_last, G, scheduler, inpaint):
    from lora_b200.host import schedulers
    from lora_b200.host.vae import DiagonalGaussianDistribution
    from lora_b200.step_ops import sample_init
    from oracle import sample_image_ref as RI
    g = torch.Generator().manual_seed(G + 2 * int(channels_last) + 4 * int(inpaint))
    B, C, H, W = 2, 4, 6, 10
    n = 10
    start = 0 if inpaint else schedulers.t_start(n, 0.5)
    tab = schedulers.pack_table(scheduler, "epsilon", n, n, start, from_image=not inpaint)
    rows = tab.shape[0]
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    mom = torch.randn(B, 2 * C, H, W, generator=g) * 2
    mom[:, C:] *= 8                                       # logvar past both clamp bounds
    mom[0, C, 0, :2] = torch.tensor([-40.0, 30.0])
    mom = mom.to(md).to(DEV).contiguous(memory_format=fmt)
    eps = torch.randn(B, C, H, W, generator=g).to(md).to(DEV)
    noise = torch.randn(rows, B, C, H, W, generator=g).to(DEV)
    Cu = 2 * C + 1 if inpaint else C
    unet_in = torch.full((G * B, Cu, H, W), float("nan"), device=DEV, dtype=torch.bfloat16).contiguous(
        memory_format=torch.channels_last)
    x = torch.zeros(B, C, H, W, device=DEV)
    idx = torch.full((1,), 7, device=DEV, dtype=torch.int32)
    cnt = torch.full((1,), 3, device=DEV, dtype=torch.int32)
    ts = torch.zeros(1, device=DEV)
    mask = _mask_u8(B, 8 * H, 8 * W, g).to(DEV) if inpaint else None
    sample_init(mom, eps, x, noise, tab.to(DEV), idx, cnt, unet_in, ts, 0.18215, mask=mask)
    torch.cuda.synchronize()
    # torch, op by op: latent_dist.sample(eps) * 0.18215 in the moments' dtype
    dist = DiagonalGaussianDistribution(mom)
    lat = (dist.mean + dist.std * eps) * 0.18215
    ref = RI.make_scheduler(scheduler, "epsilon")
    ref.set_timesteps(n, device=DEV)
    if inpaint:
        want_x = noise[0] * tab[0, 0].item()
    else:
        want_x = ref.add_noise(lat.float(), noise[0], ref.timesteps[start:start + 1])
    assert torch.equal(_bits(x), _bits(want_x))
    want_in = (tab[0, 1].item() * want_x).to(torch.bfloat16)
    for h in range(G):
        half = unet_in[h * B:(h + 1) * B]
        assert torch.equal(_bits(half[:, :C]), _bits(want_in))
        if inpaint:
            m, _ = RI.prepare_mask_and_masked_image(torch.zeros(B, 8 * H, 8 * W, 3, dtype=torch.uint8), mask.cpu())
            m = F.interpolate(m, size=(H, W))
            assert torch.equal(_bits(half[:, C:C + 1]), _bits(m.to(torch.bfloat16)))
            assert torch.equal(_bits(half[:, C + 1:]), _bits(lat.to(torch.bfloat16)))
    assert float(ts) == float(tab[0, 2]) and int(idx) == 0 and int(cnt) == 0


def test_sample_init_without_moments_is_the_txt2img_init():
    from lora_b200.host import schedulers
    from lora_b200.step_ops import sample_init, sample_step
    g = torch.Generator().manual_seed(0)
    B, C, H, W = 2, 4, 8, 8
    tab = schedulers.pack_table("euler_ancestral", "epsilon", 10, 12).to(DEV)
    noise = torch.randn(13, B, C, H, W, generator=g).to(DEV)
    outs = []
    for init in ("step", "init"):
        x = torch.zeros(B, C, H, W, device=DEV)
        unet_in = torch.zeros(2 * B, C, H, W, device=DEV, dtype=torch.bfloat16).contiguous(
            memory_format=torch.channels_last)
        idx, cnt, ts = (torch.ones(1, device=DEV, dtype=torch.int32), torch.zeros(1, device=DEV, dtype=torch.int32),
                        torch.zeros(1, device=DEV))
        if init == "step":
            sample_step(None, x, noise, tab, None, idx, cnt, unet_in, ts, None, 0.18215, init=True)
        else:
            sample_init(None, None, x, noise, tab, idx, cnt, unet_in, ts)
        outs.append((x, unet_in, ts, idx))
    for a, b in zip(*outs):
        assert torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("channels_last", [True, False])
def test_pixels_ingest_inpaint_is_prepare_mask_and_masked_image_bit_for_bit(dt, channels_last):
    from lora_b200.step_ops import pixels_ingest_inpaint
    from oracle import sample_image_ref as RI
    g = torch.Generator().manual_seed(2)
    B, H, W = 2, 24, 40
    img = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
    img[0, 0, :6] = (torch.arange(18, dtype=torch.uint8) * 15).reshape(6, 3)          # 0, 15, .., 255
    mask = _mask_u8(B, H, W, g)
    got = pixels_ingest_inpaint(img.to(DEV), mask.to(DEV), dt, channels_last=channels_last)
    assert got.is_contiguous(memory_format=torch.channels_last if channels_last else torch.contiguous_format)
    _, want = RI.prepare_mask_and_masked_image(img, mask)
    assert torch.equal(_bits(got), _bits(want.to(dt)))


@pytest.mark.parametrize("G", [1, 2])
@pytest.mark.parametrize("last", [False, True])
def test_strided_step_writes_the_latent_channels_only(G, last):
    from lora_b200.step_ops import sample_step, sample_step_ch
    g = torch.Generator().manual_seed(G)
    B, C, H, W = 2, 4, 8, 12
    rows = 4
    tab = torch.zeros(rows, 8)
    tab[1:, 0] = 1 + torch.rand(rows - 1, generator=g) * 0.1
    tab[1:, 1] = -torch.rand(rows - 1, generator=g)
    tab[1:, 2] = torch.rand(rows - 1, generator=g)
    tab[1:, 3] = torch.rand(rows - 1, generator=g)
    tab[1:, 4] = torch.tensor([900.0, 500.0, 100.0])
    tab[rows - 1, 5] = 1.0
    tab = tab.to(DEV)
    mo = torch.randn(G * B, C, H, W, generator=g).to(torch.bfloat16).to(DEV).contiguous(
        memory_format=torch.channels_last)
    noise = torch.randn(rows, B, C, H, W, generator=g).to(DEV)
    x0 = torch.randn(B, C, H, W, generator=g).to(DEV)
    gs = torch.tensor([7.0], device=DEV)
    sentinel = torch.randn(G * B, C + 1, H, W, generator=g).to(torch.bfloat16).to(DEV)
    res = []
    for Cu in (C, 2 * C + 1):
        x = x0.clone()
        idx = torch.full((1,), 2 if last else 1, device=DEV, dtype=torch.int32)
        cnt, ts = torch.zeros(1, device=DEV, dtype=torch.int32), torch.zeros(1, device=DEV)
        unet_in = torch.zeros(G * B, Cu, H, W, device=DEV, dtype=torch.bfloat16)
        if Cu > C:
            unet_in[:, C:] = sentinel
        unet_in = unet_in.contiguous(memory_format=torch.channels_last)
        vae_in = torch.zeros(B, C, H, W, device=DEV)
        (sample_step if Cu == C else sample_step_ch)(mo, x, noise, tab, gs, idx, cnt, unet_in, ts, vae_in, 0.18215)
        torch.cuda.synchronize()
        res.append((x, unet_in, ts, idx, vae_in))
    (x, u, ts, idx, v), (x2, u2, ts2, idx2, v2) = res
    assert torch.equal(_bits(x), _bits(x2)) and torch.equal(_bits(u), _bits(u2[:, :C]))
    assert torch.equal(_bits(u2[:, C:]), _bits(sentinel))
    assert torch.equal(ts, ts2) and torch.equal(idx, idx2) and torch.equal(_bits(v), _bits(v2))


# ------------------------------------------------------------------------------------ tiny models
def _models(in_channels=4, seed=0, up_std=0.05):
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
    if in_channels != 4:
        # the 9-channel UNet from its own draw; the text encoder and VAE stay the 4-channel set's. On the
        # text-encoder weights the 9-channel draw would give, the captured text encoder alone (no sampler
        # launch in the graph) differs from its eager run in the last bits, which would hide what these
        # tests check: that the inpainting graphs replay the eager path exactly.
        torch.manual_seed(seed + 1000)
        ucfg = UNetConfig.tiny()
        ucfg.in_channels = in_channels
        unet = UNet2DConditionModel(ucfg).to(DEV).to(memory_format=torch.channels_last)
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


def _images(seed=6):
    g = torch.Generator().manual_seed(seed)
    B, _, h, w = LAT
    img = torch.randint(0, 256, (B, 8 * h, 8 * w, 3), generator=g, dtype=torch.uint8)
    return img.to(DEV), _mask_u8(B, 8 * h, 8 * w, g).to(DEV)


def _sampler(unet, text, vae, graph, **kw):
    from lora_b200.sample import LoraSampler, SamplerConfig
    base = dict(num_inference_steps=10, max_steps=12, guidance_scale=7.0, autocast_dtype=torch.bfloat16,
                use_cuda_graph=graph)
    base.update(kw)
    return LoraSampler(unet, text, vae, SamplerConfig(**base), latent_shape=LAT, seq_len=77, device=DEV)


def _noise_pair(sg, se, seed=11):
    g = torch.Generator(device=DEV).manual_seed(seed)
    noise = torch.randn(sg.noise.shape, device=DEV, generator=g)
    peps = torch.randn(sg.posterior_noise.shape, device=DEV, generator=g).to(sg.posterior_noise.dtype)
    for s in (sg, se):
        s.noise.copy_(noise)
        s.posterior_noise.copy_(peps)
    return noise, peps


@pytest.mark.parametrize("scheduler", ["euler_ancestral", "ddim"])
@pytest.mark.parametrize("prediction_type", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("strength", [0.5, 1.0])
def test_tiny_img2img_graph_equals_eager_and_oracle(scheduler, prediction_type, strength):
    from oracle import sample_image_ref as RI
    unet, text, vae, unet_r, text_r = _models()
    ids, neg = _ids(text)
    img, _ = _images()
    kw = dict(task="img2img", strength=strength, scheduler=scheduler, prediction_type=prediction_type,
              external_noise=True)
    sg, se = _sampler(unet, text, vae, True, **kw), _sampler(unet, text, vae, False, **kw)
    noise, peps = _noise_pair(sg, se)
    sg.prepare()
    img_g = sg.sample(ids, neg, image=img).clone()
    img_e = se.sample(ids, neg, image=img).clone()
    assert sg.captures == 1
    assert torch.equal(img_g, img_e) and torch.equal(sg.latents, se.latents)
    n = 10
    k = int(n * strength)
    args = (ids, neg, img, noise[:k + 1], peps, 7.0)
    f64 = [copy.deepcopy(m).double() for m in (unet_r, text_r, vae)]
    _, lat64 = RI.sample_img2img(*f64, RI.make_scheduler(scheduler, prediction_type), n, strength, *args,
                                 dtype=torch.float64)
    _, lat_run = RI.sample_img2img(unet_r, text_r, vae, RI.make_scheduler(scheduler, prediction_type), n, strength,
                                   *args, dtype=torch.float32, autocast_dtype=torch.bfloat16)
    e_ours, e_ref = _rel(sg.latents, lat64), _rel(lat_run, lat64)
    assert e_ours <= 2 * e_ref, (e_ours, e_ref)


@pytest.mark.parametrize("scheduler", ["euler_ancestral", "ddim"])
def test_tiny_inpaint_graph_equals_eager_and_oracle(scheduler):
    from oracle import sample_image_ref as RI
    unet, text, vae, unet_r, text_r = _models(in_channels=9)
    ids, neg = _ids(text)
    img, mask = _images()
    kw = dict(task="inpaint", scheduler=scheduler, external_noise=True)
    sg, se = _sampler(unet, text, vae, True, **kw), _sampler(unet, text, vae, False, **kw)
    noise, peps = _noise_pair(sg, se)
    sg.prepare()
    img_g = sg.sample(ids, neg, image=img, mask_image=mask).clone()
    img_e = se.sample(ids, neg, image=img, mask_image=mask).clone()
    assert sg.captures == 1
    assert torch.equal(img_g, img_e) and torch.equal(sg.latents, se.latents)
    n = 10
    args = (ids, neg, img, mask, noise[:n + 1], peps, 7.0)
    f64 = [copy.deepcopy(m).double() for m in (unet_r, text_r, vae)]
    _, lat64 = RI.sample_inpaint(*f64, RI.make_scheduler(scheduler, "epsilon"), n, *args, dtype=torch.float64)
    _, lat_run = RI.sample_inpaint(unet_r, text_r, vae, RI.make_scheduler(scheduler, "epsilon"), n, *args,
                                   dtype=torch.float32, autocast_dtype=torch.bfloat16)
    e_ours, e_ref = _rel(sg.latents, lat64), _rel(lat_run, lat64)
    assert e_ours <= 2 * e_ref, (e_ours, e_ref)


@pytest.mark.parametrize("task", ["img2img", "inpaint"])
def test_per_call_changes_do_not_recapture(task):
    unet, text, vae, *_ = _models(in_channels=9 if task == "inpaint" else 4)
    ids, neg = _ids(text)
    img, mask = _images()
    img2, mask2 = _images(seed=7)
    s, e = _sampler(unet, text, vae, True, task=task), _sampler(unet, text, vae, False, task=task)
    m = (lambda mk: dict(mask_image=mk)) if task == "inpaint" else (lambda mk: {})
    calls = [dict(seed=1, image=img, **m(mask)), dict(seed=2, image=img2, **m(mask)),
             dict(seed=2, image=img, **m(mask2)), dict(seed=3, image=img, num_inference_steps=6, **m(mask)),
             dict(seed=3, image=img, scheduler="ddim", **m(mask))]
    if task == "img2img":
        calls += [dict(seed=1, image=img, strength=0.3), dict(seed=1, image=img, strength=1.0),
                  dict(seed=4, image=img2, strength=0.58, num_inference_steps=12)]
    for kw in calls:
        a = s.sample(ids, neg, **kw).clone()
        assert torch.equal(a, e.sample(ids, neg, **kw)), kw
        assert torch.equal(s.latents, e.latents), kw
    assert s.captures == 1
    st = torch.cuda.get_rng_state()
    a = s.sample(ids, neg, **calls[0]).clone()
    b = s.sample(ids, neg, **calls[1]).clone()
    assert not torch.equal(a, b)
    assert torch.equal(a, s.sample(ids, neg, **calls[0])) and torch.equal(st, torch.cuda.get_rng_state())
    assert s.captures == 1


def test_launches_per_denoising_step_of_the_9_channel_unet_are_the_forward_plus_one():
    from lora_b200 import ops
    unet, text, vae, *_ = _models(in_channels=9)
    ids, neg = _ids(text)
    img, mask = _images()
    s = _sampler(unet, text, vae, False, task="inpaint")
    s.sample(ids, neg, image=img, mask_image=mask)
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


# ------------------------------------------------------------------------------------ with training
def _train_inpaint(unet, text, K, sampler_fn=None):
    from lora_b200.train import LoraTrainStep, StepConfig
    cfg = StepConfig(use_cuda_graph=True, graph_warmup=2, autocast_dtype=torch.bfloat16, train_inpainting=True)
    tr = LoraTrainStep(unet, text, cfg, latent_shape=LAT, seq_len=77, device=DEV)
    torch.manual_seed(21)
    tr.latents.copy_(torch.randn(LAT, device=DEV) * 0.18215)
    tr.masked_latents.copy_(torch.randn(LAT, device=DEV) * 0.18215)
    tr.inpaint_mask.copy_((torch.rand(tr.inpaint_mask.shape, device=DEV) > 0.5).float())
    tr.input_ids.copy_(torch.randint(0, text.config.vocab_size, (LAT[0], 77), device=DEV))
    tr.prepare()
    losses = []
    for _ in range(K):
        losses.append(tr.step_device().clone())
        if sampler_fn is not None:
            sampler_fn()
    return tr, torch.stack(losses)


def test_inpaint_sampling_between_inpainting_training_steps_changes_nothing():
    import lora_b200 as L
    unet, text, vae, *_ = _models(in_channels=9)
    u2, t2 = copy.deepcopy(unet), copy.deepcopy(text)
    ids, neg = _ids(text)
    img, mask = _images()
    s = _sampler(unet, text, vae, True, task="inpaint")
    imgs = []
    tr, losses = _train_inpaint(unet, text, 3,
                                lambda: imgs.append(s.sample(ids, neg, seed=0, image=img, mask_image=mask).clone()))
    u4, t4 = copy.deepcopy(u2), copy.deepcopy(t2)
    tr2, losses2 = _train_inpaint(u2, t2, 3)
    assert torch.equal(_bits(losses), _bits(losses2))
    # a second run without sampling: the factors of two plain runs are the yardstick
    tr4, _ = _train_inpaint(u4, t4, 3)
    if torch.equal(tr2.arena.p, tr4.arena.p):
        assert torch.equal(tr.arena.p, tr2.arena.p)
    else:
        assert _rel(tr.arena.p, tr2.arena.p) <= 10 * _rel(tr4.arena.p, tr2.arena.p)
    assert s.captures == 1
    u3, t3 = copy.deepcopy(unet), copy.deepcopy(text)
    L.link_sites(u3, t3)
    fresh = _sampler(u3, t3, vae, False, task="inpaint")
    fresh.sample(ids, neg, seed=0, image=img, mask_image=mask)
    assert torch.equal(imgs[-1], fresh.image) and torch.equal(s.latents, fresh.latents)
    assert unet.training and text.training


# ------------------------------------------------------------------------------------ full size
def _full(in_channels):
    import lora_b200 as L
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    from oracle.ref_modules import ref_inject
    torch.manual_seed(0)
    ucfg = UNetConfig()
    ucfg.in_channels = in_channels
    with torch.device(DEV):
        unet = UNet2DConditionModel(ucfg)
        text = build_text_encoder()
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


@pytest.mark.parametrize("task", ["img2img", "inpaint"])
def test_full_size_sd15_512_euler_50_graph_equals_eager_and_oracle(task):
    import lora_b200 as L
    from lora_b200.sample import LoraSampler, SamplerConfig
    from oracle import sample_image_ref as RI
    n, strength, lat = 50, 0.75, (1, 4, 64, 64)
    unet, text, vae, unet_r, text_r = _full(9 if task == "inpaint" else 4)
    L.set_grouping(True)
    try:
        cfg = dict(task=task, num_inference_steps=n, max_steps=n, guidance_scale=7.0, autocast_dtype=torch.bfloat16,
                   external_noise=True)
        if task == "img2img":
            cfg["strength"] = strength
        sg = LoraSampler(unet, text, vae, SamplerConfig(**cfg), latent_shape=lat, device=DEV)
        se = LoraSampler(unet, text, vae, SamplerConfig(use_cuda_graph=False, **cfg), latent_shape=lat, device=DEV)
        noise, peps = _noise_pair(sg, se, seed=5)
        g = torch.Generator().manual_seed(8)
        img = torch.randint(0, 256, (1, 512, 512, 3), generator=g, dtype=torch.uint8).to(DEV)
        mask = torch.zeros(1, 512, 512, dtype=torch.uint8)
        mask[:, 128:384, 160:416] = 255
        mask = mask.to(DEV)
        extra = dict(image=img, mask_image=mask) if task == "inpaint" else dict(image=img)
        ids = torch.randint(0, text.config.vocab_size, (1, 77), device=DEV)
        neg = torch.randint(0, text.config.vocab_size, (1, 77), device=DEV)
        sg.prepare()
        out = sg.sample(ids, neg, **extra).clone()
        assert torch.equal(out, se.sample(ids, neg, **extra)) and torch.equal(sg.latents, se.latents)
        if task == "img2img":
            k = int(n * strength)
            run = lambda models, **kw: RI.sample_img2img(*models, RI.make_scheduler("euler_ancestral", "epsilon"),  # noqa: E731
                                                         n, strength, ids, neg, img, noise[:k + 1], peps, 7.0, **kw)
        else:
            run = lambda models, **kw: RI.sample_inpaint(*models, RI.make_scheduler("euler_ancestral", "epsilon"),  # noqa: E731
                                                         n, ids, neg, img, mask, noise[:n + 1], peps, 7.0, **kw)
        _, lat_run = run((unet_r, text_r, vae), dtype=torch.float32, autocast_dtype=torch.bfloat16)
        f64 = [copy.deepcopy(m).double() for m in (unet_r, text_r)]
        vae64 = copy.deepcopy(vae).double()
        del unet_r, text_r
        _, lat64 = run((f64[0], f64[1], vae64), dtype=torch.float64)
        e_ours, e_ref = _rel(sg.latents, lat64), _rel(lat_run, lat64)
        assert e_ours <= 2 * e_ref, (e_ours, e_ref)
    finally:
        L.set_grouping(False)
