"""Training from images on the GPU (StepConfig.encode_images): the two kernels against torch's
op-by-op evaluation bit for bit (lb_pixels_ingest against torchvision's ToTensor + Normalize,
lb_step_prologue_posterior against DiagonalGaussianDistribution.sample() * 0.18215 followed by
lb_step_prologue[_v]); the pixels step against the eager encode followed by the latents step, eager
and graph-replayed; the pixels step against the oracle step (oracle/vae_ref.py); the embedding and
textual-inversion steps from pixels against their latents-fed runs; and the launch count.

Oracle bounds are those of the suites the steps come from: test_sd2_gpu.py / test_zz_pti_variants_gpu.py
(tiny steps: loss 1e-2 relative under bf16 autocast) and test_grad_scaler_gpu.py (fp16 GradScaler
steps: same skips and scales, loss 1e-2, update direction cos > 0.95)."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
LAT = (2, 4, 16, 16)


def _bits(t):
    t = t.detach().cpu().contiguous()
    return t.view({4: torch.int32, 2: torch.int16, 1: torch.uint8}[t.element_size()])


def _same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _cpu_ingest(pixels, dtype, mask=None):
    """torchvision's ToTensor + Normalize([0.5], [0.5]) (on the CPU, as the data loader runs them), the
    inpainting dataset's masked image, then the cast to the VAE's dtype."""
    from torchvision import transforms as T
    norm = T.Normalize([0.5], [0.5])
    x = torch.stack([norm(T.ToTensor()(p.numpy())) for p in pixels.cpu()])
    xm = None if mask is None else (x * (mask.cpu() < 0.5)).to(dtype)
    return x.to(dtype), xm


# ------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("channels_last", [True, False])
@pytest.mark.parametrize("B,H,W", [(1, 64, 64), (3, 40, 72)])
def test_pixels_ingest_is_torchvision_bit_for_bit(out_dtype, channels_last, B, H, W):
    from lora_b200.step_ops import pixels_ingest
    g = torch.Generator().manual_seed(B * 1000 + H)
    px = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
    px[0, 0, :4, 0] = torch.tensor([0, 127, 128, 255], dtype=torch.uint8)
    for mask in (None, (torch.rand(B, 1, H, W, generator=g) > 0.5).float(),
                 (torch.rand(B, 1, H, W, generator=g) > 0.5).to(torch.uint8)):
        x, xm = pixels_ingest(px.to(DEV), out_dtype, None if mask is None else mask.to(DEV), channels_last)
        want, want_m = _cpu_ingest(px, out_dtype, mask)
        fmt = torch.channels_last if channels_last else torch.contiguous_format
        assert x.is_contiguous(memory_format=fmt)
        assert _same_bits(x, want)
        if mask is None:
            assert xm is None
        else:
            assert xm.is_contiguous(memory_format=fmt) and _same_bits(xm, want_m)
    # already-normalised fp32 pixels: a cast (and the same masked image)
    f = torch.randn(B, 3, H, W, generator=g)
    mask = (torch.rand(B, 1, H, W, generator=g) > 0.5).float()
    x, xm = pixels_ingest(f.to(DEV), out_dtype, mask.to(DEV), channels_last)
    assert _same_bits(x, f.to(out_dtype)) and _same_bits(xm, (f * (mask < 0.5)).to(out_dtype))


@pytest.mark.parametrize("mdt", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("eps_fp32", [False, True])
@pytest.mark.parametrize("velocity", [False, True])
@pytest.mark.parametrize("inpaint", [False, True])
def test_step_prologue_posterior_is_torch_bit_for_bit(mdt, eps_fp32, velocity, inpaint):
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.vae import DiagonalGaussianDistribution
    from lora_b200.step_ops import step_prologue, step_prologue_posterior
    g = torch.Generator(device=DEV).manual_seed(int(velocity) + 2 * int(inpaint) + 4 * int(eps_fp32))
    noiser = DDPMNoiser(device=DEV)
    B, C, h, w = 3, 4, 12, 20

    def moments():
        m = torch.randn(B, 2 * C, h, w, device=DEV, generator=g) * 3
        m[:, C:] -= 2.0
        m[0, C, 0, :6] = torch.tensor([-45.0, -30.0, -29.5, 19.75, 20.0, 31.0])   # past and at both clamp bounds
        return m.to(mdt).contiguous(memory_format=torch.channels_last)       # the VAE's layout

    edt = torch.float32 if eps_fp32 else mdt
    mom = moments()
    pe = torch.randn(B, C, h, w, device=DEV, generator=g).to(edt)
    noise = torch.randn(B, C, h, w, device=DEV, generator=g)
    t = torch.tensor([0, 517, 999], device=DEV)

    def sample(m, e):                    # diffusers' sample() * 0.18215, then the cast to fp32
        post = DiagonalGaussianDistribution(m)
        return ((post.mean + post.std * e) * 0.18215).float()

    lat = torch.full((B, C, h, w), float("nan"), device=DEV)
    kw = {}
    if inpaint:
        mmom = moments()
        mpe = torch.randn(B, C, h, w, device=DEV, generator=g).to(edt)
        mask = (torch.rand(B, 1, 8 * h, 8 * w, device=DEV, generator=g) > 0.5).float()
        ml, im = torch.empty_like(lat), torch.empty(B, 1, h, w, device=DEV)
        kw = dict(masked_moments=mmom, masked_posterior_noise=mpe, mask=mask, masked_latents=ml, inpaint_mask=im)
        want_im = torch.nn.functional.interpolate(mask, scale_factor=1 / 8)
        want_ml = sample(mmom, mpe)
    got = step_prologue_posterior(mom, pe, noise, t, noiser, torch.bfloat16, lat, 0.18215, velocity=velocity, **kw)
    want_lat = sample(mom, pe)
    assert _same_bits(lat, want_lat)
    if inpaint:
        assert _same_bits(im, want_im) and _same_bits(ml, want_ml)
        want = step_prologue(want_lat, noise, t, noiser, torch.bfloat16, want_im, want_ml, velocity=velocity)
    else:
        want = step_prologue(want_lat, noise, t, noiser, torch.bfloat16, velocity=velocity)
    if velocity:
        assert _same_bits(got[0], want[0]) and _same_bits(got[1], want[1])
    else:
        assert _same_bits(got, want)


# ------------------------------------------------------------------------------------ models
def _models(in_channels=4, vae_dtype=torch.float32, seed=0):
    """(unet, text, vae, (unet, text) before the LoRA injection): tiny host models with non-zero
    trainable LoRA factors, on the GPU."""
    import lora_b200 as L
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    torch.manual_seed(seed)
    cfg = UNetConfig.tiny()
    cfg.in_channels = in_channels
    unet = UNet2DConditionModel(cfg).to(DEV).to(memory_format=torch.channels_last)
    text = build_text_encoder(tiny=True).to(DEV)
    vae = AutoencoderKL(VAEConfig.tiny()).to(DEV, vae_dtype).to(memory_format=torch.channels_last)
    for m in (unet, text, vae):
        m.requires_grad_(False)
    plain = copy.deepcopy(unet), copy.deepcopy(text)
    L.inject_trainable_lora(unet, r=4)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=4)
    g = torch.Generator(device=DEV).manual_seed(3)
    for m in list(unet.modules()) + list(text.modules()):
        if type(m).__name__ == "LoraInjectedLinear":
            m.lora_up.weight.data.normal_(0, 0.05, generator=g)
    return unet, text, vae, plain


def _draws(n, seed=8, pe_dtype=torch.float32, inpaint=False, vocab=1000):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        d = dict(pixels=torch.randint(0, 256, (LAT[0], 8 * LAT[2], 8 * LAT[3], 3), generator=g, dtype=torch.uint8),
                 ids=torch.randint(0, vocab, (LAT[0], 77), generator=g),
                 pe=torch.randn(LAT, generator=g).to(pe_dtype), noise=torch.randn(LAT, generator=g),
                 t=torch.randint(0, 1000, (LAT[0],), generator=g))
        if inpaint:
            d["mask"] = (torch.rand(LAT[0], 1, 8 * LAT[2], 8 * LAT[3], generator=g) > 0.5).float()
            d["mpe"] = torch.randn(LAT, generator=g).to(pe_dtype)
        out.append(d)
    return out


def _feed_pixels(eng, d):
    eng.pixels.copy_(d["pixels"]); eng.input_ids.copy_(d["ids"]); eng.posterior_noise.copy_(d["pe"])
    eng.noise.copy_(d["noise"]); eng.timesteps.copy_(d["t"])
    if "mask" in d:
        eng.pixel_mask.copy_(d["mask"]); eng.masked_posterior_noise.copy_(d["mpe"])


def _factors(eng):
    return torch.cat([p.detach().flatten() for p in eng.arena.parameters()]).clone()


# ------------------------------------------------------------------------------------ latents step
def test_pixels_step_equals_eager_encode_then_latents_step_eager_and_graph():
    """Same posterior noise, noise and timesteps: the pixels step (ingest + VAE + posterior prologue in
    the step) against the user's pattern today -- an eager VAE encode outside the step, its latents
    copied into the latents step. The sampled latents are bit-equal every step and the first loss is
    equal (the forward is deterministic). The factors after 3 steps, and the graph-replayed pixels
    step against the eager one, agree within test_modules_gpu.py's bounds for two runs of one step
    (loss 2e-3 relative, factors 1e-4): the dA / dB reductions add CTA partials with unordered fp32
    atomics, so two runs of the SAME latents step on identical inputs already differ -- by 2e-9 to
    9.1e-6 relative in the factors after 3 steps on an H100 (Adam turns a last-bit gradient
    difference into a step-sized one). prepare() leaves the RNG stream untouched."""
    from lora_b200.host.vae import DiagonalGaussianDistribution
    from lora_b200.train import LoraTrainStep, StepConfig
    unet, text, vae, _ = _models()
    copies = [(copy.deepcopy(unet), copy.deepcopy(text)) for _ in range(3)]
    px = LoraTrainStep(*copies[0], StepConfig(use_cuda_graph=False, external_noise=True, encode_images=True),
                       latent_shape=LAT, device=DEV, vae=vae)
    lt = LoraTrainStep(*copies[1], StepConfig(use_cuda_graph=False, external_noise=True), latent_shape=LAT,
                       device=DEV)
    gr = LoraTrainStep(*copies[2], StepConfig(use_cuda_graph=True, graph_warmup=2, external_noise=True,
                                              encode_images=True), latent_shape=LAT, device=DEV, vae=vae)
    rng = torch.cuda.get_rng_state()
    gr.prepare()
    assert gr.graph is not None, gr.graph_error
    assert torch.equal(torch.cuda.get_rng_state(), rng)
    for k, d in enumerate(_draws(3)):
        _feed_pixels(px, d)
        _feed_pixels(gr, d)
        l_px, l_gr = float(px.step_device()), float(gr.step_device())
        x, _ = _cpu_ingest(d["pixels"], vae.dtype)
        with torch.no_grad():
            post = DiagonalGaussianDistribution(
                vae.encode(x.to(DEV).contiguous(memory_format=torch.channels_last)).latent_dist.parameters)
            lat = ((post.mean + post.std * d["pe"].to(DEV)) * 0.18215).float()
        assert _same_bits(px.latents, lat), k
        lt.latents.copy_(lat); lt.input_ids.copy_(d["ids"]); lt.noise.copy_(d["noise"]); lt.timesteps.copy_(d["t"])
        l_lt = float(lt.step_device())
        if k == 0:
            assert l_px == l_lt, (l_px, l_lt)
        assert abs(l_gr - l_px) < 2e-3 * abs(l_px), (k, l_gr, l_px)
    assert _rel(_factors(px), _factors(lt)) < 1e-4
    assert _rel(_factors(gr), _factors(px)) < 1e-4


# ------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("variant", ["plain", "inpaint", "v_prediction", "fp16_grad_scaler"])
def test_pixels_step_matches_oracle_step(variant):
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.train import LoraTrainStep, StepConfig
    from oracle.ref_modules import ref_inject
    from oracle.vae_ref import RefImageStep, encode
    inpaint, fp16 = variant == "inpaint", variant == "fp16_grad_scaler"
    unet, text, vae, (unet_r, text_r) = _models(in_channels=9 if inpaint else 4,
                                                vae_dtype=torch.float16 if fp16 else torch.float32)
    # the oracle's sites carry the same factors as ours
    ours = [m for m in list(unet.modules()) + list(text.modules()) if type(m).__name__ == "LoraInjectedLinear"]
    us = ref_inject(unet_r, {"CrossAttention", "Attention", "GEGLU"}, r=4)
    ts = ref_inject(text_r, {"CLIPAttention"}, r=4)
    assert len(ours) == len(us) + len(ts)
    for o, r in zip(ours, us + ts):
        r.up.data.copy_(o.lora_up.weight.data)
        r.down.data.copy_(o.lora_down.weight.data)
    v = "v_prediction" if variant == "v_prediction" else "epsilon"
    kw = dict(use_cuda_graph=False, external_noise=True, encode_images=True, train_inpainting=inpaint,
              prediction_type=v)
    noiser = DDPMNoiser(device=DEV)
    if fp16:
        from oracle.amp_ref import RefAmpDreamboothStep
        cfg = StepConfig(autocast_dtype=torch.float16, compute_dtype=torch.float16, grad_scaler=True, **kw)
        ref = RefAmpDreamboothStep(unet_r, text_r, noiser, us, ts, lambda k: 1.0)
    else:
        cfg = StepConfig(autocast_dtype=torch.bfloat16, **kw)
        ref = RefImageStep(vae, unet_r, text_r, noiser, us, ts, autocast_dtype=torch.bfloat16)
    tr = LoraTrainStep(unet, text, cfg, latent_shape=LAT, device=DEV, vae=vae)
    p0 = _factors(tr)
    r0 = torch.cat([p.detach().flatten() for p in ref.unet_params + ref.text_params]).clone()
    for k, d in enumerate(_draws(3, pe_dtype=vae.dtype, inpaint=inpaint)):
        mask, mpe = d.get("mask"), d.get("mpe")
        if fp16:
            lat, _ = encode(vae, d["pixels"], d["pe"])
            l_ref = float(ref.step(lat, d["ids"].to(DEV), d["noise"].to(DEV), d["t"].to(DEV)))
        else:
            l_ref = float(ref.step_from_pixels(d["pixels"], d["ids"].to(DEV), d["pe"], d["noise"].to(DEV),
                                               d["t"].to(DEV), mask=mask, masked_posterior_noise=mpe,
                                               prediction_type=v))
        _feed_pixels(tr, d)
        l_ours = float(tr.step_device())
        assert abs(l_ours - l_ref) < 1e-2 * abs(l_ref), (k, l_ours, l_ref)
    if fp16:
        torch.cuda.synchronize()
        assert ref.skipped == [False] * 3 and int(tr.arena.applied_steps) == 3
    d_ours = _factors(tr) - p0
    d_ref = torch.cat([p.detach().flatten() for p in ref.unet_params + ref.text_params]) - r0
    cos = float((d_ours.double() * d_ref.double()).sum() / (d_ours.double().norm() * d_ref.double().norm()))
    assert cos > 0.95, cos


# ------------------------------------------------------------------------------------ embedding / TI
def _latents_twin(eng_px, eng_lt, d):
    """Feed the latents engine what the pixels engine just encoded, with the same noise."""
    eng_lt.latents.copy_(eng_px.latents); eng_lt.input_ids.copy_(d["ids"])
    eng_lt.noise.copy_(d["noise"]); eng_lt.timesteps.copy_(d["t"])


@pytest.mark.parametrize("kind", ["embedding_table", "textual_inversion"])
def test_embedding_and_ti_steps_from_pixels_match_latents_fed_runs(kind):
    """Each step's latents fed to the latents engine as the pixels engine sampled them: the first loss
    equal, then the bounds of two runs of one step (see the test above). The embedding rows train at
    lr 5e-3, so one Adam element whose gradient differs in the last bits moves a row by a step of that
    size: the table's update after 3 steps differed by 3.5e-4 relative between the two engines on an
    H100, and is held to 1e-2."""
    from lora_b200.train import LoraEmbeddingStep, StepConfig, TextualInversionStep
    unet, text, vae, _ = _models()
    V = text.get_input_embeddings().weight.shape[0]
    tok = [V - 2, V - 1]
    engines = []
    for encode_images in (True, False):
        u, t = copy.deepcopy(unet), copy.deepcopy(text)
        cfg = StepConfig(use_cuda_graph=False, external_noise=True, encode_images=encode_images,
                         t_multiplier=0.8, lr_step_first=True, lr_scheduler="linear", max_train_steps=6)
        vae_arg = vae if encode_images else None
        if kind == "embedding_table":
            engines.append(LoraEmbeddingStep(u, t, tok, cfg, lr_embedding=5e-3, mode="table", latent_shape=LAT,
                                             device=DEV, vae=vae_arg))
        else:
            engines.append(TextualInversionStep(u, t, tok, cfg, lr=5e-3, latent_shape=LAT, device=DEV, vae=vae_arg))
    px, lt = engines
    for k, d in enumerate(_draws(3, vocab=60)):
        d["ids"][0, 2], d["ids"][1, 5] = tok[0], tok[1]
        _feed_pixels(px, d)
        l_px = float(px.step_device())
        _latents_twin(px, lt, d)
        l_lt = float(lt.step_device())
        if k == 0:
            assert l_px == l_lt, (l_px, l_lt)
        assert abs(l_px - l_lt) < 2e-3 * abs(l_lt), (k, l_px, l_lt)
    if kind == "embedding_table":
        px.flush(); lt.flush()
        assert _rel(_factors(px), _factors(lt)) < 1e-4
    tab_px = px.text_encoder.get_input_embeddings().weight
    tab_lt = lt.text_encoder.get_input_embeddings().weight
    assert _rel(tab_px - text.get_input_embeddings().weight, tab_lt - text.get_input_embeddings().weight) < 1e-2
    px.release(); lt.release()


# ------------------------------------------------------------------------------------ launches
# Launches of liblora_b200.so per tiny step (UNetConfig.tiny + tiny CLIP, LoRA r=4, bs 2, default
# StepConfig), counted with the previous release's library: encode_images=False must keep it.
LATENTS_STEP_LAUNCHES = 151


def _launches_per_step(eng):
    from lora_b200 import ops
    eng._body()
    ops.LAUNCH_COUNT = 0
    eng._body()
    return ops.LAUNCH_COUNT


def test_launch_count_latents_step_unchanged_and_pixels_step_adds_one():
    from lora_b200.train import LoraTrainStep, StepConfig
    counts = {}
    for encode_images in (False, True):
        unet, text, vae, _ = _models()
        eng = LoraTrainStep(unet, text, StepConfig(use_cuda_graph=False, encode_images=encode_images),
                            latent_shape=LAT, device=DEV, vae=vae if encode_images else None)
        counts[encode_images] = _launches_per_step(eng)
    print("launches per step", counts)
    assert counts[False] == LATENTS_STEP_LAUNCHES, counts
    # the ingest launch; the posterior prologue replaces the prologue
    assert counts[True] == counts[False] + 1, counts
