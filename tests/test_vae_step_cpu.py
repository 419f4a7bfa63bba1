"""Training from images without a GPU: the host VAE encoder (lora_b200/host/vae.py) -- its state-dict
names and its posterior --, the arithmetic lb_pixels_ingest restates, the step engine's
encode_images body (LoraTrainStep._fwd_bwd on CPU host models, float64 VAE) against the oracle
(oracle/vae_ref.py), and the configurations and inputs the step refuses."""
import re
import warnings

import numpy as np
import pytest
import torch

from lora_b200.host.vae import AutoencoderKL, DiagonalGaussianDistribution, VAEConfig

# original-SD (CompVis AutoencoderKL) names of the encoder half: first_stage_model.<these>
_SD_KEY = re.compile(
    r"^(quant_conv|encoder\.(conv_in|norm_out|conv_out"
    r"|down\.[0-3]\.block\.[01]\.(norm1|conv1|norm2|conv2|nin_shortcut)"
    r"|down\.[0-2]\.downsample\.conv"
    r"|mid\.block_[12]\.(norm1|conv1|norm2|conv2)"
    r"|mid\.attn_1\.(norm|q|k|v|proj_out)))\.(weight|bias)$")


@pytest.mark.parametrize("cfg", [VAEConfig.tiny(), VAEConfig.sd()], ids=["tiny", "sd"])
def test_every_vae_key_converts_to_an_original_sd_key(cfg):
    from lora_b200.to_ckpt import convert_vae_state_dict
    with torch.device("meta"):
        vae = AutoencoderKL(cfg)
    sd = vae.state_dict()
    out = convert_vae_state_dict(sd)
    assert len(out) == len(sd)
    bad = [k for k in out if not _SD_KEY.match(k)]
    assert not bad, bad
    # the attention projections become 1x1 convolutions, as in the original checkpoint
    assert out["encoder.mid.attn_1.q.weight"].dim() == 4
    c = cfg.block_out_channels
    assert out["encoder.conv_in.weight"].shape == (c[0], 3, 3, 3)
    assert out["encoder.conv_out.weight"].shape == (8, c[-1], 3, 3)
    assert out["quant_conv.weight"].shape == (8, 8, 1, 1)


def test_old_and_new_attention_names_load_the_same():
    torch.manual_seed(0)
    src = AutoencoderKL(VAEConfig.tiny()).double()
    old = src.state_dict()
    rename = {"query.": "to_q.", "key.": "to_k.", "value.": "to_v.", "proj_attn.": "to_out.0."}
    new = {}
    for k, v in old.items():
        for a, b in rename.items():
            if ".attentions.0." + a in k:
                k = k.replace(".attentions.0." + a, ".attentions.0." + b)
        new[k] = v
    assert any("to_out.0." in k for k in new) and not any("proj_attn" in k for k in new)
    a = AutoencoderKL(VAEConfig.tiny()).double()
    b = AutoencoderKL(VAEConfig.tiny()).double()
    a.load_state_dict(old)
    b.load_state_dict(new)
    x = torch.randn(2, 3, 64, 48, dtype=torch.float64)
    pa, pb, ps = (m.encode(x).latent_dist.parameters for m in (a, b, src))
    assert torch.equal(pa, pb) and torch.equal(pa, ps)
    assert pa.shape == (2, 8, 8, 6)


def test_latent_dist_float64_semantics():
    g = torch.Generator().manual_seed(3)
    params = torch.randn(2, 8, 4, 5, dtype=torch.float64, generator=g) * 10
    params[0, 4:, 0, 0] = torch.tensor([-45.0, 31.0, -30.0, 20.0], dtype=torch.float64)
    d = DiagonalGaussianDistribution(params)
    mean, logvar = params[:, :4], params[:, 4:]
    assert torch.equal(d.mean, mean) and torch.equal(d.parameters, params)
    assert torch.equal(d.logvar, logvar.clamp(-30.0, 20.0))
    assert d.logvar[0, :, 0, 0].tolist() == [-30.0, 20.0, -30.0, 20.0]
    assert torch.equal(d.std, torch.exp(0.5 * logvar.clamp(-30.0, 20.0)))
    assert torch.equal(d.var, torch.exp(logvar.clamp(-30.0, 20.0)))
    eps = torch.randn(2, 4, 4, 5, dtype=torch.float64, generator=torch.Generator().manual_seed(9))
    s = d.sample(generator=torch.Generator().manual_seed(9))
    assert s.dtype == torch.float64
    assert torch.equal(s, mean + torch.exp(0.5 * logvar.clamp(-30.0, 20.0)) * eps)
    assert torch.equal(d.mode(), mean)


def test_ingest_arithmetic_is_torchvisions():
    """lb_pixels_ingest evaluates each uint8 value as x / 255, (x - 0.5) / 0.5 in IEEE fp32 with one
    rounding per op; all 256 values give torchvision's ToTensor + Normalize([0.5], [0.5]) bits."""
    tv = pytest.importorskip("torchvision.transforms")
    v = np.arange(256, dtype=np.uint8).reshape(16, 16, 1).repeat(3, axis=2)
    want = tv.Normalize([0.5], [0.5])(tv.ToTensor()(v))
    x = np.arange(256, dtype=np.float32)
    ours = (x / np.float32(255) - np.float32(0.5)) / np.float32(0.5)
    assert np.array_equal(want[0].reshape(-1).numpy().view(np.uint32), ours.view(np.uint32))


def _cpu_step(variant, vae):
    """A LoraTrainStep assembled by hand around CPU host models (no arena, no CUDA buffers), with
    encode_images on and the oracle's eager LoRA sites in place of the product's."""
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.train import LoraTrainStep, StepConfig
    from oracle.ref_modules import ref_inject
    inpaint = variant == "inpaint"
    cfg_u = UNetConfig.tiny()
    cfg_u.in_channels = 9 if inpaint else 4
    unet, text = UNet2DConditionModel(cfg_u), build_text_encoder(tiny=True)
    us = ref_inject(unet, {"CrossAttention", "Attention", "GEGLU"}, r=4)
    ts = ref_inject(text, {"CLIPAttention"}, r=4)
    g = torch.Generator().manual_seed(1)
    for s in us + ts:
        s.up.data.normal_(0, 0.05, generator=g)
    shape = (2, 4, 8, 8)
    tr = object.__new__(LoraTrainStep)
    tr.cfg = StepConfig(use_cuda_graph=False, t_multiplier=0.8, use_mask=variant == "masked", mask_temperature=2.0,
                        train_inpainting=inpaint, with_prior_preservation=variant == "prior", prior_loss_weight=0.7,
                        encode_images=True)
    tr.unet, tr.text_encoder, tr.device = unet, text, torch.device("cpu")
    tr.noiser, tr.model_dtype = DDPMNoiser(device="cpu"), torch.float32
    tr.vae, tr.vae_dtype, tr.posterior_noise_dtype = vae, torch.float64, torch.float64
    tr.latents = torch.zeros(shape)
    tr.pixels = torch.randint(0, 256, (2, 64, 64, 3), generator=g, dtype=torch.uint8)
    tr.input_ids = torch.randint(0, 1000, (2, 77), generator=g)
    tr.loss = torch.zeros(())
    tr.mask = torch.ones(2, 1, 8, 8)
    if inpaint:
        tr.inpaint_mask, tr.masked_latents = torch.zeros(2, 1, 8, 8), torch.zeros(shape)
        tr.pixel_mask = (torch.rand(2, 1, 64, 64, generator=g) > 0.5).float()
    return tr, us, ts, g


@pytest.mark.parametrize("variant", ["plain", "masked", "inpaint", "prior"])
def test_train_step_from_pixels_body_on_cpu_doubles(variant):
    """LoraTrainStep._fwd_bwd with encode_images (the unfused body: torch ops for the ingest and the
    posterior sample, a float64 host VAE) against oracle/vae_ref.py for the same seed: the draw
    order (posterior noise of the image, of the masked image, then noise and timesteps), the
    inpainting mask resize and the masked image included."""
    from lora_b200.host.ddpm import DDPMNoiser
    from oracle.vae_ref import RefImageStep
    torch.manual_seed(0)
    vae = AutoencoderKL(VAEConfig.tiny()).double()
    tr, us, ts, g = _cpu_step(variant, vae)
    kw = {}
    if variant == "masked":
        img_mask = (torch.rand(2, 1, 64, 64, generator=g) > 0.4).float()
        tr.set_loss_mask(img_mask)
        kw.update(loss_mask=img_mask, mask_temperature=2.0)
    if variant == "prior":
        kw.update(prior_loss_weight=0.7)
    ref = RefImageStep(vae, tr.unet, tr.text_encoder, DDPMNoiser(device="cpu"), us, ts, t_multiplier=0.8)
    torch.manual_seed(77)
    pe = torch.randn(tr.latents.shape, dtype=torch.float64)
    mpe = torch.randn_like(pe) if variant == "inpaint" else None
    noise = torch.randn(tr.latents.shape)
    t = torch.randint(0, 800, (2,)).long()
    mask = tr.pixel_mask if variant == "inpaint" else None
    want = ref.forward_loss_from_pixels(tr.pixels, tr.input_ids, pe, noise, t, mask=mask,
                                        masked_posterior_noise=mpe, **kw)
    want.backward()
    g_ref = torch.cat([p.grad.flatten() for p in ref.unet_params + ref.text_params])
    ref.opt.zero_grad()
    lat_ref, inp_ref = ref.encode(tr.pixels, pe, mask, mpe)
    torch.manual_seed(77)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")             # torch.autocast("cuda", enabled=False) on a CPU-only box
        tr._fwd_bwd()
    g_ours = torch.cat([p.grad.flatten() for p in ref.unet_params + ref.text_params])
    assert torch.equal(tr.latents, lat_ref.float())
    if variant == "inpaint":
        assert torch.equal(tr.inpaint_mask, inp_ref[0].float())
        assert torch.equal(tr.masked_latents, inp_ref[1].float())
    assert abs(float(tr.loss) - float(want)) <= 1e-5 * abs(float(want))
    assert float((g_ours - g_ref).norm() / g_ref.norm()) < 1e-4


def _tiny_models():
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    return UNet2DConditionModel(UNetConfig.tiny()), build_text_encoder(tiny=True)


def test_encode_images_without_a_vae_is_refused_before_cuda():
    from lora_b200.train import LoraTrainStep, StepConfig, TextualInversionStep
    unet, text = _tiny_models()
    cfg = StepConfig(encode_images=True)
    with pytest.raises(ValueError, match="needs the frozen VAE"):
        LoraTrainStep(unet, text, cfg, latent_shape=(1, 4, 8, 8), device="cpu")
    with pytest.raises(ValueError, match="needs the frozen VAE"):
        TextualInversionStep(unet, text, [5], cfg, latent_shape=(1, 4, 8, 8), device="cpu")
    with pytest.raises(ValueError, match="pixel_dtype"):
        LoraTrainStep(unet, text, StepConfig(encode_images=True, pixel_dtype=torch.float16),
                      latent_shape=(1, 4, 8, 8), device="cpu", vae=AutoencoderKL(VAEConfig.tiny()))


def _host_step(inpaint=False, pixel_dtype=torch.uint8):
    from lora_b200.train import LoraTrainStep, StepConfig
    tr = object.__new__(LoraTrainStep)
    tr.cfg = StepConfig(encode_images=True, train_inpainting=inpaint, pixel_dtype=pixel_dtype)
    tr.latents = torch.zeros(2, 4, 8, 8)
    tr.pixels = torch.zeros((2, 64, 64, 3) if pixel_dtype == torch.uint8 else (2, 3, 64, 64), dtype=pixel_dtype)
    if inpaint:
        tr.pixel_mask = torch.zeros(2, 1, 64, 64)
    return tr


def test_step_host_refuses_images_it_cannot_take():
    ids = torch.zeros(2, 77, dtype=torch.long)
    tr = _host_step()
    with pytest.raises(ValueError, match="8x the latent grid"):
        tr.step_host(torch.zeros(2, 56, 64, 3, dtype=torch.uint8), ids)
    with pytest.raises(ValueError, match="8x the latent grid"):
        tr.step_host(torch.zeros(2, 8, 8, 3, dtype=torch.uint8), ids)
    for dt in (torch.float16, torch.int32, torch.float64):
        with pytest.raises(ValueError, match="uint8 or float32"):
            tr.step_host(torch.zeros(2, 64, 64, 3, dtype=dt), ids)
    with pytest.raises(ValueError, match="pixel_dtype"):
        tr.step_host(torch.zeros(2, 3, 64, 64), ids)
    with pytest.raises(ValueError, match="train_inpainting is off"):
        tr.step_host(torch.zeros(2, 64, 64, 3, dtype=torch.uint8), ids, mask=torch.zeros(2, 1, 64, 64))
    tr = _host_step(inpaint=True)
    with pytest.raises(ValueError, match="needs the image-resolution mask"):
        tr.step_host(torch.zeros(2, 64, 64, 3, dtype=torch.uint8), ids)
    with pytest.raises(ValueError, match="mask of shape"):
        tr.step_host(torch.zeros(2, 64, 64, 3, dtype=torch.uint8), ids, mask=torch.zeros(2, 1, 8, 8))
    tr = _host_step(pixel_dtype=torch.float32)
    with pytest.raises(ValueError, match="8x the latent grid"):
        tr.step_host(torch.zeros(2, 64, 64, 3), ids)
