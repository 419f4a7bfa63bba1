"""Sampling without a GPU: the folded scheduler tables (lora_b200/host/schedulers.py) against the
oracle's op-by-op scheduler steps (oracle/sample_ref.py) in float64, their timestep and sigma values,
the VAE decoder's keys and arithmetic, the C-ABI of lb_sample_step / lb_pixels_emit, and the sampler's
construction refusals."""
import copy
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from test_formats_cpu import _vae_keys


# ------------------------------------------------------------------------------------ tables
@pytest.mark.parametrize("scheduler", ["euler_ancestral", "ddim"])
@pytest.mark.parametrize("prediction_type", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("n", [1, 2, 10, 50])
def test_folded_table_matches_op_by_op_step_in_float64(scheduler, prediction_type, n):
    from lora_b200.host import schedulers
    from oracle.sample_ref import make_scheduler
    ref = make_scheduler(scheduler, prediction_type)
    ref.set_timesteps(n)
    # the scheduler's float32 tables widened, so that every op of its step runs in float64
    ref.alphas_cumprod = ref.alphas_cumprod.double()
    if scheduler == "euler_ancestral":
        ref.sigmas = ref.sigmas.double()
    else:
        ref.final_alpha_cumprod = ref.alphas_cumprod[0]
    (sigma0, s0, t0), steps = schedulers.coefficients(scheduler, prediction_type, n)
    assert sigma0 == float(ref.init_noise_sigma) and t0 == float(ref.timesteps[0])
    g = torch.Generator().manual_seed(n)
    gs = 7.0
    shape = (2, 4, 8, 8)
    x = torch.randn(shape, generator=g, dtype=torch.float64) * float(ref.init_noise_sigma)
    # the first UNet input
    assert torch.allclose(ref.scale_model_input(x, 0), s0 * x, rtol=1e-12, atol=0)
    for i in range(n):
        m_u, m_c, z = (torch.randn(shape, generator=g, dtype=torch.float64) for _ in range(3))
        m_hat = m_u + gs * (m_c - m_u)
        want = ref.step(m_hat, i, x, z)
        alpha, beta, gamma, s_next, t_next = steps[i]
        got = alpha * x + beta * m_hat + gamma * z
        scale = (alpha * x).abs() + (beta * m_hat).abs() + (gamma * z).abs()
        assert float(((got - want).abs() / scale).max()) < 1e-12, i
        if i + 1 < n:
            assert t_next == float(ref.timesteps[i + 1])
            assert torch.allclose(ref.scale_model_input(want, i + 1), s_next * want, rtol=1e-12, atol=0)
        x = want


def test_timestep_and_sigma_spot_values():
    from lora_b200.host import schedulers
    assert list(schedulers.timesteps("ddim", 50)) == list(range(981, 0, -20))
    ts = schedulers.timesteps("euler_ancestral", 50)
    assert ts[0] == 999.0 and ts[-1] == 0.0 and all(a > b for a, b in zip(ts, ts[1:]))
    assert abs(schedulers.init_noise_sigma("euler_ancestral", 50) - 14.6146) < 1e-4
    (sigma0, _, t0), _ = schedulers.coefficients("euler_ancestral", "epsilon", 50)
    assert sigma0 == schedulers.euler_sigmas(50)[0] and t0 == 999.0
    assert schedulers.euler_sigmas(50)[-1] == 0.0


def test_packed_table_layout():
    from lora_b200.host import schedulers
    tab = schedulers.pack_table("ddim", "epsilon", 3, 5)
    (_, _, t0), steps = schedulers.coefficients("ddim", "epsilon", 3)
    assert tab.dtype == torch.float32 and tuple(tab.shape) == (6, 8)
    assert float(tab[0, 0]) == 1.0 and float(tab[0, 2]) == t0
    assert torch.equal(tab[1:4, :5], torch.from_numpy(steps).float())
    assert tab[:, 5].tolist() == [0, 0, 0, 1, 0, 0]
    with pytest.raises(ValueError):
        schedulers.pack_table("ddim", "epsilon", 6, 5)
    with pytest.raises(ValueError):
        schedulers.coefficients("ddpm", "epsilon", 5)
    with pytest.raises(ValueError):
        schedulers.coefficients("ddim", "sample", 5)


# ------------------------------------------------------------------------------------ VAE decoder
def test_decoder_keys_are_diffusers_and_convert():
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    from lora_b200.to_ckpt import convert_vae_state_dict
    want = {k for k in _vae_keys() if k.startswith(("decoder.", "post_quant_conv."))}
    vae = AutoencoderKL(VAEConfig.sd(), with_decoder=True)
    sd = vae.state_dict()
    got = {k for k in sd if k.startswith(("decoder.", "post_quant_conv."))}
    assert got == want
    assert set(sd) == set(_vae_keys())
    conv = convert_vae_state_dict(dict(sd))
    assert len(conv) == len(sd)
    assert "decoder.up.3.block.0.norm1.weight" in conv and "post_quant_conv.weight" in conv
    # the decoder loads diffusers >= 0.14's attention names too
    new = {k.replace("attentions.0.query.", "attentions.0.to_q."): v for k, v in sd.items()}
    AutoencoderKL(VAEConfig.sd(), with_decoder=True).load_state_dict(new)


def test_without_decoder_is_unchanged():
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    torch.manual_seed(5)
    plain = AutoencoderKL(VAEConfig.tiny())
    torch.manual_seed(5)
    full = AutoencoderKL(VAEConfig.tiny(), with_decoder=True)
    enc = {k for k in _vae_keys() if not k.startswith(("decoder.", "post_quant_conv."))}
    assert set(AutoencoderKL(VAEConfig.sd()).state_dict()) == enc
    fs = full.state_dict()
    for k, v in plain.state_dict().items():
        assert torch.equal(v, fs[k]), k
    with pytest.raises(ValueError):
        plain.decode(torch.zeros(1, 4, 2, 2))


def _decode_f64(sd, cfg, z):
    """diffusers' Decoder restated functionally in float64."""
    p = {k: v.double() for k, v in sd.items()}

    def gn(x, pre):
        return F.group_norm(x, cfg.norm_num_groups, p[pre + ".weight"], p[pre + ".bias"], eps=1e-6)

    def conv(x, pre, pad=1):
        return F.conv2d(x, p[pre + ".weight"], p[pre + ".bias"], padding=pad)

    def res(x, pre):
        h = conv(F.silu(gn(x, pre + ".norm1")), pre + ".conv1")
        h = conv(F.silu(gn(h, pre + ".norm2")), pre + ".conv2")
        if pre + ".conv_shortcut.weight" in p:
            x = conv(x, pre + ".conv_shortcut", 0)
        return x + h

    def attn(x, pre):
        B, C, H, W = x.shape
        h = gn(x, pre + ".group_norm").reshape(B, C, H * W).transpose(1, 2)
        q, k, v = (F.linear(h, p[f"{pre}.{n}.weight"], p[f"{pre}.{n}.bias"]) for n in ("query", "key", "value"))
        w = torch.softmax(q @ k.transpose(1, 2) / math.sqrt(C), dim=-1)
        o = F.linear(w @ v, p[pre + ".proj_attn.weight"], p[pre + ".proj_attn.bias"])
        return o.transpose(1, 2).reshape(B, C, H, W) + x

    x = conv(z, "post_quant_conv", 0)
    x = conv(x, "decoder.conv_in")
    x = res(x, "decoder.mid_block.resnets.0")
    x = attn(x, "decoder.mid_block.attentions.0")
    x = res(x, "decoder.mid_block.resnets.1")
    for i in range(len(cfg.block_out_channels)):
        for j in range(cfg.layers_per_block + 1):
            x = res(x, f"decoder.up_blocks.{i}.resnets.{j}")
        if i < len(cfg.block_out_channels) - 1:
            x = conv(F.interpolate(x, scale_factor=2.0, mode="nearest"), f"decoder.up_blocks.{i}.upsamplers.0.conv")
    return conv(F.silu(gn(x, "decoder.conv_norm_out")), "decoder.conv_out")


def test_tiny_decoder_matches_float64_restatement():
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    torch.manual_seed(0)
    cfg = VAEConfig.tiny()
    vae = AutoencoderKL(cfg, with_decoder=True).double()
    z = torch.randn(2, 4, 5, 6, dtype=torch.float64)
    got = vae.decode(z).sample
    want = _decode_f64(vae.state_dict(), cfg, z)
    assert got.shape == (2, 3, 40, 48)
    assert float((got - want).abs().max() / want.abs().max()) < 1e-12


# ------------------------------------------------------------------------------------ C-ABI
def _lib():
    from lora_b200 import _C
    return _C


def test_new_entry_points_are_declared_and_exported():
    import os
    C = _lib()
    hdr = open(os.path.join(os.path.dirname(C.__file__), "..", "include", "lora_b200.h")).read()
    for name in ("lb_sample_step", "lb_pixels_emit"):
        assert f"int {name}(" in hdr and name in C.EXPORTED and hasattr(C.lib, name)


def test_sample_step_refuses_bad_arguments_without_gpu():
    C = _lib()
    L = C.lib
    p = ctypes.c_void_p(256)         # never dereferenced: every call below is refused before any CUDA call

    def call(model=p, mdt=C.LB_BF16, G=2, x=p, noise=p, table=p, rows=51, guid=p, idx=p, cnt=p, uin=p,
             udt=C.LB_BF16, ts=p, vin=p, vdt=C.LB_F32, scaling=0.18215, B=1, Ch=4, H=8, W=8, init=0):
        return L.lb_sample_step(model, mdt, 256, 1, 4, G, x, noise, table, rows, guid, idx, cnt, uin, udt, ts, vin,
                                vdt, 0, scaling, B, Ch, H, W, init, None)
    SHAPE, DTYPE = -1, -3
    assert call(B=0) == SHAPE and call(H=-1) == SHAPE and call(G=3) == SHAPE and call(rows=1) == SHAPE
    assert call(mdt=7) == DTYPE and call(udt=9) == DTYPE and call(vdt=-1) == DTYPE
    assert call(model=None) == SHAPE and call(guid=None) == SHAPE and call(vin=None) == SHAPE
    assert call(idx=None) == SHAPE and call(cnt=None) == SHAPE and call(x=None) == SHAPE
    assert call(scaling=0.0) == SHAPE and call(scaling=float("nan")) == SHAPE
    # init reads no model output, guidance or decoder input, but still needs the rest
    assert call(init=1, noise=None) == SHAPE and call(init=1, uin=None) == SHAPE


def test_pixels_emit_refuses_bad_arguments_without_gpu():
    C = _lib()
    p = ctypes.c_void_p(256)
    assert C.lib.lb_pixels_emit(p, C.LB_BF16, 0, p, 0, 8, 8, None) == -1
    assert C.lib.lb_pixels_emit(None, C.LB_BF16, 0, p, 1, 8, 8, None) == -1
    assert C.lib.lb_pixels_emit(p, C.LB_BF16, 0, None, 1, 8, 8, None) == -1
    assert C.lib.lb_pixels_emit(p, 5, 0, p, 1, 8, 8, None) == -3


# ------------------------------------------------------------------------------------ refusals
def _tiny(in_channels=4, sdxl=False, decoder=True):
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    cfg = UNetConfig.sdxl_tiny() if sdxl else UNetConfig.tiny()
    cfg.in_channels = in_channels
    return (UNet2DConditionModel(cfg), build_text_encoder(tiny=True),
            AutoencoderKL(VAEConfig.tiny(), with_decoder=decoder))


def test_sampler_construction_refusals():
    from lora_b200.sample import LoraSampler, SamplerConfig
    unet, text, vae = _tiny()
    shape = (1, 4, 8, 8)
    for kw in (dict(scheduler="ddpm"), dict(scheduler="pndm"), dict(prediction_type="sample"),
               dict(num_inference_steps=60, max_steps=50), dict(num_inference_steps=0)):
        with pytest.raises(ValueError):
            LoraSampler(unet, text, vae, SamplerConfig(**kw), latent_shape=shape, device="cpu")
    with pytest.raises(ValueError, match="decoder"):
        LoraSampler(unet, text, _tiny(decoder=False)[2], SamplerConfig(), latent_shape=shape, device="cpu")
    with pytest.raises(ValueError, match="inpainting"):
        LoraSampler(_tiny(in_channels=9)[0], text, vae, SamplerConfig(), latent_shape=shape, device="cpu")
    with pytest.raises(ValueError, match="SDXL"):
        LoraSampler(_tiny(sdxl=True)[0], text, vae, SamplerConfig(), latent_shape=shape, device="cpu")
    # a valid configuration constructs without a GPU
    s = LoraSampler(unet, text, vae, SamplerConfig(max_steps=10, num_inference_steps=10), latent_shape=shape,
                    device="cpu")
    assert s.captures == 0 and tuple(s.noise.shape) == (11, 1, 4, 8, 8) and tuple(s.image.shape) == (1, 64, 64, 3)
