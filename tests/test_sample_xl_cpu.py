"""SDXL sampling and guidance rescale without a GPU: the folded Euler tables (lora_b200/host/schedulers.py,
"euler") against the oracle's op-by-op EulerDiscreteScheduler (oracle/sample_xl_ref.RefEulerDiscrete) in
float64 for txt2img and img2img slices, its timestep and init_noise_sigma spot values, the oracle's
rescale_noise_cfg against a float64 restatement, the C-ABI refusals of lb_sample_step_rescale, and the
construction and call refusals of LoraXLSampler."""
import ctypes

import numpy as np
import pytest
import torch

EULER = "euler"


def _ref64(prediction_type, n):
    """The oracle scheduler after set_timesteps(n), its float32 sigmas widened to float64."""
    from oracle.sample_xl_ref import RefEulerDiscrete
    ref = RefEulerDiscrete(prediction_type)
    ref.set_timesteps(n)
    ref.sigmas = ref.sigmas.double()
    ref.init_noise_sigma = (ref.sigmas.max() ** 2 + 1) ** 0.5
    return ref


# ------------------------------------------------------------------------------------ tables
@pytest.mark.parametrize("prediction_type", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("n", [1, 7, 20, 30, 50])
def test_folded_euler_table_matches_op_by_op_step_in_float64(prediction_type, n):
    from lora_b200.host import schedulers
    ref = _ref64(prediction_type, n)
    (sig0, s0, t0), steps = schedulers.coefficients(EULER, prediction_type, n)
    assert abs(sig0 - float(ref.init_noise_sigma)) <= 1e-12 * sig0
    one = torch.ones((), dtype=torch.float64)
    assert abs(s0 - float(ref.scale_model_input(one, 0))) <= 1e-15 and t0 == float(ref.timesteps[0])
    g = torch.Generator().manual_seed(n)
    tab = schedulers.pack_table(EULER, prediction_type, n, 50)
    for i in range(n):
        x = torch.randn(64, generator=g, dtype=torch.float64) * 5
        m = torch.randn(64, generator=g, dtype=torch.float64)
        alpha, beta, gamma, s_next, t_next = steps[i]
        want = ref.step(m, i, x)
        assert gamma == 0.0 and float(tab[1 + i, 2]) == 0.0
        assert float((alpha * x + beta * m - want).abs().max()) <= 1e-12 * float(want.abs().max() + 1)
        if i + 1 < n:
            assert abs(s_next - float(ref.scale_model_input(one, i + 1))) <= 1e-15
            assert t_next == float(ref.timesteps[i + 1])
        else:
            assert t_next == 0.0 and float(tab[1 + i, 5]) == 1.0
    assert float(tab[1:n + 1, :5].double().sub(torch.from_numpy(steps)).abs().max()) <= 1e-6 * max(1.0, sig0)


def test_euler_spot_values():
    from lora_b200.host import schedulers
    t30, t50 = schedulers.timesteps(EULER, 30), schedulers.timesteps(EULER, 50)
    assert t30.dtype == np.float32 and list(t30[:3]) == [958, 925, 892] and list(t30[-2:]) == [34, 1]
    assert list(t50[:3]) == [981, 961, 941] and list(t50[-2:]) == [21, 1]
    assert round(schedulers.init_noise_sigma(EULER, 30), 4) == 11.5203
    assert round(schedulers.init_noise_sigma(EULER, 50), 4) == 13.1585
    assert schedulers.family(EULER) == "single-step"
    ref = _ref64("epsilon", 30)
    assert np.array_equal(schedulers.euler_sigmas(30, EULER), ref.sigmas.float().numpy())


@pytest.mark.parametrize("prediction_type", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("n,strength", [(10, 0.5), (30, 0.3), (30, 0.5), (50, 1.0)])
def test_sliced_euler_table_matches_op_by_op_img2img_in_float64(prediction_type, n, strength):
    from lora_b200.host import schedulers
    from oracle import sample_image_ref as RI
    ref = _ref64(prediction_type, n)
    start = schedulers.t_start(n, strength)
    ts, k = RI.get_timesteps(ref, n, strength)
    tab = schedulers.pack_table(EULER, prediction_type, n, 50, start, from_image=True).double()
    assert float(tab[0, 2]) == float(ts[0]) and float(tab[0, 3]) == 1.0
    assert float(tab[0, 0]) == float(ref.sigmas[start].float())
    assert abs(float(tab[0, 1]) - float(ref.scale_model_input(torch.ones((), dtype=torch.float64), start))) < 1e-7
    g = torch.Generator().manual_seed(n)
    for j in range(k):
        x = torch.randn(64, generator=g, dtype=torch.float64) * 5
        m = torch.randn(64, generator=g, dtype=torch.float64)
        want = ref.step(m, start + j, x)
        got = tab[1 + j, 0] * x + tab[1 + j, 1] * m
        assert float((got - want).abs().max()) <= 1e-6 * float(want.abs().max() + 1), j
    assert float(tab[k, 5]) == 1.0 and float(tab[k + 1:].abs().max() if k + 1 < tab.shape[0] else 0.0) == 0.0


@pytest.mark.parametrize("n,strength", [(10, 0.5), (30, 0.75)])
def test_euler_add_noise_row_is_the_oracle_add_noise_in_float32(n, strength):
    from lora_b200.host import schedulers
    from oracle.sample_xl_ref import RefEulerDiscrete
    ref = RefEulerDiscrete("epsilon")
    ref.set_timesteps(n)
    start = schedulers.t_start(n, strength)
    tab = schedulers.pack_table(EULER, "epsilon", n, n, start, from_image=True)
    g = torch.Generator().manual_seed(n)
    x, z = torch.randn(2, 4, 8, 8, generator=g), torch.randn(2, 4, 8, 8, generator=g)
    want = ref.add_noise(x, z, ref.timesteps[start:start + 1])
    got = tab[0, 3] * x + tab[0, 0] * z
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))


# ------------------------------------------------------------------------------------ rescale
@pytest.mark.parametrize("phi", [0.0, 0.3, 0.7, 1.0])
def test_rescale_noise_cfg_matches_a_float64_restatement(phi):
    from oracle.sample_xl_ref import rescale_noise_cfg
    g = torch.Generator().manual_seed(int(phi * 10))
    B, C, H, W = 3, 4, 9, 7
    mc = torch.randn(B, C, H, W, generator=g, dtype=torch.float64) * 1.3 + 0.2
    mu = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    cfg = mu + 5.0 * (mc - mu)
    got = rescale_noise_cfg(cfg, mc, phi)
    n = C * H * W
    for b in range(B):
        a, c = mc[b].numpy().ravel(), cfg[b].numpy().ravel()
        sa = np.sqrt(((a - a.mean()) ** 2).sum() / (n - 1))
        sc = np.sqrt(((c - c.mean()) ** 2).sum() / (n - 1))
        want = phi * c * (sa / sc) + (1 - phi) * c
        assert np.allclose(got[b].numpy().ravel(), want, rtol=1e-13, atol=0)
        if phi == 1.0:        # the rescaled prediction has the conditional prediction's std
            assert abs(got[b].std().item() - sa) <= 1e-12 * sa


# ------------------------------------------------------------------------------------ C-ABI
def test_rescale_entry_point_is_declared_and_exported():
    import os
    from lora_b200 import _C as C
    hdr = open(os.path.join(os.path.dirname(C.__file__), "..", "include", "lora_b200.h")).read()
    assert "int lb_sample_step_rescale(" in hdr and "lb_sample_step_rescale" in C.EXPORTED
    assert hasattr(C.lib, "lb_sample_step_rescale")


def test_sample_step_rescale_refuses_bad_arguments_without_gpu():
    from lora_b200 import _C as C
    p = ctypes.c_void_p(256)         # never dereferenced: every call below is refused before any CUDA call

    def call(model=p, mdt=C.LB_BF16, G=2, x=p, noise=p, hist=None, table=p, rows=51, guid=p, phi=p, idx=p, cnt=p,
             uin=p, udt=C.LB_BF16, uch=4, ts=p, vin=p, vdt=C.LB_F32, scaling=0.13025, B=1, Ch=4, H=8, W=8):
        return C.lib.lb_sample_step_rescale(model, mdt, 256, 1, 4, G, x, noise, hist, table, rows, guid, phi, idx, cnt,
                                            uin, udt, uch, ts, vin, vdt, 0, scaling, B, Ch, H, W, None)
    SHAPE, DTYPE = -1, -3
    assert call(G=1) == SHAPE and call(G=3) == SHAPE and call(G=0) == SHAPE
    assert call(phi=None) == SHAPE and call(phi=None, hist=p) == SHAPE
    assert call(B=0) == SHAPE and call(B=65536) == SHAPE and call(H=-1) == SHAPE and call(W=0) == SHAPE
    assert call(Ch=0) == SHAPE and call(rows=1) == SHAPE and call(uch=3) == SHAPE
    assert call(mdt=7) == DTYPE and call(udt=9) == DTYPE and call(vdt=-1) == DTYPE
    assert call(noise=None) == SHAPE and call(x=None) == SHAPE and call(table=None) == SHAPE
    assert call(model=None) == SHAPE and call(guid=None) == SHAPE and call(vin=None) == SHAPE
    assert call(idx=None) == SHAPE and call(cnt=None) == SHAPE and call(uin=None) == SHAPE and call(ts=None) == SHAPE
    assert call(scaling=0.0) == SHAPE and call(scaling=float("nan")) == SHAPE


# ------------------------------------------------------------------------------------ sampler refusals
def _xl(vae_dtype=torch.float32):
    from lora_b200.host.clip import build_sdxl_text_encoders
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    torch.manual_seed(0)
    te1, te2 = build_sdxl_text_encoders(tiny=True)
    return (UNet2DConditionModel(UNetConfig.sdxl_tiny()), te1, te2,
            AutoencoderKL(VAEConfig.tiny(), with_decoder=True).to(vae_dtype))


SHAPE = (1, 4, 8, 8)


def test_xl_sampler_construction_refusals():
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.sample import LoraSampler, LoraXLSampler, SamplerConfig
    unet, te1, te2, vae = _xl()
    kw = dict(latent_shape=SHAPE, device="cpu")
    with pytest.raises(ValueError, match="SDXL"):
        LoraXLSampler(UNet2DConditionModel(UNetConfig.tiny()), te1, te2, vae, SamplerConfig(), **kw)
    with pytest.raises(ValueError, match="CLIPTextModelWithProjection"):
        LoraXLSampler(unet, te1, build_text_encoder(tiny=True), vae, SamplerConfig(), **kw)
    with pytest.raises(ValueError, match="cross_attention_dim"):
        LoraXLSampler(unet, build_text_encoder(tiny=True, sd2=True), te2, vae, SamplerConfig(), **kw)
    with pytest.raises(ValueError, match="fp16"):
        LoraXLSampler(unet, te1, te2, _xl(torch.float16)[3], SamplerConfig(), **kw)
    with pytest.raises(ValueError, match="inpaint"):
        LoraXLSampler(unet, te1, te2, vae, SamplerConfig(task="inpaint"), **kw)
    for phi in (-0.1, 1.5, float("nan")):
        with pytest.raises(ValueError, match="guidance_rescale"):
            LoraXLSampler(unet, te1, te2, vae, SamplerConfig(guidance_rescale=phi), **kw)
    # LoraSampler still refuses SDXL UNets, and names the class that samples them
    with pytest.raises(ValueError, match="SDXL.*LoraXLSampler"):
        LoraSampler(unet, te1, vae, SamplerConfig(), **kw)
    s = LoraXLSampler(unet, te1, te2, vae, SamplerConfig(scheduler=EULER, max_steps=30, num_inference_steps=30),
                      **kw)
    assert s.captures == 0 and tuple(s.time_ids.shape) == (2, 6) and tuple(s.input_ids_2.shape) == (2, 77)
    assert s.time_ids[0].tolist() == [64.0, 64.0, 0.0, 0.0, 64.0, 64.0]
    assert len(s._lora_models()) == 3 and s._lora_models()[2] is te2


def test_xl_sampler_call_refusals_before_any_cuda_call():
    from lora_b200.sample import LoraXLSampler, SamplerConfig
    unet, te1, te2, vae = _xl()
    s = LoraXLSampler(unet, te1, te2, vae, SamplerConfig(scheduler=EULER), latent_shape=SHAPE, device="cpu")
    ids = torch.zeros(1, 77, dtype=torch.long)
    bad = [dict(input_ids_2=torch.zeros(2, 77, dtype=torch.long)),
           dict(input_ids_2=torch.zeros(1, 76, dtype=torch.long)),
           dict(input_ids_2=torch.zeros(1, 77)),
           dict(input_ids=torch.zeros(1, 77, dtype=torch.float16)),
           dict(negative_input_ids=ids),
           dict(negative_input_ids_2=ids),
           dict(negative_input_ids=ids, negative_input_ids_2=torch.zeros(1, 77)),
           dict(negative_input_ids=torch.zeros(1, 70, dtype=torch.long), negative_input_ids_2=ids),
           dict(guidance_rescale=1.2), dict(guidance_rescale=-0.5),
           dict(original_size=(1024,)), dict(crops_coords_top_left=None),
           dict(image=torch.zeros(1, 64, 64, 3, dtype=torch.uint8))]
    for kw in bad:
        args = dict(input_ids=ids, input_ids_2=ids)
        args.update(kw)
        with pytest.raises(ValueError):
            s.sample(args.pop("input_ids"), args.pop("input_ids_2"), **args)


def test_sd_sampler_takes_guidance_rescale_in_range_only():
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    from lora_b200.sample import LoraSampler, SamplerConfig
    unet, text = UNet2DConditionModel(UNetConfig.tiny()), build_text_encoder(tiny=True)
    vae = AutoencoderKL(VAEConfig.tiny(), with_decoder=True)
    with pytest.raises(ValueError, match="guidance_rescale"):
        LoraSampler(unet, text, vae, SamplerConfig(guidance_rescale=2.0), latent_shape=SHAPE, device="cpu")
    s = LoraSampler(unet, text, vae, SamplerConfig(scheduler=EULER, guidance_rescale=0.7), latent_shape=SHAPE,
                    device="cpu")
    ids = torch.zeros(1, 77, dtype=torch.long)
    with pytest.raises(ValueError, match="guidance_rescale"):
        s.sample(ids, ids, guidance_rescale=1.01)
    assert s._key(2, "single-step", True) == (2, "single-step", "rescale") and s._key(2, "multistep", False) == (
        2, "multistep")
