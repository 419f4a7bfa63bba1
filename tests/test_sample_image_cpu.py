"""img2img and inpainting sampling without a GPU: the strength rule (host/schedulers.t_start) against the
oracle's get_timesteps, the sliced tables and their add_noise row against the oracle's schedulers
(oracle/sample_image_ref.py), both pipelines' preprocessing against the ingest formula for every uint8
value, the C-ABI of lb_sample_init / lb_sample_step_ch / lb_pixels_ingest_inpaint, and the sampler's
construction and call refusals."""
import ctypes

import numpy as np
import pytest
import torch

N_VALUES = [1, 2, 10, 20, 50, 100]
STRENGTHS = [0.01, 0.05, 0.1, 0.29, 0.3, 0.5, 0.58, 0.7, 0.75, 0.99, 1.0]


# ------------------------------------------------------------------------------------ strength
@pytest.mark.parametrize("scheduler", ["euler_ancestral", "ddim"])
@pytest.mark.parametrize("n", N_VALUES)
def test_t_start_matches_get_timesteps(scheduler, n):
    from lora_b200.host import schedulers
    from oracle import sample_image_ref as RI
    ref = RI.make_scheduler(scheduler, "epsilon")
    ref.set_timesteps(n)
    for s in STRENGTHS:
        timesteps, k = RI.get_timesteps(ref, n, s)
        if k == 0:
            with pytest.raises(ValueError, match="no denoising step"):
                schedulers.t_start(n, s)
            continue
        start = schedulers.t_start(n, s)
        assert start == n - k, (n, s)
        assert np.array_equal(schedulers.timesteps(scheduler, n)[start:], timesteps.numpy())


def test_t_start_truncates_the_float_product():
    from lora_b200.host import schedulers
    assert 50 * 0.58 < 29 and 100 * 0.29 < 29
    assert schedulers.t_start(50, 0.58) == 50 - 28
    assert schedulers.t_start(100, 0.29) == 100 - 28
    assert schedulers.t_start(50, 0.75) == 50 - 37
    assert schedulers.t_start(50, 1.0) == 0
    for bad in (0.0, -0.5, 1.01, float("nan")):
        with pytest.raises(ValueError):
            schedulers.t_start(50, bad)


# ------------------------------------------------------------------------------------ tables
@pytest.mark.parametrize("scheduler", ["euler_ancestral", "ddim"])
@pytest.mark.parametrize("prediction_type", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("n,strength", [(10, 0.5), (20, 0.3), (50, 0.75), (50, 0.58), (50, 1.0)])
def test_sliced_table_rows_are_the_full_tables(scheduler, prediction_type, n, strength):
    from lora_b200.host import schedulers
    start = schedulers.t_start(n, strength)
    k = n - start
    full = schedulers.pack_table(scheduler, prediction_type, n, n)
    tab = schedulers.pack_table(scheduler, prediction_type, n, n, start, from_image=True)
    assert torch.equal(tab[1:k + 1, :5], full[1 + start:n + 1, :5])
    assert tab[:, 5].tolist() == [0.0] * k + [1.0] + [0.0] * (n - k)
    assert not bool(tab[k + 1:].any()) and not bool(tab[:, 6:].any())
    # s and t at t_start: those the full run's step before computes as its next input
    if start:
        assert float(tab[0, 1]) == float(full[start, 3]) and float(tab[0, 2]) == float(full[start, 4])
    else:
        assert float(tab[0, 1]) == float(full[0, 1]) and float(tab[0, 2]) == float(full[0, 2])
    # txt2img's table is unchanged by the new arguments
    assert torch.equal(schedulers.pack_table(scheduler, prediction_type, n, n, 0, from_image=False), full)
    with pytest.raises(ValueError):
        schedulers.pack_table(scheduler, prediction_type, n, n, max(start, 1), from_image=False)


@pytest.mark.parametrize("scheduler", ["euler_ancestral", "ddim"])
@pytest.mark.parametrize("n,strength", [(10, 0.5), (50, 0.75), (50, 1.0), (100, 0.29), (1, 1.0)])
def test_add_noise_row_is_the_oracle_add_noise_in_float32(scheduler, n, strength):
    from lora_b200.host import schedulers
    from oracle import sample_image_ref as RI
    ref = RI.make_scheduler(scheduler, "epsilon")
    ref.set_timesteps(n)
    start = schedulers.t_start(n, strength)
    ts = ref.timesteps[start:start + 1]
    tab = schedulers.pack_table(scheduler, "epsilon", n, n, start, from_image=True)
    c_noise, c_lat = tab[0, 0], tab[0, 3]
    one, zero = torch.ones(1), torch.zeros(1)
    assert torch.equal(ref.add_noise(one, zero, ts), c_lat.reshape(1))
    assert torch.equal(ref.add_noise(zero, one, ts), c_noise.reshape(1))
    g = torch.Generator().manual_seed(n)
    x, z = torch.randn(2, 4, 8, 8, generator=g), torch.randn(2, 4, 8, 8, generator=g)
    want = ref.add_noise(x, z, ts)
    got = c_lat * x + c_noise * z                   # the kernel's fl(fl(c_lat x) + fl(c_noise z))
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    if scheduler == "euler_ancestral":
        assert float(c_lat) == 1.0 and float(c_noise) == float(ref.sigmas[start])


@pytest.mark.parametrize("scheduler", ["euler_ancestral", "ddim"])
@pytest.mark.parametrize("prediction_type", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("n,strength", [(10, 0.5), (50, 0.75), (20, 1.0)])
def test_folded_update_over_a_sliced_run_matches_op_by_op_in_float64(scheduler, prediction_type, n, strength):
    from lora_b200.host import schedulers
    from oracle import sample_image_ref as RI
    ref = RI.make_scheduler(scheduler, prediction_type)
    ref.set_timesteps(n)
    ref.alphas_cumprod = ref.alphas_cumprod.double()
    if scheduler == "euler_ancestral":
        ref.sigmas = ref.sigmas.double()
    else:
        ref.final_alpha_cumprod = ref.alphas_cumprod[0]
    timesteps, k = RI.get_timesteps(ref, n, strength)
    start = n - k
    tab = schedulers.pack_table(scheduler, prediction_type, n, n, start, from_image=True).double()
    g = torch.Generator().manual_seed(n + k)
    shape = (2, 4, 8, 8)
    lat, z0 = torch.randn(shape, generator=g, dtype=torch.float64), torch.randn(shape, generator=g, dtype=torch.float64)
    x = ref.add_noise(lat, z0, timesteps[:1])
    got0 = tab[0, 3] * lat + tab[0, 0] * z0
    assert float((got0 - x).abs().max() / x.abs().max()) < 1e-6        # the row holds fp32-rounded scalars
    assert torch.allclose(ref.scale_model_input(x, start), tab[0, 1] * x, rtol=1e-6, atol=0)
    for j in range(k):
        i = start + j
        m_u, m_c, z = (torch.randn(shape, generator=g, dtype=torch.float64) for _ in range(3))
        m_hat = m_u + 7.0 * (m_c - m_u)
        want = ref.step(m_hat, i, x, z)
        alpha, beta, gamma, s_next, t_next = schedulers.coefficients(scheduler, prediction_type, n)[1][i]
        row = tab[1 + j]
        got = alpha * x + beta * m_hat + gamma * z
        scale = (alpha * x).abs() + (beta * m_hat).abs() + (gamma * z).abs()
        assert float(((got - want).abs() / scale).max()) < 1e-12, i
        got32 = row[0] * x + row[1] * m_hat + row[2] * z
        assert float(((got32 - want).abs() / scale).max()) < 1e-6, i
        assert bool(row[5] == (1.0 if j == k - 1 else 0.0))
        if j + 1 < k:
            assert float(row[4]) == float(np.float32(timesteps[j + 1]))      # the table is fp32
        x = want


# ------------------------------------------------------------------------------------ preprocessing
def test_both_pipelines_preprocessing_equals_the_ingest_for_every_uint8_value():
    from oracle import sample_image_ref as RI
    v = torch.arange(256, dtype=torch.uint8)
    ingest = (v.float() / 255 - 0.5) / 0.5                  # lb_pixels_ingest's normalise_u8, op by op
    img = v.reshape(1, 16, 16, 1).expand(1, 16, 16, 3).contiguous()
    i2i = RI.preprocess(img)                                 # 2.0 * (u8 / 255.0) - 1.0
    mask, masked = RI.prepare_mask_and_masked_image(img, torch.zeros(1, 16, 16, dtype=torch.uint8))
    inp = masked                                             # u8 / 127.5 - 1.0, times (0 < 0.5) = 1
    for got in (i2i, inp):
        assert got.dtype == torch.float32
        for c in range(3):
            assert torch.equal(got[0, c].reshape(-1).view(torch.int32), ingest.view(torch.int32))
    # the numpy restatement itself, value by value
    a = np.arange(256, dtype=np.float32)
    np.testing.assert_array_equal((2.0 * (a / 255.0) - 1.0).view(np.int32), ingest.numpy().view(np.int32))
    np.testing.assert_array_equal((a / np.float32(127.5) - 1.0).astype(np.float32).view(np.int32),
                                  ingest.numpy().view(np.int32))


def test_pipeline_mask_threshold_falls_between_127_and_128():
    from oracle import sample_image_ref as RI
    v = torch.arange(256, dtype=torch.uint8).reshape(1, 16, 16)
    img = torch.full((1, 16, 16, 3), 200, dtype=torch.uint8)
    mask, masked = RI.prepare_mask_and_masked_image(img, v)
    m = mask.reshape(-1)
    assert m[:128].eq(0).all() and m[128:].eq(1).all()
    # masked image: kept where the mask is 0, zeroed where it is 1
    keep = masked[0, 0].reshape(-1)
    assert keep[:128].ne(0).all() and keep[128:].eq(0).all()
    # the kernel's binarisation, v / 255.f >= 0.5
    assert ((v.float() / 255) >= 0.5).reshape(-1).float().equal(m)


# ------------------------------------------------------------------------------------ C-ABI
def _lib():
    from lora_b200 import _C
    return _C


def test_new_entry_points_are_declared_and_exported():
    import os
    C = _lib()
    hdr = open(os.path.join(os.path.dirname(C.__file__), "..", "include", "lora_b200.h")).read()
    for name in ("lb_sample_init", "lb_sample_step_ch", "lb_pixels_ingest_inpaint"):
        assert f"int {name}(" in hdr and name in C.EXPORTED and hasattr(C.lib, name)


SHAPE, DTYPE = -1, -3


def test_sample_init_refuses_bad_arguments_without_gpu():
    C = _lib()
    p = ctypes.c_void_p(256)         # never dereferenced: every call below is refused before any CUDA call

    def call(mom=p, md=C.LB_BF16, pe=p, ed=C.LB_BF16, mask=None, noise=p, table=p, rows=51, x=p, idx=p, cnt=p,
             uin=p, udt=C.LB_BF16, uch=4, ts=p, G=2, B=1, Ch=4, H=8, W=8):
        return C.lib.lb_sample_init(mom, md, 256, 64, 1, pe, ed, 0.18215, mask, noise, table, rows, x, idx, cnt,
                                    uin, udt, uch, ts, G, B, Ch, H, W, None)
    assert call(B=0) == SHAPE and call(W=-1) == SHAPE and call(G=3) == SHAPE and call(rows=1) == SHAPE
    assert call(udt=9) == DTYPE and call(md=7) == DTYPE and call(ed=C.LB_F16) == DTYPE
    assert call(x=None) == SHAPE and call(noise=None) == SHAPE and call(table=None) == SHAPE
    assert call(idx=None) == SHAPE and call(cnt=None) == SHAPE and call(uin=None) == SHAPE and call(ts=None) == SHAPE
    assert call(pe=None) == SHAPE
    # unet_channels: C without a mask, 2C + 1 with one; a mask needs the masked image's moments
    assert call(uch=9) == SHAPE and call(mask=p, uch=4) == SHAPE and call(mask=p, uch=9, mom=None) == SHAPE
    # without moments (the txt2img start) neither moments' dtype nor the posterior noise is read
    assert call(mom=None, md=7, pe=None, uch=5) == SHAPE


def test_sample_step_ch_refuses_bad_arguments_without_gpu():
    C = _lib()
    p = ctypes.c_void_p(256)

    def call(model=p, mdt=C.LB_BF16, G=2, x=p, rows=51, guid=p, uin=p, udt=C.LB_BF16, uch=9, vin=p, vdt=C.LB_F32,
             scaling=0.18215, B=1, Ch=4, init=0):
        return C.lib.lb_sample_step_ch(model, mdt, 256, 1, 4, G, x, p, p, rows, guid, p, p, uin, udt, uch, p, vin,
                                       vdt, 0, scaling, B, Ch, 8, 8, init, None)
    assert call(uch=3) == SHAPE and call(uch=-1) == SHAPE
    assert call(B=0) == SHAPE and call(G=0) == SHAPE and call(rows=1) == SHAPE
    assert call(mdt=7) == DTYPE and call(udt=9) == DTYPE and call(vdt=-1) == DTYPE
    assert call(model=None) == SHAPE and call(guid=None) == SHAPE and call(vin=None) == SHAPE
    assert call(x=None) == SHAPE and call(uin=None) == SHAPE and call(scaling=0.0) == SHAPE


def test_pixels_ingest_inpaint_refuses_bad_arguments_without_gpu():
    C = _lib()
    p = ctypes.c_void_p(256)
    f = C.lib.lb_pixels_ingest_inpaint
    assert f(p, p, p, C.LB_BF16, 1, 0, 8, 8, None) == SHAPE
    assert f(None, p, p, C.LB_BF16, 1, 1, 8, 8, None) == SHAPE
    assert f(p, None, p, C.LB_BF16, 1, 1, 8, 8, None) == SHAPE
    assert f(p, p, None, C.LB_BF16, 1, 1, 8, 8, None) == SHAPE
    assert f(p, p, p, 5, 1, 1, 8, 8, None) == DTYPE


# ------------------------------------------------------------------------------------ construction
def _tiny(in_channels=4):
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    cfg = UNetConfig.tiny()
    cfg.in_channels = in_channels
    return (UNet2DConditionModel(cfg), build_text_encoder(tiny=True),
            AutoencoderKL(VAEConfig.tiny(), with_decoder=True))


SHAPE4 = (1, 4, 8, 8)


def test_task_and_in_channels_mismatches_are_refused():
    from lora_b200.sample import LoraSampler, SamplerConfig
    unet4, text, vae = _tiny()
    unet9 = _tiny(in_channels=9)[0]
    with pytest.raises(ValueError, match="inpainting"):
        LoraSampler(unet9, text, vae, SamplerConfig(), latent_shape=SHAPE4, device="cpu")
    with pytest.raises(ValueError, match="inpainting"):
        LoraSampler(unet9, text, vae, SamplerConfig(task="img2img"), latent_shape=SHAPE4, device="cpu")
    with pytest.raises(ValueError, match="9 input channels"):
        LoraSampler(unet4, text, vae, SamplerConfig(task="inpaint"), latent_shape=SHAPE4, device="cpu")
    with pytest.raises(ValueError, match="task"):
        LoraSampler(unet4, text, vae, SamplerConfig(task="outpaint"), latent_shape=SHAPE4, device="cpu")


def test_strength_outside_the_unit_interval_is_refused():
    from lora_b200.sample import LoraSampler, SamplerConfig
    unet4, text, vae = _tiny()
    for s in (0.0, -0.1, 1.5):
        for task in ("img2img", "txt2img"):
            with pytest.raises(ValueError, match="strength"):
                LoraSampler(unet4, text, vae, SamplerConfig(task=task, strength=s), latent_shape=SHAPE4, device="cpu")
    # int(10 * 0.05) == 0: no step would run
    with pytest.raises(ValueError, match="no denoising step"):
        LoraSampler(unet4, text, vae, SamplerConfig(task="img2img", strength=0.05, num_inference_steps=10,
                                                    max_steps=10), latent_shape=SHAPE4, device="cpu")


def test_valid_img2img_and_inpaint_samplers_construct_and_check_their_inputs():
    from lora_b200.sample import LoraSampler, SamplerConfig
    unet4, text, vae = _tiny()
    unet9 = _tiny(in_channels=9)[0]
    cfg = dict(num_inference_steps=10, max_steps=10)
    s = LoraSampler(unet4, text, vae, SamplerConfig(task="img2img", strength=0.75, **cfg), latent_shape=SHAPE4,
                    device="cpu")
    assert s.captures == 0 and tuple(s.pixels.shape) == (1, 64, 64, 3)
    assert tuple(s.posterior_noise.shape) == SHAPE4 and s.posterior_noise.dtype == torch.float32
    assert tuple(s.unet_in[2].shape) == (2, 4, 8, 8)
    ids = torch.zeros(1, 77, dtype=torch.long)
    img = torch.zeros(1, 64, 64, 3, dtype=torch.uint8)
    mask = torch.zeros(1, 64, 64, dtype=torch.uint8)
    for kw in (dict(), dict(image=img[..., :2]), dict(image=img.float()), dict(image=img[:, :32]),
               dict(image=img, mask_image=mask)):
        with pytest.raises(ValueError):
            s.sample(ids, ids, **kw)
    with pytest.raises(ValueError, match="strength"):
        s.sample(ids, ids, image=img, strength=1.5)
    with pytest.raises(ValueError, match="no denoising step"):
        s.sample(ids, ids, image=img, strength=0.05)
    si = LoraSampler(unet9, text, vae, SamplerConfig(task="inpaint", **cfg), latent_shape=SHAPE4, device="cpu")
    assert tuple(si.unet_in[2].shape) == (2, 9, 8, 8) and tuple(si.mask_image.shape) == (1, 64, 64)
    for kw in (dict(image=img), dict(mask_image=mask), dict(image=img, mask_image=mask[:, :, :32]),
               dict(image=img, mask_image=mask.float()), dict(image=img, mask_image=mask[:, None]),
               dict(image=img, mask_image=mask, strength=0.5)):
        with pytest.raises(ValueError):
            si.sample(ids, ids, **kw)
    st = LoraSampler(unet4, text, vae, SamplerConfig(**cfg), latent_shape=SHAPE4, device="cpu")
    with pytest.raises(ValueError, match="txt2img"):
        st.sample(ids, ids, image=img)
    with pytest.raises(ValueError, match="strength"):
        st.sample(ids, ids, strength=0.5)
