"""DPM-Solver++(2M) sampling on the GPU: lb_sample_step_ms against a float64 evaluation of its row form
(model dtypes, layouts, G, the 9-channel UNet input, the last step, an unread NaN history), one
captured launch replayed as every step with the history chained, and the sampler -- graph replay
against its eager path and both against the oracle's op-by-op scheduler (oracle/sample_dpm_ref.py) in
the pipeline loops of oracle/sample_ref.py and oracle/sample_image_ref.py -- for txt2img, img2img and
inpainting on tiny models and at SD1.5 512 px, switching scheduler families on one sampler, and
sampling between training steps.

Oracle bound, as for Euler-ancestral and DDIM: the sampler's error against the oracle's float64 run is
at most twice the oracle's own error in the run's dtype (bf16 autocast) against that float64 run."""
import copy

import pytest
import torch

from oracle.sample_dpm_ref import RefDPMSolverMultistep
from test_sample_gpu import _train
from test_sample_image_gpu import LAT, _bits, _ids, _images, _models, _noise_pair, _rel, _sampler

pytestmark = pytest.mark.gpu
DEV = "cuda"
DPM = "dpmsolver_multistep"


# ------------------------------------------------------------------------------------ kernel
def _ms_table(rows, g):
    """Random (a, b, d, s_next, t_next, last, p, q) rows of DPM-like magnitudes, `last` on the final row."""
    tab = torch.zeros(rows, 8)
    tab[0, :3] = torch.tensor([1.0, 1.0, 999.0])
    tab[1:, 0] = 0.7 + torch.rand(rows - 1, generator=g) * 0.3
    tab[1:, 1] = 0.05 + torch.rand(rows - 1, generator=g) * 0.5
    tab[1:, 2] = -torch.rand(rows - 1, generator=g) * 0.2
    tab[1:, 3] = 0.5 + torch.rand(rows - 1, generator=g)
    tab[1:, 4] = torch.arange(rows - 1, 0, -1).float() * 50.0
    tab[1:, 6] = 1 + torch.rand(rows - 1, generator=g) * 10
    tab[1:, 7] = -torch.rand(rows - 1, generator=g) * 10
    tab[rows - 1, 5] = 1.0
    return tab


def _bufs(B, C, H, W, G, Cu, sentinel=None):
    idx, cnt = torch.zeros(1, device=DEV, dtype=torch.int32), torch.zeros(1, device=DEV, dtype=torch.int32)
    ts = torch.zeros(1, device=DEV)
    unet_in = torch.zeros(G * B, Cu, H, W, device=DEV, dtype=torch.bfloat16)
    if sentinel is not None:
        unet_in[:, C:] = sentinel
    unet_in = unet_in.contiguous(memory_format=torch.channels_last)
    vae_in = torch.full((B, C, H, W), float("nan"), device=DEV, dtype=torch.float16)
    return idx, cnt, ts, unet_in, vae_in


@pytest.mark.parametrize("mdt", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("channels_last", [True, False])
@pytest.mark.parametrize("G", [1, 2])
@pytest.mark.parametrize("Cu", [4, 9])
@pytest.mark.parametrize("last", [False, True])
def test_sample_step_ms_matches_float64(mdt, channels_last, G, Cu, last):
    from lora_b200.step_ops import sample_step_ms
    g = torch.Generator().manual_seed(G + 2 * int(channels_last) + 4 * Cu + 8 * int(last))
    B, C, H, W = 3, 4, 12, 20
    rows = 4
    tab = _ms_table(rows, g)
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    mo = (torch.randn(G * B, C, H, W, generator=g) * 2).to(mdt).to(DEV).contiguous(memory_format=fmt)
    x_start = (torch.randn(B, C, H, W, generator=g) * 3).to(DEV)
    h_start = torch.randn(B, C, H, W, generator=g).to(DEV)
    sentinel = torch.randn(G * B, Cu - C, H, W, generator=g).to(torch.bfloat16).to(DEV) if Cu > C else None
    x, hist = x_start.clone(), h_start.clone()
    gs = torch.tensor([7.0], device=DEV)
    idx, cnt, ts, unet_in, vae_in = _bufs(B, C, H, W, G, Cu, sentinel)
    k = 2 if last else 1                         # row 1 + k; the last row is rows - 1
    idx.fill_(k)
    sample_step_ms(mo, x, hist, tab.to(DEV), gs, idx, cnt, unet_in, ts, vae_in, 0.18215)
    torch.cuda.synchronize()
    row = tab[1 + k].double()
    a, b, d, s_next, t_next, _, p, q = row.tolist()
    m = mo.double().cpu()
    m_hat = m[:B] if G == 1 else m[:B] + 7.0 * (m[B:] - m[:B])
    m_mag = m[:B].abs() + (7.0 * (m[B:] - m[:B]).abs() if G == 2 else 0)
    xd, hd = x_start.double().cpu(), h_start.double().cpu()
    x0 = p * xd + q * m_hat
    want = a * xd + b * x0 + d * hd
    x0_mag = (p * xd).abs() + abs(q) * m_mag
    bound = (a * xd).abs() + abs(b) * x0_mag + (d * hd).abs()
    err = (x.double().cpu() - want).abs()
    assert bool((err <= 8 * 2 ** -23 * bound + 1e-30).all()), float((err / bound).max())
    err0 = (hist.double().cpu() - x0).abs()
    assert bool((err0 <= 4 * 2 ** -23 * x0_mag + 1e-30).all()), float((err0 / x0_mag).max())
    want_in = (s_next * x).to(torch.bfloat16)
    for h in range(G):
        assert torch.equal(_bits(unet_in[h * B:(h + 1) * B, :C]), _bits(want_in))
    if Cu > C:
        assert torch.equal(_bits(unet_in[:, C:]), _bits(sentinel))
    assert float(ts) == t_next and int(idx) == k + 1 and int(cnt) == 0
    if last:
        assert torch.equal(_bits(vae_in), _bits((1 / 0.18215 * x).to(torch.float16)))
    else:
        assert bool(torch.isnan(vae_in.float()).all())          # not the last step: the decoder input is untouched


@pytest.mark.parametrize("G", [1, 2])
def test_first_order_row_does_not_read_a_nan_history(G):
    from lora_b200.step_ops import sample_step_ms
    g = torch.Generator().manual_seed(G)
    B, C, H, W = 2, 4, 8, 12
    tab = _ms_table(3, g)
    tab[1:, 2] = 0.0                             # d = 0: first-order rows
    tab = tab.to(DEV)
    mo = torch.randn(G * B, C, H, W, generator=g).to(torch.bfloat16).to(DEV)
    x_start = torch.randn(B, C, H, W, generator=g).to(DEV)
    gs = torch.tensor([5.0], device=DEV)
    res = []
    for fill in (float("nan"), 0.0):
        x, hist = x_start.clone(), torch.full((B, C, H, W), fill, device=DEV)
        idx, cnt, ts, unet_in, vae_in = _bufs(B, C, H, W, G, C)
        sample_step_ms(mo, x, hist, tab, gs, idx, cnt, unet_in, ts, vae_in, 0.18215)
        sample_step_ms(mo, x, hist, tab, gs, idx, cnt, unet_in, ts, vae_in, 0.18215)     # the last row
        torch.cuda.synchronize()
        res.append((x, hist, unet_in, vae_in))
    (x, h, u, v), (x2, h2, u2, v2) = res
    assert bool(torch.isfinite(x).all() and torch.isfinite(h).all() and torch.isfinite(v.float()).all())
    assert torch.equal(_bits(x), _bits(x2)) and torch.equal(_bits(h), _bits(h2))
    assert torch.equal(_bits(u), _bits(u2)) and torch.equal(_bits(v), _bits(v2))


def test_sample_step_ms_replays_one_captured_launch_as_every_step():
    from lora_b200.host import schedulers
    from lora_b200.step_ops import sample_step, sample_step_ms
    g = torch.Generator().manual_seed(0)
    B, C, H, W = 2, 4, 16, 16
    N = 6
    tab = schedulers.pack_table(DPM, "epsilon", N, N).to(DEV)
    noise = torch.randn(N + 1, B, C, H, W, generator=g).to(DEV)
    mos = [torch.randn(2 * B, C, H, W, generator=g).to(DEV) for _ in range(N)]
    mo = torch.empty_like(mos[0])
    gs = torch.tensor([3.0], device=DEV)

    def state():
        x, hist = torch.zeros(B, C, H, W, device=DEV), torch.full((B, C, H, W), float("nan"), device=DEV)
        idx, cnt = torch.zeros(1, device=DEV, dtype=torch.int32), torch.zeros(1, device=DEV, dtype=torch.int32)
        ts = torch.zeros(1, device=DEV)
        unet_in = torch.zeros(2 * B, C, H, W, device=DEV).contiguous(memory_format=torch.channels_last)
        return x, hist, idx, cnt, ts, unet_in, torch.zeros(B, C, H, W, device=DEV)

    x, hist, idx, cnt, ts, unet_in, vae_in = st = state()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        sample_step(None, x, noise, tab, None, idx, cnt, unet_in, ts, None, 0.18215, init=True)
        sample_step_ms(mo, x, hist, tab, gs, idx, cnt, unet_in, ts, vae_in, 0.18215)
    torch.cuda.current_stream().wait_stream(s)
    gb = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gb):
        sample_step_ms(mo, x, hist, tab, gs, idx, cnt, unet_in, ts, vae_in, 0.18215)
    ex, eh, eidx, ecnt, ets, eu, ev = est = state()
    sample_step(None, x, noise, tab, None, idx, cnt, unet_in, ts, None, 0.18215, init=True)
    sample_step(None, ex, noise, tab, None, eidx, ecnt, eu, ets, None, 0.18215, init=True)
    hist.fill_(float("nan"))
    t = tab.double().cpu()
    xd, hd = noise[0].double().cpu(), None
    for i in range(N):
        mo.copy_(mos[i])
        gb.replay()
        sample_step_ms(mos[i], ex, eh, tab, gs, eidx, ecnt, eu, ets, ev, 0.18215)
        torch.cuda.synchronize()
        for a, b in zip(st, est):
            assert torch.equal(_bits(a), _bits(b)), i
        a_, b_, d_, _, t_next, _, p, q = t[1 + i].tolist()
        m = mos[i].double().cpu()
        x0 = p * xd + q * (m[:B] + 3.0 * (m[B:] - m[:B]))
        xd = a_ * xd + b_ * x0 + (d_ * hd if d_ != 0.0 else 0.0)
        hd = x0
        assert int(idx) == i + 1 and float(ts) == t_next
        assert _rel(x, xd) < 1e-5 and _rel(hist, x0) < 1e-5, i
    assert torch.equal(vae_in, 1 / 0.18215 * x)


# ------------------------------------------------------------------------------------ tiny models
def _oracle_txt2img(unet_r, text_r, vae, pred, n, ids, neg, noise):
    from oracle import sample_ref as R
    f64 = [copy.deepcopy(m).double() for m in (unet_r, text_r, vae)]
    args = (ids, neg, noise, 7.0)
    _, lat64 = R.sample(*f64, RefDPMSolverMultistep(pred), n, *args, dtype=torch.float64)
    _, lat_run = R.sample(unet_r, text_r, vae, RefDPMSolverMultistep(pred), n, *args, dtype=torch.float32,
                          autocast_dtype=torch.bfloat16)
    return lat64, lat_run


@pytest.mark.parametrize("prediction_type", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("n", [10, 12])
def test_tiny_txt2img_graph_equals_eager_and_oracle(prediction_type, n):
    unet, text, vae, unet_r, text_r = _models()
    ids, neg = _ids(text)
    kw = dict(scheduler=DPM, prediction_type=prediction_type, external_noise=True, num_inference_steps=n)
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
    assert torch.equal(sg.x0_hist, se.x0_hist)
    lat64, lat_run = _oracle_txt2img(unet_r, text_r, vae, prediction_type, n, ids, neg, noise[:n + 1])
    e_ours, e_ref = _rel(sg.latents, lat64), _rel(lat_run, lat64)
    assert e_ours <= 2 * e_ref, (e_ours, e_ref)


@pytest.mark.parametrize("prediction_type", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("strength", [0.3, 0.75])
def test_tiny_img2img_graph_equals_eager_and_oracle(prediction_type, strength):
    from oracle import sample_image_ref as RI
    unet, text, vae, unet_r, text_r = _models()
    ids, neg = _ids(text)
    img, _ = _images()
    n = 20
    kw = dict(task="img2img", strength=strength, scheduler=DPM, prediction_type=prediction_type,
              external_noise=True, num_inference_steps=n, max_steps=n)
    sg, se = _sampler(unet, text, vae, True, **kw), _sampler(unet, text, vae, False, **kw)
    noise, peps = _noise_pair(sg, se)
    sg.prepare()
    img_g = sg.sample(ids, neg, image=img).clone()
    img_e = se.sample(ids, neg, image=img).clone()
    assert sg.captures == 1
    assert torch.equal(img_g, img_e) and torch.equal(sg.latents, se.latents)
    k = int(n * strength)
    args = (ids, neg, img, noise[:k + 1], peps, 7.0)
    f64 = [copy.deepcopy(m).double() for m in (unet_r, text_r, vae)]
    _, lat64 = RI.sample_img2img(*f64, RefDPMSolverMultistep(prediction_type), n, strength, *args,
                                 dtype=torch.float64)
    _, lat_run = RI.sample_img2img(unet_r, text_r, vae, RefDPMSolverMultistep(prediction_type), n, strength,
                                   *args, dtype=torch.float32, autocast_dtype=torch.bfloat16)
    e_ours, e_ref = _rel(sg.latents, lat64), _rel(lat_run, lat64)
    assert e_ours <= 2 * e_ref, (e_ours, e_ref)


def test_tiny_inpaint_graph_equals_eager_and_oracle():
    from oracle import sample_image_ref as RI
    unet, text, vae, unet_r, text_r = _models(in_channels=9)
    ids, neg = _ids(text)
    img, mask = _images()
    kw = dict(task="inpaint", scheduler=DPM, external_noise=True)
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
    _, lat64 = RI.sample_inpaint(*f64, RefDPMSolverMultistep("epsilon"), n, *args, dtype=torch.float64)
    _, lat_run = RI.sample_inpaint(unet_r, text_r, vae, RefDPMSolverMultistep("epsilon"), n, *args,
                                   dtype=torch.float32, autocast_dtype=torch.bfloat16)
    e_ours, e_ref = _rel(sg.latents, lat64), _rel(lat_run, lat64)
    assert e_ours <= 2 * e_ref, (e_ours, e_ref)


# ------------------------------------------------------------------------------------ families
def test_family_switch_captures_once_and_leaves_the_euler_images_alone():
    from lora_b200 import ops
    unet, text, vae, *_ = _models()
    ids, neg = _ids(text)
    s, e = _sampler(unet, text, vae, True), _sampler(unet, text, vae, False)
    a = s.sample(ids, neg, seed=3).clone()
    la = s.latents.clone()
    assert s.captures == 1
    dpm = s.sample(ids, neg, seed=3, scheduler=DPM).clone()
    assert s.captures == 2
    assert torch.equal(dpm, e.sample(ids, neg, seed=3, scheduler=DPM)) and torch.equal(s.latents, e.latents)
    b = s.sample(ids, neg, seed=3).clone()
    assert s.captures == 2
    assert torch.equal(a, b) and torch.equal(la, s.latents)
    # within a family no call captures: DDIM after Euler, and DPM again at other steps and seeds
    s.sample(ids, neg, seed=4, scheduler="ddim")
    d2 = s.sample(ids, neg, seed=5, scheduler=DPM, num_inference_steps=12).clone()
    assert s.captures == 2
    assert torch.equal(d2, e.sample(ids, neg, seed=5, scheduler=DPM, num_inference_steps=12))
    # launches per denoising step: the UNet forward + 1, as for the single-step schedulers
    unet.eval()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        c0 = ops.LAUNCH_COUNT
        unet(e.unet_in[2], e.timestep, e._ehs[2])
        fwd = ops.LAUNCH_COUNT - c0
        c0 = ops.LAUNCH_COUNT
        e._body_b(2, "multistep")
        step = ops.LAUNCH_COUNT - c0
    unet.train()
    assert fwd > 0 and step == fwd + 1


def test_dpm_sampling_between_training_steps_changes_nothing():
    import lora_b200 as L
    unet, text, vae, *_ = _models()
    u2, t2 = copy.deepcopy(unet), copy.deepcopy(text)
    ids, neg = _ids(text)
    s = _sampler(unet, text, vae, True, scheduler=DPM)
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
    L.link_sites(u3, t3)
    fresh = _sampler(u3, t3, vae, False, scheduler=DPM)
    fresh.sample(ids, neg, seed=0)
    assert torch.equal(imgs[-1], fresh.image) and torch.equal(s.latents, fresh.latents)
    assert unet.training and text.training


# ------------------------------------------------------------------------------------ full size
def test_full_size_sd15_512_dpm_20_graph_equals_eager_and_oracle():
    import lora_b200 as L
    from lora_b200.host.unet_sd15 import UNetConfig
    from lora_b200.sample import LoraSampler, SamplerConfig
    from oracle import sample_ref as R
    from test_sample_gpu import _full
    n, lat = 20, (1, 4, 64, 64)
    unet, text, vae, unet_r, text_r = _full(UNetConfig(), False)
    L.set_grouping(True)
    try:
        cfg = dict(scheduler=DPM, num_inference_steps=n, max_steps=n, guidance_scale=7.0,
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
        _, lat_run = R.sample(unet_r, text_r, vae, RefDPMSolverMultistep("epsilon"), n, *args,
                              dtype=torch.float32, autocast_dtype=torch.bfloat16)
        f64 = [copy.deepcopy(m).double() for m in (unet_r, text_r)]
        vae64 = copy.deepcopy(vae).double()
        del unet_r, text_r
        _, lat64 = R.sample(f64[0], f64[1], vae64, RefDPMSolverMultistep("epsilon"), n, *args,
                            dtype=torch.float64)
        e_ours, e_ref = _rel(sg.latents, lat64), _rel(lat_run, lat64)
        assert e_ours <= 2 * e_ref, (e_ours, e_ref)
    finally:
        L.set_grouping(False)
