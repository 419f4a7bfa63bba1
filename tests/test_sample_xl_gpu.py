"""SDXL sampling and guidance rescale on the GPU.

Kernel: lb_sample_step_rescale against a float64 evaluation (model dtypes, layouts, B, a pixel count
that is not a multiple of the cluster's stride, 4 or 9 UNet channels, both scheduler families, phi), bit
equality with lb_sample_step_ch / lb_sample_step_ms at phi = 0, and one captured launch replayed as every
step, bit-reproducibly.
Samplers: LoraXLSampler on the tiny SDXL preset and LoraSampler with guidance rescale -- graph replay
against the eager path and both against the pipeline-style oracle loop (oracle/sample_xl_ref.py) --
zeroed and encoded negatives, per-call time ids, capture counts, launches per step, and sampling between
LoraXLTrainStep steps. Census: the fused forward at the SDXL sampling shapes (G*B = 2 at 1024 px). Full
size: SDXL 1024 px, 20 Euler steps, phi = 0 and 0.7.

Oracle bound, as for the other samplers: the sampler's error against the oracle's float64 run is at most
twice the oracle's own error in the run's dtype (bf16 autocast) against that float64 run.

On the tiny SDXL preset the graph-replayed and eager paths are not bit-identical: they differ by a few
bf16 roundings on the text side, which ten guided steps of a random UNet grow to about 1e-2 relative in
the latents (the SD samplers, the rescale launch included, do replay their eager path bit for bit). The
tiny SDXL tests therefore hold both paths to the oracle bound and the distance between them to twice the
oracle's own bf16 error, or to XL_GRAPH_EAGER where no oracle runs; a change of the result is read off the
graph path, whose replays repeat bit for bit. At full size the two paths are bit-identical."""
import contextlib
import copy

import pytest
import torch

import test_conv_kernels_gpu as CK
import test_kernels_gpu as KG
from test_sample_image_gpu import _bits, _rel
from test_sdxl_gpu import CONV_SDXL, _ids, _xl_pair

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
SCHEDULERS = ["euler", "euler_ancestral", "ddim", "dpmsolver_multistep"]
XL_GRAPH_EAGER = 3e-2          # rel. distance of graph and eager latents on the tiny SDXL preset (see above)


# ------------------------------------------------------------------------------------ kernel
def _table(rows, g, ms):
    """Random rows of scheduler-like magnitudes; single-step rows have gamma != 0, `last` on the final row."""
    tab = torch.zeros(rows, 8)
    tab[0, :3] = torch.tensor([1.0, 1.0, 999.0])
    tab[1:, 0] = 0.7 + torch.rand(rows - 1, generator=g) * 0.3
    tab[1:, 1] = -(0.05 + torch.rand(rows - 1, generator=g) * 0.5)
    tab[1:, 2] = (-torch.rand(rows - 1, generator=g) * 0.2) if ms else (0.1 + torch.rand(rows - 1, generator=g))
    tab[1:, 3] = 0.5 + torch.rand(rows - 1, generator=g)
    tab[1:, 4] = torch.arange(rows - 1, 0, -1).float() * 50.0
    if ms:
        tab[1:, 6] = 1 + torch.rand(rows - 1, generator=g) * 10
        tab[1:, 7] = -torch.rand(rows - 1, generator=g) * 10
    tab[rows - 1, 5] = 1.0
    return tab


def _state(B, C, H, W, Cu, g, sentinel):
    idx, cnt = torch.zeros(1, device=DEV, dtype=torch.int32), torch.zeros(1, device=DEV, dtype=torch.int32)
    ts = torch.zeros(1, device=DEV)
    unet_in = torch.zeros(2 * B, Cu, H, W, device=DEV, dtype=BF)
    if Cu > C:
        unet_in[:, C:] = sentinel
    unet_in = unet_in.contiguous(memory_format=torch.channels_last)
    vae_in = torch.full((B, C, H, W), float("nan"), device=DEV, dtype=torch.float16)
    return idx, cnt, ts, unet_in, vae_in


def _run_step(rescale, ms, mo, x, noise, hist, tab, gs, phi, st):
    from lora_b200.step_ops import sample_step_ch, sample_step_ms, sample_step_rescale
    idx, cnt, ts, unet_in, vae_in = st
    if rescale:
        sample_step_rescale(mo, x, None if ms else noise, hist if ms else None, tab, gs, phi, idx, cnt, unet_in, ts,
                            vae_in, 0.13025)
    elif ms:
        sample_step_ms(mo, x, hist, tab, gs, idx, cnt, unet_in, ts, vae_in, 0.13025)
    else:
        sample_step_ch(mo, x, noise, tab, gs, idx, cnt, unet_in, ts, vae_in, 0.13025)


@pytest.mark.parametrize("mdt", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("channels_last", [True, False])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("Cu", [4, 9])
@pytest.mark.parametrize("ms", [False, True])
@pytest.mark.parametrize("phi", [0.3, 0.7, 1.0])
def test_sample_step_rescale_matches_float64(mdt, channels_last, B, Cu, ms, phi):
    g = torch.Generator().manual_seed(B + 4 * Cu + 16 * int(ms) + 32 * int(channels_last) + int(phi * 64))
    C, H, W = 4, 45, 50                  # P = 2250: past one 8 x 256 stride, not a multiple of it
    rows = 4
    tab = _table(rows, g, ms)
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    mo = (torch.randn(2 * B, C, H, W, generator=g) * 2 + 0.3).to(mdt).to(DEV).contiguous(memory_format=fmt)
    x_start = (torch.randn(B, C, H, W, generator=g) * 3).to(DEV)
    h_start = torch.randn(B, C, H, W, generator=g).to(DEV)
    noise = torch.randn(rows, B, C, H, W, generator=g).to(DEV)
    sentinel = torch.randn(2 * B, Cu - C, H, W, generator=g).to(BF).to(DEV) if Cu > C else None
    x, hist = x_start.clone(), h_start.clone()
    gs, ph = torch.tensor([5.0], device=DEV), torch.tensor([phi], device=DEV)
    st = _state(B, C, H, W, Cu, g, sentinel)
    k = 2 if B == 3 else 1               # B = 3 runs the last row
    st[0].fill_(k)
    _run_step(True, ms, mo, x, noise, hist, tab.to(DEV), gs, ph, st)
    torch.cuda.synchronize()
    idx, cnt, ts, unet_in, vae_in = st
    a, b, d, s_next, t_next, last, p, q = tab[1 + k].double().tolist()
    m = mo.double().cpu()
    mu, mc = m[:B], m[B:]
    m_hat = mu + 5.0 * (mc - mu)
    r = mc.std(dim=(1, 2, 3), keepdim=True) / m_hat.std(dim=(1, 2, 3), keepdim=True)
    kb = phi * r + (1 - phi)
    m_r = kb * m_hat
    m_mag = kb.abs() * (mu.abs() + 5.0 * (mc - mu).abs())
    xd = x_start.double().cpu()
    if ms:
        hd = h_start.double().cpu()
        x0 = p * xd + q * m_r
        want = a * xd + b * x0 + d * hd
        x0_mag = (p * xd).abs() + abs(q) * m_mag
        bound = (a * xd).abs() + abs(b) * x0_mag + (d * hd).abs()
        err0 = (hist.double().cpu() - x0).abs()
        assert bool((err0 <= 8 * 2 ** -23 * x0_mag + 1e-30).all()), float((err0 / x0_mag).max())
    else:
        z = noise[1 + k].double().cpu()
        want = a * xd + b * m_r + d * z
        bound = (a * xd).abs() + abs(b) * m_mag + (d * z).abs()
    err = (x.double().cpu() - want).abs()
    assert bool((err <= 12 * 2 ** -23 * bound + 1e-30).all()), float((err / bound).max())
    want_in = (s_next * x).to(BF)
    for h in range(2):
        assert torch.equal(_bits(unet_in[h * B:(h + 1) * B, :C]), _bits(want_in))
    if Cu > C:
        assert torch.equal(_bits(unet_in[:, C:]), _bits(sentinel))
    assert float(ts) == t_next and int(idx) == k + 1 and int(cnt) == 0
    if last:
        assert torch.equal(_bits(vae_in), _bits((1 / 0.13025 * x).to(torch.float16)))
    else:
        assert bool(torch.isnan(vae_in.float()).all())


@pytest.mark.parametrize("mdt", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("channels_last", [True, False])
@pytest.mark.parametrize("Cu", [4, 9])
@pytest.mark.parametrize("ms", [False, True])
def test_phi_zero_is_bit_equal_to_the_plain_step(mdt, channels_last, Cu, ms):
    g = torch.Generator().manual_seed(Cu + 16 * int(ms) + 32 * int(channels_last))
    B, C, H, W = 3, 4, 45, 50
    rows = 4
    tab = _table(rows, g, ms).to(DEV)
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    mo = (torch.randn(2 * B, C, H, W, generator=g) * 2).to(mdt).to(DEV).contiguous(memory_format=fmt)
    x_start = (torch.randn(B, C, H, W, generator=g) * 3).to(DEV)
    h_start = torch.randn(B, C, H, W, generator=g).to(DEV)
    noise = torch.randn(rows, B, C, H, W, generator=g).to(DEV)
    sentinel = torch.randn(2 * B, Cu - C, H, W, generator=g).to(BF).to(DEV) if Cu > C else None
    gs, ph = torch.tensor([7.5], device=DEV), torch.tensor([0.0], device=DEV)
    outs = []
    for rescale in (False, True):
        x, hist = x_start.clone(), h_start.clone()
        st = _state(B, C, H, W, Cu, g, sentinel)
        for _ in range(rows - 1):                    # every row, the last included
            _run_step(rescale, ms, mo, x, noise, hist, tab, gs, ph, st)
        torch.cuda.synchronize()
        outs.append((x, hist) + st)
    for a, b in zip(*outs):
        assert torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("scheduler", ["euler", "dpmsolver_multistep"])
def test_rescale_launch_replays_as_every_step_bit_reproducibly(scheduler):
    from lora_b200.host import schedulers
    from lora_b200.step_ops import sample_step
    g = torch.Generator().manual_seed(1)
    B, C, H, W = 2, 4, 64, 64
    N = 6
    ms = scheduler == "dpmsolver_multistep"
    tab = schedulers.pack_table(scheduler, "epsilon", N, N).to(DEV)
    noise = torch.randn(N + 1, B, C, H, W, generator=g).to(DEV)
    mos = [torch.randn(2 * B, C, H, W, generator=g).to(BF).to(DEV) for _ in range(N)]
    mo = torch.empty_like(mos[0])
    gs, ph = torch.tensor([5.0], device=DEV), torch.tensor([0.7], device=DEV)

    def fresh():
        x, hist = torch.zeros(B, C, H, W, device=DEV), torch.zeros(B, C, H, W, device=DEV)
        st = _state(B, C, H, W, C, g, None)
        sample_step(None, x, noise, tab, None, st[0], st[1], st[3], st[2], None, 0.13025, init=True)
        return (x, hist) + st

    x, hist, *st = S = fresh()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _run_step(True, ms, mo, x, noise, hist, tab, gs, ph, st)
    torch.cuda.current_stream().wait_stream(s)
    gb = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gb):
        _run_step(True, ms, mo, x, noise, hist, tab, gs, ph, st)
    runs = []
    for rep in range(2):
        x, hist, *st = S
        sample_step(None, x, noise, tab, None, st[0], st[1], st[3], st[2], None, 0.13025, init=True)
        hist.zero_()
        st[4].fill_(float("nan"))                 # the decoder input is written on the last step only
        ex, eh, *est = E = fresh()
        for i in range(N):
            mo.copy_(mos[i])
            gb.replay()
            _run_step(True, ms, mos[i], ex, noise, eh, tab, gs, ph, est)
            torch.cuda.synchronize()
            for a, b in zip(S, E):
                assert torch.equal(_bits(a), _bits(b)), (rep, i)
            assert int(st[0]) == i + 1
        runs.append([t.clone() for t in S])
    for a, b in zip(*runs):                       # the replays of a second run are bit for bit the first's
        assert torch.equal(_bits(a), _bits(b))
    assert bool(torch.isfinite(S[0]).all())


# ------------------------------------------------------------------------------------ tiny SDXL samplers
TLAT = (2, 4, 16, 16)


def _xl_models(seed=0):
    """(ours (unet, te1, te2), refs (unet, te1, te2), vae): the tiny SDXL preset with equal non-zero
    LoRA factors on the engine's and the oracle's modules, and a tiny fp32 VAE."""
    from lora_b200.host.unet_sd15 import UNetConfig
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    ours, refs, *_ = _xl_pair(UNetConfig.sdxl_tiny(), tiny=True, seed=seed, up_std=0.05)
    torch.manual_seed(seed + 7)
    vae = AutoencoderKL(VAEConfig.tiny(), with_decoder=True).to(DEV).to(memory_format=torch.channels_last)
    vae.requires_grad_(False)
    return ours, refs, vae


def _xl_ids(seed=4):
    gi = torch.Generator(device=DEV).manual_seed(seed)
    return [_ids(TLAT[0], 998, 999, gi, lengths=lens) for lens in ((11, 30), (5, 40), (7, 20), (3, 60))]


def _xl_sampler(ours, vae, graph, **kw):
    from lora_b200.sample import LoraXLSampler, SamplerConfig
    base = dict(num_inference_steps=10, max_steps=12, guidance_scale=5.0, autocast_dtype=BF, vae_scaling=0.13025,
                use_cuda_graph=graph, scheduler="euler")
    base.update(kw)
    return LoraXLSampler(*ours, vae, SamplerConfig(**base), latent_shape=TLAT, seq_len=77, device=DEV)


def _external_noise(samplers, seed=11):
    g = torch.Generator(device=DEV).manual_seed(seed)
    s0 = samplers[0]
    noise = torch.randn(s0.noise.shape, device=DEV, generator=g)
    peps = torch.randn(s0.posterior_noise.shape, device=DEV, generator=g) if hasattr(s0, "posterior_noise") else None
    for s in samplers:
        s.noise.copy_(noise)
        if peps is not None:
            s.posterior_noise.copy_(peps.to(s.posterior_noise.dtype))
    return noise, peps


def _oracle_xl(refs, vae, sched, n, ids, g, phi, sizes=(128, 128, 0, 0, 128, 128), neg=None, image=None,
               strength=None, peps=None, noise=None):
    """(latents of the float64 run, latents of the fp32 + bf16-autocast run) of oracle/sample_xl_ref."""
    from oracle import sample_xl_ref as XR
    ids1, ids2 = ids
    neg1, neg2 = (None, None) if neg is None else neg
    out = []
    for dtype, ac in ((torch.float64, None), (torch.float32, BF)):
        models = [copy.deepcopy(m).to(dtype) for m in refs] if dtype == torch.float64 else list(refs)
        v = copy.deepcopy(vae).to(dtype) if dtype == torch.float64 else vae
        unet, te1, te2 = models

        def encode():
            return XR.encode_prompt_xl(te1, te2, ids1, ids2, neg1, neg2, g > 1.0)
        tid = XR.add_time_ids(sizes[:2], sizes[2:4], sizes[4:], ids1.shape[0], g > 1.0, dtype, DEV)
        _, lat = XR.sample(unet, v, XR.make_scheduler(sched, "epsilon"), n, encode, noise, g, phi,
                           added_cond_kwargs={"time_ids": tid}, image_u8=image, strength=strength,
                           posterior_eps=peps, scaling=0.13025, dtype=dtype, autocast_dtype=ac)
        out.append(lat)
    return out


def _check_xl(sg, se, lat64, lat_run):
    """Graph and eager within the oracle bound, and no further apart than twice the oracle's bf16 error."""
    e_ref = _rel(lat_run, lat64)
    for s in (sg, se):
        e_ours = _rel(s.latents, lat64)
        assert e_ours <= 2 * e_ref, (e_ours, e_ref)
    assert _rel(sg.latents, se.latents) <= 2 * e_ref, (_rel(sg.latents, se.latents), e_ref)


def _images(seed=6):
    g = torch.Generator().manual_seed(seed)
    B, _, h, w = TLAT
    return torch.randint(0, 256, (B, 8 * h, 8 * w, 3), generator=g, dtype=torch.uint8).to(DEV)


@pytest.mark.parametrize("scheduler", SCHEDULERS)
@pytest.mark.parametrize("task", ["txt2img", "img2img"])
def test_tiny_xl_graph_equals_eager_and_oracle(scheduler, task):
    ours, refs, vae = _xl_models()
    ids1, ids2, *_ = _xl_ids()
    n = 10
    kw = dict(scheduler=scheduler, external_noise=True, task=task, strength=0.6)
    sg, se = _xl_sampler(ours, vae, True, **kw), _xl_sampler(ours, vae, False, **kw)
    noise, peps = _external_noise([sg, se])
    image = _images() if task == "img2img" else None
    sg.prepare()
    sg.sample(ids1, ids2, image=image)
    se.sample(ids1, ids2, image=image)
    assert sg.captures == 1
    k = n - (n - int(n * 0.6)) if task == "img2img" else n
    lat64, lat_run = _oracle_xl(refs, vae, scheduler, n, (ids1, ids2), 5.0, 0.0, image=image,
                                strength=0.6 if image is not None else None, peps=peps, noise=noise[:k + 1])
    _check_xl(sg, se, lat64, lat_run)


@pytest.mark.parametrize("scheduler", ["euler", "dpmsolver_multistep"])
def test_tiny_xl_guidance_rescale_graph_equals_eager_and_oracle(scheduler):
    ours, refs, vae = _xl_models()
    ids1, ids2, *_ = _xl_ids()
    kw = dict(scheduler=scheduler, external_noise=True, guidance_rescale=0.7)
    sg, se = _xl_sampler(ours, vae, True, **kw), _xl_sampler(ours, vae, False, **kw)
    noise, _ = _external_noise([sg, se])
    sg.sample(ids1, ids2)
    se.sample(ids1, ids2)
    assert sg.captures == 1 and any("rescale" in key for key in sg._graphs)
    lat64, lat_run = _oracle_xl(refs, vae, scheduler, 10, (ids1, ids2), 5.0, 0.7, noise=noise[:11])
    _check_xl(sg, se, lat64, lat_run)
    # the rescale moves the result: phi = 0 lands elsewhere
    se.sample(ids1, ids2, guidance_rescale=0.0)
    assert not torch.equal(sg.latents, se.latents)


def test_tiny_xl_zeroed_and_encoded_negatives():
    ours, refs, vae = _xl_models()
    ids1, ids2, neg1, neg2 = _xl_ids()
    sg, se = _xl_sampler(ours, vae, True, external_noise=True), _xl_sampler(ours, vae, False, external_noise=True)
    noise, _ = _external_noise([sg, se])
    zeroed = sg.sample(ids1, ids2).clone()
    lz = sg.latents.clone()
    assert sg.captures == 1
    sg.sample(ids1, ids2, neg1, neg2)
    se.sample(ids1, ids2, neg1, neg2)
    assert sg.captures == 2
    assert not torch.equal(lz, sg.latents)
    lat64, lat_run = _oracle_xl(refs, vae, "euler", 10, (ids1, ids2), 5.0, 0.0, neg=(neg1, neg2), noise=noise[:11])
    _check_xl(sg, se, lat64, lat_run)
    again = sg.sample(ids1, ids2).clone()                # back to zeroed negatives: no capture
    assert sg.captures == 2 and torch.equal(again, zeroed) and torch.equal(sg.latents, lz)


def test_tiny_xl_time_ids_change_per_call_without_capture():
    ours, refs, vae = _xl_models()
    ids1, ids2, *_ = _xl_ids()
    sg, se = _xl_sampler(ours, vae, True, external_noise=True), _xl_sampler(ours, vae, False, external_noise=True)
    noise, _ = _external_noise([sg, se])
    sg.prepare()
    sg.sample(ids1, ids2)
    l0 = sg.latents.clone()
    kw = dict(original_size=(1024, 768), crops_coords_top_left=(32, 16), target_size=(512, 512))
    sg.sample(ids1, ids2, **kw)
    assert sg.captures == 1 and not torch.equal(l0, sg.latents)
    assert sg.time_ids.tolist() == [[1024.0, 768.0, 32.0, 16.0, 512.0, 512.0]] * 4
    se.sample(ids1, ids2, **kw)
    lat64, lat_run = _oracle_xl(refs, vae, "euler", 10, (ids1, ids2), 5.0, 0.0, sizes=(1024, 768, 32, 16, 512, 512),
                                noise=noise[:11])
    _check_xl(sg, se, lat64, lat_run)
    sg.sample(ids1, ids2)
    assert sg.captures == 1 and torch.equal(sg.latents, l0)


def test_tiny_xl_capture_counts_and_launches_per_step():
    from lora_b200 import ops
    ours, _, vae = _xl_models()
    ids1, ids2, *_ = _xl_ids()
    s, e = _xl_sampler(ours, vae, True), _xl_sampler(ours, vae, False)
    a = s.sample(ids1, ids2, seed=3).clone()
    assert s.captures == 1
    s.sample(ids1, ids2, seed=3, guidance_rescale=0.7)
    assert s.captures == 2
    s.sample(ids1, ids2, seed=3, guidance_rescale=0.3)
    e.sample(ids1, ids2, seed=3, guidance_rescale=0.3)
    assert s.captures == 2 and _rel(s.latents, e.latents) <= XL_GRAPH_EAGER
    assert torch.equal(a, s.sample(ids1, ids2, seed=3)) and s.captures == 2      # replays repeat bit for bit
    s.sample(ids1, ids2, seed=3, scheduler="dpmsolver_multistep")
    assert s.captures == 3
    s.sample(ids1, ids2, seed=3, scheduler="dpmsolver_multistep", guidance_rescale=0.5)
    assert s.captures == 4
    s.sample(ids1, ids2, seed=3, scheduler="euler_ancestral", guidance_rescale=0.5)     # Euler's family
    s.sample(ids1, ids2, seed=3, guidance_scale=1.0, guidance_rescale=0.5)              # G = 1: no rescale
    assert s.captures == 5 and (1, "single-step") in s._graphs
    for key in list(s._graphs):
        assert ("rescale" in key) == (key in {(2, "single-step", "rescale", "zero_negatives"),
                                              (2, "multistep", "rescale", "zero_negatives")})
    unet = ours[0]
    unet.eval()
    for m in ours[1:]:
        m.eval()
    with torch.no_grad(), torch.autocast("cuda", dtype=BF):
        for family in ("single-step", "multistep"):
            c0 = ops.LAUNCH_COUNT
            unet(e.unet_in[2], e.timestep, e._ehs[2], added_cond_kwargs=e._added[2])
            fwd = ops.LAUNCH_COUNT - c0
            c0 = ops.LAUNCH_COUNT
            e._body_b(2, family, True)
            step = ops.LAUNCH_COUNT - c0
            assert fwd > 0 and step == fwd + 1, (family, fwd, step)
    for m in ours:
        m.train()


def test_tiny_xl_sampling_between_training_steps_changes_nothing():
    import lora_b200 as L
    from lora_b200.train import LoraXLTrainStep, StepConfig
    ours, _, vae = _xl_models()
    twin = tuple(copy.deepcopy(m) for m in ours)
    ids1, ids2, *_ = _xl_ids()
    s = _xl_sampler(ours, vae, True, guidance_rescale=0.5)

    def train(models, K, sampler_fn=None):
        cfg = StepConfig(use_cuda_graph=True, graph_warmup=2, autocast_dtype=BF, train_text_encoder=True)
        tr = LoraXLTrainStep(*models, cfg, latent_shape=TLAT, seq_len=77, device=DEV)
        torch.manual_seed(21)
        tr.latents.copy_(torch.randn(TLAT, device=DEV) * 0.13025)
        tr.input_ids.copy_(ids1)
        tr.input_ids_2.copy_(ids2)
        tr.prepare()
        losses = []
        for _ in range(K):
            losses.append(tr.step_device().clone())
            if sampler_fn is not None:
                sampler_fn()
        return tr, torch.stack(losses)

    tr, losses = train(ours, 3, lambda: s.sample(ids1, ids2, seed=0))
    _, losses2 = train(twin, 3)
    assert torch.equal(_bits(losses), _bits(losses2))
    assert s.captures == 1
    fresh_models = tuple(copy.deepcopy(m) for m in ours)
    L.link_sites(*fresh_models)
    fresh = _xl_sampler(fresh_models, vae, False, guidance_rescale=0.5)
    fresh.sample(ids1, ids2, seed=0)
    assert _rel(s.latents, fresh.latents) <= XL_GRAPH_EAGER       # the trained factors, seen by the replay
    assert all(m.training for m in ours)


def test_tiny_xl_encoder_2_factor_edit_and_scale_change():
    ours, _, vae = _xl_models()
    ids1, ids2, *_ = _xl_ids()
    s, e = _xl_sampler(ours, vae, True), _xl_sampler(ours, vae, False)
    s.sample(ids1, ids2)
    l0 = s.latents.clone()
    site = next(m for m in ours[2].modules() if type(m).__name__ == "LoraInjectedLinear")
    site.lora_down.weight.data.mul_(-3.0)            # an in-place edit: seen by the next sample, no capture
    s.sample(ids1, ids2)
    assert s.captures == 1 and not torch.equal(l0, s.latents)
    e.sample(ids1, ids2)
    assert _rel(s.latents, e.latents) <= XL_GRAPH_EAGER
    site.scale = 0.5 * float(site.scale)             # a scale is baked into the launch: recapture
    s.sample(ids1, ids2)
    assert s.captures == 2
    e.sample(ids1, ids2)
    assert _rel(s.latents, e.latents) <= XL_GRAPH_EAGER


# ------------------------------------------------------------------------------------ SD with rescale
@pytest.mark.parametrize("scheduler,task", [("euler_ancestral", "txt2img"), ("dpmsolver_multistep", "img2img"),
                                            ("euler", "txt2img")])
def test_tiny_sd_guidance_rescale_graph_equals_eager_and_oracle(scheduler, task):
    from oracle import sample_image_ref as RI
    from oracle import sample_xl_ref as XR
    from test_sample_image_gpu import _ids as sd_ids
    from test_sample_image_gpu import _images as sd_images
    from test_sample_image_gpu import _models, _noise_pair, _sampler
    unet, text, vae, unet_r, text_r = _models()
    ids, neg = sd_ids(text)
    img = sd_images()[0] if task == "img2img" else None
    kw = dict(scheduler=scheduler, external_noise=True, guidance_rescale=0.7, task=task, strength=0.7)
    sg, se = _sampler(unet, text, vae, True, **kw), _sampler(unet, text, vae, False, **kw)
    if task == "img2img":
        noise, peps = _noise_pair(sg, se)
    else:
        noise, peps = _external_noise([sg, se])
    img_g = sg.sample(ids, neg, image=img).clone()
    img_e = se.sample(ids, neg, image=img).clone()
    assert sg.captures == 1 and torch.equal(img_g, img_e) and torch.equal(sg.latents, se.latents)
    n = 10
    k = int(n * 0.7) if task == "img2img" else n
    lats = []
    for dtype, ac in ((torch.float64, None), (torch.float32, BF)):
        u, t, v = ((copy.deepcopy(m).double() for m in (unet_r, text_r, vae)) if dtype == torch.float64
                   else (unet_r, text_r, vae))

        def encode(t=t):             # runs under the loop's autocast: no context of its own
            return RI._text(t, ids, neg, True, contextlib.nullcontext()), None
        _, lat = XR.sample(u, v, XR.make_scheduler(scheduler, "epsilon"), n, encode, noise[:k + 1], 7.0, 0.7,
                           image_u8=img, strength=0.7 if img is not None else None, posterior_eps=peps,
                           scaling=0.18215, dtype=dtype, autocast_dtype=ac, divide_by_scaling=False)
        lats.append(lat)
    e_ours, e_ref = _rel(sg.latents, lats[0]), _rel(lats[1], lats[0])
    assert e_ours <= 2 * e_ref, (e_ours, e_ref)


def test_oracle_loop_leaves_autocast_as_it_found_it():
    """The fp32 + bf16-autocast oracle run must not leave autocast on for whatever runs next."""
    from oracle import sample_image_ref as RI
    from oracle import sample_xl_ref as XR
    from test_sample_image_gpu import _ids as sd_ids
    from test_sample_image_gpu import _models
    _, text, vae, unet_r, text_r = _models()
    ids, neg = sd_ids(text)
    noise = torch.randn(4, 2, 4, 8, 8, device=DEV)
    XR.sample(unet_r, vae, XR.make_scheduler("euler", "epsilon"), 3, lambda: (RI._text(
        text_r, ids, neg, True, contextlib.nullcontext()), None), noise, 7.0, 0.7, scaling=0.18215,
        dtype=torch.float32, autocast_dtype=BF, divide_by_scaling=False)
    assert not torch.is_autocast_enabled("cuda")


# ------------------------------------------------------------------------------------ census
# (M, K, N) of the SDXL sites at G * B = 2, 1024 px: the shapes the training census (batch 1) did not cover
XL_SAMPLE_LINEAR = [(8192, 640, 640), (8192, 640, 5120), (2048, 1280, 1280), (2048, 1280, 10240),
                    (154, 2048, 640), (154, 2048, 1280), (154, 1280, 1280)]
XL_SAMPLE_GROUPED = [(8192, 640, 640, 3), (2048, 1280, 1280, 3), (154, 1280, 1280, 3),
                     (154, 2048, 640, 2), (154, 2048, 1280, 2)]


@pytest.mark.parametrize("M,K,N", XL_SAMPLE_LINEAR)
def test_sdxl_sampling_linear_sites_match_float64(M, K, N):
    KG.test_fused_forward_matches_oracle(M, K, N, 4, BF)


@pytest.mark.parametrize("M,K,N,n", XL_SAMPLE_GROUPED)
def test_sdxl_sampling_grouped_launches_match_float64(M, K, N, n):
    import test_sdxl_gpu as SX
    SX.test_sdxl_grouped_launches_match_float64(M, K, N, n)


@pytest.mark.parametrize("case", [(2,) + c[1:] for c in CONV_SDXL],
                         ids=lambda c: "n{}_{}x{}_{}to{}_k{}_r{}_{}".format(*c[:7], str(c[7])[6:]))
def test_sdxl_sampling_conv_sites_match_float64(case):
    CK.test_conv_kernels_match_float64(case)


# ------------------------------------------------------------------------------------ full size
def test_full_size_sdxl_1024_euler_20_graph_equals_eager_and_oracle():
    """SDXL UNet and both encoders, LoRA r = 4 everywhere, random weights, bf16 autocast, 1024 px, 20 Euler
    steps at guidance 5, phi = 0 and 0.7."""
    import lora_b200 as L
    from lora_b200.host.unet_sd15 import UNetConfig
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    from lora_b200.sample import LoraXLSampler, SamplerConfig
    ours, refs, *_ = _xl_pair(UNetConfig.sdxl(), tiny=False)
    torch.manual_seed(1)
    with torch.device(DEV):
        vae = AutoencoderKL(VAEConfig.sd(), with_decoder=True)
    vae = vae.to(torch.bfloat16).to(memory_format=torch.channels_last)
    vae.requires_grad_(False)
    n, lat = 20, (1, 4, 128, 128)
    gi = torch.Generator(device=DEV).manual_seed(9)
    ids1, ids2 = _ids(1, 49407, 49407, gi), _ids(1, 49407, 49407, gi)
    L.set_grouping(True)
    try:
        cfg = dict(scheduler="euler", num_inference_steps=n, max_steps=n, guidance_scale=5.0, vae_scaling=0.13025,
                   autocast_dtype=BF, external_noise=True)
        sg = LoraXLSampler(*ours, vae, SamplerConfig(**cfg), latent_shape=lat, device=DEV)
        se = LoraXLSampler(*ours, vae, SamplerConfig(use_cuda_graph=False, **cfg), latent_shape=lat, device=DEV)
        noise, _ = _external_noise([sg, se], seed=5)
        results = {}
        for phi in (0.0, 0.7):
            img = sg.sample(ids1, ids2, guidance_rescale=phi).clone()
            assert torch.equal(img, se.sample(ids1, ids2, guidance_rescale=phi)) and torch.equal(sg.latents, se.latents)
            results[phi] = sg.latents.clone()
        assert sg.captures == 2
        del se
        torch.cuda.empty_cache()
        for phi, got in results.items():
            lat64, lat_run = _oracle_xl(refs, vae, "euler", n, (ids1, ids2), 5.0, phi,
                                        sizes=(1024, 1024, 0, 0, 1024, 1024), noise=noise)
            e_ours, e_ref = _rel(got, lat64), _rel(lat_run, lat64)
            assert e_ours <= 2 * e_ref, (phi, e_ours, e_ref)
            del lat64, lat_run
            torch.cuda.empty_cache()
    finally:
        L.set_grouping(False)
