"""Per-image LoRA coefficients on the GPU: the _ps entry points against float64 and, row block by row
block, against the scalar-coefficient launches bit for bit; the site layer (per_sample_lora) against the
default forward after tune_lora_scale / set_lora_diag; and the samplers' per-sample graphs against default
calls, their eager path and the float64 oracle."""
import copy
import types

import pytest
import torch
import torch.nn.functional as F

import test_sample_gpu as SG
from lora_b200._C import LoraB200Error
import test_sample_image_gpu as SI

pytestmark = pytest.mark.gpu
DEV = "cuda"
_bits = SG._bits


def _l2_split(M, K, N, r):
    """Whether lb_lora_linear_fwd picks an L2 split-K plan for this shape (the planner's own answer):
    those add their partials in arrival order, so they are held to the float64 bound only."""
    from lora_b200 import _C, ops
    return _C.lib.lb_lora_linear_fwd_split_k(M, K, N, ops.rank_pad(r)) > 1


def _operands(M, K, N, r, dt, bias, S, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g).to(dt)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dt)
    a = torch.randn(r, K, generator=g) / K ** 0.5
    b = torch.randn(N, r, generator=g) * 0.5
    bs = torch.randn(N, generator=g) if bias else None
    table = torch.rand(S, r, generator=g) * 2.0 - 0.5
    table[0, 0] = 0.0
    return [t if t is None else t.to(DEV) for t in (x, w, a, b, bs, table)]


def _rows_of(M, rps, S):
    return (torch.arange(M) // rps) % S


def _ref_linear(x, w, down16, b, bias, table, rps, r):
    """float64 result and elementwise bound: the kernel rounds T' and U to the operand type."""
    x64, w64, d64 = x.double().cpu(), w.double().cpu(), down16[:r].double().cpu()
    b64 = b.double().cpu()
    M = x64.shape[0]
    coef = table.double().cpu()[_rows_of(M, rps, table.shape[0])]
    ts = (x64 @ d64.T) * coef
    y = x64 @ w64.T + ts @ b64.T
    scale = x64.abs() @ w64.abs().T + ts.abs() @ b64.abs().T
    if bias is not None:
        y = y + bias.double().cpu()
        scale = scale + bias.double().cpu().abs()
    return y, scale


def _check_f64(y, ref, scale, out_f32):
    err = (y.double().cpu() - ref).abs()
    tol = 2 ** -7 * scale + (0 if out_f32 else 2 ** -8) * ref.abs() + 1e-6
    assert bool((err <= tol).all()), float((err / tol).max())


# (M, K, N, rows_per_sample, S): one case per auto plan of 16-bit outputs at rank pad 16
LINEAR_CASES = [
    (154, 2048, 320, 77, 1),      # L2 split-K (few tiles, long K)
    (308, 768, 768, 77, 2),       # cluster split-K
    (16, 1280, 1280, 1, 8),       # cluster split-K, one row per sample, batch 2S
    (1024, 640, 2560, 128, 4),    # 192-wide tiles in one wave
    (4096, 320, 640, 256, 8),     # crowded 128-wide tiles: inline TMA
    (2048, 320, 640, 256, 4),     # crowded 64-wide tiles, two CTAs per SM
    (1232, 768, 768, 77, 8),      # one 64-wide tile per CTA, deep ring, batch 2S of 77 tokens
    (200, 320, 320, 25, 4),       # one tile per CTA, M not a multiple of 128
]


@pytest.mark.parametrize("case", LINEAR_CASES)
@pytest.mark.parametrize("r", [4, 24, 48])
@pytest.mark.parametrize("out_f32", [False, True])
def test_linear_ps_matches_scalar_rows_and_float64(case, r, out_f32):
    from lora_b200 import ops
    M, K, N, rps, S = case
    for i, (dt, bias) in enumerate(((torch.bfloat16, True), (torch.float16, False))):
        x, w, a, b, bs, table = _operands(M, K, N, r, dt, bias, S, seed=M + r + i)
        down16 = ops.cast_rows_pad16(a, K, 1, r, K, dt)
        odt = torch.float32 if out_f32 else dt
        y, t = ops.fused_linear(x, w, bs, down16, b, r, 1, None, 1.0, r, odt, False, coef_rows=(table, r, rps, S))
        assert t is None
        ref, scale = _ref_linear(x, w, down16, b, bs, table, rps, r)
        _check_f64(y, ref, scale, out_f32)
        if _l2_split(M, K, N, r):
            continue
        rows = _rows_of(M, rps, S).to(DEV)
        for s in range(S):    # row block of sample s == the scalar launch with coefficients table[s]
            ys, _ = ops.fused_linear(x, w, bs, down16, b, r, 1, table[s].contiguous(), 1.0, r, odt, False)
            sel = rows == s
            assert torch.equal(_bits(y[sel]), _bits(ys[sel])), (s, dt)


@pytest.mark.parametrize("case", [LINEAR_CASES[1], LINEAR_CASES[4], LINEAR_CASES[7]])
def test_linear_uniform_table_is_the_scalar_path_bit_for_bit(case):
    from lora_b200 import ops
    M, K, N, rps, S = case
    r = 8
    x, w, a, b, bs, _ = _operands(M, K, N, r, torch.bfloat16, True, S, seed=5)
    down16 = ops.cast_rows_pad16(a, K, 1, r, K, torch.bfloat16)
    scale, diag = 0.7, torch.linspace(0.25, 1.5, r, device=DEV)
    table = (torch.tensor(scale, dtype=torch.float32) * diag).expand(S, r).contiguous()
    y, _ = ops.fused_linear(x, w, bs, down16, b, r, 1, None, 1.0, r, torch.bfloat16, False,
                            coef_rows=(table, r, rps, S))
    y0, _ = ops.fused_linear(x, w, bs, down16, b, r, 1, diag, scale, r, torch.bfloat16, False)
    assert torch.equal(_bits(y), _bits(y0))


@pytest.mark.parametrize("n", [2, 3, 4])
@pytest.mark.parametrize("out_f32", [False, True])
def test_grouped_ps_one_table_per_problem(n, out_f32):
    from lora_b200 import ops
    dt = torch.bfloat16
    M, K = 308, 640
    shapes = [(640, 77, 2), (320, 77, 4), (1280, 154, 1), (640, 1, 4)][:n]
    x = torch.randn(M, K, generator=torch.Generator().manual_seed(n)).to(dt).to(DEV)
    probs, tabs, refs = [], [], []
    for i, (N, rps, S) in enumerate(shapes):
        _, w, a, b, bs, table = _operands(M, K, N, 4 + 3 * i, dt, i % 2 == 0, S, seed=10 * n + i)
        r = 4 + 3 * i
        d16 = ops.cast_rows_pad16(a, K, 1, r, K, dt)
        probs.append((x, w, bs, d16, b, r, 1, None, 1.0, r))
        tabs.append((table, r, rps, S))
        refs.append(_ref_linear(x, w, d16, b, bs, table, rps, r))
    odt = torch.float32 if out_f32 else dt
    ys, ts = ops.fused_linear_grouped(probs, odt, False, coef_rows=tabs)
    assert all(t is None for t in ts)
    for y, (ref, scale) in zip(ys, refs):
        _check_f64(y, ref, scale, out_f32)
    # row block of sample s of problem i == the scalar grouped launch with diag = its table row s
    for s in range(max(S for _, _, S in shapes)):
        sc = [p[:7] + (tabs[i][0][min(s, tabs[i][3] - 1)].contiguous(), 1.0, p[9]) for i, p in enumerate(probs)]
        ys0, _ = ops.fused_linear_grouped(sc, odt, False)
        for i, (y, y0) in enumerate(zip(ys, ys0)):
            _, _, rps, S = tabs[i]
            if s < S:
                sel = _rows_of(M, rps, S).to(DEV) == s
                assert torch.equal(_bits(y[sel]), _bits(y0[sel])), (i, s)


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("n_img,S", [(2, 2), (4, 2), (3, 3)])
@pytest.mark.parametrize("r", [4, 32])
def test_conv_ps_matches_scalar_images_and_float64(k, n_img, S, r):
    from lora_b200 import ops
    dt = torch.bfloat16
    H, W, cin, cout = 12, 20, 64, 128
    g = torch.Generator().manual_seed(k + n_img + r)
    x = torch.randn(n_img, cin, H, W, generator=g).to(dt).to(DEV).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).to(DEV)
    a = (torch.randn(r, cin, k, k, generator=g) / (cin * k * k) ** 0.5).to(DEV)
    b = (torch.randn(cout, r, generator=g) * 0.5).to(DEV)
    bias = torch.randn(cout, generator=g).to(DEV)
    table = (torch.rand(S, r, generator=g) * 2.0 - 0.5).to(DEV)
    w_f, _ = ops.cast_conv_weight(w, dt, True, False)
    d16 = ops.conv_down16(a, dt, {})
    pad = (k - 1) // 2
    args = (x, w_f, bias, d16, b, 0, r, 1, 0)
    y, t = ops.fused_conv2d(*args, None, 1.0, r, cout, k, k, pad, pad, False, dt, False,
                            coef_rows=(table, r, H * W, S))
    assert t is None
    x64, w64, a64 = x.double().cpu(), w.to(dt).double().cpu(), a.to(dt).double().cpu()
    coef = table.double().cpu()[torch.arange(n_img) % S]
    ts = F.conv2d(x64, a64, padding=pad) * coef[:, :, None, None]
    b64 = b.double().cpu()
    ref = F.conv2d(x64, w64, bias.double().cpu(), padding=pad) + torch.einsum("njhw,cj->nchw", ts, b64)
    scale = (F.conv2d(x64.abs(), w64.abs(), bias.double().cpu().abs(), padding=pad)
             + torch.einsum("njhw,cj->nchw", ts.abs(), b64.abs()))
    _check_f64(y, ref, scale, False)
    from lora_b200 import _C
    if _C.lib.lb_lora_conv2d_fwd_split_k(n_img, H, W, cin, cout, k, k, ops.rank_pad(r)) > 1:
        return                                        # an L2 split-K plan: float64 bound only
    for s in range(S):
        y0, _ = ops.fused_conv2d(*args, table[s].contiguous(), 1.0, r, cout, k, k, pad, pad, False, dt, False)
        sel = (torch.arange(n_img) % S == s).to(DEV)
        assert torch.equal(_bits(y[sel]), _bits(y0[sel])), s


# ------------------------------------------------------------------------------------ site level
@pytest.mark.parametrize("grouping", [False, True])
def test_unet_per_sample_rows_equal_tuned_default_forward(grouping):
    import lora_b200 as L
    unet, text, *_ = SG._models()
    unet.eval()
    text.eval()
    S = 3
    scales = [0.0, 0.6, 1.5]
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn(2 * S, 4, 8, 8, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)
    ids = torch.randint(0, text.config.vocab_size, (2 * S, 77), device=DEV, generator=g)
    ts = torch.tensor([500.0], device=DEV)
    L.set_grouping(grouping)
    try:
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            def run():
                ehs = text(ids)[0]
                return ehs, unet(x, ts, ehs).sample
            run()                                     # grouping learns its families
            with L.per_sample_lora(unet, scale=scales, samples=S), L.per_sample_lora(text, scale=scales, samples=S):
                e_ps, y_ps = run()
            for s, sc in enumerate(scales):
                L.tune_lora_scale(unet, sc)
                L.tune_lora_scale(text, sc)
                e0, y0 = run()
                rows = torch.arange(2 * S, device=DEV) % S == s
                assert torch.equal(_bits(e_ps[rows]), _bits(e0[rows])), s
                assert torch.equal(_bits(y_ps[rows]), _bits(y0[rows])), s
    finally:
        L.set_grouping(False)


def test_diag_rows_and_selector_per_sample_equal_set_lora_diag():
    import lora_b200 as L
    unet, *_ = SG._models()
    unet.eval()
    mgr = L.LoRAManager.__new__(L.LoRAManager)      # a join of two rank-2 LoRAs into the rank-4 sites
    mgr.ranklist, mgr.pipe = [2, 2], types.SimpleNamespace(unet=unet)
    mixes = [[1.0, 0.0], [0.0, 1.0], [0.5, 1.25]]
    rows = mgr.diag_rows(mixes)
    g = torch.Generator(device=DEV).manual_seed(2)
    x = torch.randn(3, 4, 8, 8, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)
    ehs = torch.randn(3, 77, unet.cfg.cross_attention_dim, device=DEV, generator=g)
    ts = torch.tensor([300.0], device=DEV)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        with L.per_sample_lora(unet, diag=rows, scale=0.8):
            y = unet(x, ts, ehs).sample
        L.tune_lora_scale(unet, 0.8)
        for s, mix in enumerate(mixes):
            mgr.tune(mix)
            y0 = unet(x, ts, ehs).sample
            assert torch.equal(_bits(y[s]), _bits(y0[s])), s


def test_conv_site_per_sample_rows_and_refusals():
    import lora_b200 as L
    torch.manual_seed(0)
    m = L.LoraInjectedConv2d(64, 64, 3, padding=1, r=4, dropout_p=0.1).to(DEV)
    m.lora_up.weight.data.normal_(0, 0.1)
    m.eval()
    x = torch.randn(4, 64, 12, 12, device=DEV).to(torch.bfloat16)
    with torch.no_grad():
        with L.per_sample_lora(m, scale=[0.0, 2.0], samples=2):
            y = m(x)
        for s, sc in enumerate([0.0, 2.0]):
            m.scale = sc
            y0 = m(x)
            assert torch.equal(_bits(y[s::2]), _bits(y0[s::2]))
    with L.per_sample_lora(m, scale=[1.0, 2.0]):
        with pytest.raises(LoraB200Error, match="forward only"):
            m(x)                                      # factors require grad
        with torch.no_grad():
            with pytest.raises(LoraB200Error, match="multiple"):
                m(x[:3])
            m.train()
            with pytest.raises(LoraB200Error, match="dropout"):
                m(x)
            m.eval()


def test_linear_site_refusals():
    import lora_b200 as L
    lin = L.LoraInjectedLinear(64, 128, r=4, dropout_p=0.0).to(DEV)
    wide = L.LoraInjectedLinear(128, 128, r=80, dropout_p=0.0).to(DEV)
    x = torch.randn(2, 77, 64, device=DEV)
    with torch.no_grad():
        with L.per_sample_lora(lin, scale=[0.5, 1.0]):
            L.set_fp32_mode("split")
            try:
                with pytest.raises(LoraB200Error, match="split"):
                    lin(x)
            finally:
                L.set_fp32_mode("bf16")
            assert lin(x).shape == (2, 77, 128)
        with L.per_sample_lora(wide, scale=[0.5, 1.0]):
            with pytest.raises(LoraB200Error, match="ranks up to 64"):
                wide(torch.randn(2, 5, 128, device=DEV))


# ------------------------------------------------------------------------------------ samplers
LAT4 = (4, 4, 8, 8)
SCALES = [0.0, 0.5, 1.0, 1.5]


def _sampler4(unet, text, vae, graph, **kw):
    from lora_b200.sample import LoraSampler, SamplerConfig
    base = dict(num_inference_steps=6, max_steps=8, guidance_scale=7.0, autocast_dtype=torch.bfloat16,
                use_cuda_graph=graph, external_noise=True)
    base.update(kw)
    return LoraSampler(unet, text, vae, SamplerConfig(**base), latent_shape=LAT4, seq_len=77, device=DEV)


def _ids4(text, seed=4):
    g = torch.Generator().manual_seed(seed)
    v = text.config.vocab_size
    return (torch.randint(0, v, (4, 77), generator=g).to(DEV), torch.randint(0, v, (4, 77), generator=g).to(DEV))


def _set_noise(samplers, seed=11):
    g = torch.Generator(device=DEV).manual_seed(seed)
    noise = torch.randn(samplers[0].noise.shape, device=DEV, generator=g)
    peps = None
    if hasattr(samplers[0], "posterior_noise"):
        peps = torch.randn(samplers[0].posterior_noise.shape, device=DEV, generator=g)
    for s in samplers:
        s.noise.copy_(noise)
        if peps is not None:
            s.posterior_noise.copy_(peps.to(s.posterior_noise.dtype))
    return noise


def test_sampler_per_image_scales_match_tuned_calls_eager_and_oracle():
    import lora_b200 as L
    from oracle import sample_ref as R
    unet, text, vae, unet_r, text_r = SG._models()
    ids, neg = _ids4(text)
    sg, se, sd = (_sampler4(unet, text, vae, True), _sampler4(unet, text, vae, False),
                  _sampler4(unet, text, vae, True))
    noise = _set_noise([sg, se, sd])
    lora = {"unet": SCALES, "text_encoder": SCALES}
    img = sg.sample(ids, neg, lora_scale=lora).clone()
    lat = sg.latents.clone()
    assert torch.equal(img, se.sample(ids, neg, lora_scale=lora)) and torch.equal(lat, se.latents)
    n = 6
    for b, sc in enumerate(SCALES):
        L.tune_lora_scale(unet, sc)
        L.tune_lora_scale(text, sc)
        ib = sd.sample(ids, neg).clone()
        assert torch.equal(img[b], ib[b]) and torch.equal(_bits(lat[b]), _bits(sd.latents[b])), b
        for m in list(unet_r.modules()) + list(text_r.modules()):
            if type(m).__name__ == "RefLoraSite":
                m.scale = sc
        args = (ids, neg, noise[:n + 1], 7.0)
        f64 = [copy.deepcopy(m).double() for m in (unet_r, text_r, vae)]
        _, lat64 = R.sample(*f64, R.make_scheduler("euler_ancestral", "epsilon"), n, *args, dtype=torch.float64)
        _, lat_run = R.sample(unet_r, text_r, vae, R.make_scheduler("euler_ancestral", "epsilon"), n, *args,
                              dtype=torch.float32, autocast_dtype=torch.bfloat16)
        assert SG._rel(lat[b], lat64[b]) <= 2 * SG._rel(lat_run[b], lat64[b]), b
    assert sd.captures == len(SCALES)          # default calls still recapture on a scale change
    # per-sample graphs: new values, tune_lora_scale and set_lora_diag between calls cost no capture
    sg.sample(ids, neg, lora_scale={"unet": [1.0, 0.2, 0.3, 0.4]})
    L.tune_lora_scale(unet, 0.25)
    L.set_lora_diag(text, torch.tensor([1.0, 0.5, 0.0, 2.0]))
    diag = torch.rand(4, 4, generator=torch.Generator().manual_seed(7))
    a = sg.sample(ids, neg, lora_scale={"text_encoder": 0.5}, lora_diag={"unet": diag}).clone()
    assert sg.captures == 1
    assert torch.equal(a, se.sample(ids, neg, lora_scale={"text_encoder": 0.5}, lora_diag={"unet": diag}))


def test_sampler_diag_rows_mix_per_image_and_no_recapture():
    import lora_b200 as L
    unet, text, vae, *_ = SG._models()
    ids, neg = _ids4(text)
    sg, sd = _sampler4(unet, text, vae, True), _sampler4(unet, text, vae, True)
    _set_noise([sg, sd])
    mgr = L.LoRAManager.__new__(L.LoRAManager)
    mgr.ranklist, mgr.pipe = [2, 2], types.SimpleNamespace(unet=unet)
    mixes = [[1.0, 0.0], [0.0, 1.0], [0.5, 0.5], [1.0, 1.0]]
    rows = mgr.diag_rows(mixes)
    img = sg.sample(ids, neg, lora_diag={"unet": rows}).clone()
    for b, mix in enumerate(mixes):
        mgr.tune(mix)
        assert torch.equal(img[b], sd.sample(ids, neg)[b]), b
    mgr.tune([0.3, 0.3])
    again = sg.sample(ids, neg, lora_diag={"unet": rows})
    assert torch.equal(img, again) and sg.captures == 1


@pytest.mark.parametrize("task", ["img2img", "inpaint"])
def test_image_tasks_per_image_scales_match_tuned_calls(task):
    import lora_b200 as L
    unet, text, vae, *_ = SI._models(in_channels=9 if task == "inpaint" else 4)
    ids, neg = _ids4(text)
    g = torch.Generator().manual_seed(6)
    image = torch.randint(0, 256, (4, 64, 64, 3), generator=g, dtype=torch.uint8).to(DEV)
    mask = SI._mask_u8(4, 64, 64, g).to(DEV)
    kw = dict(image=image) if task == "img2img" else dict(image=image, mask_image=mask)
    sg, se, sd = (_sampler4(unet, text, vae, True, task=task), _sampler4(unet, text, vae, False, task=task),
                  _sampler4(unet, text, vae, True, task=task))
    _set_noise([sg, se, sd])
    scales = [0.0, 1.5, 0.5, 1.0]
    img = sg.sample(ids, neg, lora_scale={"unet": scales}, **kw).clone()
    lat = sg.latents.clone()
    for b, sc in enumerate(scales):
        L.tune_lora_scale(unet, sc)
        sd.sample(ids, neg, **kw)
        assert torch.equal(_bits(lat[b]), _bits(sd.latents[b])), (b, SG._rel(lat[b], sd.latents[b]))
        assert torch.equal(img[b], sd.image[b]), b
    # graph against eager: as bit-exact as the default path is at this batch. The text encoder's eager and
    # captured runs can differ in the last bits at some batch sizes (test_sample_image_gpu.py, _models);
    # where the default path's graph and eager runs differ, the per-sample pair is held to the same distance
    se.sample(ids, neg, **kw)
    default_gap = SG._rel(sd.latents, se.latents)
    se.sample(ids, neg, lora_scale={"unet": scales}, **kw)
    if default_gap == 0.0:
        assert torch.equal(_bits(lat), _bits(se.latents)) and torch.equal(img, se.image)
    else:
        assert SG._rel(lat, se.latents) <= max(2 * default_gap, 3e-2), default_gap


def test_shared_noise_is_the_batch_1_noise_for_every_image():
    unet, text, vae, *_ = SG._models()
    ids, neg = _ids4(text)
    s4 = _sampler4(unet, text, vae, True, external_noise=False)
    from lora_b200.sample import LoraSampler, SamplerConfig
    s1 = LoraSampler(unet, text, vae, SamplerConfig(num_inference_steps=6, max_steps=8, guidance_scale=7.0,
                                                    autocast_dtype=torch.bfloat16),
                     latent_shape=(1, 4, 8, 8), seq_len=77, device=DEV)
    img = s4.sample(ids, neg, seed=5, shared_noise=True, lora_scale={"unet": SCALES}).clone()
    s1.sample(ids[:1], neg[:1], seed=5)
    for b in range(4):
        assert torch.equal(s4.noise[:7, b], s1.noise[:7, 0])
    # the image whose scale is the module's own (1.0) is the batch-1 call's image up to batch effects: the
    # same prompt everywhere makes every image a one-scale batch-1 sample
    s4.sample(ids[:1].expand(4, -1), neg[:1].expand(4, -1), seed=5, shared_noise=True,
              lora_scale={"unet": 1.0, "text_encoder": 1.0})
    assert all(torch.equal(s4.image[0], s4.image[b]) for b in range(4))
    assert img.shape == (4, 64, 64, 3)
    with pytest.raises(ValueError, match="external_noise"):
        _sampler4(unet, text, vae, True).sample(ids, neg, shared_noise=True)


def test_per_sample_step_graph_keeps_its_launch_count():
    import lora_b200 as L
    from lora_b200 import ops
    from lora_b200 import per_sample
    unet, text, vae, *_ = SG._models()
    ids, neg = _ids4(text)
    s = _sampler4(unet, text, vae, False)
    s.sample(ids, neg, lora_scale={"unet": SCALES})
    unet.eval()
    with torch.no_grad():
        c0 = ops.LAUNCH_COUNT
        s._body_b(2)
        default = ops.LAUNCH_COUNT - c0
        sites, views = s._per_sample_tables({"unet": (torch.tensor(SCALES), None)})
        with per_sample.bound(sites, views, 4):
            c0 = ops.LAUNCH_COUNT
            s._body_b(2)
            ps = ops.LAUNCH_COUNT - c0
    unet.train()
    assert default > 0 and ps == default


def test_xl_sampler_text_encoder_2_scale_per_image():
    import lora_b200 as L
    import test_sample_xl_gpu as SX
    ours, refs, vae = SX._xl_models()
    unet, te1, te2 = ours
    from lora_b200.sample import LoraXLSampler, SamplerConfig
    lat = (2,) + tuple(SX.TLAT[1:])

    def mk(graph):
        cfg = SamplerConfig(num_inference_steps=4, max_steps=6, guidance_scale=5.0, autocast_dtype=torch.bfloat16,
                            vae_scaling=0.13025, use_cuda_graph=graph, scheduler="euler", external_noise=True)
        return LoraXLSampler(unet, te1, te2, vae, cfg, latent_shape=lat, seq_len=77, device=DEV)
    sg, se, sd = mk(True), mk(False), mk(True)
    _set_noise([sg, se, sd])
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(0, 998, (2, 77), generator=g).to(DEV)
    ids2 = torch.randint(0, 998, (2, 77), generator=g).to(DEV)
    scales = [0.0, 1.5]
    img = sg.sample(ids, ids2, lora_scale={"text_encoder_2": scales}).clone()
    lat = sg.latents.clone()
    # graph against graph bit for bit; the tiny SDXL preset's graph and eager paths differ by a few bf16
    # roundings on the text side (test_sample_xl_gpu.py), so the eager run is held to that module's bound
    for b, sc in enumerate(scales):
        L.tune_lora_scale(te2, sc)
        assert torch.equal(img[b], sd.sample(ids, ids2)[b]) and torch.equal(_bits(lat[b]), _bits(sd.latents[b])), b
    assert sg.captures == 1
    se.sample(ids, ids2, lora_scale={"text_encoder_2": scales})
    assert SG._rel(lat, se.latents) <= SX.XL_GRAPH_EAGER


def test_grouped_per_sample_graphs_survive_selector_changes(monkeypatch):
    """Grouping on (the benchmarked setting), selectors installed before the capture: bound sites never
    read their selector or scale (a per-sample graph must not hold a copy of a selector weight that the
    next set_lora_diag frees); images equal tuned default calls; a new selector and an emptied allocator
    cache between calls cost no capture and replay the new values."""
    import lora_b200 as L
    from lora_b200 import modules
    unet, text, vae, *_ = SG._models()
    ids, neg = _ids4(text)
    L.set_grouping(True)
    try:
        sg, se, sd = (_sampler4(unet, text, vae, True), _sampler4(unet, text, vae, False),
                      _sampler4(unet, text, vae, True))
        _set_noise([sg, se, sd])
        L.set_lora_diag(unet, torch.tensor([1.0, 0.5, 0.0, 2.0]))
        L.set_lora_diag(text, torch.tensor([0.25, 1.0, 1.5, 0.75]))
        real = modules._selector_diag

        def guarded(self):
            assert self._lb.ps is None, "a site bound to a per-sample table read its selector"
            return real(self)
        monkeypatch.setattr(modules.LoraInjectedLinear, "_selector_diag", guarded)
        lora = {"unet": SCALES, "text_encoder": SCALES}
        img = sg.sample(ids, neg, lora_scale=lora).clone()
        assert torch.equal(img, se.sample(ids, neg, lora_scale=lora))
        for b, sc in enumerate(SCALES):
            L.tune_lora_scale(unet, sc)
            L.tune_lora_scale(text, sc)
            assert torch.equal(img[b], sd.sample(ids, neg)[b]), b
        L.set_lora_diag(unet, torch.tensor([2.0, 0.0, 1.0, 0.5]))      # frees the previous selector weights
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        a = sg.sample(ids, neg, lora_scale=lora).clone()
        assert sg.captures == 1
        assert torch.equal(a, se.sample(ids, neg, lora_scale=lora)) and not torch.equal(a, img)
    finally:
        L.set_grouping(False)


def test_coef_table_row_pitch_is_checked():
    from lora_b200 import ops
    wide = torch.rand(4, 8, device=DEV)
    with pytest.raises(AssertionError):
        ops._coef_args((wide[:, :4], 4, 1, 4), 4)        # rows 8 apart, not ld = 4
    assert ops._coef_args((wide[:, :4].contiguous(), 4, 1, 4), 4)[1] == 4
    assert ops._coef_args((wide, 8, 1, 4), 4)[1] == 8     # a wider pitch given as ld
