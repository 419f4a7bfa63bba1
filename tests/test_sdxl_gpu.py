"""SDXL on the GPU: the fused linear, grouped and conv kernels at SDXL 1024 px site shapes against
float64, and SDXL LoRA training steps (LoraXLTrainStep) against the oracle step
(oracle/ref_step_xl.py): full-size SDXL at 1024 px, eager and graph-replayed, and tiny-preset variants.

Bounds are those of the suites the checks come from: test_kernels_gpu.py (linear kernels),
test_conv_kernels_gpu.py (conv kernels, whose checks are called here on the new shapes),
test_grouping_gpu.py (grouped launches), test_sd2_gpu.py (full-size step: loss 1e-2 relative, first-step
gradient 3e-2, update direction < 0.5 after 4 steps; tiny steps: loss 1e-2 relative under autocast) and
test_checkpointing_gpu.py (checkpointed against plain: first loss equal, factors within 1e-5).

Prompts end with the eos id (the CLIP tokenizers pad with it), so the pooled token of the second encoder
is a real position."""
import pytest
import torch
import torch.nn as nn

import test_conv_kernels_gpu as CK
import test_kernels_gpu as KG

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF, FP = torch.bfloat16, torch.float16


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ------------------------------------------------------------------------------------ linear census
# (M, K, N) of the SDXL sites at batch 1, 1024 px (128 x 128 latents)
SDXL_LINEAR = [
    (4096, 640, 640), (4096, 640, 5120),          # level 2 (64 x 64 tokens): q/k/v/out, GEGLU proj
    (1024, 1280, 1280), (1024, 1280, 10240),      # level 3 (32 x 32) and the mid block
    (77, 2048, 640), (77, 2048, 1280),            # attn2 to_k / to_v on the concatenated 2048-wide context
    (77, 1280, 1280),                             # text encoder 2 (OpenCLIP bigG)
]


@pytest.mark.parametrize("r", [4, 16, 64])
@pytest.mark.parametrize("M,K,N", SDXL_LINEAR)
def test_sdxl_linear_sites_match_float64(M, K, N, r):
    """test_kernels_gpu.py's checks and bounds: frozen GEMM + T (fp32 out), fused forward (bf16
    operands, fp32 and bf16 out), input gradient and dA / dB."""
    KG.test_base_gemm_and_T_fp32_out(M, K, N, r)
    KG.test_fused_forward_matches_oracle(M, K, N, r, torch.bfloat16)
    KG.test_backward_kernels_match_oracle(M, K, N, r)


# ------------------------------------------------------------------------------------ grouped census
# (M, K, N, family): the self-attention q/k/v and the text encoder's q/k/v (3 sites on one input), the
# cross-attention k/v (2 sites on the context)
SDXL_GROUPED = [(4096, 640, 640, 3), (1024, 1280, 1280, 3), (77, 1280, 1280, 3),
                (77, 2048, 640, 2), (77, 2048, 1280, 2)]


@pytest.mark.parametrize("M,K,N,n", SDXL_GROUPED)
def test_sdxl_grouped_launches_match_float64(M, K, N, n):
    """One grouped forward and one grouped dX launch per family (lora_b200.set_grouping): each site's
    output, the summed input gradient and every dA / dB against the float64 oracle, with
    test_grouping_gpu.py's forward bound and test_kernels_gpu.py's backward bound."""
    import lora_b200 as L
    from oracle import lora_ops as O

    class Attention(nn.Module):
        def __init__(self):
            super().__init__()
            for name in ("to_q", "to_k", "to_v")[3 - n:]:
                setattr(self, name, nn.Linear(K, N, bias=False))

    torch.manual_seed(0)
    att = Attention().to(DEV).to(torch.bfloat16)
    att.requires_grad_(False)
    L.inject_trainable_lora(att, r=4)
    sites = [m for m in att.modules() if type(m).__name__ == "LoraInjectedLinear"]
    assert len(sites) == n
    for m in sites:
        m.lora_up.weight.data.normal_(0, 0.05)
    x = torch.randn(M, K, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    gys = [torch.randn(M, N, device=DEV, dtype=torch.bfloat16) for _ in sites]
    L.set_grouping(True)
    try:
        for _ in range(2):                                # learning: the sites share x
            for m in sites:
                m(x)
        fam = att.__dict__["_lb_groups"].groups[id(sites[0])]
        assert fam is not None and len(fam) == n
        for m in sites:
            m.lora_up.weight.grad = m.lora_down.weight.grad = None
        ys = [m(x) for m in sites]                        # the first call launches the family
        torch.autograd.backward(ys, gys)
        torch.cuda.synchronize()
    finally:
        L.set_grouping(False)
    dx = torch.zeros(M, K, dtype=torch.float64)
    for m, y, gy in zip(sites, ys, gys):
        W = m.linear.weight.detach()
        want = O.lora_linear_forward(x.detach(), W, None, m.lora_down.weight, m.lora_up.weight, 1.0)
        assert rel(y, want) < 2 ** -7
        dX, dA, dB = O.lora_linear_backward(gy, x.detach(), W, m.lora_down.weight, m.lora_up.weight, 1.0)
        dx += dX
        assert rel(m.lora_down.weight.grad, dA) < 2e-2 and rel(m.lora_up.weight.grad, dB) < 2e-2
    assert rel(x.grad, dx) < 2e-2


# ------------------------------------------------------------------------------------ conv census
def _sdxl_conv_sites():
    """(H, W, Cin, Cout, k) of every conv site of the extended target set (the ResnetBlock2D convs) of
    UNetConfig.sdxl() at 128 x 128 latents, read from a meta-device forward of the preset."""
    import lora_b200 as L
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from oracle.ref_modules import ref_find_sites
    with torch.device("meta"):
        unet = UNet2DConditionModel(UNetConfig.sdxl())
    seen = set()

    def hook(m, inp, out):
        seen.add((inp[0].shape[2], inp[0].shape[3], m.in_channels, m.out_channels, m.kernel_size[0]))

    for _, _, m in ref_find_sites(unet, set(L.UNET_EXTENDED_TARGET_REPLACE), (nn.Conv2d,)):
        m.register_forward_hook(hook)
    meta = dict(device="meta")
    unet(torch.zeros(1, 4, 128, 128, **meta), torch.zeros(1, dtype=torch.long, **meta),
         torch.zeros(1, 77, 2048, **meta),
         added_cond_kwargs={"text_embeds": torch.zeros(1, 1280, **meta), "time_ids": torch.zeros(1, 6, **meta)})
    return sorted(seen, reverse=True)


# ranks and output dtypes cycle over the sites: every rank pad (16, 32, 64) and both 16-bit types
_RANKS = (4, 8, 16, 32, 64)
CONV_SDXL = [(1, H, W, cin, cout, k, _RANKS[i % 5], (BF, FP)[i % 2])
             for i, (H, W, cin, cout, k) in enumerate(_sdxl_conv_sites())]


def test_sdxl_conv_census_covers_128_64_32():
    assert {c[1] for c in CONV_SDXL} == {128, 64, 32} and len(CONV_SDXL) == 21


@pytest.mark.parametrize("case", CONV_SDXL, ids=lambda c: "n{}_{}x{}_{}to{}_k{}_r{}_{}".format(*c[:7], str(c[7])[6:]))
def test_conv_sites_at_128_64_32_match_float64(case):
    """test_conv_kernels_gpu.py's census check (frozen conv, T, full output, input gradient, dA / dB;
    whole image, border ring and last tile row / column)."""
    CK.test_conv_kernels_match_float64(case)


# ------------------------------------------------------------------------------------ models
def _tie(dst: nn.Module, src: nn.Module):
    """dst (same architecture, built on the meta device) uses src's parameters and buffers."""
    for (_, md), (_, ms) in zip(dst.named_modules(), src.named_modules()):
        for k in ms._parameters:
            md._parameters[k] = ms._parameters[k]
        for k in ms._buffers:
            md._buffers[k] = ms._buffers[k]


def _xl_pair(unet_cfg, tiny, seed=0, r=4, up_std=0.02):
    """(ours (unet, te1, te2), reference (unet, te1, te2), ref unet sites, ref te1 sites, ref te2 sites):
    fp32 weights, shared frozen weights and equal non-zero LoRA factors on both sides."""
    import lora_b200 as L
    from lora_b200.host.clip import build_sdxl_text_encoders
    from lora_b200.host.unet_sd15 import UNet2DConditionModel
    from oracle.ref_modules import ref_inject
    torch.manual_seed(seed)
    with torch.device(DEV):
        unet = UNet2DConditionModel(unet_cfg)
        te1, te2 = build_sdxl_text_encoders(tiny=tiny)
    unet = unet.to(memory_format=torch.channels_last)
    ours = (unet, te1, te2)
    for m in ours:
        m.requires_grad_(False)
    with torch.device("meta"):
        refs = (UNet2DConditionModel(unet_cfg),) + tuple(build_sdxl_text_encoders(tiny=tiny))
    for d, s in zip(refs, ours):
        _tie(d, s)
    L.inject_trainable_lora(unet, r=r)
    for te in (te1, te2):
        L.inject_trainable_lora(te, target_replace_module={"CLIPAttention"}, r=r)
    us = ref_inject(refs[0], {"CrossAttention", "Attention", "GEGLU"}, r=r)
    ts1 = ref_inject(refs[1], {"CLIPAttention"}, r=r)
    ts2 = ref_inject(refs[2], {"CLIPAttention"}, r=r)
    mine = [m for mdl in ours for m in mdl.modules() if type(m).__name__ == "LoraInjectedLinear"]
    assert len(mine) == len(us) + len(ts1) + len(ts2)
    g = torch.Generator(device=DEV).manual_seed(3)
    for o, rs in zip(mine, us + ts1 + ts2):
        o.lora_up.weight.data.normal_(0, up_std, generator=g)
        rs.up.data.copy_(o.lora_up.weight.data)
        rs.down.data.copy_(o.lora_down.weight.data)
    return ours, refs, us, ts1, ts2


def _ids(batch, vocab_hi, eos, gen, lengths=(11, 30)):
    ids = torch.randint(0, vocab_hi, (batch, 77), device=DEV, generator=gen)
    for b in range(batch):
        ids[b, lengths[b % len(lengths)]:] = eos
    return ids


def _draw(step, shape):
    g = torch.Generator(device=DEV).manual_seed(2000 + step)
    noise = torch.randn(shape, device=DEV, generator=g)
    t = torch.randint(0, 1000, (shape[0],), device=DEV, generator=g).long()
    return noise, t


def _live_ref_params(ref, ts1):
    """The oracle's factors that get a gradient, in the arena's order: encoder 1's last layer (its last
    4 sites) feeds only hidden_states[-1]."""
    dead = {id(p) for s in ts1[-4:] for p in (s.up, s.down)}
    return [p for p in ref.unet_params + ref.text_params if id(p) not in dead]


def test_sdxl_1024_bf16_step_eager_and_graph_match_reference_step():
    """Full-size SDXL UNet and both encoders, LoRA r=4 on 630 + 176 sites, 1024 px, bf16 autocast,
    grouping on: the first step eager, then graph replays, against RefXLStep."""
    import lora_b200 as L
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNetConfig
    from lora_b200.train import LoraXLTrainStep, StepConfig
    from oracle.ref_step_xl import RefXLStep
    ours, refs, us, ts1, ts2 = _xl_pair(UNetConfig.sdxl(), tiny=False)
    assert len(us) == 630 and len(ts1) == 48 and len(ts2) == 128
    shape = (1, 4, 128, 128)
    L.set_grouping(True)
    try:
        cfg = StepConfig(use_cuda_graph=True, graph_warmup=2, autocast_dtype=torch.bfloat16, external_noise=True)
        tr = LoraXLTrainStep(*ours, cfg, latent_shape=shape, seq_len=77, device=DEV)
        assert len(tr.arena.base_lr) == 3
        ref = RefXLStep(*refs, DDPMNoiser(device=DEV), us, ts1, ts2, autocast_dtype=torch.bfloat16)
        gi = torch.Generator(device=DEV).manual_seed(7)
        lat = torch.randn(shape, device=DEV, generator=gi) * 0.13025
        ids, ids2 = _ids(1, 49406, 49407, gi), _ids(1, 49406, 49407, gi, lengths=(17,))
        tid = tr.time_ids.clone()
        assert tid.tolist() == [[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]]
        tr.latents.copy_(lat); tr.input_ids.copy_(ids); tr.input_ids_2.copy_(ids2)
        xl = dict(input_ids_2=ids2, time_ids=tid)

        live = _live_ref_params(ref, ts1)
        noise, t = _draw(0, shape)
        loss_r = ref.forward_loss(lat, ids, noise, t, **xl)
        loss_r.backward()
        g_ref = torch.cat([p.grad.flatten() for p in live]).clone()
        ref.opt.zero_grad()
        tr.noise.copy_(noise); tr.timesteps.copy_(t)
        tr._fwd_bwd()
        g_ours = torch.cat([p.grad.flatten() for p in tr.arena.parameters()]).clone()
        assert g_ours.numel() == g_ref.numel()
        assert abs(float(tr.loss) - float(loss_r)) < 1e-2 * abs(float(loss_r))
        assert rel(g_ours, g_ref) < 3e-2
        n_te2 = sum(p.numel() for s in ts2 for p in (s.up, s.down))
        assert float(g_ours[-n_te2:].norm()) > 0                    # encoder 2 trained
        tr.arena.zero_grad()

        p0 = torch.cat([p.detach().flatten() for p in tr.arena.parameters()]).clone()
        traj = []
        for step in range(4):
            noise, t = _draw(step, shape)
            l_ref = float(ref.step(lat, ids, noise=noise, timesteps=t, **xl))
            tr.noise.copy_(noise); tr.timesteps.copy_(t)
            if step == 0:
                tr._body()
                l_ours = float(tr.loss)
                tr.prepare()
                assert tr.graph is not None, tr.graph_error
                assert tr.graph_update is None                      # one graph per step
                assert int(tr.arena.step_dev) == 1
            else:
                l_ours = float(tr.step_device())
            traj.append((l_ours, l_ref))
            assert abs(l_ours - l_ref) < 1e-2 * abs(l_ref), (step, traj)
        assert int(tr.arena.step_dev) == 4
        p_ref = torch.cat([p.detach().flatten().float() for p in live])
        p_ours = torch.cat([p.detach().flatten() for p in tr.arena.parameters()])
        assert rel(p_ours - p0, p_ref - p0) < 0.5
        # encoder 1's last layer is not trained, as torch's AdamW leaves a parameter without gradient
        for s in ts1[-4:]:
            assert s.up.grad is None
    finally:
        L.set_grouping(False)


# ------------------------------------------------------------------------------------ tiny variants
TINY = (2, 4, 16, 16)


def _tiny_inputs(seed=8):
    gi = torch.Generator(device=DEV).manual_seed(seed)
    lat = torch.randn(TINY, device=DEV, generator=gi) * 0.13025
    return lat, _ids(2, 998, 999, gi), _ids(2, 998, 999, gi, lengths=(5, 40))


@pytest.mark.parametrize("variant", ["plain", "plain_unfused", "prior", "encode_images", "grad_scaler"])
def test_tiny_sdxl_step_variants_match_oracle(variant):
    """Three steps of LoraXLTrainStep against RefXLStep with the same draws; grad_scaler runs fp16 autocast
    with torch.amp.GradScaler's constants, the oracle fp16 autocast without a scaler (an applied step
    updates the same)."""
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNetConfig
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    from lora_b200.train import LoraXLTrainStep, StepConfig
    from oracle.ref_step_xl import RefXLStep
    from oracle.vae_ref import encode
    ours, refs, us, ts1, ts2 = _xl_pair(UNetConfig.sdxl_tiny(), tiny=True, up_std=0.05)
    fp16 = variant == "grad_scaler"
    ac = FP if fp16 else BF
    kw = dict(use_cuda_graph=False, autocast_dtype=ac, external_noise=True, t_multiplier=0.8,
              with_prior_preservation=variant == "prior", prior_loss_weight=0.7,
              fused_glue=variant != "plain_unfused")
    vae = None
    if fp16:
        kw.update(compute_dtype=FP, grad_scaler=True, init_scale=1024.0)
    if variant == "encode_images":
        kw.update(encode_images=True, vae_scaling=0.13025)
        torch.manual_seed(4)
        vae = AutoencoderKL(VAEConfig.tiny()).to(DEV).to(memory_format=torch.channels_last)
        vae.requires_grad_(False)
    tr = LoraXLTrainStep(*ours, StepConfig(**kw), latent_shape=TINY, seq_len=77, device=DEV, vae=vae)
    ref = RefXLStep(*refs, DDPMNoiser(device=DEV), us, ts1, ts2, autocast_dtype=ac, t_multiplier=0.8)
    lat, ids, ids2 = _tiny_inputs()
    tid = torch.tensor([[128.0, 128, 0, 0, 128, 128], [160, 96, 16, 0, 128, 128]], device=DEV)
    tr.input_ids.copy_(ids); tr.input_ids_2.copy_(ids2); tr.time_ids.copy_(tid)
    lk = dict(input_ids_2=ids2, time_ids=tid)
    if variant == "prior":
        lk.update(prior_loss_weight=0.7)
    gi = torch.Generator(device=DEV).manual_seed(9)
    for step in range(3):
        noise, t = _draw(100 + step, TINY)
        t = t % 800
        tr.noise.copy_(noise); tr.timesteps.copy_(t)
        if variant == "encode_images":
            pixels = torch.randint(0, 256, (2, 128, 128, 3), device=DEV, generator=gi, dtype=torch.uint8)
            pe = torch.randn(TINY, device=DEV, generator=gi)
            tr.pixels.copy_(pixels); tr.posterior_noise.copy_(pe)
            latents, _ = encode(vae, pixels, pe, scaling=0.13025)
        else:
            latents = lat
            tr.latents.copy_(lat)
        l_ref = float(ref.step(latents, ids, noise=noise, timesteps=t, **lk))
        l_ours = float(tr.step_device())
        assert l_ours == l_ours and l_ref == l_ref
        assert abs(l_ours - l_ref) < 1e-2 * abs(l_ref), (step, l_ours, l_ref)
        if variant == "encode_images":
            assert rel(tr.latents, latents) < 1e-5
        if fp16:
            assert not tr.arena.step_was_skipped()


def _tiny_engine(graph, ckpt=False, grouping=False, time_gain=1.0):
    import lora_b200 as L
    from lora_b200.host.unet_sd15 import UNetConfig
    from lora_b200.train import LoraXLTrainStep, StepConfig
    L.set_grouping(grouping)
    ours, *_ = _xl_pair(UNetConfig.sdxl_tiny(), tiny=True, up_std=0.05)
    ours[0].add_embedding.linear_2.weight.data.mul_(time_gain)     # a louder text_time branch
    cfg = StepConfig(use_cuda_graph=graph, graph_warmup=2, autocast_dtype=BF, external_noise=True,
                     gradient_checkpointing=ckpt)
    return LoraXLTrainStep(*ours, cfg, latent_shape=TINY, seq_len=77, device=DEV)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_tiny_sdxl_checkpointed_step_matches_plain_step(graph):
    """gradient_checkpointing recomputes the UNet blocks and BOTH encoders' layers: the same first loss and
    first-step gradients, and factors within 1e-5 after 3 steps."""
    import lora_b200 as L
    lat, ids, ids2 = _tiny_inputs()
    out = []
    try:
        for ckpt in (False, True):
            tr = _tiny_engine(graph, ckpt)
            assert tr.unet.is_gradient_checkpointing == ckpt
            assert tr.text_encoder.is_gradient_checkpointing == ckpt
            assert tr.text_encoder_2.is_gradient_checkpointing == ckpt
            tr.latents.copy_(lat); tr.input_ids.copy_(ids); tr.input_ids_2.copy_(ids2)
            noise, t = _draw(0, TINY)
            tr.noise.copy_(noise); tr.timesteps.copy_(t)
            tr._fwd_bwd()
            g0 = tr.arena.g[:tr.arena.n_params].clone()
            tr.arena.zero_grad()
            if graph:
                tr.prepare()
                assert tr.graph is not None, tr.graph_error
            p_init = tr.arena.p[:tr.arena.n_params].clone()
            losses = []
            for step in range(3):
                noise, t = _draw(step, TINY)
                tr.noise.copy_(noise); tr.timesteps.copy_(t)
                losses.append(tr.step_device().clone())
            torch.cuda.synchronize()
            out.append((g0, torch.stack(losses), p_init, tr.arena.p[:tr.arena.n_params].clone()))
    finally:
        L.set_grouping(False)
    (g_a, l_a, i_a, p_a), (g_b, l_b, i_b, p_b) = out
    assert torch.equal(i_a, i_b) and not torch.equal(p_a, i_a)
    assert float(g_a.norm()) > 0 and rel(g_b, g_a) < 1e-5
    assert torch.equal(l_a[0], l_b[0]), (l_a, l_b)
    assert rel(l_b, l_a) < 1e-5 and rel(p_b, p_a) < 1e-5


def test_time_ids_written_between_replays_change_the_loss_as_an_eager_step_does():
    """Graph replays read `time_ids` from its static buffer: new ids given to step_host between two
    replays move the loss as they move an eager step's. A replay and an eager step of the same step
    differ by bf16 rounding (the frozen layers' cuBLAS and cuDNN calls may pick other kernels under
    capture), so the check is that the replay with the new ids stays as close to the eager step with
    the new ids as the first replay was to the first eager step, while the new ids move the loss far
    more than that."""
    lat, ids, ids2 = _tiny_inputs()
    new = torch.tensor([[1024.0, 64, 512, 256, 96, 2048], [64, 1024, 0, 768, 2048, 64]])
    g_eng = _tiny_engine(graph=True, time_gain=8.0)
    g_eng.prepare()
    assert g_eng.graph is not None and g_eng.graph_update is None, g_eng.graph_error
    e_eng = _tiny_engine(graph=False, time_gain=8.0)
    assert torch.equal(g_eng.arena.p, e_eng.arena.p)
    losses = {"graph": [], "eager": []}
    for step, tid in enumerate((None, new)):
        noise, t = _draw(step, TINY)
        for eng in (g_eng, e_eng):
            eng.noise.copy_(noise); eng.timesteps.copy_(t)
        e_eng.latents.copy_(lat); e_eng.input_ids.copy_(ids); e_eng.input_ids_2.copy_(ids2)
        if tid is not None:                  # the eager engine's loss with the old ids, no update
            e_eng._fwd_bwd()
            old = float(e_eng.loss)
            e_eng.arena.zero_grad()
            e_eng.time_ids.copy_(tid)
        h = g_eng.step_host(lat.cpu(), ids.cpu(), ids2.cpu(), time_ids=tid)
        torch.cuda.synchronize()
        losses["graph"].append(float(h))
        losses["eager"].append(float(e_eng.step_device()))
    assert torch.equal(g_eng.time_ids.cpu(), new)
    (g0, g1), (e0, e1) = losses["graph"], losses["eager"]
    floor = max(abs(g0 - e0), 1e-6 * abs(e0))
    assert abs(g0 - e0) <= 2e-3 * abs(e0), losses             # bf16 rounding
    assert abs(g1 - e1) <= 4 * floor, (floor, losses)
    assert abs(e1 - old) > 5 * max(abs(g1 - e1), floor), (old, losses)


def test_sdxl_step_is_one_graph_and_its_launch_count_is_stable():
    """With grouping on, the captured step is one graph (no second graph around a collective, no host
    sync refused by the capture), and an eager step's launch count is stable from step to step."""
    from lora_b200 import ops
    import lora_b200 as L
    tr = _tiny_engine(graph=False, grouping=True)
    try:
        lat, ids, ids2 = _tiny_inputs()
        tr.latents.copy_(lat); tr.input_ids.copy_(ids); tr.input_ids_2.copy_(ids2)
        noise, t = _draw(0, TINY)
        tr.noise.copy_(noise); tr.timesteps.copy_(t)
        counts = []
        for _ in range(3):
            ops.LAUNCH_COUNT = 0
            tr._body()
            counts.append(ops.LAUNCH_COUNT)
        assert counts[1] == counts[2] > 0, counts
        tr.cfg.use_cuda_graph = True
        tr.prepare()
        assert tr.graph is not None and tr.graph_update is None, tr.graph_error
        loss = float(tr.step_device())
        assert loss == loss
    finally:
        L.set_grouping(False)
