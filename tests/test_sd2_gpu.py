"""SD 2.x on the GPU: the v-prediction target from the step prologue (lb_step_prologue_v), the fused
linear and conv kernels at SD2.1-768 site shapes against float64, and v-prediction training steps
(full-size SD2.1-768, fp32 split mode, the tiny step variants, textual inversion, the joint
embedding step) against the oracle step (oracle/ref_step_v.py, pinned to the reference's `loss_step`
with a v-prediction scheduler by tests/golden/pti_loss_step_v.pt).

Bounds are those of the suites the checks come from: test_kernels_gpu.py (linear kernels),
test_conv_kernels_gpu.py (conv kernels, whose checks are called here on the new shapes),
test_zz_fullsize_parity_gpu.py (full-size step: loss 1e-2 relative, first-step gradient 3e-2,
update direction < 0.5 after 4 steps; fp32 split mode: |loss - oracle| <= 1e-4) and
test_zz_pti_variants_gpu.py (tiny steps: loss 1e-2 relative under bf16 autocast)."""
import copy

import pytest
import torch

import test_conv_kernels_gpu as CK
import test_kernels_gpu as KG

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF, FP = torch.bfloat16, torch.float16


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ------------------------------------------------------------------------------------ prologue
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("inpaint", [False, True])
def test_step_prologue_velocity_is_bit_exact(out_dtype, inpaint):
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.step_ops import step_prologue
    torch.manual_seed(0)
    noiser = DDPMNoiser(device=DEV)
    lat = torch.randn(3, 4, 24, 40, device=DEV) * 0.18215
    eps = torch.randn_like(lat)
    t = torch.tensor([0, 517, 999], device=DEV)
    mask = (torch.rand(3, 1, 24, 40, device=DEV) > 0.5).float() if inpaint else None
    ml = torch.randn_like(lat) if inpaint else None
    noisy, v = step_prologue(lat, eps, t, noiser, out_dtype, mask, ml, velocity=True)
    a = noiser.sqrt_acp[t].view(-1, 1, 1, 1)
    s = noiser.sqrt_one_minus_acp[t].view(-1, 1, 1, 1)
    assert v.dtype == torch.float32 and v.shape == lat.shape and v.is_contiguous()
    assert torch.equal(v, a * eps - s * lat)
    assert torch.equal(v, noiser.get_velocity(lat, eps, t))
    noisy_eps = step_prologue(lat, eps, t, noiser, out_dtype, mask, ml)      # lb_step_prologue
    assert torch.equal(noisy, noisy_eps)
    assert noisy.is_contiguous(memory_format=torch.channels_last)


def test_step_prologue_velocity_inside_a_cuda_graph():
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.step_ops import step_prologue
    noiser = DDPMNoiser(device=DEV)
    lat = torch.zeros(2, 4, 96, 96, device=DEV)
    eps, t = torch.zeros_like(lat), torch.zeros(2, dtype=torch.long, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step_prologue(lat, eps, t, noiser, torch.bfloat16, velocity=True)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        noisy, v = step_prologue(lat, eps, t, noiser, torch.bfloat16, velocity=True)
    for rep in range(3):
        gen = torch.Generator(device=DEV).manual_seed(rep)
        lat.copy_(torch.randn(lat.shape, device=DEV, generator=gen))
        eps.copy_(torch.randn(lat.shape, device=DEV, generator=gen))
        t.copy_(torch.randint(0, 1000, (2,), device=DEV, generator=gen))
        v.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(v, noiser.get_velocity(lat, eps, t)), rep
        assert torch.equal(noisy, noiser.add_noise(lat, eps, t).to(torch.bfloat16)), rep


# ------------------------------------------------------------------------------------ linear census
# (M, K, N) of the SD2.1 768-v sites at batch 1 (96 x 96 latents)
SD21_LINEAR = [
    (9216, 320, 320), (9216, 320, 2560),          # level 1: q/k/v/out, GEGLU proj
    (2304, 640, 640), (2304, 640, 5120),          # level 2
    (576, 1280, 1280), (576, 1280, 10240),        # level 3
    (144, 1280, 1280),                            # mid block
    (77, 1024, 320), (77, 1024, 640), (77, 1024, 1280),   # attn2 to_k / to_v on the OpenCLIP-H states
    (77, 1024, 1024),                             # text encoder
]


@pytest.mark.parametrize("r", [4, 16, 64])
@pytest.mark.parametrize("M,K,N", SD21_LINEAR)
def test_sd21_linear_sites_match_float64(M, K, N, r):
    """test_kernels_gpu.py's checks and bounds: frozen GEMM + T (fp32 out), fused forward (bf16
    operands, fp32 and bf16 out), input gradient and dA / dB."""
    KG.test_base_gemm_and_T_fp32_out(M, K, N, r)
    KG.test_fused_forward_matches_oracle(M, K, N, r, torch.bfloat16)
    KG.test_backward_kernels_match_oracle(M, K, N, r)


# ------------------------------------------------------------------------------------ conv census
# Every (Cin, Cout, k) of the ResnetBlock2D convs (the extended sites) at 96 / 48 / 24 / 12: SD2.1
# 768-v and the SD1.5 768-px shape share them. 24 and 12 have ragged last tiles (TW 16 / 8).
CONV_96 = [
    (1, 96, 96, 320, 320, 3, 4, BF), (1, 96, 96, 960, 320, 3, 8, FP), (1, 96, 96, 640, 320, 3, 16, BF),
    (1, 96, 96, 960, 320, 1, 4, FP), (1, 96, 96, 640, 320, 1, 64, BF),
    (1, 48, 48, 320, 640, 3, 4, BF), (1, 48, 48, 640, 640, 3, 32, BF), (1, 48, 48, 1920, 640, 3, 8, FP),
    (1, 48, 48, 1280, 640, 3, 4, BF), (1, 48, 48, 960, 640, 3, 16, BF),
    (1, 48, 48, 320, 640, 1, 4, BF), (1, 48, 48, 1920, 640, 1, 8, FP), (1, 48, 48, 1280, 640, 1, 4, BF),
    (1, 48, 48, 960, 640, 1, 16, FP),
    (1, 24, 24, 640, 1280, 3, 4, BF), (1, 24, 24, 1280, 1280, 3, 8, FP), (1, 24, 24, 2560, 1280, 3, 16, BF),
    (1, 24, 24, 1920, 1280, 3, 64, BF),
    (1, 24, 24, 640, 1280, 1, 4, FP), (1, 24, 24, 2560, 1280, 1, 8, BF), (1, 24, 24, 1920, 1280, 1, 4, BF),
    (1, 12, 12, 1280, 1280, 3, 4, BF), (1, 12, 12, 2560, 1280, 3, 32, FP),
    (1, 12, 12, 2560, 1280, 1, 4, BF),
]


@pytest.mark.parametrize("case", CONV_96, ids=lambda c: "n{}_{}x{}_{}to{}_k{}_r{}_{}".format(*c[:7], str(c[7])[6:]))
def test_conv_sites_at_96_48_24_12_match_float64(case):
    """test_conv_kernels_gpu.py's census check (frozen conv, T, full output, input gradient, dA / dB;
    whole image, border ring and last tile row / column)."""
    CK.test_conv_kernels_match_float64(case)


# ------------------------------------------------------------------------------------ models
def _pair(unet_cfg, sd2_text, seed=0, r=4, tiny=False, up_std=0.02, in_channels=None):
    """(ours unet, ours text, ref unet, ref text, ref unet sites, ref text sites): fp32 weights,
    identical frozen weights and non-zero LoRA factors on both sides."""
    import lora_b200 as L
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel
    from oracle.ref_modules import ref_inject
    if in_channels is not None:
        unet_cfg.in_channels = in_channels
    torch.manual_seed(seed)
    with torch.device(DEV):
        unet = UNet2DConditionModel(unet_cfg)
        text = build_text_encoder(tiny=tiny, sd2=sd2_text)
    unet.requires_grad_(False)
    text.requires_grad_(False)
    unet = unet.to(memory_format=torch.channels_last)
    unet_r, text_r = copy.deepcopy(unet), copy.deepcopy(text)
    L.inject_trainable_lora(unet, r=r)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=r)
    us = ref_inject(unet_r, {"CrossAttention", "Attention", "GEGLU"}, r=r)
    ts = ref_inject(text_r, {"CLIPAttention"}, r=r)
    ours = [m for m in list(unet.modules()) + list(text.modules()) if type(m).__name__ == "LoraInjectedLinear"]
    assert len(ours) == len(us) + len(ts)
    g = torch.Generator(device=DEV).manual_seed(3)
    for o, rs in zip(ours, us + ts):
        o.lora_up.weight.data.normal_(0, up_std, generator=g)
        rs.up.data.copy_(o.lora_up.weight.data)
        rs.down.data.copy_(o.lora_down.weight.data)
    return unet, text, unet_r, text_r, us, ts


def _draw(step, shape):
    g = torch.Generator(device=DEV).manual_seed(2000 + step)
    noise = torch.randn(shape, device=DEV, generator=g)
    t = torch.randint(0, 1000, (shape[0],), device=DEV, generator=g).long()
    return noise, t


def test_sd21_768_v_bf16_step_eager_and_graph_match_reference_step():
    import lora_b200 as L
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNetConfig
    from lora_b200.train import LoraTrainStep, StepConfig
    from oracle.ref_step_v import RefDreamboothStepV as RefDreamboothStep
    unet, text, unet_r, text_r, us, ts = _pair(UNetConfig.sd21(), True)
    assert len(us) == 144 and len(ts) == 92
    shape = (1, 4, 96, 96)
    V = "v_prediction"
    L.set_grouping(True)
    try:
        cfg = StepConfig(use_cuda_graph=True, graph_warmup=2, autocast_dtype=torch.bfloat16, external_noise=True,
                         prediction_type=V)
        tr = LoraTrainStep(unet, text, cfg, latent_shape=shape, seq_len=77, device=DEV)
        ref = RefDreamboothStep(unet_r, text_r, DDPMNoiser(device=DEV), us, ts, autocast_dtype=torch.bfloat16)
        torch.manual_seed(7)
        lat = torch.randn(shape, device=DEV) * 0.18215
        ids = torch.randint(0, text.config.vocab_size, (1, 77), device=DEV)
        tr.latents.copy_(lat)
        tr.input_ids.copy_(ids)

        noise, t = _draw(0, shape)
        loss_r = ref.forward_loss(lat, ids, noise, t, prediction_type=V)
        loss_r.backward()
        g_ref = torch.cat([p.grad.flatten() for p in ref.unet_params + ref.text_params]).clone()
        ref.opt.zero_grad()
        tr.noise.copy_(noise); tr.timesteps.copy_(t)
        tr._fwd_bwd()
        g_ours = torch.cat([p.grad.flatten() for p in tr.arena.parameters()]).clone()
        assert abs(float(tr.loss) - float(loss_r)) < 1e-2 * abs(float(loss_r))
        assert rel(g_ours, g_ref) < 3e-2
        tr.arena.zero_grad()

        p0 = torch.cat([p.detach().flatten() for p in tr.arena.parameters()]).clone()
        traj = []
        for step in range(4):
            noise, t = _draw(step, shape)
            l_ref = float(ref.step(lat, ids, noise=noise, timesteps=t, prediction_type=V))
            tr.noise.copy_(noise); tr.timesteps.copy_(t)
            if step == 0:
                tr._body()
                l_ours = float(tr.loss)
                tr.prepare()
                assert tr.graph is not None, tr.graph_error
                assert int(tr.arena.step_dev) == 1
            else:
                l_ours = float(tr.step_device())
            traj.append((l_ours, l_ref))
            assert abs(l_ours - l_ref) < 1e-2 * abs(l_ref), (step, traj)
        assert int(tr.arena.step_dev) == 4
        p_ref = torch.cat([p.detach().flatten().float() for p in ref.unet_params + ref.text_params])
        p_ours = torch.cat([p.detach().flatten() for p in tr.arena.parameters()])
        assert rel(p_ours - p0, p_ref - p0) < 0.5
    finally:
        L.set_grouping(False)


def test_sd2_64_fp32_split_mode_v_loss_within_1e4():
    import lora_b200 as L
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNetConfig
    from lora_b200.train import LoraTrainStep, StepConfig
    from oracle.ref_step_v import RefDreamboothStepV as RefDreamboothStep
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    L.set_fp32_mode("split")
    try:
        unet, text, unet_r, text_r, us, ts = _pair(UNetConfig.sd21(), True, seed=1)
        shape = (1, 4, 64, 64)
        cfg = StepConfig(use_cuda_graph=False, autocast_dtype=None, external_noise=True, prediction_type="v_prediction")
        tr = LoraTrainStep(unet, text, cfg, latent_shape=shape, seq_len=77, device=DEV)
        ref = RefDreamboothStep(unet_r, text_r, DDPMNoiser(device=DEV), us, ts)
        torch.manual_seed(8)
        lat = torch.randn(shape, device=DEV) * 0.18215
        ids = torch.randint(0, text.config.vocab_size, (1, 77), device=DEV)
        tr.latents.copy_(lat)
        tr.input_ids.copy_(ids)
        for step in range(2):
            noise, t = _draw(10 + step, shape)
            l_ref = float(ref.step(lat, ids, noise=noise, timesteps=t, prediction_type="v_prediction"))
            tr.noise.copy_(noise); tr.timesteps.copy_(t)
            l_ours = float(tr.step_device())
            assert abs(l_ours - l_ref) <= 1e-4, (step, l_ours, l_ref)
    finally:
        L.set_fp32_mode("bf16")
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


# ------------------------------------------------------------------------------------ tiny variants
@pytest.mark.parametrize("variant", ["plain", "plain_unfused", "masked", "prior", "inpaint"])
def test_tiny_sd2_v_step_variants_match_oracle(variant):
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNetConfig
    from lora_b200.train import LoraTrainStep, StepConfig
    from oracle.ref_step_v import RefDreamboothStepV as RefDreamboothStep
    inpaint = variant == "inpaint"
    unet, text, unet_r, text_r, us, ts = _pair(UNetConfig.sd2_tiny(), True, tiny=True, up_std=0.05,
                                              in_channels=9 if inpaint else 4)
    shape = (2, 4, 16, 16)
    cfg = StepConfig(use_cuda_graph=False, autocast_dtype=torch.bfloat16, t_multiplier=0.8,
                     prediction_type="v_prediction", use_mask=variant == "masked", train_inpainting=inpaint,
                     with_prior_preservation=variant == "prior", prior_loss_weight=0.7,
                     fused_glue=variant != "plain_unfused")
    tr = LoraTrainStep(unet, text, cfg, latent_shape=shape, seq_len=77, device=DEV)
    ref = RefDreamboothStep(unet_r, text_r, DDPMNoiser(device=DEV), us, ts, autocast_dtype=torch.bfloat16,
                            t_multiplier=0.8)
    gi = torch.Generator(device=DEV).manual_seed(8)
    lat = torch.randn(shape, device=DEV, generator=gi) * 0.18215
    ids = torch.randint(0, 1000, (2, 77), device=DEV, generator=gi)
    tr.latents.copy_(lat)
    tr.input_ids.copy_(ids)
    kw = {"prediction_type": "v_prediction"}
    if variant == "masked":
        img_mask = (torch.rand(2, 1, 128, 128, device=DEV, generator=gi) > 0.4).float()
        tr.set_loss_mask(img_mask)
        kw.update(loss_mask=img_mask, mask_temperature=1.0)
    if variant == "prior":
        kw.update(prior_loss_weight=0.7)
    if inpaint:
        im = (torch.rand(2, 1, 16, 16, device=DEV, generator=gi) > 0.5).float()
        ml = torch.randn(shape, device=DEV, generator=gi) * 0.18215
        tr.inpaint_mask.copy_(im)
        tr.masked_latents.copy_(ml)
        kw.update(inpaint=(im, ml))
    for step in range(3):
        torch.manual_seed(100 + step)
        l_ref = float(ref.step(lat, ids, **kw))
        torch.manual_seed(100 + step)
        l_ours = float(tr.step_device())
        assert l_ours == l_ours and l_ref == l_ref
        assert abs(l_ours - l_ref) < 1e-2 * abs(l_ref), (step, l_ours, l_ref)


def test_textual_inversion_v_step_matches_oracle():
    """TextualInversionStep with prediction_type "v_prediction" against the oracle's full-table update
    (oracle/ti_ref.py) fed the dense gradient of the same v-prediction loss by plain autograd."""
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.train import StepConfig, TextualInversionStep
    from oracle.ti_ref import ti_table_step
    torch.manual_seed(0)
    unet = UNet2DConditionModel(UNetConfig.sd2_tiny()).to(DEV)
    te = build_text_encoder(tiny=True, sd2=True).to(DEV)
    unet.requires_grad_(False); te.requires_grad_(False)
    unet_r, te_r = copy.deepcopy(unet), copy.deepcopy(te)
    emb_r = te_r.get_input_embeddings()
    emb_r.weight.requires_grad_(True)
    V, D = emb_r.weight.shape
    tok = [V - 3, V - 1]
    index_updates = torch.zeros(V, dtype=torch.bool)
    index_updates[tok] = True
    orig = emb_r.weight.detach().clone()
    cfg = StepConfig(use_cuda_graph=False, external_noise=True, prediction_type="v_prediction")
    lr0 = 5e-3
    eng = TextualInversionStep(unet, te, tok, cfg, lr=lr0, latent_shape=(2, 4, 16, 16), device=DEV)
    noiser = DDPMNoiser(device=DEV)
    lat = torch.randn(2, 4, 16, 16, device=DEV) * 0.18215
    ids = torch.randint(0, V - 3, (2, 77), device=DEV)
    ids[0, 3], ids[1, 7] = tok[0], tok[1]
    eng.latents.copy_(lat); eng.input_ids.copy_(ids)
    o_table, o_m, o_v = orig.clone(), torch.zeros(V, D), torch.zeros(V, D)
    unet_r.eval(); te_r.train()
    for step in range(1, 3):
        g = torch.Generator(device=DEV).manual_seed(step)
        noise = torch.randn(2, 4, 16, 16, device=DEV, generator=g)
        t = torch.randint(0, 1000, (2,), device=DEV, generator=g)
        with torch.no_grad():
            emb_r.weight.copy_(o_table.to(DEV, torch.float32))
        emb_r.weight.grad = None
        pred = unet_r(noiser.add_noise(lat, noise, t), t, te_r(ids)[0]).sample
        a = noiser.sqrt_acp[t].view(-1, 1, 1, 1)
        s = noiser.sqrt_one_minus_acp[t].view(-1, 1, 1, 1)
        loss_r = torch.nn.functional.mse_loss(pred.float(), (a * noise - s * lat).float())
        loss_r.backward()
        o_table, o_m, o_v = ti_table_step(o_table, emb_r.weight.grad, o_m, o_v, step, lr0, index_updates, orig)
        eng.noise.copy_(noise); eng.timesteps.copy_(t)
        l_ours = float(eng.step_device())
        assert abs(l_ours - float(loss_r)) <= 1e-4 * abs(float(loss_r)) + 1e-6, (step, l_ours, float(loss_r))
        got = te.get_input_embeddings().weight.detach().double().cpu()
        assert float((got[tok] - o_table[tok]).norm() / o_table[tok].norm()) < 1e-3
        assert torch.equal(te.get_input_embeddings().weight.detach()[: V - 3], orig[: V - 3].to(DEV))
    eng.release()


def test_embedding_table_v_step_matches_oracle():
    """LoraEmbeddingStep(mode="table") with prediction_type "v_prediction" against RefJointStep (the
    oracle of cli_lora_pti.py's continue_inversion loop) with the same prediction type."""
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNetConfig
    from lora_b200.train import LoraEmbeddingStep, StepConfig
    from oracle.ref_step_v import RefJointStepV as RefJointStep
    unet, text, unet_r, text_r, us, ts = _pair(UNetConfig.sd2_tiny(), True, tiny=True, up_std=0.05)
    V = text.get_input_embeddings().weight.shape[0]
    tok = [V - 2, V - 1]
    lr, lr_text, lr_emb, wd = 1e-4, 1e-5, 5e-5, 1e-3
    cfg = StepConfig(use_cuda_graph=False, autocast_dtype=torch.bfloat16, t_multiplier=0.8, lr_step_first=True,
                     lr_scheduler="linear", max_train_steps=6, learning_rate=lr, learning_rate_text=lr_text,
                     adam_weight_decay=wd, external_noise=True, prediction_type="v_prediction")
    eng = LoraEmbeddingStep(unet, text, tok, cfg, lr_embedding=lr_emb, mode="table", latent_shape=(2, 4, 16, 16))
    ref = RefJointStep(unet_r, text_r, DDPMNoiser(device=DEV), us, ts, "table", lr=lr, lr_text=lr_text,
                       lr_embedding=lr_emb, lr_lambda=lambda k: max(0.0, 1.0 - k / 6), weight_decay=wd,
                       t_multiplier=0.8, autocast_dtype=torch.bfloat16)
    table0 = text.get_input_embeddings().weight.detach().clone()
    gi = torch.Generator(device=DEV).manual_seed(8)
    seen = set(tok)
    for _ in range(2):
        lat = torch.randn(2, 4, 16, 16, device=DEV, generator=gi) * 0.18215
        ids = torch.randint(0, 60, (2, 77), device=DEV, generator=gi)
        ids[0, 2], ids[1, 5] = tok[0], tok[1]
        noise = torch.randn(2, 4, 16, 16, device=DEV, generator=gi)
        t = torch.randint(0, 800, (2,), device=DEV, generator=gi)
        seen |= set(ids.reshape(-1).tolist())
        l_ref = float(ref.step(lat, ids, noise, t, prediction_type="v_prediction"))
        eng.latents.copy_(lat); eng.input_ids.copy_(ids); eng.noise.copy_(noise); eng.timesteps.copy_(t)
        l_ours = float(eng.step_device())
        assert abs(l_ours - l_ref) < 1e-2 * abs(l_ref), (l_ours, l_ref)
        got = text.get_input_embeddings().weight.detach().double()
        want = ref.table.detach().double()
        s = torch.tensor(sorted(seen), device=DEV)
        assert float((got[s] - want[s]).norm() / want[s].norm()) < 1e-3
        d_ours, d_ref = got[s] - table0[s].double(), want[s] - table0[s].double()
        assert float((d_ours * d_ref).sum() / (d_ours.norm() * d_ref.norm())) > 0.95
    eng.release()


def test_v_prediction_step_has_the_epsilon_step_launch_count():
    from lora_b200 import ops
    from lora_b200.host.unet_sd15 import UNetConfig
    from lora_b200.train import LoraTrainStep, StepConfig
    counts = {}
    for pt in ("epsilon", "v_prediction"):
        unet, text, *_ = _pair(UNetConfig.sd2_tiny(), True, tiny=True)
        cfg = StepConfig(use_cuda_graph=False, autocast_dtype=torch.bfloat16, prediction_type=pt)
        tr = LoraTrainStep(unet, text, cfg, latent_shape=(1, 4, 16, 16), device=DEV)
        tr._body()
        ops.LAUNCH_COUNT = 0
        tr._body()
        counts[pt] = ops.LAUNCH_COUNT
    assert counts["epsilon"] == counts["v_prediction"] > 0, counts
