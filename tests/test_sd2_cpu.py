"""SD 2.x on the CPU: the v-prediction oracle against the reference's own `loss_step`, the
prediction_type check, argument validation of lb_step_prologue_v through the C ABI, the SD2 LoRA
site census, and SD1.5 host models left exactly as they were (module tree, state_dict keys and
values for seed 0: the goldens depend on them)."""
import ctypes
import hashlib
import json
import os

import pytest
import torch

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def test_oracle_v_prediction_loss_matches_reference_loss_step_golden():
    """oracle/ref_step_v.py::forward_loss(prediction_type="v_prediction") against the losses of the
    reference's `loss_step` run with a v-prediction scheduler (scripts/make_golden.py::gen_loss_step_v):
    plain, t_mutliplier 0.8, masked, inpainting on the tiny SD1.5 models, plain on the tiny SD2 ones."""
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from oracle.ref_modules import ref_inject
    from oracle.ref_step_v import RefDreamboothStepV as RefDreamboothStep
    G = torch.load(os.path.join(GOLD, "pti_loss_step_v.pt"))
    assert G["prediction_type"] == "v_prediction"
    lat, ids = G["latents"], G["input_ids"]
    assert [c["name"] for c in G["cases"]] == ["plain", "t_mult_0.8", "masked_T1", "inpaint", "sd2_plain"]
    for case in G["cases"]:
        sd2 = case["model"] == "sd2_tiny"
        torch.manual_seed(G["model_seed"])
        cfg = UNetConfig.sd2_tiny() if sd2 else UNetConfig.tiny()
        cfg.in_channels = case["in_channels"]
        unet = UNet2DConditionModel(cfg)
        text = build_text_encoder(tiny=True, sd2=sd2)
        sites = ref_inject(unet, {"CrossAttention", "Attention", "GEGLU"}, r=4)
        gg = torch.Generator().manual_seed(G["up_seed"])
        for s in sites:
            s.down.data.normal_(0, 0.25, generator=gg)
            s.up.data.normal_(0, 0.05, generator=gg)
        kw = case["kwargs"]
        ref = RefDreamboothStep(unet, text, DDPMNoiser(device="cpu"), sites, None,
                                t_multiplier=kw.get("t_mutliplier", 1.0))
        unet.train(False), text.train(False)
        torch.manual_seed(G["step_seed"])
        noise = torch.randn_like(lat)
        t = torch.randint(0, int(1000 * ref.t_multiplier), (lat.shape[0],)).long()
        loss = ref.forward_loss(
            lat, ids, noise, t, prediction_type="v_prediction",
            loss_mask=G["loss_mask"] if case["with_mask"] else None,
            mask_temperature=kw.get("mask_temperature", 1.0),
            inpaint=(G["inpaint_mask"], G["masked_latents"]) if kw.get("train_inpainting") else None)
        assert abs(float(loss) - case["loss"]) <= 2e-6 * abs(case["loss"]), (case["name"], float(loss), case["loss"])
        # the epsilon loss of the same draw is a different number: the golden really pins the target
        torch.manual_seed(G["step_seed"])
        noise = torch.randn_like(lat)
        eps_loss = ref.forward_loss(lat, ids, noise, t, loss_mask=G["loss_mask"] if case["with_mask"] else None,
                                    inpaint=(G["inpaint_mask"], G["masked_latents"]) if kw.get("train_inpainting") else None)
        assert abs(float(eps_loss) - case["loss"]) > 1e-3 * abs(case["loss"])


def test_unknown_prediction_type_raises():
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.train import LoraEmbeddingStep, LoraTrainStep, StepConfig, TextualInversionStep
    from oracle.ref_step_v import RefDreamboothStepV as RefDreamboothStep
    torch.manual_seed(0)
    unet, text = UNet2DConditionModel(UNetConfig.tiny()), build_text_encoder(tiny=True)
    cfg = StepConfig(prediction_type="sample")
    with pytest.raises(ValueError, match="Unknown prediction type sample"):
        LoraTrainStep(unet, text, cfg, device="cpu")
    with pytest.raises(ValueError, match="Unknown prediction type sample"):
        TextualInversionStep(unet, text, [998], cfg, device="cpu")
    with pytest.raises(ValueError, match="Unknown prediction type sample"):
        LoraEmbeddingStep(unet, text, [998], cfg, lr_embedding=1e-3, device="cpu")
    ref = RefDreamboothStep(unet, text, DDPMNoiser(), [], None)
    with pytest.raises(ValueError, match="Unknown prediction type sample"):
        ref.forward_loss(torch.zeros(1, 4, 8, 8), torch.zeros(1, 77, dtype=torch.long), torch.zeros(1, 4, 8, 8),
                         torch.zeros(1, dtype=torch.long), prediction_type="sample")


def test_noiser_get_velocity_is_diffusers_formula():
    from lora_b200.host.ddpm import DDPMNoiser
    n = DDPMNoiser()
    g = torch.Generator().manual_seed(3)
    x0, eps = torch.randn(3, 4, 5, 6, generator=g), torch.randn(3, 4, 5, 6, generator=g)
    t = torch.tensor([0, 400, 999])
    v = n.get_velocity(x0, eps, t)
    for b in range(3):
        assert torch.equal(v[b], n.sqrt_acp[t[b]] * eps[b] - n.sqrt_one_minus_acp[t[b]] * x0[b])
    # x0 and eps are recovered from (noisy, v): the pair is a rotation of (x0, eps)
    noisy = n.add_noise(x0, eps, t)
    a, s = n.sqrt_acp[t].view(-1, 1, 1, 1), n.sqrt_one_minus_acp[t].view(-1, 1, 1, 1)
    assert torch.allclose(a * noisy - s * v, x0, atol=1e-5)


def test_step_prologue_v_argument_validation_without_gpu():
    from lora_b200 import _C
    L = _C.lib
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.c_void_p((ctypes.addressof(buf) + 255) & ~255)
    # null velocity, bad dtype, empty shape, inpainting mask without masked latents: refused before any CUDA call
    assert L.lb_step_prologue_v(p, p, p, p, p, 1000, None, None, p, 0, None, 1, 4, 8, 8, None) == -1
    assert L.lb_step_prologue_v(p, p, p, p, p, 1000, None, None, p, 7, p, 1, 4, 8, 8, None) == -3
    assert L.lb_step_prologue_v(p, p, p, p, p, 1000, None, None, p, 0, p, 0, 4, 8, 8, None) == -1
    assert L.lb_step_prologue_v(p, p, p, p, p, 0, None, None, p, 0, p, 1, 4, 8, 8, None) == -1
    assert L.lb_step_prologue_v(p, p, p, p, p, 1000, p, None, p, 0, p, 1, 4, 8, 8, None) == -1
    # the epsilon entry point keeps its signature and its checks
    assert L.lb_step_prologue(p, p, p, p, p, 1000, None, None, p, 7, 1, 4, 8, 8, None) == -3


def _sites(model):
    return [(n, m) for n, m in model.named_modules() if type(m).__name__ == "LoraInjectedLinear"]


def test_sd2_site_census_and_safeloras_layout(tmp_path):
    """SD2.1 (UNetConfig.sd21 + the OpenCLIP-H text encoder): 144 UNet default sites with the
    cross-attention to_k / to_v at K = 1024, 92 text sites of 1024 x 1024, linear proj_in / proj_out
    that are not sites; the saved file has the SD1.5 fixtures' key layout."""
    import lora_b200 as L
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    torch.manual_seed(0)
    unet = UNet2DConditionModel(UNetConfig.sd21())
    text = build_text_encoder(sd2=True)
    heads = [m.heads for n, m in unet.named_modules() if n.endswith("attn1")]
    # down 5, 5, 10, 10, 20, 20; up 20 x 3, 10 x 3, 5 x 3; mid 20: head dim 64 everywhere
    assert heads == [5, 5, 10, 10, 20, 20] + [20] * 3 + [10] * 3 + [5] * 3 + [20]
    for n, m in unet.named_modules():
        if type(m).__name__ == "Transformer2DModel":
            assert type(m.proj_in) is torch.nn.Linear and type(m.proj_out) is torch.nn.Linear
            assert m.transformer_blocks[0].attn1.to_q.out_features // m.transformer_blocks[0].attn1.heads == 64
    L.inject_trainable_lora(unet, r=4)
    L.inject_trainable_lora(text, target_replace_module=L.TEXT_ENCODER_DEFAULT_TARGET_REPLACE, r=4)
    us, ts = _sites(unet), _sites(text)
    assert len(us) == 144 and len(ts) == 92
    assert not any("proj_in" in n or "proj_out" in n for n, _ in us)
    kv = [(n, m) for n, m in us if ".attn2.to_k" in n or ".attn2.to_v" in n]
    assert len(kv) == 32 and all(m.linear.in_features == 1024 for _, m in kv)
    assert all(m.linear.in_features != 1024 for n, m in us if (n, m) not in kv)
    assert all((m.linear.in_features, m.linear.out_features) == (1024, 1024) for _, m in ts)
    path = str(tmp_path / "sd2.safetensors")
    L.save_safeloras({"unet": (unet, L.UNET_DEFAULT_TARGET_REPLACE),
                      "text_encoder": (text, L.TEXT_ENCODER_DEFAULT_TARGET_REPLACE)}, path)
    from safetensors import safe_open
    f = safe_open(path, framework="pt", device="cpu")
    want = {f"unet:{i}:{w}" for i in range(144) for w in ("up", "down")} | \
           {f"text_encoder:{i}:{w}" for i in range(92) for w in ("up", "down")}
    assert set(f.keys()) == want
    for i, (_, m) in enumerate(us):
        assert f.get_tensor(f"unet:{i}:down").shape == (4, m.linear.in_features)
        assert f.get_tensor(f"unet:{i}:up").shape == (m.linear.out_features, 4)
    # the same key scheme as the SD1.5 fixture files of the reference
    man = json.load(open(os.path.join(GOLD, "example_loras_manifest.json")))
    fixture_keys = next(set(e["tensors"]) for e in man.values() if any(k.startswith("unet:143:") for k in e["tensors"]))
    assert {k for k in fixture_keys if k.startswith("unet:")} == {k for k in want if k.startswith("unet:")}
    parsed = L.parse_safeloras(f)
    assert len(parsed["unet"][0]) == 288 and set(parsed["unet"][1]) == {4}
    assert len(parsed["text_encoder"][0]) == 184


def _fingerprint(model):
    sd = model.state_dict()
    h = hashlib.sha256()
    for k, v in sd.items():
        h.update(k.encode())
        h.update(str(tuple(v.shape)).encode())
    checksum = sum(float(v.double().sum()) + float((v.double() ** 2).sum()) for v in sd.values())
    return h.hexdigest()[:16], checksum, len(sd), len(list(model.modules()))


# measured with the host models before SD2 support was added (seed 0)
SD15_FINGERPRINTS = {
    "tiny": ("84eedbbe393fd8c6", 9037.468430077615, 324, 327),
    "tiny_text": ("a19b31f33308b8ff", 813.6650914183201, 36, 32),
    "sd15": ("5a7c305f603eb877", 306101.4317265935, 686, 684),
    "sd15_text": ("00126acd4c0abe6e", 83971.9111464127, 196, 152),
}


@pytest.mark.parametrize("name", list(SD15_FINGERPRINTS))
def test_sd15_host_models_unchanged(name):
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    make = {"tiny": lambda: UNet2DConditionModel(UNetConfig.tiny()),
            "tiny_text": lambda: build_text_encoder(tiny=True),
            "sd15": lambda: UNet2DConditionModel(UNetConfig.sd15()),
            "sd15_text": lambda: build_text_encoder()}[name]
    torch.manual_seed(0)
    keys, checksum, n_tensors, n_modules = _fingerprint(make())
    want = SD15_FINGERPRINTS[name]
    assert (keys, n_tensors, n_modules) == (want[0], want[2], want[3])
    assert abs(checksum - want[1]) <= 1e-9 * want[1]


def test_sd2_tiny_forward_shapes():
    """The tiny SD2 pair runs end to end on the CPU: cross-attention K (64) differs from the UNet width."""
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    torch.manual_seed(0)
    unet, text = UNet2DConditionModel(UNetConfig.sd2_tiny()), build_text_encoder(tiny=True, sd2=True)
    ehs = text(torch.randint(0, 1000, (2, 77)))[0]
    assert ehs.shape == (2, 77, 64)
    out = unet(torch.randn(2, 4, 8, 8), torch.tensor([3, 700]), ehs).sample
    assert out.shape == (2, 4, 8, 8) and torch.isfinite(out).all()
    with pytest.raises(ValueError):
        UNet2DConditionModel(UNetConfig(attention_head_dim=(5, 10, 20)))
