"""SDXL on the CPU: the LoRA site census of the SDXL UNet and both text encoders, the site order of
each preset, diffusers' state_dict names, the text_time embedding against a float64 restatement, the
SDXL step's conditioning (LoraXLTrainStep._fwd_bwd on CPU host models) against oracle/ref_step_xl.py,
the step's refusals, and the LoRA file round trip with three models.

The full-size models are built on the meta device: the census needs their structure, not weights."""
import copy
import json
import math
import struct
import warnings

import pytest
import torch
import torch.nn as nn

import lora_b200 as L
from lora_b200.host.clip import build_sdxl_text_encoders, build_text_encoder
from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig


def _site_names(model):
    return [n for n, m in model.named_modules() if type(m).__name__ == "LoraInjectedLinear"]


@pytest.fixture(scope="module")
def sdxl_meta():
    torch.manual_seed(0)
    with torch.device("meta"):
        unet = UNet2DConditionModel(UNetConfig.sdxl())
        te1, te2 = build_sdxl_text_encoders()
    L.inject_trainable_lora(unet, r=4)
    L.inject_trainable_lora(te1, target_replace_module=L.TEXT_ENCODER_DEFAULT_TARGET_REPLACE, r=4)
    L.inject_trainable_lora(te2, target_replace_module=L.TEXT_ENCODER_DEFAULT_TARGET_REPLACE, r=4)
    return unet, te1, te2


def test_sdxl_site_census(sdxl_meta):
    """630 default UNet sites (70 BasicTransformerBlocks x 9), 48 + 128 text sites; the 140
    cross-attention to_k / to_v read the 2048-wide context, no other site does."""
    unet, te1, te2 = sdxl_meta
    us = [(n, m) for n, m in unet.named_modules() if type(m).__name__ == "LoraInjectedLinear"]
    t1 = [m for m in te1.modules() if type(m).__name__ == "LoraInjectedLinear"]
    t2 = [m for m in te2.modules() if type(m).__name__ == "LoraInjectedLinear"]
    assert len(us) == 630 and len(t1) == 48 and len(t2) == 128 and len(t1) + len(t2) == 176
    assert sum(type(m).__name__ == "BasicTransformerBlock" for m in unet.modules()) == 70
    kv = [(n, m) for n, m in us if ".attn2.to_k" in n or ".attn2.to_v" in n]
    assert len(kv) == 140 and all(m.linear.in_features == 2048 for _, m in kv)
    assert all(m.linear.in_features != 2048 for n, m in us if ".attn2.to_k" not in n and ".attn2.to_v" not in n)
    assert all((m.linear.in_features, m.linear.out_features) == (768, 768) for m in t1)
    assert all((m.linear.in_features, m.linear.out_features) == (1280, 1280) for m in t2)
    # stacks: down 1 x 2 x 2, down 2 x 2 x 10, up 0 x 3 x 10, up 1 x 3 x 2, mid 10
    depth = {n: len(m.transformer_blocks) for n, m in unet.named_modules() if type(m).__name__ == "Transformer2DModel"}
    assert sorted(set(depth.values())) == [2, 10]
    assert depth["mid_block.attentions.0"] == 10 and depth["up_blocks.0.attentions.2"] == 10
    assert depth["down_blocks.1.attentions.1"] == 2 and depth["up_blocks.1.attentions.0"] == 2
    assert not hasattr(unet.down_blocks[0], "attentions") and not hasattr(unet.up_blocks[2], "attentions")
    # head dim 64 everywhere
    assert all(m.to_q.linear.out_features // m.heads == 64 for m in unet.modules() if type(m).__name__ == "CrossAttention")


def _block_orders(names):
    """Per BasicTransformerBlock, the order its sites are registered in."""
    out = {}
    for n in names:
        blk, rest = n.split(".transformer_blocks.")
        idx, sub = rest.split(".", 1)
        out.setdefault(f"{blk}.{idx}", []).append(sub)
    return set(tuple(v) for v in out.values())


ATTN1 = ("attn1.to_q", "attn1.to_k", "attn1.to_v", "attn1.to_out.0")
ATTN2 = ("attn2.to_q", "attn2.to_k", "attn2.to_v", "attn2.to_out.0")
FF = ("ff.net.0.proj",)


def test_site_order_per_preset(sdxl_meta):
    """SDXL registers attn1 -> attn2 -> ff (diffusers >= 0.19); SD1.5 and SD2 keep attn1 -> ff -> attn2."""
    assert _block_orders(_site_names(sdxl_meta[0])) == {ATTN1 + ATTN2 + FF}
    for cfg in (UNetConfig.tiny(), UNetConfig.sd2_tiny(), UNetConfig.sdxl_tiny()):
        torch.manual_seed(0)
        unet = UNet2DConditionModel(cfg)
        L.inject_trainable_lora(unet, r=2)
        want = ATTN1 + ATTN2 + FF if cfg.transformer_block_order == "attn1_attn2_ff" else ATTN1 + FF + ATTN2
        assert _block_orders(_site_names(unet)) == {want}
    with torch.device("meta"):
        for cfg in (UNetConfig.sd15(), UNetConfig.sd21()):
            unet = UNet2DConditionModel(cfg)
            L.inject_trainable_lora(unet, r=4)
            names = _site_names(unet)
            assert len(names) == 144 and _block_orders(names) == {ATTN1 + FF + ATTN2}
    with pytest.raises(ValueError, match="transformer_block_order"):
        UNet2DConditionModel(UNetConfig(transformer_block_order="ff_first"))
    with pytest.raises(ValueError, match="transformer_layers_per_block"):
        UNet2DConditionModel(UNetConfig(transformer_layers_per_block=(1, 2)))
    with pytest.raises(ValueError, match="addition_embed_type"):
        UNet2DConditionModel(UNetConfig(addition_embed_type="text"))


def test_sdxl_state_dict_uses_diffusers_names():
    with torch.device("meta"):
        unet = UNet2DConditionModel(UNetConfig.sdxl())
        te1, te2 = build_sdxl_text_encoders()
    sd = {k: tuple(v.shape) for k, v in unet.state_dict().items()}
    want = {
        "add_embedding.linear_1.weight": (1280, 2816), "add_embedding.linear_1.bias": (1280,),
        "add_embedding.linear_2.weight": (1280, 1280),
        "time_embedding.linear_1.weight": (1280, 320),
        "down_blocks.1.attentions.1.transformer_blocks.1.attn2.to_k.weight": (640, 2048),
        "down_blocks.2.attentions.0.transformer_blocks.9.ff.net.0.proj.weight": (10240, 1280),
        "down_blocks.2.attentions.0.proj_in.weight": (1280, 1280),
        "mid_block.attentions.0.transformer_blocks.9.attn2.to_v.weight": (1280, 2048),
        "up_blocks.0.attentions.2.transformer_blocks.9.norm3.weight": (1280,),
        "up_blocks.1.resnets.2.conv_shortcut.weight": (640, 960, 1, 1),
        "up_blocks.2.resnets.0.conv1.weight": (320, 960, 3, 3),
        "conv_in.weight": (320, 4, 3, 3), "conv_out.weight": (4, 320, 3, 3),
    }
    for k, shape in want.items():
        assert sd.get(k) == shape, (k, sd.get(k))
    assert not any(k.startswith("down_blocks.0.attentions") or k.startswith("up_blocks.2.attentions") for k in sd)
    assert not any("add_time_proj" in k for k in sd)              # sinusoidal, no parameters
    # the parameter count of diffusers' stable-diffusion-xl-base-1.0 UNet
    assert sum(v.numel() for v in unet.state_dict().values()) == 2_567_463_684
    # encoder 2: transformers' CLIPTextModelWithProjection names
    sd2 = {k: tuple(v.shape) for k, v in te2.state_dict().items()}
    assert sd2["text_projection.weight"] == (1280, 1280)
    assert sd2["text_model.encoder.layers.31.self_attn.q_proj.weight"] == (1280, 1280)
    assert sd2["text_model.encoder.layers.31.mlp.fc1.weight"] == (5120, 1280)
    assert "text_model.encoder.layers.32.self_attn.q_proj.weight" not in sd2
    assert te1.config.hidden_size == 768 and te1.config.num_hidden_layers == 12


def _text_time_float64(unet, text_embeds, time_ids):
    """diffusers' text_time branch, restated in float64 from the formulas."""
    dim = unet.cfg.addition_time_embed_dim
    half = dim // 2
    k = torch.arange(half, dtype=torch.float64)
    freqs = torch.exp(-math.log(10000.0) * k / half)
    arg = time_ids.double().reshape(-1)[:, None] * freqs[None, :]
    proj = torch.cat([torch.cos(arg), torch.sin(arg)], dim=-1).reshape(text_embeds.shape[0], 6 * dim)
    x = torch.cat([text_embeds.double(), proj], dim=-1)
    e = unet.add_embedding
    h = x @ e.linear_1.weight.double().T + e.linear_1.bias.double()
    h = h * torch.sigmoid(h)
    return h @ e.linear_2.weight.double().T + e.linear_2.bias.double()


def test_text_time_embedding_matches_float64_restatement():
    torch.manual_seed(0)
    unet = UNet2DConditionModel(UNetConfig.sdxl_tiny())
    g = torch.Generator().manual_seed(1)
    te = torch.randn(3, 40, generator=g)
    tid = torch.tensor([[1024.0, 1024, 0, 0, 1024, 1024], [768, 1344, 64, 32, 768, 1344], [512, 512, 0, 0, 1024, 1024]])
    got = unet.text_time_embedding({"text_embeds": te, "time_ids": tid}, torch.float32)
    want = _text_time_float64(unet, te, tid)
    # the sinusoid is evaluated in fp32 (diffusers' get_timestep_embedding): arguments up to 1344 rad
    assert float((got.double() - want).norm() / want.norm()) < 1e-5
    # the branch is added to the timestep embedding: a different time_ids changes the prediction
    x, t = torch.randn(3, 4, 8, 8, generator=g), torch.tensor([1, 500, 999])
    ehs = torch.randn(3, 77, 88, generator=g)
    a = unet(x, t, ehs, added_cond_kwargs={"text_embeds": te, "time_ids": tid}).sample
    b = unet(x, t, ehs, added_cond_kwargs={"text_embeds": te, "time_ids": tid + 8}).sample
    assert a.shape == x.shape and not torch.equal(a, b)
    with pytest.raises(ValueError, match="added_cond_kwargs"):
        unet(x, t, ehs)
    # an SD UNet keeps its three-argument call
    sd = UNet2DConditionModel(UNetConfig.tiny())
    assert sd(x, t, torch.randn(3, 77, 48)).sample.shape == x.shape


def _eos_ids(batch, gen, eos=999, lengths=(9, 23)):
    """Prompts of random tokens followed by eos up to 77, as the CLIP tokenizers pad them."""
    ids = torch.randint(0, 998, (batch, 77), generator=gen)
    for b in range(batch):
        ids[b, lengths[b % len(lengths)]:] = eos
    return ids


def _xl_cpu_step(variant):
    """A LoraXLTrainStep assembled by hand around float64 CPU host models with the oracle's eager LoRA
    sites in place of the product's (no arena, no CUDA buffers)."""
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.train import LoraXLTrainStep, StepConfig
    from oracle.ref_modules import ref_inject
    torch.manual_seed(0)
    unet = UNet2DConditionModel(UNetConfig.sdxl_tiny()).double()
    te1, te2 = (m.double() for m in build_sdxl_text_encoders(tiny=True))
    us = ref_inject(unet, {"CrossAttention", "Attention", "GEGLU"}, r=4)
    ts1 = ref_inject(te1, {"CLIPAttention"}, r=4)
    ts2 = ref_inject(te2, {"CLIPAttention"}, r=4)
    g = torch.Generator().manual_seed(1)
    for s in us + ts1 + ts2:
        s.up.data.normal_(0, 0.05, generator=g)
    shape = (2, 4, 8, 8)
    tr = object.__new__(LoraXLTrainStep)
    tr.cfg = StepConfig(use_cuda_graph=False, t_multiplier=0.8, with_prior_preservation=variant == "prior",
                        prior_loss_weight=0.7)
    tr.unet, tr.text_encoder, tr.text_encoder_2, tr.device = unet, te1, te2, torch.device("cpu")
    tr.noiser, tr.model_dtype = DDPMNoiser(device="cpu"), torch.float64
    tr.latents = torch.randn(shape, generator=g) * 0.13025
    tr.input_ids, tr.input_ids_2 = _eos_ids(2, g), _eos_ids(2, g)
    tr.time_ids = torch.tensor([[64.0, 64, 0, 0, 64, 64], [96, 48, 8, 0, 64, 64]])
    tr.loss = torch.zeros(())
    tr.mask = torch.ones(2, 1, 8, 8)
    return tr, us, ts1, ts2


@pytest.mark.parametrize("variant", ["plain", "prior"])
def test_xl_step_body_matches_oracle_on_cpu_doubles(variant):
    """LoraXLTrainStep._fwd_bwd (the unfused body) against RefXLStep for the same seed: loss and every
    factor gradient of the UNet and both encoders."""
    from lora_b200.host.ddpm import DDPMNoiser
    from oracle.ref_step_xl import RefXLStep
    tr, us, ts1, ts2 = _xl_cpu_step(variant)
    ref = RefXLStep(tr.unet, tr.text_encoder, tr.text_encoder_2, DDPMNoiser(device="cpu"), us, ts1, ts2,
                    t_multiplier=0.8)
    assert len(ref.text_params) == 2 * (len(ts1) + len(ts2))
    kw = {"prior_loss_weight": 0.7} if variant == "prior" else {}
    torch.manual_seed(77)
    noise = torch.randn(tr.latents.shape)
    t = torch.randint(0, 800, (2,)).long()
    want = ref.forward_loss(tr.latents, tr.input_ids, noise, t, input_ids_2=tr.input_ids_2, time_ids=tr.time_ids, **kw)
    want.backward()
    # hidden_states[-2]: encoder 1's last layer (its 4 sites) gets no gradient, every other factor does
    dead = {id(p) for s in ts1[-4:] for p in (s.up, s.down)}
    assert all((p.grad is None) == (id(p) in dead) for p in ref.unet_params + ref.text_params)
    live = [p for p in ref.unet_params + ref.text_params if id(p) not in dead]
    g_ref = torch.cat([p.grad.flatten() for p in live]).clone()
    ref.opt.zero_grad()
    assert ref.text_encoder is tr.text_encoder and ref.unet is tr.unet        # the stand-ins are gone
    torch.manual_seed(77)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")             # torch.autocast("cuda", enabled=False) on a CPU-only box
        tr._fwd_bwd()
    assert all(p.grad is None for s in ts1[-4:] for p in (s.up, s.down))
    g_ours = torch.cat([p.grad.flatten() for p in live])
    # float64 models, fp32 loss (pred.float()): the loss agrees to a few fp32 ulps
    assert abs(float(tr.loss) - float(want)) <= 1e-6 * abs(float(want))
    assert float((g_ours - g_ref).norm() / g_ref.norm()) < 1e-6
    assert all(float(s.up.grad.abs().sum()) > 0 for s in ts2)                # encoder 2 is trained
    # the conditioning matters: other time ids give another loss
    ref.opt.zero_grad()
    other = ref.forward_loss(tr.latents, tr.input_ids, noise, t, input_ids_2=tr.input_ids_2,
                             time_ids=tr.time_ids * 2, **kw)
    assert abs(float(other) - float(want)) > 1e-6 * abs(float(want))


def _tiny_xl():
    torch.manual_seed(0)
    unet = UNet2DConditionModel(UNetConfig.sdxl_tiny())
    te1, te2 = build_sdxl_text_encoders(tiny=True)
    return unet, te1, te2


def test_xl_step_refuses_mismatched_models_before_cuda():
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    from lora_b200.train import LoraXLTrainStep, StepConfig
    unet, te1, te2 = _tiny_xl()
    cfg = StepConfig()
    with pytest.raises(ValueError, match="SDXL UNet"):
        LoraXLTrainStep(UNet2DConditionModel(UNetConfig.tiny()), te1, te2, cfg, device="cpu")
    with pytest.raises(ValueError, match="CLIPTextModelWithProjection"):
        LoraXLTrainStep(unet, te1, build_text_encoder(tiny=True), cfg, device="cpu")
    with pytest.raises(ValueError, match="cross_attention_dim"):
        LoraXLTrainStep(unet, build_text_encoder(tiny=True, sd2=True), te2, cfg, device="cpu")
    wrong = CLIPTextModelWithProjection(CLIPTextConfig(vocab_size=1000, hidden_size=40, intermediate_size=80,
                                                       num_hidden_layers=1, num_attention_heads=2,
                                                       max_position_embeddings=77, projection_dim=32))
    with pytest.raises(ValueError, match="projection_class_embeddings_input_dim"):
        LoraXLTrainStep(unet, te1, wrong, cfg, device="cpu")
    with pytest.raises(ValueError, match="needs the frozen VAE"):
        LoraXLTrainStep(unet, te1, te2, StepConfig(encode_images=True), device="cpu")


def test_xl_step_host_refuses_wrong_shapes():
    from lora_b200.train import LoraXLTrainStep, StepConfig
    tr = object.__new__(LoraXLTrainStep)
    tr.cfg = StepConfig()
    tr.input_ids_2 = torch.zeros(2, 77, dtype=torch.long)
    tr.time_ids = torch.zeros(2, 6)
    lat, ids = torch.zeros(2, 4, 8, 8), torch.zeros(2, 77, dtype=torch.long)
    with pytest.raises(ValueError, match="input_ids_2 of shape"):
        tr.step_host(lat, ids, torch.zeros(1, 77, dtype=torch.long))
    with pytest.raises(ValueError, match="input_ids_2 of shape"):
        tr.step_host(lat, ids, torch.zeros(2, 76, dtype=torch.long))
    with pytest.raises(ValueError, match="integer token ids"):
        tr.step_host(lat, ids, torch.zeros(2, 77))
    with pytest.raises(ValueError, match="time_ids of shape"):
        tr.step_host(lat, ids, ids, time_ids=torch.zeros(2, 5))
    with pytest.raises(ValueError, match="time_ids of shape"):
        tr.step_host(lat, ids, ids, time_ids=torch.zeros(12))
    with pytest.raises(ValueError, match="time_ids of shape"):
        tr.step_host(lat, ids, ids, time_ids=torch.zeros(1, 6))


def _load(path):
    """(parsed header, tensor bytes) of a safetensors file."""
    raw = open(path, "rb").read()
    n = struct.unpack("<Q", raw[:8])[0]
    return json.loads(raw[8:8 + n]), raw[8 + n:]


def test_sdxl_safeloras_round_trip_equals_reference_layout(tmp_path):
    """save_safeloras with unet, text_encoder and text_encoder_2 writes the file the reference's
    save_safeloras writes from the same factors (oracle/ref_step_xl.py::save_ref_safeloras): the same
    tensors, offsets, bytes and metadata. safetensors serialises the metadata from a hash map whose
    order changes from one write to the next, so the header is compared parsed and the tensor section
    byte for byte. monkeypatch_or_replace_safeloras and patch_pipe load it into a pipeline-like object
    with the three attributes, which then saves the same file again."""
    from oracle.ref_modules import ref_inject
    from oracle.ref_step_xl import save_ref_safeloras
    unet, te1, te2 = _tiny_xl()
    refs = [copy.deepcopy(m) for m in (unet, te1, te2)]
    ut, tt = L.UNET_DEFAULT_TARGET_REPLACE, L.TEXT_ENCODER_DEFAULT_TARGET_REPLACE
    L.inject_trainable_lora(unet, r=4)
    L.inject_trainable_lora(te1, target_replace_module=tt, r=4)
    L.inject_trainable_lora(te2, target_replace_module=tt, r=4)
    rsites = [ref_inject(refs[0], set(ut), r=4), ref_inject(refs[1], set(tt), r=4), ref_inject(refs[2], set(tt), r=4)]
    g = torch.Generator().manual_seed(5)
    for model, rs in zip((unet, te1, te2), rsites):
        ours = [m for m in model.modules() if type(m).__name__ == "LoraInjectedLinear"]
        assert len(ours) == len(rs)
        for o, r in zip(ours, rs):
            o.lora_up.weight.data.normal_(0, 0.1, generator=g)
            r.up.data.copy_(o.lora_up.weight.data)
            r.down.data.copy_(o.lora_down.weight.data)
    L.tune_lora_scale(unet, 0.5)
    rsites[0] = [setattr(s, "scale", 0.5) or s for s in rsites[0]]
    ours_path, ref_path = str(tmp_path / "ours.safetensors"), str(tmp_path / "ref.safetensors")
    L.save_safeloras({"unet": (unet, ut), "text_encoder": (te1, tt), "text_encoder_2": (te2, tt)}, ours_path)
    save_ref_safeloras({"unet": (rsites[0], ut), "text_encoder": (rsites[1], tt), "text_encoder_2": (rsites[2], tt)},
                       ref_path)
    h_ours, b_ours = _load(ours_path)
    h_ref, b_ref = _load(ref_path)
    assert h_ours == h_ref and b_ours == b_ref
    meta = h_ours["__metadata__"]
    assert {k.split(":")[0] for k in h_ours if k != "__metadata__"} == {"unet", "text_encoder", "text_encoder_2"}
    n_u, n_1, n_2 = (sum(1 for k in h_ours if k.startswith(p + ":") and k.endswith(":up"))
                     for p in ("unet", "text_encoder", "text_encoder_2"))
    assert (n_u, n_1, n_2) == (len(rsites[0]), len(rsites[1]), len(rsites[2]))
    assert set(json.loads(meta["text_encoder_2"])) == set(tt)

    class Pipe:
        pass

    from safetensors import safe_open
    for how in ("monkeypatch", "patch_pipe"):
        pipe = Pipe()
        pipe.unet, pipe.text_encoder, pipe.text_encoder_2 = _tiny_xl()
        if how == "monkeypatch":
            L.monkeypatch_or_replace_safeloras(pipe, safe_open(ref_path, framework="pt", device="cpu"))
        else:
            L.patch_pipe(pipe, ref_path, patch_ti=False)
        again = str(tmp_path / f"{how}.safetensors")
        L.save_safeloras({"unet": (pipe.unet, ut), "text_encoder": (pipe.text_encoder, tt),
                          "text_encoder_2": (pipe.text_encoder_2, tt)}, again)
        h, b = _load(again)
        assert b == b_ref, how
        assert {k: v for k, v in h.items() if k != "__metadata__"} == {k: v for k, v in h_ref.items()
                                                                         if k != "__metadata__"}
        assert h["__metadata__"] == meta
