"""On the GPU: the PTI step variants either side of the UNet call --
masked loss (cli_lora_pti.py:340-368), t_mutliplier (:298-304), the inpainting input
(:279-313, 9-channel UNet) -- through lora_b200.train.LoraTrainStep (fused LoRA kernels, arena
optimizer) against the oracle step (oracle/ref_step.py, itself pinned to the reference's
`loss_step` by tests/golden/pti_loss_step.pt)."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _models(in_channels, seed=0):
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    torch.manual_seed(seed)
    cfg = UNetConfig.tiny()
    cfg.in_channels = in_channels
    unet = UNet2DConditionModel(cfg).to(DEV)
    text = build_text_encoder(tiny=True).to(DEV)
    unet.requires_grad_(False)
    text.requires_grad_(False)
    return unet, text


@pytest.mark.parametrize("inpaint,masked,temperature", [(False, True, 1.0), (True, False, 1.0), (True, True, 2.0)])
def test_pti_step_variants_match_oracle_step(inpaint, masked, temperature):
    import lora_b200 as L
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.train import LoraTrainStep, StepConfig
    from oracle.ref_modules import ref_inject
    from oracle.ref_step import RefDreamboothStep

    unet, text = _models(9 if inpaint else 4)
    unet_r, text_r = copy.deepcopy(unet), copy.deepcopy(text)
    L.inject_trainable_lora(unet, r=4)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=4)
    us = ref_inject(unet_r, {"CrossAttention", "Attention", "GEGLU"}, r=4)
    ts = ref_inject(text_r, {"CLIPAttention"}, r=4)
    ours = [m for m in list(unet.modules()) + list(text.modules()) if type(m).__name__ == "LoraInjectedLinear"]
    assert len(ours) == len(us) + len(ts)
    g = torch.Generator(device=DEV).manual_seed(3)
    for o, r in zip(ours, us + ts):
        o.lora_up.weight.data.normal_(0, 0.05, generator=g)
        r.up.data.copy_(o.lora_up.weight.data)
        r.down.data.copy_(o.lora_down.weight.data)

    shape = (2, 4, 16, 16)
    cfg = StepConfig(use_cuda_graph=False, autocast_dtype=torch.bfloat16, t_multiplier=0.8,
                     use_mask=masked, mask_temperature=temperature, train_inpainting=inpaint)
    tr = LoraTrainStep(unet, text, cfg, latent_shape=shape, seq_len=77, device=DEV)
    ref = RefDreamboothStep(unet_r, text_r, DDPMNoiser(device=DEV), us, ts, autocast_dtype=torch.bfloat16,
                            t_multiplier=0.8)
    gi = torch.Generator(device=DEV).manual_seed(8)
    lat = torch.randn(shape, device=DEV, generator=gi) * 0.18215
    ids = torch.randint(0, 1000, (2, 77), device=DEV, generator=gi)
    tr.latents.copy_(lat)
    tr.input_ids.copy_(ids)
    kw = {}
    if masked:
        img_mask = (torch.rand(2, 1, 128, 128, device=DEV, generator=gi) > 0.4).float()
        tr.set_loss_mask(img_mask)
        kw.update(loss_mask=img_mask, mask_temperature=temperature)
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
