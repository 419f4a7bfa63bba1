"""ORACLE (test infrastructure only): the LoRA training step on SDXL, in plain PyTorch eager.

The reference has no SDXL trainer, so no golden from the reference pins the SDXL conditioning. It is
restated from diffusers:

  examples/dreambooth/train_dreambooth_lora_sdxl.py, `encode_prompt`:
      for each text encoder: out = text_encoder(ids, output_hidden_states=True)
                             prompt_embeds = out.hidden_states[-2]
      prompt_embeds = cat(prompt_embeds of both encoders, dim=-1)
      pooled_prompt_embeds = the last encoder's out[0] (CLIPTextModelWithProjection's text_embeds)
  the same script's `compute_time_ids`: time_ids = original_size + crops_coords_top_left + target_size
  UNet2DConditionModel with addition_embed_type="text_time": the UNet's own `added_cond_kwargs`
      branch (the host model restates it: add_time_proj, concatenation, add_embedding, + temb).

Only the conditioning is overridden. Noise, noising, the loss and its options, clip_grad_norm_ and
AdamW are oracle/ref_step.py's, unchanged; the existing goldens pin them. The second encoder's LoRA
factors join the text parameter group (same lr), so one clip covers UNet + both encoders. The first
encoder's last layer feeds only hidden_states[-1], which nothing reads: its factors keep grad None, so
clip_grad_norm_ and AdamW skip them, as in the diffusers script. Imports nothing from the product
package.

`save_ref_safeloras` writes a LoRA file the way the reference's `save_safeloras` does
(lora_diffusion/lora.py:451-483: `{model}:{i}:up` = up * scale and `{model}:{i}:down` in fp16,
metadata `{model}` = json list of the target names and `{model}:{i}:rank`) from RefLoraSite lists.
"""
import json
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from .ref_step import RefDreamboothStep


class _XLText:
    """Stands in for the text encoder inside one forward_loss call: both encoders, concatenated."""

    def __init__(self, step, input_ids_2):
        self.step, self.input_ids_2 = step, input_ids_2

    def __call__(self, input_ids):
        st = self.step
        out1 = st.text_encoder_1(input_ids, output_hidden_states=True)
        out2 = st.text_encoder_2(self.input_ids_2, output_hidden_states=True)
        st._text_embeds = out2.text_embeds
        return (torch.cat([out1.hidden_states[-2], out2.hidden_states[-2]], dim=-1),)


class _XLUNet:
    """Stands in for the UNet inside one forward_loss call: adds the text_time conditioning."""

    def __init__(self, step, unet, time_ids):
        self.step, self.unet, self.time_ids = step, unet, time_ids

    def parameters(self):
        return self.unet.parameters()

    def __call__(self, sample, timesteps, encoder_hidden_states):
        added = {"text_embeds": self.step._text_embeds, "time_ids": self.time_ids}
        return self.unet(sample, timesteps, encoder_hidden_states, added_cond_kwargs=added)


def default_time_ids(batch: int, height: int, width: int, device=None) -> torch.Tensor:
    """compute_time_ids with original = target = (height, width) pixels and no crop."""
    row = [float(height), float(width), 0.0, 0.0, float(height), float(width)]
    return torch.tensor([row] * batch, dtype=torch.float32, device=device)


class RefXLStep(RefDreamboothStep):
    """RefDreamboothStep with SDXL's two text encoders and text_time conditioning.

    forward_loss / step take `input_ids_2` (the second tokenizer's ids) and `time_ids` [B, 6]; time_ids
    None means the Dreambooth default for the latents' size (8h, 8w, 0, 0, 8h, 8w)."""

    def __init__(self, unet, text_encoder, text_encoder_2, noiser, unet_sites: List,
                 text_sites: Optional[List], text_sites_2: Optional[List], **kw):
        for p in text_encoder_2.parameters():
            p.requires_grad_(False)
        super().__init__(unet, text_encoder, noiser, unet_sites, list(text_sites or []) + list(text_sites_2 or []),
                         **kw)
        self.text_encoder_1, self.text_encoder_2 = text_encoder, text_encoder_2
        self._unet = unet
        text_encoder_2.train()

    def forward_loss(self, latents, input_ids, noise, timesteps, input_ids_2=None, time_ids=None, **loss_kw):
        if input_ids_2 is None:
            raise ValueError("RefXLStep needs input_ids_2, the second text encoder's ids")
        if time_ids is None:
            time_ids = default_time_ids(latents.shape[0], 8 * latents.shape[2], 8 * latents.shape[3], latents.device)
        self.text_encoder = _XLText(self, input_ids_2)
        self.unet = _XLUNet(self, self._unet, time_ids)
        try:
            return super().forward_loss(latents, input_ids, noise, timesteps, **loss_kw)
        finally:
            self.text_encoder, self.unet = self.text_encoder_1, self._unet
            self._text_embeds = None


def save_ref_safeloras(modelmap: Dict[str, Tuple[Sequence, Sequence[str]]], outpath: str):
    """{model name: (RefLoraSite list in site order, target names)} -> one safetensors file, laid out as
    the reference's save_safeloras writes it."""
    from safetensors.torch import save_file
    weights, metadata = {}, {}
    for name, (sites, targets) in modelmap.items():
        metadata[name] = json.dumps(list(targets))
        for i, s in enumerate(sites):
            up = (s.up.detach() * s.scale).to("cpu", torch.float16)
            down = s.down.detach().to("cpu", torch.float16)
            metadata[f"{name}:{i}:rank"] = str(down.shape[0])
            weights[f"{name}:{i}:up"] = up.contiguous()
            weights[f"{name}:{i}:down"] = down.contiguous()
    save_file(weights, outpath, metadata)
