"""Export a saved diffusers pipeline directory as one CompVis / A1111 `.ckpt` file.

Mirrors `lora_diffusion/to_ckpt_v2.py:91-232` of the reference: the same
key names come out for the SD1.x topology (4 levels, 2 down / 3 up resnets per level), but the
renaming is done by parsing each key into (block, index, rest) rather than by a table of string
replacements. Keys that are not part of that topology pass through unchanged, as they do there.

  model.diffusion_model.*          <- unet/diffusion_pytorch_model.{bin,safetensors}
  first_stage_model.*              <- vae/diffusion_pytorch_model.{bin,safetensors}
  cond_stage_model.transformer.*   <- text_encoder/{pytorch_model.bin,model.safetensors}
"""
import os.path as osp
import re

import torch

# ------------------------------------------------------------------------------------------ UNet
_UNET_TOP = {
    "time_embedding.linear_1": "time_embed.0",
    "time_embedding.linear_2": "time_embed.2",
    "conv_in": "input_blocks.0.0",
    "conv_norm_out": "out.0",
    "conv_out": "out.2",
}
_RESNET_PART = {
    "norm1": "in_layers.0", "conv1": "in_layers.2", "norm2": "out_layers.0", "conv2": "out_layers.3",
    "time_emb_proj": "emb_layers.1", "conv_shortcut": "skip_connection",
}
_RESNET_RE = re.compile("|".join(sorted(_RESNET_PART, key=len, reverse=True)))
_BLOCK = re.compile(r"^(down_blocks|up_blocks)\.(\d+)\.(resnets|attentions)\.(\d+)\.(.*)$")
_DOWNSAMPLE = re.compile(r"^down_blocks\.(\d+)\.downsamplers\.0\.conv\.(.*)$")
_UPSAMPLE = re.compile(r"^up_blocks\.(\d+)\.upsamplers\.0\.(.*)$")
_MID = re.compile(r"^mid_block\.(resnets|attentions)\.(\d+)\.(.*)$")
N_LEVELS = 4


def _resnet_inner(rest: str) -> str:
    return _RESNET_RE.sub(lambda m: _RESNET_PART[m.group(0)], rest)


def _unet_key(k: str) -> str:
    stem, _, leaf = k.rpartition(".")
    if stem in _UNET_TOP and leaf in ("weight", "bias"):
        return f"{_UNET_TOP[stem]}.{leaf}"
    m = _BLOCK.match(k)
    if m:
        side, i, kind, j, rest = m.group(1), int(m.group(2)), m.group(3), int(m.group(4)), m.group(5)
        is_res = kind == "resnets"
        if is_res:
            rest = _resnet_inner(rest)
        if i < N_LEVELS:
            if side == "down_blocks" and j < 2 and (is_res or i < N_LEVELS - 1):
                return f"input_blocks.{3 * i + j + 1}.{0 if is_res else 1}.{rest}"
            if side == "up_blocks" and j < 3 and (is_res or i > 0):
                return f"output_blocks.{3 * i + j}.{0 if is_res else 1}.{rest}"
        return f"{side}.{i}.{kind}.{j}.{rest}"
    m = _DOWNSAMPLE.match(k)
    if m and int(m.group(1)) < N_LEVELS - 1:
        return f"input_blocks.{3 * (int(m.group(1)) + 1)}.0.op.{m.group(2)}"
    m = _UPSAMPLE.match(k)
    if m and int(m.group(1)) < N_LEVELS - 1:
        i = int(m.group(1))
        return f"output_blocks.{3 * i + 2}.{1 if i == 0 else 2}.{m.group(2)}"
    m = _MID.match(k)
    if m:
        kind, j, rest = m.group(1), int(m.group(2)), m.group(3)
        if kind == "attentions" and j == 0:
            return f"middle_block.1.{rest}"
        if kind == "resnets":
            rest = _resnet_inner(rest)
            return f"middle_block.{2 * j}.{rest}" if j < 2 else f"mid_block.resnets.{j}.{rest}"
    return k


def convert_unet_state_dict(unet_state_dict):
    """diffusers UNet2DConditionModel keys -> `openaimodel.UNetModel` keys (to_ckpt_v2.py:91-109)."""
    return {_unet_key(k): v for k, v in unet_state_dict.items()}


# ------------------------------------------------------------------------------------------- VAE
_VAE_ATTN_LEAF = {"group_norm": "norm", "query": "q", "key": "k", "value": "v", "proj_attn": "proj_out"}
_VAE_RES = re.compile(r"^(encoder|decoder)\.(down_blocks|up_blocks)\.(\d+)\.resnets\.(\d+)\.(.*)$")
_VAE_SAMPLER = re.compile(r"^(.*?)(down_blocks|up_blocks)\.(\d+)\.(downsamplers|upsamplers)\.0\.(.*)$")
_VAE_MID_RES = re.compile(r"^(.*?)mid_block\.resnets\.(\d+)\.(.*)$")
_VAE_MID_ATTN = re.compile(r"^(.*?)mid_block\.attentions\.0\.(.*)$")
_CONV_LIKE = ("q", "k", "v", "proj_out")


def _vae_key(k: str) -> str:
    k = k.replace("conv_shortcut", "nin_shortcut").replace("conv_norm_out", "norm_out")
    m = _VAE_RES.match(k)
    if m:
        coder, side, i, j, rest = m.group(1), m.group(2), int(m.group(3)), int(m.group(4)), m.group(5)
        if coder == "encoder" and side == "down_blocks" and i < N_LEVELS and j < 2:
            return f"encoder.down.{i}.block.{j}.{rest}"
        if coder == "decoder" and side == "up_blocks" and i < N_LEVELS and j < 3:
            return f"decoder.up.{N_LEVELS - 1 - i}.block.{j}.{rest}"     # SD numbers the decoder bottom-up
        return k
    m = _VAE_SAMPLER.match(k)
    if m:
        head, side, i, kind, rest = m.group(1), m.group(2), int(m.group(3)), m.group(4), m.group(5)
        if i < N_LEVELS - 1:
            if side == "down_blocks" and kind == "downsamplers":
                return f"{head}down.{i}.downsample.{rest}"
            if side == "up_blocks" and kind == "upsamplers":
                return f"{head}up.{N_LEVELS - 1 - i}.upsample.{rest}"
        return k
    m = _VAE_MID_RES.match(k)
    if m and int(m.group(2)) < 2:
        return f"{m.group(1)}mid.block_{int(m.group(2)) + 1}.{m.group(3)}"
    m = _VAE_MID_ATTN.match(k)
    if m:
        parts = m.group(2).split(".")
        parts = [_VAE_ATTN_LEAF.get(p, p) for p in parts[:-1]] + parts[-1:]
        return f"{m.group(1)}mid.attn_1." + ".".join(parts)
    return k


def reshape_weight_for_sd(w):
    """A Linear [out, in] weight as the 1x1 Conv2d weight [out, in, 1, 1] the CompVis VAE holds."""
    return w.reshape(*w.shape, 1, 1)


def convert_vae_state_dict(vae_state_dict):
    """diffusers AutoencoderKL keys -> CompVis `AutoencoderKL` keys; the mid-block attention
    projections become 1x1 convolutions (to_ckpt_v2.py:167-187)."""
    out = {}
    for k, v in vae_state_dict.items():
        nk = _vae_key(k)
        if any(f"mid.attn_1.{n}.weight" in nk for n in _CONV_LIKE):
            print(f"Reshaping {nk} for SD format")
            v = reshape_weight_for_sd(v)
        out[nk] = v
    return out


def convert_text_enc_state_dict(text_enc_dict):
    return text_enc_dict


# ----------------------------------------------------------------------------------------- files
def _load_weights(folder, names):
    for n in names:
        p = osp.join(folder, n)
        if osp.exists(p):
            if p.endswith(".safetensors"):
                from safetensors.torch import load_file
                return load_file(p, device="cpu")
            return torch.load(p, map_location="cpu")
    raise FileNotFoundError(f"none of {names} under {folder}")


def convert_to_ckpt(model_path, checkpoint_path, as_half):
    assert model_path is not None, "Must provide a model path!"
    assert checkpoint_path is not None, "Must provide a checkpoint path!"
    unet = _load_weights(osp.join(model_path, "unet"),
                         ["diffusion_pytorch_model.bin", "diffusion_pytorch_model.safetensors"])
    vae = _load_weights(osp.join(model_path, "vae"),
                        ["diffusion_pytorch_model.bin", "diffusion_pytorch_model.safetensors"])
    text = _load_weights(osp.join(model_path, "text_encoder"), ["pytorch_model.bin", "model.safetensors"])
    sd = {"model.diffusion_model." + k: v for k, v in convert_unet_state_dict(unet).items()}
    sd.update({"first_stage_model." + k: v for k, v in convert_vae_state_dict(vae).items()})
    sd.update({"cond_stage_model.transformer." + k: v for k, v in convert_text_enc_state_dict(text).items()})
    if as_half:
        sd = {k: v.half() for k, v in sd.items()}
    torch.save({"state_dict": sd}, checkpoint_path)
