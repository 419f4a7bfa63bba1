"""Pack `.pt` LoRA pair lists and textual-inversion `.pt` dicts into ONE `.safetensors` file
(behaviour of the reference's `cli_pt_to_safetensors.convert`, :19-77).

File kinds are told apart by what unpickles: a dict is a {token: embedding} table, anything else
is the flat list [up_0, down_0, up_1, down_1, ...] that `save_lora_weight` writes. The model a
list belongs to is read off the file name -- `<stem>.<model>.pt`, plain `<stem>.pt` meaning the
UNet. Keyword arguments of the form `"<model>.rank"` / `"<model>.target_modules"` override the
defaults (rank 4, the model's default target set).
"""
import os
from typing import Dict, Tuple

import torch

from . import inject as _inject
from .persist import convert_loras_to_safeloras_with_embeds


def model_name_of(path: str) -> str:
    pieces = os.path.basename(path).split(".")
    return "unet" if len(pieces) <= 2 else pieces[-2]


def _defaults_for(model: str) -> Dict[str, object]:
    targets = {"unet": _inject.UNET_DEFAULT_TARGET_REPLACE,
               "text_encoder": _inject.TEXT_ENCODER_DEFAULT_TARGET_REPLACE}.get(model, _inject.DEFAULT_TARGET_REPLACE)
    return {"target_modules": targets, "rank": 4}


def _overrides_for(model: str, settings: Dict[str, object]) -> Dict[str, object]:
    lead = model + "."
    return {key[len(lead):]: value for key, value in settings.items() if key.startswith(lead)}


def convert(*paths, outpath, overwrite=False, **settings):
    if not overwrite and os.path.exists(outpath):
        raise ValueError(f"Output path {outpath} already exists, and overwrite is not True")
    embeds: Dict[str, torch.Tensor] = {}
    modelmap: Dict[str, Tuple[str, object, int]] = {}
    for path in paths:
        payload = torch.load(path)
        if isinstance(payload, dict):
            print(f"Loading textual inversion embeds {payload.keys()} from {path}")
            embeds.update(payload)
        else:
            model = model_name_of(path)
            opts = {**_defaults_for(model), **_overrides_for(model, settings)}
            print(f"Loading Lora for {model} from {path} with settings {opts}")
            modelmap[model] = (path, opts["target_modules"], opts["rank"])
    convert_loras_to_safeloras_with_embeds(modelmap, embeds, outpath)
