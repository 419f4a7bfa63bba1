"""`lora_add`: arithmetic on LoRA files and merging a LoRA into a pipeline's frozen weights.

Mirrors `lora_diffusion/cli_lora_add.py:24-183` of the reference, modes
  lpl          LoRA (+) LoRA: alpha_1 * factors_1 + alpha_2 * factors_2, `.pt` pair lists or safetensors
  ljl          join: rank-concatenate two safetensors LoRAs (`join.lora_join`)
  upl          pipeline (+) LoRA: W += alpha_1 * B·A on every site, LoRA removed, pipeline saved
  upl-ckpt-v2  the same, then exported as a CompVis `.ckpt` + an A1111 textual-inversion `.pt`

The two `upl` modes need a pipeline loader (`diffusers.StableDiffusionPipeline.from_pretrained`
in the reference). diffusers is not a dependency of this package: pass `pipeline_loader=` (any
callable path -> object with `.unet`, `.text_encoder`, `.tokenizer`, `.save_pretrained`), or
call `merge_lora_into_pipeline` on a pipeline you already hold. On a CUDA pipeline the merge runs
`lb_lora_merge` (csrc/lora_aux.cu) per site through `collapse_lora`.
"""
import os
import shutil
from typing import Callable, Optional

import torch

from .join import lora_join
from .patch import collapse_lora, monkeypatch_remove_lora, patch_pipe
from .persist import _text_lora_path

MODES = ("lpl", "upl", "upl-ckpt-v2", "ljl")


def _blend_pt(path_1, path_2, out_path, alpha_1, alpha_2):
    """`.pt` files hold [up, down, up, down, ...]; blend tensor by tensor (cli_lora_add.py:55-66)."""
    l1, l2 = torch.load(path_1), torch.load(path_2)
    out = []
    for t1, t2 in zip(l1, l2):
        t1.data = alpha_1 * t1.data + alpha_2 * t2.data
        out.append(t1)
    if len(out) % 2:                      # the reference walks (up, down) pairs: an odd tail is dropped
        out = out[:-1]
    torch.save(out, out_path)


def _blend_safetensors(path_1, path_2, out_path, alpha_1, alpha_2):
    """cli_lora_add.py:82-108: LoRA factors are blended, anything else (embeddings) is taken from
    file 1 when it has the key, else from file 2; metadata of 2 overrides 1."""
    from safetensors.torch import safe_open, save_file
    f1 = safe_open(path_1, framework="pt", device="cpu")
    f2 = safe_open(path_2, framework="pt", device="cpu")
    metadata = dict(f1.metadata())
    metadata.update(dict(f2.metadata()))
    k1 = set(f1.keys())
    out = {}
    for key in k1 | set(f2.keys()):
        if key.startswith("text_encoder") or key.startswith("unet"):
            out[key] = alpha_1 * f1.get_tensor(key) + alpha_2 * f2.get_tensor(key)
        else:
            out[key] = f1.get_tensor(key) if key in k1 else f2.get_tensor(key)
    save_file(out, out_path, metadata)


def merge_lora_into_pipeline(pipe, lora_path: str, alpha: float = 1.0, patch_ti: bool = True):
    """The body of the `upl` modes (cli_lora_add.py:116-128,140-148): patch the LoRA in, fold
    `alpha * B·A` into every frozen weight, put plain Linear/Conv2d modules back.
    Returns what `patch_pipe` returned (the token -> embedding dict when `patch_ti` is False)."""
    ret = patch_pipe(pipe, lora_path, patch_ti=patch_ti)
    collapse_lora(pipe.unet, alpha)
    collapse_lora(pipe.text_encoder, alpha)
    monkeypatch_remove_lora(pipe.unet)
    monkeypatch_remove_lora(pipe.text_encoder)
    return ret


def _default_loader(path):
    try:
        from diffusers import StableDiffusionPipeline
    except ImportError as e:              # same failure the reference has at import time
        raise ImportError("mode 'upl'/'upl-ckpt-v2' loads a diffusers pipeline; diffusers is not "
                          "installed - pass pipeline_loader=") from e
    return StableDiffusionPipeline.from_pretrained(path).to("cpu")


def add(path_1: str, path_2: str, output_path: str, alpha_1: float = 0.5, alpha_2: float = 0.5,
        mode: str = "lpl", with_text_lora: bool = False,
        pipeline_loader: Optional[Callable] = None):
    print("Lora Add, mode " + mode)
    if mode == "lpl":
        if path_1.endswith(".pt") and path_2.endswith(".pt"):
            print("Saving merged UNET to", output_path)
            _blend_pt(path_1, path_2, output_path, alpha_1, alpha_2)
            if with_text_lora:
                t1, t2 = _text_lora_path(path_1), _text_lora_path(path_2)
                missing = [p for p in (t1, t2) if not os.path.exists(p)]
                if missing:
                    print(f"No text encoder found in {missing[0]}, skipping...")
                else:
                    print("Saving merged text encoder to", _text_lora_path(output_path))
                    _blend_pt(t1, t2, _text_lora_path(output_path), alpha_1, alpha_2)
        elif path_1.endswith(".safetensors") and path_2.endswith(".safetensors"):
            _blend_safetensors(path_1, path_2, output_path, alpha_1, alpha_2)
        # mixed extensions: the reference does nothing, silently (cli_lora_add.py:40,82)
    elif mode == "upl":
        print(f"Merging UNET/CLIP from {path_1} with LoRA from {path_2} to {output_path}. "
              f"Merging ratio : {alpha_1}.")
        pipe = (pipeline_loader or _default_loader)(path_1)
        merge_lora_into_pipeline(pipe, path_2, alpha_1)
        pipe.save_pretrained(output_path)
    elif mode == "upl-ckpt-v2":
        assert output_path.endswith(".ckpt"), "Only .ckpt files are supported"
        name = os.path.basename(output_path)[:-5]
        print(f"You will be using {name} as the token in A1111 webui. Make sure {name} is unique enough token.")
        from .to_ckpt import convert_to_ckpt
        pipe = (pipeline_loader or _default_loader)(path_1)
        tok_dict = merge_lora_into_pipeline(pipe, path_2, alpha_1, patch_ti=False)
        tmp = output_path + ".tmp"
        pipe.save_pretrained(tmp)
        convert_to_ckpt(tmp, output_path, as_half=True)
        shutil.rmtree(tmp)
        stacked = torch.stack([tok_dict[k] for k in sorted(tok_dict.keys())])
        torch.save({"string_to_token": {"*": torch.tensor(265)}, "string_to_param": {"*": stacked},
                    "name": name}, output_path[:-5] + ".pt")
        print(f"Textual embedding saved as {output_path[:-5]}.pt, put it in the embedding folder "
              f"and use it as {name} in A1111 repo, ")
    elif mode == "ljl":
        print("Using Join mode : alpha will not have an effect here.")
        assert path_1.endswith(".safetensors") and path_2.endswith(".safetensors"), \
            "Only .safetensors files are supported"
        from safetensors.torch import safe_open, save_file
        tensors, metadata, _, _ = lora_join([safe_open(path_1, framework="pt", device="cpu"),
                                             safe_open(path_2, framework="pt", device="cpu")])
        save_file(tensors, output_path, metadata)
    else:
        print("Unknown mode", mode)
        raise ValueError(f"Unknown mode {mode}")
