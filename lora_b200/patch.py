"""Load / replace / remove / merge LoRAs on a live model and pipeline-level helpers.

Contract restated from /root/reference/lora_diffusion/lora.py:635-1042. All functions are tree
surgery or small weight arithmetic; the numerical hot path lives in modules.py / liblora_b200.so.
"""
import weakref
from typing import List, Optional, Union

import torch
import torch.nn as nn

from .inject import (DEFAULT_TARGET_REPLACE, TEXT_ENCODER_DEFAULT_TARGET_REPLACE,
                     TEXT_ENCODER_EXTENDED_TARGET_REPLACE, UNET_EXTENDED_TARGET_REPLACE,
                     _find_modules)
from .modules import LoraInjectedConv2d, LoraInjectedLinear
from .persist import (_text_lora_path, _ti_lora_path, parse_safeloras, parse_safeloras_embeds,
                      safe_open)

_LORA_CLASS_NAMES = ["LoraInjectedLinear", "LoraInjectedConv2d"]


def collapse_lora(model, alpha=1.0):
    """Fold every LoRA into its frozen weight: W <- W + alpha * up @ down (lora.py:635-669).
    The module stays a LoRA module (its factors are left untouched), as in the reference."""
    targets = UNET_EXTENDED_TARGET_REPLACE | TEXT_ENCODER_EXTENDED_TARGET_REPLACE
    for _, name, site in _find_modules(model, targets,
                                       search_class=[LoraInjectedLinear, LoraInjectedConv2d]):
        is_lin = isinstance(site, LoraInjectedLinear)
        holder = site.linear if is_lin else site.conv
        print("Collapsing Lin Lora in" if is_lin else "Collapsing Conv Lora in", name)
        w = holder.weight.data
        if w.is_cuda and site.r <= 64 and w.dtype in (torch.float32, torch.bfloat16, torch.float16):
            from . import ops   # one HBM pass over W (lb_lora_merge) instead of GEMM + cast + add
            holder.weight = nn.Parameter(ops.merge_lora(w, site.lora_up.weight.data.to(w.device),
                                                        site.lora_down.weight.data.to(w.device), alpha))
            continue
        delta = site.lora_up.weight.data.flatten(start_dim=1) @ site.lora_down.weight.data.flatten(start_dim=1)
        holder.weight = nn.Parameter(w + alpha * delta.reshape(w.shape).type(w.dtype).to(w.device))


def _next_rank(r):
    return r.pop(0) if isinstance(r, list) else r


def _install_factors(parent, name, new, loras, like):
    parent._modules[name] = new
    up = loras.pop(0)
    down = loras.pop(0)
    site = parent._modules[name]
    site._lb.parent = weakref.ref(parent)
    site.lora_up.weight = nn.Parameter(up.type(like.dtype))
    site.lora_down.weight = nn.Parameter(down.type(like.dtype))
    site.to(like.device)


def monkeypatch_or_replace_lora(model, loras, target_replace_module=DEFAULT_TARGET_REPLACE,
                                r: Union[int, List[int]] = 4):
    """Linear-only (re)patch from a flat [up0, down0, ...] list (lora.py:672-713).
    New operator modules get the class defaults dropout_p = 0.1, scale = 1.0."""
    for parent, name, child in _find_modules(model, target_replace_module,
                                             search_class=[nn.Linear, LoraInjectedLinear]):
        src = child.linear if isinstance(child, LoraInjectedLinear) else child
        new = LoraInjectedLinear(src.in_features, src.out_features, src.bias is not None,
                                 r=_next_rank(r))
        new.linear.weight = src.weight
        if src.bias is not None:
            new.linear.bias = src.bias
        _install_factors(parent, name, new, loras, src.weight)


def monkeypatch_or_replace_lora_extended(model, loras, target_replace_module=DEFAULT_TARGET_REPLACE,
                                         r: Union[int, List[int]] = 4):
    """Linear + Conv2d (re)patch (lora.py:716-796). A site whose kind does not match the rank of
    the next factor in `loras` (2-D vs 4-D) is skipped, exactly like the reference."""
    kinds = [nn.Linear, LoraInjectedLinear, nn.Conv2d, LoraInjectedConv2d]
    for parent, name, child in _find_modules(model, target_replace_module, search_class=kinds):
        cls = type(child)
        if cls is nn.Linear or cls is LoraInjectedLinear:
            if len(loras[0].shape) != 2:
                continue
            src = child.linear if isinstance(child, LoraInjectedLinear) else child
            new = LoraInjectedLinear(src.in_features, src.out_features, src.bias is not None,
                                     r=_next_rank(r))
            new.linear.weight = src.weight
            if src.bias is not None:
                new.linear.bias = src.bias
        elif cls is nn.Conv2d or cls is LoraInjectedConv2d:
            if len(loras[0].shape) != 4:
                continue
            src = child.conv if isinstance(child, LoraInjectedConv2d) else child
            new = LoraInjectedConv2d(src.in_channels, src.out_channels, src.kernel_size, src.stride,
                                     src.padding, src.dilation, src.groups, src.bias is not None,
                                     r=_next_rank(r))
            new.conv.weight = src.weight
            if src.bias is not None:
                new.conv.bias = src.bias
        else:
            continue
        _install_factors(parent, name, new, loras, src.weight)


def monkeypatch_or_replace_safeloras(models, safeloras):
    """`models` is any object with attributes named like the file's model keys (a pipeline)."""
    for name, (lora, ranks, target) in parse_safeloras(safeloras).items():
        model = getattr(models, name, None)
        if not model:
            print(f"No model provided for {name}, contained in Lora")
            continue
        monkeypatch_or_replace_lora_extended(model, lora, target, ranks)


def monkeypatch_remove_lora(model):
    """Put plain nn.Linear / nn.Conv2d layers back, sharing the frozen Parameters (lora.py:812-847)."""
    for parent, name, site in _find_modules(model, search_class=[LoraInjectedLinear, LoraInjectedConv2d]):
        if isinstance(site, LoraInjectedLinear):
            src = site.linear
            plain = nn.Linear(src.in_features, src.out_features, src.bias is not None)
        else:
            src = site.conv
            plain = nn.Conv2d(in_channels=src.in_channels, out_channels=src.out_channels,
                              kernel_size=src.kernel_size, stride=src.stride, padding=src.padding,
                              dilation=src.dilation, groups=src.groups, bias=src.bias is not None)
        plain.weight = src.weight
        if src.bias is not None:
            plain.bias = src.bias
        parent._modules[name] = plain


def monkeypatch_add_lora(model, loras, target_replace_module=DEFAULT_TARGET_REPLACE,
                         alpha: float = 1.0, beta: float = 1.0):
    """factors <- alpha * new + beta * current, Linear sites only (lora.py:850-874)."""
    for parent, name, site in _find_modules(model, target_replace_module,
                                            search_class=[LoraInjectedLinear]):
        w = site.linear.weight
        up, down = loras.pop(0), loras.pop(0)
        cur = parent._modules[name]
        cur.lora_up.weight = nn.Parameter(
            up.type(w.dtype).to(w.device) * alpha + cur.lora_up.weight.to(w.device) * beta)
        cur.lora_down.weight = nn.Parameter(
            down.type(w.dtype).to(w.device) * alpha + cur.lora_down.weight.to(w.device) * beta)
        cur.to(w.device)


def tune_lora_scale(model, alpha: float = 1.0):
    """Set the python-float `scale` of every LoRA operator, matched by class NAME (lora.py:877-880)."""
    for m in model.modules():
        if type(m).__name__ in _LORA_CLASS_NAMES:
            m.scale = alpha


def set_lora_diag(model, diag: torch.Tensor):
    for m in model.modules():
        if type(m).__name__ in _LORA_CLASS_NAMES:
            m.set_selector_from_diag(diag)


def apply_learned_embed_in_clip(learned_embeds, text_encoder, tokenizer,
                                token: Optional[Union[str, List[str]]] = None, idempotent=False):
    """Install textual-inversion vectors as new tokenizer entries (lora.py:899-942)."""
    if isinstance(token, str):
        names = [token]
    elif isinstance(token, list):
        assert len(learned_embeds.keys()) == len(token), \
            "The number of tokens and the number of embeds should be the same"
        names = token
    else:
        names = list(learned_embeds.keys())
    for token in names:
        print(token)
        vec = learned_embeds[token]
        added = tokenizer.add_tokens(token)
        if not idempotent:
            i = 1
            while added == 0:
                print(f"The tokenizer already contains the token {token}.")
                token = f"{token[:-1]}-{i}>"
                print(f"Attempting to add the token {token}.")
                added = tokenizer.add_tokens(token)
                i += 1
        elif added == 0:
            print(f"The tokenizer already contains the token {token}.")
            print(f"Replacing {token} embedding.")
        text_encoder.resize_token_embeddings(len(tokenizer))
        token_id = tokenizer.convert_tokens_to_ids(token)
        text_encoder.get_input_embeddings().weight.data[token_id] = vec
    return token


def load_learned_embed_in_clip(learned_embeds_path, text_encoder, tokenizer,
                               token: Optional[Union[str, List[str]]] = None, idempotent=False):
    apply_learned_embed_in_clip(torch.load(learned_embeds_path), text_encoder, tokenizer, token,
                                idempotent)


def patch_pipe(pipe, maybe_unet_path, token: Optional[str] = None, r: int = 4, patch_unet=True,
               patch_text=True, patch_ti=True, idempotent_token=True,
               unet_target_replace_module=DEFAULT_TARGET_REPLACE,
               text_target_replace_module=TEXT_ENCODER_DEFAULT_TARGET_REPLACE):
    """Load a LoRA (+ TI embeds) into a pipeline-like object with .unet/.text_encoder/.tokenizer
    (lora.py:958-1022). `.pt` triplets and single `.safetensors` files are both accepted."""
    if maybe_unet_path.endswith(".pt"):
        if maybe_unet_path.endswith(".ti.pt"):
            unet_path = maybe_unet_path[:-6] + ".pt"
        elif maybe_unet_path.endswith(".text_encoder.pt"):
            unet_path = maybe_unet_path[:-16] + ".pt"
        else:
            unet_path = maybe_unet_path
        if patch_unet:
            print("LoRA : Patching Unet")
            monkeypatch_or_replace_lora(pipe.unet, torch.load(unet_path), r=r,
                                        target_replace_module=unet_target_replace_module)
        if patch_text:
            print("LoRA : Patching text encoder")
            monkeypatch_or_replace_lora(pipe.text_encoder, torch.load(_text_lora_path(unet_path)),
                                        target_replace_module=text_target_replace_module, r=r)
        if patch_ti:
            print("LoRA : Patching token input")
            token = load_learned_embed_in_clip(_ti_lora_path(unet_path), pipe.text_encoder,
                                               pipe.tokenizer, token=token,
                                               idempotent=idempotent_token)
    elif maybe_unet_path.endswith(".safetensors"):
        f = safe_open(maybe_unet_path, framework="pt", device="cpu")
        monkeypatch_or_replace_safeloras(pipe, f)
        tok_dict = parse_safeloras_embeds(f)
        if patch_ti:
            apply_learned_embed_in_clip(tok_dict, pipe.text_encoder, pipe.tokenizer, token=token,
                                        idempotent=idempotent_token)
        return tok_dict


@torch.no_grad()
def inspect_lora(model):
    """{site name: [mean |up @ down|]} -- how far each LoRA has moved (lora.py:1025-1042)."""
    moved = {}
    for name, m in model.named_modules():
        if type(m).__name__ in _LORA_CLASS_NAMES:
            prod = m.lora_up.weight.data.clone().flatten(1) @ m.lora_down.weight.data.clone().flatten(1)
            moved.setdefault(name, []).append(prod.flatten().abs().mean().item())
    return moved
