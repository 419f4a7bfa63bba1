"""Parity with the reference module (lora_diffusion/lora.py of cloneofsimo/lora). Every test is a
scenario that runs against a module namespace: scripts/make_golden_live.py ran it against the
reference and stored what it returned in tests/golden/reference_live.json (one digest per checked
item; equal digests mean bitwise-equal results) and tests/golden/reference_modules.pt (operator
outputs); here it runs against lora_b200 and the oracle and is compared with that record."""
import copy
import inspect
import json
import os

import pytest
import torch
import torch.nn as nn
from safetensors import safe_open

import lora_b200 as L
from lora_b200.host.clip import build_text_encoder
from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
from oracle.fingerprint import digest, fingerprint
from oracle.ref_modules import RefLoraSite, ref_inject

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

SIGNATURE_NAMES = ("inject_trainable_lora", "inject_trainable_lora_extended", "monkeypatch_or_replace_lora",
                   "monkeypatch_or_replace_lora_extended", "patch_pipe", "save_all", "tune_lora_scale",
                   "monkeypatch_add_lora", "apply_learned_embed_in_clip", "extract_lora_as_tensor")


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(GOLD, "reference_live.json")) as fh:
        return json.load(fh)


def _sites(model):
    return [m for m in model.modules() if type(m).__name__.startswith("LoraInjected")]


def _signature(fn):
    """Parameter names in order with their defaults (sets compare by value)."""
    out = []
    for k, p in inspect.signature(fn).parameters.items():
        d = p.default
        out.append([k, "<none>" if d is inspect.Parameter.empty else fingerprint(d)])
    return out


def public_names(M):
    names = {n for n in dir(M) if not n.startswith("_") and (callable(getattr(M, n)) or n.isupper()
             or n in ("safetensors_available",))}
    skip = {"Callable", "Dict", "List", "Optional", "Set", "Tuple", "Type", "Union", "groupby", "F", "nn",
            "np", "PIL", "torch", "json", "math", "_find_modules_old"}
    return sorted(n for n in names if n not in skip and not inspect.ismodule(getattr(M, n)))


def signatures(M):
    sig = {n: _signature(getattr(M, n)) for n in SIGNATURE_NAMES}
    sig["LoraInjectedLinear"] = _signature(M.LoraInjectedLinear.__init__)
    sig["LoraInjectedConv2d"] = _signature(M.LoraInjectedConv2d.__init__)
    return sig


def test_public_names_cover_the_reference_namespace(golden):
    missing = sorted(n for n in golden["public_names"] if not hasattr(L, n))
    assert missing == [], missing
    assert fingerprint(signatures(L)) == golden["signatures"]


def inject_save_load(M, tmp_path):
    """Inject, save, patch a fresh model from the saved file, collapse: what each step produced."""
    torch.manual_seed(0)
    unet = UNet2DConditionModel(UNetConfig.tiny())
    te = build_text_encoder(tiny=True)
    torch.manual_seed(1)
    _, n_unet = M.inject_trainable_lora_extended(unet, r=4)
    _, n_text = M.inject_trainable_lora(te, target_replace_module={"CLIPAttention"}, r=4)
    sites = _sites(unet) + _sites(te)
    g = torch.Generator().manual_seed(2)
    for s in sites:
        s.lora_up.weight.data.normal_(0, 0.05, generator=g)
    M.tune_lora_scale(unet, 0.7)
    path = str(tmp_path / "lora.safetensors")
    M.save_all(unet, te, path, save_ti=False, target_replace_module_unet=M.UNET_EXTENDED_TARGET_REPLACE)
    f = safe_open(path, "pt")
    saved = {k: f.get_tensor(k) for k in sorted(f.keys())}

    class P:
        pass
    pipe = P()
    torch.manual_seed(0)
    pipe.unet, pipe.text_encoder = UNet2DConditionModel(UNetConfig.tiny()), build_text_encoder(tiny=True)
    M.monkeypatch_or_replace_safeloras(pipe, f)
    patched = [[type(s).__name__, s.lora_up.weight, s.lora_down.weight]
               for s in _sites(pipe.unet) + _sites(pipe.text_encoder)]
    M.collapse_lora(pipe.unet, 0.5)
    collapsed = [s.linear.weight if hasattr(s, "linear") else s.conv.weight for s in _sites(pipe.unet)]
    return {"n": [n_unet, n_text], "site_types": [type(s).__name__ for s in sites],
            "downs": [s.lora_down.weight for s in sites], "saved": saved, "patched": patched,
            "collapsed": collapsed}


def test_inject_save_load_equal_reference_on_tiny_models(golden, tmp_path):
    got = inject_save_load(L, tmp_path)
    want = golden["inject_save_load"]
    for k in want:      # one key at a time: a mismatch names the stage that differs
        assert digest(got[k]) == want[k], k


def operator_cases():
    """Seeded inputs of the two operator cases: (conv?, base weight, base bias, down, up, x, gy)."""
    g = torch.Generator().manual_seed(3)
    cases = []
    for conv in (False, True):
        if conv:
            w, b, x = torch.randn(12, 8, 3, 3, generator=g) * 0.1, torch.randn(12, generator=g), torch.randn(2, 8, 7, 7, generator=g)
            down = torch.randn(4, 8, 3, 3, generator=g) * 0.1
            up = torch.randn(12, 4, 1, 1, generator=g) * 0.1
            gy = torch.randn(2, 12, 7, 7, generator=g)
        else:
            w, b, x = torch.randn(40, 24, generator=g) * 0.2, torch.randn(40, generator=g), torch.randn(3, 5, 24, generator=g)
            down = torch.randn(4, 24, generator=g) * 0.2
            up = torch.randn(40, 4, generator=g) * 0.1
            gy = torch.randn(3, 5, 40, generator=g)
        cases.append((conv, w, b, down, up, x, gy))
    return cases


def reference_module_outputs(M):
    """The reference's operator classes on operator_cases(), fp32, forward + backward."""
    outs = []
    for conv, w, b, down, up, x, gy in operator_cases():
        if conv:
            mod = M.LoraInjectedConv2d(8, 12, 3, 1, 1, r=4, dropout_p=0.0, scale=1.3)
            mod.conv.weight.data.copy_(w); mod.conv.bias.data.copy_(b)
        else:
            mod = M.LoraInjectedLinear(24, 40, True, r=4, dropout_p=0.0, scale=1.3)
            mod.linear.weight.data.copy_(w); mod.linear.bias.data.copy_(b)
        mod.lora_down.weight.data.copy_(down); mod.lora_up.weight.data.copy_(up)
        x1 = x.clone().requires_grad_(True)
        y = mod(x1)
        y.backward(gy)
        outs.append({"y": y.detach(), "dx": x1.grad, "ddown": mod.lora_down.weight.grad,
                     "dup": mod.lora_up.weight.grad})
    return outs


def test_oracle_modules_equal_reference_modules_fp32():
    """oracle/ref_modules.RefLoraSite vs the reference operator classes, random inputs, fwd+bwd."""
    want = torch.load(os.path.join(GOLD, "reference_modules.pt"))
    for (conv, w, b, down, up, x, gy), ref in zip(operator_cases(), want):
        base = nn.Conv2d(8, 12, 3, padding=1) if conv else nn.Linear(24, 40)
        base.weight.data.copy_(w); base.bias.data.copy_(b)
        site = RefLoraSite(base, r=4, dropout_p=0.0, scale=1.3)
        site.down.data.copy_(down); site.up.data.copy_(up)
        x2 = x.clone().requires_grad_(True)
        y2 = site(x2)
        y2.backward(gy)
        assert torch.allclose(ref["y"], y2, atol=1e-5)
        assert torch.allclose(ref["dx"], x2.grad, atol=1e-5)
        assert torch.allclose(ref["ddown"], site.down.grad, atol=1e-5)
        assert torch.allclose(ref["dup"], site.up.grad, atol=1e-5)


def inject_order(M):
    """Site shapes and frozen weights, in order, of the reference's extended inject on the tiny UNet."""
    torch.manual_seed(0)
    u = UNet2DConditionModel(UNetConfig.tiny())
    M.inject_trainable_lora_extended(u, r=4)
    return [[list(s.lora_up.weight.shape), list(s.lora_down.weight.shape),
             s.linear.weight if hasattr(s, "linear") else s.conv.weight] for s in _sites(u)]


def test_oracle_inject_order_equals_reference(golden):
    torch.manual_seed(0)
    u = UNet2DConditionModel(UNetConfig.tiny())
    sites = ref_inject(u, L.UNET_EXTENDED_TARGET_REPLACE, r=4, extended=True)
    got = digest([[list(a.up.shape), list(a.down.shape), a.weight] for a in sites])
    assert got == golden["inject_order"]


class Tok:
    def __init__(self, n):
        self.v = {f"w{i}": i for i in range(n)}

    def add_tokens(self, t):
        if t in self.v:
            return 0
        self.v[t] = len(self.v)
        return 1

    def convert_tokens_to_ids(self, t):
        return self.v[t]

    def __len__(self):
        return len(self.v)


def small_helpers(M, tmp_path):
    """_find_children, extract_lora_ups_down, save_lora_as_json, save_lora_weight (.pt),
    load_safeloras / load_safeloras_embeds / load_safeloras_both, _ti_lora_path, _text_lora_path,
    load_learned_embed_in_clip -- on the tiny UNet / text encoder."""
    import warnings
    out = {}
    torch.manual_seed(0)
    model = UNet2DConditionModel(UNetConfig.tiny())
    out["find_children"] = [[type(p).__name__, n, list(c.weight.shape)]
                            for p, n, c in M._find_children(model, [nn.Linear, nn.Conv2d])]
    torch.manual_seed(1)
    M.inject_trainable_lora(model, r=4)
    g = torch.Generator().manual_seed(2)
    for s in _sites(model):
        s.lora_up.weight.data.normal_(0, 0.02, generator=g)
    out["downs"] = [s.lora_down.weight for s in _sites(model)]
    out["ups_down"] = [[u.weight, d.weight] for u, d in M.extract_lora_ups_down(model)]
    M.save_lora_as_json(model, str(tmp_path / "l.json"))
    with open(tmp_path / "l.json", "rb") as fh:
        out["json"] = fh.read()
    M.save_lora_weight(model, str(tmp_path / "l.pt"))
    out["pt"] = list(torch.load(tmp_path / "l.pt"))
    emb = {"<tok>": torch.randn(48, generator=g)}
    M.save_safeloras_with_embeds({"unet": (model, M.UNET_DEFAULT_TARGET_REPLACE)}, emb, str(tmp_path / "x.safetensors"))
    flat = lambda d: {k: [[torch.as_tensor(t) for t in v[0]], v[1], sorted(v[2])] for k, v in d.items()}
    out["load_safeloras"] = flat(M.load_safeloras(str(tmp_path / "x.safetensors")))
    out["load_safeloras_embeds"] = M.load_safeloras_embeds(str(tmp_path / "x.safetensors"))
    both = M.load_safeloras_both(str(tmp_path / "x.safetensors"))
    out["load_safeloras_both"] = [flat(both[0]), both[1]]
    out["paths"] = [M._ti_lora_path("a/b.c.pt"), M._text_lora_path("a/b.c.pt")]
    torch.manual_seed(3)
    te = build_text_encoder(tiny=True)
    V = te.get_input_embeddings().weight.shape[0]
    torch.save(emb, tmp_path / "e.pt")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        torch.manual_seed(4)
        M.load_learned_embed_in_clip(str(tmp_path / "e.pt"), te, Tok(V), token=None, idempotent=True)
    out["embeddings"] = te.get_input_embeddings().weight
    out["learned_row"] = te.get_input_embeddings().weight[V]
    return out


def test_small_helpers_equal_reference(golden, tmp_path):
    got = small_helpers(L, tmp_path)
    assert len(got["find_children"]) > 20
    assert torch.equal(got["learned_row"], torch.load(tmp_path / "e.pt")["<tok>"])
    want = golden["small_helpers"]
    for k in want:
        assert digest(got[k]) == want[k], k
