"""Gradient checkpointing of the host UNet (lora_b200/host/unet_sd15.py): diffusers' API, and the same
outputs and parameter gradients with and without it (plain nn.Linear / nn.Conv2d, no LoRA sites, CPU)."""
import pytest
import torch

from lora_b200.host import unet_sd15
from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig

CONFIGS = {"sd15_tiny": UNetConfig.tiny, "sd2_tiny": UNetConfig.sd2_tiny}


def _model_and_inputs(name):
    cfg = CONFIGS[name]()
    torch.manual_seed(0)
    unet = UNet2DConditionModel(cfg)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 4, 16, 16, generator=g)
    ctx = torch.randn(2, 7, cfg.cross_attention_dim, generator=g)
    t = torch.tensor([10, 500])
    return unet, x, ctx, t


def _run(unet, x, ctx, t):
    unet.zero_grad(set_to_none=True)
    xi = x.clone().requires_grad_(True)
    y = unet(xi, t, ctx).sample
    (y.float().square().mean() + y.sum() * 1e-3).backward()
    return y.detach(), xi.grad, [p.grad for p in unet.parameters()]


def _counting(monkeypatch):
    calls = []
    real = unet_sd15.checkpoint

    def counted(fn, *args, **kw):
        calls.append(type(fn).__name__)
        return real(fn, *args, **kw)

    monkeypatch.setattr(unet_sd15, "checkpoint", counted)
    return calls


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_checkpointed_unet_is_bit_equal(name, monkeypatch):
    unet, x, ctx, t = _model_and_inputs(name)
    y0, gx0, g0 = _run(unet, x, ctx, t)
    assert not unet.is_gradient_checkpointing
    calls = _counting(monkeypatch)
    unet.enable_gradient_checkpointing()
    assert unet.is_gradient_checkpointing
    y1, gx1, g1 = _run(unet, x, ctx, t)
    assert torch.equal(y0, y1) and torch.equal(gx0, gx1)
    assert len(g0) == len(g1) and all(torch.equal(a, b) for a, b in zip(g0, g1))
    # every ResnetBlock2D and Transformer2DModel call of the down, mid and up blocks, nothing else
    n_res = sum(type(m).__name__ == "ResnetBlock2D" for m in unet.modules())
    n_attn = sum(type(m).__name__ == "Transformer2DModel" for m in unet.modules())
    assert sorted(set(calls)) == ["ResnetBlock2D", "Transformer2DModel"]
    assert calls.count("ResnetBlock2D") == n_res and calls.count("Transformer2DModel") == n_attn


def test_checkpointing_only_in_training_mode(monkeypatch):
    unet, x, ctx, t = _model_and_inputs("sd15_tiny")
    unet.enable_gradient_checkpointing()
    calls = _counting(monkeypatch)
    unet.eval()
    y_eval = unet(x, t, ctx).sample
    assert calls == []
    unet.train()
    y_train = unet(x, t, ctx).sample
    assert len(calls) > 0 and torch.equal(y_eval, y_train)


def test_disable_gradient_checkpointing(monkeypatch):
    unet, x, ctx, t = _model_and_inputs("sd2_tiny")
    unet.enable_gradient_checkpointing()
    unet.disable_gradient_checkpointing()
    assert not unet.is_gradient_checkpointing
    calls = _counting(monkeypatch)
    _run(unet, x, ctx, t)
    assert calls == []


def test_step_config_default_is_off():
    from lora_b200.train import StepConfig
    assert StepConfig().gradient_checkpointing is False
