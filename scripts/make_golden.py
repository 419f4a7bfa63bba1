"""Generate tests/golden/* by RUNNING THE REAL REFERENCE (/root/reference/lora_diffusion/lora.py
and cli_svd.py, loaded by file path because the package import needs fire/diffusers) on small
seeded inputs. Run in the build container (the reference tree does not exist on the GPU box):

    python scripts/make_golden.py

Outputs (all small, committed):
  golden/ops_linear.pt, ops_conv.pt     operator forward + autograd grads (fp32, CPU)
  golden/ctor_rng.pt                    lora_down init values after manual_seed(0) (RNG parity)
  golden/inject_tiny.json               site names/order from the reference's inject on the tiny
                                        host UNet / CLIP (default + extended target sets)
  golden/tiny_saved.safetensors         save_safeloras output of the reference on the tiny models
  golden/example_loras_manifest.json    keys / shapes / dtypes / metadata / sha256 of the ten
                                        fixture files in /root/reference/example_loras
  golden/svd_distill.pt                 cli_svd.overwrite_base outputs on small matrices
  golden/adamw_clip.pt                  clip_grad_norm_ + torch.optim.AdamW trajectories
  golden/pti_loss_step.pt               cli_lora_pti.loss_step losses (plain / t_mult / masked / inpainting)
  golden/pti_loss_step_v.pt             the same with prediction_type "v_prediction" (+ one SD2 tiny case)
  golden/ti_train_inversion.pt          cli_lora_pti.train_inversion: 3 real steps (grads, lr, rows after)
  golden/pti_perform_tuning.pt          cli_lora_pti.perform_tuning: 3 real steps (losses, lrs, all factors after)
  golden/pti_continue_inversion.pt      the same loop with continue_inversion: 3 real steps (losses, lrs,
                                        the whole token-embedding table after each)

`python scripts/make_golden.py continue_inversion` regenerates one file only.
"""
import hashlib
import importlib.util
import itertools
import json
import os
import sys
import types

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden")
os.makedirs(OUT, exist_ok=True)


def load_ref_lora():
    spec = importlib.util.spec_from_file_location("ref_lora", f"{REF}/lora_diffusion/lora.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_ref_svd(ref_lora):
    """cli_svd.py imports fire and diffusers at module top; stub them, and satisfy its relative
    import `.lora` with the already-loaded reference module."""
    pkg = types.ModuleType("lora_diffusion_ref")
    pkg.__path__ = [f"{REF}/lora_diffusion"]
    sys.modules["lora_diffusion_ref"] = pkg
    sys.modules["lora_diffusion_ref.lora"] = ref_lora
    sys.modules.setdefault("fire", types.ModuleType("fire"))
    d = types.ModuleType("diffusers")
    d.StableDiffusionPipeline = object
    sys.modules.setdefault("diffusers", d)
    spec = importlib.util.spec_from_file_location("lora_diffusion_ref.cli_svd", f"{REF}/lora_diffusion/cli_svd.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def gen_ops(R):
    cases = []
    for i, (M, K, N, r, bias, scale, diag) in enumerate([
            (24, 16, 24, 4, True, 1.0, False), (10, 32, 8, 1, False, 0.5, False),
            (33, 40, 48, 8, True, 1.7, True), (7, 64, 64, 16, True, 0.25, True)]):
        torch.manual_seed(100 + i)
        m = R.LoraInjectedLinear(K, N, bias, r=r, dropout_p=0.0, scale=scale)
        m.lora_up.weight.data.normal_(0, 0.1)
        d = None
        if diag:
            d = torch.rand(r) + 0.5
            m.set_selector_from_diag(d)
        x = torch.randn(2, M, K, requires_grad=True)
        y = m(x)
        gy = torch.randn_like(y)
        y.backward(gy)
        cases.append(dict(x=x.detach(), W=m.linear.weight.detach(), b=None if not bias else m.linear.bias.detach(),
                          A=m.lora_down.weight.detach(), B=m.lora_up.weight.detach(), scale=scale, diag=d,
                          y=y.detach(), gy=gy, dX=x.grad, dA=m.lora_down.weight.grad, dB=m.lora_up.weight.grad,
                          dW_is_none=True))
    torch.save(cases, f"{OUT}/ops_linear.pt")

    conv = []
    for i, (Cin, Cout, k, pad, r, bias, scale, HW) in enumerate([
            (8, 16, 3, 1, 4, True, 1.0, 6), (16, 8, 1, 0, 4, False, 0.5, 5), (12, 12, 3, 1, 8, True, 2.0, 9)]):
        torch.manual_seed(200 + i)
        m = R.LoraInjectedConv2d(Cin, Cout, k, 1, pad, 1, 1, bias, r=r, dropout_p=0.0, scale=scale)
        m.lora_up.weight.data.normal_(0, 0.1)
        x = torch.randn(2, Cin, HW, HW, requires_grad=True)
        y = m(x)
        gy = torch.randn_like(y)
        y.backward(gy)
        conv.append(dict(x=x.detach(), W=m.conv.weight.detach(), b=None if not bias else m.conv.bias.detach(),
                         A=m.lora_down.weight.detach(), B=m.lora_up.weight.detach(), scale=scale, padding=pad,
                         y=y.detach(), gy=gy, dX=x.grad, dA=m.lora_down.weight.grad, dB=m.lora_up.weight.grad))
    torch.save(conv, f"{OUT}/ops_conv.pt")

    # dropout statistics are not golden-able (Philox stream); keep the p>0 eval-mode identity
    torch.manual_seed(7)
    m = R.LoraInjectedLinear(16, 16, False, r=4, dropout_p=0.1)
    m.lora_up.weight.data.normal_(0, 0.1)
    m.eval()
    x = torch.randn(5, 16)
    torch.save(dict(x=x, W=m.linear.weight.detach(), A=m.lora_down.weight.detach(), B=m.lora_up.weight.detach(),
                    y_eval=m(x).detach()), f"{OUT}/ops_dropout_eval.pt")


def gen_ctor_rng(R):
    out = {}
    torch.manual_seed(0)
    m = R.LoraInjectedLinear(16, 24, True, r=4)
    out["linear_down"] = m.lora_down.weight.detach().clone()
    out["linear_next_rand"] = torch.rand(3)
    torch.manual_seed(0)
    c = R.LoraInjectedConv2d(8, 12, 3, 1, 1, r=4)
    out["conv_down"] = c.lora_down.weight.detach().clone()
    out["conv_next_rand"] = torch.rand(3)
    torch.save(out, f"{OUT}/ctor_rng.pt")


def gen_inject(R):
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    res = {}
    torch.manual_seed(0)
    unet = UNet2DConditionModel(UNetConfig.tiny())
    _, names = R.inject_trainable_lora(unet, r=4)
    res["unet_default_names"] = names
    res["unet_default_shapes"] = [[list(m.lora_up.weight.shape), list(m.lora_down.weight.shape)]
                                  for m in unet.modules() if m.__class__.__name__.startswith("LoraInjected")]
    torch.manual_seed(0)
    unet2 = UNet2DConditionModel(UNetConfig.tiny())
    _, names2 = R.inject_trainable_lora_extended(unet2, r=4)
    res["unet_extended_names"] = names2
    res["unet_extended_kinds"] = [m.__class__.__name__ for m in unet2.modules()
                                  if m.__class__.__name__.startswith("LoraInjected")]
    res["unet_extended_shapes"] = [[list(m.lora_up.weight.shape), list(m.lora_down.weight.shape)]
                                   for m in unet2.modules() if m.__class__.__name__.startswith("LoraInjected")]
    torch.manual_seed(0)
    te = build_text_encoder(tiny=True)
    _, names3 = R.inject_trainable_lora(te, target_replace_module={"CLIPAttention"}, r=4)
    res["text_names"] = names3
    # a saved file from the reference, with non-trivial factors and scale
    g = torch.Generator().manual_seed(5)
    for mdl in (unet, te):
        for m in mdl.modules():
            if m.__class__.__name__ == "LoraInjectedLinear":
                m.lora_up.weight.data.normal_(0, 0.05, generator=g)
    R.tune_lora_scale(unet, 0.5)
    R.save_safeloras_with_embeds({"unet": (unet, R.DEFAULT_TARGET_REPLACE),
                                  "text_encoder": (te, R.TEXT_ENCODER_DEFAULT_TARGET_REPLACE)},
                                 {"<s1>": torch.arange(48, dtype=torch.float32)},
                                 f"{OUT}/tiny_saved.safetensors")
    # the raw factors that produced it (so the test can rebuild the same state with our API)
    raw = {"unet": [], "text_encoder": []}
    for key, mdl in (("unet", unet), ("text_encoder", te)):
        for m in mdl.modules():
            if m.__class__.__name__ == "LoraInjectedLinear":
                raw[key].append((m.lora_up.weight.detach().clone(), m.lora_down.weight.detach().clone()))
    torch.save(raw, f"{OUT}/tiny_saved_raw.pt")
    json.dump(res, open(f"{OUT}/inject_tiny.json", "w"), indent=1)


def gen_manifest(R):
    from safetensors import safe_open
    man = {}
    d = f"{REF}/example_loras"
    for fn in sorted(os.listdir(d)):
        if not fn.endswith(".safetensors"):
            continue
        f = safe_open(f"{d}/{fn}", framework="pt", device="cpu")
        ent = {"metadata": f.metadata(), "tensors": {}}
        for k in sorted(f.keys()):
            t = f.get_tensor(k)
            ent["tensors"][k] = [list(t.shape), str(t.dtype).replace("torch.", ""),
                                 hashlib.sha256(t.contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()[:16]]
        parsed = R.parse_safeloras(f)
        ent["parsed"] = {name: {"n_weights": len(w), "ranks": r, "targets": sorted(t)}
                         for name, (w, r, t) in parsed.items()}
        ent["embeds"] = sorted(R.parse_safeloras_embeds(f).keys())
        man[fn] = ent
    json.dump(man, open(f"{OUT}/example_loras_manifest.json", "w"))


def gen_svd(R):
    S = load_ref_svd(R)
    out = []
    for i, (N, K, rank, conv) in enumerate([(48, 32, 4, False), (24, 64, 8, False), (16, 8, 4, True)]):
        torch.manual_seed(300 + i)

        class Holder(nn.Module):
            def __init__(self):
                super().__init__()
                if conv:
                    self.m = R.LoraInjectedConv2d(K, N, 3, 1, 1, r=rank)
                else:
                    self.m = R.LoraInjectedLinear(K, N, False, r=rank)

            @property
            def device(self):
                return torch.device("cpu")

            @property
            def dtype(self):
                return torch.float32

        base, tuned = Holder(), Holder()
        wb = (base.m.conv if conv else base.m.linear).weight
        wt = (tuned.m.conv if conv else tuned.m.linear).weight
        low = torch.randn(N, rank) @ torch.randn(rank, wb[0].numel()) * 0.02
        wt.data = wb.data + low.reshape(wb.shape) + torch.randn_like(wb) * 1e-3
        S.overwrite_base(base, tuned, rank=rank, clamp_quantile=0.99)
        out.append(dict(Wb=wb.detach().clone(), Wt=wt.detach().clone(), rank=rank, conv=conv, q=0.99,
                        up=base.m.lora_up.weight.detach().clone(), down=base.m.lora_down.weight.detach().clone()))
    torch.save(out, f"{OUT}/svd_distill.pt")


def gen_adamw():
    torch.manual_seed(400)
    ps = [torch.randn(6, 4), torch.randn(4, 10), torch.randn(3, 3)]
    lrs = [1e-3, 1e-3, 5e-4]
    twins = [p.clone().requires_grad_(True) for p in ps]
    opt = torch.optim.AdamW([{"params": twins[:2], "lr": 1e-3}, {"params": twins[2:], "lr": 5e-4}],
                            betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    traj = []
    for step in range(1, 5):
        gs = [torch.randn_like(p) * (2.0 if step % 2 else 0.05) for p in ps]
        for t, g in zip(twins, gs):
            t.grad = g.clone()
        total = torch.nn.utils.clip_grad_norm_(twins, 1.0)
        opt.step()
        traj.append(dict(grads=gs, total_norm=float(total), params=[t.detach().clone() for t in twins]))
    torch.save(dict(p0=ps, lrs=lrs, traj=traj), f"{OUT}/adamw_clip.pt")


def load_ref_pti(ref_lora):
    """cli_lora_pti.py pulls diffusers / fire / the lora_diffusion package at module top; none of
    them is touched by `loss_step` itself. Stand-ins whose attributes are inert placeholders let the
    real file execute so that the real function object can be called."""
    class _Inert(types.ModuleType):
        def __getattr__(self, name):
            if name.startswith("__"):
                raise AttributeError(name)
            return type(name, (), {"__init__": lambda self, *a, **k: None})
    saved = {}
    # huggingface_hub is installed but no longer has the names the file asks for: shadow it too
    for name in ("fire", "diffusers", "diffusers.optimization", "lora_diffusion", "wandb", "huggingface_hub"):
        saved[name] = sys.modules.get(name)
        sys.modules[name] = _Inert(name)
    try:
        spec = importlib.util.spec_from_file_location("ref_cli_lora_pti", f"{REF}/lora_diffusion/cli_lora_pti.py")
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        for name, old in saved.items():
            if old is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = old
    return mod


def gen_loss_step(R):
    """The PTI/Dreambooth loss of one step, computed by the reference's own `loss_step`
    (cli_lora_pti.py:260-370) on the tiny host models, CPU fp32, cached latents: plain, t_mutliplier
    0.8, masked loss (two temperatures), inpainting (9-channel input), inpainting + mask."""
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    P = load_ref_pti(R)
    noiser = DDPMNoiser(device="cpu")

    class Sched:                      # what loss_step reads from a diffusers DDPMScheduler
        config = types.SimpleNamespace(num_train_timesteps=noiser.num_train_timesteps, prediction_type="epsilon")
        add_noise = staticmethod(noiser.add_noise)

    g = torch.Generator().manual_seed(77)
    lat = torch.randn(2, 4, 8, 8, generator=g) * 0.18215
    ids = torch.randint(0, 1000, (2, 77), generator=g)
    loss_mask = (torch.rand(2, 1, 64, 64, generator=g) > 0.4).float()          # image resolution
    inp_mask = (torch.rand(2, 1, 8, 8, generator=g) > 0.5).float()             # cached: latent resolution
    inp_lat = torch.randn(2, 4, 8, 8, generator=g) * 0.18215
    cases = []
    for name, in_ch, kw, with_mask in [
            ("plain", 4, dict(), False),
            ("t_mult_0.8", 4, dict(t_mutliplier=0.8), False),
            ("masked_T1", 4, dict(mask_temperature=1.0), True),
            ("masked_T2.5", 4, dict(mask_temperature=2.5), True),
            ("inpaint", 9, dict(train_inpainting=True), False),
            ("inpaint_masked", 9, dict(train_inpainting=True, mask_temperature=1.0), True)]:
        torch.manual_seed(0)
        cfg = UNetConfig.tiny()
        cfg.in_channels = in_ch
        unet = UNet2DConditionModel(cfg)
        text = build_text_encoder(tiny=True)
        # a live LoRA branch (reference modules, non-zero up) so that the loss depends on it
        R.inject_trainable_lora(unet, r=4)
        gg = torch.Generator().manual_seed(5)
        for m in unet.modules():
            if type(m).__name__ == "LoraInjectedLinear":
                m.lora_down.weight.data.normal_(0, 0.25, generator=gg)     # explicit: independent of ctor RNG
                m.lora_up.weight.data.normal_(0, 0.05, generator=gg)
                m.dropout.p = 0.0
        batch = {"pixel_values": lat, "input_ids": ids}
        if in_ch == 9:
            batch.update(masked_image_latents=inp_lat, mask_values=inp_mask)
        if with_mask:
            batch["mask"] = loss_mask
        text.train(False), unet.train(False)
        torch.manual_seed(1234)
        loss = P.loss_step(batch, unet, None, text, Sched, cached_latents=True, **kw)
        cases.append(dict(name=name, in_channels=in_ch, kwargs=kw, with_mask=with_mask, loss=float(loss)))
    torch.save(dict(latents=lat, input_ids=ids, loss_mask=loss_mask, inpaint_mask=inp_mask,
                    masked_latents=inp_lat, model_seed=0, up_seed=5, step_seed=1234, cases=cases),
               f"{OUT}/pti_loss_step.pt")
    print({c["name"]: c["loss"] for c in cases})


def gen_loss_step_v(R):
    """`loss_step` (cli_lora_pti.py:260-370) with the scheduler's prediction_type = "v_prediction", so
    that its :333-338 branch regresses `scheduler.get_velocity(latents, noise, timesteps)`: plain,
    t_mutliplier 0.8, masked, inpainting on the tiny SD1.5 models, and plain on the tiny SD2 models
    (UNetConfig.sd2_tiny + the tiny SD2 text encoder). CPU fp32, cached latents."""
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    P = load_ref_pti(R)
    noiser = DDPMNoiser(device="cpu")

    class Sched:                      # what loss_step reads from a diffusers DDPMScheduler
        config = types.SimpleNamespace(num_train_timesteps=noiser.num_train_timesteps,
                                       prediction_type="v_prediction")
        add_noise = staticmethod(noiser.add_noise)
        # a restatement of diffusers' DDPMScheduler.get_velocity (scaled_linear betas 0.00085 -> 0.012):
        # sqrt(acp[t]) * noise - sqrt(1 - acp[t]) * sample, computed from alphas_cumprod like diffusers
        alphas_cumprod = torch.cumprod(1.0 - torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000,
                                                            dtype=torch.float32) ** 2, dim=0)

        @staticmethod
        def get_velocity(sample, noise, timesteps):
            acp = Sched.alphas_cumprod.to(device=sample.device, dtype=sample.dtype)
            sqrt_alpha_prod = (acp[timesteps] ** 0.5).flatten()
            while len(sqrt_alpha_prod.shape) < len(sample.shape):
                sqrt_alpha_prod = sqrt_alpha_prod.unsqueeze(-1)
            sqrt_one_minus_alpha_prod = ((1 - acp[timesteps]) ** 0.5).flatten()
            while len(sqrt_one_minus_alpha_prod.shape) < len(sample.shape):
                sqrt_one_minus_alpha_prod = sqrt_one_minus_alpha_prod.unsqueeze(-1)
            return sqrt_alpha_prod * noise - sqrt_one_minus_alpha_prod * sample

    g = torch.Generator().manual_seed(78)
    lat = torch.randn(2, 4, 8, 8, generator=g) * 0.18215
    ids = torch.randint(0, 1000, (2, 77), generator=g)
    loss_mask = (torch.rand(2, 1, 64, 64, generator=g) > 0.4).float()
    inp_mask = (torch.rand(2, 1, 8, 8, generator=g) > 0.5).float()
    inp_lat = torch.randn(2, 4, 8, 8, generator=g) * 0.18215
    cases = []
    for name, model, in_ch, kw, with_mask in [
            ("plain", "sd15_tiny", 4, dict(), False),
            ("t_mult_0.8", "sd15_tiny", 4, dict(t_mutliplier=0.8), False),
            ("masked_T1", "sd15_tiny", 4, dict(mask_temperature=1.0), True),
            ("inpaint", "sd15_tiny", 9, dict(train_inpainting=True), False),
            ("sd2_plain", "sd2_tiny", 4, dict(), False)]:
        torch.manual_seed(0)
        sd2 = model == "sd2_tiny"
        cfg = UNetConfig.sd2_tiny() if sd2 else UNetConfig.tiny()
        cfg.in_channels = in_ch
        unet = UNet2DConditionModel(cfg)
        text = build_text_encoder(tiny=True, sd2=sd2)
        R.inject_trainable_lora(unet, r=4)
        gg = torch.Generator().manual_seed(5)
        for m in unet.modules():
            if type(m).__name__ == "LoraInjectedLinear":
                m.lora_down.weight.data.normal_(0, 0.25, generator=gg)
                m.lora_up.weight.data.normal_(0, 0.05, generator=gg)
                m.dropout.p = 0.0
        batch = {"pixel_values": lat, "input_ids": ids}
        if in_ch == 9:
            batch.update(masked_image_latents=inp_lat, mask_values=inp_mask)
        if with_mask:
            batch["mask"] = loss_mask
        text.train(False), unet.train(False)
        torch.manual_seed(1235)
        loss = P.loss_step(batch, unet, None, text, Sched, cached_latents=True, **kw)
        cases.append(dict(name=name, model=model, in_channels=in_ch, kwargs=kw, with_mask=with_mask,
                          loss=float(loss)))
    torch.save(dict(latents=lat, input_ids=ids, loss_mask=loss_mask, inpaint_mask=inp_mask,
                    masked_latents=inp_lat, model_seed=0, up_seed=5, step_seed=1235,
                    prediction_type="v_prediction", cases=cases),
               f"{OUT}/pti_loss_step_v.pt")
    print({c["name"]: c["loss"] for c in cases})


def gen_ti(R):
    """Textual-inversion phase: the reference's own `train_inversion` loop (cli_lora_pti.py:373-542)
    run for 3 steps on the tiny models, CPU fp32, with torch.optim.AdamW over the embedding table
    built as at :889-895 and a LambdaLR warm-up so that the learning rate (and the norm-decay
    lambda that follows it, :456) changes every step. Recorded: per step the gradient rows of the
    placeholder tokens, the lr in force, and the placeholder rows + whole-table sum afterwards."""
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    P = load_ref_pti(R)
    noiser = DDPMNoiser(device="cpu")

    class Sched:
        config = types.SimpleNamespace(num_train_timesteps=noiser.num_train_timesteps, prediction_type="epsilon")
        add_noise = staticmethod(noiser.add_noise)

    torch.manual_seed(0)
    unet = UNet2DConditionModel(UNetConfig.tiny())
    text = build_text_encoder(tiny=True)
    unet.requires_grad_(False)
    for prm in itertools.chain(text.text_model.encoder.parameters(), text.text_model.final_layer_norm.parameters(),
                               text.text_model.embeddings.position_embedding.parameters()):
        prm.requires_grad = False
    emb = text.get_input_embeddings()
    V, D = emb.weight.shape
    tok = [V - 2, V - 1]
    index_no_updates = torch.arange(V) != -1
    for t in tok:
        index_no_updates[t] = False
    g = torch.Generator().manual_seed(21)
    batches = []
    for _ in range(3):
        ids = torch.randint(0, V - 2, (2, 77), generator=g)
        ids[0, 5], ids[1, 9], ids[1, 10] = tok[0], tok[1], tok[0]
        batches.append({"pixel_values": torch.randn(2, 4, 8, 8, generator=g) * 0.18215, "input_ids": ids})
    base_lr, wd = 5e-3, 1e-2
    steps = []

    class Recording(torch.optim.AdamW):
        def step(self, closure=None):
            steps.append(dict(grad_rows=emb.weight.grad[tok].detach().clone(), lr=self.param_groups[0]["lr"]))
            return super().step(closure)

    opt = Recording(emb.parameters(), lr=base_lr, betas=(0.9, 0.999), eps=1e-08, weight_decay=wd)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda k: min(1.0, (k + 1) / 4))

    class Snap:                     # lr_scheduler as train_inversion uses it; snapshots the table it finds
        def step(self_inner):
            if steps:
                steps[-1].update(rows_after=emb.weight.data[tok].clone(), table_sum=float(emb.weight.data.double().sum()))
            sched.step()

        def get_last_lr(self_inner):
            return sched.get_last_lr()

    table0_rows = emb.weight.data[tok].clone()
    table0_sum = float(emb.weight.data.double().sum())
    torch.manual_seed(4321)
    import contextlib, io
    with contextlib.redirect_stdout(io.StringIO()):
        P.train_inversion(unet, None, text, batches, 3, Sched, index_no_updates, opt, 10 ** 9, tok, ["<a>", "<b>"],
                          "/nonexistent", None, Snap(), "/nonexistent", True, clip_ti_decay=True)
    steps[-1].update(rows_after=emb.weight.data[tok].clone(), table_sum=float(emb.weight.data.double().sum()))
    assert len(steps) == 3 and all("rows_after" in s for s in steps)
    torch.save(dict(model_seed=0, token_ids=tok, base_lr=base_lr, weight_decay=wd, table0_rows=table0_rows,
                    table0_sum=table0_sum, steps=steps), f"{OUT}/ti_train_inversion.pt")
    print("ti lrs", [s["lr"] for s in steps], "row norms", [s["rows_after"].norm(dim=-1).tolist() for s in steps])


def gen_tuning(R):
    """LoRA-tuning phase: the reference's own `perform_tuning` loop (cli_lora_pti.py:545-680) for 3
    steps, CPU fp32 (its `torch.cuda.amp.autocast()` is inert without CUDA), on the tiny UNet + text
    encoder injected by the reference's `inject_trainable_lora` (r=4), AdamW param groups built as
    at :958-997 (unet_lr 1e-4 / text_encoder_lr 1e-5, weight_decay_lora 1e-3), a LambdaLR linear
    decay. Every factor is set from a seeded generator first, so the trajectory depends on no
    constructor RNG. Recorded: per-step loss and lr, and every factor after the 3 steps."""
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    P = load_ref_pti(R)
    noiser = DDPMNoiser(device="cpu")

    class Sched:
        config = types.SimpleNamespace(num_train_timesteps=noiser.num_train_timesteps, prediction_type="epsilon")
        add_noise = staticmethod(noiser.add_noise)

    torch.manual_seed(0)
    unet = UNet2DConditionModel(UNetConfig.tiny())
    text = build_text_encoder(tiny=True)
    unet.requires_grad_(False)
    text.requires_grad_(False)
    up, _ = R.inject_trainable_lora(unet, r=4)
    tp, _ = R.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=4)
    gg = torch.Generator().manual_seed(6)
    sites = [m for m in list(unet.modules()) + list(text.modules()) if type(m).__name__ == "LoraInjectedLinear"]
    for m in sites:
        m.lora_down.weight.data.normal_(0, 0.25, generator=gg)
        m.lora_up.weight.data.normal_(0, 0.05, generator=gg)
    opt = torch.optim.AdamW([{"params": itertools.chain(*up), "lr": 1e-4},
                             {"params": itertools.chain(*tp), "lr": 1e-5}], weight_decay=1e-3)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda k: max(0.0, 1.0 - k / 6))
    g = torch.Generator().manual_seed(22)
    V = text.get_input_embeddings().weight.shape[0]
    batches = [{"pixel_values": torch.randn(2, 4, 8, 8, generator=g) * 0.18215,
                "input_ids": torch.randint(0, V, (2, 77), generator=g),
                "mask": (torch.rand(2, 1, 64, 64, generator=g) > 0.4).float()} for _ in range(3)]
    rec = []

    class Recording:
        def step(self_inner):
            sched.step()
            rec.append(dict(lrs=[grp["lr"] for grp in opt.param_groups]))

        def get_last_lr(self_inner):
            return sched.get_last_lr()

    real_loss_step = P.loss_step

    def spy(*a, **k):
        out = real_loss_step(*a, **k)
        rec[-1]["loss"] = float(out.detach())
        rec[-1]["kwargs"] = {kk: vv for kk, vv in k.items() if isinstance(vv, (int, float, bool))}
        return out

    P.loss_step = spy
    torch.manual_seed(999)
    import contextlib, io
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            P.perform_tuning(unet, None, text, batches, 3, Sched, opt, 10 ** 9, [], [], "/nonexistent",
                             Recording(), {"CrossAttention", "Attention", "GEGLU"}, {"CLIPAttention"}, 1.0,
                             "out", None, "/nonexistent", True)
    finally:
        P.loss_step = real_loss_step
    assert len(rec) == 3 and rec[0]["kwargs"]["t_mutliplier"] == 0.8
    keep = sorted({0, 1, 2, len(up) // 2 - 1, len(up) // 2, len(sites) - 1})      # a few sites in full ...
    factors = {i: (sites[i].lora_up.weight.detach().clone(), sites[i].lora_down.weight.detach().clone()) for i in keep}
    sums = [(float(m.lora_up.weight.double().sum()), float(m.lora_down.weight.double().sum()),     # ... all by moments
             float((m.lora_up.weight.double() ** 2).sum()), float((m.lora_down.weight.double() ** 2).sum())) for m in sites]
    for b in batches:
        b["mask"] = b["mask"].bool()
    torch.save(dict(model_seed=0, factor_seed=6, step_seed=999, n_unet_sites=len(up) // 2, batches=batches,
                    steps=rec, factors=factors, factor_moments=sums), f"{OUT}/pti_perform_tuning.pt")
    print("tuning", [(r["loss"], r["lrs"]) for r in rec], len(sites))


def gen_continue_inversion(R):
    """LoRA-tuning phase with `continue_inversion=True`: the reference's own `perform_tuning` loop
    (cli_lora_pti.py:545-620) for 3 steps, CPU fp32, with the param groups and requires_grad flags
    built as at :958-997 -- [unet LoRA (1e-4), the whole token-embedding table (continue_inversion_lr
    5e-3), text LoRA (1e-5)], one AdamW(weight_decay_lora=1e-3), encoder / final layer norm /
    position embedding frozen -- and a LambdaLR linear decay. Recorded: per-step loss and per-group
    lr, and the full table after every step."""
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    P = load_ref_pti(R)
    noiser = DDPMNoiser(device="cpu")

    class Sched:
        config = types.SimpleNamespace(num_train_timesteps=noiser.num_train_timesteps, prediction_type="epsilon")
        add_noise = staticmethod(noiser.add_noise)

    torch.manual_seed(0)
    unet = UNet2DConditionModel(UNetConfig.tiny())
    text = build_text_encoder(tiny=True)
    unet.requires_grad_(False)
    up, _ = R.inject_trainable_lora(unet, r=4)
    params = [{"params": itertools.chain(*up), "lr": 1e-4}]
    text.requires_grad_(False)
    params.append({"params": text.get_input_embeddings().parameters(), "lr": 5e-3})      # :962-971
    text.requires_grad_(True)
    for prm in itertools.chain(text.text_model.encoder.parameters(), text.text_model.final_layer_norm.parameters(),
                               text.text_model.embeddings.position_embedding.parameters()):
        prm.requires_grad = False
    tp, _ = R.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=4)
    params.append({"params": itertools.chain(*tp), "lr": 1e-5})
    gg = torch.Generator().manual_seed(6)
    sites = [m for m in list(unet.modules()) + list(text.modules()) if type(m).__name__ == "LoraInjectedLinear"]
    for m in sites:
        m.lora_down.weight.data.normal_(0, 0.25, generator=gg)
        m.lora_up.weight.data.normal_(0, 0.05, generator=gg)
    opt = torch.optim.AdamW(params, weight_decay=1e-3)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda k: max(0.0, 1.0 - k / 6))
    emb = text.get_input_embeddings()
    V = emb.weight.shape[0]
    tok = [V - 2, V - 1]
    g = torch.Generator().manual_seed(23)
    batches = []
    for _ in range(3):
        ids = torch.randint(0, V - 2, (2, 77), generator=g)
        ids[0, 4], ids[1, 6] = tok[0], tok[1]
        batches.append({"pixel_values": torch.randn(2, 4, 8, 8, generator=g) * 0.18215, "input_ids": ids})
    table0 = emb.weight.detach().clone()
    rec = []

    class Recording:                    # lr_scheduler_lora: stepped first, snapshots the table it finds
        def step(self_inner):
            if rec:
                rec[-1]["table_after"] = emb.weight.detach().clone()
            sched.step()
            rec.append(dict(lrs=[grp["lr"] for grp in opt.param_groups]))

        def get_last_lr(self_inner):
            return sched.get_last_lr()

    real_loss_step = P.loss_step

    def spy(*a, **k):
        out = real_loss_step(*a, **k)
        rec[-1]["loss"] = float(out.detach())
        rec[-1]["kwargs"] = {kk: vv for kk, vv in k.items() if isinstance(vv, (int, float, bool))}
        return out

    P.loss_step = spy
    torch.manual_seed(1001)
    import contextlib, io
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            P.perform_tuning(unet, None, text, batches, 3, Sched, opt, 10 ** 9, tok, ["<a>", "<b>"], "/nonexistent",
                             Recording(), {"CrossAttention", "Attention", "GEGLU"}, {"CLIPAttention"}, 1.0,
                             "out", None, "/nonexistent", True)
    finally:
        P.loss_step = real_loss_step
    rec[-1]["table_after"] = emb.weight.detach().clone()
    assert len(rec) == 3 and rec[0]["kwargs"]["t_mutliplier"] == 0.8
    assert not torch.equal(rec[0]["table_after"], table0)
    torch.save(dict(model_seed=0, factor_seed=6, step_seed=1001, n_unet_sites=len(up) // 2, token_ids=tok,
                    lrs0=[1e-4, 5e-3, 1e-5], weight_decay=1e-3, table0=table0, batches=batches, steps=rec),
               f"{OUT}/pti_continue_inversion.pt")
    print("continue_inversion", [(r["loss"], r["lrs"]) for r in rec])


GENERATORS = {"ops": gen_ops, "ctor_rng": gen_ctor_rng, "inject": gen_inject, "manifest": gen_manifest,
              "svd": gen_svd, "adamw": gen_adamw, "loss_step": gen_loss_step, "loss_step_v": gen_loss_step_v, "ti": gen_ti, "tuning": gen_tuning,
              "continue_inversion": gen_continue_inversion}


if __name__ == "__main__":
    # `python scripts/make_golden.py [name ...]` regenerates only the named files
    R = load_ref_lora()
    for name in (sys.argv[1:] or list(GENERATORS)):
        fn = GENERATORS[name]
        fn() if fn is gen_adamw else fn(R)
    for fn in sorted(os.listdir(OUT)):
        print(fn, os.path.getsize(f"{OUT}/{fn}"))
