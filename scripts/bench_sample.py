"""Sampling throughput: LoraSampler's graph replay, its eager path and the pipeline-style oracle loop
(oracle/sample_ref.py), alternated in one process, on full-size host models with LoRA r=4 on the UNet
and the text encoder, bf16 autocast, guidance 7:
  SD1.5 512 px, Euler-ancestral, 50 steps, batch 1 and 4;  SD2.1 768-v, DDIM, 50 steps, batch 1;
  SD1.5 512 px img2img, Euler-ancestral, 50 steps at strength 0.75 (37 steps run), batch 1;
  SD1.5-inpainting shape (a 9-channel UNet), 512 px, Euler-ancestral, 50 steps, batch 1;
  DPM-Solver++(2M): SD1.5 512 px 20 and 25 steps, SD2.1 768-v 25 steps, SD1.5 512 px img2img 25 steps at
  strength 0.75 (18 steps run), batch 1.
Prints per workload: s/image and ms per denoising step (the call's time over its steps), the time of
one replay of the denoising-step graph alone, the decode's share of a graph-replayed call,
liblora_b200 launches per denoising step (ops counter), peak memory, and the GPU's name and power limit.
The img2img and inpainting workloads also print the share of graph A (text encoder, image ingest, VAE
encoder and lb_sample_init) in a graph-replayed call, and the denoising steps run. The DPM-Solver++
workloads also print the peak memory once the same graph sampler holds the captures of both scheduler
families (one Euler-ancestral call after the timed ones).
Weights are random: the timings do not depend on them."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _gpu():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
    except Exception:
        name, power = torch.cuda.get_device_name(), "unknown"
    return name, power


def _models(sd2: bool, in_channels: int = 4):
    import lora_b200 as L
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    from oracle.ref_modules import ref_inject
    import copy
    torch.manual_seed(0)
    with torch.device("cuda"):
        ucfg = UNetConfig.sd21() if sd2 else UNetConfig()
        ucfg.in_channels = in_channels
        unet = UNet2DConditionModel(ucfg)
        text = build_text_encoder(sd2=sd2)
        vae = AutoencoderKL(VAEConfig.sd(), with_decoder=True)
    for m in (unet, text, vae):
        m.requires_grad_(False)
    unet = unet.to(memory_format=torch.channels_last)
    vae = vae.to(torch.bfloat16).to(memory_format=torch.channels_last)
    unet_r, text_r = copy.deepcopy(unet), copy.deepcopy(text)
    L.inject_trainable_lora(unet, r=4)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=4)
    ref_inject(unet_r, {"CrossAttention", "Attention", "GEGLU"}, r=4)
    ref_inject(text_r, {"CLIPAttention"}, r=4)
    return unet, text, vae, unet_r, text_r


def _time(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def _ref_scheduler(mod, sched, pred):
    """The oracle scheduler of that name: oracle/sample_dpm_ref.py's DPM-Solver++, otherwise oracle module
    `mod`'s (sample_ref or sample_image_ref)."""
    from oracle.sample_dpm_ref import RefDPMSolverMultistep
    return RefDPMSolverMultistep(pred) if sched == "dpmsolver_multistep" else mod.make_scheduler(sched, pred)


def run(name, sd2, B, res, sched, pred, n, reps, task="txt2img", strength=0.75):
    import lora_b200 as L
    from lora_b200 import ops
    from lora_b200.host import schedulers
    from lora_b200.sample import LoraSampler, SamplerConfig
    from oracle import sample_image_ref as RI
    from oracle import sample_ref as R
    unet, text, vae, unet_r, text_r = _models(sd2, 9 if task == "inpaint" else 4)
    L.set_grouping(True)
    lat = (B, 4, res // 8, res // 8)
    cfg = dict(scheduler=sched, prediction_type=pred, num_inference_steps=n, max_steps=n, guidance_scale=7.0,
               autocast_dtype=torch.bfloat16, task=task, strength=strength)
    sg = LoraSampler(unet, text, vae, SamplerConfig(**cfg), latent_shape=lat)
    se = LoraSampler(unet, text, vae, SamplerConfig(use_cuda_graph=False, **cfg), latent_shape=lat)
    ids = torch.randint(0, text.config.vocab_size, (B, 77), device="cuda")
    neg = torch.randint(0, text.config.vocab_size, (B, 77), device="cuda")
    g = torch.Generator().manual_seed(0)
    image = torch.randint(0, 256, (B, res, res, 3), generator=g, dtype=torch.uint8).cuda()
    mask = torch.zeros(B, res, res, dtype=torch.uint8)
    mask[:, res // 4:3 * res // 4, res // 4:3 * res // 4] = 255
    mask = mask.cuda()
    extra = {"txt2img": {}, "img2img": dict(image=image), "inpaint": dict(image=image, mask_image=mask)}[task]
    k = n - schedulers.t_start(n, strength) if task == "img2img" else n        # denoising steps run
    torch.cuda.reset_peak_memory_stats()
    sg.prepare()
    sg.sample(ids, neg, **extra)
    se.sample(ids, neg, **extra)
    noise = sg.noise[:k + 1].clone()
    if task == "txt2img":
        oracle = lambda: R.sample(unet_r, text_r, vae, _ref_scheduler(R, sched, pred), n, ids, neg, noise, 7.0,  # noqa: E731
                                  dtype=torch.float32, autocast_dtype=torch.bfloat16)
    elif task == "img2img":
        peps = sg.posterior_noise.clone()
        oracle = lambda: RI.sample_img2img(unet_r, text_r, vae, _ref_scheduler(RI, sched, pred), n, strength, ids,  # noqa: E731
                                           neg, image, noise, peps, 7.0, dtype=torch.float32,
                                           autocast_dtype=torch.bfloat16)
    else:
        peps = sg.posterior_noise.clone()
        oracle = lambda: RI.sample_inpaint(unet_r, text_r, vae, _ref_scheduler(RI, sched, pred), n, ids, neg,  # noqa: E731
                                           image, mask, noise, peps, 7.0, dtype=torch.float32,
                                           autocast_dtype=torch.bfloat16)
    oracle()
    t = {"graph": [], "eager": [], "oracle": []}
    for _ in range(reps):                      # alternated: the three paths see the same machine state
        t["graph"].append(_time(lambda: sg.sample(ids, neg, **extra), 1))
        t["eager"].append(_time(lambda: se.sample(ids, neg, **extra), 1))
        t["oracle"].append(_time(oracle, 1))
    family = schedulers.family(sched)
    ga, gb, gc = sg._graphs[(2, family)]
    decode = _time(gc.replay, 3)
    graph_a = _time(ga.replay, 3)
    # graph B alone (the UNet forward and the one step launch), replayed as many times as a call does; the
    # step index runs past the table, whose last row the kernel then repeats: the same work per replay
    denoise_step = _time(gb.replay, k)
    with torch.no_grad():
        unet.eval()
        c0 = ops.LAUNCH_COUNT
        se._body_b(2, family)
        launches = ops.LAUNCH_COUNT - c0
        unet.train()
    med = {key: sorted(v)[len(v) // 2] for key, v in t.items()}
    out = {"workload": name, "batch": B, "steps": n,
           **{f"{key}_s_per_image": round(v / B, 4) for key, v in med.items()},
           **{f"{key}_ms_per_step": round(1e3 * v / k, 3) for key, v in med.items()},
           "graph_b_ms_per_replay": round(1e3 * denoise_step, 3),
           "decode_share_graph": round(decode / med["graph"], 4),
           "launches_per_step": launches,
           "peak_mib": round(torch.cuda.max_memory_allocated() / 2 ** 20)}
    if family == "multistep":
        out["scheduler"] = sched
        sg.sample(ids, neg, scheduler="euler_ancestral", **extra)          # the other family's captures
        torch.cuda.synchronize()
        out.update(captures=sg.captures, peak_mib_both_families=round(torch.cuda.max_memory_allocated() / 2 ** 20))
    if task != "txt2img":
        out.update(task=task, denoising_steps=k, graph_a_share_graph=round(graph_a / med["graph"], 4))
        if task == "img2img":
            out["strength"] = strength
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--only", default=None,
                    help="comma-separated workloads (sd15_b1, sd15_b4, sd21_768v, sd15_img2img, sd15_inpaint, "
                         "sd15_dpm20, sd15_dpm25, sd21_768v_dpm25, sd15_img2img_dpm25)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample.py needs a CUDA device")
    name, power = _gpu()
    work = [("sd15_b1", False, 1, 512, "euler_ancestral", "epsilon"),
            ("sd15_b4", False, 4, 512, "euler_ancestral", "epsilon"),
            ("sd21_768v", True, 1, 768, "ddim", "v_prediction"),
            ("sd15_img2img", False, 1, 512, "euler_ancestral", "epsilon", "img2img"),
            ("sd15_inpaint", False, 1, 512, "euler_ancestral", "epsilon", "inpaint"),
            ("sd15_dpm20", False, 1, 512, "dpmsolver_multistep", "epsilon", "txt2img", 20),
            ("sd15_dpm25", False, 1, 512, "dpmsolver_multistep", "epsilon", "txt2img", 25),
            ("sd21_768v_dpm25", True, 1, 768, "dpmsolver_multistep", "v_prediction", "txt2img", 25),
            ("sd15_img2img_dpm25", False, 1, 512, "dpmsolver_multistep", "epsilon", "img2img", 25)]
    only = set(a.only.split(",")) if a.only else None
    for w in work:
        if only and w[0] not in only:
            continue
        steps = w[7] if len(w) > 7 else a.steps           # the DPM-Solver++ rows fix their step counts
        r = run(*w[:6], steps, a.reps, *w[6:7])
        r.update(gpu=name, power_limit=power)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
