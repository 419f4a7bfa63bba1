"""Sampling throughput: LoraSampler's graph replay, its eager path and the pipeline-style oracle loop
(oracle/sample_ref.py), alternated in one process, on full-size host models with LoRA r=4 on the UNet
and the text encoder, bf16 autocast, guidance 7:
  SD1.5 512 px, Euler-ancestral, 50 steps, batch 1 and 4;  SD2.1 768-v, DDIM, 50 steps, batch 1.
Prints per workload: s/image and ms per denoising step, the decode's share of a graph-replayed call,
liblora_b200 launches per denoising step (ops counter), peak memory, and the GPU's name and power limit.
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


def _models(sd2: bool):
    import lora_b200 as L
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    from oracle.ref_modules import ref_inject
    import copy
    torch.manual_seed(0)
    with torch.device("cuda"):
        unet = UNet2DConditionModel(UNetConfig.sd21() if sd2 else UNetConfig())
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


def run(name, sd2, B, res, sched, pred, n, reps):
    import lora_b200 as L
    from lora_b200 import ops
    from lora_b200.sample import LoraSampler, SamplerConfig
    from oracle import sample_ref as R
    unet, text, vae, unet_r, text_r = _models(sd2)
    L.set_grouping(True)
    lat = (B, 4, res // 8, res // 8)
    cfg = dict(scheduler=sched, prediction_type=pred, num_inference_steps=n, max_steps=n, guidance_scale=7.0,
               autocast_dtype=torch.bfloat16)
    sg = LoraSampler(unet, text, vae, SamplerConfig(**cfg), latent_shape=lat)
    se = LoraSampler(unet, text, vae, SamplerConfig(use_cuda_graph=False, **cfg), latent_shape=lat)
    ids = torch.randint(0, text.config.vocab_size, (B, 77), device="cuda")
    neg = torch.randint(0, text.config.vocab_size, (B, 77), device="cuda")
    torch.cuda.reset_peak_memory_stats()
    sg.prepare()
    sg.sample(ids, neg)
    se.sample(ids, neg)
    noise = sg.noise[:n + 1].clone()
    oracle = lambda: R.sample(unet_r, text_r, vae, R.make_scheduler(sched, pred), n, ids, neg, noise, 7.0,  # noqa: E731
                              dtype=torch.float32, autocast_dtype=torch.bfloat16)
    oracle()
    t = {"graph": [], "eager": [], "oracle": []}
    for _ in range(reps):                      # alternated: the three paths see the same machine state
        t["graph"].append(_time(lambda: sg.sample(ids, neg), 1))
        t["eager"].append(_time(lambda: se.sample(ids, neg), 1))
        t["oracle"].append(_time(oracle, 1))
    gc = sg._graphs[2][2]
    decode = _time(gc.replay, 3)
    with torch.no_grad():
        unet.eval()
        c0 = ops.LAUNCH_COUNT
        se._body_b(2)
        launches = ops.LAUNCH_COUNT - c0
        unet.train()
    med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
    return {"workload": name, "batch": B, "steps": n,
            **{f"{k}_s_per_image": round(v / B, 4) for k, v in med.items()},
            **{f"{k}_ms_per_step": round(1e3 * v / n, 3) for k, v in med.items()},
            "decode_share_graph": round(decode / med["graph"], 4),
            "launches_per_step": launches,
            "peak_mib": round(torch.cuda.max_memory_allocated() / 2 ** 20)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--only", default=None, help="run one workload (sd15_b1, sd15_b4, sd21_768v)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample.py needs a CUDA device")
    name, power = _gpu()
    work = [("sd15_b1", False, 1, 512, "euler_ancestral", "epsilon"),
            ("sd15_b4", False, 4, 512, "euler_ancestral", "epsilon"),
            ("sd21_768v", True, 1, 768, "ddim", "v_prediction")]
    for w in work:
        if a.only and w[0] != a.only:
            continue
        r = run(*w, a.steps, a.reps)
        r.update(gpu=name, power_limit=power)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
