"""What training from images costs: the LoRA step fed latents, the same step fed images
(StepConfig.encode_images: ingest + frozen VAE encode + posterior sample inside the captured step),
and the pattern users run without it -- an eager VAE encode outside the graph, its sample copied
into the latents step. Workloads: SD1.5 UNet + text LoRA r = 4 at 512 px, batch 1 and 4, fp32
frozen weights and fp32 VAE (the PTI trainer's weight_dtype); the same with bf16 autocast and a bf16
VAE; SD2.1 768-v (v-prediction) at batch 1. Every step is one CUDA-graph replay on inputs already on
the device; the three steps' timed windows alternate.

Prints one JSON line per workload: ms/step and images/s of each step, launches per step of this
library (eager body, the ops counter), the VAE's share of the pixels step ((pixels - latents) /
pixels), and the GPU name and power limit read in the same run.

    python scripts/bench_image_step.py [--steps 20] [--warmup 5] [--rounds 3] [--only sd15_bs1,...]
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {
    # name: (unet config, SD2 text encoder, latent grid, batch, autocast / VAE dtype, prediction type)
    "sd15_512_bs1_fp32vae": ("sd15", False, 64, 1, None, "epsilon"),
    "sd15_512_bs4_fp32vae": ("sd15", False, 64, 4, None, "epsilon"),
    "sd15_512_bs1_bf16": ("sd15", False, 64, 1, torch.bfloat16, "epsilon"),
    "sd15_512_bs4_bf16": ("sd15", False, 64, 4, torch.bfloat16, "epsilon"),
    "sd21_768v_bs1_fp32vae": ("sd21", True, 96, 1, None, "v_prediction"),
}


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        q = f"{torch.cuda.get_device_name()}, power limit unavailable ({type(e).__name__})"
    return q


def timed(fn, steps):
    """ms per call over `steps` calls, host clock around work that ends in a device synchronise."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / steps


def run(name, spec, args, dev):
    import lora_b200 as L
    from lora_b200 import ops
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.host.vae import AutoencoderKL, DiagonalGaussianDistribution, VAEConfig
    from lora_b200.train import LoraTrainStep, StepConfig
    ucfg, sd2, grid, bs, dt, pred = spec
    shape = (bs, 4, grid, grid)
    torch.manual_seed(0)
    with torch.device(dev):
        unet = UNet2DConditionModel(UNetConfig.sd21() if ucfg == "sd21" else UNetConfig.sd15())
        text = build_text_encoder(sd2=sd2)
        vae = AutoencoderKL(VAEConfig.sd())
    for m in (unet, text, vae):
        m.requires_grad_(False)
    unet = unet.to(memory_format=torch.channels_last)
    vae = vae.to(dtype=dt or torch.float32, memory_format=torch.channels_last)
    L.inject_trainable_lora(unet, r=args.rank)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=args.rank)
    g = torch.Generator(device=dev).manual_seed(1)
    for m in list(unet.modules()) + list(text.modules()):
        if type(m).__name__ == "LoraInjectedLinear":
            m.lora_up.weight.data.normal_(0.0, 0.01, generator=g)
    gen = torch.Generator().manual_seed(5)
    pixels = torch.randint(0, 256, (bs, 8 * grid, 8 * grid, 3), generator=gen, dtype=torch.uint8).to(dev)
    ids = torch.randint(0, 49406, (bs, 77), generator=gen).to(dev)

    steps, launches = {}, {}
    for kind in ("latents", "pixels"):
        u, t = (unet, text) if kind == "latents" else (copy.deepcopy(unet), copy.deepcopy(text))
        cfg = StepConfig(autocast_dtype=dt, use_cuda_graph=True, prediction_type=pred,
                         encode_images=kind == "pixels")
        st = LoraTrainStep(u, t, cfg, latent_shape=shape, device=dev, vae=vae if kind == "pixels" else None)
        st.input_ids.copy_(ids)
        if kind == "pixels":
            st.pixels.copy_(pixels)
        else:
            st.latents.normal_().mul_(0.18215)
        st._body()
        ops.LAUNCH_COUNT = 0
        st._body()
        launches[kind] = ops.LAUNCH_COUNT
        st.prepare()
        if st.graph is None:
            raise SystemExit(f"{name} {kind}: capture failed: {st.graph_error}")
        for _ in range(args.warmup):
            st.step_device()
        steps[kind] = st
    lat_step = steps["latents"]

    def eager_vae_then_latents():          # the pattern without encode_images: the VAE outside the graph
        with torch.no_grad():
            x = pixels.permute(0, 3, 1, 2).float().div(255).sub(0.5).div(0.5)
            x = x.to(vae.dtype).contiguous(memory_format=torch.channels_last)
            post = DiagonalGaussianDistribution(vae.encode(x).latent_dist.parameters)
            eps = torch.randn(post.mean.shape, device=dev, dtype=post.mean.dtype)
            lat_step.latents.copy_((post.mean + post.std * eps) * 0.18215)
        lat_step.step_device()

    for _ in range(args.warmup):
        eager_vae_then_latents()
    fns = {"latents": lat_step.step_device, "pixels": steps["pixels"].step_device,
           "eager_vae_then_latents": eager_vae_then_latents}
    ms = {k: [] for k in fns}
    for _ in range(args.rounds):
        for k, fn in fns.items():
            ms[k].append(timed(fn, args.steps))
    best = {k: min(v) for k, v in ms.items()}
    res = {"workload": f"{name}_lora_r{args.rank}_graph", "gpu": gpu_info(), "steps": args.steps,
           "warmup": args.warmup, "rounds": args.rounds,
           "ms_per_step": {k: [round(x, 3) for x in v] for k, v in ms.items()},
           "images_per_s": {k: round(1e3 * shape[0] / v, 3) for k, v in best.items()},
           "launches_per_step": launches,
           "vae_share_of_pixels_step": round((best["pixels"] - best["latents"]) / best["pixels"], 4),
           "pixels_vs_eager_vae_speedup": round(best["eager_vae_then_latents"] / best["pixels"], 4)}
    del steps, lat_step, fns
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3, help="alternated timed windows per step kind")
    ap.add_argument("--rank", type=int, default=4)
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    names = list(WORKLOADS) if args.only is None else args.only.split(",")
    unknown = [n for n in names if n not in WORKLOADS]
    if unknown:
        raise SystemExit(f"unknown workloads {unknown}: one of {list(WORKLOADS)}")
    if not torch.cuda.is_available():
        raise SystemExit("bench_image_step.py needs a CUDA device")
    import lora_b200 as L
    torch.backends.cudnn.benchmark = True
    L.set_grouping(True)
    lines = []
    for n in names:
        line = json.dumps(run(n, WORKLOADS[n], args, torch.device("cuda")))
        print(line, flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_image_step.json"), "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
