"""The SDXL LoRA training step: UNetConfig.sdxl() + both SDXL text encoders, LoRA r = 4 on the 630 UNet
and 176 text sites, 1024 px (128 x 128 latents), batch 1, fp32 frozen weights under bf16 autocast (the
accelerate configuration of diffusers' train_dreambooth_lora_sdxl.py), grouping on, one CUDA-graph
replay per step (lora_b200.train.LoraXLTrainStep).

Prints one JSON line: ms/step and images/s over device-synchronised steps after warm-up, launches per
step (eager, the ops counter), the peak memory of the steady-state step (weights, arena and the graph's
pool), the same with StepConfig.gradient_checkpointing, the oracle's step (oracle/ref_step_xl.py, torch
eager on the same models and weights) as a comparator, and the GPU name and power limit read in the same
run.

    python scripts/bench_sdxl_step.py [--steps 10] [--warmup 3] [--res 1024] [--ref-steps 3] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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


def _tie(dst, src):
    """dst (same architecture, built on the meta device) uses src's parameters and buffers."""
    for (_, md), (_, ms) in zip(dst.named_modules(), src.named_modules()):
        for k in ms._parameters:
            md._parameters[k] = ms._parameters[k]
        for k in ms._buffers:
            md._buffers[k] = ms._buffers[k]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--res", type=int, default=1024)
    ap.add_argument("--rank", type=int, default=4)
    ap.add_argument("--ref-steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sdxl_step.py needs a CUDA device")
    import lora_b200 as L
    from lora_b200 import ops
    from lora_b200.host.clip import build_sdxl_text_encoders
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.train import LoraXLTrainStep, StepConfig
    from oracle.ref_modules import ref_inject
    from oracle.ref_step_xl import RefXLStep
    torch.backends.cudnn.benchmark = True
    dev, dt = torch.device("cuda"), torch.bfloat16
    lat_hw = args.res // 8
    shape = (1, 4, lat_hw, lat_hw)
    torch.manual_seed(0)
    with torch.device(dev):
        unet = UNet2DConditionModel(UNetConfig.sdxl())
        te1, te2 = build_sdxl_text_encoders()
    unet = unet.to(memory_format=torch.channels_last)
    models = (unet, te1, te2)
    for m in models:
        m.requires_grad_(False)
    with torch.device("meta"):
        refs = (UNet2DConditionModel(UNetConfig.sdxl()),) + tuple(build_sdxl_text_encoders())
    for d, s in zip(refs, models):
        _tie(d, s)                          # the oracle runs on the same frozen weights
    L.inject_trainable_lora(unet, r=args.rank)
    for te in (te1, te2):
        L.inject_trainable_lora(te, target_replace_module={"CLIPAttention"}, r=args.rank)
    g = torch.Generator(device=dev).manual_seed(1)
    for mdl in models:
        for m in mdl.modules():
            if type(m).__name__ == "LoraInjectedLinear":
                m.lora_up.weight.data.normal_(0.0, 0.01, generator=g)
    gen = torch.Generator().manual_seed(5)
    lat = (torch.randn(shape, generator=gen) * 0.13025).to(dev)
    ids = torch.randint(0, 49406, (1, 77), generator=gen)
    ids[:, 20:] = 49407                     # eos-padded prompts
    ids = ids.to(dev)

    def run(ckpt):
        L.set_grouping(True)
        cfg = StepConfig(use_cuda_graph=True, autocast_dtype=dt, gradient_checkpointing=ckpt)
        st = LoraXLTrainStep(unet, te1, te2, cfg, latent_shape=shape, device=dev)
        st.latents.copy_(lat); st.input_ids.copy_(ids); st.input_ids_2.copy_(ids)
        st._body()
        ops.LAUNCH_COUNT = 0
        st._body()
        launches = ops.LAUNCH_COUNT
        st.prepare()
        if st.graph is None:
            raise SystemExit(f"capture failed: {st.graph_error}")
        for _ in range(args.warmup):
            st.step_device()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        ms = timed(st.step_device, args.steps)
        peak = torch.cuda.max_memory_allocated() / 2 ** 20
        out = {"ms_per_step": round(ms, 3), "images_per_s": round(1e3 / ms, 3), "launches_per_step": launches,
               "peak_mib": round(peak), "loss": float(st.loss), "graphs_per_step": 1 + (st.graph_update is not None)}
        L.set_grouping(False)
        unet.disable_gradient_checkpointing()
        for te in (te1, te2):
            te.gradient_checkpointing_disable()
        del st
        torch.cuda.empty_cache()
        return out

    plain = run(False)
    ckpt = run(True)

    us = ref_inject(refs[0], {"CrossAttention", "Attention", "GEGLU"}, r=args.rank)
    ts1 = ref_inject(refs[1], {"CLIPAttention"}, r=args.rank)
    ts2 = ref_inject(refs[2], {"CLIPAttention"}, r=args.rank)
    ref = RefXLStep(*refs, DDPMNoiser(device=dev), us, ts1, ts2, autocast_dtype=dt)

    def ref_step():
        ref.step(lat, ids, input_ids_2=ids)

    for _ in range(2):
        ref_step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms_ref = timed(ref_step, args.ref_steps)
    peak_ref = torch.cuda.max_memory_allocated() / 2 ** 20

    result = {"workload": f"sdxl_lora_r{args.rank}_{args.res}px_bs1_bf16_autocast_graph",
              "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup, **plain,
              "gradient_checkpointing": ckpt,
              "reference_eager_ms_per_step": round(ms_ref, 3), "reference_eager_images_per_s": round(1e3 / ms_ref, 3),
              "reference_eager_peak_mib": round(peak_ref), "speedup_vs_reference": round(ms_ref / plain["ms_per_step"], 3)}
    line = json.dumps(result)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_sdxl_step.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
