"""The SD 2.x LoRA training step: UNetConfig.sd21() + the OpenCLIP-H text encoder, UNet and text LoRA
r = 4, batch 1, bf16 weights, one CUDA-graph replay per step (lora_b200.train.LoraTrainStep).
Default: stable-diffusion-2-1 768-v (96 x 96 latents, prediction_type "v_prediction");
`--res 512 --prediction epsilon` is the 2-1-base shape.

Prints one JSON line: images/s and ms/step over device-synchronised steps after warm-up, launches
per step (eager, the ops counter), the oracle's reference step (oracle/ref_step_v.py, torch eager on
the same bf16 models) on the same GPU as a comparator, and the GPU name and power limit read in the
same run.

    python scripts/bench_sd2_step.py [--steps 20] [--warmup 5] [--res 768] [--prediction v_prediction]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--res", type=int, default=768)
    ap.add_argument("--prediction", default="v_prediction", choices=("epsilon", "v_prediction"))
    ap.add_argument("--rank", type=int, default=4)
    ap.add_argument("--ref-steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sd2_step.py needs a CUDA device")
    import lora_b200 as L
    from lora_b200 import ops
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.train import LoraTrainStep, StepConfig
    from oracle.ref_modules import ref_inject
    from oracle.ref_step_v import RefDreamboothStepV as RefDreamboothStep
    torch.backends.cudnn.benchmark = True
    dev, dt = torch.device("cuda"), torch.bfloat16
    lat_hw = args.res // 8
    shape = (1, 4, lat_hw, lat_hw)
    torch.manual_seed(0)
    with torch.device(dev):
        unet = UNet2DConditionModel(UNetConfig.sd21())
        text = build_text_encoder(sd2=True)
    unet.requires_grad_(False); text.requires_grad_(False)
    unet, text = unet.to(dt).to(memory_format=torch.channels_last), text.to(dt)
    unet_r, text_r = copy.deepcopy(unet), copy.deepcopy(text)
    L.inject_trainable_lora(unet, r=args.rank)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=args.rank)
    g = torch.Generator(device=dev).manual_seed(1)
    for m in list(unet.modules()) + list(text.modules()):
        if type(m).__name__ == "LoraInjectedLinear":
            m.lora_up.weight.data.normal_(0.0, 0.01, generator=g)
    gen = torch.Generator().manual_seed(5)
    lat = (torch.randn(shape, generator=gen) * 0.18215).to(dev)
    ids = torch.randint(0, 49406, (1, 77), generator=gen).to(dev)

    L.set_grouping(True)
    cfg = StepConfig(compute_dtype=dt, use_cuda_graph=True, prediction_type=args.prediction)
    st = LoraTrainStep(unet, text, cfg, latent_shape=shape, device=dev)
    st.latents.copy_(lat); st.input_ids.copy_(ids)
    st._body()
    ops.LAUNCH_COUNT = 0
    st._body()
    launches = ops.LAUNCH_COUNT
    st.prepare()
    if st.graph is None:
        raise SystemExit(f"capture failed: {st.graph_error}")
    for _ in range(args.warmup):
        st.step_device()
    ms = timed(st.step_device, args.steps)
    loss = float(st.loss)
    L.set_grouping(False)
    del st
    torch.cuda.empty_cache()

    us = ref_inject(unet_r, {"CrossAttention", "Attention", "GEGLU"}, r=args.rank)
    ts = ref_inject(text_r, {"CLIPAttention"}, r=args.rank)
    ref = RefDreamboothStep(unet_r, text_r, DDPMNoiser(device=dev), us, ts)

    def ref_step():
        ref.step(lat, ids, prediction_type=args.prediction)

    for _ in range(2):
        ref_step()
    ms_ref = timed(ref_step, args.ref_steps)

    result = {"workload": f"sd21_lora_r{args.rank}_{args.res}px_{args.prediction}_bs1_bf16_graph",
              "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup,
              "ms_per_step": round(ms, 3), "images_per_s": round(1e3 / ms, 3), "launches_per_step": launches,
              "loss": loss, "reference_eager_ms_per_step": round(ms_ref, 3),
              "reference_eager_images_per_s": round(1e3 / ms_ref, 3), "speedup_vs_reference": round(ms_ref / ms, 3)}
    line = json.dumps(result)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_sd2_step.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
