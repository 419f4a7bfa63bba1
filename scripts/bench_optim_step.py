"""Times the optimizer launch on its own: `LoraArena.step` over the SD1.5 UNet + text-encoder LoRA
arena (r = 4, the arena bench.py trains), with CUDA events around back-to-back launches (captured in
one CUDA graph and replayed) after an eager warm-up, for four flavours:

  local          lb_optim_step_fused, no loss scaling
  local_scaled   lb_optim_step_fused with fp16 loss scaling and a linear warm-up schedule
  peer           lb_optim_step_dp at world 1 (own gradient buffer as the only peer)
  peer_scaled    the same with loss scaling

The gradients are zero after the first launch; the launch's work does not depend on their values.
A step-level benchmark's spread hides a change in this one launch, hence the separate timing. The
flavours' timed windows alternate over --rounds; the median is reported.

Prints one JSON line: microseconds per launch per flavour (every round, and the median), the arena
size and block counts, and the GPU name and power limit read in the same run.

    python scripts/bench_optim_step.py [--launches 1000] [--warmup 100] [--rounds 5] [--library-tree DIR]

--library-tree imports lora_b200 from another built checkout (e.g. an earlier release) to compare
two builds with the same script.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FLAVOURS = ("local", "local_scaled", "peer", "peer_scaled")


def gpu_info():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        q = f"{torch.cuda.get_device_name()}, power limit unavailable ({type(e).__name__})"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=1000, help="back-to-back launches per timed window")
    ap.add_argument("--warmup", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--rank", type=int, default=4)
    ap.add_argument("--library-tree", default=ROOT, help="built checkout to import lora_b200 from")
    args = ap.parse_args()
    tree = os.path.abspath(args.library_tree)
    sys.path.insert(0, tree)
    import torch
    import lora_b200 as L
    from lora_b200.arena import LoraArena, LrSchedule
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    if os.path.dirname(os.path.abspath(L.__file__)) != os.path.join(tree, "lora_b200"):
        raise SystemExit(f"lora_b200 was imported from {L.__file__}, not from {tree}")
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim_step.py needs a CUDA device")
    dev = torch.device("cuda")
    torch.manual_seed(0)
    with torch.device(dev):
        unet = UNet2DConditionModel(UNetConfig.sd15())
        text = build_text_encoder()
    unet.requires_grad_(False)
    text.requires_grad_(False)
    unet, text = unet.to(torch.bfloat16), text.to(torch.bfloat16)
    L.inject_trainable_lora(unet, r=args.rank)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=args.rank)
    g = torch.Generator(device=dev).manual_seed(1)
    for m in list(unet.modules()) + list(text.modules()):
        if type(m).__name__ == "LoraInjectedLinear":
            m.lora_up.weight.data.normal_(0.0, 0.01, generator=g)

    schedule = LrSchedule("linear", 10, 1 << 20, (0, 1))
    steps = {}
    for name in FLAVOURS:
        # one arena per flavour over the same sites: each step touches only its own buffers
        arena = LoraArena([(unet, 1e-4), (text, 5e-5)], compute_dtype=torch.bfloat16, device=dev)
        if name.startswith("peer"):
            arena._dp_flags = torch.zeros(2, device=dev, dtype=torch.int32)
            arena._dp_epoch = torch.zeros(1, device=dev, dtype=torch.int32)
            arena.gsum = torch.zeros_like(arena.g)
            one = ctypes.c_void_p * 1
            arena._dp = (one(arena.g.data_ptr()), one(arena._dp_flags.data_ptr()), 1, 0)
        scaled = name.endswith("scaled")
        if scaled:
            arena.enable_loss_scaling(init_scale=2.0 ** 16, growth_interval=2000)
        arena.g.normal_(0.0, 1e-3)
        steps[name] = (lambda a=arena, s=scaled: a.step(0.9, 0.999, 1e-8, 1e-2, 1.0, world_size=1,
                                                       schedule=schedule if s else None))
    # the launches are captured into one graph per flavour: replayed, they run back to back without
    # the host-side cost of arena.step (ctypes call, operand-cache bookkeeping) in the timed window
    graphs = {}
    for name in FLAVOURS:
        for _ in range(args.warmup):
            steps[name]()
        torch.cuda.synchronize()
        graphs[name] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[name]):
            for _ in range(args.launches):
                steps[name]()
        graphs[name].replay()
    torch.cuda.synchronize()

    us = {name: [] for name in FLAVOURS}
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for name in FLAVOURS:
            start.record()
            graphs[name].replay()
            stop.record()
            stop.synchronize()
            us[name].append(1e3 * start.elapsed_time(stop) / args.launches)
    n = arena.n
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    result = {"workload": f"sd15_unet_text_lora_r{args.rank}_optimizer_launch", "library": tree,
              "gpu": gpu_info(), "arena_elements": n, "launches": args.launches, "warmup": args.warmup,
              "rounds": args.rounds,
              "blocks": {"local": min((n + 255) // 256, sms), "peer": min((n // 4 + 255) // 256, sms)},
              "us_per_launch": {k: [round(x, 3) for x in v] for k, v in us.items()},
              "us_per_launch_median": {k: round(statistics.median(v), 3) for k, v in us.items()}}
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
