"""Gradient checkpointing (StepConfig.gradient_checkpointing) against the plain step: peak memory,
time per step and launches per step, and the largest batch that fits at 768 px either way.

Per configuration both engines are built in one process (bf16 weights, UNet + text-encoder LoRA,
grouped launches on, one CUDA-graph replay per step) and timed alternately, `--reps` rounds of
`--steps` replays each; ms/step is the median round, host clock around device-synchronised replays.
Peak memory is torch.cuda.max_memory_allocated over one eager step, less what was allocated before
that engine's models were built (the other engine of the pair is resident then): weights, arena and
activations of one engine. A replay allocates nothing, so the eager step stands for it. Launches per
step count the lora_b200 kernels of that eager step; `wgrad_launches` are its batched weight-gradient launches
(lb_lora_wgrad_batch) and `wgrad_items` the reductions they carry, so ceil(items / 24) is what one
end-of-backward flush takes. A checkpointed step is also counted with defer_wgrad=False (every
reduction launched by its site's backward at once).

The largest batch: peaks at two batch sizes give bytes per sample; the predicted largest batch
is run eagerly, then one more (an allocator OutOfMemoryError there is the expected outcome).

Prints one JSON line per measurement and the GPU's name and power limit read in the same run.

    python scripts/bench_checkpointing.py [--steps 10] [--reps 3] [--out DIR] [--dry-run]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (name, model, LoRA rank, resolution px, batch, prediction type)
CONFIGS = [
    ("sd15_r4_512_bs1", "sd15", 4, 512, 1, "epsilon"),
    ("sd15_r4_512_bs8", "sd15", 4, 512, 8, "epsilon"),
    ("sd15_r16_768_bs4", "sd15", 16, 768, 4, "epsilon"),
    ("sd21_768v_r4_bs4", "sd21", 4, 768, 4, "v_prediction"),
]
# largest batch at 768 px: (name, model, rank, prediction, the two probe batches)
MAX_BATCH = [
    ("sd15_r16_768", "sd15", 16, "epsilon", (2, 4)),
    ("sd21_768v_r4", "sd21", 4, "v_prediction", (2, 4)),
]
BATCH_CAP = 64       # largest batch tried: keeps every site's row count far inside the kernels' int32 indexing


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        q = f"{torch.cuda.get_device_name()}, power limit unavailable ({type(e).__name__})"
    return q


def latent_shape(res, batch):
    if res % 64:
        raise ValueError(f"resolution {res}: a multiple of 64 (three 2x down-samplings of res / 8)")
    return (batch, 4, res // 8, res // 8)


def build(model, rank, res, batch, prediction, ckpt, graph=True, seed=0):
    import lora_b200 as L
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.train import LoraTrainStep, StepConfig
    dev, dt = torch.device("cuda"), torch.bfloat16
    torch.manual_seed(seed)
    with torch.device(dev):
        unet = UNet2DConditionModel(UNetConfig.sd21() if model == "sd21" else UNetConfig.sd15())
        text = build_text_encoder(sd2=model == "sd21")
    unet.requires_grad_(False); text.requires_grad_(False)
    unet, text = unet.to(dt).to(memory_format=torch.channels_last), text.to(dt)
    L.inject_trainable_lora(unet, r=rank)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=rank)
    g = torch.Generator(device=dev).manual_seed(1)
    for m in list(unet.modules()) + list(text.modules()):
        if type(m).__name__ == "LoraInjectedLinear":
            m.lora_up.weight.data.normal_(0.0, 0.01, generator=g)
    cfg = StepConfig(compute_dtype=dt, use_cuda_graph=graph, prediction_type=prediction, gradient_checkpointing=ckpt)
    shape = latent_shape(res, batch)
    st = LoraTrainStep(unet, text, cfg, latent_shape=shape, device=dev)
    gen = torch.Generator().manual_seed(5)
    st.latents.copy_(torch.randn(shape, generator=gen) * 0.18215)
    st.input_ids.copy_(torch.randint(0, 49406, (batch, 77), generator=gen))
    return st


def eager_step_stats(st, base=0):
    """(peak bytes above `base`, launches, batched wgrad launches, queued wgrad reductions) of one eager step."""
    from lora_b200 import ops
    wg = {"launches": 0, "items": 0}
    real = ops._wgrad_launch

    def counted(dtype, items):
        n = real(dtype, items)
        wg["launches"] += n
        wg["items"] += len(items)
        return n

    ops._wgrad_launch = counted
    try:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        ops.LAUNCH_COUNT = 0
        st._body()
        torch.cuda.synchronize()
    finally:
        ops._wgrad_launch = real
    return torch.cuda.max_memory_allocated() - base, ops.LAUNCH_COUNT, wg["launches"], wg["items"]


def timed(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / steps


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(os.path.join(out, "bench_checkpointing.jsonl"), "a") as fh:
            fh.write(line + "\n")


def compare(cfg, args):
    import lora_b200 as L
    name, model, rank, res, batch, pred = cfg
    L.set_grouping(True)
    engines, rec = {}, {"config": name, "latent_shape": list(latent_shape(res, batch)), "rank": rank}
    for ckpt in (False, True):
        key = "checkpointed" if ckpt else "plain"
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        st = build(model, rank, res, batch, pred, ckpt)
        st._body()                                   # first call: cuDNN / allocator warm-up
        peak, launches, wgl, wgi = eager_step_stats(st, base)
        rec[key] = {"peak_mib": round(peak / 2 ** 20, 1), "launches_per_step": launches,
                    "wgrad_launches": wgl, "wgrad_items": wgi, "ceil_items_over_24": math.ceil(wgi / 24)}
        st.prepare()
        if st.graph is None:
            raise SystemExit(f"{name} {key}: capture failed: {st.graph_error}")
        for _ in range(args.warmup):
            st.step_device()
        engines[key] = st
    rounds = {k: [] for k in engines}
    for _ in range(args.reps):                      # alternate the two engines
        for k, st in engines.items():
            rounds[k].append(timed(st.step_device, args.steps))
    for k in engines:
        rec[k]["ms_per_step"] = round(statistics.median(rounds[k]), 3)
        rec[k]["ms_rounds"] = [round(v, 3) for v in rounds[k]]
    st = None
    del engines
    torch.cuda.empty_cache()
    # the checkpointed step with every reduction launched at once (defer_wgrad=False)
    base = torch.cuda.memory_allocated()
    st = build(model, rank, res, batch, pred, True, graph=False)
    st.cfg.defer_wgrad = False
    st._body()
    peak, launches, _, _ = eager_step_stats(st, base)
    rec["checkpointed_immediate_wgrad"] = {"peak_mib": round(peak / 2 ** 20, 1), "launches_per_step": launches}
    del st
    torch.cuda.empty_cache()
    L.set_grouping(False)
    return rec


def fits(model, rank, batch, pred, ckpt):
    """Peak bytes of one eager step at `batch` (768 px), or None on an allocator OutOfMemoryError."""
    st = None
    try:
        st = build(model, rank, 768, batch, pred, ckpt, graph=False)
        st._body()
        torch.cuda.synchronize()
        return eager_step_stats(st)[0]
    except torch.cuda.OutOfMemoryError:
        return None
    finally:
        del st
        import gc
        gc.collect()
        torch.cuda.empty_cache()


def max_batch(spec):
    import lora_b200 as L
    name, model, rank, pred, (b0, b1) = spec
    L.set_grouping(True)
    total = torch.cuda.get_device_properties(0).total_memory
    rec = {"config": name, "res": 768, "device_bytes": total}
    for ckpt in (False, True):
        key = "checkpointed" if ckpt else "plain"
        p0, p1 = fits(model, rank, b0, pred, ckpt), fits(model, rank, b1, pred, ckpt)
        if p0 is None or p1 is None:
            rec[key] = {"probe_oom": [b0 if p0 is None else None, b1 if p1 is None else None]}
            continue
        per = (p1 - p0) / (b1 - b0)
        pred_b = max(1, min(BATCH_CAP, int((0.98 * total - (p0 - per * b0)) // per)))
        largest, tried = None, {}
        b = pred_b
        while b >= 1:                              # walk down until one fits
            tried[b] = fits(model, rank, b, pred, ckpt)
            if tried[b] is not None:
                largest = b
                break
            b -= max(1, b // 16)
        if largest is not None and largest < BATCH_CAP:
            tried[largest + 1] = fits(model, rank, largest + 1, pred, ckpt)
            if tried[largest + 1] is not None:
                largest += 1                       # the prediction was conservative by one
        rec[key] = {"mib_per_sample": round(per / 2 ** 20, 1), "predicted": pred_b, "largest_fitting": largest,
                    "capped_at": BATCH_CAP if largest == BATCH_CAP else None,
                    "tried": {str(k): (None if v is None else round(v / 2 ** 20, 1)) for k, v in tried.items()}}
    L.set_grouping(False)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--configs", default=",".join(c[0] for c in CONFIGS))
    ap.add_argument("--max-batch", default=",".join(m[0] for m in MAX_BATCH),
                    help="configurations of the largest-batch search ('' for none)")
    ap.add_argument("--out", default=None)
    ap.add_argument("--dry-run", action="store_true", help="print the plan (shapes) and stop before any CUDA call")
    args = ap.parse_args()
    chosen = [c for c in CONFIGS if c[0] in args.configs.split(",")]
    searches = [m for m in MAX_BATCH if m[0] in args.max_batch.split(",")]
    plan = {"configs": [{"config": c[0], "latent_shape": list(latent_shape(c[3], c[4])), "rank": c[2],
                         "prediction": c[5]} for c in chosen],
            "max_batch": [{"config": m[0], "probe_batches": list(m[4]), "cap": BATCH_CAP} for m in searches],
            "steps": args.steps, "reps": args.reps}
    if args.dry_run:
        print(json.dumps(plan))
        return
    if not torch.cuda.is_available():
        raise SystemExit("bench_checkpointing.py needs a CUDA device")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    torch.backends.cudnn.benchmark = True
    emit({"gpu": gpu_info(), **plan}, args.out)
    for c in chosen:
        emit(compare(c, args), args.out)
    for m in searches:
        emit(max_batch(m), args.out)
    emit({"gpu": gpu_info(), "done": True}, args.out)


if __name__ == "__main__":
    main()
