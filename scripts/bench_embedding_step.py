"""Cost of training the token-embedding table with the LoRA factors (lora_b200.train.LoraEmbeddingStep)
against the plain LoRA step, on the flagship workload: SD1.5 UNet + CLIP text encoder at 512 px, bf16,
batch 1, LoRA r = 1 and r = 4, two placeholder tokens, prompt ids drawn from a fixed pool of 300
tokens. In one process the plain step, mode "table" and mode "placeholders" run alternately as CUDA
graph replays; prints ms/step and launches per step of each, CUDA-event times of the scatter and
write-back kernels (a captured sweep of each), and the GPU name and power limit read in the same run.

    python scripts/bench_embedding_step.py [--steps 20] [--warmup 5] [--rounds 2] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:       # name from torch at least
        q = f"{torch.cuda.get_device_name()}, power limit unavailable ({type(e).__name__})"
    return q


def build(rank, kind, lat_hw):
    import lora_b200 as L
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.train import LoraEmbeddingStep, LoraTrainStep, StepConfig
    dev = torch.device("cuda")
    torch.manual_seed(0)
    with torch.device(dev):
        unet = UNet2DConditionModel(UNetConfig.sd15())
        text = build_text_encoder()
    unet.requires_grad_(False); text.requires_grad_(False)
    unet, text = unet.to(torch.bfloat16).to(memory_format=torch.channels_last), text.to(torch.bfloat16)
    L.inject_trainable_lora(unet, r=rank)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=rank)
    g = torch.Generator(device=dev).manual_seed(1)
    for m in list(unet.modules()) + list(text.modules()):
        if type(m).__name__ == "LoraInjectedLinear":
            m.lora_up.weight.data.normal_(0.0, 0.01, generator=g)
    cfg = StepConfig(compute_dtype=torch.bfloat16, use_cuda_graph=True)
    shape = (1, 4, lat_hw, lat_hw)
    if kind == "plain":
        return LoraTrainStep(unet, text, cfg, latent_shape=shape)
    V = text.get_input_embeddings().weight.shape[0]
    ph = [V - 2, V - 1]
    if kind == "table":
        return LoraEmbeddingStep(unet, text, ph, cfg, lr_embedding=1e-4, mode="table", latent_shape=shape)
    return LoraEmbeddingStep(unet, text, ph, cfg, lr_embedding=5e-4, mode="placeholders", unfreeze_lora_step=10 ** 6,
                             latent_shape=shape)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_embedding_step.py needs a CUDA device")
    from lora_b200 import ops
    torch.backends.cudnn.benchmark = True
    lat_hw = args.res // 8
    gen = torch.Generator().manual_seed(5)
    pool = torch.randint(0, 49406, (300,), generator=gen)
    data = []
    for _ in range(4):
        ids = pool[torch.randint(0, 300, (1, 77), generator=gen)]
        ids[0, 1], ids[0, 2] = 49406, 49407                     # the two placeholders
        data.append((torch.randn(1, 4, lat_hw, lat_hw, generator=gen) * 0.18215, ids))
    result = {"gpu": gpu_info(), "res": args.res, "steps": args.steps, "runs": []}
    for rank in (1, 4):
        steps = {}
        for kind in ("plain", "table", "placeholders"):
            st = build(rank, kind, lat_hw)
            st.latents.copy_(data[0][0]); st.input_ids.copy_(data[0][1])
            st._body()
            ops.LAUNCH_COUNT = 0
            st._body()
            launches = ops.LAUNCH_COUNT
            st.prepare()
            assert st.graph is not None, st.graph_error
            steps[kind] = (st, launches)
        times = {k: [] for k in steps}
        for _ in range(args.rounds):
            for kind, (st, _) in steps.items():          # alternate the three engines
                for i in range(args.warmup):
                    st.latents.copy_(data[i % 4][0]); st.input_ids.copy_(data[i % 4][1])
                    st.step_device()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(args.steps):
                    st.step_device()
                e1.record()
                torch.cuda.synchronize()
                times[kind].append(e0.elapsed_time(e1) / args.steps)
        # kernel times: a captured sweep of 50 scatters / write-backs on the "table" engine's state
        st = steps["table"][0]
        rows = st.rows
        snap = st._snapshot()
        ids = st.input_ids
        gout = torch.randn(1, 77, rows.D, device="cuda", dtype=torch.bfloat16)
        kern = {}
        for name, fn in (("scatter", lambda: rows._scatter(ids, gout)), ("write_back", rows.write_back)):
            fn()
            torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                for _ in range(50):
                    fn()
            gr.replay()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            gr.replay()
            e1.record()
            torch.cuda.synchronize()
            kern[name + "_us"] = round(1000 * e0.elapsed_time(e1) / 50, 2)
        st._restore(snap)
        st.rows.check()
        for kind, (s, launches) in steps.items():
            result["runs"].append({"rank": rank, "step": kind, "launches_per_step": launches,
                                   "ms_per_step": [round(t, 3) for t in times[kind]]})
        result["runs"].append({"rank": rank, "kernels": kern, "claimed_rows": st.rows.claimed()})
        for s, _ in steps.values():
            if hasattr(s, "release"):
                s.release()
        del steps, st, rows
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_embedding_step.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
