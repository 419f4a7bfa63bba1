"""Data-parallel cost of training the token-embedding table with the LoRA factors, in the
pivotal-tuning shape: SD1.5 UNet + CLIP text encoder, LoRA r = 16, 768 px, bf16, batch 1 per GPU, two
placeholder tokens, LoraEmbeddingStep mode "table" (PTI `continue_inversion`), at world 1, 2 and 4.
Each world size is one torchrun job in which the plain LoraTrainStep and LoraEmbeddingStep run
alternately as CUDA-graph replays (each rank with its own prompt ids); prints one JSON line with
images/s, ms/step and launches per step of each, plus the GPU name and power limit read in this call.
World sizes above the visible GPU count are reported as not run.

    python scripts/bench_embedding_dp.py [--steps 20] [--warmup 5] [--rounds 2] [--worlds 1,2,4] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)


def worker(args):
    import torch.distributed as dist
    from bench_embedding_step import build
    from lora_b200 import ops
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    torch.backends.cudnn.benchmark = True
    lat_hw = args.res // 8
    gen = torch.Generator().manual_seed(5 + rank)
    pool = torch.randint(0, 49406, (300,), generator=gen)
    data = []
    for _ in range(4):
        ids = pool[torch.randint(0, 300, (1, 77), generator=gen)]
        ids[0, 1], ids[0, 2] = 49406, 49407                     # the two placeholders
        data.append((torch.randn(1, 4, lat_hw, lat_hw, generator=gen) * 0.18215, ids))
    steps = {}
    for kind in ("plain", "table"):
        st = build(args.rank, kind, lat_hw)
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
        for kind, (st, _) in steps.items():              # alternate the two engines
            for i in range(args.warmup):
                st.latents.copy_(data[i % 4][0]); st.input_ids.copy_(data[i % 4][1])
                st.step_device()
            torch.cuda.synchronize()
            if world > 1:
                dist.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(args.steps):
                st.step_device()
            e1.record()
            torch.cuda.synchronize()
            times[kind].append(e0.elapsed_time(e1) / args.steps)
    steps["table"][0].flush()                            # raises if the union overflowed the rows
    if rank == 0:
        st = steps["table"][0]
        out = {"world": world, "exchange": ("nvlink-peer" if st.peer_allreduce else "nccl") if world > 1 else None,
               "claimed_rows": st.rows.claimed(), "runs": []}
        for kind, (s, launches) in steps.items():
            ms = [round(t, 3) for t in times[kind]]
            out["runs"].append({"step": kind, "launches_per_step": launches, "ms_per_step": ms,
                                "images_per_s": [round(1000.0 * world / t, 2) for t in ms]})
        print("RESULT " + json.dumps(out), flush=True)
    for s, _ in steps.values():
        if hasattr(s, "release"):
            s.release()
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--res", type=int, default=768)
    ap.add_argument("--rank", type=int, default=16)
    ap.add_argument("--worlds", default="1,2,4")
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_embedding_dp.py needs a CUDA device")
    if args.worker:
        return worker(args)
    from bench_embedding_step import gpu_info
    n_gpus = torch.cuda.device_count()
    result = {"gpu": gpu_info(), "gpus_visible": n_gpus, "res": args.res, "lora_rank": args.rank,
              "steps": args.steps, "worlds": []}
    for w in (int(x) for x in args.worlds.split(",")):
        if w > n_gpus:
            result["worlds"].append({"world": w, "not_run": f"{n_gpus} GPU(s) visible"})
            continue
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(w),
               "--master-addr", "127.0.0.1", "--master-port", str(29561 + w), os.path.abspath(__file__), "--worker",
               "--steps", str(args.steps), "--warmup", str(args.warmup), "--rounds", str(args.rounds),
               "--res", str(args.res), "--rank", str(args.rank)]
        p = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
        lines = [ln for ln in p.stdout.splitlines() if ln.startswith("RESULT ")]
        if p.returncode != 0 or not lines:
            result["worlds"].append({"world": w, "error": (p.stdout + p.stderr)[-1500:]})
            continue
        result["worlds"].append(json.loads(lines[-1][len("RESULT "):]))
    line = json.dumps(result)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_embedding_dp.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
