"""SDXL sampling throughput: LoraXLSampler's graph replay, its eager path and the pipeline-style oracle
loop (oracle/sample_xl_ref.py), alternated in one process, on the full-size SDXL host models with LoRA
r=4 on the UNet and both text encoders, random weights, bf16 autocast, guidance 5, 1024 px, batch 1:
  Euler 30 steps;  DPM-Solver++(2M) 25 steps;  Euler 30 steps with guidance_rescale 0.7;
  img2img, Euler 30 steps at strength 0.5 (15 steps run).
Prints per workload: s/image and ms per denoising step for the three paths, the time of one replay of
the denoising-step graph alone, the decode's share of a graph-replayed call, liblora_b200 launches per
denoising step (ops counter), peak memory, and the GPU's name and power limit. Then a CUDA-event
microbenchmark of the step launch alone at 128 x 128 latents with G = 2: lb_sample_step_rescale against
lb_sample_step_ch, 2000 launches each, alternated in blocks.
Weights are random: the timings do not depend on them."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_sample import _gpu, _time  # noqa: E402


def _models():
    """(ours (unet, te1, te2), oracle (unet, te1, te2) sharing the frozen weights, bf16 VAE)."""
    import lora_b200 as L
    from lora_b200.host.clip import build_sdxl_text_encoders
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    from oracle.ref_modules import ref_inject
    torch.manual_seed(0)
    with torch.device("cuda"):
        unet = UNet2DConditionModel(UNetConfig.sdxl())
        te1, te2 = build_sdxl_text_encoders()
        vae = AutoencoderKL(VAEConfig.sd(), with_decoder=True)
    ours = (unet.to(memory_format=torch.channels_last), te1, te2)
    for m in ours + (vae,):
        m.requires_grad_(False)
    vae = vae.to(torch.bfloat16).to(memory_format=torch.channels_last)
    with torch.device("meta"):
        refs = (UNet2DConditionModel(UNetConfig.sdxl()),) + tuple(build_sdxl_text_encoders())
    for dst, src in zip(refs, ours):                    # the oracle's models use ours' frozen weights
        for (_, md), (_, ms) in zip(dst.named_modules(), src.named_modules()):
            md._parameters.update(ms._parameters)
            md._buffers.update(ms._buffers)
    L.inject_trainable_lora(ours[0], r=4)
    for te in ours[1:]:
        L.inject_trainable_lora(te, target_replace_module={"CLIPAttention"}, r=4)
    ref_inject(refs[0], {"CrossAttention", "Attention", "GEGLU"}, r=4)
    for te in refs[1:]:
        ref_inject(te, {"CLIPAttention"}, r=4)
    return ours, refs, vae


def run(models, name, sched, n, reps, phi=0.0, task="txt2img", strength=0.5):
    from lora_b200 import ops
    from lora_b200.host import schedulers
    from lora_b200.sample import LoraXLSampler, SamplerConfig
    from oracle import sample_xl_ref as XR
    ours, refs, vae = models
    lat = (1, 4, 128, 128)
    cfg = dict(scheduler=sched, num_inference_steps=n, max_steps=n, guidance_scale=5.0, vae_scaling=0.13025,
               autocast_dtype=torch.bfloat16, guidance_rescale=phi, task=task, strength=strength)
    sg = LoraXLSampler(*ours, vae, SamplerConfig(**cfg), latent_shape=lat)
    se = LoraXLSampler(*ours, vae, SamplerConfig(use_cuda_graph=False, **cfg), latent_shape=lat)
    ids1 = torch.randint(0, 49407, (1, 77), device="cuda")
    ids2 = torch.randint(0, 49407, (1, 77), device="cuda")
    g = torch.Generator().manual_seed(0)
    image = torch.randint(0, 256, (1, 1024, 1024, 3), generator=g, dtype=torch.uint8).cuda()
    extra = dict(image=image) if task == "img2img" else {}
    k = n - schedulers.t_start(n, strength) if task == "img2img" else n
    torch.cuda.reset_peak_memory_stats()
    sg.prepare()
    sg.sample(ids1, ids2, **extra)
    se.sample(ids1, ids2, **extra)
    noise = sg.noise[:k + 1].clone()
    peps = sg.posterior_noise.clone() if task == "img2img" else None
    tid = XR.add_time_ids((1024, 1024), (0, 0), (1024, 1024), 1, True, torch.float32, "cuda")

    def oracle():
        def encode():
            return XR.encode_prompt_xl(refs[1], refs[2], ids1, ids2)
        XR.sample(refs[0], vae, XR.make_scheduler(sched, "epsilon"), n, encode, noise, 5.0, phi,
                  added_cond_kwargs={"time_ids": tid}, image_u8=extra.get("image"),
                  strength=strength if task == "img2img" else None, posterior_eps=peps, scaling=0.13025,
                  dtype=torch.float32, autocast_dtype=torch.bfloat16)
    oracle()
    t = {"graph": [], "eager": [], "oracle": []}
    for _ in range(reps):                      # alternated: the three paths see the same machine state
        t["graph"].append(_time(lambda: sg.sample(ids1, ids2, **extra), 1))
        t["eager"].append(_time(lambda: se.sample(ids1, ids2, **extra), 1))
        t["oracle"].append(_time(oracle, 1))
    family = schedulers.family(sched)
    ga, gb, gc = sg._graphs[sg._key(2, family, phi > 0.0)]
    decode = _time(gc.replay, 3)
    denoise_step = _time(gb.replay, k)          # past the table's end the kernel repeats its last row
    with torch.no_grad():
        for m in ours:
            m.eval()
        c0 = ops.LAUNCH_COUNT
        se._body_b(2, family, phi > 0.0)
        launches = ops.LAUNCH_COUNT - c0
        for m in ours:
            m.train()
    med = {key: sorted(v)[len(v) // 2] for key, v in t.items()}
    out = {"workload": name, "scheduler": sched, "steps": n, "denoising_steps": k, "guidance_rescale": phi,
           **{f"{key}_s_per_image": round(v, 4) for key, v in med.items()},
           **{f"{key}_ms_per_step": round(1e3 * v / k, 3) for key, v in med.items()},
           "graph_b_ms_per_replay": round(1e3 * denoise_step, 3),
           "decode_share_graph": round(decode / med["graph"], 4),
           "launches_per_step": launches,
           "peak_mib": round(torch.cuda.max_memory_allocated() / 2 ** 20)}
    if task == "img2img":
        out.update(task=task, strength=strength)
    del sg, se
    torch.cuda.empty_cache()
    return out


def step_launch_microbench(launches=2000, block=100):
    """us per launch of the step alone at 128 x 128 latents, B = 1, G = 2, bf16 model output (an
    Euler table; the step index runs past its end, where the kernel repeats the last row)."""
    from lora_b200.host import schedulers
    from lora_b200.step_ops import sample_step_ch, sample_step_rescale
    dev = "cuda"
    B, C, H, W = 1, 4, 128, 128
    tab = schedulers.pack_table("euler", "epsilon", 30, 30).to(dev)
    noise = torch.randn(31, B, C, H, W, device=dev)
    mo = torch.randn(2 * B, C, H, W, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    x = torch.randn(B, C, H, W, device=dev)
    gs, phi = torch.tensor([5.0], device=dev), torch.tensor([0.7], device=dev)
    idx, cnt = torch.zeros(1, device=dev, dtype=torch.int32), torch.zeros(1, device=dev, dtype=torch.int32)
    ts = torch.zeros(1, device=dev)
    unet_in = torch.zeros(2 * B, C, H, W, device=dev, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    vae_in = torch.zeros(B, C, H, W, device=dev, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    fns = {"sample_step_ch": lambda: sample_step_ch(mo, x, noise, tab, gs, idx, cnt, unet_in, ts, vae_in, 0.13025),
           "sample_step_rescale": lambda: sample_step_rescale(mo, x, noise, None, tab, gs, phi, idx, cnt, unet_in, ts,
                                                              vae_in, 0.13025)}
    # each path's `block` launches captured in one graph: the replays time the device, not the host's
    # enqueue rate (the Python wrapper takes longer per launch than the kernel)
    graphs = {}
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for f in fns.values():
            f()
    torch.cuda.current_stream().wait_stream(side)
    for key, f in fns.items():
        graphs[key] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[key]):
            for _ in range(block):
                f()
    total = {k: 0.0 for k in fns}
    for gr in graphs.values():
        gr.replay()
    for _ in range(launches // block):
        for key, gr in graphs.items():
            x.normal_()                                  # keep the latents finite
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            gr.replay()
            e1.record()
            e1.synchronize()
            total[key] += e0.elapsed_time(e1)
    return {f"{k}_us_per_launch": round(1e3 * v / launches, 2) for k, v in total.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", default=None,
                    help="comma-separated workloads (xl_euler30, xl_dpm25, xl_euler30_rescale, xl_img2img_euler30, "
                         "step_launch)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample_xl.py needs a CUDA device")
    name, power = _gpu()
    only = set(a.only.split(",")) if a.only else None
    work = [("xl_euler30", "euler", 30, 0.0, "txt2img"),
            ("xl_dpm25", "dpmsolver_multistep", 25, 0.0, "txt2img"),
            ("xl_euler30_rescale", "euler", 30, 0.7, "txt2img"),
            ("xl_img2img_euler30", "euler", 30, 0.0, "img2img")]
    import lora_b200 as L
    if not only or "step_launch" in only:
        r = step_launch_microbench()
        r.update(workload="step_launch", latents="1x4x128x128", G=2, gpu=name, power_limit=power)
        print(json.dumps(r), flush=True)
    work = [w for w in work if not only or w[0] in only]
    if not work:
        return
    models = _models()
    L.set_grouping(True)
    for w in work:
        r = run(models, w[0], w[1], w[2], a.reps, phi=w[3], task=w[4])
        r.update(gpu=name, power_limit=power)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
