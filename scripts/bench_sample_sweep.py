"""Per-image LoRA scales: what the per-sample coefficient path costs and what it saves, on full-size SD1.5
host models (LoRA r=4 on the UNet and the text encoder, bf16 autocast, guidance 7, Euler-ancestral,
512 px, grouping on). Weights are random: the timings do not depend on them.

  (a) graph B (one denoising step: the UNet at batch 2B and the step launch), ms per replay, default
      graphs vs per-sample graphs, at B = 1, 4, 8; the two replays alternated, median of --reps rounds;
  (b) an 8-frame LoRA-scale sweep (scales 0 .. 1, one seed), three ways: 8 batch-1 calls with
      tune_lora_scale before each (each one a capture), 8 batch-1 calls with lora_scale (one capture),
      one batch-8 call with lora_scale and shared_noise. Seconds per frame (host clock around each way,
      ending in a device synchronise) and the captures each way took;
  (c) CUDA-event time of ops.fused_linear with scalar coefficients and with a per-sample table
      (coef_rows, S = 4) at SD1.5 site shapes of a batch-4 guided step, alternated, median of --reps.
Prints one JSON line per measurement with the GPU's name and power limit."""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_sample import _gpu, _models  # noqa: E402


def _sync_time(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def _median(v):
    return sorted(v)[len(v) // 2]


def _sampler(unet, text, vae, B, n):
    from lora_b200.sample import LoraSampler, SamplerConfig
    cfg = SamplerConfig(scheduler="euler_ancestral", num_inference_steps=n, max_steps=n, guidance_scale=7.0,
                        autocast_dtype=torch.bfloat16)
    return LoraSampler(unet, text, vae, cfg, latent_shape=(B, 4, 64, 64))


def graph_b(models, B, n, reps):
    unet, text, vae = models
    s = _sampler(unet, text, vae, B, n)
    ids = torch.randint(0, text.config.vocab_size, (B, 77), device="cuda")
    neg = torch.randint(0, text.config.vocab_size, (B, 77), device="cuda")
    scales = [i / max(1, B - 1) for i in range(B)]
    s.sample(ids, neg)
    s.sample(ids, neg, lora_scale={"unet": scales, "text_encoder": scales})
    gb_d = s._graphs[(2, "single-step")][1]
    gb_p = s._graphs[(2, "single-step", "per_sample")][1]
    events = lambda: (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))  # noqa: E731
    t = {"default": [], "per_sample": []}
    for _ in range(reps):
        for key, g in (("default", gb_d), ("per_sample", gb_p)):
            a, b = events()
            a.record()
            for _ in range(n):
                g.replay()
            b.record()
            b.synchronize()
            t[key].append(a.elapsed_time(b) / n)
    return {"measure": "graph_b_ms_per_step", "batch": B, "steps_per_rep": n,
            "default_ms": round(_median(t["default"]), 3), "per_sample_ms": round(_median(t["per_sample"]), 3),
            "captures": s.captures}


def sweep(models, n, frames=8):
    import lora_b200 as L
    unet, text, vae = models
    scales = [i / (frames - 1) for i in range(frames)]
    ids = torch.randint(0, text.config.vocab_size, (1, 77), device="cuda")
    neg = torch.randint(0, text.config.vocab_size, (1, 77), device="cuda")
    out = {"measure": "scale_sweep", "frames": frames, "steps": n}
    s1 = _sampler(unet, text, vae, 1, n)

    def tuned():
        for sc in scales:
            L.tune_lora_scale(unet, sc)
            L.tune_lora_scale(text, sc)
            s1.sample(ids, neg, seed=0)
    out["tune_batch1_s_per_frame"] = round(_sync_time(tuned) / frames, 4)
    out["tune_batch1_captures"] = s1.captures
    L.tune_lora_scale(unet, 1.0)
    L.tune_lora_scale(text, 1.0)
    sp = _sampler(unet, text, vae, 1, n)

    def per_sample():
        for sc in scales:
            sp.sample(ids, neg, seed=0, lora_scale={"unet": sc, "text_encoder": sc})
    out["per_sample_batch1_s_per_frame"] = round(_sync_time(per_sample) / frames, 4)
    out["per_sample_batch1_captures"] = sp.captures
    s8 = _sampler(unet, text, vae, frames, n)
    ids8, neg8 = ids.expand(frames, -1).contiguous(), neg.expand(frames, -1).contiguous()
    out["batch8_shared_noise_s_per_frame"] = round(_sync_time(
        lambda: s8.sample(ids8, neg8, seed=0, shared_noise=True,
                          lora_scale={"unet": scales, "text_encoder": scales})) / frames, 4)
    out["batch8_shared_noise_captures"] = s8.captures
    # steady state of the same three ways once every capture exists (the per-sample ones need none)
    out["per_sample_batch1_warm_s_per_frame"] = round(_sync_time(per_sample) / frames, 4)
    out["batch8_shared_noise_warm_s_per_frame"] = round(_sync_time(
        lambda: s8.sample(ids8, neg8, seed=0, shared_noise=True,
                          lora_scale={"unet": scales, "text_encoder": scales})) / frames, 4)
    return out


# (site, M, K, N) of a guided batch-4 SD1.5 512-px step (2B = 8 latents / prompts)
SITES = [("attn1 q 64x64", 8 * 4096, 320, 320), ("ff in 64x64", 8 * 4096, 320, 2560),
         ("ff out 64x64", 8 * 4096, 1280, 320), ("attn2 k 77", 8 * 77, 768, 320),
         ("attn1 q 32x32", 8 * 1024, 640, 640), ("attn1 q 16x16", 8 * 256, 1280, 1280),
         ("attn1 q 8x8", 8 * 64, 1280, 1280), ("clip q", 8 * 77, 768, 768)]


def kernels(reps, iters=50):
    from lora_b200 import ops
    out = []
    S, r = 4, 4
    for name, M, K, N in SITES:
        x = torch.randn(M, K, device="cuda").to(torch.bfloat16)
        w = (torch.randn(N, K, device="cuda") / K ** 0.5).to(torch.bfloat16)
        d16 = ops.cast_rows_pad16(torch.randn(r, K, device="cuda"), K, 1, r, K, torch.bfloat16)
        up = torch.randn(N, r, device="cuda")
        table = torch.rand(S, r, device="cuda")
        rps = M // (2 * S)
        scalar = lambda: ops.fused_linear(x, w, None, d16, up, r, 1, None, 0.8, r, torch.bfloat16, False)  # noqa: E731
        per = lambda: ops.fused_linear(x, w, None, d16, up, r, 1, None, 1.0, r, torch.bfloat16, False,  # noqa: E731
                                       coef_rows=(table, r, rps, S))
        for f in (scalar, per):
            f()
        t = {"scalar": [], "per_sample": []}
        for _ in range(reps):
            for key, f in (("scalar", scalar), ("per_sample", per)):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(iters):
                    f()
                b.record()
                b.synchronize()
                t[key].append(1e3 * a.elapsed_time(b) / iters)
        out.append({"measure": "fused_linear_us", "site": name, "M": M, "K": K, "N": N,
                    "scalar_us": round(_median(t["scalar"]), 2), "per_sample_us": round(_median(t["per_sample"]), 2)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--only", default=None, help="comma-separated parts: a, b, c")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample_sweep.py needs a CUDA device")
    import lora_b200 as L
    name, power = _gpu()
    parts = set(a.only.split(",")) if a.only else {"a", "b", "c"}
    L.set_grouping(True)
    rows = []
    if "c" in parts:
        rows += kernels(a.reps)
    if parts & {"a", "b"}:
        unet, text, vae, *_ = _models(False)
        if "a" in parts:
            for B in (1, 4, 8):
                rows.append(graph_b((unet, text, vae), B, a.steps, a.reps))
        if "b" in parts:
            rows.append(sweep((unet, text, vae), a.steps))
    for r in rows:
        r.update(gpu=name, power_limit=power)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
