"""BASELINE.json configs[4]: cli_svd distill full-finetune -> rank 8 over all SD1.5 attention/GEGLU
weight deltas + CLIP attention, on 1 x H100. Synthetic fp16 weight pairs (
dW = lowrank(8)*0.02 + noise*1e-3). Prints matrices/s and algorithmic GB/s (ONE read of both
fp16 models = 2*2*sum(N*K) bytes) against the measured HBM peak, and the reference's way
(serial torch.linalg.svd, full_matrices default, cli_svd.py:35) timed on a subset."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lora_b200.svd import svd_lowrank_ragged

SHAPES = [(320, 320, 30), (2560, 320, 5), (320, 768, 10), (640, 640, 30), (5120, 640, 5), (640, 768, 10),
          (1280, 1280, 36), (10240, 1280, 6), (1280, 768, 12), (768, 768, 48)]
dev = "cuda"
rank = 8
torch.manual_seed(0)
groups = []
total_bytes = 0
n_mats = 0
for (N, K, cnt) in SHAPES:
    Wb = [(torch.randn(N, K, device=dev) * 0.05).half() for _ in range(cnt)]
    Wt = []
    for w in Wb:
        low = (torch.randn(N, rank, device=dev) @ torch.randn(rank, K, device=dev)) * 0.02 / (K ** 0.5)
        Wt.append((w.float() + low + torch.randn(N, K, device=dev) * 1e-3).half())
    groups.append((Wt, Wb))
    total_bytes += 2 * 2 * N * K * cnt
    n_mats += cnt


ALL_T = [w for Wt, _ in groups for w in Wt]
ALL_B = [w for _, Wb in groups for w in Wb]


def run():
    """ONE call for all 240 weight deltas (ragged over the 10 shapes), quantile clamp included."""
    ups, downs, sigma, hi = svd_lowrank_ragged(ALL_T, ALL_B, rank, clamp_quantile=0.99)
    outs, i = [], 0
    for Wt, _ in groups:
        n = len(Wt)
        outs.append((ups[i:i + n], downs[i:i + n], sigma[i:i + n]))
        i += n
    return outs


run(); torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
reps = 5
e0.record()
for _ in range(reps):
    outs = run()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / reps
# accuracy spot check vs exact SVD on one matrix per group
worst = 0.0
for (Wt, Wb), (up, down, sig) in zip(groups, outs):
    resid = (Wt[0].float() - Wb[0].float()).double()
    S = torch.linalg.svdvals(resid)
    worst = max(worst, float((sig[0, :rank].double() - S[:rank]).abs().max() / S[0]))
# the reference's way on a subset: serial full SVD (fp32, full_matrices=True)
sub = [(g[0][0], g[1][0]) for g in groups]
torch.cuda.synchronize()
t0 = time.perf_counter()
for wt, wb in sub:
    U, S, Vh = torch.linalg.svd((wt - wb).float())
torch.cuda.synchronize()
ref_ms_per_mat = (time.perf_counter() - t0) * 1e3 / len(sub)
peak = 6585.8
if os.path.exists("MEASURED_PEAKS.json"):
    peak = json.load(open("MEASURED_PEAKS.json")).get("hbm_gbs", peak)
out = {"workload": "SD1.5 svd_distill rank 8: 192 UNet attention/GEGLU + 48 CLIP weight deltas (fp16 pairs)",
       "matrices": n_mats, "ms_total": ms, "matrices_per_s": n_mats / ms * 1e3,
       "algorithmic_GBps": total_bytes / ms / 1e6, "frac_of_hbm_peak": total_bytes / ms / 1e6 / peak,
       "passes_over_weights": 4, "max_rel_sigma_err": worst,
       "reference_way_ms_per_matrix_subset(torch.linalg.svd full, cuSOLVER)": ref_ms_per_mat,
       "reference_way_est_ms_total": ref_ms_per_mat * n_mats}
print(json.dumps(out))
os.makedirs("gpurun_out", exist_ok=True)
json.dump(out, open("gpurun_out/bench_svd.json", "w"), indent=1)
