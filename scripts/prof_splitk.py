"""Time the cluster split-K schedule (lb_debug_set_linear_mode schedule 3, csrc/fused_core.cuh with
CL > 1) against the other schedules on the small-M / long-K SD1.5 sites.

Launches are enqueued back to back (REPS per measurement, one CUDA-event pair around the batch,
rotating over enough operand sets to exceed the 50 MB L2 when COLD=1), so the GPU never waits for
Python -- scripts/prof_site.py's per-launch event pairs measure CPU launch latency for kernels this
short. Run the parity test first (pytest tests/test_zz_splitk_experimental_gpu.py).
    python scripts/prof_splitk.py            # -> gpurun_out/splitk_times.json
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lora_b200 import _C, ops

SHAPES = [(77, 768, 768, 4), (77, 768, 320, 4), (77, 768, 1280, 4), (256, 1280, 1280, 4), (64, 1280, 1280, 4),
          (1024, 640, 640, 4), (256, 5120, 1280, 4), (256, 10240, 1280, 4), (64, 10240, 1280, 4),
          (1024, 5120, 640, 4)]
MODES = [(0, "default")] + [(3 + 4 * 1 + 16 * (s - 1), f"splitk{s}/bn64") for s in (2, 3, 4)] + \
        [(3 + 4 * 2 + 16 * 1, "splitk2/bn128")]
REPS = int(os.environ.get("REPS", 200))
COLD = os.environ.get("COLD", "0") == "1"
dev, dt = "cuda", torch.bfloat16
rows = []
for (M, K, N, r) in SHAPES:
    per_set = 2 * (M * K + N * K + M * N)
    n_sets = max(1, min(64, (192 << 20) // per_set)) if COLD else 1
    sets = []
    for i in range(n_sets):
        x = torch.randn(M, K, device=dev, dtype=dt)
        w = torch.randn(N, K, device=dev, dtype=dt) * 0.02
        a = torch.randn(r, K, device=dev)
        b = torch.randn(N, r, device=dev) * 0.01
        sets.append((x, w, ops.cast_rows_pad16(a, K, 1, r, K, dt), b, torch.zeros(N, device=dev)))
    ref = None
    for mode, name in MODES:
        if _C.lib.lb_debug_set_linear_mode(mode) != 0:
            continue
        run = lambda i: ops.fused_linear(sets[i][0], sets[i][1], sets[i][4], sets[i][2], sets[i][3], r, 1,
                                         None, 1.0, r, dt, True)
        y, t = run(0)
        torch.cuda.synchronize()
        if ref is None:
            ref = (y.float(), t.clone())
        err_y = float((y.float() - ref[0]).norm() / ref[0].norm())
        err_t = float((t - ref[1]).norm() / ref[1].norm())
        for i in range(10):
            run(i % n_sets)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(REPS):
            run(i % n_sets)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / REPS
        rows.append({"M": M, "K": K, "N": N, "r": r, "mode": name, "us_per_launch": round(us, 2),
                     "cold_sets": n_sets, "rel_err_y_vs_default": err_y, "rel_err_t_vs_default": err_t})
        print(rows[-1], flush=True)
    _C.lib.lb_debug_set_linear_mode(0)
os.makedirs("gpurun_out", exist_ok=True)
json.dump(rows, open("gpurun_out/splitk_times.json", "w"), indent=1)
