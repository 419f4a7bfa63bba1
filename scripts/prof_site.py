"""Launch the fused LoRA-linear kernel on representative SD1.5 site shapes and print CUDA-event
timings per shape and tile schedule (algorithmic GB/s, TFLOP/s). Launches are enqueued back to back,
REPS per event pair, rotating over enough operand sets that the working set exceeds the 50 MB L2: a
per-launch event pair would time the host's launch latency on the short sites."""
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lora_b200 import _C, ops

SHAPES = [(4096, 320, 2560, 4), (4096, 320, 320, 4), (1024, 640, 640, 4), (1024, 640, 5120, 4),
          (256, 1280, 1280, 4), (256, 1280, 10240, 4), (64, 1280, 10240, 4), (77, 768, 768, 4),
          (77, 768, 320, 4), (9216, 320, 2560, 16),
          # dX launches of the same sites (K and N swapped)
          (4096, 2560, 320, 4), (1024, 5120, 640, 4), (256, 10240, 1280, 4)]
if os.environ.get("PROF_SHAPES"):      # e.g. PROF_SHAPES="4096,320,320,4;9216,320,2560,16"
    SHAPES = [tuple(int(v) for v in t.split(",")) for t in os.environ["PROF_SHAPES"].split(";")]
if os.environ.get("PROF_AUTO_ONLY"):
    MODES = [(0, "auto")]
else:
    MODES = [(0, "auto"), (1 + 4, "1tile/bn64"), (1 + 8, "1tile/bn128"), (2 + 8, "1cta-per-sm/bn128"),
             (3 + 16, "cluster2/bn64"), (3 + 48, "cluster4/bn64")]
dev, dt = "cuda", torch.bfloat16
rows = []
flush = torch.empty(256 << 20, device=dev, dtype=torch.uint8)


REPS = 40


def timed(fn, n_sets=1):
    """Median over 5 batches of the per-launch time of REPS back-to-back calls fn(i % n_sets)."""
    ts = []
    for _ in range(5):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(REPS):
            fn(i % n_sets)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / REPS)
    ts.sort()
    return ts[len(ts) // 2]


for (M, K, N, r) in SHAPES:
    n_sets = max(1, min(8, -(-(120 << 20) // (2 * (M * K + N * K + M * N)))))
    xs = [torch.randn(M, K, device=dev, dtype=dt) for _ in range(n_sets)]
    ws = [torch.randn(N, K, device=dev, dtype=dt) * 0.02 for _ in range(n_sets)]
    a = torch.randn(r, K, device=dev)
    b = torch.randn(N, r, device=dev) * 0.01
    d16 = ops.cast_rows_pad16(a, K, 1, r, K, dt)
    bias = torch.zeros(N, device=dev)
    byts = 2 * (M * K + N * K + r * K + M * N) + 4 * N * r + 4 * N + 4 * M * 16
    fl = 2 * M * K * N + 2 * M * r * (K + N)
    for mode, mname in MODES:
        _C.lib.lb_debug_set_linear_mode(mode)
        run = lambda i: ops.fused_linear(xs[i], ws[i], bias, d16, b, r, 1, None, 1.0, r, dt, True)
        for i in range(n_sets):
            run(i)
        torch.cuda.synchronize()
        ms = timed(run, n_sets)
        rows.append({"mode": mname, "M": M, "K": K, "N": N, "r": r, "us": round(ms * 1e3, 2),
                     "GBps": round(byts / ms / 1e6, 1), "TFLOPs": round(fl / ms / 1e9, 1)})
        print(rows[-1], flush=True)
    # library GEMM of the same base shape, for scale (cuBLAS bf16, no LoRA, no bias)
    ms = timed(lambda i: torch.matmul(xs[i], ws[i].t()), n_sets)
    rows.append({"mode": "torch.matmul (base GEMM only)", "M": M, "K": K, "N": N, "us": round(ms * 1e3, 2)})
    print(rows[-1], flush=True)
_C.lib.lb_debug_set_linear_mode(0)

# skinny weight-gradient reduction
for (M, C, r) in [(4096, 320, 4), (4096, 2560, 4), (1024, 640, 4), (256, 10240, 4), (77, 768, 4), (9216, 320, 16)]:
    S = torch.randn(M, C, device=dev, dtype=dt)
    V = torch.randn(M, 16, device=dev)
    out = torch.zeros(r, C, device=dev)
    run = lambda i: ops.wgrad(S, V, None, 1.0, out, C, 1, r)
    for _ in range(3):
        run(0)
    ms = timed(run)
    rows.append({"mode": "wgrad", "M": M, "C": C, "r": r, "us": round(ms * 1e3, 2),
                 "GBps": round((2 * M * C + 64 * M) / ms / 1e6, 1)})
    print(rows[-1], flush=True)

os.makedirs("gpurun_out", exist_ok=True)
json.dump(rows, open("gpurun_out/site_times.json", "w"), indent=1)

# ---- phase breakdown of one CTA (globaltimer stamps inside the one-tile-per-CTA kernel)
names = ["entry", "first TMA issue", "first stage landed", "main-loop MMAs completed", "accumulator parked",
         "T' ready", "LoRA MMA done", "stores issued", "staging released", "exit"]
stamps = torch.zeros(16, device=dev, dtype=torch.int64)
phase = []
for (M, K, N, r) in [(77, 768, 768, 4), (256, 1280, 1280, 4), (1024, 640, 640, 4), (4096, 320, 320, 4)]:
    x = torch.randn(M, K, device=dev, dtype=dt)
    w = torch.randn(N, K, device=dev, dtype=dt) * 0.02
    a = torch.randn(r, K, device=dev)
    b = torch.randn(N, r, device=dev) * 0.01
    d16 = ops.cast_rows_pad16(a, K, 1, r, K, dt)
    _C.lib.lb_debug_set_linear_mode(1)           # one tile per CTA (stamps live in that kernel)
    for cold in (True, False):
        ops.fused_linear(x, w, None, d16, b, r, 1, None, 1.0, r, dt, True)
        if cold:
            flush.zero_()
        torch.cuda.synchronize()
        stamps.zero_()
        _C.lib.lb_debug_set_stamp_buffer(ctypes.c_void_p(stamps.data_ptr()))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ops.fused_linear(x, w, None, d16, b, r, 1, None, 1.0, r, dt, True)
        e1.record()
        torch.cuda.synchronize()
        _C.lib.lb_debug_set_stamp_buffer(None)
        t = stamps.cpu().tolist()
        rel = {names[i]: (t[i] - t[0]) for i in range(10) if t[i]}
        row = {"mode": "phases_ns", "M": M, "K": K, "N": N, "cold_L2": cold,
               "event_us": round(e0.elapsed_time(e1) * 1e3, 2), **rel}
        phase.append(row)
        print(row, flush=True)
_C.lib.lb_debug_set_linear_mode(0)
json.dump(rows + phase, open("gpurun_out/site_times.json", "w"), indent=1)
