"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list: time per kernel family,
share of the step. Usage: python scripts/summarize_launches.py launches.csv [first_id last_id | last]
(`last` = the launches of the LAST training step only: everything after the second-to-last optimizer launch)"""
import csv, re, sys, collections

path = sys.argv[1]
rows = []
with open(path) as fh:
    lines = [l for l in fh if l.startswith('"')]
rd = csv.reader(lines)
hdr = next(rd)
ik, iv, iid = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("ID")
for r in rd:
    rows.append((int(r[iid]), r[ik], float(r[iv].replace(",", ""))))
if len(sys.argv) > 2 and sys.argv[2] == "last":
    opt = [i for i, r in enumerate(rows) if re.search(r"optim_step_(fused|dp)_kernel", r[1])]
    if len(opt) >= 2:
        rows = rows[opt[-2] + 1: opt[-1] + 1]
else:
    lo = int(sys.argv[2]) if len(sys.argv) > 2 else 0
    hi = int(sys.argv[3]) if len(sys.argv) > 3 else 10 ** 9
    rows = [r for r in rows if lo <= r[0] <= hi]


def family(name):
    n = name
    for pat, fam in [(r"fused_lora", "OURS fused_lora (wgmma fwd/dX)"), (r"wgrad_kernel", "OURS wgrad (dA/dB)"),
                     (r"optim_step_", "OURS clip+AdamW (one launch)"), (r"prologue_kernel|masked_mse_kernel", "OURS step prologue / loss"), (r"refresh_shadows|cast_rows|cast_weight|cast_conv", "OURS casts/shadows"),
                     (r"up_dropout|dropout_dt", "OURS dropout branch"),
                     (r"fmha|flash|attention|sdp", "attention (SDPA)"), (r"cudnn|conv|implicit_gemm|xmma|cutlass.*conv|sm\d+_xmma|wgrad|dgrad", "cuDNN conv"),
                     (r"nvjet|gemm|cublas|gemv|cutlass", "cuBLAS GEMM (non-LoRA linears)"),
                     (r"group_norm|GroupNorm|RowwiseMoments|ComputeFusedParams|GammaBeta|ComputeInternalGradients|ComputeBackwardFusedParams", "GroupNorm"),
                     (r"layer_norm|LayerNorm|layernorm", "LayerNorm"),
                     (r"elementwise|vectorized|unrolled|copy|Copy|fill|cat|Cat|index|gelu|silu|reduce|upsample|nearest|softmax", "ATen elementwise/copy/reduce")]:
        if re.search(pat, n):
            return fam
    return "other: " + n[:60]


tot = sum(r[2] for r in rows)
fam = collections.defaultdict(lambda: [0, 0.0])
for _, k, v in rows:
    f = family(k)
    fam[f][0] += 1
    fam[f][1] += v
print(f"launches {len(rows)}  total {tot/1e6:.3f} ms (cold-cache, serialised: compare SHARES)")
for f, (c, v) in sorted(fam.items(), key=lambda kv: -kv[1][1]):
    print(f"{v/1e6:9.3f} ms {100*v/tot:6.2f}%  n={c:5d}  avg {v/c/1e3:8.2f} us  {f}")
