"""In-tree build of the C-ABI library (nvcc, sm_90a only). No torch headers are involved.

`python -m lora_b200.build` or `__graft_entry__.build()`; output: lora_b200/liblora_b200.so
(git-ignored, travels to the GPU box with the gpurun snapshot).
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "liblora_b200.so")
STAMP = os.path.join(HERE, ".liblora_b200.stamp")

SOURCES = ["fused_linear.cu", "fused_conv.cu", "lora_aux.cu", "svd.cu", "svd_batched.cu", "step_glue.cu", "embed_rows.cu"]
# every header under csrc/ takes part in the rebuild digest (a stale .so after a header edit is silent)
HEADERS = sorted(f for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))) + [
    os.path.join(ROOT, "include", "lora_b200.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "-shared",
    "-I", os.path.join(ROOT, "include"), "-I", CSRC,
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _digest(srcs):
    h = hashlib.sha256()
    for f in srcs:
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    hdrs = [h if os.path.isabs(h) else os.path.join(CSRC, h) for h in HEADERS]
    hdrs = [h for h in hdrs if os.path.exists(h)]
    dig = _digest(srcs + hdrs)
    if not force and os.path.exists(OUT) and os.path.exists(STAMP):
        with open(STAMP) as fh:
            if fh.read().strip() == dig:
                return OUT
    cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + srcs + ["-o", OUT]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed building liblora_b200.so")
    with open(STAMP, "w") as fh:
        fh.write(dig)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
