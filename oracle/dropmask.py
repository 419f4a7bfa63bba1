"""ORACLE (test infrastructure only -- never imported by the product path).

Exact host restatement of the dropout keep-mask of the fused kernels, lora_b200/csrc/dropmask.cuh
(`mix32`, `drop_bits`, `drop_threshold`, `drop_keep`), in numpy uint32 wrap-around arithmetic. The
kernels apply nn.Dropout on the LoRA branch (lora_diffusion/lora.py:45,56,115,133) with this mask
instead of ATen's Philox stream; with it, a dropout test compares against the float64 oracle
(oracle/lora_ops.py, keep_mask=...) deterministically instead of recovering the mask from the output.

Element indices (include/lora_b200.h):
  linear  m * N + n
  conv    pixel * Cout + n,  pixel = (img * H + h) * W + w
"""
import numpy as np

_U32 = np.uint32


def mix32(x: np.ndarray) -> np.ndarray:
    """dropmask.cuh `mix32` ("lowbias32" finaliser) on a uint32 array."""
    x = np.asarray(x, dtype=_U32)
    x = x ^ (x >> _U32(16))
    x = x * _U32(0x7FEB352D)
    x = x ^ (x >> _U32(15))
    x = x * _U32(0x846CA68B)
    x = x ^ (x >> _U32(16))
    return x


def drop_bits(s0: int, s1: int, pair: np.ndarray) -> np.ndarray:
    """dropmask.cuh `drop_bits`: one 32-bit hash per element pair (pair = idx >> 1, uint64)."""
    pair = np.asarray(pair, dtype=np.uint64)
    lo = (pair & np.uint64(0xFFFFFFFF)).astype(_U32)
    hi = (pair >> np.uint64(32)).astype(_U32)
    return mix32(mix32(lo ^ _U32(s0)) + hi * _U32(0x9E3779B1) + _U32(s1))


def drop_threshold(p: float) -> int:
    """dropmask.cuh `drop_threshold`: (uint32)(p * 65536.f + 0.5f), evaluated in float32."""
    return int(np.float32(np.float32(p) * np.float32(65536.0) + np.float32(0.5)))


def keep(seed: int, p: float, idx: np.ndarray) -> np.ndarray:
    """dropmask.cuh `drop_keep` for every element index in `idx`: {0, 1} uint8 array of idx's shape.
    `seed` is the int64 the kernels read from device memory (taken as its 64-bit two's complement)."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    idx = np.asarray(idx, dtype=np.uint64)
    bits = drop_bits(seed & 0xFFFFFFFF, seed >> 32, idx >> np.uint64(1))
    lane = np.where((idx & np.uint64(1)) != 0, bits >> _U32(16), bits & _U32(0xFFFF))
    return (lane >= _U32(drop_threshold(p))).astype(np.uint8)


def linear_mask(seed: int, p: float, M: int, N: int) -> np.ndarray:
    """Keep-mask [M, N] of a linear site (element m * N + n)."""
    return keep(seed, p, np.arange(M * N, dtype=np.uint64)).reshape(M, N)


def conv_mask(seed: int, p: float, n_img: int, H: int, W: int, cout: int) -> np.ndarray:
    """Keep-mask of a conv site as an NCHW [n_img, cout, H, W] array (element pixel * cout + n)."""
    m = keep(seed, p, np.arange(n_img * H * W * cout, dtype=np.uint64))
    return np.ascontiguousarray(m.reshape(n_img, H, W, cout).transpose(0, 3, 1, 2))
