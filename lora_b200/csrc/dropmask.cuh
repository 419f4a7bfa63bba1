// Counter-based keep decision for element `idx` of the LoRA-branch output (nn.Dropout on the
// branch, /root/reference/lora_diffusion/lora.py:45,56,115,133). Forward (inside the fused
// kernel's drain) and the backward kernels recompute the same bit from (seed, idx); nothing is
// stored. One 32-bit hash serves the element PAIR (idx >> 1): its low / high 16 bits decide the
// even / odd element, keep iff lane >= round(p * 65536) -- so the fused epilogue, where only four
// warps drain a 128 x BLOCK_N tile, pays 8 integer operations per element instead of a 64-bit
// splitmix per element. The stream differs from ATen's Philox, so parity with the reference under
// dropout is statistical (keep probability 1-p to 8e-6, survivors scaled by 1/(1-p), identical
// mask in forward and backward).
#pragma once
#include <stdint.h>

namespace lb {

__device__ __forceinline__ uint32_t mix32(uint32_t x) {   // "lowbias32" integer finaliser
  x ^= x >> 16;
  x *= 0x7feb352du;
  x ^= x >> 15;
  x *= 0x846ca68bu;
  x ^= x >> 16;
  return x;
}
__device__ __forceinline__ uint32_t drop_bits(uint32_t s0, uint32_t s1, unsigned long long pair) {
  return mix32(mix32(static_cast<uint32_t>(pair) ^ s0) + static_cast<uint32_t>(pair >> 32) * 0x9E3779B1u + s1);
}
__host__ __device__ __forceinline__ uint32_t drop_threshold(float p) {
  return static_cast<uint32_t>(p * 65536.f + 0.5f);
}
__device__ __forceinline__ bool drop_keep(unsigned long long seed, unsigned long long idx, float p) {
  const uint32_t bits = drop_bits(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32), idx >> 1);
  const uint32_t lane = (idx & 1ull) ? (bits >> 16) : (bits & 0xffffu);
  return lane >= drop_threshold(p);
}

}  // namespace lb
