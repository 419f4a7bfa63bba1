// The two ends of a training step, either side of the UNet call:
//   lb_step_prologue      scheduler.add_noise + cast + NCHW -> NHWC (+ the inpainting concat)
//                         cli_lora_pti.py:295-313, train_lora_dreambooth.py:822-840
//   lb_step_prologue_v    the same, plus the v-prediction target scheduler.get_velocity
//                         cli_lora_pti.py:333-338, train_lora_dreambooth.py:846-853
//   lb_masked_mse_fwd_bwd the (mask-weighted) MSE of cli_lora_pti.py:340-370 /
//                         train_lora_dreambooth.py:855-875 and its gradient w.r.t. the prediction,
//                         in one pass (the loss is a scalar: its backward is known in the forward)
// Both are HBM-bound over a few hundred KB: what they buy is launch count (about ten small torch
// kernels per step and their intermediates), not bandwidth.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "lora_b200.h"

namespace lbglue {

__device__ __forceinline__ float ld_any(const void* p, long long i, int dt) {
  if (dt == LB_F32) return reinterpret_cast<const float*>(p)[i];
  if (dt == LB_BF16) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
  return __half2float(reinterpret_cast<const __half*>(p)[i]);
}
__device__ __forceinline__ void st_any(void* p, long long i, int dt, float x) {
  if (dt == LB_F32) reinterpret_cast<float*>(p)[i] = x;
  else if (dt == LB_BF16) reinterpret_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(x);
  else reinterpret_cast<__half*>(p)[i] = __float2half_rn(x);
}

// out[b, p, c] (NHWC, C_out = C or C + 1 + C) = sqrt_acp[t_b] * x0[b, c, p] + sqrt_1m[t_b] * eps[b, c, p]
// for c < C; channel C = inpaint mask[b, p]; channels C+1.. = masked-image latents[b, c', p].
// velocity (optional, fp32 NCHW like x0): v[b, c, p] = sqrt_acp[t_b] * eps[b, c, p] - sqrt_1m[t_b] * x0[b, c, p].
__global__ void __launch_bounds__(256)
prologue_kernel(const float* __restrict__ x0, const float* __restrict__ eps, const long long* __restrict__ t,
                const float* __restrict__ sqrt_acp, const float* __restrict__ sqrt_1m,
                const float* __restrict__ inp_mask, const float* __restrict__ masked_lat, void* __restrict__ out,
                int out_dt, float* __restrict__ velocity, int B, int C, int P, int T) {
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= static_cast<long long>(B) * P) return;
  const int b = static_cast<int>(i / P), px = static_cast<int>(i % P);
  long long tt = t[b];
  tt = tt < 0 ? 0 : (tt >= T ? T - 1 : tt);
  const float a = sqrt_acp[tt], s = sqrt_1m[tt];
  const int c_out = inp_mask ? 2 * C + 1 : C;
  const long long obase = i * c_out;
  for (int c = 0; c < C; ++c) {
    const long long src = (static_cast<long long>(b) * C + c) * P + px;
    const float x = x0[src], e = eps[src];
    // two rounded products and one rounded sum (difference), as torch evaluates add_noise and
    // get_velocity (no FMA contraction): both equal torch's result bit for bit
    st_any(out, obase + c, out_dt, __fadd_rn(__fmul_rn(a, x), __fmul_rn(s, e)));
    if (velocity) velocity[src] = __fsub_rn(__fmul_rn(a, e), __fmul_rn(s, x));   // consecutive px: coalesced
  }
  if (inp_mask) {
    st_any(out, obase + C, out_dt, inp_mask[static_cast<long long>(b) * P + px]);
    for (int c = 0; c < C; ++c)
      st_any(out, obase + C + 1 + c, out_dt, masked_lat[(static_cast<long long>(b) * C + c) * P + px]);
  }
}

// loss = sum_b w_b / (C P) * sum_{c,p} (m[b,p] (pred - target))^2 ;  grad = 2 w_b m^2 (pred - target) / (C P)
// pred / grad: element (b, c, p) at b*sb + c*sc + p*sp (NCHW: sc = P, sp = 1; NHWC: sc = 1, sp = C);
// target: fp32 NCHW. Block partials + last-block reduction in fixed order (deterministic).
__global__ void __launch_bounds__(256)
masked_mse_kernel(const void* __restrict__ pred, int pred_dt, long long sb, long long sc, long long sp,
                  const float* __restrict__ target, const float* __restrict__ mask,
                  const float* __restrict__ weights, void* __restrict__ grad, float* __restrict__ loss,
                  float* __restrict__ partials, unsigned int* __restrict__ counter, int B, int C, int P) {
  __shared__ float sh[8];
  __shared__ bool last;
  const long long total = static_cast<long long>(B) * C * P;
  const float inv_cp = 1.f / (static_cast<float>(C) * static_cast<float>(P));
  float acc = 0.f;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * 256) {
    // i enumerates (b, p, c) with c fastest: coalesced for NHWC predictions, the usual case
    const int c = static_cast<int>(i % C);
    const long long bp = i / C;
    const int px = static_cast<int>(bp % P), b = static_cast<int>(bp / P);
    const long long pi = b * sb + c * sc + px * sp;
    const float d = ld_any(pred, pi, pred_dt) - target[(static_cast<long long>(b) * C + c) * P + px];
    const float m = mask ? mask[static_cast<long long>(b) * P + px] : 1.f;
    const float w = (weights ? weights[b] : 1.f / B) * inv_cp;
    const float md = m * d;
    acc += w * md * md;
    st_any(grad, pi, pred_dt, 2.f * w * m * md);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < 8; ++i) s += sh[i];
    partials[blockIdx.x] = s;
    __threadfence();
    last = atomicAdd(counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence();
    float s = 0.f;
    for (unsigned int i = 0; i < gridDim.x; ++i) s += __ldcg(partials + i);
    loss[0] = s;
    *counter = 0u;
  }
}

}  // namespace lbglue

using namespace lbglue;

static int launch_prologue(const float* latents, const float* noise, const long long* timesteps,
                           const float* sqrt_acp, const float* sqrt_one_minus_acp, int n_timesteps,
                           const float* inpaint_mask, const float* masked_latents, void* out, int out_dtype,
                           float* velocity, int B, int C, int H, int W, void* stream) {
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || n_timesteps <= 0) return LB_ERR_SHAPE;
  if (out_dtype != LB_BF16 && out_dtype != LB_F16 && out_dtype != LB_F32) return LB_ERR_DTYPE;
  if ((inpaint_mask == nullptr) != (masked_latents == nullptr)) return LB_ERR_SHAPE;
  const long long n = static_cast<long long>(B) * H * W;
  prologue_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      latents, noise, timesteps, sqrt_acp, sqrt_one_minus_acp, inpaint_mask, masked_latents, out, out_dtype,
      velocity, B, C, H * W, n_timesteps);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_step_prologue(const float* latents, const float* noise, const long long* timesteps,
                                const float* sqrt_acp, const float* sqrt_one_minus_acp, int n_timesteps,
                                const float* inpaint_mask, const float* masked_latents, void* out,
                                int out_dtype, int B, int C, int H, int W, void* stream) {
  return launch_prologue(latents, noise, timesteps, sqrt_acp, sqrt_one_minus_acp, n_timesteps, inpaint_mask,
                         masked_latents, out, out_dtype, nullptr, B, C, H, W, stream);
}

extern "C" int lb_step_prologue_v(const float* latents, const float* noise, const long long* timesteps,
                                  const float* sqrt_acp, const float* sqrt_one_minus_acp, int n_timesteps,
                                  const float* inpaint_mask, const float* masked_latents, void* out,
                                  int out_dtype, float* velocity, int B, int C, int H, int W, void* stream) {
  if (velocity == nullptr) return LB_ERR_SHAPE;
  return launch_prologue(latents, noise, timesteps, sqrt_acp, sqrt_one_minus_acp, n_timesteps, inpaint_mask,
                         masked_latents, out, out_dtype, velocity, B, C, H, W, stream);
}

extern "C" int lb_masked_mse_fwd_bwd(const void* pred, int pred_dtype, long long stride_b, long long stride_c,
                                     long long stride_p, const float* target, const float* mask,
                                     const float* weights, void* grad, float* loss, float* partials64,
                                     unsigned int* counter, int B, int C, int H, int W, void* stream) {
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0) return LB_ERR_SHAPE;
  if (pred_dtype != LB_BF16 && pred_dtype != LB_F16 && pred_dtype != LB_F32) return LB_ERR_DTYPE;
  if (partials64 == nullptr || counter == nullptr || loss == nullptr || grad == nullptr) return LB_ERR_SHAPE;
  const long long total = static_cast<long long>(B) * C * H * W;
  long long blocks = (total + 256 * 8 - 1) / (256 * 8);
  if (blocks > 64) blocks = 64;
  if (blocks < 1) blocks = 1;
  masked_mse_kernel<<<static_cast<int>(blocks), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      pred, pred_dtype, stride_b, stride_c, stride_p, target, mask, weights, grad, loss, partials64, counter, B, C,
      H * W);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}
