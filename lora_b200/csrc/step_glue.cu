// The two ends of a training step, either side of the UNet call:
//   lb_pixels_ingest      uint8 HWC images -> ToTensor + Normalize([0.5], [0.5]) -> the VAE's dtype and
//                         layout (+ the inpainting masked image), dataset.py:108-116, 240-252
//   lb_step_prologue      scheduler.add_noise + cast + NCHW -> NHWC (+ the inpainting concat)
//                         cli_lora_pti.py:295-313, train_lora_dreambooth.py:822-840
//   lb_step_prologue_v    the same, plus the v-prediction target scheduler.get_velocity
//                         cli_lora_pti.py:333-338, train_lora_dreambooth.py:846-853
//   lb_step_prologue_posterior  the same with the VAE posterior sample in front:
//                         latent_dist.sample() * 0.18215 (+ the latent-grid inpainting mask),
//                         train_lora_dreambooth.py:818-821, cli_lora_pti.py:273-290
//   lb_masked_mse_fwd_bwd the (mask-weighted) MSE of cli_lora_pti.py:340-370 /
//                         train_lora_dreambooth.py:855-875 and its gradient w.r.t. the prediction,
//                         in one pass (the loss is a scalar: its backward is known in the forward),
//                         optionally times the fp16 loss scale (GradScaler.scale(loss).backward())
// and the two ends of a sampling step (the denoising loop of diffusers' StableDiffusionPipeline):
//   lb_sample_step        the guidance sum, the scheduler's update as folded coefficients, the next UNet
//                         input and timestep (+ the decoder input on the last step); or, with init, the
//                         first UNet input from the initial noise
//   lb_sample_step_ch     the same into a UNet input of more channels than the latents (the 9-channel
//                         inpainting UNet): only the latent channels are written
//   lb_sample_step_ms     the same for a multistep scheduler (DPM-Solver++(2M)): the data prediction, the
//                         update from it and the previous step's, and that history kept in place
//   lb_sample_step_rescale  either step (single-step or multistep) with guidance rescale: the per-sample
//                         std ratio of the conditional and guided predictions, in the same one launch
//   lb_sample_init       the start of an img2img or inpainting loop: the posterior sample of the encoded
//                         image, scheduler.add_noise at the first kept timestep, the first UNet input,
//                         and for inpainting the constant mask and masked-image channels
//   lb_pixels_ingest_inpaint  uint8 image + uint8 0..255 mask -> the inpainting pipeline's masked image
//                         (prepare_mask_and_masked_image) in the VAE's dtype and layout
//   lb_pixels_emit        the decoded image -> (x / 2 + 0.5).clamp(0, 1) -> uint8 HWC (numpy_to_pil)
// All are HBM-bound over a few hundred KB (a few MB of pixels): what they buy is launch count (about
// ten small torch kernels per step and their intermediates), not bandwidth.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "lora_b200.h"

namespace cg = cooperative_groups;

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
// x rounded to dt and widened back: torch's result of one bf16 / fp16 op evaluated in fp32
__device__ __forceinline__ float round_to(int dt, float x) {
  if (dt == LB_BF16) return __bfloat162float(__float2bfloat16_rn(x));
  if (dt == LB_F16) return __half2float(__float2half_rn(x));
  return x;
}

// two rounded products and one rounded sum (difference), as torch evaluates add_noise and
// get_velocity (no FMA contraction): both equal torch's result bit for bit
__device__ __forceinline__ void noise_one(void* out, long long o, int out_dt, float* velocity, long long src,
                                          float a, float s, float x, float e) {
  st_any(out, o, out_dt, __fadd_rn(__fmul_rn(a, x), __fmul_rn(s, e)));
  if (velocity) velocity[src] = __fsub_rn(__fmul_rn(a, e), __fmul_rn(s, x));   // consecutive px: coalesced
}

__device__ __forceinline__ float clamp_timestep_coef(const long long* t, const float* tab, int b, int T) {
  long long tt = t[b];
  tt = tt < 0 ? 0 : (tt >= T ? T - 1 : tt);
  return tab[tt];
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
  const float a = clamp_timestep_coef(t, sqrt_acp, b, T), s = clamp_timestep_coef(t, sqrt_1m, b, T);
  const int c_out = inp_mask ? 2 * C + 1 : C;
  const long long obase = i * c_out;
  for (int c = 0; c < C; ++c) {
    const long long src = (static_cast<long long>(b) * C + c) * P + px;
    noise_one(out, obase + c, out_dt, velocity, src, a, s, x0[src], eps[src]);
  }
  if (inp_mask) {
    st_any(out, obase + C, out_dt, inp_mask[static_cast<long long>(b) * P + px]);
    for (int c = 0; c < C; ++c)
      st_any(out, obase + C + 1 + c, out_dt, masked_lat[(static_cast<long long>(b) * C + c) * P + px]);
  }
}

// One pixel of torchvision's ToTensor + Normalize([0.5], [0.5]) on a uint8 value, op by op as the
// data loader evaluates it on the CPU: x.float() / 255, then (x - 0.5) / 0.5, each rounded once.
__device__ __forceinline__ float normalise_u8(unsigned char v) {
  return __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(v), 255.f), 0.5f), 0.5f);
}

// diffusers' prepare_mask_and_masked_image on one uint8 L-mode mask value: v / 255 in fp32, then
// binarised (< 0.5 -> 0, >= 0.5 -> 1). 127 -> 0, 128 -> 1.
__device__ __forceinline__ float binarise_u8(unsigned char v) {
  return __fdiv_rn(static_cast<float>(v), 255.f) < 0.5f ? 0.f : 1.f;
}

enum { MASK_F32 = 0, MASK_U8 = 1, MASK_U8_PIPELINE = 2 };

// out (VAE input, [B, 3, H, W] NCHW or channels_last, out_dt) <- pixels: uint8 [B, H, W, 3] (normalised
// here) or fp32 [B, 3, H, W] (already normalised: a cast). With mask [B, 1, H, W]: masked = image *
// (mask < 0.5), the product in fp32, then the same cast. mask_mode MASK_F32 / MASK_U8: the mask's value
// as stored (the training dataset's 0 / 1 mask, dataset.py:115); MASK_U8_PIPELINE: a 0..255 mask
// binarised first (binarise_u8). out may be NULL when only the masked image is wanted.
__global__ void __launch_bounds__(256)
pixels_ingest_kernel(const void* __restrict__ pixels, int pixels_u8, const void* __restrict__ mask, int mask_mode,
                     void* __restrict__ out, void* __restrict__ masked, int out_dt, int channels_last, int B,
                     long long P) {
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= B * P) return;
  const long long b = i / P, p = i % P;
  float keep = 0.f;
  if (mask) {
    const unsigned char* m8 = reinterpret_cast<const unsigned char*>(mask);
    const float m = mask_mode == MASK_U8_PIPELINE ? binarise_u8(m8[i])
                    : mask_mode == MASK_U8        ? static_cast<float>(m8[i])
                                                  : reinterpret_cast<const float*>(mask)[i];
    keep = m < 0.5f ? 1.f : 0.f;          // NaN < 0.5 is false, as in torch
  }
  for (int c = 0; c < 3; ++c) {
    const long long nchw = (b * 3 + c) * P + p;
    const float x = pixels_u8 ? normalise_u8(reinterpret_cast<const unsigned char*>(pixels)[i * 3 + c])
                              : reinterpret_cast<const float*>(pixels)[nchw];
    const long long o = channels_last ? i * 3 + c : nchw;
    if (out) st_any(out, o, out_dt, x);
    if (mask) st_any(masked, o, out_dt, __fmul_rn(x, keep));   // x * 0 keeps the sign of x, as torch does
  }
}

// diffusers' DiagonalGaussianDistribution(moments).sample() * scaling, each op rounded as torch rounds
// it: logvar.clamp(-30, 20) -> std = exp(0.5 * logvar) in the moments' dtype md; std * eps and
// mean + that in the promoted dtype td (md when eps has md, else fp32); then * scaling in td.
__device__ __forceinline__ float posterior_sample(const void* mom, int md, long long i_mean, long long i_logvar,
                                                  const void* post_eps, int ed, long long i_eps, int td,
                                                  float scaling) {
  const float mean = ld_any(mom, i_mean, md);
  float lv = ld_any(mom, i_logvar, md);
  lv = lv < -30.f ? -30.f : (lv > 20.f ? 20.f : lv);     // torch.clamp: NaN stays NaN
  const float sd = round_to(md, expf(round_to(md, __fmul_rn(0.5f, lv))));
  const float x = round_to(td, __fadd_rn(mean, round_to(td, __fmul_rn(sd, ld_any(post_eps, i_eps, ed)))));
  return round_to(td, __fmul_rn(x, scaling));
}

// prologue_kernel's output from VAE moments instead of latents: latents[b, c, p] = the posterior sample
// (moments element (b, c, p) at b*sb + c*sc + p*sp, logvar C channels further; post_eps fp32 NCHW or
// the moments' dtype), written out in fp32 and noised as prologue_kernel does. Inpainting (mask != NULL):
// the latent-grid mask is mask[b, 0, 8h, 8w] of the image-resolution mask (F.interpolate(scale_factor=
// 1/8), nearest), the masked-image latents the posterior sample of the masked moments; both are written
// out (fp32 NCHW) and into the concat.
__global__ void __launch_bounds__(256)
prologue_posterior_kernel(const void* __restrict__ mom, int md, long long sb, long long sc, long long sp,
                          const void* __restrict__ post_eps, int ed, float scaling, float* __restrict__ lat_out,
                          const void* __restrict__ mmom, const void* __restrict__ mpost_eps,
                          const void* __restrict__ mask, int mask_u8, float* __restrict__ mlat_out,
                          float* __restrict__ mask_out, const float* __restrict__ eps,
                          const long long* __restrict__ t, const float* __restrict__ sqrt_acp,
                          const float* __restrict__ sqrt_1m, void* __restrict__ out, int out_dt,
                          float* __restrict__ velocity, int B, int C, int H, int W, int T) {
  const int P = H * W;
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= static_cast<long long>(B) * P) return;
  const int b = static_cast<int>(i / P), px = static_cast<int>(i % P);
  const float a = clamp_timestep_coef(t, sqrt_acp, b, T), s = clamp_timestep_coef(t, sqrt_1m, b, T);
  const int td = ed == md ? md : LB_F32;
  const int c_out = mask ? 2 * C + 1 : C;
  const long long obase = i * c_out;
  const long long mbase = b * sb + px * sp;
  for (int c = 0; c < C; ++c) {
    const long long src = (static_cast<long long>(b) * C + c) * P + px;
    const long long mi = mbase + c * sc;
    const float x = posterior_sample(mom, md, mi, mi + C * sc, post_eps, ed, src, td, scaling);
    lat_out[src] = x;
    noise_one(out, obase + c, out_dt, velocity, src, a, s, x, eps[src]);
  }
  if (mask) {
    const int h = px / W, w = px % W;
    const long long mpix = (static_cast<long long>(b) * 8 * H + 8 * h) * (8ll * W) + 8 * w;
    const float m = mask_u8 ? static_cast<float>(reinterpret_cast<const unsigned char*>(mask)[mpix])
                            : reinterpret_cast<const float*>(mask)[mpix];
    mask_out[static_cast<long long>(b) * P + px] = m;
    st_any(out, obase + C, out_dt, m);
    for (int c = 0; c < C; ++c) {
      const long long src = (static_cast<long long>(b) * C + c) * P + px;
      const long long mi = mbase + c * sc;
      const float x = posterior_sample(mmom, md, mi, mi + C * sc, mpost_eps, ed, src, td, scaling);
      mlat_out[src] = x;
      st_any(out, obase + C + 1 + c, out_dt, x);
    }
  }
}

// loss = sum_b w_b / (C P) * sum_{c,p} (m[b,p] (pred - target))^2 ;  grad = 2 w_b m^2 (pred - target) / (C P)
// pred / grad: element (b, c, p) at b*sb + c*sc + p*sp (NCHW: sc = P, sp = 1; NHWC: sc = 1, sp = C);
// target: fp32 NCHW. Block partials + last-block reduction in fixed order (deterministic).
__global__ void __launch_bounds__(256)
masked_mse_kernel(const void* __restrict__ pred, int pred_dt, long long sb, long long sc, long long sp,
                  const float* __restrict__ target, const float* __restrict__ mask,
                  const float* __restrict__ weights, void* __restrict__ grad, float* __restrict__ loss,
                  float* __restrict__ partials, unsigned int* __restrict__ counter, int B, int C, int P,
                  const float* __restrict__ grad_scale) {
  __shared__ float sh[8];
  __shared__ bool last;
  const long long total = static_cast<long long>(B) * C * P;
  const float inv_cp = 1.f / (static_cast<float>(C) * static_cast<float>(P));
  const float gs = grad_scale ? grad_scale[0] : 1.f;
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
    const float gd = 2.f * w * m * md;
    // the loss scale multiplies the finished fp32 gradient (one more rounding, exact for a power of
    // two); NULL leaves the product untouched
    st_any(grad, pi, pred_dt, grad_scale ? __fmul_rn(gd, gs) : gd);
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

// One sampling step, element (b, c, p) of the latents [B, C, P] (fp32 NCHW), step row k = 1 + *step_index
// of the [rows, 8] table: (alpha, beta, gamma, s_next, t_next, last, -, -):
//   m_hat = m_u + g (m_c - m_u)      (G = 2: m_u row b, m_c row B + b of the UNet output; G = 1: m_hat = m)
//   x'    = alpha x + beta m_hat + gamma z      (z: noise slice k of [rows, B, C, P]; unread when gamma = 0)
//   unet_in[g B + b, c, p] = (s_next x') in the UNet's dtype, NHWC with Cu >= C channels (only channels
//   [0, C) are written: the inpainting UNet's mask and masked-image channels stay as sample_init_kernel
//   wrote them), for each of the G halves
//   last row: vae_in[b, c, p] = (1 / scaling) x' in the VAE's dtype (NCHW or NHWC), the pipeline's
//   `1 / scaling * latents` with the reciprocal rounded to fp32 as torch rounds a scalar factor
// init: x = z_0 * init_noise_sigma (row 0: (sigma, s_0, t_0)), the first UNet input and timestep, and the
// step index and arrival counter reset. Every block reads *step_index; the last block to arrive
// advances it, so one captured launch replays as every step in turn.
// MS (the multistep family, lb_sample_step_ms; no init, no noise): row 1 + i is
// (a, b, d, s_next, t_next, last, p, q) and, with h = x0_hist [B, C, P] fp32 NCHW,
//   x0 = p x + q m_hat        (the data prediction: convert_model_output of DPM-Solver++)
//   x' = a x + b x0 + d h     (h unread when d = 0);  then h = x0, in place
// Each element of x and h is read and written by the one thread that owns it.
template <bool MS>
__global__ void __launch_bounds__(256)
sample_step_kernel(const void* __restrict__ mo, int mdt, long long sb, long long sc, long long sp, int G,
                   float* __restrict__ x, const float* __restrict__ noise, float* __restrict__ x0_hist,
                   const float* __restrict__ table, int rows, const float* __restrict__ guidance,
                   int* __restrict__ step_index, unsigned int* __restrict__ counter, void* __restrict__ unet_in,
                   int udt, int Cu, float* __restrict__ timestep, void* __restrict__ vae_in, int vdt, int vae_cl,
                   float vae_inv_scaling, int B, int C, int P, int init_arg) {
  const bool init = !MS && init_arg;
  __shared__ int s_row;
  __shared__ bool last_block;
  if (threadIdx.x == 0) {
    int k = init ? 0 : 1 + *step_index;
    s_row = k < 0 ? 0 : (k >= rows ? rows - 1 : k);
  }
  __syncthreads();
  const float* row = table + 8ll * s_row;
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  const long long slice = static_cast<long long>(B) * C * P;
  if (i < static_cast<long long>(B) * P) {
    const int b = static_cast<int>(i / P), px = static_cast<int>(i % P);
    float s_next, alpha = 0.f, beta = 0.f, gamma = 0.f, g = 0.f, p = 0.f, q = 0.f;
    bool last = false;
    if (init) {
      s_next = row[1];
    } else {
      alpha = row[0]; beta = row[1]; gamma = row[2]; s_next = row[3]; last = row[5] != 0.f;
      g = *guidance;
      if (MS) { p = row[6]; q = row[7]; }
    }
    const float* z = MS ? nullptr : noise + (init ? 0ll : s_row * slice);
    for (int c = 0; c < C; ++c) {
      const long long xi = (static_cast<long long>(b) * C + c) * P + px;
      float xn;
      if (init) {
        xn = __fmul_rn(z[xi], row[0]);
      } else {
        float m = ld_any(mo, b * sb + c * sc + px * sp, mdt);
        if (G == 2) {
          const float mc = ld_any(mo, (B + b) * sb + c * sc + px * sp, mdt);
          m = fmaf(g, mc - m, m);
        }
        if (MS) {
          const float xc = x[xi];
          const float x0 = fmaf(p, xc, q * m);
          xn = fmaf(alpha, xc, beta * x0);
          if (gamma != 0.f) xn = fmaf(gamma, x0_hist[xi], xn);
          x0_hist[xi] = x0;
        } else {
          xn = fmaf(alpha, x[xi], beta * m);
          if (gamma != 0.f) xn = fmaf(gamma, z[xi], xn);
        }
      }
      x[xi] = xn;
      const float u = __fmul_rn(s_next, xn);
      for (int h = 0; h < G; ++h) st_any(unet_in, (static_cast<long long>(h * B + b) * P + px) * Cu + c, udt, u);
      if (last) st_any(vae_in, vae_cl ? i * C + c : xi, vdt, __fmul_rn(vae_inv_scaling, xn));
    }
  }
  if (init) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      *timestep = row[2];
      *step_index = 0;
      *counter = 0u;
    }
    return;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *timestep = row[4];
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    last_block = atomicAdd(counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (last_block && threadIdx.x == 0) {
    *step_index += 1;
    *counter = 0u;
    __threadfence();
  }
}

// lb_sample_step_rescale: sample_step_kernel's step (G = 2) with guidance rescale ("Common Diffusion Noise
// Schedules are Flawed", diffusers' rescale_noise_cfg) between the guidance sum and the update:
//   m_hat = m_u + g (m_c - m_u);  r_b = std(m_c[b]) / std(m_hat[b]) (unbiased, over C x P; the (n - 1)
//   cancels in the ratio);  m_hat <- k_b m_hat,  k_b = fl32(1 + phi (r_b - 1)) = phi r_b + (1 - phi)
// k_b is exactly 1 at phi = 0 (set so, whatever r_b is), and m_hat * 1 is m_hat bit for bit: the update
// then equals sample_step_kernel's, whose float operations this kernel repeats in the same order.
//
// The statistics of sample b need every element of b before any element can be updated, so the launch
// is one 8-CTA thread-block cluster per sample (8 is the portable cluster size; grid (8, B)). Its CTAs
// stride over the sample's pixels twice. Pass 1 sums (m_c, m_c^2, m_hat, m_hat^2) in fp64 per thread,
// then over the warp by shuffles, over the CTA in warp order, and over the cluster through distributed
// shared memory in rank order: a fixed order, so replays are bit-reproducible. A cluster barrier needs no
// grid-wide co-residency (a cooperative launch would) and keeps the whole exchange on chip. Pass 2
// re-reads the model output (L2-resident: 256 KiB at 128 x 128 latents in bf16) and applies the update.
// The step index advances as in sample_step_kernel: every CTA reads it first, the last CTA to arrive
// advances it, so one captured launch replays as every step. MS selects lb_sample_step_ms's update.
constexpr int RS_CLUSTER = 8;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <bool MS>
__global__ void __cluster_dims__(RS_CLUSTER, 1, 1) __launch_bounds__(256)
sample_step_rescale_kernel(const void* __restrict__ mo, int mdt, long long sb, long long sc, long long sp,
                           float* __restrict__ x, const float* __restrict__ noise, float* __restrict__ x0_hist,
                           const float* __restrict__ table, int rows, const float* __restrict__ guidance,
                           const float* __restrict__ guidance_rescale, int* __restrict__ step_index,
                           unsigned int* __restrict__ counter, void* __restrict__ unet_in, int udt, int Cu,
                           float* __restrict__ timestep, void* __restrict__ vae_in, int vdt, int vae_cl,
                           float vae_inv_scaling, int B, int C, int P) {
  cg::cluster_group cluster = cg::this_cluster();
  __shared__ int s_row;
  __shared__ double s_warp[8][4];
  __shared__ double s_part[4];
  __shared__ float s_k;
  __shared__ bool last_block;
  if (threadIdx.x == 0) {
    const int k = 1 + *step_index;
    s_row = k < 0 ? 0 : (k >= rows ? rows - 1 : k);
  }
  __syncthreads();
  const float* row = table + 8ll * s_row;
  const int b = blockIdx.y;
  const int stride = RS_CLUSTER * 256;
  const int first = static_cast<int>(cluster.block_rank()) * 256 + threadIdx.x;
  const float g = *guidance;
  const long long ub = static_cast<long long>(b) * sb, cb = static_cast<long long>(B + b) * sb;

  double acc[4] = {0.0, 0.0, 0.0, 0.0};       // sum m_c, sum m_c^2, sum m_hat, sum m_hat^2
  for (int px = first; px < P; px += stride) {
    for (int c = 0; c < C; ++c) {
      const long long o = c * sc + px * sp;
      const float mu = ld_any(mo, ub + o, mdt), mc = ld_any(mo, cb + o, mdt);
      const double dc = mc, dh = fmaf(g, mc - mu, mu);
      acc[0] += dc;
      acc[1] += dc * dc;
      acc[2] += dh;
      acc[3] += dh * dh;
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const double v = warp_sum(acc[j]);
    if (lane == 0) s_warp[warp][j] = v;
  }
  __syncthreads();
  if (threadIdx.x < 4) {
    double v = 0.0;
    for (int w = 0; w < 8; ++w) v += s_warp[w][threadIdx.x];
    s_part[threadIdx.x] = v;
  }
  cluster.sync();
  if (threadIdx.x == 0) {
    double a[4] = {0.0, 0.0, 0.0, 0.0};
    for (unsigned int r = 0; r < RS_CLUSTER; ++r) {
      const double* part = cluster.map_shared_rank(s_part, r);
#pragma unroll
      for (int j = 0; j < 4; ++j) a[j] += part[j];
    }
    const double n = static_cast<double>(C) * P;
    const double ss_c = a[1] - a[0] * a[0] / n, ss_h = a[3] - a[2] * a[2] / n;
    const double phi = *guidance_rescale;
    s_k = phi == 0.0 ? 1.f : static_cast<float>(1.0 + phi * (sqrt(ss_c / ss_h) - 1.0));
  }
  cluster.sync();            // s_k is set, and no CTA leaves while another still reads its s_part

  const float kf = s_k;
  const float alpha = row[0], beta = row[1], gamma = row[2], s_next = row[3];
  const bool last = row[5] != 0.f;
  const float p = MS ? row[6] : 0.f, q = MS ? row[7] : 0.f;
  const long long slice = static_cast<long long>(B) * C * P;
  const float* z = MS ? nullptr : noise + s_row * slice;
  for (int px = first; px < P; px += stride) {
    const long long i = static_cast<long long>(b) * P + px;
    for (int c = 0; c < C; ++c) {
      const long long xi = (static_cast<long long>(b) * C + c) * P + px;
      const long long o = c * sc + px * sp;
      float m = ld_any(mo, ub + o, mdt);
      const float mc = ld_any(mo, cb + o, mdt);
      m = fmaf(g, mc - m, m);
      m = __fmul_rn(m, kf);
      float xn;
      if (MS) {
        const float xc = x[xi];
        const float x0 = fmaf(p, xc, q * m);
        xn = fmaf(alpha, xc, beta * x0);
        if (gamma != 0.f) xn = fmaf(gamma, x0_hist[xi], xn);
        x0_hist[xi] = x0;
      } else {
        xn = fmaf(alpha, x[xi], beta * m);
        if (gamma != 0.f) xn = fmaf(gamma, z[xi], xn);
      }
      x[xi] = xn;
      const float u = __fmul_rn(s_next, xn);
      for (int h = 0; h < 2; ++h) st_any(unet_in, (static_cast<long long>(h * B + b) * P + px) * Cu + c, udt, u);
      if (last) st_any(vae_in, vae_cl ? i * C + c : xi, vdt, __fmul_rn(vae_inv_scaling, xn));
    }
  }
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *timestep = row[4];
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    last_block = atomicAdd(counter, 1u) == gridDim.x * gridDim.y - 1;
  }
  __syncthreads();
  if (last_block && threadIdx.x == 0) {
    *step_index += 1;
    *counter = 0u;
    __threadfence();
  }
}

// The start of an img2img or inpainting sampling loop (StableDiffusionImg2ImgPipeline /
// StableDiffusionInpaintPipeline), element (b, c, p) of the latents [B, C, P], from row 0 of the table:
// (c_noise, s_start, t_start, c_lat). With moments and no mask (img2img):
//   lat = the posterior sample of the image's moments * scaling (posterior_sample)
//   x   = fl(fl(c_lat lat) + fl(c_noise z_0))       scheduler.add_noise(init_latents, z_0, t_start)
// Without moments, or with the mask (inpainting): x = z_0 * c_noise (randn * init_noise_sigma).
// unet_in[g B + b, :, p] (NHWC, Cu channels) = s_start x in channels [0, C) of each of the G halves; with
// the mask also channel C = the binarised mask at pixel (8h, 8w) of the image-resolution uint8 mask
// (F.interpolate to the latent grid, nearest) and channels C+1 .. 2C = the posterior sample of the
// masked image's moments * scaling. Those channels are constant over the loop: only this launch writes
// them. Then *timestep = t_start, and the step index and arrival counter reset as lb_sample_step's init.
__global__ void __launch_bounds__(256)
sample_init_kernel(const void* __restrict__ mom, int md, long long sb, long long sc, long long sp,
                   const void* __restrict__ post_eps, int ed, float scaling,
                   const unsigned char* __restrict__ mask, const float* __restrict__ noise,
                   const float* __restrict__ table, float* __restrict__ x, int* __restrict__ step_index,
                   unsigned int* __restrict__ counter, void* __restrict__ unet_in, int udt, int Cu,
                   float* __restrict__ timestep, int G, int B, int C, int H, int W) {
  const int P = H * W;
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    *timestep = table[2];
    *step_index = 0;
    *counter = 0u;
  }
  if (i >= static_cast<long long>(B) * P) return;
  const int b = static_cast<int>(i / P), px = static_cast<int>(i % P);
  const float c_noise = table[0], s = table[1], c_lat = table[3];
  const int td = ed == md ? md : LB_F32;
  const bool from_image = mom != nullptr && mask == nullptr;
  const long long mbase = b * sb + px * sp;
  for (int c = 0; c < C; ++c) {
    const long long xi = (static_cast<long long>(b) * C + c) * P + px;
    float xn;
    if (from_image) {
      const long long mi = mbase + c * sc;
      const float lat = posterior_sample(mom, md, mi, mi + C * sc, post_eps, ed, xi, td, scaling);
      xn = __fadd_rn(__fmul_rn(c_lat, lat), __fmul_rn(c_noise, noise[xi]));
    } else {
      xn = __fmul_rn(noise[xi], c_noise);
    }
    x[xi] = xn;
    const float u = __fmul_rn(s, xn);
    for (int h = 0; h < G; ++h) st_any(unet_in, (static_cast<long long>(h * B + b) * P + px) * Cu + c, udt, u);
  }
  if (mask) {
    const int h = px / W, w = px % W;
    const float m = binarise_u8(mask[(static_cast<long long>(b) * 8 * H + 8 * h) * (8ll * W) + 8 * w]);
    for (int g = 0; g < G; ++g) st_any(unet_in, (static_cast<long long>(g * B + b) * P + px) * Cu + C, udt, m);
    for (int c = 0; c < C; ++c) {
      const long long mi = mbase + c * sc;
      const long long xi = (static_cast<long long>(b) * C + c) * P + px;
      const float ml = posterior_sample(mom, md, mi, mi + C * sc, post_eps, ed, xi, td, scaling);
      for (int g = 0; g < G; ++g)
        st_any(unet_in, (static_cast<long long>(g * B + b) * P + px) * Cu + C + 1 + c, udt, ml);
    }
  }
}

// diffusers' image post-processing, op by op: (image / 2 + 0.5).clamp(0, 1), each op rounded in the
// image's dtype; then .float() * 255, round half to even, cast to uint8 (numpy_to_pil). in: [B, 3, P]
// NCHW or NHWC; out: uint8 [B, P, 3].
__global__ void __launch_bounds__(256)
pixels_emit_kernel(const void* __restrict__ img, int dt, int channels_last, unsigned char* __restrict__ out, int B,
                   long long P) {
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= B * P) return;
  const long long b = i / P, p = i % P;
  for (int c = 0; c < 3; ++c) {
    const float v = ld_any(img, channels_last ? i * 3 + c : (b * 3 + c) * P + p, dt);
    float y = round_to(dt, __fadd_rn(round_to(dt, __fdiv_rn(v, 2.f)), 0.5f));
    y = y < 0.f ? 0.f : (y > 1.f ? 1.f : y);       // NaN stays NaN
    const float q = rintf(__fmul_rn(y, 255.f));
    out[i * 3 + c] = q == q ? static_cast<unsigned char>(q) : 0;
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

static bool float_dtype(int dt) { return dt == LB_BF16 || dt == LB_F16 || dt == LB_F32; }

extern "C" int lb_pixels_ingest(const void* pixels, int pixels_u8, const void* mask, int mask_u8, void* out,
                                void* masked_out, int out_dtype, int channels_last, int B, int H, int W,
                                void* stream) {
  if (B <= 0 || H <= 0 || W <= 0 || pixels == nullptr || out == nullptr) return LB_ERR_SHAPE;
  if (!float_dtype(out_dtype)) return LB_ERR_DTYPE;
  if ((mask == nullptr) != (masked_out == nullptr)) return LB_ERR_SHAPE;
  const long long P = static_cast<long long>(H) * W, n = B * P;
  pixels_ingest_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      pixels, pixels_u8 != 0, mask, mask_u8 != 0, out, masked_out, out_dtype, channels_last != 0, B, P);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_step_prologue_posterior(const void* moments, int moments_dtype, long long stride_b,
                                          long long stride_c, long long stride_p, const void* posterior_noise,
                                          int posterior_noise_dtype, float scaling, float* latents,
                                          const void* masked_moments, const void* masked_posterior_noise,
                                          const void* mask, int mask_u8, float* masked_latents,
                                          float* inpaint_mask, const float* noise, const long long* timesteps,
                                          const float* sqrt_acp, const float* sqrt_one_minus_acp,
                                          int n_timesteps, void* out, int out_dtype, float* velocity, int B,
                                          int C, int H, int W, void* stream) {
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || n_timesteps <= 0) return LB_ERR_SHAPE;
  if (!float_dtype(moments_dtype) || !float_dtype(out_dtype)) return LB_ERR_DTYPE;
  if (posterior_noise_dtype != moments_dtype && posterior_noise_dtype != LB_F32) return LB_ERR_DTYPE;
  if (moments == nullptr || posterior_noise == nullptr || latents == nullptr) return LB_ERR_SHAPE;
  const bool inp = mask != nullptr;
  if (inp && (masked_moments == nullptr || masked_posterior_noise == nullptr || masked_latents == nullptr ||
              inpaint_mask == nullptr))
    return LB_ERR_SHAPE;
  const long long n = static_cast<long long>(B) * H * W;
  prologue_posterior_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      moments, moments_dtype, stride_b, stride_c, stride_p, posterior_noise, posterior_noise_dtype, scaling,
      latents, masked_moments, masked_posterior_noise, mask, mask_u8 != 0, masked_latents, inpaint_mask, noise,
      timesteps, sqrt_acp, sqrt_one_minus_acp, out, out_dtype, velocity, B, C, H, W, n_timesteps);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_masked_mse_fwd_bwd(const void* pred, int pred_dtype, long long stride_b, long long stride_c,
                                     long long stride_p, const float* target, const float* mask,
                                     const float* weights, void* grad, float* loss, float* partials64,
                                     unsigned int* counter, int B, int C, int H, int W, const float* grad_scale,
                                     void* stream) {
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0) return LB_ERR_SHAPE;
  if (pred_dtype != LB_BF16 && pred_dtype != LB_F16 && pred_dtype != LB_F32) return LB_ERR_DTYPE;
  if (partials64 == nullptr || counter == nullptr || loss == nullptr || grad == nullptr) return LB_ERR_SHAPE;
  const long long total = static_cast<long long>(B) * C * H * W;
  long long blocks = (total + 256 * 8 - 1) / (256 * 8);
  if (blocks > 64) blocks = 64;
  if (blocks < 1) blocks = 1;
  masked_mse_kernel<<<static_cast<int>(blocks), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      pred, pred_dtype, stride_b, stride_c, stride_p, target, mask, weights, grad, loss, partials64, counter, B, C,
      H * W, grad_scale);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_pixels_ingest_inpaint(const void* pixels, const unsigned char* mask, void* masked_out,
                                        int out_dtype, int channels_last, int B, int H, int W, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0 || pixels == nullptr || mask == nullptr || masked_out == nullptr)
    return LB_ERR_SHAPE;
  if (!float_dtype(out_dtype)) return LB_ERR_DTYPE;
  const long long P = static_cast<long long>(H) * W, n = B * P;
  pixels_ingest_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      pixels, 1, mask, MASK_U8_PIPELINE, nullptr, masked_out, out_dtype, channels_last != 0, B, P);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

// MS: the multistep launch (lb_sample_step_ms): x0_hist in place of noise, never init
template <bool MS>
static int launch_sample_step(const void* model_out, int model_dtype, long long stride_b, long long stride_c,
                              long long stride_p, int G, float* x, const float* noise, float* x0_hist,
                              const float* table, int table_rows, const float* guidance, int* step_index,
                              unsigned int* counter, void* unet_in, int unet_dtype, int unet_channels,
                              float* timestep, void* vae_in, int vae_dtype, int vae_channels_last,
                              float vae_inv_scaling, int B, int C, int H, int W, int init, void* stream) {
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || (G != 1 && G != 2) || table_rows < 2) return LB_ERR_SHAPE;
  if (unet_channels < C) return LB_ERR_SHAPE;
  if (!float_dtype(unet_dtype) || !float_dtype(vae_dtype) || (!init && !float_dtype(model_dtype)))
    return LB_ERR_DTYPE;
  if (x == nullptr || (MS ? x0_hist == nullptr : noise == nullptr) || table == nullptr || step_index == nullptr ||
      counter == nullptr || unet_in == nullptr || timestep == nullptr)
    return LB_ERR_SHAPE;
  if (!init && (model_out == nullptr || guidance == nullptr || vae_in == nullptr || !(vae_inv_scaling > 0.f)))
    return LB_ERR_SHAPE;
  const long long n = static_cast<long long>(B) * H * W;
  sample_step_kernel<MS><<<static_cast<int>((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      model_out, model_dtype, stride_b, stride_c, stride_p, G, x, noise, x0_hist, table, table_rows, guidance,
      step_index, counter, unet_in, unet_dtype, unet_channels, timestep, vae_in, vae_dtype, vae_channels_last != 0,
      vae_inv_scaling, B, C, H * W, init != 0);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_sample_step(const void* model_out, int model_dtype, long long stride_b, long long stride_c,
                              long long stride_p, int G, float* x, const float* noise, const float* table,
                              int table_rows, const float* guidance, int* step_index, unsigned int* counter,
                              void* unet_in, int unet_dtype, float* timestep, void* vae_in, int vae_dtype,
                              int vae_channels_last, float vae_inv_scaling, int B, int C, int H, int W, int init,
                              void* stream) {
  return launch_sample_step<false>(model_out, model_dtype, stride_b, stride_c, stride_p, G, x, noise, nullptr,
                                   table, table_rows, guidance, step_index, counter, unet_in, unet_dtype, C,
                                   timestep, vae_in, vae_dtype, vae_channels_last, vae_inv_scaling, B, C, H, W, init,
                                   stream);
}

extern "C" int lb_sample_step_ch(const void* model_out, int model_dtype, long long stride_b, long long stride_c,
                                 long long stride_p, int G, float* x, const float* noise, const float* table,
                                 int table_rows, const float* guidance, int* step_index, unsigned int* counter,
                                 void* unet_in, int unet_dtype, int unet_channels, float* timestep, void* vae_in,
                                 int vae_dtype, int vae_channels_last, float vae_inv_scaling, int B, int C, int H,
                                 int W, int init, void* stream) {
  return launch_sample_step<false>(model_out, model_dtype, stride_b, stride_c, stride_p, G, x, noise, nullptr,
                                   table, table_rows, guidance, step_index, counter, unet_in, unet_dtype,
                                   unet_channels, timestep, vae_in, vae_dtype, vae_channels_last, vae_inv_scaling, B,
                                   C, H, W, init, stream);
}

extern "C" int lb_sample_step_ms(const void* model_out, int model_dtype, long long stride_b, long long stride_c,
                                 long long stride_p, int G, float* x, float* x0_hist, const float* table,
                                 int table_rows, const float* guidance, int* step_index, unsigned int* counter,
                                 void* unet_in, int unet_dtype, int unet_channels, float* timestep, void* vae_in,
                                 int vae_dtype, int vae_channels_last, float vae_inv_scaling, int B, int C, int H,
                                 int W, void* stream) {
  return launch_sample_step<true>(model_out, model_dtype, stride_b, stride_c, stride_p, G, x, nullptr, x0_hist,
                                  table, table_rows, guidance, step_index, counter, unet_in, unet_dtype,
                                  unet_channels, timestep, vae_in, vae_dtype, vae_channels_last, vae_inv_scaling, B,
                                  C, H, W, 0, stream);
}

extern "C" int lb_sample_step_rescale(const void* model_out, int model_dtype, long long stride_b,
                                      long long stride_c, long long stride_p, int G, float* x, const float* noise,
                                      float* x0_hist, const float* table, int table_rows, const float* guidance,
                                      const float* guidance_rescale, int* step_index, unsigned int* counter,
                                      void* unet_in, int unet_dtype, int unet_channels, float* timestep,
                                      void* vae_in, int vae_dtype, int vae_channels_last, float vae_inv_scaling,
                                      int B, int C, int H, int W, void* stream) {
  if (B <= 0 || B > 65535 || C <= 0 || H <= 0 || W <= 0 || G != 2 || table_rows < 2 || unet_channels < C)
    return LB_ERR_SHAPE;
  if (static_cast<long long>(H) * W > 0x7fffffffll - RS_CLUSTER * 256) return LB_ERR_SHAPE;
  if (!float_dtype(model_dtype) || !float_dtype(unet_dtype) || !float_dtype(vae_dtype)) return LB_ERR_DTYPE;
  if (model_out == nullptr || x == nullptr || (x0_hist == nullptr && noise == nullptr) || table == nullptr ||
      guidance == nullptr || guidance_rescale == nullptr || step_index == nullptr || counter == nullptr ||
      unet_in == nullptr || timestep == nullptr || vae_in == nullptr || !(vae_inv_scaling > 0.f))
    return LB_ERR_SHAPE;
  const dim3 grid(RS_CLUSTER, B);
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (x0_hist)
    sample_step_rescale_kernel<true><<<grid, 256, 0, s>>>(
        model_out, model_dtype, stride_b, stride_c, stride_p, x, nullptr, x0_hist, table, table_rows, guidance,
        guidance_rescale, step_index, counter, unet_in, unet_dtype, unet_channels, timestep, vae_in, vae_dtype,
        vae_channels_last != 0, vae_inv_scaling, B, C, H * W);
  else
    sample_step_rescale_kernel<false><<<grid, 256, 0, s>>>(
        model_out, model_dtype, stride_b, stride_c, stride_p, x, noise, nullptr, table, table_rows, guidance,
        guidance_rescale, step_index, counter, unet_in, unet_dtype, unet_channels, timestep, vae_in, vae_dtype,
        vae_channels_last != 0, vae_inv_scaling, B, C, H * W);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_sample_init(const void* moments, int moments_dtype, long long stride_b, long long stride_c,
                              long long stride_p, const void* posterior_noise, int posterior_noise_dtype,
                              float scaling, const unsigned char* mask, const float* noise, const float* table,
                              int table_rows, float* x, int* step_index, unsigned int* counter, void* unet_in,
                              int unet_dtype, int unet_channels, float* timestep, int G, int B, int C, int H, int W,
                              void* stream) {
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || (G != 1 && G != 2) || table_rows < 2) return LB_ERR_SHAPE;
  if (!float_dtype(unet_dtype)) return LB_ERR_DTYPE;
  if (x == nullptr || noise == nullptr || table == nullptr || step_index == nullptr || counter == nullptr ||
      unet_in == nullptr || timestep == nullptr)
    return LB_ERR_SHAPE;
  if (unet_channels != (mask ? 2 * C + 1 : C)) return LB_ERR_SHAPE;
  if (mask && moments == nullptr) return LB_ERR_SHAPE;
  if (moments) {
    if (!float_dtype(moments_dtype)) return LB_ERR_DTYPE;
    if (posterior_noise_dtype != moments_dtype && posterior_noise_dtype != LB_F32) return LB_ERR_DTYPE;
    if (posterior_noise == nullptr) return LB_ERR_SHAPE;
  }
  const long long n = static_cast<long long>(B) * H * W;
  sample_init_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      moments, moments_dtype, stride_b, stride_c, stride_p, posterior_noise, posterior_noise_dtype, scaling, mask,
      noise, table, x, step_index, counter, unet_in, unet_dtype, unet_channels, timestep, G, B, C, H, W);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_pixels_emit(const void* image, int image_dtype, int channels_last, unsigned char* out, int B,
                              int H, int W, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0 || image == nullptr || out == nullptr) return LB_ERR_SHAPE;
  if (!float_dtype(image_dtype)) return LB_ERR_DTYPE;
  const long long P = static_cast<long long>(H) * W, n = B * P;
  pixels_emit_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      image, image_dtype, channels_last != 0, out, B, P);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}
