// C-ABI entry point for the fused LoRA Conv2d (NHWC implicit GEMM, stride 1, dilation 1,
// groups 1; 1x1 and 3x3 in the SD1.5 ResnetBlock2D sites). Forward and, on flipped/transposed
// frozen weights, the input gradient. Replaces LoraInjectedConv2d.forward
// (lora_diffusion/lora.py:130-135 of cloneofsimo/lora) and the dX part of its autograd backward.
// Kernel: fused_core.cuh.
#include "fused_core.cuh"
#include "lora_b200.h"
#include "tmap.h"

namespace lb {

int launch_t_from16(const void* gY, int fmt, const void* down, int C, int M, int r, int rp, float* T,
                    cudaStream_t st);   // lora_aux.cu

template <int BLOCK_N, int STAGES, typename OutT, int G, bool DROP = false, bool SPLITK = false, int RP = R_PAD>
static int launch_conv(const void* X, const void* W, const void* Dn, void* Y, const FusedParams& p_in,
                       int n_img, int down_cols, int out_dtype, cudaStream_t stream, int split = 1) {
  using S = Smem<BLOCK_N, STAGES, OutT, G, DROP, 1, RP>;
  auto kern = fused_lora_kernel<BLOCK_N, STAGES, OutT, true, G, 1, DROP, SPLITK, 1, false, RP>;
  FusedParams p = p_in;
  p.split = 1;
  if constexpr (SPLITK) {
    const size_t tiles = static_cast<size_t>((p.N + BLOCK_N - 1) / BLOCK_N) * n_img * p.tiles_h * p.tiles_w;
    p.split = split;
    if (!split_ws_reserve(stream, tiles * BLOCK_M * (BLOCK_N + R_PAD * G) * sizeof(float),
                          static_cast<unsigned int>(tiles), &p.ws, &p.counters))
      return LB_ERR_CUDA;
  }
  static unsigned long long attr_mask = 0;
  if (!ensure_dyn_smem(reinterpret_cast<const void*>(kern), S::DYN_BYTES, attr_mask)) return LB_ERR_CUDA;
  const CUtensorMapDataType in_dt = p.fmt ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const CUtensorMapDataType out_dt = out_dtype == LB_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : in_dt;
  CUtensorMap tmX, tmW, tmD, tmY;
  if (!tmap_nhwc(&tmX, X, in_dt, 2, p.C, p.W, p.H, n_img, BLOCK_K, p.TW, p.TH)) return LB_ERR_TMAP;
  if (!tmap_2d(&tmW, W, in_dt, 2, p.K, p.N, BLOCK_K, BLOCK_N, true)) return LB_ERR_TMAP;
  if (!tmap_2d(&tmD, Dn, in_dt, 2, down_cols, RP, BLOCK_K, RP, true)) return LB_ERR_TMAP;
  if (!tmap_nhwc(&tmY, Y, out_dt, sizeof(OutT), p.N, p.W, p.H, n_img, S::BOX_COLS, p.TW, p.TH)) return LB_ERR_TMAP;
  dim3 grid((p.N + BLOCK_N - 1) / BLOCK_N, n_img * p.tiles_h * p.tiles_w, SPLITK ? split : 1);
  return launch_ex(kern, grid, dim3(NUM_THREADS), S::DYN_BYTES, stream, 1, tmX, tmW, tmD, tmY, p) == cudaSuccess
             ? LB_OK : LB_ERR_CUDA;
}

// Split-K plan for one conv problem (same cost model as the linear planner, fused_linear.cu; K = taps x
// Cin runs to 23040 on the SD1.5 ResnetBlock2D sites while
// the 8x8 / 16x16 levels have only 10-40 output tiles). g = T groups (1 forward, taps for dX).
struct ConvPlan { int block_n, split; };
static ConvPlan plan_conv_split(long long m_tiles, int num_kb, int N, int g, int n_sms) {
  if (!splitk_enabled() || n_sms <= 0) return {0, 1};
  ConvPlan best = {0, 1};
  double best_t = 1e30, base_t = 1e30;
  {
    const int bn = 64;   // split plans use BLOCK_N 64 (see plan_split in fused_linear.cu)
    const long long tiles = m_tiles * ((N + bn - 1) / bn);
    const double per_kb = (128.0 + bn + 16.0) * 128.0 / 92e3;
    const double waves = static_cast<double>((tiles + n_sms - 1) / n_sms);
    const double t1 = waves * (2.0 + num_kb * per_kb);
    if (t1 < base_t) base_t = t1;
    for (int sp = 2; sp <= 8; ++sp) {
      if (tiles * sp > n_sms || num_kb / sp < 4) break;
      const double t = 2.0 + ((num_kb + sp - 1) / sp) * per_kb + 3.0 + (g > 1 ? 2.0 : 0.0);
      if (t < best_t) { best_t = t; best = {bn, sp}; }
    }
  }
  if (best.split > 1 && best_t < 0.75 * base_t) return best;
  return {0, 1};
}

// Ranks 17..64 (RP = 32 or 64): one tile per CTA, 64 wide while those tiles fit one wave, else 128;
// no split-K plans at these pads (a scope choice, not a measured one). The 3x3 input gradient runs the
// tap loop (T from t_in, fused_core.cuh TAPLOOP). A 128-wide fp32-output dropout tile at RP = 64 does not
// fit shared memory; it runs 64 wide.
template <int RP>
static int launch_conv_wide(const void* X, const void* W, const void* Dn, void* Y, const FusedParams& p,
                            int n_img, int down_cols, int out_dtype, cudaStream_t st, bool drop, bool groups,
                            bool narrow) {
#define LB_CONVW(BN, OT, GG, DR) launch_conv<BN, 4, OT, GG, DR, false, RP>(X, W, Dn, Y, p, n_img, down_cols, out_dtype, st)
  if (drop) {
    if (out_dtype == LB_F32) {
      if (narrow || RP == 64) return LB_CONVW(64, float, 1, true);
      if constexpr (RP != 64) return LB_CONVW(128, float, 1, true);
    }
    return narrow ? LB_CONVW(64, uint16_t, 1, true) : LB_CONVW(128, uint16_t, 1, true);
  }
  if (groups) {
    if (out_dtype == LB_F32) return narrow ? LB_CONVW(64, float, 9, false) : LB_CONVW(128, float, 9, false);
    return narrow ? LB_CONVW(64, uint16_t, 9, false) : LB_CONVW(128, uint16_t, 9, false);
  }
  if (out_dtype == LB_F32) return narrow ? LB_CONVW(64, float, 1, false) : LB_CONVW(128, float, 1, false);
  return narrow ? LB_CONVW(64, uint16_t, 1, false) : LB_CONVW(128, uint16_t, 1, false);
#undef LB_CONVW
}

}  // namespace lb

static int conv2d_fwd_impl(const void* X, const void* W, const float* bias,
                                  const void* down16, const float* up, long long up_rs,
                                  long long up_cs, long long up_gs, const float* diag, float scale,
                                  void* Y, float* T_out, const float* T_in, int n_img, int H, int Wd, int Cin,
                                  int Cout, int kh, int kw, int pad_h, int pad_w, int r, int r_pad,
                                  int per_tap_T, int in_dtype, int out_dtype, float drop_p,
                                  const void* seed_dev, void* stream) {
  using namespace lb;
  if (r_pad != 16 && r_pad != 32 && r_pad != 64) return LB_ERR_SHAPE;
  if (!(drop_p >= 0.f && drop_p < 1.f) || (drop_p > 0.f && (seed_dev == nullptr || T_in != nullptr || per_tap_T != 0)))
    return LB_ERR_SHAPE;
  if (n_img <= 0 || H <= 0 || Wd <= 0 || Cin <= 0 || Cout <= 0) return LB_ERR_SHAPE;
  if (!((kh == 1 && kw == 1) || (kh == 3 && kw == 3))) return LB_ERR_SHAPE;
  // "same" geometry only (output extent == input extent), which is what stride-1 SD convs use
  if (2 * pad_h != kh - 1 || 2 * pad_w != kw - 1) return LB_ERR_SHAPE;
  if (r < 1 || r > r_pad) return LB_ERR_RANK;
  // the wide-rank 3x3 input gradient reads its per-tap T from T_in; without T_in it first computes
  // T_out = X . down^T (one extra pass over X) and reads that
  const bool t_first = r_pad > R_PAD && per_tap_T != 0 && kh * kw > 1 && T_in == nullptr;
  if (t_first && T_out == nullptr) return LB_ERR_SHAPE;
  if (r_pad > R_PAD && per_tap_T != 0 && kh * kw > 1 && T_in != nullptr && T_out != nullptr) return LB_ERR_SHAPE;
  if (in_dtype != LB_BF16 && in_dtype != LB_F16) return LB_ERR_DTYPE;
  if (out_dtype != in_dtype && out_dtype != LB_F32) return LB_ERR_DTYPE;
  if ((Cin % 8) != 0 || (Cout % 8) != 0) return LB_ERR_SHAPE;
  if ((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(W) |
       reinterpret_cast<uintptr_t>(down16) | reinterpret_cast<uintptr_t>(Y) |
       reinterpret_cast<uintptr_t>(T_out) | reinterpret_cast<uintptr_t>(T_in)) & 15)
    return LB_ERR_ALIGN;

  const int taps = kh * kw;
  FusedParams p = {};
  p.bias = bias; p.up = up; p.up_rs = up_rs; p.up_cs = up_cs; p.up_gs = up_gs; p.diag = diag;
  p.t_out = T_out; p.t_in = T_in; p.scale = scale;
  p.M = n_img * H * Wd; p.N = Cout; p.K = taps * Cin; p.r = r;
  p.fmt = (in_dtype == LB_BF16) ? 1 : 0;
  p.H = H; p.W = Wd; p.C = Cin; p.kh = kh; p.kw = kw; p.pad_h = pad_h; p.pad_w = pad_w;
  p.TW = Wd >= 16 ? 16 : 8; p.TH = BLOCK_M / p.TW;
  p.tiles_h = (H + p.TH - 1) / p.TH; p.tiles_w = (Wd + p.TW - 1) / p.TW;
  const bool groups = per_tap_T != 0 && taps > 1;
  p.down_per_tap = groups ? 0 : 1;
  p.drop_p = drop_p; p.drop_inv = 1.f / (1.f - drop_p);
  p.seed = reinterpret_cast<const unsigned long long*>(seed_dev);
  p.t_group = groups ? pad_h * kw + pad_w : 0;   // the tap with zero shift
  const int down_cols = groups ? Cin : taps * Cin;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);

  // 64-wide tiles only while they still fit ONE wave (one CTA per SM: two of these rings do not fit an SM):
  // the 64x64-pixel, Cout = 320 sites are 96 tiles of 128 but 160 of 64 -- a second wave over 45-135 K blocks
  const long long tiles64c = static_cast<long long>(n_img) * p.tiles_h * p.tiles_w * ((Cout + 63) / 64);
  const bool narrow = tiles64c <= sm_count();
  if (t_first) {
    const int rc = launch_t_from16(X, p.fmt, down16, Cin, p.M, r, r_pad, T_out, st);
    if (rc != LB_OK) return rc;
    p.t_in = T_out;
    p.t_out = nullptr;
  }
  if (r_pad > R_PAD)
    return r_pad == 32 ? launch_conv_wide<32>(X, W, down16, Y, p, n_img, down_cols, out_dtype, st, drop_p > 0.f, groups, narrow)
                       : launch_conv_wide<64>(X, W, down16, Y, p, n_img, down_cols, out_dtype, st, drop_p > 0.f, groups, narrow);
#define LB_CONV(BN, OT, GG) launch_conv<BN, 4, OT, GG>(X, W, down16, Y, p, n_img, down_cols, out_dtype, st)
  const int cblocks = (Cin + BLOCK_K - 1) / BLOCK_K;
  const ConvPlan sp = plan_conv_split(static_cast<long long>(n_img) * p.tiles_h * p.tiles_w, taps * cblocks, Cout,
                                      groups ? taps : 1, sm_count());
  if (drop_p > 0.f) {   // forward with dropout on the branch: masked in the drain (DROP kernels)
#define LB_CONVD(BN, OT) launch_conv<BN, 4, OT, 1, true>(X, W, down16, Y, p, n_img, down_cols, out_dtype, st)
#define LB_CONVDS(BN, OT) launch_conv<BN, 4, OT, 1, true, true>(X, W, down16, Y, p, n_img, down_cols, out_dtype, st, sp.split)
    if (sp.split > 1) {
      if (out_dtype == LB_F32) return LB_CONVDS(64, float);
      return LB_CONVDS(64, uint16_t);
    }
    if (out_dtype == LB_F32) return narrow ? LB_CONVD(64, float) : LB_CONVD(128, float);
    return narrow ? LB_CONVD(64, uint16_t) : LB_CONVD(128, uint16_t);
#undef LB_CONVD
#undef LB_CONVDS
  }
  {
    if (sp.split > 1) {
#define LB_CONVS(BN, ST, OT, GG) launch_conv<BN, ST, OT, GG, false, true>(X, W, down16, Y, p, n_img, down_cols, out_dtype, st, sp.split)
      if (groups) {
        if (out_dtype == LB_F32) return LB_CONVS(64, 4, float, 9);
        return LB_CONVS(64, 4, uint16_t, 9);
      }
      if (out_dtype == LB_F32) return LB_CONVS(64, 4, float, 1);
      return LB_CONVS(64, 4, uint16_t, 1);
#undef LB_CONVS
    }
  }
  if (groups) {
    if (out_dtype == LB_F32) return narrow ? LB_CONV(64, float, 9) : LB_CONV(128, float, 9);
    return narrow ? LB_CONV(64, uint16_t, 9) : LB_CONV(128, uint16_t, 9);
  }
  if (out_dtype == LB_F32) return narrow ? LB_CONV(64, float, 1) : LB_CONV(128, float, 1);
  return narrow ? LB_CONV(64, uint16_t, 1) : LB_CONV(128, uint16_t, 1);
#undef LB_CONV
}

extern "C" int lb_lora_conv2d_fwd(const void* X, const void* W, const float* bias,
                                  const void* down, const float* up, long long up_rs,
                                  long long up_cs, long long up_gs, const float* diag, float scale,
                                  void* Y, float* T_out, const float* T_in, int n_img, int H, int Wd, int Cin,
                                  int Cout, int kh, int kw, int pad_h, int pad_w, int r, int r_pad,
                                  int per_tap_T, int in_dtype, int out_dtype, void* stream) {
  return conv2d_fwd_impl(X, W, bias, down, up, up_rs, up_cs, up_gs, diag, scale, Y, T_out, T_in, n_img, H,
                         Wd, Cin, Cout, kh, kw, pad_h, pad_w, r, r_pad, per_tap_T, in_dtype, out_dtype, 0.f,
                         nullptr, stream);
}

extern "C" int lb_lora_conv2d_fwd_dropout(const void* X, const void* W, const float* bias,
                                          const void* down, const float* up, long long up_rs,
                                          long long up_cs, const float* diag, float scale, void* Y,
                                          float* T_out, int n_img, int H, int Wd, int Cin, int Cout, int kh,
                                          int kw, int pad_h, int pad_w, int r, int r_pad, int in_dtype,
                                          int out_dtype, float drop_p, const void* seed_dev, void* stream) {
  return conv2d_fwd_impl(X, W, bias, down, up, up_rs, up_cs, 0, diag, scale, Y, T_out, nullptr, n_img, H,
                         Wd, Cin, Cout, kh, kw, pad_h, pad_w, r, r_pad, 0, in_dtype, out_dtype, drop_p, seed_dev,
                         stream);
}
