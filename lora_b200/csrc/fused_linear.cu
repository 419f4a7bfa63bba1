// C-ABI entry point for the fused LoRA linear (forward and, on transposed operands, dX).
// Replaces LoraInjectedLinear.forward (lora_diffusion/lora.py:53-58 of cloneofsimo/lora) and the dX
// part of its autograd backward. Kernel: fused_core.cuh.
#include "fused_core.cuh"
#include "lora_b200.h"
#include "tmap.h"

namespace lb {

// Tensor map of the frozen weight: row-major [N, K] (box BLOCK_N x 64) or, pre-tiled by lb_tile_weight,
// [n64 * num_kb * 64, 64] (box 64 x 64: one contiguous 8 KB block per box).
static bool tmap_weight(CUtensorMap* tm, const void* W, CUtensorMapDataType dt, int N, int K, int block_n, int tiled) {
  if (!tiled) return tmap_2d(tm, W, dt, 2, K, N, BLOCK_K, block_n, true);
  const unsigned long long n64 = (N + 63) / 64, nkb = (K + BLOCK_K - 1) / BLOCK_K;
  return tmap_2d(tm, W, dt, 2, 64, n64 * nkb * 64, 64, 64, true);
}

template <int BLOCK_N, int STAGES, typename OutT, int MIN_CTAS, bool DROP = false, bool SPLITK = false,
          int CL = 1, bool INLINE_TMA = false, int RP = R_PAD>
static int launch_linear(const void* X, const void* W, const void* Dn, void* Y, const FusedParams& p_in,
                         int out_dtype, cudaStream_t stream, int split = 1) {
  using S = Smem<BLOCK_N, STAGES, OutT, 1, DROP, CL, RP>;
  auto kern = fused_lora_kernel<BLOCK_N, STAGES, OutT, false, 1, MIN_CTAS, DROP, SPLITK, CL, INLINE_TMA, RP>;
  FusedParams p = p_in;
  p.split = 1;
  if constexpr (SPLITK) {
    const size_t tiles = static_cast<size_t>((p.N + BLOCK_N - 1) / BLOCK_N) * ((p.M + BLOCK_M - 1) / BLOCK_M);
    p.split = split;
    if (!split_ws_reserve(stream, tiles * BLOCK_M * (BLOCK_N + R_PAD) * sizeof(float),
                          static_cast<unsigned int>(tiles), &p.ws, &p.counters))
      return LB_ERR_CUDA;
  }
  static_assert(MIN_CTAS * (S::DYN_BYTES + 1024) <= 233472, "occupancy target does not fit");
  static unsigned long long attr_mask = 0;
  if (!ensure_dyn_smem(reinterpret_cast<const void*>(kern), S::DYN_BYTES, attr_mask)) return LB_ERR_CUDA;
  const CUtensorMapDataType in_dt = p.fmt ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const CUtensorMapDataType out_dt = out_dtype == LB_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : in_dt;
  CUtensorMap tmX, tmW, tmD, tmY;
  if (!tmap_2d(&tmX, X, in_dt, 2, p.K, p.M, BLOCK_K, BLOCK_M, true)) return LB_ERR_TMAP;
  if (!tmap_weight(&tmW, W, in_dt, p.N, p.K, BLOCK_N, p.w_tiled)) return LB_ERR_TMAP;
  if (!tmap_2d(&tmD, Dn, in_dt, 2, p.K, RP, BLOCK_K, RP, true)) return LB_ERR_TMAP;
  if (!tmap_2d(&tmY, Y, out_dt, sizeof(OutT), p.N, p.M, S::BOX_COLS, BLOCK_M, true)) return LB_ERR_TMAP;
  dim3 grid((p.N + BLOCK_N - 1) / BLOCK_N, (p.M + BLOCK_M - 1) / BLOCK_M, SPLITK ? split : CL);
  return launch_ex(kern, dim3(grid), dim3(kernel_threads<INLINE_TMA>()), S::DYN_BYTES, stream, CL, tmX, tmW, tmD, tmY,
                   p) == cudaSuccess
             ? LB_OK : LB_ERR_CUDA;
}

// Split-K plan for one linear problem (fused_core.cuh, SPLITK): a lone CTA streams its operands at a
// bounded per-SM rate, so sites with few tiles and long K leave most SMs idle while a handful stream.
// Cost model in microseconds (a planning heuristic, its parameters are not H100 measurements): fixed
// 2.0 (prologue + tail) + K blocks x per-SM ingest at 92 GB/s; a split adds 3.0 (L2 reductions of the
// partials, election, one burst read of the reduced row), independent of the split factor. Only
// single-wave plans (tiles x split <= SMs), and a split must win by > 25 %. Split plans use BLOCK_N 64:
// a 128-wide tile's reduced row and accumulator do not fit the registers together.
struct SplitPlan { int block_n, split; };
static SplitPlan plan_split(int M, int K, int N, int n_sms) {
  if (!splitk_enabled() || n_sms <= 0) return {0, 1};
  const int num_kb = (K + BLOCK_K - 1) / BLOCK_K;
  const int m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
  SplitPlan best = {0, 1};
  double best_t = 1e30, base_t = 1e30;
  {
    const int bn = 64;
    const long long tiles = static_cast<long long>(m_tiles) * ((N + bn - 1) / bn);
    const double per_kb = (128.0 + bn + 16.0) * 128.0 / 92e3;
    const double waves = static_cast<double>((tiles + n_sms - 1) / n_sms);
    const double t1 = waves * (2.0 + num_kb * per_kb);
    if (t1 < base_t) base_t = t1;
    for (int sp = 2; sp <= 8; ++sp) {
      if (tiles * sp > n_sms || num_kb / sp < 4) break;
      const double t = 2.0 + ((num_kb + sp - 1) / sp) * per_kb + 3.0;
      if (t < best_t) { best_t = t; best = {bn, sp}; }
    }
  }
  if (best.split > 1 && best_t < 0.75 * base_t) return best;
  return {0, 1};
}

template <int BLOCK_N, int STAGES, typename OutT, int MIN_CTAS, bool INLINE_TMA = false>
static int launch_grouped(GroupedArgs& a, const void* const* X, const void* const* W,
                          const void* const* Dn, void* const* Y, int out_dtype, cudaStream_t stream) {
  using S = Smem<BLOCK_N, STAGES, OutT, 1>;
  static_assert(MIN_CTAS * (S::DYN_BYTES + 1024) <= 233472, "occupancy target does not fit");
  auto kern = fused_lora_grouped_kernel<BLOCK_N, STAGES, OutT, MIN_CTAS, INLINE_TMA>;
  static unsigned long long attr_mask = 0;
  if (!ensure_dyn_smem(reinterpret_cast<const void*>(kern), S::DYN_BYTES, attr_mask)) return LB_ERR_CUDA;
  const int fmt = a.p[0].fmt;
  const CUtensorMapDataType in_dt = fmt ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const CUtensorMapDataType out_dt = out_dtype == LB_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : in_dt;
  int total = 0;
  for (int i = 0; i < a.n_problems; ++i) {
    const FusedParams& p = a.p[i];
    if (!tmap_2d(&a.tmX[i], X[i], in_dt, 2, p.K, p.M, BLOCK_K, BLOCK_M, true)) return LB_ERR_TMAP;
    if (!tmap_weight(&a.tmW[i], W[i], in_dt, p.N, p.K, BLOCK_N, p.w_tiled)) return LB_ERR_TMAP;
    if (!tmap_2d(&a.tmD[i], Dn[i], in_dt, 2, p.K, R_PAD, BLOCK_K, R_PAD, true)) return LB_ERR_TMAP;
    if (!tmap_2d(&a.tmY[i], Y[i], out_dt, sizeof(OutT), p.N, p.M, S::BOX_COLS, BLOCK_M, true)) return LB_ERR_TMAP;
    a.tile_start[i] = total;
    a.n_tiles_n[i] = (p.N + BLOCK_N - 1) / BLOCK_N;
    total += a.n_tiles_n[i] * ((p.M + BLOCK_M - 1) / BLOCK_M);
  }
  for (int i = a.n_problems; i <= MAX_GROUP; ++i) a.tile_start[i] = total;
  return launch_ex(kern, dim3(total), dim3(kernel_threads<INLINE_TMA>()), S::DYN_BYTES, stream, 1, a) == cudaSuccess
             ? LB_OK : LB_ERR_CUDA;
}


// Ranks 17..64 (RP = 32 or 64): one tile per CTA, 64 or 128 wide, one CTA per SM. 64-wide tiles while
// they fit one wave. Split-K, cluster split-K, inline-TMA and 192-wide plans are not built at these
// pads: a scope choice, not a measured one. A 128-wide fp32-output dropout tile at RP = 64 does not
// fit shared memory (accumulator + LoRA product + fp32 staging); it runs 64 wide.
template <int RP>
static int launch_linear_wide(const void* X, const void* W, const void* Dn, void* Y, const FusedParams& p,
                              int out_dtype, cudaStream_t st, bool drop, bool narrow) {
  if (out_dtype == LB_F32) {
    if (drop) {
      if (narrow || RP == 64) return launch_linear<64, 4, float, 1, true, false, 1, false, RP>(X, W, Dn, Y, p, out_dtype, st);
      if constexpr (RP != 64) return launch_linear<128, 4, float, 1, true, false, 1, false, RP>(X, W, Dn, Y, p, out_dtype, st);
    }
    return narrow ? launch_linear<64, 4, float, 1, false, false, 1, false, RP>(X, W, Dn, Y, p, out_dtype, st)
                  : launch_linear<128, 4, float, 1, false, false, 1, false, RP>(X, W, Dn, Y, p, out_dtype, st);
  }
  if (drop)
    return narrow ? launch_linear<64, 4, uint16_t, 1, true, false, 1, false, RP>(X, W, Dn, Y, p, out_dtype, st)
                  : launch_linear<128, 4, uint16_t, 1, true, false, 1, false, RP>(X, W, Dn, Y, p, out_dtype, st);
  return narrow ? launch_linear<64, 4, uint16_t, 1, false, false, 1, false, RP>(X, W, Dn, Y, p, out_dtype, st)
                : launch_linear<128, 4, uint16_t, 1, false, false, 1, false, RP>(X, W, Dn, Y, p, out_dtype, st);
}

static int g_linear_mode = 0;
static unsigned long long* g_dbg = nullptr;  // profiling: device buffer of 16 timestamps

}  // namespace lb

// Tuning knob (benchmarks / profiling only): force the tile schedule of lb_lora_linear_fwd.
extern "C" int lb_debug_set_linear_mode(int mode) {
  // schedule (0 auto, 1 one tile per CTA, 2 one tile per CTA and one CTA per SM, 3 cluster split-K
  // over 2..4 CTAs per tile)
  // + 4 * block_n choice (0 auto, 1: 64, 2: 128) + 16 * split-K factor choice (0: auto, 1..3: 2..4 CTAs)
  if (mode < 0 || mode > 63) return LB_ERR_SHAPE;          // block_n choice 3 = 192 (16-bit outputs, one tile per CTA)
  lb::g_linear_mode = mode;
  return LB_OK;
}

// Programmatic dependent launch for the fused kernels (0 off, 1 on; default from env LB_PDL).
extern "C" int lb_debug_set_pdl(int on) {
  lb::pdl_flag() = on ? 1 : 0;
  return LB_OK;
}

// Profiling knob: CTA (0,0) of the next lb_lora_linear_fwd launches writes %globaltimer stamps
// (entry, first TMA, first stage landed, MMAs issued, accumulator ready, T' ready, LoRA MMA done,
// stores issued, staging released, exit) into this device buffer of 16 uint64 (NULL: off).
extern "C" int lb_debug_set_stamp_buffer(void* dev_buf) {
  lb::g_dbg = reinterpret_cast<unsigned long long*>(dev_buf);
  return LB_OK;
}

static int linear_fwd_impl(const void* X, const void* W, const float* bias,
                                  const void* down16, const float* up, long long up_rs,
                                  long long up_cs, const float* diag, float scale, void* Y,
                                  float* T_out, const float* T_in, int M, int K, int N, int r, int r_pad,
                                  int in_dtype, int out_dtype, float drop_p, const void* seed_dev,
                                  void* stream) {
  using namespace lb;
  const int w_tiled = (in_dtype & LB_W_TILED) ? 1 : 0;
  in_dtype &= ~LB_W_TILED;
  if (r_pad != 16 && r_pad != 32 && r_pad != 64) return LB_ERR_SHAPE;
  if (!(drop_p >= 0.f && drop_p < 1.f) || (drop_p > 0.f && (seed_dev == nullptr || T_in != nullptr)))
    return LB_ERR_SHAPE;
  if (M <= 0 || N <= 0 || K <= 0) return LB_ERR_SHAPE;
  if (r < 1 || r > r_pad) return LB_ERR_RANK;
  if (in_dtype != LB_BF16 && in_dtype != LB_F16) return LB_ERR_DTYPE;
  if (out_dtype != in_dtype && out_dtype != LB_F32) return LB_ERR_DTYPE;
  // TMA: 16-byte aligned base pointers and row pitches
  if ((K % 8) != 0) return LB_ERR_SHAPE;
  if (out_dtype == LB_F32 ? (N % 4) != 0 : (N % 8) != 0) return LB_ERR_SHAPE;
  if ((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(W) |
       reinterpret_cast<uintptr_t>(down16) | reinterpret_cast<uintptr_t>(Y) |
       reinterpret_cast<uintptr_t>(T_out) | reinterpret_cast<uintptr_t>(T_in)) & 15)
    return LB_ERR_ALIGN;

  FusedParams p = {};
  p.bias = bias; p.up = up; p.up_rs = up_rs; p.up_cs = up_cs; p.up_gs = 0; p.diag = diag;
  p.t_out = T_out; p.t_in = T_in; p.scale = scale; p.M = M; p.N = N; p.K = K; p.r = r;
  p.fmt = (in_dtype == LB_BF16) ? 1 : 0; p.t_group = 0; p.dbg = g_dbg; p.w_tiled = w_tiled;
  p.drop_p = drop_p; p.drop_inv = 1.f / (1.f - drop_p);
  p.seed = reinterpret_cast<const unsigned long long*>(seed_dev);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (r_pad > R_PAD) {
    const int bn_choice = (g_linear_mode >> 2) & 3;
    const long long tiles64 = static_cast<long long>((M + 127) / 128) * ((N + 63) / 64);
    const bool narrow = bn_choice == 1 || (bn_choice != 2 && tiles64 <= sm_count());
    return r_pad == 32 ? launch_linear_wide<32>(X, W, down16, Y, p, out_dtype, st, drop_p > 0.f, narrow)
                       : launch_linear_wide<64>(X, W, down16, Y, p, out_dtype, st, drop_p > 0.f, narrow);
  }
  if (drop_p > 0.f) {
    // Dropout on the branch: the LoRA product keeps its own accumulator and is masked in the
    // drain (fused_core.cuh, DROP). One tile per CTA; BLOCK_N 64 (2 CTAs/SM) unless the site has
    // plenty of 128-wide tiles.
    const SplitPlan spd = plan_split(M, K, N, sm_count());
    if (spd.split > 1) {
      if (out_dtype == LB_F32)
        return launch_linear<64, 4, float, 1, true, true>(X, W, down16, Y, p, out_dtype, st, spd.split);
      return launch_linear<64, 5, uint16_t, 1, true, true>(X, W, down16, Y, p, out_dtype, st, spd.split);
    }
    const long long t128 = static_cast<long long>((M + 127) / 128) * ((N + 127) / 128);
    const bool nar = t128 < 120 && !(K >= 2048 && t128 >= 64);
    if (out_dtype == LB_F32)
      return nar ? launch_linear<64, 3, float, 2, true>(X, W, down16, Y, p, out_dtype, st)
                 : launch_linear<128, 4, float, 1, true>(X, W, down16, Y, p, out_dtype, st);
    return nar ? launch_linear<64, 3, uint16_t, 2, true>(X, W, down16, Y, p, out_dtype, st)
               : launch_linear<128, 4, uint16_t, 1, true>(X, W, down16, Y, p, out_dtype, st);
  }

  if ((g_linear_mode & 3) == 0) {
    const SplitPlan sp = plan_split(M, K, N, sm_count());
    if (sp.split > 1) {
      if (out_dtype == LB_F32)
        return launch_linear<64, 5, float, 1, false, true>(X, W, down16, Y, p, out_dtype, st, sp.split);
      return launch_linear<64, 6, uint16_t, 1, false, true>(X, W, down16, Y, p, out_dtype, st, sp.split);
    }
  }
  const int sched = g_linear_mode & 3, bn_choice = (g_linear_mode >> 2) & 3, split_choice = g_linear_mode >> 4;
  const long long m_tiles = (M + 127) / 128;
  const long long tiles128 = m_tiles * ((N + 127) / 128);
  const long long tiles64 = m_tiles * ((N + 63) / 64);
  const int n_sms = sm_count();
  if (g_linear_mode == 0 && T_in == nullptr && splitk_enabled() && n_sms > 0) {
    // Cluster split-K: few tiles and a K loop of >= 10 blocks -- the attention projections of the
    // 16x16 / 8x8 levels, the 77-token k/v sites, CLIP. Two CTAs of a cluster halve the K loop and
    // merge through distributed shared memory (one bulk copy, no global round trip).
    if (K >= 640 && tiles64 * 2 <= n_sms) {
      if (out_dtype == LB_F32) return launch_linear<64, 4, float, 1, false, false, 2>(X, W, down16, Y, p, out_dtype, st);
      return launch_linear<64, 6, uint16_t, 1, false, false, 2>(X, W, down16, Y, p, out_dtype, st);
    }
    // One balanced wave of 192-wide tiles instead of 1.1 waves of 128-wide ones (256x1280->10240:
    // 160 tiles of 128, 80 of 192)
    if (out_dtype != LB_F32 && tiles128 > n_sms && m_tiles * ((N + 191) / 192) <= n_sms && K >= 640)
      return launch_linear<192, 4, uint16_t, 1>(X, W, down16, Y, p, out_dtype, st);
  }
  // not enough tiles to fill the SMs with 128-wide ones: halve BLOCK_N -- as long as the 64-wide tiles
  // still fit ONE wave (at 2 CTAs per SM for short K and many row tiles: 4096x320->320 on an H100,
  // 96 tiles of 128 at one CTA per SM ~37-40 us, 160 tiles of 64 at two per SM ~21 us)
  bool narrow = tiles64 <= n_sms || (tiles64 <= 2LL * n_sms && K < 2048 && m_tiles >= 8);
  if (K >= 2048 && tiles128 >= 64) narrow = false;  // long K: per-tile work is large, keep W reuse
  if (bn_choice == 1) narrow = true;
  if (bn_choice == 2) narrow = false;
  const long long tiles_n = narrow ? tiles64 : tiles128;
  if (sched == 3 && T_in == nullptr) {
    // opt-in: split the K loop of every tile across a cluster of 2..4 CTAs (as the auto rule above)
    const int num_kb = (K + BLOCK_K - 1) / BLOCK_K;
    int split = split_choice ? split_choice + 1 : 4;
    if (split > num_kb) split = num_kb;
    if (bn_choice == 2 && split > 2) split = 2;        // 128-wide partials: one peer slot fits
    if (split >= 2) {
      if (out_dtype == LB_F32) {
        if (split == 2) return launch_linear<64, 4, float, 1, false, false, 2>(X, W, down16, Y, p, out_dtype, st);
        if (split == 3) return launch_linear<64, 3, float, 1, false, false, 3>(X, W, down16, Y, p, out_dtype, st);
        return launch_linear<64, 2, float, 1, false, false, 4>(X, W, down16, Y, p, out_dtype, st);
      }
      if (bn_choice == 2) return launch_linear<128, 3, uint16_t, 1, false, false, 2>(X, W, down16, Y, p, out_dtype, st);
      if (split == 2) return launch_linear<64, 6, uint16_t, 1, false, false, 2>(X, W, down16, Y, p, out_dtype, st);
      if (split == 3) return launch_linear<64, 4, uint16_t, 1, false, false, 3>(X, W, down16, Y, p, out_dtype, st);
      return launch_linear<64, 2, uint16_t, 1, false, false, 4>(X, W, down16, Y, p, out_dtype, st);
    }
  }
  if (bn_choice == 3 && out_dtype != LB_F32)
    return launch_linear<192, 4, uint16_t, 1>(X, W, down16, Y, p, out_dtype, st);
  // One tile per CTA. More tiles than SMs: 2 CTAs per SM with a short smem ring, so one CTA's
  // park / LoRA MMA / drain / store overlaps its neighbour's loads and MMAs (16-bit 128-wide tiles:
  // the 256-thread inline-TMA kernel, see fused_core.cuh). Fewer tiles than SMs (small-M / long-K
  // sites): one CTA per SM with a DEEP ring (7 x 26 KB or 4 x 34 KB in flight), because a lone CTA
  // streaming K = 768..10240 is bound by load latency, not bandwidth. Schedule 2 forces one CTA per
  // SM (deep ring) everywhere, to measure the overlap against.
  const bool crowded = tiles_n > n_sms && sched != 2;
  if (out_dtype == LB_F32) {
    return narrow ? launch_linear<64, 3, float, 2>(X, W, down16, Y, p, out_dtype, st)
                  : launch_linear<128, 4, float, 1>(X, W, down16, Y, p, out_dtype, st);
  }
  if (narrow)
    return crowded ? launch_linear<64, 2, uint16_t, 2>(X, W, down16, Y, p, out_dtype, st)
                   : launch_linear<64, 7, uint16_t, 1>(X, W, down16, Y, p, out_dtype, st);
  return crowded ? launch_linear<128, 2, uint16_t, 2, false, false, 1, true>(X, W, down16, Y, p, out_dtype, st)
                 : launch_linear<128, 4, uint16_t, 1>(X, W, down16, Y, p, out_dtype, st);
}


extern "C" int lb_lora_linear_fwd(const void* X, const void* W, const float* bias,
                                  const void* down, const float* up, long long up_rs,
                                  long long up_cs, const float* diag, float scale, void* Y,
                                  float* T_out, const float* T_in, int M, int K, int N, int r, int r_pad,
                                  int in_dtype, int out_dtype, void* stream) {
  return linear_fwd_impl(X, W, bias, down, up, up_rs, up_cs, diag, scale, Y, T_out, T_in, M, K, N, r, r_pad,
                         in_dtype, out_dtype, 0.f, nullptr, stream);
}

extern "C" int lb_lora_linear_fwd_dropout(const void* X, const void* W, const float* bias,
                                          const void* down, const float* up, long long up_rs,
                                          long long up_cs, const float* diag, float scale, void* Y,
                                          float* T_out, int M, int K, int N, int r, int r_pad, int in_dtype,
                                          int out_dtype, float drop_p, const void* seed_dev, void* stream) {
  return linear_fwd_impl(X, W, bias, down, up, up_rs, up_cs, diag, scale, Y, T_out, nullptr, M, K, N, r, r_pad,
                         in_dtype, out_dtype, drop_p, seed_dev, stream);
}

extern "C" int lb_lora_linear_fwd_grouped(int n, const void* const* X, const void* const* W,
                                          const float* const* bias, const void* const* down16,
                                          const float* const* up, const long long* up_rs,
                                          const long long* up_cs, const float* const* diag,
                                          const float* scale, void* const* Y, float* const* T_out,
                                          const int* M, const int* K, const int* N, const int* r,
                                          int in_dtype, int out_dtype, void* stream) {
  using namespace lb;
  const int w_tiled = (in_dtype & LB_W_TILED) ? 1 : 0;
  in_dtype &= ~LB_W_TILED;
  if (n < 1 || n > MAX_GROUP) return LB_ERR_SHAPE;
  if (in_dtype != LB_BF16 && in_dtype != LB_F16) return LB_ERR_DTYPE;
  if (out_dtype != in_dtype && out_dtype != LB_F32) return LB_ERR_DTYPE;
  GroupedArgs a = {};     // ~2.7 KB of kernel parameters (tensor maps + per-problem arguments)
  a.n_problems = n;
  long long tiles128 = 0, tiles64 = 0;
  for (int i = 0; i < n; ++i) {
    if (M[i] <= 0 || N[i] <= 0 || K[i] <= 0 || (K[i] % 8) != 0) return LB_ERR_SHAPE;
    if (out_dtype == LB_F32 ? (N[i] % 4) != 0 : (N[i] % 8) != 0) return LB_ERR_SHAPE;
    if (r[i] < 1 || r[i] > R_PAD) return LB_ERR_RANK;
    if ((reinterpret_cast<uintptr_t>(X[i]) | reinterpret_cast<uintptr_t>(W[i]) |
         reinterpret_cast<uintptr_t>(down16[i]) | reinterpret_cast<uintptr_t>(Y[i]) |
         reinterpret_cast<uintptr_t>(T_out ? T_out[i] : nullptr)) & 15)
      return LB_ERR_ALIGN;
    FusedParams p = {};
    p.bias = bias ? bias[i] : nullptr; p.up = up[i]; p.up_rs = up_rs[i]; p.up_cs = up_cs[i]; p.up_gs = 0;
    p.diag = diag ? diag[i] : nullptr; p.t_out = T_out ? T_out[i] : nullptr; p.t_in = nullptr;
    p.scale = scale[i]; p.M = M[i]; p.N = N[i]; p.K = K[i]; p.r = r[i];
    p.fmt = (in_dtype == LB_BF16) ? 1 : 0; p.t_group = 0; p.dbg = nullptr; p.w_tiled = w_tiled;
    a.p[i] = p;
    tiles128 += static_cast<long long>((M[i] + 127) / 128) * ((N[i] + 127) / 128);
    tiles64 += static_cast<long long>((M[i] + 127) / 128) * ((N[i] + 63) / 64);
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const bool narrow = tiles128 < 120;
  const bool crowded = (narrow ? tiles64 : tiles128) > sm_count();
  if (out_dtype == LB_F32)
    return narrow ? launch_grouped<64, 3, float, 2>(a, X, W, down16, Y, out_dtype, st)
                  : launch_grouped<128, 4, float, 1>(a, X, W, down16, Y, out_dtype, st);
  if (narrow)
    return crowded ? launch_grouped<64, 2, uint16_t, 2>(a, X, W, down16, Y, out_dtype, st)
                   : launch_grouped<64, 7, uint16_t, 1>(a, X, W, down16, Y, out_dtype, st);
  return crowded ? launch_grouped<128, 2, uint16_t, 2, true>(a, X, W, down16, Y, out_dtype, st)
                 : launch_grouped<128, 4, uint16_t, 1>(a, X, W, down16, Y, out_dtype, st);
}
