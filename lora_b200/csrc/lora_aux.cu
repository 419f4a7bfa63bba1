// HBM-bound helper kernels around the fused wgmma path:
//   - skinny weight-gradient reduction (dA, dB)        lora.py:53-58 autograd backward
//   - 16-bit shadow / frozen-weight casts + transposes
//   - global-norm clip + AdamW over the flat LoRA arena  train_lora_dreambooth.py:878-888
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "dropmask.cuh"
#include "lora_b200.h"
#include "ptx.cuh"
#include "tmap.h"

namespace lb {

__device__ __forceinline__ float2 ld16x2(const uint32_t w, int fmt) {
  if (fmt) {
    __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&w);
    return __bfloat1622float2(v);
  }
  __half2 v = *reinterpret_cast<const __half2*>(&w);
  return __half22float2(v);
}
__device__ __forceinline__ uint16_t to16(float x, int fmt) {
  if (fmt) {
    __nv_bfloat16 v = __float2bfloat16_rn(x);
    return *reinterpret_cast<uint16_t*>(&v);
  }
  __half v = __float2half_rn(x);
  return *reinterpret_cast<uint16_t*>(&v);
}
__device__ __forceinline__ float from16(uint16_t x, int fmt) {
  if (fmt) return __bfloat162float(*reinterpret_cast<__nv_bfloat16*>(&x));
  return __half2float(*reinterpret_cast<__half*>(&x));
}

// ------------------------------------------------------------------------------- wgrad
// out[j, c] += coef_j * sum_m V[m, j] * S[m, c]   -- a [r x M] . [M x C] product with r <= 64:
// pure streaming over S (HBM/L2-bound), so the kernel is organised for memory-level parallelism:
// CTA = 8 warps over a [64-row x 128-column] slab; a lane owns 4 adjacent columns (one 8-byte
// load; a warp covers 256 B of a row), a warp owns 8 rows and issues all 8 row loads before the
// first FMA. Partials are combined with shared-memory atomics, then one global atomicAdd per
// output element per CTA. Ranks above 16 (RG kernels) split into 16-wide rank groups on grid z, each
// re-reading its S slab (through L2): 64 accumulators per lane instead of 256.
constexpr int WG_COLS = 128;
constexpr int WG_WARPS = 8;
constexpr int WG_RPW = 8;                    // rows per warp
constexpr int WG_ROWS = WG_WARPS * WG_RPW;   // 64 rows per CTA

struct WgProblem {
  const uint2* S;      // [M, C] 16-bit rows (8-byte words)
  const float* V;      // [M, vp] fp32
  float* out;          // out[j*js + c*cs]
  long long js, cs;
  int C;
  float drop_p;        // > 0: S is masked (dropout site), mask index m*C + c
  const float* diag;   // selector diagonal of this problem's site (or null)
  float scale;
  int r;
  int M;               // rows of this problem (0: the launch-wide WgArgs::M)
  const unsigned long long* seed;  // mask seed of this problem (null: the launch-wide seed_dev)
  // conv weight-gradient: rows of S are pixels of NHWC images [M/(cH*cW), cH, cW, C] read at the
  // pixel shifted by (dy, dx) (zero outside the image); taps > 1: blockIdx.z = filter tap t with
  // shift (dy + t/kw, dx + t%kw) and out += t. cH == 0: plain rows.
  int cH, cW, dy, dx, kw, taps;
  int vp;              // row pitch of V (the rank pad: 16, 32 or 64)
};
constexpr int WG_MAXP = 24;
struct WgArgs {
  WgProblem pr[WG_MAXP];  // dA / dB of several sites share a launch (lb_lora_wgrad_batch: up to 24)
  int nb_start[WG_MAXP + 1];  // prefix sum of 128-column blocks per problem
  int n_pr;
  const unsigned long long* seed_dev;
  int M, fmt;
  int slabs;           // 64-row slabs per CTA
  int rgroups;         // RG kernels: 16-wide rank groups per tap on grid z (grid.z = taps x rgroups)
};

template <int RQ, bool RG = false>  // RQ: float4 groups of V used: ceil(r/4); RG: r > 16, rank groups
__global__ void __launch_bounds__(WG_WARPS * 32)
wgrad_kernel(const WgArgs a) {
  __shared__ float red[RQ * 4][WG_COLS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int which = 0;
#pragma unroll
  for (int i = 1; i < WG_MAXP; ++i)
    if (i < a.n_pr && static_cast<int>(blockIdx.x) >= a.nb_start[i]) which = i;
  const WgProblem& P = a.pr[which];
  const int cblk = blockIdx.x - a.nb_start[which];
  const int C = P.C;
  const int c0 = cblk * WG_COLS + lane * 4;
  const bool col_ok = c0 < C;                          // C % 8 == 0 => whole 4-column group valid
  const bool f32in = a.fmt == 2;                       // fp32 rows: 16 bytes per lane
  const size_t pitch = static_cast<size_t>(C) >> 2;    // row pitch in 8-byte words (16-bit rows)
  const int cH = P.cH, cW = P.cW;
  const int ntaps = (cH > 0 && P.taps > 1) ? P.taps : 1;
  const int tap = RG ? static_cast<int>(blockIdx.z) / a.rgroups : static_cast<int>(blockIdx.z);
  const int j0 = RG ? (static_cast<int>(blockIdx.z) % a.rgroups) * 16 : 0;   // first rank of this group
  if (tap >= ntaps) return;     // grid.z = most taps of any problem in the launch (x rank groups)
  if (RG && j0 >= P.r) return;
  const int sdy = P.dy + (ntaps > 1 ? tap / P.kw : 0), sdx = P.dx + (ntaps > 1 ? tap % P.kw : 0);
  for (int i = threadIdx.x; i < RQ * 4 * WG_COLS; i += WG_WARPS * 32) (&red[0][0])[i] = 0.f;
  __syncthreads();

  float acc[RQ * 4][4];
#pragma unroll
  for (int j = 0; j < RQ * 4; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  const float drop_p = P.drop_p;
  const int PM = P.M > 0 ? P.M : a.M;                 // rows of THIS problem
  if (static_cast<long long>(blockIdx.y) * a.slabs * WG_ROWS >= PM) return;   // batch: shorter problem
  const unsigned long long sd = (drop_p > 0.f) ? (P.seed ? P.seed[0] : a.seed_dev[0]) : 0ull;
  const float inv = (drop_p > 0.f) ? 1.f / (1.f - drop_p) : 1.f;

  auto load_rows = [&](int m_base, uint4 (&raw)[WG_RPW]) {
#pragma unroll
    for (int i = 0; i < WG_RPW; ++i) {
      const int m = m_base + i;
      bool ok = col_ok && m < PM;
      long long src = m;
      if (cH > 0 && ok) {
        // conv weight-gradient tap: row m is pixel (h, w) of an NHWC image; S is read at the pixel
        // shifted by (dy, dx), zero outside the image (= the convolution's zero padding)
        const int ww = m % cW + sdx, hh = (m / cW) % cH + sdy;
        ok = hh >= 0 && hh < cH && ww >= 0 && ww < cW;
        src = static_cast<long long>(m) + sdy * cW + sdx;
      }
      if (!ok) {
        raw[i] = make_uint4(0u, 0u, 0u, 0u);
      } else if (f32in) {
        raw[i] = __ldg(reinterpret_cast<const uint4*>(P.S) + static_cast<size_t>(src) * pitch + (c0 >> 2));
      } else {
        const uint2 v = __ldg(P.S + static_cast<size_t>(src) * pitch + (c0 >> 2));
        raw[i] = make_uint4(v.x, v.y, 0u, 0u);
      }
    }
  };

  const int m_first = blockIdx.y * a.slabs * WG_ROWS + warp * WG_RPW;
  uint4 cur[WG_RPW], nxt[WG_RPW];
  load_rows(m_first, cur);
  for (int sl = 0; sl < a.slabs; ++sl) {
    const int m_base = m_first + sl * WG_ROWS;
    if (m_base >= PM) break;
    if (sl + 1 < a.slabs) load_rows(m_base + WG_ROWS, nxt);   // next slab's rows in flight
#pragma unroll
    for (int i = 0; i < WG_RPW; ++i) {
      const int m = m_base + i;
      if (m < PM) {
        float x[4];
        if (f32in) {
          x[0] = __uint_as_float(cur[i].x); x[1] = __uint_as_float(cur[i].y);
          x[2] = __uint_as_float(cur[i].z); x[3] = __uint_as_float(cur[i].w);
        } else {
          const float2 lo = ld16x2(cur[i].x, a.fmt), hi = ld16x2(cur[i].y, a.fmt);
          x[0] = lo.x; x[1] = lo.y; x[2] = hi.x; x[3] = hi.y;
        }
        if (drop_p > 0.f) {  // S = gY of a dropout site: the branch saw mask/(1-p)
          const unsigned long long e = static_cast<unsigned long long>(m) * C + c0;
#pragma unroll
          for (int k = 0; k < 4; ++k) x[k] = drop_keep(sd, e + k, drop_p) ? x[k] * inv : 0.f;
        }
        const float4* vrow = reinterpret_cast<const float4*>(P.V + static_cast<size_t>(m) * (RG ? P.vp : 16) + j0);
#pragma unroll
        for (int qd = 0; qd < RQ; ++qd) {
          const float4 v = __ldg(vrow + qd);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            acc[qd * 4 + 0][k] += v.x * x[k];
            acc[qd * 4 + 1][k] += v.y * x[k];
            acc[qd * 4 + 2][k] += v.z * x[k];
            acc[qd * 4 + 3][k] += v.w * x[k];
          }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < WG_RPW; ++i) cur[i] = nxt[i];
  }
  if (col_ok) {
#pragma unroll
    for (int j = 0; j < RQ * 4; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k) atomicAdd(&red[j][lane * 4 + k], acc[j][k]);
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < RQ * 4 * WG_COLS; idx += WG_WARPS * 32) {
    const int j = idx / WG_COLS, c = idx % WG_COLS;
    const int cg = cblk * WG_COLS + c;
    if (j0 + j < P.r && cg < C) {
      const float coef = P.scale * (P.diag ? P.diag[j0 + j] : 1.f);
      atomicAdd(P.out + (j0 + j) * P.js + cg * P.cs + tap, coef * red[j][c]);
    }
  }
}

// ------------------------------------------------------------------------------- dropout branch
// Y[m, n] += scale/(1-p) * keep(m,n) * sum_j (T[m,j] * diag[j]) * up[n, j]     (in place)
// one thread = 8 consecutive columns of one row (16-byte access for 16-bit Y)
template <typename YT, int RP = 16>   // RP: row pitch of T (the rank pad)
__global__ void __launch_bounds__(256)
up_dropout_kernel(YT* __restrict__ Y, int y_fmt, const float* __restrict__ T,
                  const float* __restrict__ up, long long up_rs, long long up_cs,
                  const float* __restrict__ diag, float scale, float drop_p,
                  const unsigned long long* __restrict__ seed_dev, int M, int N, int r) {
  const int groups = N >> 3;  // N % 8 == 0
  const long long gid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (gid >= static_cast<long long>(M) * groups) return;
  const int m = static_cast<int>(gid / groups);
  const int n0 = static_cast<int>(gid % groups) << 3;
  const unsigned long long sd = seed_dev[0];
  const float inv = scale / (1.f - drop_p);
  float t[RP];
#pragma unroll
  for (int j = 0; j < RP; ++j) t[j] = (j < r) ? T[static_cast<size_t>(m) * RP + j] * (diag ? diag[j] : 1.f) : 0.f;
  float add[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float u = 0.f;
    for (int j = 0; j < r; ++j) u += t[j] * __ldg(up + (n0 + i) * up_rs + j * up_cs);
    add[i] = drop_keep(sd, static_cast<unsigned long long>(m) * N + n0 + i, drop_p) ? u * inv : 0.f;
  }
  YT* yp = Y + static_cast<size_t>(m) * N + n0;
  if constexpr (sizeof(YT) == 2) {
    uint4 raw = *reinterpret_cast<uint4*>(yp);
    uint16_t* h = reinterpret_cast<uint16_t*>(&raw);
#pragma unroll
    for (int i = 0; i < 8; ++i) h[i] = to16(from16(h[i], y_fmt) + add[i], y_fmt);
    *reinterpret_cast<uint4*>(yp) = raw;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) yp[i] += add[i];
  }
}

// dTs[m, j] = sum_n keep(m,n)/(1-p) * gY[m,n] * up[n, j]
// CTA = 8 warps over a [32-row x 512-column] slab of gY; the slab's up rows are staged transposed
// in shared memory ([j][n]: lanes read consecutive n), a lane owns 16 consecutive columns (two
// 16-byte loads, 8 pair-hashes), a warp owns 4 rows and re-uses the staged factors across them.
// Column slabs are combined with fp32 atomics (dTs zeroed by the launcher when there are several),
// so small-M sites (the 8x8 convs, time_emb_proj with M = 1) still spread over the chip.
// RG kernels (r > 16): dTs has row pitch rp, grid z = 16-wide rank group (gY slab re-read through L2).
// UP16 (RG only, p = 0, no seed): `up` is a 16-bit operand in gY's format -- T = gY . B of the wide-rank
// 3x3 conv input gradient, from the same padded B^T [rp, N] rows the fused kernel reads.
constexpr int DT_ROWS = 32, DT_COLS = 512;
template <bool RG = false, bool UP16 = false>
__global__ void __launch_bounds__(256)
dropout_dt_kernel(const uint4* __restrict__ gY, int fmt, const float* __restrict__ up,
                  long long up_rs, long long up_cs, float drop_p,
                  const unsigned long long* __restrict__ seed_dev, float* __restrict__ dTs, int M,
                  int N, int r, int use_atomics, int rp = 16) {
  __shared__ float ups[16][DT_COLS + 4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pitch_t = RG ? rp : 16;
  if (RG) {   // this group's ranks [16 z, 16 z + 16): shift the factor and the output, r = ranks left
    const int j0 = static_cast<int>(blockIdx.z) * 16;
    up = UP16 ? reinterpret_cast<const float*>(reinterpret_cast<const uint16_t*>(up) + j0 * up_cs) : up + j0 * up_cs;
    dTs += j0; r = r - j0 < 16 ? r - j0 : 16;
  }
  const int n_base = blockIdx.x * DT_COLS;
  const int m_base = blockIdx.y * DT_ROWS + warp * 4;
  for (int i = threadIdx.x; i < 16 * DT_COLS; i += 256) {
    const int j = i / DT_COLS, c = i % DT_COLS;
    const int n = n_base + c;
    // column c = lane*16 + 4q + w is stored at (q*32 + lane)*4 + w: a warp's float4 reads are contiguous
    const int pos = ((((c >> 2) & 3) * 32 + (c >> 4)) << 2) + (c & 3);
    if constexpr (UP16)
      ups[j][pos] = (j < r && n < N) ? from16(reinterpret_cast<const uint16_t*>(up)[n * up_rs + j * up_cs], fmt) : 0.f;
    else
      ups[j][pos] = (j < r && n < N) ? __ldg(up + n * up_rs + j * up_cs) : 0.f;
  }
  __syncthreads();
  const unsigned long long sd = UP16 ? 0ull : seed_dev[0];
  const uint32_t s0 = static_cast<uint32_t>(sd), s1 = static_cast<uint32_t>(sd >> 32);
  const uint32_t thr = drop_threshold(drop_p);
  const float inv = 1.f / (1.f - drop_p);
  const int c0 = lane * 16, n0 = n_base + c0;
  const size_t pitch = static_cast<size_t>(N) >> 3;           // row pitch in 16-byte words
  float g[4][16];
#pragma unroll
  for (int rr = 0; rr < 4; ++rr) {
    const int m = m_base + rr;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = n0 + 8 * h;
      uint4 raw = make_uint4(0u, 0u, 0u, 0u);
      if (m < M && n < N) raw = __ldg(gY + static_cast<size_t>(m) * pitch + (n >> 3));
      const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
      const unsigned long long e = (static_cast<unsigned long long>(m) * N + n) >> 1;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 v = ld16x2(w[q], fmt);
        const uint32_t bits = drop_bits(s0, s1, e + q);
        g[rr][8 * h + 2 * q] = (bits & 0xffffu) >= thr ? v.x * inv : 0.f;
        g[rr][8 * h + 2 * q + 1] = (bits >> 16) >= thr ? v.y * inv : 0.f;
      }
    }
  }
  for (int j = 0; j < r; ++j) {
    float u[16];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 t = *reinterpret_cast<const float4*>(&ups[j][(q * 32 + lane) << 2]);
      u[4 * q] = t.x; u[4 * q + 1] = t.y; u[4 * q + 2] = t.z; u[4 * q + 3] = t.w;
    }
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
      float acc = 0.f;
#pragma unroll
      for (int c = 0; c < 16; ++c) acc += g[rr][c] * u[c];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      const int m = m_base + rr;
      if (lane == 0 && m < M) {
        if (use_atomics) atomicAdd(dTs + static_cast<size_t>(m) * pitch_t + j, acc);
        else dTs[static_cast<size_t>(m) * pitch_t + j] = acc;
      }
    }
  }
  if (!use_atomics && lane < 16 && lane >= r) {                 // padded ranks stay zero
#pragma unroll
    for (int rr = 0; rr < 4; ++rr)
      if (m_base + rr < M) dTs[static_cast<size_t>(m_base + rr) * pitch_t + lane] = 0.f;
  }
}

// ------------------------------------------------------------------------------- casts
__global__ void cast_rows_pad16_kernel(const float* __restrict__ src, long long rs, long long cs,
                                       uint16_t* __restrict__ dst, int r, int C, int fmt) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int j = blockIdx.y;
  if (c >= C) return;
  const float x = (j < r) ? src[j * rs + c * cs] : 0.f;
  dst[static_cast<size_t>(j) * C + c] = to16(x, fmt);
}

// One entry {src_off, src_rs, src_cs, r, C, dst_off, dst_rs, rows} of the shadow table (lb_refresh_shadows):
// columns c = c0, c0 + dc, ... < C of the `rows` zero-padded 16-bit rows of one LoRA factor. p is read
// through L2 because the optimizer kernels write it earlier in the same launch.
__device__ __forceinline__ void refresh_shadow_entry(const float* __restrict__ p, const long long* __restrict__ e,
                                                     uint16_t* __restrict__ dst, int fmt, int c0, int dc) {
  const long long src_off = __ldg(e), rs = __ldg(e + 1), cs = __ldg(e + 2);
  const int r = static_cast<int>(__ldg(e + 3)), C = static_cast<int>(__ldg(e + 4));
  const long long dst_off = __ldg(e + 5), dst_rs = __ldg(e + 6);
  const int rows = static_cast<int>(__ldg(e + 7));
  for (int c = c0; c < C; c += dc) {
#pragma unroll 2   // deeper unrolling hoists the row loads and raises the optimizer kernels' registers
    for (int j = 0; j < rows; ++j) {
      const float x = (j < r) ? __ldcg(p + src_off + j * rs + c * cs) : 0.f;
      dst[dst_off + j * dst_rs + c] = to16(x, fmt);
    }
  }
}

// grid (column blocks, table entries)
__global__ void refresh_shadows_kernel(const float* __restrict__ p,
                                       const long long* __restrict__ table,
                                       uint16_t* __restrict__ dst_base, int fmt) {
  refresh_shadow_entry(p, table + static_cast<size_t>(blockIdx.y) * 8, dst_base, fmt,
                       blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x);
}

// src [R,C] -> dst [R,C] (optional) and dstT [C,R] (optional), 32x32 tiles through smem
template <typename SrcT>
__global__ void cast_weight_kernel(const SrcT* __restrict__ src, int src_fmt,
                                   uint16_t* __restrict__ dst, uint16_t* __restrict__ dstT, int R,
                                   int C, int fmt) {
  __shared__ float tile[32][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int rr = blockIdx.y * 32 + i;
    float x = 0.f;
    if (rr < R && c < C) {
      if constexpr (sizeof(SrcT) == 4) x = src[static_cast<size_t>(rr) * C + c];
      else x = from16(src[static_cast<size_t>(rr) * C + c], src_fmt);
      if (dst) dst[static_cast<size_t>(rr) * C + c] = to16(x, fmt);
    }
    tile[i][threadIdx.x] = x;
  }
  __syncthreads();
  if (dstT) {
    const int rr = blockIdx.y * 32 + threadIdx.x;  // becomes the contiguous index of dstT
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
      const int cc = blockIdx.x * 32 + i;
      if (rr < R && cc < C) dstT[static_cast<size_t>(cc) * R + rr] = to16(tile[threadIdx.x][i], fmt);
    }
  }
}

// Frozen weight -> 16-bit, 64 x 64-block layout (LB_W_TILED): dst block (n64, kb) = rows
// [(n64 * nkb + kb) * 64, +64) x 64 columns; element (n, k) of the logical [N, K] operand is read from
// src[n * src_rs + k * src_cs] (src_rs = K, src_cs = 1: W itself; src_rs = 1, src_cs = N_out... the
// transpose for dX), zero padded to multiples of 64. One-time preparation: simplicity over speed.
template <typename SrcT>
__global__ void __launch_bounds__(256)
tile_weight_kernel(const SrcT* __restrict__ src, int src_fmt, long long src_rs, long long src_cs,
                   uint16_t* __restrict__ dst, int N, int K, int nkb, int fmt) {
  __shared__ float tile[64][65];
  const int kb = blockIdx.x, n64 = blockIdx.y;
  const bool k_fast = src_cs == 1;     // which index is contiguous in the source decides the read order
  for (int i = threadIdx.x; i < 64 * 64; i += 256) {
    const int a = i >> 6, b = i & 63;
    const int rr = k_fast ? a : b, cc = k_fast ? b : a;       // (row in block, column in block)
    const int n = n64 * 64 + rr, k = kb * 64 + cc;
    float x = 0.f;
    if (n < N && k < K) {
      const size_t off = static_cast<size_t>(n) * src_rs + static_cast<size_t>(k) * src_cs;
      if constexpr (sizeof(SrcT) == 4) x = src[off];
      else x = from16(src[off], src_fmt);
    }
    tile[rr][cc] = x;
  }
  __syncthreads();
  uint16_t* d = dst + (static_cast<size_t>(n64) * nkb + kb) * 64 * 64;
  for (int i = threadIdx.x; i < 64 * 64; i += 256) d[i] = to16(tile[i >> 6][i & 63], fmt);
}

// fp32 -> three bf16 terms laid side by side along K ("split-bf16" operands for the fp32-faithful
// mode): x = hi + lo + O(2^-16 |x|), hi = bf16(x), lo = bf16(x - hi).
//   pattern 0 (activation side): [hi | lo | hi]      pattern 1 (weight side): [hi | hi | lo]
// so that  sum_k a3[k] w3[k] = a_hi w_hi + a_lo w_hi + a_hi w_lo  (the dropped lo*lo term is 2^-16).
__global__ void split_bf16x3_kernel(const float* __restrict__ src, long long src_rs,
                                    uint16_t* __restrict__ dst, int R, int C, int pattern) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int r = blockIdx.y;
  if (c >= C) return;
  const float x = src[r * src_rs + c];
  const __nv_bfloat16 hi = __float2bfloat16_rn(x);
  const __nv_bfloat16 lo = __float2bfloat16_rn(x - __bfloat162float(hi));
  const uint16_t h = *reinterpret_cast<const uint16_t*>(&hi), l = *reinterpret_cast<const uint16_t*>(&lo);
  uint16_t* row = dst + static_cast<size_t>(r) * 3 * C;
  row[c] = h;
  row[C + c] = pattern == 0 ? l : h;
  row[2 * C + c] = pattern == 0 ? h : l;
}

// ------------------------------------------------------------------------------- merge / collapse
// out[n,k] = W[n,k] + alpha * sum_j up[n,j] * down[j,k]   (lora.py:646-669; conv: flattened [Cout, Cin*kh*kw])
// HBM-bound over W: one read + one write of the weight, the rank-r factors stay in L1/L2.
template <typename WT, int RMAX = 16>
__global__ void __launch_bounds__(256)
merge_kernel(const WT* __restrict__ W, int w_fmt, const float* __restrict__ up,
             const float* __restrict__ down, float alpha, WT* __restrict__ out, int N, int K, int r) {
  const int k = blockIdx.x * 256 + threadIdx.x;
  const int n0 = blockIdx.y * 8;
  if (k >= K) return;
  float d[RMAX];
#pragma unroll
  for (int j = 0; j < RMAX; ++j) d[j] = (j < r) ? __ldg(down + static_cast<size_t>(j) * K + k) : 0.f;
  for (int n = n0; n < min(N, n0 + 8); ++n) {
    float acc = 0.f;
    for (int j = 0; j < r; ++j) acc += __ldg(up + static_cast<size_t>(n) * r + j) * d[j];
    const size_t i = static_cast<size_t>(n) * K + k;
    if constexpr (sizeof(WT) == 4) out[i] = W[i] + alpha * acc;
    else out[i] = to16(from16(W[i], w_fmt) + alpha * acc, w_fmt);
  }
}

// frozen conv weight [Cout,Cin,T] -> forward operand [Cout, T*Cin] and flipped-transposed
// input-gradient operand [Cin, T*Cout]; one-time per frozen weight, one thread per element
template <typename SrcT>
__global__ void cast_conv_weight_kernel(const SrcT* __restrict__ src, int src_fmt,
                                        uint16_t* __restrict__ dst, uint16_t* __restrict__ dstT,
                                        int Cout, int Cin, int T, int fmt) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long total = static_cast<long long>(Cout) * Cin * T;
  if (i >= total) return;
  const int t = static_cast<int>(i % T);
  const int c = static_cast<int>((i / T) % Cin);
  const int o = static_cast<int>(i / (static_cast<long long>(T) * Cin));
  float x;
  if constexpr (sizeof(SrcT) == 4) x = src[i];
  else x = from16(src[i], src_fmt);
  const uint16_t v = to16(x, fmt);
  if (dst) dst[(static_cast<long long>(o) * T + t) * Cin + c] = v;
  if (dstT) dstT[(static_cast<long long>(c) * T + (T - 1 - t)) * Cout + o] = v;
}

// ------------------------------------------------------------------------------- clip + AdamW
constexpr int OPT_THREADS = 256;
constexpr int OPT_MAX_PARTIALS = 1024;
constexpr int OPT_MAX_GROUPS = 8;

struct OptGroups {
  long long off[OPT_MAX_GROUPS + 1];
  int n;
};

__device__ __forceinline__ float block_sum(float x, float* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) sh[warp] = x;
  __syncthreads();
  float t = (threadIdx.x < OPT_THREADS / 32) ? sh[threadIdx.x] : 0.f;
  if (warp == 0) {
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (lane == 0) sh[0] = t;
  }
  __syncthreads();
  const float rsum = sh[0];
  __syncthreads();
  return rsum;
}

// pass 1: per-block partial sums of g^2 (fixed summation order => run-to-run deterministic)
__global__ void __launch_bounds__(OPT_THREADS)
sqnorm_partial_kernel(const float* __restrict__ g, long long n, float* __restrict__ partials,
                      int* __restrict__ step_dev) {
  __shared__ float sh[OPT_THREADS / 32];
  float s = 0.f;
  const long long n4 = n >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (long long i = blockIdx.x * static_cast<long long>(OPT_THREADS) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * OPT_THREADS) {
    const float4 x = g4[i];
    s += x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const float x = g[(n4 << 2) + threadIdx.x];
    s += x * x;
  }
  const float tot = block_sum(s, sh);
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = tot;
    if (blockIdx.x == 0) step_dev[0] += 1;  // t for the update pass that follows on the stream
  }
}

// pass 2: every block re-reduces the partials (same order everywhere), then updates its slice
__global__ void __launch_bounds__(OPT_THREADS)
adamw_update_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
                    float* __restrict__ v, long long n, OptGroups groups,
                    const float* __restrict__ lr_dev, float beta1, float beta2, float eps,
                    float wd, float max_norm, float inv_world, const int* __restrict__ step_dev,
                    const float* __restrict__ partials, int n_partials,
                    float* __restrict__ gnorm_out) {
  __shared__ float sh[OPT_THREADS / 32];
  float s = 0.f;
  for (int i = threadIdx.x; i < n_partials; i += OPT_THREADS) s += partials[i];
  const float sq = block_sum(s, sh);
  const float total = sqrtf(sq) * inv_world;
  float coef = inv_world;
  if (max_norm > 0.f) coef *= fminf(1.f, max_norm / (total + 1e-6f));
  if (blockIdx.x == 0 && threadIdx.x == 0 && gnorm_out) gnorm_out[0] = total;

  const int t = step_dev[0];
  const float bc1 = static_cast<float>(1.0 - pow(static_cast<double>(beta1), static_cast<double>(t)));
  const float bc2_sqrt = static_cast<float>(sqrt(1.0 - pow(static_cast<double>(beta2), static_cast<double>(t))));

  for (long long i = blockIdx.x * static_cast<long long>(OPT_THREADS) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * OPT_THREADS) {
    int gi = 0;
#pragma unroll
    for (int k = 1; k < OPT_MAX_GROUPS; ++k)
      if (k < groups.n && i >= groups.off[k]) gi = k;
    const float lr = lr_dev[gi];
    const float gg = g[i] * coef;
    float pp = p[i];
    pp *= (1.f - lr * wd);
    const float mm = beta1 * m[i] + (1.f - beta1) * gg;
    const float vv = beta2 * v[i] + (1.f - beta2) * gg * gg;
    const float denom = sqrtf(vv) / bc2_sqrt + eps;
    pp -= (lr / bc1) * (mm / denom);
    p[i] = pp;
    m[i] = mm;
    v[i] = vv;
    g[i] = 0.f;
  }
}

// ------------------------------------------------------------------------------- one-launch optimizer step
// clip_grad_norm_ + AdamW + zero_grad + refresh of the 16-bit operand shadows in ONE cooperative
// launch (train_lora_dreambooth.py:878-888 is ~10 foreach launches over hundreds of tiny tensors):
//   phase 1  per-block partial sum of g^2 (fixed order => deterministic)          -- grid barrier --
//   phase 2  every block re-reduces the partials, forms coef, updates its slice of p/m/v, zeroes g
//                                                                                  -- grid barrier --
//   phase 3  re-casts every LoRA factor into the zero-padded 16-bit [rows, C] operands the wgmma
//            kernels read (table walk, same rows as lb_refresh_shadows)
// The grid is launched with cudaLaunchAttributeCooperative (co-residency guaranteed) and at most
// one CTA per SM; the barrier is a generation counter in `bar` (2 x uint32, zero-initialised).
__device__ __forceinline__ void grid_barrier(unsigned int* bar, unsigned int nblocks) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned int gen = atomicAdd(&bar[1], 0u);
    if (atomicAdd(&bar[0], 1u) == nblocks - 1) {
      bar[0] = 0u;
      __threadfence();
      atomicAdd(&bar[1], 1u);
    } else {
      const long long t0 = clock64();
      while (atomicAdd(&bar[1], 0u) == gen) {
        if (clock64() - t0 > 4000000000ll) __trap();   // a protocol bug traps instead of hanging the box
      }
    }
    __threadfence();
  }
  __syncthreads();
}

__global__ void __launch_bounds__(OPT_THREADS)
optim_step_fused_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
                        float* __restrict__ v, long long n, OptGroups groups,
                        const float* __restrict__ lr_dev, float beta1, float beta2, float eps, float wd,
                        float max_norm, float inv_world, int* __restrict__ step_dev,
                        float* __restrict__ partials, float* __restrict__ gnorm_out,
                        const long long* __restrict__ table, int n_entries, int max_c,
                        uint16_t* __restrict__ shadow, int fmt, unsigned int* __restrict__ bar) {
  __shared__ float sh[OPT_THREADS / 32];
  const unsigned int nb = gridDim.x;
  // ---- phase 1
  {
    float s = 0.f;
    const long long n4 = n >> 2;
    const float4* g4 = reinterpret_cast<const float4*>(g);
    for (long long i = blockIdx.x * static_cast<long long>(OPT_THREADS) + threadIdx.x; i < n4;
         i += static_cast<long long>(nb) * OPT_THREADS) {
      const float4 x = g4[i];
      s += x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
      const float x = g[(n4 << 2) + threadIdx.x];
      s += x * x;
    }
    const float tot = block_sum(s, sh);
    if (threadIdx.x == 0) {
      partials[blockIdx.x] = tot;
      if (blockIdx.x == 0) step_dev[0] += 1;
    }
  }
  grid_barrier(bar, nb);
  // ---- phase 2
  {
    float s = 0.f;
    for (unsigned int i = threadIdx.x; i < nb; i += OPT_THREADS) s += __ldcg(partials + i);
    const float sq = block_sum(s, sh);
    const float total = sqrtf(sq) * inv_world;
    float coef = inv_world;
    if (max_norm > 0.f) coef *= fminf(1.f, max_norm / (total + 1e-6f));
    if (blockIdx.x == 0 && threadIdx.x == 0 && gnorm_out) gnorm_out[0] = total;
    const int t = __ldcg(step_dev);
    const float bc1 = static_cast<float>(1.0 - pow(static_cast<double>(beta1), static_cast<double>(t)));
    const float bc2_sqrt = static_cast<float>(sqrt(1.0 - pow(static_cast<double>(beta2), static_cast<double>(t))));
    for (long long i = blockIdx.x * static_cast<long long>(OPT_THREADS) + threadIdx.x; i < n;
         i += static_cast<long long>(nb) * OPT_THREADS) {
      int gi = 0;
#pragma unroll
      for (int k = 1; k < OPT_MAX_GROUPS; ++k)
        if (k < groups.n && i >= groups.off[k]) gi = k;
      const float lr = lr_dev[gi];
      const float gg = g[i] * coef;
      float pp = p[i];
      pp *= (1.f - lr * wd);
      const float mm = beta1 * m[i] + (1.f - beta1) * gg;
      const float vv = beta2 * v[i] + (1.f - beta2) * gg * gg;
      const float denom = sqrtf(vv) / bc2_sqrt + eps;
      pp -= (lr / bc1) * (mm / denom);
      p[i] = pp;
      m[i] = mm;
      v[i] = vv;
      g[i] = 0.f;
    }
  }
  if (n_entries <= 0) return;
  grid_barrier(bar, nb);
  // ---- phase 3: one table entry per block iteration (entries have 64 ... 10240 columns: no empty work items)
  for (int e_i = blockIdx.x; e_i < n_entries; e_i += nb)
    refresh_shadow_entry(p, table + static_cast<size_t>(e_i) * 8, shadow, fmt, threadIdx.x, OPT_THREADS);
}

// ------------------------------------------------------------------------------- data-parallel optimizer step
// The gradient all-reduce FUSED into the optimizer step (train_lora_dreambooth.py:744-757,877-888:
// DDP's bucketed all-reduce, then clip_grad_norm_ + AdamW + zero_grad): one cooperative launch per
// rank, no NCCL call, so the whole training step is ONE CUDA graph at any world size.
//   barrier 1 (NVLink flags)  every rank's backward has finished: its flat gradient buffer is final
//   phase 1   one-shot all-reduce by peer reads: gsum[i] = sum_r g_r[i], r = 0..world-1 in the SAME
//             order on every rank (bitwise identical sums => replicas stay identical), 16-byte loads
//             straight from the peers' HBM over NVLink/NVSwitch; per-block partial of gsum^2
//   grid barrier, then signal barrier 2 ("this rank has finished reading everybody's gradients")
//   phase 2   clip coefficient (1/world folded in) + AdamW on the local replica from gsum
//   wait barrier 2, zero the local gradient buffer (peers are done with it)
//   grid barrier, phase 3: refresh the 16-bit operand shadows
// Flags: flags[(b * world + r)] in each rank's own memory, b = barrier 0/1, written by rank r with
// the step's epoch (monotonic, so nothing is ever reset); peers' flag and gradient buffers are
// CUDA-IPC mappings. Every wait is bounded (~20 s) and traps instead of hanging the box.
constexpr int DP_MAX_WORLD = 16;
struct DpPeers {
  const float* g[DP_MAX_WORLD];       // gradient buffers in rank order (own one included)
  unsigned int* flags[DP_MAX_WORLD];  // flag arrays in rank order (own one included)
};

__device__ __forceinline__ float4 ld_peer16(const float* p) {
  float4 v;
  asm volatile("ld.volatile.global.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
// all ranks have written `epoch` into this rank's flags[b*world + r]
__device__ __forceinline__ void dp_wait_all(const unsigned int* flags, int b, int world, unsigned int epoch) {
  if (threadIdx.x < world) wait_flag_reached(flags + b * world + threadIdx.x, epoch);
  __syncthreads();
}

__global__ void __launch_bounds__(OPT_THREADS)
optim_step_dp_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ gsum,
                     float* __restrict__ m, float* __restrict__ v, long long n, OptGroups groups,
                     const float* __restrict__ lr_dev, float beta1, float beta2, float eps, float wd,
                     float max_norm, int* __restrict__ step_dev, float* __restrict__ partials,
                     float* __restrict__ gnorm_out, const long long* __restrict__ table, int n_entries,
                     int max_c, uint16_t* __restrict__ shadow, int fmt, unsigned int* __restrict__ bar,
                     DpPeers peers, int world, int rank, unsigned int* __restrict__ epoch_dev) {
  __shared__ float sh[OPT_THREADS / 32];
  const unsigned int nb = gridDim.x;
  const unsigned int epoch = epoch_dev[0] + 1u;          // bumped by block 0 at the very end
  unsigned int* my_flags = peers.flags[rank];
  const float inv_world = 1.f / static_cast<float>(world);
  // ---- barrier 1: announce "my gradients are final" to every rank, wait for everybody's
  if (blockIdx.x == 0 && threadIdx.x < world) {
    __threadfence_system();
    st_release_sys(peers.flags[threadIdx.x] + 0 * world + rank, epoch);
  }
  dp_wait_all(my_flags, 0, world, epoch);
  // ---- phase 1: gsum = sum over ranks (fixed order), partial sum of squares
  {
    float s = 0.f;
    const long long n4 = n >> 2;
    for (long long i = blockIdx.x * static_cast<long long>(OPT_THREADS) + threadIdx.x; i < n4;
         i += static_cast<long long>(nb) * OPT_THREADS) {
      float4 part[DP_MAX_WORLD];
#pragma unroll
      for (int r = 0; r < DP_MAX_WORLD; ++r)
        if (r < world) part[r] = ld_peer16(peers.g[r] + 4 * i);
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int r = 0; r < DP_MAX_WORLD; ++r)
        if (r < world) { a.x += part[r].x; a.y += part[r].y; a.z += part[r].z; a.w += part[r].w; }
      reinterpret_cast<float4*>(gsum)[i] = a;
      s += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
      const long long i = (n4 << 2) + threadIdx.x;
      float a = 0.f;
      for (int r = 0; r < world; ++r) a += *reinterpret_cast<const volatile float*>(peers.g[r] + i);
      gsum[i] = a;
      s += a * a;
    }
    const float tot = block_sum(s, sh);
    if (threadIdx.x == 0) {
      partials[blockIdx.x] = tot;
      if (blockIdx.x == 0) step_dev[0] += 1;
    }
  }
  grid_barrier(bar, nb);
  // ---- barrier 2 (signal only): every block of this rank has finished reading the peers
  if (blockIdx.x == 0 && threadIdx.x < world) {
    __threadfence_system();
    st_release_sys(peers.flags[threadIdx.x] + 1 * world + rank, epoch);
  }
  // ---- phase 2: clip + AdamW from gsum
  {
    float s = 0.f;
    for (unsigned int i = threadIdx.x; i < nb; i += OPT_THREADS) s += __ldcg(partials + i);
    const float sq = block_sum(s, sh);
    const float total = sqrtf(sq) * inv_world;
    float coef = inv_world;
    if (max_norm > 0.f) coef *= fminf(1.f, max_norm / (total + 1e-6f));
    if (blockIdx.x == 0 && threadIdx.x == 0 && gnorm_out) gnorm_out[0] = total;
    const int t = __ldcg(step_dev);
    const float bc1 = static_cast<float>(1.0 - pow(static_cast<double>(beta1), static_cast<double>(t)));
    const float bc2_sqrt = static_cast<float>(sqrt(1.0 - pow(static_cast<double>(beta2), static_cast<double>(t))));
    for (long long i = blockIdx.x * static_cast<long long>(OPT_THREADS) + threadIdx.x; i < n;
         i += static_cast<long long>(nb) * OPT_THREADS) {
      int gi = 0;
#pragma unroll
      for (int k = 1; k < OPT_MAX_GROUPS; ++k)
        if (k < groups.n && i >= groups.off[k]) gi = k;
      const float lr = lr_dev[gi];
      const float gg = __ldcg(gsum + i) * coef;
      float pp = p[i];
      pp *= (1.f - lr * wd);
      const float mm = beta1 * m[i] + (1.f - beta1) * gg;
      const float vv = beta2 * v[i] + (1.f - beta2) * gg * gg;
      const float denom = sqrtf(vv) / bc2_sqrt + eps;
      pp -= (lr / bc1) * (mm / denom);
      p[i] = pp;
      m[i] = mm;
      v[i] = vv;
    }
  }
  // ---- peers are done with this rank's gradients: zero them for the next backward pass
  dp_wait_all(my_flags, 1, world, epoch);
  for (long long i = blockIdx.x * static_cast<long long>(OPT_THREADS) + threadIdx.x; i < n;
       i += static_cast<long long>(nb) * OPT_THREADS)
    g[i] = 0.f;
  grid_barrier(bar, nb);
  if (blockIdx.x == 0 && threadIdx.x == 0) epoch_dev[0] = epoch;
  // ---- phase 3: operand shadows, one table entry per block iteration
  for (int e_i = blockIdx.x; e_i < n_entries; e_i += nb)
    refresh_shadow_entry(p, table + static_cast<size_t>(e_i) * 8, shadow, fmt, threadIdx.x, OPT_THREADS);
}

// ------------------------------------------------------------------------------- textual inversion step
__global__ void bump_step_kernel(int* step_dev) { step_dev[0] += 1; }

// One CTA per trained token row: AdamW on the row (the reference runs AdamW over the whole
// 49408 x 768 table and then copies every other row back: cli_lora_pti.py:448,477-479 -- the net
// effect is an update of the placeholder rows only), then the norm "decay" of
// cli_lora_pti.py:451-468:  w <- w/||w|| * (n + lambda (0.4 - n)),  n = ||w||, lambda = min(1, 100 lr),
// and the write-back of the row into the embedding table used by the text encoder.
__global__ void __launch_bounds__(256)
ti_step_kernel(float* __restrict__ rows, float* __restrict__ grad, float* __restrict__ m,
               float* __restrict__ v, const long long* __restrict__ token_ids, void* __restrict__ table,
               int table_dtype, int D, const float* __restrict__ lr_dev, float beta1, float beta2,
               float eps, float wd, const int* __restrict__ step_dev, int clip_decay, float target_norm) {
  __shared__ float sh[8];
  const int j = blockIdx.x;
  float* w = rows + static_cast<size_t>(j) * D;
  float* g = grad + static_cast<size_t>(j) * D;
  float* mm = m + static_cast<size_t>(j) * D;
  float* vv = v + static_cast<size_t>(j) * D;
  const float lr = lr_dev[0];
  const int t = step_dev[0];
  const float bc1 = static_cast<float>(1.0 - pow(static_cast<double>(beta1), static_cast<double>(t)));
  const float bc2_sqrt = static_cast<float>(sqrt(1.0 - pow(static_cast<double>(beta2), static_cast<double>(t))));
  float sq = 0.f;
  for (int i = threadIdx.x; i < D; i += 256) {
    const float gi = g[i];
    float p = w[i] * (1.f - lr * wd);
    const float m1 = beta1 * mm[i] + (1.f - beta1) * gi;
    const float v1 = beta2 * vv[i] + (1.f - beta2) * gi * gi;
    p -= (lr / bc1) * (m1 / (sqrtf(v1) / bc2_sqrt + eps));
    w[i] = p; mm[i] = m1; vv[i] = v1; g[i] = 0.f;
    sq += p * p;
  }
  const float norm = sqrtf(block_sum(sq, sh));
  float mult = 1.f;
  if (clip_decay) {
    const float lambda = fminf(1.f, 100.f * lr);
    mult = (norm + lambda * (target_norm - norm)) / fmaxf(norm, 1e-12f);
  }
  const long long tok = token_ids[j];
  for (int i = threadIdx.x; i < D; i += 256) {
    const float p = w[i] * mult;
    w[i] = p;
    const size_t o = static_cast<size_t>(tok) * D + i;
    if (table_dtype == LB_F32) reinterpret_cast<float*>(table)[o] = p;
    else reinterpret_cast<uint16_t*>(table)[o] = to16(p, table_dtype == LB_BF16);
  }
}


// T[m, j] = sum_c gY[m, c] * down[j, c] for j < r (16-bit gY [M, C] and down [rp, C], fp32 T [M, rp]):
// the per-pixel T of the wide-rank conv input gradient (fused_conv.cu)
int launch_t_from16(const void* gY, int fmt, const void* down, int C, int M, int r, int rp, float* T,
                    cudaStream_t st) {
  dim3 grid((C + DT_COLS - 1) / DT_COLS, (M + DT_ROWS - 1) / DT_ROWS, rp / 16);
  const int use_atomics = grid.x > 1;
  if (use_atomics && cudaMemsetAsync(T, 0, sizeof(float) * static_cast<size_t>(M) * rp, st) != cudaSuccess)
    return LB_ERR_CUDA;
  dropout_dt_kernel<true, true><<<grid, 256, 0, st>>>(reinterpret_cast<const uint4*>(gY), fmt,
                                                      reinterpret_cast<const float*>(down), 1, C, 0.f, nullptr, T,
                                                      M, C, r, use_atomics, rp);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

}  // namespace lb

// =============================================================================== C ABI
using namespace lb;

extern "C" int lb_abi_version(void) { return 6; }

static int wgrad_run(WgArgs& a, int in_dtype, void* stream) {
  if (a.M <= 0 || a.n_pr < 1 || a.n_pr > WG_MAXP) return LB_ERR_SHAPE;
  if (in_dtype != LB_BF16 && in_dtype != LB_F16 && in_dtype != LB_F32) return LB_ERR_DTYPE;
  int nblk = 0, rmax = 0;
  bool wide = false;   // any V pitch other than 16: the rank-group kernel (it reads the pitch)
  for (int i = 0; i < a.n_pr; ++i) {
    const WgProblem& P = a.pr[i];
    if (P.vp != 16 && P.vp != 32 && P.vp != 64) return LB_ERR_SHAPE;
    if (P.r < 1 || P.r > P.vp) return LB_ERR_RANK;
    if (P.C <= 0 || (P.C % 8) != 0) return LB_ERR_SHAPE;
    if ((reinterpret_cast<uintptr_t>(P.S) | reinterpret_cast<uintptr_t>(P.V)) & 15) return LB_ERR_ALIGN;
    a.nb_start[i] = nblk;
    nblk += (P.C + WG_COLS - 1) / WG_COLS;
    rmax = P.r > rmax ? P.r : rmax;
    wide = wide || P.vp != 16;
  }
  for (int i = a.n_pr; i <= WG_MAXP; ++i) a.nb_start[i] = nblk;
  a.fmt = in_dtype == LB_BF16 ? 1 : (in_dtype == LB_F32 ? 2 : 0);
  // rows per CTA: keep >= ~2 CTAs per SM, but fold slabs together when the grid would be far
  // larger (fewer global atomics per output element)
  const int slabs_total = (a.M + WG_ROWS - 1) / WG_ROWS;
  int slabs = 1;
  while (slabs < 8 && static_cast<long long>(nblk) * ((slabs_total + 2 * slabs - 1) / (2 * slabs)) >= 296) slabs *= 2;
  a.slabs = slabs;
  int max_taps = 1;
  for (int i = 0; i < a.n_pr; ++i)
    if (a.pr[i].cH > 0 && a.pr[i].taps > max_taps) max_taps = a.pr[i].taps;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (wide) {
    a.rgroups = (rmax + 15) / 16;
    dim3 grid(nblk, (slabs_total + slabs - 1) / slabs, max_taps * a.rgroups);
    wgrad_kernel<4, true><<<grid, WG_WARPS * 32, 0, st>>>(a);
    return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
  }
  dim3 grid(nblk, (slabs_total + slabs - 1) / slabs, max_taps);
  switch ((rmax + 3) / 4) {
    case 1: wgrad_kernel<1><<<grid, WG_WARPS * 32, 0, st>>>(a); break;
    case 2: wgrad_kernel<2><<<grid, WG_WARPS * 32, 0, st>>>(a); break;
    case 3: wgrad_kernel<3><<<grid, WG_WARPS * 32, 0, st>>>(a); break;
    default: wgrad_kernel<4><<<grid, WG_WARPS * 32, 0, st>>>(a); break;
  }
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

static int wgrad_launch(const void* S, const float* V, const float* diag, float scale, float* out,
                        long long out_js, long long out_cs, int M, int C, int r, int r_pad, float drop_p,
                        const void* seed_dev, int in_dtype, void* stream) {
  WgArgs a = {};
  a.pr[0].S = reinterpret_cast<const uint2*>(S); a.pr[0].V = V; a.pr[0].out = out;
  a.pr[0].js = out_js; a.pr[0].cs = out_cs; a.pr[0].C = C; a.pr[0].drop_p = drop_p;
  a.pr[0].diag = diag; a.pr[0].scale = scale; a.pr[0].r = r; a.pr[0].vp = r_pad;
  a.n_pr = 1;
  a.seed_dev = reinterpret_cast<const unsigned long long*>(seed_dev);
  a.M = M; a.pr[0].kw = 1; a.pr[0].taps = 1;
  return wgrad_run(a, in_dtype, stream);
}

extern "C" int lb_lora_wgrad(const void* S, const float* V, const float* diag, float scale,
                             float* out, long long out_js, long long out_cs, int M, int C, int r,
                             int r_pad, int in_dtype, void* stream) {
  return wgrad_launch(S, V, diag, scale, out, out_js, out_cs, M, C, r, r_pad, 0.f, nullptr, in_dtype, stream);
}

extern "C" int lb_lora_wgrad_masked(const void* S, const float* V, const float* diag, float scale,
                                    float* out, long long out_js, long long out_cs, int M, int C,
                                    int r, int r_pad, float drop_p, const void* seed_dev, int in_dtype,
                                    void* stream) {
  if (!(drop_p >= 0.f && drop_p < 1.f) || (drop_p > 0.f && seed_dev == nullptr)) return LB_ERR_SHAPE;
  return wgrad_launch(S, V, diag, scale, out, out_js, out_cs, M, C, r, r_pad, drop_p, seed_dev, in_dtype,
                      stream);
}

// All kh*kw taps of a conv down-factor gradient in one launch: tap t reads S shifted by
// (t/kw - pad_h, t%kw - pad_w) and accumulates into out[j*out_js + c*out_cs + t].
extern "C" int lb_lora_wgrad_conv(const void* S, const float* V, const float* diag, float scale,
                                  float* out, int M, int C, int r, int r_pad, int H, int W, int kh, int kw,
                                  int pad_h, int pad_w, int in_dtype, void* stream) {
  if (H <= 0 || W <= 0 || kh <= 0 || kw <= 0 || (M % (H * W)) != 0) return LB_ERR_SHAPE;
  WgArgs a = {};
  const int taps = kh * kw;
  a.pr[0].S = reinterpret_cast<const uint2*>(S); a.pr[0].V = V; a.pr[0].out = out;
  a.pr[0].js = static_cast<long long>(C) * taps; a.pr[0].cs = taps; a.pr[0].C = C; a.pr[0].drop_p = 0.f;
  a.pr[0].diag = diag; a.pr[0].scale = scale; a.pr[0].r = r; a.pr[0].vp = r_pad;
  a.n_pr = 1;
  a.M = M; a.pr[0].cH = H; a.pr[0].cW = W; a.pr[0].dy = -pad_h; a.pr[0].dx = -pad_w; a.pr[0].kw = kw; a.pr[0].taps = taps;
  return wgrad_run(a, in_dtype, stream);
}

extern "C" int lb_lora_wgrad_pair(const void* X, const float* dTs, float* dA, long long dA_js,
                                  long long dA_cs, int K, const void* gY, const float* T, float* dB,
                                  long long dB_js, long long dB_cs, int N, const float* diag,
                                  float scale, int M, int r, int r_pad, float drop_p, const void* seed_dev,
                                  int in_dtype, void* stream) {
  if (!(drop_p >= 0.f && drop_p < 1.f) || (drop_p > 0.f && seed_dev == nullptr)) return LB_ERR_SHAPE;
  WgArgs a = {};
  a.pr[0].S = reinterpret_cast<const uint2*>(X); a.pr[0].V = dTs; a.pr[0].out = dA;
  a.pr[0].js = dA_js; a.pr[0].cs = dA_cs; a.pr[0].C = K; a.pr[0].drop_p = 0.f;
  a.pr[1].S = reinterpret_cast<const uint2*>(gY); a.pr[1].V = T; a.pr[1].out = dB;
  a.pr[1].js = dB_js; a.pr[1].cs = dB_cs; a.pr[1].C = N; a.pr[1].drop_p = drop_p;
  for (int i = 0; i < 2; ++i) { a.pr[i].diag = diag; a.pr[i].scale = scale; a.pr[i].r = r; a.pr[i].vp = r_pad; }
  a.n_pr = 2;
  a.seed_dev = reinterpret_cast<const unsigned long long*>(seed_dev);
  a.M = M;
  return wgrad_run(a, in_dtype, stream);
}

// dA and dB of up to 4 sites that share X (a grouped family) in one launch. HOST arrays of length n.
extern "C" int lb_lora_wgrad_multi(int n, const void* X, const float* const* dTs, float* const* dA,
                                   const void* const* gY, const float* const* T, float* const* dB,
                                   const int* N, const float* const* diag, const float* scale,
                                   const int* r, int M, int K, int in_dtype, void* stream) {
  if (n < 1 || 2 * n > WG_MAXP) return LB_ERR_SHAPE;
  WgArgs a = {};
  for (int i = 0; i < n; ++i) {
    WgProblem& pa = a.pr[2 * i];
    WgProblem& pb = a.pr[2 * i + 1];
    pa.S = reinterpret_cast<const uint2*>(X); pa.V = dTs[i]; pa.out = dA[i]; pa.js = K; pa.cs = 1; pa.C = K;
    pb.S = reinterpret_cast<const uint2*>(gY[i]); pb.V = T[i]; pb.out = dB[i]; pb.js = 1; pb.cs = r[i]; pb.C = N[i];
    pa.drop_p = pb.drop_p = 0.f;
    pa.diag = pb.diag = diag ? diag[i] : nullptr;
    pa.scale = pb.scale = scale[i];
    pa.r = pb.r = r[i];
    pa.vp = pb.vp = 16;
  }
  a.n_pr = 2 * n;
  a.M = M;
  return wgrad_run(a, in_dtype, stream);
}

// Many independent reductions out[j,c] += scale*diag[j] * sum_m V[m,j] S[m,c] in as few launches as
// possible (24 problems per launch): the dA / dB of EVERY linear site of a step, queued during
// backward and flushed once at its end -- they feed only the optimizer, and one launch over
// hundreds of MB fills the chip where 120-270 launches over a few MB each were latency-bound.
extern "C" int lb_lora_wgrad_batch(const lb_wgrad_problem* probs, int n, int in_dtype, void* stream) {
  if (probs == nullptr || n < 1) return LB_ERR_SHAPE;
  for (int base = 0; base < n; base += WG_MAXP) {
    const int cnt = (n - base) < WG_MAXP ? (n - base) : WG_MAXP;
    WgArgs a = {};
    int max_m = 0;
    for (int i = 0; i < cnt; ++i) {
      const lb_wgrad_problem& q = probs[base + i];
      if (q.M <= 0 || !(q.drop_p >= 0.f && q.drop_p < 1.f) || (q.drop_p > 0.f && q.seed_dev == nullptr))
        return LB_ERR_SHAPE;
      WgProblem& w = a.pr[i];
      w.S = reinterpret_cast<const uint2*>(q.S); w.V = q.V; w.out = q.out; w.js = q.out_js; w.cs = q.out_cs;
      w.C = q.C; w.drop_p = q.drop_p; w.diag = q.diag; w.scale = q.scale; w.r = q.r; w.M = q.M;
      w.seed = reinterpret_cast<const unsigned long long*>(q.seed_dev);
      w.vp = q.r_pad;
      if (q.conv_H > 0) {       // conv lora_down weight-gradient: all taps of one site as one problem
        if (q.conv_W <= 0 || q.kh <= 0 || q.kw <= 0 || (q.M % (q.conv_H * q.conv_W)) != 0) return LB_ERR_SHAPE;
        w.cH = q.conv_H; w.cW = q.conv_W; w.dy = -q.pad_h; w.dx = -q.pad_w; w.kw = q.kw; w.taps = q.kh * q.kw;
      }
      max_m = q.M > max_m ? q.M : max_m;
    }
    a.n_pr = cnt;
    a.M = max_m;
    const int rc = wgrad_run(a, in_dtype, stream);
    if (rc != LB_OK) return rc;
  }
  return LB_OK;
}

template <int RP>
static void up_dropout_launch(void* Y, int y_dtype, const float* T, const float* up, long long up_rs,
                              long long up_cs, const float* diag, float scale, float drop_p,
                              const unsigned long long* sd, int M, int N, int r, int blocks, cudaStream_t st) {
  if (y_dtype == LB_F32)
    up_dropout_kernel<float, RP><<<blocks, 256, 0, st>>>(reinterpret_cast<float*>(Y), 0, T, up, up_rs, up_cs, diag, scale, drop_p, sd, M, N, r);
  else
    up_dropout_kernel<uint16_t, RP><<<blocks, 256, 0, st>>>(reinterpret_cast<uint16_t*>(Y), y_dtype == LB_BF16, T, up, up_rs, up_cs, diag, scale, drop_p, sd, M, N, r);
}

extern "C" int lb_lora_up_dropout(void* Y, int y_dtype, const float* T, const float* up,
                                  long long up_rs, long long up_cs, const float* diag, float scale,
                                  float drop_p, const void* seed_dev, int M, int N, int r, int r_pad,
                                  void* stream) {
  if (r_pad != 16 && r_pad != 32 && r_pad != 64) return LB_ERR_SHAPE;
  if (M <= 0 || N <= 0 || (N % 8) != 0) return LB_ERR_SHAPE;
  if (r < 1 || r > r_pad) return LB_ERR_RANK;
  if (!(drop_p >= 0.f && drop_p < 1.f) || seed_dev == nullptr) return LB_ERR_SHAPE;
  if (reinterpret_cast<uintptr_t>(Y) & 15) return LB_ERR_ALIGN;
  if (y_dtype != LB_F32 && y_dtype != LB_BF16 && y_dtype != LB_F16) return LB_ERR_DTYPE;
  const long long threads = static_cast<long long>(M) * (N / 8);
  const int blocks = static_cast<int>((threads + 255) / 256);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const unsigned long long* sd = reinterpret_cast<const unsigned long long*>(seed_dev);
  if (r_pad == 16) up_dropout_launch<16>(Y, y_dtype, T, up, up_rs, up_cs, diag, scale, drop_p, sd, M, N, r, blocks, st);
  else if (r_pad == 32) up_dropout_launch<32>(Y, y_dtype, T, up, up_rs, up_cs, diag, scale, drop_p, sd, M, N, r, blocks, st);
  else up_dropout_launch<64>(Y, y_dtype, T, up, up_rs, up_cs, diag, scale, drop_p, sd, M, N, r, blocks, st);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_lora_dropout_dt(const void* gY, int in_dtype, const float* up, long long up_rs,
                                  long long up_cs, float drop_p, const void* seed_dev, float* dTs,
                                  int M, int N, int r, int r_pad, void* stream) {
  if (r_pad != 16 && r_pad != 32 && r_pad != 64) return LB_ERR_SHAPE;
  if (M <= 0 || N <= 0 || (N % 8) != 0) return LB_ERR_SHAPE;
  if (r < 1 || r > r_pad) return LB_ERR_RANK;
  if (in_dtype != LB_BF16 && in_dtype != LB_F16) return LB_ERR_DTYPE;
  if (!(drop_p >= 0.f && drop_p < 1.f) || seed_dev == nullptr) return LB_ERR_SHAPE;
  if (reinterpret_cast<uintptr_t>(gY) & 15) return LB_ERR_ALIGN;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  dim3 grid((N + DT_COLS - 1) / DT_COLS, (M + DT_ROWS - 1) / DT_ROWS, r_pad / 16);
  const int use_atomics = grid.x > 1;
  if (use_atomics && cudaMemsetAsync(dTs, 0, sizeof(float) * static_cast<size_t>(M) * r_pad, st) != cudaSuccess)
    return LB_ERR_CUDA;
  const uint4* g4 = reinterpret_cast<const uint4*>(gY);
  const unsigned long long* sd = reinterpret_cast<const unsigned long long*>(seed_dev);
  if (r_pad == 16)
    dropout_dt_kernel<<<grid, 256, 0, st>>>(g4, in_dtype == LB_BF16, up, up_rs, up_cs, drop_p, sd, dTs, M, N, r,
                                            use_atomics);
  else
    dropout_dt_kernel<true><<<grid, 256, 0, st>>>(g4, in_dtype == LB_BF16, up, up_rs, up_cs, drop_p, sd, dTs, M,
                                                  N, r, use_atomics, r_pad);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_cast_rows_pad(const float* src, long long src_rs, long long src_cs,
                                void* dst16, int r, int r_pad, int C, int out_dtype, void* stream) {
  if (r_pad != 16 && r_pad != 32 && r_pad != 64) return LB_ERR_SHAPE;
  if (C <= 0) return LB_ERR_SHAPE;
  if (r < 1 || r > r_pad) return LB_ERR_RANK;
  if (out_dtype != LB_BF16 && out_dtype != LB_F16) return LB_ERR_DTYPE;
  dim3 grid((C + 255) / 256, r_pad);
  cast_rows_pad16_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      src, src_rs, src_cs, reinterpret_cast<uint16_t*>(dst16), r, C, out_dtype == LB_BF16);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_refresh_shadows(const float* p, const long long* table, int n_entries,
                                  int max_C, void* dst16_base, int out_dtype, void* stream) {
  if (n_entries <= 0 || max_C <= 0) return LB_ERR_SHAPE;
  if (out_dtype != LB_BF16 && out_dtype != LB_F16) return LB_ERR_DTYPE;
  dim3 grid((max_C + 255) / 256, n_entries);
  refresh_shadows_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      p, table, reinterpret_cast<uint16_t*>(dst16_base), out_dtype == LB_BF16);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_cast_weight(const void* src, int src_dtype, void* dst16, void* dstT16, int R,
                              int C, int out_dtype, void* stream) {
  if (R <= 0 || C <= 0) return LB_ERR_SHAPE;
  if (out_dtype != LB_BF16 && out_dtype != LB_F16) return LB_ERR_DTYPE;
  dim3 grid((C + 31) / 32, (R + 31) / 32), block(32, 8);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint16_t* d = reinterpret_cast<uint16_t*>(dst16);
  uint16_t* dT = reinterpret_cast<uint16_t*>(dstT16);
  const int fmt = out_dtype == LB_BF16;
  if (src_dtype == LB_F32)
    cast_weight_kernel<float><<<grid, block, 0, st>>>(reinterpret_cast<const float*>(src), 0, d, dT, R, C, fmt);
  else if (src_dtype == LB_BF16 || src_dtype == LB_F16)
    cast_weight_kernel<uint16_t><<<grid, block, 0, st>>>(reinterpret_cast<const uint16_t*>(src), src_dtype == LB_BF16, d, dT, R, C, fmt);
  else
    return LB_ERR_DTYPE;
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" long long lb_tiled_weight_elems(int N, int K) {
  if (N <= 0 || K <= 0) return 0;
  return static_cast<long long>((N + 63) / 64) * ((K + 63) / 64) * 64 * 64;
}

extern "C" int lb_tile_weight(const void* src, int src_dtype, long long src_rs, long long src_cs, int N, int K,
                              void* dst16, int out_dtype, void* stream) {
  if (N <= 0 || K <= 0) return LB_ERR_SHAPE;
  if (out_dtype != LB_BF16 && out_dtype != LB_F16) return LB_ERR_DTYPE;
  if (reinterpret_cast<uintptr_t>(dst16) & 15) return LB_ERR_ALIGN;
  const int nkb = (K + 63) / 64;
  dim3 grid(nkb, (N + 63) / 64);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint16_t* d = reinterpret_cast<uint16_t*>(dst16);
  const int fmt = out_dtype == LB_BF16;
  if (src_dtype == LB_F32)
    tile_weight_kernel<float><<<grid, 256, 0, st>>>(reinterpret_cast<const float*>(src), 0, src_rs, src_cs, d, N, K, nkb, fmt);
  else if (src_dtype == LB_BF16 || src_dtype == LB_F16)
    tile_weight_kernel<uint16_t><<<grid, 256, 0, st>>>(reinterpret_cast<const uint16_t*>(src), src_dtype == LB_BF16, src_rs,
                                                      src_cs, d, N, K, nkb, fmt);
  else
    return LB_ERR_DTYPE;
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_ti_embed_step(float* rows, float* grad, float* m, float* v, const long long* token_ids,
                                void* table, int table_dtype, int n_rows, int D, const float* lr_dev,
                                float beta1, float beta2, float eps, float weight_decay, int* step_dev,
                                int clip_decay, float target_norm, void* stream) {
  if (n_rows <= 0 || D <= 0) return LB_ERR_SHAPE;
  if (table_dtype != LB_F32 && table_dtype != LB_BF16 && table_dtype != LB_F16) return LB_ERR_DTYPE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // t = ++(*step_dev) on the stream, before the update reads it
  bump_step_kernel<<<1, 1, 0, st>>>(step_dev);
  ti_step_kernel<<<n_rows, 256, 0, st>>>(rows, grad, m, v, token_ids, table, table_dtype, D, lr_dev, beta1,
                                         beta2, eps, weight_decay, step_dev, clip_decay, target_norm);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_lora_merge(const void* W, int w_dtype, const float* up, const float* down, float alpha,
                             void* out, int N, int K, int r, void* stream) {
  if (N <= 0 || K <= 0) return LB_ERR_SHAPE;
  if (r < 1 || r > 64) return LB_ERR_RANK;
  if (w_dtype != LB_F32 && w_dtype != LB_BF16 && w_dtype != LB_F16) return LB_ERR_DTYPE;
  dim3 grid((K + 255) / 256, (N + 7) / 8);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int wf = w_dtype == LB_BF16;
  float* o32 = reinterpret_cast<float*>(out);
  uint16_t* o16 = reinterpret_cast<uint16_t*>(out);
  const float* w32 = reinterpret_cast<const float*>(W);
  const uint16_t* w16 = reinterpret_cast<const uint16_t*>(W);
  if (r <= 16) {
    if (w_dtype == LB_F32) merge_kernel<float><<<grid, 256, 0, st>>>(w32, 0, up, down, alpha, o32, N, K, r);
    else merge_kernel<uint16_t><<<grid, 256, 0, st>>>(w16, wf, up, down, alpha, o16, N, K, r);
  } else {   // ranks 17..64 (joined or wide LoRAs)
    if (w_dtype == LB_F32) merge_kernel<float, 64><<<grid, 256, 0, st>>>(w32, 0, up, down, alpha, o32, N, K, r);
    else merge_kernel<uint16_t, 64><<<grid, 256, 0, st>>>(w16, wf, up, down, alpha, o16, N, K, r);
  }
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_split_bf16x3(const float* src, long long src_rs, void* dst16, int R, int C,
                               int pattern, void* stream) {
  if (R <= 0 || C <= 0 || (pattern != 0 && pattern != 1)) return LB_ERR_SHAPE;
  dim3 grid((C + 255) / 256, R);
  split_bf16x3_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      src, src_rs, reinterpret_cast<uint16_t*>(dst16), R, C, pattern);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_cast_conv_weight(const void* src, int src_dtype, void* dst16, void* dstT16,
                                   int Cout, int Cin, int kh, int kw, int out_dtype,
                                   void* stream) {
  if (Cout <= 0 || Cin <= 0 || kh <= 0 || kw <= 0) return LB_ERR_SHAPE;
  if (out_dtype != LB_BF16 && out_dtype != LB_F16) return LB_ERR_DTYPE;
  const int T = kh * kw;
  const long long total = static_cast<long long>(Cout) * Cin * T;
  const int blocks = static_cast<int>((total + 255) / 256);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint16_t* d = reinterpret_cast<uint16_t*>(dst16);
  uint16_t* dT = reinterpret_cast<uint16_t*>(dstT16);
  const int fmt = out_dtype == LB_BF16;
  if (src_dtype == LB_F32)
    cast_conv_weight_kernel<float><<<blocks, 256, 0, st>>>(reinterpret_cast<const float*>(src), 0, d, dT, Cout, Cin, T, fmt);
  else if (src_dtype == LB_BF16 || src_dtype == LB_F16)
    cast_conv_weight_kernel<uint16_t><<<blocks, 256, 0, st>>>(reinterpret_cast<const uint16_t*>(src), src_dtype == LB_BF16, d, dT, Cout, Cin, T, fmt);
  else
    return LB_ERR_DTYPE;
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_adamw_clip_step(float* p, float* g, float* m, float* v, long long n,
                                  const long long* group_off, int n_groups, const float* lr_dev,
                                  float beta1, float beta2, float eps, float weight_decay,
                                  float max_norm, float inv_world, int* step_dev, float* partials,
                                  float* gnorm_out, void* stream) {
  if (n <= 0 || n_groups < 1 || n_groups > OPT_MAX_GROUPS) return LB_ERR_SHAPE;
  if (reinterpret_cast<uintptr_t>(g) & 15) return LB_ERR_ALIGN;
  OptGroups groups;
  groups.n = n_groups;
  for (int i = 0; i <= n_groups; ++i) groups.off[i] = group_off[i];
  for (int i = n_groups + 1; i <= OPT_MAX_GROUPS; ++i) groups.off[i] = n;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  long long want = (n / 4 + OPT_THREADS - 1) / OPT_THREADS;
  int nblk = static_cast<int>(want < 1 ? 1 : (want > OPT_MAX_PARTIALS ? OPT_MAX_PARTIALS : want));
  sqnorm_partial_kernel<<<nblk, OPT_THREADS, 0, st>>>(g, n, partials, step_dev);
  long long want2 = (n + OPT_THREADS - 1) / OPT_THREADS;
  const int cap2 = 8 * (sm_count() > 0 ? sm_count() : 132);
  int nblk2 = static_cast<int>(want2 > cap2 ? cap2 : want2);
  adamw_update_kernel<<<nblk2, OPT_THREADS, 0, st>>>(p, g, m, v, n, groups, lr_dev, beta1, beta2,
                                                     eps, weight_decay, max_norm, inv_world,
                                                     step_dev, partials, nblk, gnorm_out);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_optim_step_fused(float* p, float* g, float* m, float* v, long long n,
                                   const long long* group_off, int n_groups, const float* lr_dev,
                                   float beta1, float beta2, float eps, float weight_decay,
                                   float max_norm, float inv_world, int* step_dev, float* partials,
                                   float* gnorm_out, const long long* table, int n_entries, int max_C,
                                   void* shadow16, int shadow_dtype, unsigned int* barrier2,
                                   void* stream) {
  if (n <= 0 || n_groups < 1 || n_groups > OPT_MAX_GROUPS) return LB_ERR_SHAPE;
  if (reinterpret_cast<uintptr_t>(g) & 15) return LB_ERR_ALIGN;
  if (n_entries > 0 && (table == nullptr || shadow16 == nullptr || max_C <= 0)) return LB_ERR_SHAPE;
  if (n_entries > 0 && shadow_dtype != LB_BF16 && shadow_dtype != LB_F16) return LB_ERR_DTYPE;
  if (barrier2 == nullptr || partials == nullptr) return LB_ERR_SHAPE;
  OptGroups groups;
  groups.n = n_groups;
  for (int i = 0; i <= n_groups; ++i) groups.off[i] = group_off[i];
  for (int i = n_groups + 1; i <= OPT_MAX_GROUPS; ++i) groups.off[i] = n;
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
    return LB_ERR_CUDA;
  long long want = (n + OPT_THREADS - 1) / OPT_THREADS;
  int nblk = static_cast<int>(want < 1 ? 1 : (want > sms ? sms : want));
  if (nblk > OPT_MAX_PARTIALS) nblk = OPT_MAX_PARTIALS;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(nblk);
  cfg.blockDim = dim3(OPT_THREADS);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = reinterpret_cast<cudaStream_t>(stream);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const int fmt = shadow_dtype == LB_BF16;
  uint16_t* sh = reinterpret_cast<uint16_t*>(shadow16);
  cudaError_t e = cudaLaunchKernelEx(&cfg, optim_step_fused_kernel, p, g, m, v, n, groups, lr_dev, beta1,
                                     beta2, eps, weight_decay, max_norm, inv_world, step_dev, partials, gnorm_out,
                                     table, n_entries, max_C, sh, fmt, barrier2);
  return e == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

// ------------------------------------------------------------------------------- CUDA IPC helpers
// Peer mappings for lb_optim_step_dp: export a device pointer (any pointer inside a cudaMalloc'ed
// block, e.g. a slice of a torch caching-allocator segment) as (IPC handle of the block, byte offset
// inside it); open such a handle in another process of the same node. Opening enables peer access
// from the current device to the exporting one (cudaIpcMemLazyEnablePeerAccess).
extern "C" int lb_ipc_export(const void* ptr, void* handle64, long long* offset) {
  if (ptr == nullptr || handle64 == nullptr || offset == nullptr) return LB_ERR_SHAPE;
  typedef CUresult (*GetRangeFn)(CUdeviceptr*, size_t*, CUdeviceptr);
  static GetRangeFn fn = nullptr;
  if (fn == nullptr) {
    void* pfn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &pfn, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return LB_ERR_CUDA;
    fn = reinterpret_cast<GetRangeFn>(pfn);
  }
  CUdeviceptr base = 0;
  size_t size = 0;
  if (fn(&base, &size, reinterpret_cast<CUdeviceptr>(ptr)) != CUDA_SUCCESS) return LB_ERR_CUDA;
  cudaIpcMemHandle_t h;
  if (cudaIpcGetMemHandle(&h, reinterpret_cast<void*>(base)) != cudaSuccess) {
    cudaGetLastError();
    return LB_ERR_CUDA;
  }
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle64, &h, 64);
  *offset = static_cast<long long>(reinterpret_cast<CUdeviceptr>(ptr) - base);
  return LB_OK;
}

extern "C" int lb_ipc_open(const void* handle64, void** base_out) {
  if (handle64 == nullptr || base_out == nullptr) return LB_ERR_SHAPE;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  void* p = nullptr;
  if (cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
    cudaGetLastError();
    return LB_ERR_CUDA;
  }
  *base_out = p;
  return LB_OK;
}

extern "C" int lb_optim_step_dp(float* p, float* g, float* gsum, float* m, float* v, long long n,
                                const long long* group_off, int n_groups, const float* lr_dev,
                                float beta1, float beta2, float eps, float weight_decay, float max_norm,
                                int* step_dev, float* partials, float* gnorm_out, const long long* table,
                                int n_entries, int max_C, void* shadow16, int shadow_dtype,
                                unsigned int* barrier2, const void* const* peer_g,
                                void* const* peer_flags, int world, int rank, unsigned int* epoch_dev,
                                void* stream) {
  if (n <= 0 || n_groups < 1 || n_groups > OPT_MAX_GROUPS) return LB_ERR_SHAPE;
  if (world < 1 || world > DP_MAX_WORLD || rank < 0 || rank >= world) return LB_ERR_SHAPE;
  if (peer_g == nullptr || peer_flags == nullptr || gsum == nullptr || epoch_dev == nullptr) return LB_ERR_SHAPE;
  if ((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(gsum)) & 15) return LB_ERR_ALIGN;
  if (n_entries > 0 && (table == nullptr || shadow16 == nullptr || max_C <= 0)) return LB_ERR_SHAPE;
  if (n_entries > 0 && shadow_dtype != LB_BF16 && shadow_dtype != LB_F16) return LB_ERR_DTYPE;
  if (barrier2 == nullptr || partials == nullptr) return LB_ERR_SHAPE;
  OptGroups groups;
  groups.n = n_groups;
  for (int i = 0; i <= n_groups; ++i) groups.off[i] = group_off[i];
  for (int i = n_groups + 1; i <= OPT_MAX_GROUPS; ++i) groups.off[i] = n;
  DpPeers peers = {};
  for (int r = 0; r < world; ++r) {
    if (peer_g[r] == nullptr || peer_flags[r] == nullptr || (reinterpret_cast<uintptr_t>(peer_g[r]) & 15))
      return LB_ERR_ALIGN;
    peers.g[r] = reinterpret_cast<const float*>(peer_g[r]);
    peers.flags[r] = reinterpret_cast<unsigned int*>(peer_flags[r]);
  }
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
    return LB_ERR_CUDA;
  long long want = (n / 4 + OPT_THREADS - 1) / OPT_THREADS;
  int nblk = static_cast<int>(want < 1 ? 1 : (want > sms ? sms : want));
  if (nblk > OPT_MAX_PARTIALS) nblk = OPT_MAX_PARTIALS;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(nblk);
  cfg.blockDim = dim3(OPT_THREADS);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = reinterpret_cast<cudaStream_t>(stream);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const int fmt = shadow_dtype == LB_BF16;
  uint16_t* sh = reinterpret_cast<uint16_t*>(shadow16);
  cudaError_t e = cudaLaunchKernelEx(&cfg, optim_step_dp_kernel, p, g, gsum, m, v, n, groups, lr_dev, beta1,
                                     beta2, eps, weight_decay, max_norm, step_dev, partials, gnorm_out, table,
                                     n_entries, max_C, sh, fmt, barrier2, peers, world, rank, epoch_dev);
  return e == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}
