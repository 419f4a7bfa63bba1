// lb_svd_truncated_batched: the whole SVD distillation of /root/reference/lora_diffusion/cli_svd.py:24-92
// (`overwrite_base`: per site  dW = W_tuned - W_base -> SVD -> U_r diag(S_r), Vh_r -> quantile clamp)
// for ALL sites of a model in one C call, ragged over shapes.
//
// Algorithm (per matrix, all matrices in flight together): randomized range finder with L = 32
// Rademacher probes and q power iterations, then the exact SVD of the projected 32 x K problem:
//     Y = dW Om ; [ Z = dW^T orth(Y) ; Y = dW orth(Z) ] x q ; Q = orth2(Y) ; B^T = dW^T Q ;
//     B B^T = Uh diag(s^2) Uh^T ;  up = Q Uh_r diag(s_r) ;  down = diag(1/s_r) Uh_r^T B
// = 2q + 2 streaming passes over (W_tuned, W_base); dW is formed in registers and never stored.
// orth() = Gram matrix -> 32 x 32 Jacobi eigen-decomposition -> multiply by V diag(1/s)
// (rank-revealing: numerically null directions become zero columns -- an exactly low-rank delta,
// i.e. a merged LoRA, is a real input).
//
// Kernels:
//   mul_right / mul_left   the passes. HBM-bound: AI = 2*32 flop per 4 bytes = 16 flop/B, i.e.
//       ~54 TFLOP/s at the H100's 3.35 TB/s data-sheet bandwidth -- near the fp32 CUDA cores' 67
//       TFLOP/s data-sheet peak, so the contraction runs on the tensor cores: the fp32 delta tile is split in registers into
//       bf16 hi + lo, the tall-skinny operand likewise, and hi.hi + lo.hi + hi.lo are accumulated
//       in fp32 with mma.sync.m16n8k16 (2^-16 relative per product: fp32-faithful; wgmma would
//       need the operands staged in its shared-memory layouts and buys nothing on a memory-bound
//       pass). Weights come in through 16-byte vector loads, one tile ahead in registers.
//   mul_right also accumulates the Gram matrix of its output tile (no separate pass over Y).
//   tall_transform         Y <- Y V diag(1/s) (+ Gram of the result), or Gram only
//   jacobi32               block-wide cyclic Jacobi, 16 disjoint rotations per step in parallel
//   factors                up / down from (Q, B^T, Uh, s)
//   quantile_clamp         exact radix select of torch.quantile's two order statistics over
//                          cat(up, down) (cli_svd.py:43-47), lerp, symmetric clamp, in place
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include <vector>

#include "lora_b200.h"

namespace lbsvd2 {

constexpr int L = 32;     // probe / subspace width
constexpr int TM = 128;   // rows of a weight tile
constexpr int THREADS = 256;

struct MatDesc {
  const void* wt;
  const void* wb;          // may be null (dW = W_tuned)
  int N, K;
  long long yoff;          // first row of this matrix in the [sum N, 32] workspace
  long long zoff;          // first row in the [sum K, 32] workspace
  long long out_off;       // element offset of [up (N x r) | down (r x K)] in the flat fp32 output
};
struct RItem { int b, row0; };            // mul_right: one 128-row block of matrix b
struct LItem { int b, k0, n0, n1; };      // mul_left : one KT-column block x row slab [n0, n1)
struct TItem { int b, row0; };            // tall kernels: one 256-row block

// ------------------------------------------------------------------------------------ helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint4 ldg16(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2_t(uint32_t addr, uint32_t (&r)[2]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];"
               : "=r"(r[0]), "=r"(r[1]) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// fp32 pair -> (bf16 hi pair, bf16 lo pair); x = hi + lo + O(2^-16 |x|)
__device__ __forceinline__ void split2(float x, float y, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat16 hx = __float2bfloat16_rn(x), hy = __float2bfloat16_rn(y);
  const __nv_bfloat16 lx = __float2bfloat16_rn(x - __bfloat162float(hx));
  const __nv_bfloat16 ly = __float2bfloat16_rn(y - __bfloat162float(hy));
  hi = static_cast<uint32_t>(*reinterpret_cast<const uint16_t*>(&hx)) |
       (static_cast<uint32_t>(*reinterpret_cast<const uint16_t*>(&hy)) << 16);
  lo = static_cast<uint32_t>(*reinterpret_cast<const uint16_t*>(&lx)) |
       (static_cast<uint32_t>(*reinterpret_cast<const uint16_t*>(&ly)) << 16);
}

template <typename WT> struct WTraits;
template <> struct WTraits<__half> {
  static constexpr int KT = 64, VEC = 8;
  static __device__ __forceinline__ void diff(const uint4& t, const uint4& b, float (&d)[8]) {
    const __half2* a = reinterpret_cast<const __half2*>(&t);
    const __half2* c = reinterpret_cast<const __half2*>(&b);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 x = __half22float2(a[i]), y = __half22float2(c[i]);
      d[2 * i] = x.x - y.x; d[2 * i + 1] = x.y - y.y;
    }
  }
};
template <> struct WTraits<__nv_bfloat16> {
  static constexpr int KT = 64, VEC = 8;
  static __device__ __forceinline__ void diff(const uint4& t, const uint4& b, float (&d)[8]) {
    const __nv_bfloat162* a = reinterpret_cast<const __nv_bfloat162*>(&t);
    const __nv_bfloat162* c = reinterpret_cast<const __nv_bfloat162*>(&b);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 x = __bfloat1622float2(a[i]), y = __bfloat1622float2(c[i]);
      d[2 * i] = x.x - y.x; d[2 * i + 1] = x.y - y.y;
    }
  }
};
template <> struct WTraits<float> {
  static constexpr int KT = 32, VEC = 4;
  static __device__ __forceinline__ void diff(const uint4& t, const uint4& b, float (&d)[4]) {
    d[0] = __uint_as_float(t.x) - __uint_as_float(b.x);
    d[1] = __uint_as_float(t.y) - __uint_as_float(b.y);
    d[2] = __uint_as_float(t.z) - __uint_as_float(b.z);
    d[3] = __uint_as_float(t.w) - __uint_as_float(b.w);
  }
};

// A [rows x KT] bf16 tile in shared memory: row pitch KT*2 bytes (128 or 64), 16-byte chunks
// XOR-swizzled so that both ldmatrix (8 rows, same chunk) and the 16-byte row stores are
// bank-conflict free. Also used for the [k or n][32] tall-skinny chunks (pitch 64 bytes).
template <int KT>
__device__ __forceinline__ uint32_t tile_off(int row, int chunk) {
  if constexpr (KT == 64) return row * 128 + ((chunk ^ (row & 7)) << 4);
  else return row * 64 + ((chunk ^ ((row >> 1) & 3)) << 4);
}

// Weight tiles [128 rows x 128 bytes] of both models travel global -> shared through a 2-slot
// cp.async ring (slot = 2 weights x 16 KB, raw element type), issued one whole step ahead -- at the
// START of the step that converts the previous tile, which a register prefetch could not do without
// doubling its registers; with 2 CTAs per SM that keeps 64 KB per SM in flight. Thread mapping:
// 16-byte chunk c = tid & 7 of rows (tid >> 3) + 32 j, j = 0..3: a warp touches 4 full 128-byte rows
// per instruction (coalesced in global memory, conflict-free in shared memory), and every thread later
// reads back exactly the chunks it requested (no barrier needed for the raw data).
constexpr int RAW_W_BYTES = TM * 128;            // one weight's tile
constexpr int RAW_STAGE_BYTES = 2 * RAW_W_BYTES;
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void st_zero16(uint32_t dst) {
  asm volatile("st.shared.v4.b32 [%0], {%1,%1,%1,%1};" ::"r"(dst), "r"(0u) : "memory");
}
__device__ __forceinline__ uint4 lds16(uint32_t src) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(src));
  return v;
}
// request the [128 x KT] tile whose first row is `row0` (rows >= row_end or >= N: zeros) and first
// column `k0` into ring slot `slot`; one commit group per call
template <typename WT>
__device__ __forceinline__ void issue_tile(uint32_t raw, int slot, const MatDesc& m, int row0, int row_end, int k0) {
  constexpr int VEC = WTraits<WT>::VEC;
  const int c = threadIdx.x & 7;
  const int k = k0 + c * VEC;
  const bool k_ok = k + VEC <= m.K;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int r = (threadIdx.x >> 3) + 32 * j;
    const int n = row0 + r;
    const bool ok = k_ok && n < row_end && n < m.N;
    const uint32_t dst = raw + slot * RAW_STAGE_BYTES + r * 128 + c * 16;
    if (ok) {
      cp_async16(dst, reinterpret_cast<const WT*>(m.wt) + static_cast<size_t>(n) * m.K + k);
      if (m.wb) cp_async16(dst + RAW_W_BYTES, reinterpret_cast<const WT*>(m.wb) + static_cast<size_t>(n) * m.K + k);
      else st_zero16(dst + RAW_W_BYTES);
    } else {
      st_zero16(dst);
      st_zero16(dst + RAW_W_BYTES);
    }
  }
  cp_async_commit();
}
// raw slot -> (W_tuned - W_base) split into bf16 hi / lo tiles in the swizzled MMA layout
template <typename WT, bool LO = true>
__device__ __forceinline__ void convert_tile(uint32_t raw, int slot, uint32_t s_hi, uint32_t s_lo) {
  constexpr int KT = WTraits<WT>::KT;
  const int c = threadIdx.x & 7;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int r = (threadIdx.x >> 3) + 32 * j;
    const uint32_t src = raw + slot * RAW_STAGE_BYTES + r * 128 + c * 16;
    const uint4 t = lds16(src), b = lds16(src + RAW_W_BYTES);
    if constexpr (sizeof(WT) == 2) {
      float d[8];
      WTraits<WT>::diff(t, b, d);
      uint32_t h[4], l[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) split2(d[2 * q], d[2 * q + 1], h[q], l[q]);
      const uint32_t off = tile_off<KT>(r, c);
      asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(s_hi + off), "r"(h[0]), "r"(h[1]), "r"(h[2]), "r"(h[3]) : "memory");
      if constexpr (LO)
        asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(s_lo + off), "r"(l[0]), "r"(l[1]), "r"(l[2]), "r"(l[3]) : "memory");
    } else {
      float d[4];
      WTraits<WT>::diff(t, b, d);
      uint32_t h[2], l[2];
      split2(d[0], d[1], h[0], l[0]);
      split2(d[2], d[3], h[1], l[1]);
      const uint32_t off = tile_off<KT>(r, c >> 1) + (c & 1) * 8;    // 4 fp32 = half a 16-byte bf16 chunk
      asm volatile("st.shared.v2.b32 [%0], {%1,%2};" ::"r"(s_hi + off), "r"(h[0]), "r"(h[1]) : "memory");
      if constexpr (LO)
        asm volatile("st.shared.v2.b32 [%0], {%1,%2};" ::"r"(s_lo + off), "r"(l[0]), "r"(l[1]) : "memory");
    }
  }
}

// 8 consecutive fp32 of one row of a [rows, 32] tall-skinny operand -> one 16-byte chunk (hi, lo)
template <bool LO = true>
__device__ __forceinline__ void store_tall8(const float4& a, const float4& b, uint32_t s_hi, uint32_t s_lo,
                                            int row, int chunk) {
  uint32_t h[4], l[4];
  split2(a.x, a.y, h[0], l[0]); split2(a.z, a.w, h[1], l[1]);
  split2(b.x, b.y, h[2], l[2]); split2(b.z, b.w, h[3], l[3]);
  const uint32_t off = tile_off<32>(row, chunk);
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(s_hi + off), "r"(h[0]), "r"(h[1]), "r"(h[2]), "r"(h[3]) : "memory");
  if constexpr (LO)
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(s_lo + off), "r"(l[0]), "r"(l[1]), "r"(l[2]), "r"(l[3]) : "memory");
}

// ------------------------------------------------------------------------------------ Y = dW . Z
// CTA = one 128-row block of one matrix, K walked in KT-column steps. Warp w owns rows
// [16w, 16w+16) x all 32 columns (4 n8 tiles). Optional fused Gram of the output tile.
// TERMS = how many of the split products are accumulated: 3 = hi.hi + lo.hi + hi.lo (fp32-faithful),
// 2 = hi.hi + lo.hi (dW exact, the tall operand rounded to bf16: exact for the +-1 probes, and a
// product with a rounded operand still lies in range(dW), which is what the basis needs),
// 1 = hi.hi (bf16 product: only ever for an intermediate power-iteration pass).
template <typename WT, int TERMS>
__global__ void __launch_bounds__(THREADS, 2)
mul_right_kernel(const MatDesc* __restrict__ mats, const RItem* __restrict__ items,
                 const float* __restrict__ Zin, float* __restrict__ Yout, float* __restrict__ G) {
  constexpr int KT = WTraits<WT>::KT;
  constexpr int TILE_BYTES = TM * KT * 2;
  constexpr int ZS_BYTES = KT * 64;
  extern __shared__ __align__(128) uint8_t smem[];   // [raw ring 2 x 32 KB | hi | lo | Zs hi | Zs lo]
  const uint32_t raw = smem_u32(smem);
  const uint32_t s_hi = raw + 2 * RAW_STAGE_BYTES, s_lo = s_hi + TILE_BYTES;
  const uint32_t z_hi = s_lo + TILE_BYTES, z_lo = z_hi + ZS_BYTES;

  const RItem it = items[blockIdx.x];
  const MatDesc m = mats[it.b];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nsteps = (m.K + KT - 1) / KT;
  const float* z = Zin + static_cast<size_t>(m.zoff) * L;

  // tall-skinny chunk [KT x 32]: thread -> row zr, 8 columns starting at zc*8 (two rounds for KT = 64)
  const int zr = tid >> 2, zc = tid & 3;
  constexpr int ZROUNDS = KT / 64 + (KT % 64 ? 1 : 0);   // 1 (KT = 32 uses half the threads) or 1 (64)
  auto load_z = [&](int k0, float4 (&v)[2]) {
    const int k = k0 + zr;
    if (zr < KT && k < m.K) {
      const float4* src = reinterpret_cast<const float4*>(z + static_cast<size_t>(k) * L + zc * 8);
      v[0] = __ldg(src); v[1] = __ldg(src + 1);
    } else {
      v[0] = v[1] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  (void)ZROUNDS;

  float4 zv[2];
  issue_tile<WT>(raw, 0, m, it.row0, m.N, 0);
  load_z(0, zv);

  float acc[4][4] = {};
  for (int step = 0; step < nsteps; ++step) {
    if (step + 1 < nsteps) {                           // next tile: requested a whole step ahead
      issue_tile<WT>(raw, (step + 1) & 1, m, it.row0, m.N, (step + 1) * KT);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();                                   // previous step's MMAs have read the operand tiles
    convert_tile<WT, (TERMS >= 2)>(raw, step & 1, s_hi, s_lo);
    if (zr < KT) store_tall8<(TERMS == 3)>(zv[0], zv[1], z_hi, z_lo, zr, zc);
    __syncthreads();
    if (step + 1 < nsteps) load_z((step + 1) * KT, zv);
#pragma unroll
    for (int ks = 0; ks < KT / 16; ++ks) {
      uint32_t ah[4], al[4];
      const uint32_t a_off = tile_off<KT>(warp * 16 + (lane & 15), ks * 2 + (lane >> 4));
      ldsm_x4(s_hi + a_off, ah);
      if constexpr (TERMS >= 2) ldsm_x4(s_lo + a_off, al);
#pragma unroll
      for (int np = 0; np < 2; ++np) {
        uint32_t bh[4], bl[4];
        const uint32_t b_off = tile_off<32>(ks * 16 + ((lane >> 3) & 1) * 8 + (lane & 7), np * 2 + (lane >> 4));
        ldsm_x4_t(z_hi + b_off, bh);
        if constexpr (TERMS == 3) ldsm_x4_t(z_lo + b_off, bl);
        mma_bf16(acc[2 * np], ah, bh[0], bh[1]);
        if constexpr (TERMS >= 2) mma_bf16(acc[2 * np], al, bh[0], bh[1]);
        if constexpr (TERMS == 3) mma_bf16(acc[2 * np], ah, bl[0], bl[1]);
        mma_bf16(acc[2 * np + 1], ah, bh[2], bh[3]);
        if constexpr (TERMS >= 2) mma_bf16(acc[2 * np + 1], al, bh[2], bh[3]);
        if constexpr (TERMS == 3) mma_bf16(acc[2 * np + 1], ah, bl[2], bl[3]);
      }
    }
  }
  // ---- output: c0,c1 = (row g, cols 2t,2t+1), c2,c3 = (row g+8, same cols) of each n8 tile
  const int g = lane >> 2, t = lane & 3;
  float* y = Yout + static_cast<size_t>(m.yoff) * L;
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    const int r0 = it.row0 + warp * 16 + g, c = nt * 8 + 2 * t;
    if (r0 < m.N) *reinterpret_cast<float2*>(y + static_cast<size_t>(r0) * L + c) = make_float2(acc[nt][0], acc[nt][1]);
    if (r0 + 8 < m.N) *reinterpret_cast<float2*>(y + static_cast<size_t>(r0 + 8) * L + c) = make_float2(acc[nt][2], acc[nt][3]);
  }
  if (G != nullptr) {
    // Gram of the tile through shared memory (rows beyond N are zero: they came from zero tiles)
    __syncthreads();
    float* ys = reinterpret_cast<float*>(smem);        // [128][33] fp32 = 16.9 KB <= tile bytes
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      const int r0 = warp * 16 + g, c = nt * 8 + 2 * t;
      ys[r0 * 33 + c] = acc[nt][0]; ys[r0 * 33 + c + 1] = acc[nt][1];
      ys[(r0 + 8) * 33 + c] = acc[nt][2]; ys[(r0 + 8) * 33 + c + 1] = acc[nt][3];
    }
    __syncthreads();
    const int i = tid >> 3, j0 = (tid & 7) * 4;
    float s[4] = {};
#pragma unroll 8
    for (int r = 0; r < TM; ++r) {
      const float a = ys[r * 33 + i];
#pragma unroll
      for (int q = 0; q < 4; ++q) s[q] += a * ys[r * 33 + j0 + q];
    }
    float* gdst = G + static_cast<size_t>(it.b) * L * L + i * L + j0;
#pragma unroll
    for (int q = 0; q < 4; ++q) atomicAdd(gdst + q, s[q]);
  }
}

// ------------------------------------------------------------------------------------ Z += dW^T . Q
// CTA = one KT-column block x row slab of one matrix; computes the [32 x KT] partial
// (Q^T)[32 x n] . dW[n x KT] (A = Q^T through ldmatrix.trans of the [n][32] chunk, B = the weight
// tile through ldmatrix.trans) and adds it into Z[k][col] with fp32 atomics (Z zeroed beforehand).
// Warp w: m16 tile (w & 1) of the 32 Q-columns, n8 tiles [(w>>1)*NT, +NT) of the KT weight columns.
template <typename WT, int TERMS>
__global__ void __launch_bounds__(THREADS, 2)
mul_left_kernel(const MatDesc* __restrict__ mats, const LItem* __restrict__ items,
                const float* __restrict__ Qin, float* __restrict__ Zout) {
  constexpr int KT = WTraits<WT>::KT;
  constexpr int NT = KT / 32;                           // n8 tiles per warp: 2 (KT 64) or 1 (KT 32)
  constexpr int TILE_BYTES = TM * KT * 2;
  constexpr int QS_BYTES = TM * 64;
  extern __shared__ __align__(128) uint8_t smem[];   // [raw ring 2 x 32 KB | hi | lo | Qs hi | Qs lo]
  const uint32_t raw = smem_u32(smem);
  const uint32_t s_hi = raw + 2 * RAW_STAGE_BYTES, s_lo = s_hi + TILE_BYTES;
  const uint32_t q_hi = s_lo + TILE_BYTES, q_lo = q_hi + QS_BYTES;

  const LItem it = items[blockIdx.x];
  const MatDesc m = mats[it.b];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int row = tid >> 1, half = tid & 1;
  const int mt = warp & 1, ng = warp >> 1;
  const float* qsrc = Qin + static_cast<size_t>(m.yoff) * L;
  const int nsteps = (it.n1 - it.n0 + TM - 1) / TM;

  // Q chunk [128 x 32]: thread -> row tid/2, 16 columns starting at (tid&1)*16 (2 chunks of 8)
  auto load_q = [&](int n_base, float4 (&v)[4]) {
    const int n = n_base + row;
    if (n < it.n1) {
      const float4* src = reinterpret_cast<const float4*>(qsrc + static_cast<size_t>(n) * L + half * 16);
      v[0] = __ldg(src); v[1] = __ldg(src + 1); v[2] = __ldg(src + 2); v[3] = __ldg(src + 3);
    } else {
      v[0] = v[1] = v[2] = v[3] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  // rows beyond the slab are zero in both operands (Q rows and weight tile rows)
  float4 qv[4];
  issue_tile<WT>(raw, 0, m, it.n0, it.n1, it.k0);
  load_q(it.n0, qv);

  float acc[NT][4] = {};
  for (int step = 0; step < nsteps; ++step) {
    if (step + 1 < nsteps) {
      issue_tile<WT>(raw, (step + 1) & 1, m, it.n0 + (step + 1) * TM, it.n1, it.k0);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    convert_tile<WT, (TERMS >= 2)>(raw, step & 1, s_hi, s_lo);
    store_tall8<(TERMS == 3)>(qv[0], qv[1], q_hi, q_lo, row, half * 2);
    store_tall8<(TERMS == 3)>(qv[2], qv[3], q_hi, q_lo, row, half * 2 + 1);
    __syncthreads();
    if (step + 1 < nsteps) load_q(it.n0 + (step + 1) * TM, qv);
#pragma unroll
    for (int ks = 0; ks < TM / 16; ++ks) {
      // A = Q^T: a0 (m 0-7, kk 0-7), a1 (m 8-15, kk 0-7), a2 (m 0-7, kk 8-15), a3 (m 8-15, kk 8-15);
      // source 8x8 blocks are rows kk (n), 16-byte chunk = 8 Q-columns, transposed on load
      uint32_t ah[4], al[4];
      const uint32_t a_off = tile_off<32>(ks * 16 + (lane >> 4) * 8 + (lane & 7), mt * 2 + ((lane >> 3) & 1));
      ldsm_x4_t(q_hi + a_off, ah);
      if constexpr (TERMS == 3) ldsm_x4_t(q_lo + a_off, al);     // tall operand's low half
      if constexpr (NT == 2) {
        uint32_t bh[4], bl[4];
        const uint32_t b_off = tile_off<KT>(ks * 16 + ((lane >> 3) & 1) * 8 + (lane & 7), ng * 2 + (lane >> 4));
        ldsm_x4_t(s_hi + b_off, bh);
        if constexpr (TERMS >= 2) ldsm_x4_t(s_lo + b_off, bl);   // dW's low half
        mma_bf16(acc[0], ah, bh[0], bh[1]);
        if constexpr (TERMS == 3) mma_bf16(acc[0], al, bh[0], bh[1]);
        if constexpr (TERMS >= 2) mma_bf16(acc[0], ah, bl[0], bl[1]);
        mma_bf16(acc[1], ah, bh[2], bh[3]);
        if constexpr (TERMS == 3) mma_bf16(acc[1], al, bh[2], bh[3]);
        if constexpr (TERMS >= 2) mma_bf16(acc[1], ah, bl[2], bl[3]);
      } else {
        uint32_t bh[2], bl[2];
        const uint32_t b_off = tile_off<KT>(ks * 16 + ((lane >> 3) & 1) * 8 + (lane & 7), ng);
        ldsm_x2_t(s_hi + b_off, bh);
        if constexpr (TERMS >= 2) ldsm_x2_t(s_lo + b_off, bl);
        mma_bf16(acc[0], ah, bh[0], bh[1]);
        if constexpr (TERMS == 3) mma_bf16(acc[0], al, bh[0], bh[1]);
        if constexpr (TERMS >= 2) mma_bf16(acc[0], ah, bl[0], bl[1]);
      }
    }
  }
  // c0,c1 = (Q column mt*16+g, weight columns k0 + n8*8 + 2t, +1); c2,c3 = Q column +8
  const int g = lane >> 2, t = lane & 3;
  float* zdst = Zout + static_cast<size_t>(m.zoff) * L;
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    const int k = it.k0 + (ng * NT + j) * 8 + 2 * t;
    const int c = mt * 16 + g;
    if (k < m.K) {
      atomicAdd(zdst + static_cast<size_t>(k) * L + c, acc[j][0]);
      atomicAdd(zdst + static_cast<size_t>(k) * L + c + 8, acc[j][2]);
    }
    if (k + 1 < m.K) {
      atomicAdd(zdst + static_cast<size_t>(k + 1) * L + c, acc[j][1]);
      atomicAdd(zdst + static_cast<size_t>(k + 1) * L + c + 8, acc[j][3]);
    }
  }
}

// ------------------------------------------------------------------------------------ probes
// Rademacher (+-1) probes: as good a test matrix as Gaussians for the range finder (sub-Gaussian),
// one hash per 32 entries.
__global__ void probes_kernel(float* __restrict__ Z, long long rows, unsigned long long seed) {
  const long long r = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (r >= rows) return;
  unsigned long long z = seed + static_cast<unsigned long long>(r) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  const uint32_t bits = static_cast<uint32_t>(z >> 16);
  float4* dst = reinterpret_cast<float4*>(Z + r * L);
#pragma unroll
  for (int i = 0; i < 8; ++i)
    dst[i] = make_float4((bits >> (4 * i)) & 1 ? 1.f : -1.f, (bits >> (4 * i + 1)) & 1 ? 1.f : -1.f,
                         (bits >> (4 * i + 2)) & 1 ? 1.f : -1.f, (bits >> (4 * i + 3)) & 1 ? 1.f : -1.f);
}

// ------------------------------------------------------------------------------------ tall transform
// out_row = in_row . M with M = V diag(1/s) (null directions, s_j <= 1e-6 s_0, dropped), in place
// allowed; optional Gram of the OUTPUT rows (mode bit 1) -- or Gram only, no multiply (mode bit 0
// clear). space: 0 = rows indexed through yoff / N, 1 = through zoff / K.
__global__ void __launch_bounds__(THREADS)
tall_transform_kernel(const MatDesc* __restrict__ mats, const TItem* __restrict__ items, int space,
                      float* __restrict__ buf, const float* __restrict__ V, const float* __restrict__ sig,
                      int do_mul, float* __restrict__ G) {
  __shared__ float Ms[L][L + 1];
  __shared__ float rows_s[THREADS][L + 1];
  const TItem it = items[blockIdx.x];
  const MatDesc m = mats[it.b];
  const int rows = space ? m.K : m.N;
  float* base = buf + static_cast<size_t>(space ? m.zoff : m.yoff) * L;
  const int tid = threadIdx.x;
  if (do_mul) {
    const float* v = V + static_cast<size_t>(it.b) * L * L;
    const float* s = sig + static_cast<size_t>(it.b) * L;
    const float smax = s[0];
    for (int i = tid; i < L * L; i += THREADS) {
      const int r = i >> 5, c = i & 31;
      const float sc = s[c];
      Ms[r][c] = (sc > 1e-6f * smax && sc > 0.f) ? v[i] / sc : 0.f;
    }
  }
  __syncthreads();
  const int row = it.row0 + tid;
  float x[L];
  if (row < rows) {
    const float4* src = reinterpret_cast<const float4*>(base + static_cast<size_t>(row) * L);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 a = src[i];
      x[4 * i] = a.x; x[4 * i + 1] = a.y; x[4 * i + 2] = a.z; x[4 * i + 3] = a.w;
    }
  } else {
#pragma unroll
    for (int i = 0; i < L; ++i) x[i] = 0.f;
  }
  if (do_mul) {
    float o[L];
#pragma unroll
    for (int j = 0; j < L; ++j) o[j] = 0.f;
#pragma unroll
    for (int i = 0; i < L; ++i) {
      const float xi = x[i];
#pragma unroll
      for (int j = 0; j < L; ++j) o[j] += xi * Ms[i][j];
    }
#pragma unroll
    for (int j = 0; j < L; ++j) x[j] = o[j];
    if (row < rows) {
      float4* dst = reinterpret_cast<float4*>(base + static_cast<size_t>(row) * L);
#pragma unroll
      for (int i = 0; i < 8; ++i) dst[i] = make_float4(x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
    }
  }
  if (G != nullptr) {
#pragma unroll
    for (int j = 0; j < L; ++j) rows_s[tid][j] = x[j];
    __syncthreads();
    const int i = tid >> 3, j0 = (tid & 7) * 4;
    float s4[4] = {};
#pragma unroll 8
    for (int r = 0; r < THREADS; ++r) {
      const float a = rows_s[r][i];
#pragma unroll
      for (int q = 0; q < 4; ++q) s4[q] += a * rows_s[r][j0 + q];
    }
    float* gdst = G + static_cast<size_t>(it.b) * L * L + i * L + j0;
#pragma unroll
    for (int q = 0; q < 4; ++q) atomicAdd(gdst + q, s4[q]);
  }
}

// ------------------------------------------------------------------------------------ Jacobi
// One CTA (256 threads) per symmetric 32x32 matrix: cyclic two-sided Jacobi, round-robin ordering.
// A step applies 16 disjoint rotations J = diag(J_0..J_15); A <- J^T A J decomposes into 16 x 16
// independent 2x2 blocks {p_k,q_k} x {p_l,q_l}, ONE PER THREAD (k = tid / 16 rotates the block's
// rows, l = tid % 16 its columns), so a step is: read (block + the column rotation's pivots) ->
// barrier -> write -> barrier. Every lane derives the rotation of its column pair and fetches the
// row pair's from a lane of its own warp (no serial 16-thread phase); the round-robin pairing is
// tabulated once (no permutation array to maintain): 2 barriers per step instead of 5 (a solve is
// latency-bound on the barriers).
// Outputs eigenvectors (columns, descending eigenvalue) and sqrt(max(eig, 0)).
__device__ __forceinline__ int rr_elem(int pos, int step) {   // element at tournament position `pos` after `step` rotations
  if (pos == 0) return 0;
  int e = (pos - 1 - step) % (L - 1);
  if (e < 0) e += L - 1;
  return e + 1;
}
__device__ __forceinline__ void jacobi_rot(float app, float aqq, float apq, float& c, float& s) {
  c = 1.f; s = 0.f;
  if (fabsf(apq) > 1e-30f) {
    const float tau = (aqq - app) / (2.f * apq);
    const float tt = (tau >= 0.f ? 1.f : -1.f) / (fabsf(tau) + sqrtf(1.f + tau * tau));
    c = rsqrtf(1.f + tt * tt);
    s = tt * c;
  }
}
__global__ void __launch_bounds__(256)
jacobi32_kernel(const float* __restrict__ G, float* __restrict__ V, float* __restrict__ sigma, int sweeps,
                float tol) {
  __shared__ float A[L][L + 1];
  __shared__ float Q[L][L + 1];
  __shared__ float wmax[8];
  __shared__ unsigned char pair_p[L - 1][16], pair_q[L - 1][16];   // the tournament, tabulated once
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* g = G + static_cast<size_t>(b) * L * L;
  for (int i = tid; i < L * L; i += 256) {
    A[i >> 5][i & 31] = g[i];
    Q[i >> 5][i & 31] = ((i >> 5) == (i & 31)) ? 1.f : 0.f;
  }
  for (int i = tid; i < (L - 1) * 16; i += 256) {
    const int step = i >> 4, kk = i & 15;
    int pp = rr_elem(kk, step), qq = rr_elem(L - 1 - kk, step);
    if (pp > qq) { const int t = pp; pp = qq; qq = t; }
    pair_p[step][kk] = static_cast<unsigned char>(pp);
    pair_q[step][kk] = static_cast<unsigned char>(qq);
  }
  __syncthreads();
  // lane = (k & 1) * 16 + l: every lane derives the rotation of ITS COLUMN pair l; the row pair k's
  // rotation is the one lane (k & 1) * 16 + k of the same warp derived (k < 16): two shuffles
  const int k = tid >> 4, l = tid & 15;
  const int src_lane = (tid & 16) + k;
  for (int sw = 0; sw < sweeps; ++sw) {
    float seen = 0.f;       // largest relative off-diagonal this thread met in the sweep
    for (int step = 0; step < L - 1; ++step) {
      const int pk = pair_p[step][k], qk = pair_q[step][k];
      const int pl = pair_p[step][l], ql = pair_q[step][l];
      float cl, sl;
      {
        const float apq = A[pl][ql], app = A[pl][pl], aqq = A[ql][ql];
        jacobi_rot(app, aqq, apq, cl, sl);
        seen = fmaxf(seen, fabsf(apq) * rsqrtf(fmaxf(fabsf(app * aqq), 1e-37f)));
      }
      const float ck = __shfl_sync(0xffffffffu, cl, src_lane);
      const float sk = __shfl_sync(0xffffffffu, sl, src_lane);
      const float a00 = A[pk][pl], a01 = A[pk][ql], a10 = A[qk][pl], a11 = A[qk][ql];
      const float v0p = Q[k][pl], v0q = Q[k][ql], v1p = Q[k + 16][pl], v1q = Q[k + 16][ql];
      __syncthreads();                       // every read of the old matrix is done
      // columns (p_l, q_l) by J_l, then rows (p_k, q_k) by J_k^T
      const float b00 = cl * a00 - sl * a01, b01 = sl * a00 + cl * a01;
      const float b10 = cl * a10 - sl * a11, b11 = sl * a10 + cl * a11;
      A[pk][pl] = ck * b00 - sk * b10;
      A[pk][ql] = ck * b01 - sk * b11;
      A[qk][pl] = sk * b00 + ck * b10;
      A[qk][ql] = sk * b01 + ck * b11;
      Q[k][pl] = cl * v0p - sl * v0q;
      Q[k][ql] = sl * v0p + cl * v0q;
      Q[k + 16][pl] = cl * v1p - sl * v1q;
      Q[k + 16][ql] = sl * v1p + cl * v1q;
      __syncthreads();
    }
    // converged: every off-diagonal met in this sweep was below `tol` relative to its diagonal pair
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) seen = fmaxf(seen, __shfl_xor_sync(0xffffffffu, seen, o));
    if ((tid & 31) == 0) wmax[tid >> 5] = seen;
    __syncthreads();
    float all = wmax[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) all = fmaxf(all, wmax[w]);
    __syncthreads();
    if (all < tol) break;
  }
  if (tid < L) {
    const float w = A[tid][tid];
    int rank = 0;
    for (int j = 0; j < L; ++j) {
      const float wj = A[j][j];
      rank += (wj > w) || (wj == w && j < tid);
    }
    sigma[static_cast<size_t>(b) * L + rank] = sqrtf(fmaxf(w, 0.f));
    float* v = V + static_cast<size_t>(b) * L * L;
    for (int i = 0; i < L; ++i) v[i * L + rank] = Q[i][tid];
  }
}

// ------------------------------------------------------------------------------------ factors
// up[n, j]   = s_j * sum_i Q[n, i] Uh[i, j]                      (space 0, rows = N)   -> out[n*r + j]
// down[j, k] = (1/s_j) * sum_i Bt[k, i] Uh[i, j]  (0 if null)    (space 1, rows = K)   -> out[N*r + j*K + k]
__global__ void __launch_bounds__(THREADS)
factors_kernel(const MatDesc* __restrict__ mats, const TItem* __restrict__ items, int space,
               const float* __restrict__ buf, const float* __restrict__ V, const float* __restrict__ sig,
               int r, float* __restrict__ out) {
  __shared__ float Ms[L][17];
  const TItem it = items[blockIdx.x];
  const MatDesc m = mats[it.b];
  const int rows = space ? m.K : m.N;
  const float* base = buf + static_cast<size_t>(space ? m.zoff : m.yoff) * L;
  const float* v = V + static_cast<size_t>(it.b) * L * L;
  const float* s = sig + static_cast<size_t>(it.b) * L;
  const int tid = threadIdx.x;
  const float smax = s[0];
  for (int i = tid; i < L * 16; i += THREADS) {
    const int rr = i >> 4, c = i & 15;
    float val = 0.f;
    if (c < r) {
      const float sc = s[c];
      val = space ? ((sc > 1e-6f * smax && sc > 0.f) ? v[rr * L + c] / sc : 0.f) : v[rr * L + c] * sc;
    }
    Ms[rr][c] = val;
  }
  __syncthreads();
  const int row = it.row0 + tid;
  if (row >= rows) return;
  float x[L];
  const float4* src = reinterpret_cast<const float4*>(base + static_cast<size_t>(row) * L);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 a = src[i];
    x[4 * i] = a.x; x[4 * i + 1] = a.y; x[4 * i + 2] = a.z; x[4 * i + 3] = a.w;
  }
  float* o = out + m.out_off;
  for (int j = 0; j < r; ++j) {
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < L; ++i) acc += x[i] * Ms[i][j];
    if (space) o[static_cast<size_t>(m.N) * r + static_cast<size_t>(j) * m.K + row] = acc;
    else o[static_cast<size_t>(row) * r + j] = acc;
  }
}

// ------------------------------------------------------------------------------------ quantile clamp
// cli_svd.py:43-47: hi = torch.quantile(cat(U.flatten(), Vh.flatten()), q); clamp both to [-hi, hi].
// torch.quantile ("linear"): pos = q (n-1) evaluated in fp32, v = sorted[floor pos].lerp(sorted[ceil pos],
// frac). The two order statistics are found EXACTLY by a 4 x 8-bit radix select on the
// order-preserving integer image of the floats (one CTA per matrix, data is L2-resident).
__device__ __forceinline__ uint32_t fkey(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
__global__ void __launch_bounds__(1024)
quantile_clamp_kernel(const MatDesc* __restrict__ mats, int r, float q, float* __restrict__ out,
                      float* __restrict__ hi_out) {
  __shared__ unsigned int hist[256];
  __shared__ unsigned int sel_prefix, sel_rank, s_min_above, s_count_le;
  const MatDesc m = mats[blockIdx.x];
  float* x = out + m.out_off;
  const long long n = static_cast<long long>(r) * (static_cast<long long>(m.N) + m.K);
  const int tid = threadIdx.x;
  const float pos = q * static_cast<float>(n - 1);
  const long long k_lo = static_cast<long long>(floorf(pos));
  const long long k_hi = static_cast<long long>(ceilf(pos));
  const float w = pos - floorf(pos);
  // ---- k_lo-th smallest (0-based)
  uint32_t prefix = 0, mask = 0;
  unsigned int rank = static_cast<unsigned int>(k_lo);
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += 1024) hist[i] = 0;
    __syncthreads();
    for (long long i = tid; i < n; i += 1024) {
      const uint32_t key = fkey(x[i]);
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      unsigned int cum = 0, b = 0;
      for (; b < 256; ++b) {
        if (cum + hist[b] > rank) break;
        cum += hist[b];
      }
      sel_prefix = prefix | (static_cast<uint32_t>(b) << shift);
      sel_rank = rank - cum;
    }
    __syncthreads();
    prefix = sel_prefix;
    rank = sel_rank;
    mask |= 0xffu << shift;
    __syncthreads();
  }
  const float v_lo = fkey_inv(prefix);
  // ---- the next order statistic: equal to v_lo if it has duplicates past k_lo, else the
  // smallest element above it
  if (tid == 0) { s_min_above = 0xffffffffu; s_count_le = 0; }
  __syncthreads();
  unsigned int cnt = 0, mn = 0xffffffffu;
  for (long long i = tid; i < n; i += 1024) {
    const uint32_t key = fkey(x[i]);
    cnt += key <= prefix;
    if (key > prefix) mn = min(mn, key);
  }
  atomicAdd(&s_count_le, cnt);
  atomicMin(&s_min_above, mn);
  __syncthreads();
  float v_hi = v_lo;
  if (k_hi > k_lo && static_cast<long long>(s_count_le) <= k_hi && s_min_above != 0xffffffffu)
    v_hi = fkey_inv(s_min_above);
  // torch.lerp
  const float d = v_hi - v_lo;
  const float hi = (w < 0.5f) ? v_lo + w * d : v_hi - d * (1.f - w);
  if (tid == 0 && hi_out) hi_out[blockIdx.x] = hi;
  for (long long i = tid; i < n; i += 1024) x[i] = fminf(fmaxf(x[i], -hi), hi);
}

// ------------------------------------------------------------------------------------ host side
struct Plan {
  std::vector<MatDesc> mats;
  std::vector<RItem> ritems;
  std::vector<LItem> litems;
  std::vector<TItem> ty, tz;
  long long sumN = 0, sumK = 0, out_elems = 0;
};

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

static void make_plan(Plan& p, const void* const* Wt, const void* const* Wb, const int* N, const int* K,
                      int batch, int rank, int kt) {
  p.mats.resize(batch);
  for (int b = 0; b < batch; ++b) {
    MatDesc& m = p.mats[b];
    m.wt = Wt[b]; m.wb = Wb ? Wb[b] : nullptr; m.N = N[b]; m.K = K[b];
    m.yoff = p.sumN; m.zoff = p.sumK; m.out_off = p.out_elems;
    p.sumN += N[b]; p.sumK += K[b];
    p.out_elems += static_cast<long long>(rank) * (static_cast<long long>(N[b]) + K[b]);
    for (int r0 = 0; r0 < N[b]; r0 += TM) p.ritems.push_back({b, r0});
    // row slabs of <= 1024 rows: bounds the serial length of one CTA (per-SM ingest ~100 GB/s)
    const int slabs = (N[b] + 1023) / 1024;
    const int per = ((N[b] + slabs - 1) / slabs + TM - 1) / TM * TM;
    for (int k0 = 0; k0 < K[b]; k0 += kt)
      for (int n0 = 0; n0 < N[b]; n0 += per) p.litems.push_back({b, k0, n0, n0 + per < N[b] ? n0 + per : N[b]});
    for (int r0 = 0; r0 < N[b]; r0 += THREADS) p.ty.push_back({b, r0});
    for (int r0 = 0; r0 < K[b]; r0 += THREADS) p.tz.push_back({b, r0});
  }
}

struct Layout {
  size_t mats, ritems, litems, ty, tz, Y, Z, G, V, sig, total;
};
static Layout make_layout(const Plan& p, int batch) {
  Layout l;
  size_t o = 0;
  l.mats = o; o = align_up(o + p.mats.size() * sizeof(MatDesc), 256);
  l.ritems = o; o = align_up(o + p.ritems.size() * sizeof(RItem), 256);
  l.litems = o; o = align_up(o + p.litems.size() * sizeof(LItem), 256);
  l.ty = o; o = align_up(o + p.ty.size() * sizeof(TItem), 256);
  l.tz = o; o = align_up(o + p.tz.size() * sizeof(TItem), 256);
  l.Y = o; o = align_up(o + static_cast<size_t>(p.sumN) * L * 4, 256);
  l.Z = o; o = align_up(o + static_cast<size_t>(p.sumK) * L * 4, 256);
  l.G = o; o = align_up(o + static_cast<size_t>(batch) * L * L * 4, 256);
  l.V = o; o = align_up(o + static_cast<size_t>(batch) * L * L * 4, 256);
  l.sig = o; o = align_up(o + static_cast<size_t>(batch) * L * 4, 256);
  l.total = o;
  return l;
}

}  // namespace lbsvd2

using namespace lbsvd2;

static inline int kt_of(int w_dtype) { return w_dtype == LB_F32 ? 32 : 64; }

extern "C" long long lb_svd_workspace_bytes(const int* N, const int* K, int batch, int w_dtype) {
  if (batch <= 0 || N == nullptr || K == nullptr) return LB_ERR_SHAPE;
  Plan p;
  std::vector<const void*> dummy(batch, nullptr);
  make_plan(p, dummy.data(), nullptr, N, K, batch, 16, kt_of(w_dtype));
  return static_cast<long long>(make_layout(p, batch).total);
}

#define LB_SVD_CHECK() do { if (cudaGetLastError() != cudaSuccess) return LB_ERR_CUDA; } while (0)

extern "C" int lb_svd_truncated_batched(const void* const* Wt, const void* const* Wb, const int* N,
                                        const int* K, int batch, int w_dtype, int rank, int power_iters,
                                        float clamp_q, unsigned long long seed, float* out,
                                        float* sigma_out, float* hi_out, void* workspace,
                                        long long workspace_bytes, void* stream) {
  if (batch <= 0 || Wt == nullptr || N == nullptr || K == nullptr || out == nullptr || workspace == nullptr)
    return LB_ERR_SHAPE;
  if (rank < 1 || rank > 16) return LB_ERR_RANK;
  if (w_dtype != LB_F32 && w_dtype != LB_BF16 && w_dtype != LB_F16) return LB_ERR_DTYPE;
  if (power_iters < 0 || power_iters > 8) return LB_ERR_SHAPE;
  const int vec = w_dtype == LB_F32 ? 4 : 8;
  for (int b = 0; b < batch; ++b) {
    if (N[b] <= 0 || K[b] <= 0 || (K[b] % vec) != 0) return LB_ERR_SHAPE;   // 16-byte row pitch
    if ((reinterpret_cast<uintptr_t>(Wt[b]) | reinterpret_cast<uintptr_t>(Wb ? Wb[b] : nullptr)) & 15) return LB_ERR_ALIGN;
  }
  const int kt = kt_of(w_dtype);
  Plan p;
  make_plan(p, Wt, Wb, N, K, batch, rank, kt);
  const Layout lay = make_layout(p, batch);
  if (static_cast<long long>(lay.total) > workspace_bytes) return LB_ERR_SHAPE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  // tables: pageable host -> device (the runtime stages pageable sources before returning)
  if (cudaMemcpyAsync(ws + lay.mats, p.mats.data(), p.mats.size() * sizeof(MatDesc), cudaMemcpyHostToDevice, st) != cudaSuccess ||
      cudaMemcpyAsync(ws + lay.ritems, p.ritems.data(), p.ritems.size() * sizeof(RItem), cudaMemcpyHostToDevice, st) != cudaSuccess ||
      cudaMemcpyAsync(ws + lay.litems, p.litems.data(), p.litems.size() * sizeof(LItem), cudaMemcpyHostToDevice, st) != cudaSuccess ||
      cudaMemcpyAsync(ws + lay.ty, p.ty.data(), p.ty.size() * sizeof(TItem), cudaMemcpyHostToDevice, st) != cudaSuccess ||
      cudaMemcpyAsync(ws + lay.tz, p.tz.data(), p.tz.size() * sizeof(TItem), cudaMemcpyHostToDevice, st) != cudaSuccess)
    return LB_ERR_CUDA;
  const MatDesc* mats = reinterpret_cast<const MatDesc*>(ws + lay.mats);
  const RItem* ritems = reinterpret_cast<const RItem*>(ws + lay.ritems);
  const LItem* litems = reinterpret_cast<const LItem*>(ws + lay.litems);
  const TItem* ty = reinterpret_cast<const TItem*>(ws + lay.ty);
  const TItem* tz = reinterpret_cast<const TItem*>(ws + lay.tz);
  float* Y = reinterpret_cast<float*>(ws + lay.Y);
  float* Z = reinterpret_cast<float*>(ws + lay.Z);
  float* G = reinterpret_cast<float*>(ws + lay.G);
  float* V = reinterpret_cast<float*>(ws + lay.V);
  float* sig = sigma_out ? sigma_out : reinterpret_cast<float*>(ws + lay.sig);
  const size_t g_bytes = static_cast<size_t>(batch) * L * L * 4;
  const int nR = static_cast<int>(p.ritems.size()), nL = static_cast<int>(p.litems.size());
  const int nTy = static_cast<int>(p.ty.size()), nTz = static_cast<int>(p.tz.size());

  // dynamic shared memory: raw ring 64 KB + converted hi/lo tiles + the tall-skinny chunk (hi/lo)
  const int tile_bytes = TM * kt * 2;
  const int smem_r = 2 * RAW_STAGE_BYTES + 2 * tile_bytes + 2 * kt * 64;
  const int smem_l = 2 * RAW_STAGE_BYTES + 2 * tile_bytes + 2 * TM * 64;
  static unsigned long long attr_done = 0;      // bit per device ordinal
  {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return LB_ERR_CUDA;
    if (dev < 0 || dev >= 64 || !((attr_done >> dev) & 1ull)) {
      const int big_r = 2 * RAW_STAGE_BYTES + 2 * TM * 64 * 2 + 2 * 64 * 64;
      const int big_l = 2 * RAW_STAGE_BYTES + 2 * TM * 64 * 2 + 2 * TM * 64;
      bool ok = true;
      auto set_r = [&](auto kern) { ok = ok && cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, big_r) == cudaSuccess; };
      auto set_l = [&](auto kern) { ok = ok && cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, big_l) == cudaSuccess; };
      set_r(mul_right_kernel<__half, 1>); set_r(mul_right_kernel<__half, 2>); set_r(mul_right_kernel<__half, 3>);
      set_r(mul_right_kernel<__nv_bfloat16, 1>); set_r(mul_right_kernel<__nv_bfloat16, 2>); set_r(mul_right_kernel<__nv_bfloat16, 3>);
      set_r(mul_right_kernel<float, 1>); set_r(mul_right_kernel<float, 2>); set_r(mul_right_kernel<float, 3>);
      set_l(mul_left_kernel<__half, 1>); set_l(mul_left_kernel<__half, 2>); set_l(mul_left_kernel<__half, 3>);
      set_l(mul_left_kernel<__nv_bfloat16, 1>); set_l(mul_left_kernel<__nv_bfloat16, 2>); set_l(mul_left_kernel<__nv_bfloat16, 3>);
      set_l(mul_left_kernel<float, 1>); set_l(mul_left_kernel<float, 2>); set_l(mul_left_kernel<float, 3>);
      if (!ok)
        return LB_ERR_CUDA;
      if (dev >= 0 && dev < 64) attr_done |= 1ull << dev;
    }
  }
  // split terms per pass (see mul_right_kernel): pass 1 multiplies by +-1 probes (exact in bf16), the
  // power-iteration passes only shape a basis that is re-orthonormalised anyway and whose columns stay
  // in range(dW) / range(dW^T) because dW itself keeps both halves; the LAST pass (B^T = dW^T Q, which
  // the factors are read from) is fp32-faithful. LB_SVD_TERMS=3333 restores three terms everywhere.
  static int terms_cfg[4] = {0, 0, 0, 0};
  if (terms_cfg[0] == 0) {
    const char* e = getenv("LB_SVD_TERMS");
    const char* d = (e && e[0] && e[1] && e[2] && e[3]) ? e : "2223";
    int tmp[4];
    for (int i = 0; i < 4; ++i) tmp[i] = (d[i] >= '1' && d[i] <= '3') ? d[i] - '0' : 3;
    tmp[3] = 3;
    for (int i = 3; i >= 0; --i) terms_cfg[i] = tmp[i];
  }
  auto mul_right = [&](bool gram, int terms) -> bool {
    if (gram && cudaMemsetAsync(G, 0, g_bytes, st) != cudaSuccess) return false;
    float* g = gram ? G : nullptr;
#define LB_MR(WT_)                                                                                         \
    do {                                                                                                   \
      if (terms == 1) mul_right_kernel<WT_, 1><<<nR, THREADS, smem_r, st>>>(mats, ritems, Z, Y, g);        \
      else if (terms == 2) mul_right_kernel<WT_, 2><<<nR, THREADS, smem_r, st>>>(mats, ritems, Z, Y, g);   \
      else mul_right_kernel<WT_, 3><<<nR, THREADS, smem_r, st>>>(mats, ritems, Z, Y, g);                   \
    } while (0)
    if (w_dtype == LB_F16) LB_MR(__half);
    else if (w_dtype == LB_BF16) LB_MR(__nv_bfloat16);
    else LB_MR(float);
#undef LB_MR
    return cudaGetLastError() == cudaSuccess;
  };
  auto mul_left = [&](int terms) -> bool {
    if (cudaMemsetAsync(Z, 0, static_cast<size_t>(p.sumK) * L * 4, st) != cudaSuccess) return false;
#define LB_ML(WT_)                                                                                     \
    do {                                                                                               \
      if (terms == 1) mul_left_kernel<WT_, 1><<<nL, THREADS, smem_l, st>>>(mats, litems, Y, Z);        \
      else if (terms == 2) mul_left_kernel<WT_, 2><<<nL, THREADS, smem_l, st>>>(mats, litems, Y, Z);   \
      else mul_left_kernel<WT_, 3><<<nL, THREADS, smem_l, st>>>(mats, litems, Y, Z);                   \
    } while (0)
    if (w_dtype == LB_F16) LB_ML(__half);
    else if (w_dtype == LB_BF16) LB_ML(__nv_bfloat16);
    else LB_ML(float);
#undef LB_ML
    return cudaGetLastError() == cudaSuccess;
  };
  // orth(buf): [Gram given in G] -> Jacobi -> buf <- buf V diag(1/s) (+ Gram of the result)
  // at most `sweeps` cyclic sweeps; stops after the first sweep whose rotations were all below `tol`
  // (relative off-diagonal): 1e-4 is plenty for an intermediate basis, 1e-7 (fp32) for the last two
  auto jacobi = [&](int sweeps, float tol) -> bool {
    jacobi32_kernel<<<batch, 256, 0, st>>>(G, V, sig, sweeps, tol);
    return cudaGetLastError() == cudaSuccess;
  };
  auto transform = [&](int space, bool mul, bool gram) -> bool {
    if (gram && cudaMemsetAsync(G, 0, g_bytes, st) != cudaSuccess) return false;
    tall_transform_kernel<<<space ? nTz : nTy, THREADS, 0, st>>>(mats, space ? tz : ty, space, space ? Z : Y, V, sig,
                                                               mul ? 1 : 0, gram ? G : nullptr);
    return cudaGetLastError() == cudaSuccess;
  };

  probes_kernel<<<static_cast<int>((p.sumK + 255) / 256), 256, 0, st>>>(Z, p.sumK, seed);
  LB_SVD_CHECK();
  if (!mul_right(true, terms_cfg[0])) return LB_ERR_CUDA;         // Y = dW Om, G = Y^T Y
  for (int it = 0; it < power_iters; ++it) {
    if (!jacobi(6, 1e-4f) || !transform(0, true, false)) return LB_ERR_CUDA;    // Y <- orth(Y)
    if (!mul_left(terms_cfg[1])) return LB_ERR_CUDA;                       // Z = dW^T Y
    if (!transform(1, false, true) || !jacobi(6, 1e-4f) || !transform(1, true, false)) return LB_ERR_CUDA;   // Z <- orth(Z)
    if (!mul_right(true, terms_cfg[2])) return LB_ERR_CUDA;                // Y = dW Z, G
  }
  // Q = orth2(Y): the basis the projected problem is solved in must be orthonormal to fp32 accuracy
  if (!jacobi(6, 1e-4f) || !transform(0, true, true) || !jacobi(8, 1e-7f) || !transform(0, true, false)) return LB_ERR_CUDA;
  if (!mul_left(3)) return LB_ERR_CUDA;                                    // B^T = dW^T Q (fp32-faithful)
  if (!transform(1, false, true) || !jacobi(10, 1e-7f)) return LB_ERR_CUDA;       // B B^T = Uh diag(s^2) Uh^T
  factors_kernel<<<nTy, THREADS, 0, st>>>(mats, ty, 0, Y, V, sig, rank, out);
  LB_SVD_CHECK();
  factors_kernel<<<nTz, THREADS, 0, st>>>(mats, tz, 1, Z, V, sig, rank, out);
  LB_SVD_CHECK();
  if (clamp_q > 0.f) {
    quantile_clamp_kernel<<<batch, 1024, 0, st>>>(mats, rank, clamp_q, out, hi_out);
    LB_SVD_CHECK();
  }
  return LB_OK;
}
