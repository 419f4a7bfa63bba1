// Fused frozen-weight GEMM / implicit-GEMM conv + rank-r LoRA for sm_90a (wgmma + TMA + mbarrier).
//
//   Y[M,N] = X[M,K] . W[N,K]^T (+ bias) + sum_g ((X_g . D^T) * (scale * diag)) . U_g^T
//
// LINEAR  (CONV = false):  X is a row-major [M,K] matrix, one T group (G = 1).
// CONV    (CONV = true):   X is an NHWC activation; a CTA owns a TH x TW pixel rectangle
//                          (TH*TW = 128 rows) and walks K = (filter tap, 64-channel block); each
//                          tap is the same rectangle shifted by (dy - pad, dx - pad), fetched by a
//                          4-D TMA box whose out-of-image part is zero-filled by the hardware
//                          (that IS the padding). Stride 1, dilation 1, groups 1.
//
// The LoRA down factor D ([RP, K] 16-bit, rank zero-padded to RP = 16, 32 or 64) rides the main K
// loop: its RP rows are appended below every W tile in shared memory, so the tensor core produces
// T = X.D^T alongside the base accumulator from the same X tile -- X is read from HBM exactly once.
//   G == 1: one wgmma per K-step with N = BLOCK_N + RP; T is accumulator columns [BLOCK_N, +RP).
//                                                         (linear fwd / dX, conv fwd, 1x1 conv dX)
//   G  > 1: the conv input-gradient. dX needs a separate T_t = gY(shifted by tap t) . B per tap,
//           so each K-step issues N = BLOCK_N into the base accumulator and N = 16 into the tap's
//           own accumulator (RP = 16). At RP > 16 the taps' T come from t_in instead (TAPLOOP in
//           Smem): the K loop issues N = BLOCK_N only, and the epilogue adds T'_t . U_t^T tap by tap.
// The up-projection is a K = RP wgmma chain (RP / 16 K-steps per T group) over an interleaved
// core-matrix layout of T' and U.
//
// Roles: warps 0-7 are two consumer warpgroups -- warpgroup w owns accumulator rows [64 w, 64 w + 64)
// and issues wgmma.m64nNk16 on the shared-memory stages, the accumulators live in its registers;
// warp 8 is the TMA producer. After the K loop the warpgroups park their accumulators in shared
// memory (ACC, which aliases the drained stage ring), and warpgroup 0 works row-per-thread: it
// scales the T group(s), writes them back as 16-bit K-major operands, and both warpgroups
// accumulate acc += T'_g . U_g^T (K = 16 each) into their registers. Bias is added in the drain and
// the tile leaves through a swizzled staging buffer and TMA stores.
//
// Cluster split-K (CL > 1, linear G == 1 only): the CL CTAs of a (1, 1, CL) cluster share one output
// tile, CTA `rank` reducing K blocks [rank * nkb / CL, (rank + 1) * nkb / CL). Each peer pushes its
// parked accumulator (base AND T columns -- both are linear in K) into the leader's slot rank - 1 with
// ONE cp.async.bulk over distributed shared memory (completion = complete_tx on the leader's
// mbarrier); the leader adds the slots to its own before the epilogue. Lifetimes: the leader waits for
// every copy; a peer leaves only after the closing cluster barrier, which the leader's threads arrive
// at once the copies have landed (so the source buffers have been read).
#pragma once
#include "dropmask.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace lb {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 x 16-bit = 128 B = one SWIZZLE_128B row
constexpr int R_PAD = 16;    // LoRA rank padded to one MMA K-step
constexpr int MMA_K = 16;
constexpr int CONSUMER_THREADS = 256;                // two warpgroups of 64 accumulator rows each
constexpr int NUM_THREADS = CONSUMER_THREADS + 32;   // + the TMA producer warp
// INLINE_TMA kernels have no producer warp: consumer thread 0 issues the loads (a stage is refilled
// as soon as both warpgroups have released it). 256 threads let two 128-wide CTAs share an SM's
// registers (a 288-thread CTA is allocated as 10 warps), so one CTA's epilogue overlaps the other's
// loads and MMAs -- the Hopper form of the epilogue overlap for sites with many tiles.
template <bool INLINE_TMA>
constexpr int kernel_threads() { return INLINE_TMA ? CONSUMER_THREADS : NUM_THREADS; }
constexpr int EPI_THREADS = 128;                     // row-per-thread epilogue: warpgroup 0
constexpr int BAR_CONSUMERS = 1, BAR_EPI = 2;        // named barriers (0 is __syncthreads)

struct FusedParams {
  const float* bias;   // [N] or null
  const float* up;     // fp32 LoRA-up factor: element (n, g, j) at up[n*up_rs + j*up_cs + g*up_gs]
  long long up_rs, up_cs, up_gs;
  const float* diag;   // [r] or null (selector diagonal)
  float* t_out;        // [M,RP] fp32 side output (group t_group, unscaled), n_blk == 0 CTAs; or null
  const float* t_in;   // [M,RP] fp32 or null: when set, the rank-r activations are TAKEN from here
                       // (row = this row / the tap-shifted pixel) instead of from the accumulator. Used
                       // by the dropout path, where T = (mask o gY).B cannot share the base operand.
  float scale;
  int M, N, K, r;      // K = total reduction length (conv: taps * C)
  int fmt;             // 1 = bf16 operands, 0 = fp16
  int t_group;         // which T group goes to t_out
  // conv geometry
  int H, W, C;         // image height/width, input channels
  int kh, kw, pad_h, pad_w;
  int TH, TW, tiles_h, tiles_w;
  int down_per_tap;    // 1: D columns advance with the tap (forward); 0: D restarts every tap (dX)
  // dropout on the LoRA branch (DROP kernels only): keep(m, n) from dropmask.cuh on element index
  // row * N + n, survivors scaled by drop_inv = 1/(1-p); seed lives in device memory (graph-safe)
  float drop_p, drop_inv;
  const unsigned long long* seed;
  // split-K (SPLITK kernels only): gridDim.z = split CTAs share one output tile, each reducing a
  // contiguous range of K blocks. Every CTA adds its partial accumulator (base + T columns) into the
  // tile's [128][BLOCK_N + 16 G] fp32 buffer in `ws` with vector reductions at L2; `counters[tile]`
  // elects the last CTA to arrive, which reads the reduced row back in one burst, wipes it and runs
  // the ordinary epilogue. Buffer and counters must be zero on entry; the elected CTA leaves them so.
  int w_tiled;         // 1: the frozen weight is stored as 64 x 64 blocks, block (n64, kb) = rows
                       // [(n64 * num_kb + kb) * 64, +64) of a [rows, 64] tensor (lb_tile_weight): every TMA box
                       // is ONE contiguous 8 KB run of HBM instead of 64 rows a whole K apart
  int split;
  float* ws;
  unsigned int* counters;
  unsigned long long* dbg;  // profiling only: 16 x %globaltimer stamps written by CTA (0,0), or null
};

// B-operand tile of the frozen weight: rows [n0, n0 + BLOCK_N) x K block kb (global index, conv: tap-major).
template <int BLOCK_N>
__device__ __forceinline__ void load_w_tile(const CUtensorMap* tmW, uint32_t bar, uint32_t dst, int k_elem, int kb,
                                            int num_kb, int n0, int w_tiled) {
  if (w_tiled) {
#pragma unroll
    for (int j = 0; j < BLOCK_N / 64; ++j)
      tma_load_2d(tmW, bar, dst + j * (64 * 128), 0, (((n0 >> 6) + j) * num_kb + kb) * 64);
  } else {
    tma_load_2d(tmW, bar, dst, k_elem, n0);
  }
}

__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
#define LB_STAMP(i) do { if (p.dbg != nullptr && blockIdx.x == 0 && blockIdx.y == 0) p.dbg[i] = gtimer(); } while (0)

template <int BLOCK_N, int STAGES, typename OutT, int G, bool DROP = false, int CL = 1, int RP = R_PAD>
struct Smem {
  // TAPLOOP: conv input-gradient (G taps) at RP > 16. Per-tap T accumulators would not fit, so T is
  // taken from t_in and the epilogue runs the taps one after another through ONE T'/U buffer pair;
  // the main loop carries no D rows and no T columns.
  static constexpr bool TAPLOOP = G > 1 && RP > R_PAD;
  static constexpr int DROWS = TAPLOOP ? 0 : RP;        // D rows below each W tile
  static constexpr int TCOLS = TAPLOOP ? 0 : RP * G;    // T columns of the parked accumulator
  static constexpr int TG = TAPLOOP ? 1 : G;            // T'/U groups staged at once
  static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
  static constexpr int B_BYTES = (BLOCK_N + DROWS) * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;   // one TMA transaction: X tile, W tile + D rows
  // fp32 accumulator parked after the K loop: base columns, T group(s), and (DROP) the LoRA product,
  // which the mask separates from the sum. Row pitch padded by 8 floats against bank conflicts.
  static constexpr int L_COL0 = BLOCK_N + TCOLS;
  static constexpr int ACC_COLS = BLOCK_N + TCOLS + (DROP ? BLOCK_N : 0);
  static constexpr int ACC_LD = ACC_COLS + 8;
  static constexpr int ACC_BYTES = BLOCK_M * ACC_LD * 4;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  static constexpr int BOX_COLS = 128 / sizeof(OutT);  // columns per 128-byte store box
  static constexpr int NUM_BOXES = BLOCK_N / BOX_COLS;
  static constexpr int BOX_BYTES = BLOCK_M * 128;
  static constexpr int T_BYTES = BLOCK_M * RP * TG * 2;   // T' operand(s)
  static constexpr int UP_BYTES = BLOCK_N * RP * TG * 2;  // U tile(s)
  // the accumulator is parked only after the last stage has been consumed: it aliases the ring
  static constexpr int OFF_ACC = 0;
  static constexpr int OFF_EPI = (((RING_BYTES > ACC_BYTES ? RING_BYTES : ACC_BYTES) + 1023) / 1024) * 1024;
  // output staging is written only after the LoRA MMAs have consumed T'/U: the regions alias
  static constexpr int OFF_OUT = OFF_EPI;
  static constexpr int OFF_T = OFF_EPI;
  static constexpr int OFF_UP = OFF_T + T_BYTES;
  static constexpr int EPI_BYTES =
      (NUM_BOXES * BOX_BYTES > T_BYTES + UP_BYTES) ? NUM_BOXES * BOX_BYTES : T_BYTES + UP_BYTES;
  // cluster split-K, leader: one parked accumulator per peer (never aliased: peers push at any time)
  static constexpr int OFF_SLOTS = OFF_EPI + ((EPI_BYTES + 1023) / 1024) * 1024;
  static constexpr int OFF_BIAS = OFF_SLOTS + (CL - 1) * ACC_BYTES;
  static constexpr int OFF_BAR = OFF_BIAS + BLOCK_N * 4;
  static constexpr int NUM_BARS = 2 * STAGES + 1;     // full[], empty[], peers' partials landed
  static constexpr int OFF_FLAG = OFF_BAR + NUM_BARS * 8;   // split-K election result
  static constexpr int TOTAL = OFF_FLAG + 16;
  static constexpr int DYN_BYTES = TOTAL + 1024;  // slack for manual 1024-B alignment
  static_assert(DYN_BYTES <= 232448, "shared memory budget exceeded");
};

// Park a warpgroup's m64nNC accumulator fragment in the ACC rows it owns, columns [col0, col0 + NC)
// (ADD: added to what is parked there).
template <int NC, int LD, bool ADD = false>
__device__ __forceinline__ void park_acc(float* acc_s, const float* d, int wg_row0, int col0) {
  const int t = threadIdx.x & 127;
  const int r = wg_row0 + 16 * (t >> 5) + ((t & 31) >> 2);
  const int c = col0 + 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < NC / 8; ++j) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float2* q = reinterpret_cast<float2*>(acc_s + (r + 8 * i) * LD + c + 8 * j);
      float2 v = make_float2(d[4 * j + 2 * i], d[4 * j + 2 * i + 1]);
      if constexpr (ADD) { const float2 o = *q; v.x += o.x; v.y += o.y; }
      *q = v;
    }
  }
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// relaxed: nothing is published through the cluster barrier itself (barrier initialisation is
// released by fence.mbarrier_init, the partials travel by bulk copy + mbarrier)
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait_acquire() { asm volatile("barrier.cluster.wait.acquire;" ::: "memory"); }
// shared::cta address of THIS CTA -> shared::cluster address of the same offset in CTA `rank`
__device__ __forceinline__ uint32_t mapa_u32(uint32_t local_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(rank));
  return r;
}
// bulk copy own shared memory -> a peer CTA's shared memory; completes on the PEER's mbarrier
__device__ __forceinline__ void dsmem_bulk_copy(uint32_t dst_cluster, uint32_t src_cta, uint32_t bytes,
                                                uint32_t bar_cluster) {
  asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst_cluster), "r"(src_cta), "r"(bytes), "r"(bar_cluster) : "memory");
}
// 16 consecutive fp32 of a parked accumulator row
__device__ __forceinline__ void ld_acc16(const float* src, float* v) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 q = reinterpret_cast<const float4*>(src)[i];
    v[4 * i] = q.x; v[4 * i + 1] = q.y; v[4 * i + 2] = q.z; v[4 * i + 3] = q.w;
  }
}

// One output tile (n_blk, m_blk) of one problem; called by the single-problem and the grouped kernel.
template <int BLOCK_N, int STAGES, typename OutT, bool CONV, int G, bool DROP = false, bool SPLITK = false,
          int CL = 1, bool INLINE_TMA = false, int RP = R_PAD>
__device__ __forceinline__ void fused_tile(const CUtensorMap& tmX, const CUtensorMap& tmW,
                                           const CUtensorMap& tmD, const CUtensorMap& tmY,
                                           const FusedParams& p, const int n_blk, const int m_blk) {
  using S = Smem<BLOCK_N, STAGES, OutT, G, DROP, CL, RP>;
  static_assert(CL == 1 || (!CONV && G == 1 && !DROP && !SPLITK), "cluster split-K: plain linear tiles");
  static_assert(!INLINE_TMA || (!CONV && G == 1 && !DROP && !SPLITK && CL == 1), "inline TMA: plain linear tiles");
  // wider ranks run the one-tile-per-CTA schedules only (a scope choice, not a measured one)
  static_assert(RP == R_PAD || ((RP == 32 || RP == 64) && !SPLITK && CL == 1 && !INLINE_TMA), "rank pad");
  static_assert(!S::TAPLOOP || (CONV && !DROP), "tap loop: conv input-gradient");
  constexpr bool TAPLOOP = S::TAPLOOP;
  constexpr int GQ = RP / 16;                         // 16-wide K-steps per T group
  constexpr int KG = S::TG * GQ;                      // 16-wide K-steps of the staged up-projection
  constexpr int PCOLS = BLOCK_N + S::TCOLS;           // columns of one partial accumulator
  constexpr bool WIDE = G == 1;                       // T rides the base MMA as RP extra columns
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* sgen = smem_raw + (sbase - smem_u32(smem_raw));  // generic pointer to the aligned base
  float* acc_s = reinterpret_cast<float*>(sgen + S::OFF_ACC);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) LB_STAMP(0);   // kernel entry
  const int n0 = n_blk * BLOCK_N;
  // row-tile origin
  int m0 = m_blk * BLOCK_M;   // LINEAR: first row
  int img = 0, h0 = 0, w0 = 0;  // CONV: image index and rectangle origin
  if constexpr (CONV) {
    const int per_img = p.tiles_h * p.tiles_w;
    img = m_blk / per_img;
    const int rem = m_blk - img * per_img;
    h0 = (rem / p.tiles_w) * p.TH;
    w0 = (rem % p.tiles_w) * p.TW;
  }
  const int taps = CONV ? p.kh * p.kw : 1;
  const int cblocks = CONV ? (p.C + BLOCK_K - 1) / BLOCK_K : (p.K + BLOCK_K - 1) / BLOCK_K;
  const int num_kb = taps * cblocks;
  // this CTA's share of the K loop (split-K: blockIdx.z of gridDim.z; launcher keeps split <= num_kb)
  // (cluster split-K: this CTA's rank of CL; the launcher keeps CL <= num_kb)
  const int part = SPLITK ? static_cast<int>(blockIdx.z) : (CL > 1 ? static_cast<int>(cluster_ctarank()) : 0);
  const int parts = SPLITK ? p.split : CL;
  const int kb_begin = static_cast<int>((static_cast<long long>(part) * num_kb) / parts);
  const int kb_end = static_cast<int>((static_cast<long long>(part + 1) * num_kb) / parts);
  const bool leader = part == 0;
  const uint32_t bar_red = sbase + S::OFF_BAR + 8 * (2 * STAGES);   // cluster: peers' partials landed
  auto finish = [&]() { if constexpr (CL > 1) cluster_wait_acquire(); };

  auto bar_full = [&](int s) { return sbase + S::OFF_BAR + 8 * s; };
  auto bar_empty = [&](int s) { return sbase + S::OFF_BAR + 8 * (STAGES + s); };

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmD);
    tma_prefetch_desc(&tmY);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(bar_full(s), 1);
      mbar_init(bar_empty(s), CONSUMER_THREADS);
    }
    mbar_init(bar_red, 1);
    fence_mbar_init();
    if (CL > 1 && leader) mbar_expect_tx(bar_red, (CL - 1) * S::ACC_BYTES);   // the one arrival + all peer bytes
  }
  __syncthreads();  // barriers initialised
  if constexpr (CL > 1) {   // cluster-wide: every CTA's barriers exist before any peer signals them
    cluster_arrive_relaxed();
    cluster_wait_acquire();
  }
  pdl_launch_dependents();   // the next kernel in the stream may start its own prologue now
  pdl_wait();                // predecessor grid complete, its writes visible: global reads may start

  // K block kb -> its ring stage (after that stage's previous use has been released)
  auto load_stage = [&](const int kb) {
    const int it = kb - kb_begin;
    const int s = it % STAGES;
    mbar_wait(bar_empty(s), ((it / STAGES) & 1) ^ 1);
    mbar_expect_tx(bar_full(s), S::STAGE_BYTES);
    const uint32_t sa = sbase + s * S::STAGE_BYTES;
    const uint32_t sb = sa + S::A_BYTES;
    if constexpr (CONV) {
      const int tap = kb / cblocks, cb = kb - tap * cblocks;
      const int dy = tap / p.kw, dx = tap - dy * p.kw;
      tma_load_4d(&tmX, bar_full(s), sa, cb * BLOCK_K, w0 + dx - p.pad_w, h0 + dy - p.pad_h, img);
      load_w_tile<BLOCK_N>(&tmW, bar_full(s), sb, tap * p.C + cb * BLOCK_K, kb, num_kb, n0, p.w_tiled);
      if constexpr (!TAPLOOP)
        tma_load_2d(&tmD, bar_full(s), sb + BLOCK_N * 128,
                    (p.down_per_tap ? tap * p.C : 0) + cb * BLOCK_K, 0);
    } else {
      tma_load_2d(&tmX, bar_full(s), sa, kb * BLOCK_K, m0);
      load_w_tile<BLOCK_N>(&tmW, bar_full(s), sb, kb * BLOCK_K, kb, num_kb, n0, p.w_tiled);
      tma_load_2d(&tmD, bar_full(s), sb + BLOCK_N * 128, kb * BLOCK_K, 0);
    }
  };
  if (INLINE_TMA && threadIdx.x == 0)   // fill the ring
    for (int kb = kb_begin; kb < kb_end && kb < kb_begin + STAGES; ++kb) load_stage(kb);

  if (!INLINE_TMA && warp == CONSUMER_THREADS / 32) {
    // ------------------------------------------------------------ TMA producer
    if (lane == 0) {
      LB_STAMP(1);                       // first TMA about to be issued
      for (int kb = kb_begin; kb < kb_end; ++kb) load_stage(kb);
    }
    if constexpr (CL > 1) {
      __syncwarp();
      cluster_arrive_relaxed();        // this warp has no distributed-shared-memory business
    }
    finish();
    return;
  }

  // ------------------------------------------------------------ consumer warpgroups
  const int ct = threadIdx.x;          // 0..255
  const int wg = ct >> 7;              // accumulator rows [64 wg, 64 wg + 64)
  float* bias_s = reinterpret_cast<float*>(sgen + S::OFF_BIAS);

  // Stage the U tile(s) (fp32 master -> 16-bit, interleaved core-matrix layout: 16-wide K-step kk of
  // row i at (i >> 3) * 256 KG + kk * 256 + (i & 7) * 16) and the bias; the TMA producer is already
  // streaming the first stages. TAPLOOP stages each tap's U in the epilogue instead.
  for (int i = ct; i < BLOCK_N; i += CONSUMER_THREADS) {
    const int n = n0 + i;
    const bool ok = n < p.N;
#pragma unroll
    for (int g = 0; g < S::TG * !TAPLOOP; ++g)
#pragma unroll
    for (int q = 0; q < GQ; ++q) {
      float u[16];
#pragma unroll
      for (int j = 0; j < 16; ++j)
        u[j] = (ok && 16 * q + j < p.r) ? __ldg(p.up + n * p.up_rs + (16 * q + j) * p.up_cs + g * p.up_gs) : 0.f;
      const uint32_t dst = sbase + S::OFF_UP + (i >> 3) * (256 * KG) + (g * GQ + q) * 256 + (i & 7) * 16;
      st_shared_v4(dst, pack2(u[0], u[1], p.fmt), pack2(u[2], u[3], p.fmt),
                   pack2(u[4], u[5], p.fmt), pack2(u[6], u[7], p.fmt));
      st_shared_v4(dst + 128, pack2(u[8], u[9], p.fmt), pack2(u[10], u[11], p.fmt),
                   pack2(u[12], u[13], p.fmt), pack2(u[14], u[15], p.fmt));
    }
    bias_s[i] = (p.bias != nullptr && ok) ? __ldg(p.bias + n) : 0.f;
  }

  // register accumulators (zero-initialised: every wgmma accumulates)
  constexpr int AREG = (WIDE ? PCOLS : BLOCK_N) / 2;
  constexpr int TG = (WIDE || TAPLOOP) ? 1 : G;   // separate T accumulators (unused when WIDE / TAPLOOP)
  float acc[AREG];
  float tacc[TG][R_PAD / 2];
#pragma unroll
  for (int i = 0; i < AREG; ++i) acc[i] = 0.f;
#pragma unroll
  for (int g = 0; g < TG; ++g)
#pragma unroll
    for (int i = 0; i < R_PAD / 2; ++i) tacc[g][i] = 0.f;

  // one K block; `tdst` = the T accumulator of the block's tap (unused when WIDE). The caller picks
  // it with a compile-time index: a wgmma under a data-dependent branch would be serialized.
  auto k_block = [&](const int kb, float* tdst) {
    const int it = kb - kb_begin;
    const int s = it % STAGES;
    const uint32_t ph = (it / STAGES) & 1;
    mbar_wait(bar_full(s), ph);
    if (it == 0 && ct == 0) LB_STAMP(2);          // first stage landed
    const uint32_t sa = sbase + s * S::STAGE_BYTES;
    const uint32_t sb = sa + S::A_BYTES;
    reg_fence<AREG>(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
      // K-major SWIZZLE_128B: 8-row groups 1024 B apart; one K-step = 32 B along the row
      const uint64_t ad = wgmma_desc(sa + wg * (64 * 128) + k * MMA_K * 2, 16, 1024, 1);
      const uint64_t bd = wgmma_desc(sb + k * MMA_K * 2, 16, 1024, 1);
      if constexpr (WIDE) {
        wgmma_ss<BLOCK_N + RP>(acc, ad, bd, p.fmt);
      } else if constexpr (TAPLOOP) {
        wgmma_ss<BLOCK_N>(acc, ad, bd, p.fmt);
      } else {
        const uint64_t dd = wgmma_desc(sb + BLOCK_N * 128 + k * MMA_K * 2, 16, 1024, 1);
        wgmma_ss<BLOCK_N>(acc, ad, bd, p.fmt);
        wgmma_ss<R_PAD>(tdst, ad, dd, p.fmt);
      }
    }
    wgmma_commit();
    // keep this stage's MMAs in flight; the previous stage's have retired: release its slot
    wgmma_wait<1>();
    reg_fence<AREG>(acc);
    if (it > 0) mbar_arrive(bar_empty((it - 1) % STAGES));
    // inline TMA: the stage just released takes K block kb - 1 + STAGES
    if (INLINE_TMA && ct == 0 && it > 0 && kb - 1 + STAGES < kb_end) load_stage(kb - 1 + STAGES);
  };
  if constexpr (WIDE || TAPLOOP) {
    for (int kb = kb_begin; kb < kb_end; ++kb) k_block(kb, nullptr);
  } else {
#pragma unroll
    for (int g = 0; g < TG; ++g) {   // tap g's K blocks within this CTA's range
      const int b0 = g * cblocks > kb_begin ? g * cblocks : kb_begin;
      const int b1 = (g + 1) * cblocks < kb_end ? (g + 1) * cblocks : kb_end;
      for (int kb = b0; kb < b1; ++kb) k_block(kb, tacc[g]);
    }
  }
  wgmma_wait<0>();
  reg_fence<AREG>(acc);
#pragma unroll
  for (int g = 0; g < TG; ++g) reg_fence<R_PAD / 2>(tacc[g]);
  if (ct == 0) LB_STAMP(3);            // main-loop MMAs completed
  // the ring is drained (every stage consumed, no loads outstanding) once BOTH warpgroups' MMAs have
  // retired: park the accumulator over it
  named_bar_sync(BAR_CONSUMERS, CONSUMER_THREADS);
  park_acc<WIDE ? PCOLS : BLOCK_N, S::ACC_LD>(acc_s, acc, wg * 64, 0);
  if constexpr (!WIDE && !TAPLOOP) {
#pragma unroll
    for (int g = 0; g < TG; ++g) park_acc<R_PAD, S::ACC_LD>(acc_s, tacc[g], wg * 64, BLOCK_N + R_PAD * g);
  }
  if constexpr (CL > 1) fence_proxy_async_smem();   // peers: the parked partial is read by a bulk copy
  named_bar_sync(BAR_CONSUMERS, CONSUMER_THREADS);
  if (ct == 0) LB_STAMP(4);            // accumulator parked
  if constexpr (CL > 1) {
    if (!leader) {   // partial -> the leader's slot (part - 1), then wait for the leader to read it
      if (ct == 0)
        dsmem_bulk_copy(mapa_u32(sbase + S::OFF_SLOTS + (part - 1) * S::ACC_BYTES, 0), sbase + S::OFF_ACC,
                        S::ACC_BYTES, mapa_u32(bar_red, 0));
      __syncwarp();
      cluster_arrive_relaxed();
      finish();
      return;
    }
    mbar_wait(bar_red, 0);             // every peer's partial is in its slot
    __syncwarp();
    cluster_arrive_relaxed();          // peers may retire: their buffers have been read
    const float4* slots = reinterpret_cast<const float4*>(sgen + S::OFF_SLOTS);
    float4* own = reinterpret_cast<float4*>(acc_s);
    for (int i = ct; i < S::ACC_BYTES / 16; i += CONSUMER_THREADS) {
      float4 v = own[i];
#pragma unroll
      for (int q = 0; q < CL - 1; ++q) {
        const float4 o = slots[q * (S::ACC_BYTES / 16) + i];
        v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w;
      }
      own[i] = v;
    }
    named_bar_sync(BAR_CONSUMERS, CONSUMER_THREADS);
  }

  volatile uint32_t* flag = reinterpret_cast<volatile uint32_t*>(sgen + S::OFF_FLAG);
  // split-K, G == 1: the whole reduced row (base + T columns) in registers after ONE burst of L2
  // reads; G > 1 (conv dX): T groups first, base columns chunk by chunk in the drain
  constexpr int ROW_REGS = (SPLITK && G == 1) ? PCOLS : 1;
  float rowv[ROW_REGS];
  float* acc_row = nullptr;     // split-K: this thread's row of the tile's fp32 accumulation buffer
  const int row = ct;           // epilogue row (warpgroup 0 only)
  const float* arow = acc_s + row * S::ACC_LD;
  long long grow = -1;          // global row (pixel) this thread owns, for the T side output
  if (ct < EPI_THREADS) {
    // ------------------------------------------------------------ epilogue part 1 (row per thread)
    // T is scaled 16 columns at a time: t[RP] and coef[RP] at once would not fit beside the accumulator
    float coef[16];
    auto load_coef = [&](const int j0) {
#pragma unroll
      for (int j = 0; j < 16; ++j)
        coef[j] = (j0 + j < p.r) ? p.scale * (p.diag ? __ldg(p.diag + j0 + j) : 1.f) : 0.f;
    };
    if constexpr (RP == R_PAD) load_coef(0);
    if constexpr (CONV) {
      const int hh = h0 + row / p.TW, ww = w0 + row % p.TW;
      if (hh < p.H && ww < p.W) grow = (static_cast<long long>(img) * p.H + hh) * p.W + ww;
    } else {
      if (m0 + row < p.M) grow = m0 + row;
    }
    auto tap_touched = [&](int g) {   // did this CTA's K range feed tap g's T columns?
      return !SPLITK || G == 1 || (kb_begin < (g + 1) * cblocks && kb_end > g * cblocks);
    };
    bool elected = true;          // split-K: is this the CTA that finishes the tile?
    if constexpr (SPLITK) {
      const unsigned tile_id = blockIdx.y * gridDim.x + blockIdx.x;
      acc_row = p.ws + (static_cast<size_t>(tile_id) * BLOCK_M + row) * PCOLS;
      // every CTA adds its partial into the tile's accumulation buffer (vector fp32 reductions at
      // L2, fire-and-forget); T columns of taps this CTA never fed are skipped
      if (CONV || grow >= 0) {       // rows past M hold zeros: nothing to add (the buffer row stays zero)
#pragma unroll 1
        for (int c = 0; c < PCOLS / 16; ++c) {
          if (c >= BLOCK_N / 16 && (p.t_in != nullptr || !tap_touched(c - BLOCK_N / 16))) continue;
#pragma unroll
          for (int w4 = 0; w4 < 4; ++w4) {
            const float4 v = *reinterpret_cast<const float4*>(arow + c * 16 + w4 * 4);
            asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1,%2,%3,%4};"
                         ::"l"(acc_row + c * 16 + w4 * 4), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                         : "memory");
          }
        }
      }
      named_bar_sync(BAR_EPI, EPI_THREADS);                  // all 128 rows issued
      if (ct == 0) {
        __threadfence();                               // cumulative: the CTA's reductions before the count
        const unsigned old = atomicAdd(p.counters + tile_id, 1u);
        const bool last = old == static_cast<unsigned>(p.split - 1);
        if (last) p.counters[tile_id] = 0u;            // ready for the next launch on this stream
        __threadfence();
        *flag = last ? 1u : 0u;
      }
      named_bar_sync(BAR_EPI, EPI_THREADS);
      elected = *flag != 0u;
      if (elected && G == 1) {
        // one burst: the reduced row (all CTAs' partials, this one's included), then wipe it for
        // the next launch that gets this workspace region
        const float4* src = reinterpret_cast<const float4*>(acc_row);
#pragma unroll
        for (int i = 0; i < PCOLS / 4; ++i) {
          const float4 t4 = __ldcg(src + i);
          rowv[4 * i] = t4.x; rowv[4 * i + 1] = t4.y; rowv[4 * i + 2] = t4.z; rowv[4 * i + 3] = t4.w;
        }
        float4* dstz = reinterpret_cast<float4*>(acc_row);
#pragma unroll
        for (int i = 0; i < PCOLS / 4; ++i) __stcg(dstz + i, make_float4(0.f, 0.f, 0.f, 0.f));
      }
    }
    if (!TAPLOOP && elected) {
#pragma unroll
      for (int g = 0; g < S::TG; ++g)
#pragma unroll
      for (int q = 0; q < GQ; ++q) {
        float t[16];
        if (p.t_in == nullptr) {
          if constexpr (SPLITK) {
            if constexpr (G == 1) {
#pragma unroll
              for (int j = 0; j < R_PAD; ++j) t[j] = rowv[BLOCK_N + j];
            } else {
              float4* src = reinterpret_cast<float4*>(acc_row + BLOCK_N + R_PAD * g);
#pragma unroll
              for (int w4 = 0; w4 < 4; ++w4) {
                const float4 t4 = __ldcg(src + w4);
                t[4 * w4] = t4.x; t[4 * w4 + 1] = t4.y; t[4 * w4 + 2] = t4.z; t[4 * w4 + 3] = t4.w;
                __stcg(src + w4, make_float4(0.f, 0.f, 0.f, 0.f));
              }
            }
          } else {
            ld_acc16(arow + BLOCK_N + RP * g + 16 * q, t);
          }
        } else {
          long long srow = grow;
          if constexpr (CONV && G > 1) {   // group g = tap g: the pixel shifted by (dy - pad, dx - pad)
            const int hh = h0 + row / p.TW + g / p.kw - p.pad_h;
            const int ww = w0 + row % p.TW + g % p.kw - p.pad_w;
            srow = (grow >= 0 && hh >= 0 && hh < p.H && ww >= 0 && ww < p.W)
                       ? (static_cast<long long>(img) * p.H + hh) * p.W + ww : -1;
          }
          if (srow >= 0) {
            const float4* src = reinterpret_cast<const float4*>(p.t_in + srow * RP + 16 * q);
            const float4 a = __ldg(src), b = __ldg(src + 1), c = __ldg(src + 2), d = __ldg(src + 3);
            t[0] = a.x; t[1] = a.y; t[2] = a.z; t[3] = a.w; t[4] = b.x; t[5] = b.y; t[6] = b.z; t[7] = b.w;
            t[8] = c.x; t[9] = c.y; t[10] = c.z; t[11] = c.w; t[12] = d.x; t[13] = d.y; t[14] = d.z; t[15] = d.w;
          } else {
#pragma unroll
            for (int j = 0; j < 16; ++j) t[j] = 0.f;
          }
        }
        if (p.t_out != nullptr && n_blk == 0 && g == p.t_group && grow >= 0) {
          float4* dst = reinterpret_cast<float4*>(p.t_out + grow * RP + 16 * q);
          dst[0] = make_float4(t[0], t[1], t[2], t[3]);
          dst[1] = make_float4(t[4], t[5], t[6], t[7]);
          dst[2] = make_float4(t[8], t[9], t[10], t[11]);
          dst[3] = make_float4(t[12], t[13], t[14], t[15]);
        }
        if constexpr (RP > R_PAD) load_coef(16 * q);
#pragma unroll
        for (int j = 0; j < 16; ++j) t[j] *= coef[j];
        const uint32_t dst = sbase + S::OFF_T + (row >> 3) * (256 * KG) + (g * GQ + q) * 256 + (row & 7) * 16;
        st_shared_v4(dst, pack2(t[0], t[1], p.fmt), pack2(t[2], t[3], p.fmt),
                     pack2(t[4], t[5], p.fmt), pack2(t[6], t[7], p.fmt));
        st_shared_v4(dst + 128, pack2(t[8], t[9], p.fmt), pack2(t[10], t[11], p.fmt),
                     pack2(t[12], t[13], p.fmt), pack2(t[14], t[15], p.fmt));
      }
    }
  }
  fence_proxy_async_smem();  // generic-proxy smem writes (T', U) -> visible to the tensor-core proxy
  named_bar_sync(BAR_CONSUMERS, CONSUMER_THREADS);
  if (ct == 0) LB_STAMP(5);            // T' operand visible to both warpgroups
  // split-K: only the elected CTA continues (the others have delivered their partial)
  if (SPLITK && *flag == 0u) return;

  // LoRA up-projection(s): acc[:, 0:BLOCK_N] += T'_g[128,RP] . U_g[BLOCK_N,RP]^T, this warpgroup's rows.
  // No-swizzle K-major operand of total K = 16 KG: core matrix = 8 rows x 16 B (128 B contiguous);
  // LBO = 128 B (next K core matrix), SBO = 256 KG bytes (next 8-row group).
  if constexpr (TAPLOOP) {
    // one tap at a time through the one T'/U buffer pair: stage U_t (all consumers) and T'_t
    // (warpgroup 0, row per thread, from t_in at the tap-shifted pixel), then K = RP into acc
#pragma unroll 1
    for (int g = 0; g < G; ++g) {
      for (int i = ct; i < BLOCK_N; i += CONSUMER_THREADS) {   // U_t
        const int n = n0 + i;
#pragma unroll
        for (int q = 0; q < GQ; ++q) {
          float u[16];
#pragma unroll
          for (int j = 0; j < 16; ++j)
            u[j] = (n < p.N && 16 * q + j < p.r) ? __ldg(p.up + n * p.up_rs + (16 * q + j) * p.up_cs + g * p.up_gs) : 0.f;
          const uint32_t dst = sbase + S::OFF_UP + (i >> 3) * (256 * KG) + q * 256 + (i & 7) * 16;
          st_shared_v4(dst, pack2(u[0], u[1], p.fmt), pack2(u[2], u[3], p.fmt),
                       pack2(u[4], u[5], p.fmt), pack2(u[6], u[7], p.fmt));
          st_shared_v4(dst + 128, pack2(u[8], u[9], p.fmt), pack2(u[10], u[11], p.fmt),
                       pack2(u[12], u[13], p.fmt), pack2(u[14], u[15], p.fmt));
        }
      }
      if (ct < EPI_THREADS) {
        const int hh = h0 + row / p.TW + g / p.kw - p.pad_h;
        const int ww = w0 + row % p.TW + g % p.kw - p.pad_w;
        const bool in = grow >= 0 && hh >= 0 && hh < p.H && ww >= 0 && ww < p.W;
        const float4* src = reinterpret_cast<const float4*>(
            p.t_in + (in ? ((static_cast<long long>(img) * p.H + hh) * p.W + ww) * RP : 0));
#pragma unroll
        for (int q = 0; q < GQ; ++q) {
          float t[16];
#pragma unroll
          for (int j = 0; j < 16; j += 4) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (in) v = __ldg(src + (16 * q + j) / 4);
            t[j] = v.x; t[j + 1] = v.y; t[j + 2] = v.z; t[j + 3] = v.w;
          }
#pragma unroll
          for (int j = 0; j < 16; ++j)
            t[j] *= (16 * q + j < p.r) ? p.scale * (p.diag ? __ldg(p.diag + 16 * q + j) : 1.f) : 0.f;
          const uint32_t dst = sbase + S::OFF_T + (row >> 3) * (256 * KG) + q * 256 + (row & 7) * 16;
          st_shared_v4(dst, pack2(t[0], t[1], p.fmt), pack2(t[2], t[3], p.fmt),
                       pack2(t[4], t[5], p.fmt), pack2(t[6], t[7], p.fmt));
          st_shared_v4(dst + 128, pack2(t[8], t[9], p.fmt), pack2(t[10], t[11], p.fmt),
                       pack2(t[12], t[13], p.fmt), pack2(t[14], t[15], p.fmt));
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(BAR_CONSUMERS, CONSUMER_THREADS);   // T'_t, U_t staged
      reg_fence<AREG>(acc);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KG; ++kk) {
        const uint64_t ad = wgmma_desc(sbase + S::OFF_T + wg * (8 * 256 * KG) + kk * 256, 128, 256 * KG, 0);
        const uint64_t bd = wgmma_desc(sbase + S::OFF_UP + kk * 256, 128, 256 * KG, 0);
        wgmma_ss<BLOCK_N>(acc, ad, bd, p.fmt);
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence<AREG>(acc);
      named_bar_sync(BAR_CONSUMERS, CONSUMER_THREADS);   // both warpgroups done with the buffers
    }
    park_acc<BLOCK_N, S::ACC_LD>(acc_s, acc, wg * 64, 0);
  } else {
    constexpr int LREG = DROP ? BLOCK_N / 2 : 1;
    float lacc[LREG];              // DROP: the LoRA product's own accumulator (masked in the drain)
#pragma unroll
    for (int i = 0; i < LREG; ++i) lacc[i] = 0.f;
    if constexpr ((SPLITK || CL > 1) && !DROP) {   // the base lives in the reduced row / summed ACC
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
    }
    reg_fence<AREG>(acc);
    reg_fence<LREG>(lacc);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KG; ++kk) {
      const uint64_t ad = wgmma_desc(sbase + S::OFF_T + wg * (8 * 256 * KG) + kk * 256, 128, 256 * KG, 0);
      const uint64_t bd = wgmma_desc(sbase + S::OFF_UP + kk * 256, 128, 256 * KG, 0);
      if constexpr (DROP) wgmma_ss<BLOCK_N>(lacc, ad, bd, p.fmt);
      else wgmma_ss<BLOCK_N>(acc, ad, bd, p.fmt);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<AREG>(acc);
    reg_fence<LREG>(lacc);
    if constexpr (DROP) park_acc<BLOCK_N, S::ACC_LD>(acc_s, lacc, wg * 64, S::L_COL0);
    else if constexpr (CL > 1) park_acc<BLOCK_N, S::ACC_LD, true>(acc_s, acc, wg * 64, 0);
    else park_acc<BLOCK_N, S::ACC_LD>(acc_s, acc, wg * 64, 0);
  }
  named_bar_sync(BAR_CONSUMERS, CONSUMER_THREADS);   // LoRA MMAs of both warpgroups finished
  if (ct >= EPI_THREADS) {
    finish();
    return;
  }
  if (ct == 0) LB_STAMP(6);            // LoRA MMA completed

  // ------------------------------------------------------------ drain (row per thread)
  // Final accumulator -> (+bias) -> OutT -> swizzled staging -> TMA store
  uint32_t ds0 = 0, ds1 = 0, dthr = 0;
  if constexpr (DROP) {
    const unsigned long long sd = __ldg(p.seed);
    ds0 = static_cast<uint32_t>(sd);
    ds1 = static_cast<uint32_t>(sd >> 32);
    dthr = drop_threshold(p.drop_p);
  }
  auto drain_chunk = [&](const int c) {
    float v[32];
    ld_acc16(arow + c * 32, v);
    ld_acc16(arow + c * 32 + 16, v + 16);
    float f[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] = v[j] + bias_s[c * 32 + j];
    if constexpr (SPLITK) {
      // the parked base columns hold only the LoRA product here (this CTA's own partial is already
      // inside the reduced row); non-DROP: v = T'.U^T, DROP: v is stale and ignored
      if constexpr (G == 1) {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          f[j] = (DROP ? 0.f : v[j]) + bias_s[c * 32 + j] + rowv[c * 32 + j];
      } else {
        float4* src = reinterpret_cast<float4*>(acc_row + c * 32);
#pragma unroll
        for (int w4 = 0; w4 < 8; ++w4) {
          const float4 t4 = __ldcg(src + w4);
          f[4 * w4] = (DROP ? 0.f : v[4 * w4]) + bias_s[c * 32 + 4 * w4] + t4.x;
          f[4 * w4 + 1] = (DROP ? 0.f : v[4 * w4 + 1]) + bias_s[c * 32 + 4 * w4 + 1] + t4.y;
          f[4 * w4 + 2] = (DROP ? 0.f : v[4 * w4 + 2]) + bias_s[c * 32 + 4 * w4 + 2] + t4.z;
          f[4 * w4 + 3] = (DROP ? 0.f : v[4 * w4 + 3]) + bias_s[c * 32 + 4 * w4 + 3] + t4.w;
          __stcg(src + w4, make_float4(0.f, 0.f, 0.f, 0.f));
        }
      }
    }
    if constexpr (DROP) {
      float lv[32];
      ld_acc16(arow + S::L_COL0 + c * 32, lv);
      ld_acc16(arow + S::L_COL0 + c * 32 + 16, lv + 16);
      // element index row*N + n; N % 8 == 0 and the chunk starts at a multiple of 32, so the
      // chunk's first element is even: 16 pair-hashes cover its 32 columns
      const unsigned long long e0 =
          (static_cast<unsigned long long>(grow < 0 ? 0 : grow) * p.N + n0 + c * 32) >> 1;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        const uint32_t bits = drop_bits(ds0, ds1, e0 + jj);
        if ((bits & 0xffffu) >= dthr) f[2 * jj] += lv[2 * jj] * p.drop_inv;
        if ((bits >> 16) >= dthr) f[2 * jj + 1] += lv[2 * jj + 1] * p.drop_inv;
      }
    }
    if constexpr (sizeof(OutT) == 2) {
      const int box = c >> 1;
      const uint32_t rbase = sbase + S::OFF_OUT + box * S::BOX_BYTES + row * 128;
#pragma unroll
      for (int qq = 0; qq < 4; ++qq) {
        const int piece = ((c & 1) * 4 + qq) ^ (row & 7);
        st_shared_v4(rbase + piece * 16, pack2(f[qq * 8 + 0], f[qq * 8 + 1], p.fmt),
                     pack2(f[qq * 8 + 2], f[qq * 8 + 3], p.fmt),
                     pack2(f[qq * 8 + 4], f[qq * 8 + 5], p.fmt),
                     pack2(f[qq * 8 + 6], f[qq * 8 + 7], p.fmt));
      }
    } else {
      const uint32_t rbase = sbase + S::OFF_OUT + c * S::BOX_BYTES + row * 128;
#pragma unroll
      for (int qq = 0; qq < 8; ++qq) {
        const int piece = qq ^ (row & 7);
        st_shared_v4(rbase + piece * 16, __float_as_uint(f[qq * 4 + 0]),
                     __float_as_uint(f[qq * 4 + 1]), __float_as_uint(f[qq * 4 + 2]),
                     __float_as_uint(f[qq * 4 + 3]));
      }
    }
  };
  if constexpr (SPLITK && G == 1) {   // fully unrolled: the reduced row is indexed statically (registers)
#pragma unroll
    for (int c = 0; c < BLOCK_N / 32; ++c) drain_chunk(c);
  } else {
#pragma unroll 1
    for (int c = 0; c < BLOCK_N / 32; ++c) drain_chunk(c);
  }
  fence_proxy_async_smem();
  named_bar_sync(BAR_EPI, EPI_THREADS);
  if (ct == 0) {
    for (int b = 0; b < S::NUM_BOXES; ++b) {
      const int col = n0 + b * S::BOX_COLS;
      if (col >= p.N) break;
      if constexpr (CONV)
        tma_store_4d(&tmY, sbase + S::OFF_OUT + b * S::BOX_BYTES, col, w0, h0, img);
      else
        tma_store_2d(&tmY, sbase + S::OFF_OUT + b * S::BOX_BYTES, col, m0);
    }
    LB_STAMP(7);                       // drain done, stores issued
    tma_store_commit();
    tma_store_wait_read0();
    LB_STAMP(8);                       // staging buffer released
  }
  finish();
}

template <int BLOCK_N, int STAGES, typename OutT, bool CONV, int G, int MIN_CTAS = 1, bool DROP = false,
          bool SPLITK = false, int CL = 1, bool INLINE_TMA = false, int RP = R_PAD>
__global__ void __launch_bounds__(kernel_threads<INLINE_TMA>(), MIN_CTAS)
fused_lora_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW,
                  const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmY,
                  const FusedParams p) {
  fused_tile<BLOCK_N, STAGES, OutT, CONV, G, DROP, SPLITK, CL, INLINE_TMA, RP>(tmX, tmW, tmD, tmY, p, blockIdx.x,
                                                                             blockIdx.y);
}

// Several same-dtype linear problems in ONE launch (sites that share an input: q/k/v of an
// attention block, k/v of every cross-attention, CLIP's k/v/q): a CTA looks up which problem its
// tile belongs to. Small sites under-fill 132 SMs on their own; together they run in the time of one.
constexpr int MAX_GROUP = 4;
struct GroupedArgs {
  CUtensorMap tmX[MAX_GROUP], tmW[MAX_GROUP], tmD[MAX_GROUP], tmY[MAX_GROUP];
  FusedParams p[MAX_GROUP];
  int tile_start[MAX_GROUP + 1];   // prefix sum of tiles per problem
  int n_tiles_n[MAX_GROUP];        // tiles along N per problem
  int n_problems;
};

template <int BLOCK_N, int STAGES, typename OutT, int MIN_CTAS = 1, bool INLINE_TMA = false>
__global__ void __launch_bounds__(kernel_threads<INLINE_TMA>(), MIN_CTAS)
fused_lora_grouped_kernel(const __grid_constant__ GroupedArgs a) {
  int q = 0;
#pragma unroll
  for (int i = 1; i < MAX_GROUP; ++i)
    if (i < a.n_problems && static_cast<int>(blockIdx.x) >= a.tile_start[i]) q = i;
  const int local = blockIdx.x - a.tile_start[q];
  const int n_blk = local % a.n_tiles_n[q], m_blk = local / a.n_tiles_n[q];
  fused_tile<BLOCK_N, STAGES, OutT, false, 1, false, false, 1, INLINE_TMA>(a.tmX[q], a.tmW[q], a.tmD[q], a.tmY[q],
                                                                         a.p[q], n_blk, m_blk);
}

}  // namespace lb
