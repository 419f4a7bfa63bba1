// Sparse, exact AdamW over the token-embedding table: the gradient scatter that replaces the dense
// embedding backward, the write-back of the trained rows, and the lazy weight decay of the rows no
// gradient has touched yet. The AdamW update itself is the arena's optimizer launch: the claimed
// rows are one more param-group of the LoRA arena (see lora_b200/embed_rows.py). Under data
// parallelism the scatter claims slots over the union of every rank's ids (lb_embed_rows_scatter_dp),
// so the ranks' rows groups hold the same tokens in the same slots and the arena's all-reduce can sum
// them.
//
// Row state (all device memory, owned by the caller):
//   slot_of  int32 [V]         token -> slot, -1 = unclaimed
//   slot_tok int32 [capacity]  slot -> token
//   state    int32 [4]         {claimed, claimed after this step's scatter, flush ticket, flags}
//                              flags: bit 0 = a token found no free slot (its gradient was dropped),
//                                     bit 1 = a token id outside [0, V) was skipped
//   decay    fp64  [1]         product of the per-step decay factors since the last flush
//   master / slot_grad         fp32 [capacity, D]: the rows group of the arena's p / g buffers
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "lora_b200.h"
#include "ptx.cuh"

namespace lb_embed {

constexpr int THREADS = 256;
constexpr int MAX_TOKENS = 2048;        // world * B * S per scatter launch (shared-memory bookkeeping)
constexpr int MAX_CTAS = 264;

__device__ __forceinline__ float load_elem(const void* base, size_t i, int dtype) {
  if (dtype == LB_F32) return reinterpret_cast<const float*>(base)[i];
  const uint16_t h = reinterpret_cast<const uint16_t*>(base)[i];
  if (dtype == LB_BF16) return __bfloat162float(__ushort_as_bfloat16(h));
  return __half2float(__ushort_as_half(h));
}

__device__ __forceinline__ void store_elem(void* base, size_t i, int dtype, float x) {
  if (dtype == LB_F32) {
    reinterpret_cast<float*>(base)[i] = x;
  } else if (dtype == LB_BF16) {
    reinterpret_cast<uint16_t*>(base)[i] = __bfloat16_as_ushort(__float2bfloat16_rn(x));
  } else {
    reinterpret_cast<uint16_t*>(base)[i] = __half_as_ushort(__float2half_rn(x));
  }
}

constexpr int MAX_WORLD = 16;

// Every rank's id buffer, in rank order (this rank's own one included), and for the peer handshake
// every rank's one-word flag. Passed by value: the launch needs no device-side pointer table.
struct RankIds {
  const long long* ids[MAX_WORLD];
  const unsigned int* flags[MAX_WORLD];
};

// Every CTA redoes the (cheap, shared-memory) bookkeeping of the whole batch, so that it knows
// every distinct token's slot without a second launch; CTA b then owns the distinct tokens
// b, b + grid, ... in first-occurrence order. A slot claimed by this launch has an index >= the
// committed count state[0], which this launch never writes: whether another CTA has already
// published a new token's slot or not, every CTA classifies that token as "new" and computes the
// same slot for it.
//
// Data parallel (world > 1): the "whole batch" is the concatenation [ids of rank 0; ids of rank 1;
// ...] of n_per_rank positions each, so every rank claims the same slots for the same tokens in the
// same order as one process running the concatenated batch -- tokens that occur only on other ranks
// included (master = stored row * decay, no local gradient). Only this rank's positions
// [rank * n_per_rank, (rank + 1) * n_per_rank) add into slot_grad (grad holds just those rows); the
// arena's all-reduce sums the ranks.
//
// Handshake (flags given): CTA 0 publishes this rank's epoch in its own flag with a system-scope
// release (the ids were written before this launch, in stream order); every CTA then waits until
// every peer's flag has reached the epoch before it reads that peer's ids. epoch_dev = {epoch of the
// last scatter, CTA ticket}: every CTA reads the epoch before taking its ticket, the last CTA to
// finish advances it, so the counter moves once per launch on every rank and is never restored.
// Buffer lifetime: a peer's ids buffer is not rewritten while this rank may still read it. Rank r
// writes its next step's ids only after its lb_optim_step_dp of this step has returned; that launch
// waits for every rank's barrier-2 signal, and each rank signals barrier 2 from its own
// lb_optim_step_dp, which its stream runs after its scatter has finished reading every rank's ids.
__global__ void __launch_bounds__(THREADS)
embed_rows_scatter_kernel(RankIds src, int world, int rank, int n_per_rank, unsigned int* __restrict__ my_flag,
                          unsigned int* __restrict__ epoch_dev, const void* __restrict__ grad, int grad_dtype,
                          int D, int V, int* __restrict__ slot_of, int* __restrict__ slot_tok,
                          int capacity, int* __restrict__ state, const void* __restrict__ table,
                          int table_dtype, const double* __restrict__ decay, float* __restrict__ master,
                          float* __restrict__ slot_grad) {
  __shared__ int s_id[MAX_TOKENS];      // token id per position (-1: skipped)
  __shared__ int s_next[MAX_TOKENS];    // next position holding the same token, -1 at the last one
  __shared__ int s_first[MAX_TOKENS];   // k-th distinct token's first position
  __shared__ int s_slot[MAX_TOKENS];    // its slot (>= capacity: no free slot)
  __shared__ int s_new[MAX_TOKENS];     // 1 if this launch claims the slot
  __shared__ int s_scan[THREADS];
  const int tid = threadIdx.x;
  const int claimed0 = state[0];
  const int n_tok = world * n_per_rank;
  const int lo_local = rank * n_per_rank, hi_local = lo_local + n_per_rank;
  unsigned int epoch = 0;
  if (my_flag != nullptr) {
    epoch = epoch_dev[0] + 1u;
    if (blockIdx.x == 0 && tid == 0) {
      __threadfence_system();
      lb::st_release_sys(my_flag, epoch);
    }
    if (tid < world && tid != rank) lb::wait_flag_reached(src.flags[tid], epoch);
    __syncthreads();
  }

  for (int r = 0; r < world; ++r) {
    // volatile: a peer's buffer may have been rewritten since an earlier launch, never cache it
    const volatile long long* ids = src.ids[r];
    for (int i = tid; i < n_per_rank; i += THREADS) {
      const long long t = ids[i];
      s_id[r * n_per_rank + i] = (t >= 0 && t < V) ? static_cast<int>(t) : -1;
    }
  }
  __syncthreads();
  // first occurrence / next occurrence, per position (early exits keep repeated tokens cheap)
  const int chunk = (n_tok + THREADS - 1) / THREADS;
  const int lo = tid * chunk, hi = min(lo + chunk, n_tok);
  int n_first = 0, n_new = 0;
  for (int i = lo; i < hi; ++i) {
    const int id = s_id[i];
    int nx = -1;
    if (id >= 0) {
      bool first = true;
      for (int j = 0; j < i; ++j)
        if (s_id[j] == id) { first = false; break; }
      for (int j = i + 1; j < n_tok; ++j)
        if (s_id[j] == id) { nx = j; break; }
      if (first) {
        const int s = slot_of[id];
        n_first += 1;
        n_new += (s >= 0 && s < claimed0) ? 0 : 1;
      }
    }
    s_next[i] = nx;
  }
  // inclusive scan of (n_first | n_new << 16) over the threads' contiguous chunks (counts <= 2048)
  s_scan[tid] = n_first | (n_new << 16);
  __syncthreads();
  for (int o = 1; o < THREADS; o <<= 1) {
    const int add = tid >= o ? s_scan[tid - o] : 0;
    __syncthreads();
    s_scan[tid] += add;
    __syncthreads();
  }
  const int excl = tid ? s_scan[tid - 1] : 0;
  int k = excl & 0xffff, r = excl >> 16;
  for (int i = lo; i < hi; ++i) {
    const int id = s_id[i];
    if (id < 0) continue;
    bool first = true;
    for (int j = 0; j < i; ++j)
      if (s_id[j] == id) { first = false; break; }
    if (!first) continue;
    const int s = slot_of[id];
    const bool old = s >= 0 && s < claimed0;
    s_first[k] = i;
    s_slot[k] = old ? s : claimed0 + r;
    s_new[k] = old ? 0 : 1;
    r += old ? 0 : 1;
    ++k;
  }
  const int total = s_scan[THREADS - 1];
  const int n_distinct = total & 0xffff, n_claim = total >> 16;
  __syncthreads();

  if (blockIdx.x == 0 && tid == 0) {
    int flags = 0;
    for (int i = 0; i < n_tok; ++i)
      if (s_id[i] < 0) flags |= 2;
    if (claimed0 + n_claim > capacity) flags |= 1;
    if (flags) atomicOr(state + 3, flags);
    state[1] = min(claimed0 + n_claim, capacity);
  }
  const double dk = decay[0];
  for (int d = blockIdx.x; d < n_distinct; d += gridDim.x) {
    const int slot = s_slot[d];
    if (slot >= capacity) continue;          // flagged above; never written
    const int p0 = s_first[d];
    const int tok = s_id[p0];
    float* mrow = master + static_cast<size_t>(slot) * D;
    float* grow = slot_grad + static_cast<size_t>(slot) * D;
    if (s_new[d]) {
      if (tid == 0) { slot_of[tok] = slot; slot_tok[slot] = tok; }
      // what dense AdamW would have left in this row: the stored value times the decay since the flush
      for (int c = tid; c < D; c += THREADS)
        mrow[c] = static_cast<float>(static_cast<double>(load_elem(table, static_cast<size_t>(tok) * D + c, table_dtype)) * dk);
    }
    // this rank's positions of the token: a contiguous run of its position chain (ranks in order)
    int pl = p0;
    while (pl >= 0 && pl < lo_local) pl = s_next[pl];
    if (pl < 0 || pl >= hi_local) continue;  // the token occurs on other ranks only
    for (int c = tid; c < D; c += THREADS) {
      float acc = 0.f;
      for (int p = pl; p >= 0 && p < hi_local; p = s_next[p])
        acc += load_elem(grad, static_cast<size_t>(p - lo_local) * D + c, grad_dtype);
      grow[c] += acc;
    }
  }
  if (my_flag != nullptr) {
    __syncthreads();
    if (tid == 0) {
      __threadfence();
      if (atomicAdd(epoch_dev + 1, 1u) == gridDim.x - 1) {
        epoch_dev[0] = epoch;                // every CTA has read the old epoch before taking its ticket
        epoch_dev[1] = 0u;
      }
    }
  }
}

__global__ void __launch_bounds__(THREADS)
embed_rows_write_back_kernel(const float* __restrict__ master, const int* __restrict__ slot_tok, int* __restrict__ state,
                             int n_write, void* __restrict__ table, int table_dtype, int D, int V,
                             double* __restrict__ decay, const float* __restrict__ lr_dev, int lr_index, float wd) {
  const int claimed = state[1];
  const int n = n_write < 0 ? claimed : min(n_write, claimed);
  for (int s = blockIdx.x; s < n; s += gridDim.x) {
    const int tok = slot_tok[s];
    if (tok < 0 || tok >= V) continue;
    const float* mrow = master + static_cast<size_t>(s) * D;
    for (int c = threadIdx.x; c < D; c += THREADS) store_elem(table, static_cast<size_t>(tok) * D + c, table_dtype, mrow[c]);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    state[0] = claimed;                      // commit this step's claims for the next scatter
    if (decay != nullptr && lr_dev != nullptr) {
      const float lr = lr_dev[lr_index];
      const float f = 1.f - lr * wd;         // the factor the optimizer launch applied to every row
      decay[0] = decay[0] * static_cast<double>(f);
    }
  }
}

__global__ void __launch_bounds__(THREADS)
embed_rows_flush_kernel(void* __restrict__ table, int table_dtype, int V, int D, const int* __restrict__ slot_of,
                        double* __restrict__ decay, int* __restrict__ state) {
  const double dk = decay[0];
  if (dk == 1.0) return;                     // every CTA sees the same value: nothing to do, nothing to reset
  for (int row = blockIdx.x; row < V; row += gridDim.x) {
    if (slot_of[row] >= 0) continue;         // claimed rows hold their written-back masters
    const size_t o = static_cast<size_t>(row) * D;
    for (int c = threadIdx.x; c < D; c += THREADS)
      store_elem(table, o + c, table_dtype, static_cast<float>(static_cast<double>(load_elem(table, o + c, table_dtype)) * dk));
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(reinterpret_cast<unsigned int*>(state + 2), 1u) == gridDim.x - 1) {
      decay[0] = 1.0;                        // every CTA has read decay[0] before taking its ticket
      state[2] = 0;
    }
  }
}

inline bool dtype_ok(int t) { return t == LB_F32 || t == LB_BF16 || t == LB_F16; }

}  // namespace lb_embed

using namespace lb_embed;

extern "C" int lb_embed_rows_scatter_dp(const long long* const* ids_by_rank, int world, int rank, int n_per_rank,
                                        const void* grad, int grad_dtype, int D, int V, int* slot_of, int* slot_tok,
                                        int capacity, int* state, const void* table, int table_dtype,
                                        const double* decay, float* master, float* slot_grad,
                                        const unsigned int* const* flags_by_rank, unsigned int* epoch_dev,
                                        void* stream) {
  if (ids_by_rank == nullptr || grad == nullptr || slot_of == nullptr || slot_tok == nullptr ||
      state == nullptr || table == nullptr || decay == nullptr || master == nullptr || slot_grad == nullptr)
    return LB_ERR_SHAPE;
  if (world < 1 || world > MAX_WORLD || rank < 0 || rank >= world) return LB_ERR_SHAPE;
  if (n_per_rank <= 0 || n_per_rank > MAX_TOKENS / world || D <= 0 || V <= 0 || capacity <= 0)
    return LB_ERR_SHAPE;
  if ((flags_by_rank == nullptr) != (epoch_dev == nullptr)) return LB_ERR_SHAPE;
  if (!dtype_ok(grad_dtype) || !dtype_ok(table_dtype)) return LB_ERR_DTYPE;
  RankIds src = {};
  for (int r = 0; r < world; ++r) {
    if (ids_by_rank[r] == nullptr) return LB_ERR_SHAPE;
    src.ids[r] = ids_by_rank[r];
    if (flags_by_rank != nullptr) {
      if (flags_by_rank[r] == nullptr) return LB_ERR_SHAPE;
      src.flags[r] = flags_by_rank[r];
    }
  }
  unsigned int* my_flag = flags_by_rank ? const_cast<unsigned int*>(flags_by_rank[rank]) : nullptr;
  const int n_tok = world * n_per_rank;
  const int grid = n_tok < MAX_CTAS ? n_tok : MAX_CTAS;
  embed_rows_scatter_kernel<<<grid, THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      src, world, rank, n_per_rank, my_flag, epoch_dev, grad, grad_dtype, D, V, slot_of, slot_tok, capacity, state,
      table, table_dtype, decay, master, slot_grad);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_embed_rows_scatter(const long long* ids, const void* grad, int grad_dtype, int n_tok, int D, int V,
                                     int* slot_of, int* slot_tok, int capacity, int* state, const void* table,
                                     int table_dtype, const double* decay, float* master, float* slot_grad,
                                     void* stream) {
  if (ids == nullptr) return LB_ERR_SHAPE;
  const long long* one[1] = {ids};
  return lb_embed_rows_scatter_dp(one, 1, 0, n_tok, grad, grad_dtype, D, V, slot_of, slot_tok, capacity, state, table,
                                  table_dtype, decay, master, slot_grad, nullptr, nullptr, stream);
}

extern "C" int lb_embed_rows_write_back(const float* master, const int* slot_tok, int capacity, int* state,
                                        int n_write, void* table, int table_dtype, int D, int V, double* decay,
                                        const float* lr_dev, int lr_index, float weight_decay, void* stream) {
  if (master == nullptr || slot_tok == nullptr || state == nullptr || table == nullptr) return LB_ERR_SHAPE;
  if (capacity <= 0 || D <= 0 || V <= 0 || lr_index < 0) return LB_ERR_SHAPE;
  if ((decay == nullptr) != (lr_dev == nullptr)) return LB_ERR_SHAPE;
  if (!dtype_ok(table_dtype)) return LB_ERR_DTYPE;
  const int grid = capacity < MAX_CTAS ? capacity : MAX_CTAS;
  embed_rows_write_back_kernel<<<grid, THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      master, slot_tok, state, n_write, table, table_dtype, D, V, decay, lr_dev, lr_index, weight_decay);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}

extern "C" int lb_embed_rows_flush(void* table, int table_dtype, int V, int D, const int* slot_of, double* decay,
                                   int* state, void* stream) {
  if (table == nullptr || slot_of == nullptr || decay == nullptr || state == nullptr) return LB_ERR_SHAPE;
  if (V <= 0 || D <= 0) return LB_ERR_SHAPE;
  if (!dtype_ok(table_dtype)) return LB_ERR_DTYPE;
  const int grid = V < 4 * MAX_CTAS ? V : 4 * MAX_CTAS;
  embed_rows_flush_kernel<<<grid, THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(table, table_dtype, V, D,
                                                                                      slot_of, decay, state);
  return cudaGetLastError() == cudaSuccess ? LB_OK : LB_ERR_CUDA;
}
