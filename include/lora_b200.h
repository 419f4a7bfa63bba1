/* lora_b200 C-ABI: the drop-in boundary for the LoRA hot path of cloneofsimo/lora on H100 (sm_90a).
 *
 * Plain C: raw device pointers, sizes, dtype enums and a cudaStream_t passed as void*. No torch
 * or ATen types cross this boundary. Every entry point enqueues work on `stream` and returns an
 * int status immediately (0 = LB_OK, negative = refused, nothing was launched); kernels never
 * synchronise the host. The reference has no FFI of its own (it is pure Python on top of torch
 * eager); each entry point below names the reference code it replaces, and INTEGRATION.md shows
 * the ctypes stub that binds it under the reference's own module classes.
 *
 * Conventions
 *   - "16-bit" operands are bf16 (LB_BF16) or fp16 (LB_F16), chosen per call by in_dtype.
 *   - LoRA master factors are fp32:   down A[r,K] row-major,   up B[N,r] row-major
 *     (reference: lora_down.weight / lora_up.weight, lora_diffusion/lora.py:44-46).
 *   - Rank pad: entry points whose operands hold the rank take `r_pad` (16, 32 or 64) right after
 *     `r`, with 1 <= r <= r_pad <= 64. "down" operands are 16-bit copies zero-padded to r_pad
 *     rows: [r_pad,K] row-major (built by lb_cast_rows_pad). T / dT / V buffers are fp32
 *     [M,r_pad] row-major, columns >= r are zero. r_pad outside {16, 32, 64}: LB_ERR_SHAPE;
 *     r > r_pad: LB_ERR_RANK (both before any CUDA call). The grouped entry points
 *     (lb_lora_linear_fwd_grouped, lb_lora_wgrad_multi) take r <= 16 at a pad of 16 only.
 *   - All base pointers 16-byte aligned; K % 8 == 0; N % 8 == 0 (N % 4 for fp32 outputs).
 */
#ifndef LORA_B200_H
#define LORA_B200_H

#ifdef __cplusplus
extern "C" {
#endif

enum lb_status {
  LB_OK = 0,
  LB_ERR_SHAPE = -1, /* unsupported / misaligned extent */
  LB_ERR_RANK = -2,  /* r outside [1,r_pad] */
  LB_ERR_DTYPE = -3,
  LB_ERR_ALIGN = -4, /* pointer not 16-byte aligned */
  LB_ERR_TMAP = -5,  /* cuTensorMapEncodeTiled unavailable or failed */
  LB_ERR_CUDA = -6   /* launch error (cudaGetLastError) */
};

enum lb_dtype { LB_BF16 = 0, LB_F16 = 1, LB_F32 = 2 };
/* OR-ed into `in_dtype` of the fused linear entries: the frozen weight argument (W, or Wt of the dX
 * entry) is NOT row-major [N, K] but the 64 x 64-block layout written by lb_tile_weight -- block
 * (n64, kb) occupies rows [(n64 * ceil(K/64) + kb) * 64, +64) of a [rows, 64] 16-bit tensor, zero padded
 * -- so that every TMA box of the weight stream is one contiguous 8 KB run of HBM (a row-major box is
 * 64-192 rows of 128 bytes a whole K apart). Optional; off by default. */
#define LB_W_TILED 0x100

/* ABI version of this header (bumped on any signature change). */
int lb_abi_version(void);

/* Fused frozen linear + LoRA forward (wgmma/TMA), one launch:
 *     Y[M,N] = X[M,K] . W[N,K]^T (+ bias[N]) + ((X . down^T) * (scale * diag)) . up^T
 * up element (n, j) is read from the fp32 master at up[n*up_rs + j*up_cs]; diag is the optional
 * selector diagonal [r] (NULL = identity); T_out (NULL = skip) receives X . down^T (unscaled);
 * T_in (normally NULL): when given, the rank-r activations are read from this fp32 [M,r_pad] buffer
 * instead of being computed (dropout path: T = (mask o gY) . B comes from lb_lora_dropout_dt).
 * At r_pad > 16 only one-tile-per-CTA plans run (no split-K).
 * Replaces LoraInjectedLinear.forward, lora_diffusion/lora.py:53-58 (F.linear + lora_down +
 * selector + lora_up + scale + add), dropout handled by the caller (see INTEGRATION.md).
 *
 * The SAME entry point is the backward-dX kernel: with W := W^T[K,N] (pre-transposed frozen
 * weight), down := B^T padded [r_pad,N], up := A read transposed (up_rs = 1, up_cs = K) it returns
 *     dX[M,K] = gY . W + ((gY . B) * (scale * diag)) . A       and  T_out = gY . B.
 */
int lb_lora_linear_fwd(const void* X, const void* W, const float* bias, const void* down,
                       const float* up, long long up_rs, long long up_cs, const float* diag,
                       float scale, void* Y, float* T_out, const float* T_in, int M, int K, int N,
                       int r, int r_pad, int in_dtype, int out_dtype, void* stream);

/* lb_lora_linear_fwd with an ACTIVE nn.Dropout(p) on the LoRA branch (lora.py:45,56: module in
 * training mode, p > 0 -- the state of every site built by inject_trainable_lora_extended and the
 * monkeypatch_* loaders), still ONE launch:
 *     Y = X . W^T (+ bias) + keep(m,n)/(1-p) * (((X . down^T) * (scale * diag)) . up^T)[m,n]
 * The LoRA product keeps its own accumulator and the keep-mask (csrc/dropmask.cuh: a counter hash
 * of (*seed_dev, m*N + n); seed_dev points to one uint64 in DEVICE memory so that a captured graph
 * draws a new mask per replay) is applied while the tile is drained. Backward recomputes the same
 * mask: lb_lora_dropout_dt, lb_lora_wgrad_masked / lb_lora_wgrad_pair(drop_p). */
int lb_lora_linear_fwd_dropout(const void* X, const void* W, const float* bias, const void* down,
                               const float* up, long long up_rs, long long up_cs, const float* diag,
                               float scale, void* Y, float* T_out, int M, int K, int N, int r,
                               int r_pad, int in_dtype, int out_dtype, float drop_p,
                               const void* seed_dev, void* stream);

/* Up to 4 independent lb_lora_linear_fwd problems of the same operand/output dtype in ONE launch
 * (sites that share an input -- q/k/v of a self-attention, k/v of a cross-attention, CLIP's k/v/q --
 * each under-fill 132 SMs on their own). All array arguments are HOST arrays of length n; per-problem
 * semantics are exactly lb_lora_linear_fwd's at r_pad = 16 (r <= 16; T_in unsupported). */
int lb_lora_linear_fwd_grouped(int n, const void* const* X, const void* const* W,
                               const float* const* bias, const void* const* down16,
                               const float* const* up, const long long* up_rs, const long long* up_cs,
                               const float* const* diag, const float* scale, void* const* Y,
                               float* const* T_out, const int* M, const int* K, const int* N,
                               const int* r, int in_dtype, int out_dtype, void* stream);

/* Benchmark/profiling knob: tile schedule of lb_lora_linear_fwd.
 *   mode = schedule + 4 * block_n + 16 * split
 *   schedule: 0 = auto (default), 1 and 2 = one tile per CTA, 3 = split-K with the partials
 *             reduced at L2 (never chosen by `auto` for these shapes)
 *   block_n:  0 = auto, 1 = 64, 2 = 128, 3 = 192 (16-bit outputs)
 *   split:    (schedule 3 only) 0 = auto (4), 1..3 = 2..4 CTAs share a tile's K loop */
int lb_debug_set_linear_mode(int mode);
/* Profiling knob: device buffer (16 x uint64) receiving %globaltimer phase stamps of CTA (0,0) of
 * subsequent lb_lora_linear_fwd launches; NULL switches it off. */
int lb_debug_set_stamp_buffer(void* dev_buf);
/* Programmatic dependent launch for the fused kernels (cudaLaunchAttributeProgrammaticStream-
 * Serialization): the prologue of a launch (barrier init, descriptor prefetch)
 * overlaps the tail of the previous kernel in the stream. 0 = off, 1 = on; initial value from the
 * environment variable LB_PDL. */
int lb_debug_set_pdl(int on);

/* Skinny weight-gradient reduction (streams S once, fp32 atomics into out):
 *     out[j*out_js + c*out_cs] += scale * diag[j] * sum_m V[m,j] * S[m,c]     j < r, c < C
 * S may also be fp32 (in_dtype = LB_F32; the fp32-faithful mode keeps X and gY in fp32).
 * V is fp32 [M, r_pad]; ranks above 16 run as 16-wide rank groups, each re-reading S.
 * dA[r,K]: S = X[M,K],  V = gY.B (T_out of the dX call), out_js = K, out_cs = 1
 * dB[N,r]: S = gY[M,N], V = X.A^T (T_out of the forward), out_js = 1, out_cs = r
 * Replaces the autograd-generated dA/dB GEMMs of lora.py:53-58 (W frozen: no dW).
 */
int lb_lora_wgrad(const void* S, const float* V, const float* diag, float scale, float* out,
                  long long out_js, long long out_cs, int M, int C, int r, int r_pad, int in_dtype,
                  void* stream);

/* Both factor gradients of one linear site in ONE launch (the two reductions are independent):
 *   dA[j*dA_js + k*dA_cs] += scale*diag[j] * sum_m dTs[m,j] * X[m,k]      k < K
 *   dB[j*dB_js + n*dB_cs] += scale*diag[j] * sum_m T[m,j]  * gY[m,n]      n < N
 * drop_p > 0: gY is masked like in lb_lora_wgrad_masked (mask index m*N + n). */
int lb_lora_wgrad_pair(const void* X, const float* dTs, float* dA, long long dA_js, long long dA_cs,
                       int K, const void* gY, const float* T, float* dB, long long dB_js,
                       long long dB_cs, int N, const float* diag, float scale, int M, int r,
                       int r_pad, float drop_p, const void* seed_dev, int in_dtype, void* stream);

/* One reduction  out[j*out_js + c*out_cs] += scale*diag[j] * sum_{m<M} V[m,j] * S[m,c]  (see
 * lb_lora_wgrad; drop_p > 0: S masked like lb_lora_wgrad_masked with the uint64 at seed_dev). */
typedef struct lb_wgrad_problem {
  const void* S;        /* [M, C] rows of in_dtype                         */
  const float* V;       /* [M, r_pad] fp32                                 */
  float* out;
  long long out_js, out_cs;
  int M, C, r;
  float scale;
  const float* diag;    /* selector diagonal [r] or NULL                   */
  float drop_p;
  const void* seed_dev; /* device uint64 (drop_p > 0) or NULL              */
  /* conv_H > 0: the lora_down weight-gradient of a conv site (lb_lora_wgrad_conv as one problem):
   * S = NHWC input rows [M/(H*W), H, W, C], every tap (ty, tx) of the kh x kw filter reads the pixel
   * shifted by (ty - pad_h, tx - pad_w), out = dA[r, C, kh, kw] flat with out_js = C*kh*kw,
   * out_cs = kh*kw (+ tap). 0: plain rows. */
  int conv_H, conv_W, kh, kw, pad_h, pad_w;
  int r_pad;
} lb_wgrad_problem;

/* n independent reductions (HOST array) in ceil(n/24) launches. The step engine queues the dA / dB
 * of every linear site during backward and flushes them here once: the factor gradients feed only
 * the optimizer (autograd's dA/dB GEMMs of lora.py:53-58 for all sites at once). */
int lb_lora_wgrad_batch(const lb_wgrad_problem* probs, int n, int in_dtype, void* stream);

/* lb_lora_wgrad_pair for up to 4 sites that share X (a grouped family), one launch; HOST arrays.
 * r <= 16, dTs / T at a pad of 16. */
int lb_lora_wgrad_multi(int n, const void* X, const float* const* dTs, float* const* dA,
                        const void* const* gY, const float* const* T, float* const* dB, const int* N,
                        const float* const* diag, const float* scale, const int* r, int M, int K,
                        int in_dtype, void* stream);

/* ---- dropout on the LoRA branch (nn.Dropout inside the operator, lora.py:45,56,115,133; active
 * only when module.training and p > 0). keep(m,n) is a counter-based hash of (*seed_dev, m*N+n),
 * recomputed by every kernel; seed_dev is a DEVICE uint64 so CUDA-graph replays draw new masks.
 * Forward:  Y = lb_lora_linear_fwd(scale = 0)  ->  lb_lora_up_dropout adds the masked branch.
 * Backward: dTs = lb_lora_dropout_dt(gY) -> lb_lora_linear_fwd(T_in = dTs) for dX ->
 *           lb_lora_wgrad(X, dTs) for dA, lb_lora_wgrad_masked(gY, T) for dB. */
/* Y[m,n] += scale/(1-p) * keep(m,n) * sum_j T[m,j]*diag[j]*up[n*up_rs + j*up_cs]   (in place) */
int lb_lora_up_dropout(void* Y, int y_dtype, const float* T, const float* up, long long up_rs,
                       long long up_cs, const float* diag, float scale, float drop_p,
                       const void* seed_dev, int M, int N, int r, int r_pad, void* stream);
/* dTs[m,j] = sum_n keep(m,n)/(1-p) * gY[m,n] * up[n*up_rs + j*up_cs]    (fp32 [M,r_pad]) */
int lb_lora_dropout_dt(const void* gY, int in_dtype, const float* up, long long up_rs,
                       long long up_cs, float drop_p, const void* seed_dev, float* dTs, int M, int N,
                       int r, int r_pad, void* stream);
/* lb_lora_wgrad with S := keep o S / (1-p)  (S = gY [M,C], mask index m*C + c) */
int lb_lora_wgrad_masked(const void* S, const float* V, const float* diag, float scale, float* out,
                         long long out_js, long long out_cs, int M, int C, int r, int r_pad,
                         float drop_p, const void* seed_dev, int in_dtype, void* stream);

/* dA[r,Cin,kh,kw] of a LoraInjectedConv2d in ONE launch, the lora_down wgrad of lora.py:130-135:
 * rows of S are the pixels of NHWC images [M = n_img*H*W, C = Cin]; tap t = (ty,tx) reads S at pixel
 * (h + ty - pad_h, w + tx - pad_w), zero outside the image (the convolution's zero padding), and
 * accumulates into dA[j, c, ty, tx]. V = gY.B per pixel [M,r_pad]. */
int lb_lora_wgrad_conv(const void* S, const float* V, const float* diag, float scale, float* out, int M,
                       int C, int r, int r_pad, int H, int W, int kh, int kw, int pad_h, int pad_w,
                       int in_dtype, void* stream);

/* Fused frozen Conv2d + LoRA (NHWC implicit GEMM on wgmma; stride 1, dilation 1, groups 1,
 * 1x1 or 3x3 "same" padding -- the ResnetBlock2D sites of SD1.5):
 *     Y[n,h,w,:] = sum_tap X[n,h+ty-pad,w+tx-pad,:] . W[:, tap, :]^T (+ bias)
 *                  + ((sum_tap X[..] . down[:, tap, :]^T) * (scale*diag)) . up^T
 * X: NHWC 16-bit [n_img,H,W,Cin]; W: 16-bit [Cout, kh*kw*Cin] with K ordered tap-major,
 * channel-minor (built once from the frozen [Cout,Cin,kh,kw] weight); down: [r_pad, kh*kw*Cin] in
 * the same K order; up element (n, j) at up[n*up_rs + j*up_cs]; Y: NHWC [n_img,H,W,Cout];
 * T_out: fp32 [n_img*H*W, r_pad] = the rank-r activations (unscaled).
 * At r_pad > 16 only one-tile-per-CTA plans run (no split-K).
 * Replaces LoraInjectedConv2d.forward, lora_diffusion/lora.py:130-135.
 *
 * per_tap_T = 1 is the input-gradient form (dX = conv_T(gY, W) + conv_T((gY.B)*s*d, A)): call it
 * with X := gY [n_img,H,W,Cout'], W := the flipped+transposed frozen weight [Cin', taps*Cout'],
 * down := B^T padded [r_pad, Cout'] (restarts every tap), up := A read flipped:
 * element (c, tap g, j) at up[c*up_rs + j*up_cs + g*up_gs] (up_gs = -1 from the last tap).
 * T_out then receives gY.B of the unshifted tap. At r_pad > 16 a 3x3 input gradient reads its
 * per-tap T from T_in; without T_in it first writes T_out = X . down^T (one more launch, so T_out
 * is required) and reads that. T_in and T_out together are refused there. */
int lb_lora_conv2d_fwd(const void* X, const void* W, const float* bias, const void* down,
                       const float* up, long long up_rs, long long up_cs, long long up_gs,
                       const float* diag, float scale, void* Y, float* T_out, const float* T_in,
                       int n_img, int H, int Wd, int Cin, int Cout, int kh, int kw, int pad_h,
                       int pad_w, int r, int r_pad, int per_tap_T, int in_dtype, int out_dtype,
                       void* stream);

/* lb_lora_conv2d_fwd (forward direction) with an active nn.Dropout(p) on the LoRA branch
 * (lora.py:115,133; every conv site of inject_trainable_lora_extended): one launch, mask applied in
 * the drain exactly as in lb_lora_linear_fwd_dropout; mask index = pixel * Cout + n with
 * pixel = (img*H + h)*W + w. */
int lb_lora_conv2d_fwd_dropout(const void* X, const void* W, const float* bias, const void* down,
                               const float* up, long long up_rs, long long up_cs, const float* diag,
                               float scale, void* Y, float* T_out, int n_img, int H, int Wd, int Cin,
                               int Cout, int kh, int kw, int pad_h, int pad_w, int r, int r_pad,
                               int in_dtype, int out_dtype, float drop_p, const void* seed_dev,
                               void* stream);

/* Frozen conv-weight preparation: src [Cout,Cin,kh,kw] (LB_F32/LB_BF16/LB_F16) ->
 *   dst16  [Cout, kh*kw*Cin]  (tap-major K; forward operand)              and/or
 *   dstT16 [Cin, kh*kw*Cout]  with taps flipped (input-gradient operand). Either may be NULL. */
int lb_cast_conv_weight(const void* src, int src_dtype, void* dst16, void* dstT16, int Cout,
                        int Cin, int kh, int kw, int out_dtype, void* stream);

/* dst16[j, c] = (j < r) ? src[j*src_rs + c*src_cs] : 0   for j < r_pad, c < C  (16-bit, [r_pad,C]).
 * A[r,K] -> down:  src_rs = K, src_cs = 1.    B[N,r] -> B^T padded: src_rs = 1, src_cs = r. */
int lb_cast_rows_pad(const float* src, long long src_rs, long long src_cs, void* dst16, int r,
                     int r_pad, int C, int out_dtype, void* stream);

/* Pivotal-tuning phase 1 (textual inversion) update of the n trained token rows, one launch:
 * AdamW on rows [n,D] (fp32 masters; grad is zeroed), t = ++(*step_dev), then, if clip_decay,
 *   w <- w/||w|| * (||w|| + min(1, 100*lr) * (target_norm - ||w||))        (target_norm = 0.4)
 * and the row is written into table[token_ids[j], :] (LB_F32/LB_BF16/LB_F16). Equivalent to the
 * reference's AdamW over the WHOLE embedding table followed by restoring every untouched row,
 * lora_diffusion/cli_lora_pti.py:448-479. */
int lb_ti_embed_step(float* rows, float* grad, float* m, float* v, const long long* token_ids, void* table,
                     int table_dtype, int n_rows, int D, const float* lr_dev, float beta1, float beta2,
                     float eps, float weight_decay, int* step_dev, int clip_decay, float target_norm,
                     void* stream);

/* ---- sparse, exact AdamW over the token-embedding table (pivotal tuning's `continue_inversion`,
 * train_lora_w_ti.py). The claimed rows are one more param-group of the LoRA arena: `master` and
 * `slot_grad` are that group's [capacity, D] fp32 slices of the arena's p and g, and the unchanged
 * lb_optim_step_fused launch clips and updates them with the LoRA factors. Device-resident state:
 *   slot_of  int32 [V] (token -> slot, -1 = unclaimed), slot_tok int32 [capacity] (slot -> token),
 *   state    int32 [4] {claimed, claimed after this step's scatter, flush ticket (zero), flags},
 *            flags bit 0 = a token found no free slot (sticky; its gradient was dropped),
 *            bit 1 = an id outside [0, V) was skipped,
 *   decay    fp64  [1] product of the per-step decay factors fl32(1 - lr*wd) since the last flush.
 * An unclaimed row's stored value times `decay` is what dense AdamW would hold in it (its gradient
 * and moments are zero, so only the decoupled weight decay has moved it). */

/* Backward of the embedding lookup, one launch (replaces the dense [V, D] gradient autograd builds
 * for text_encoder.get_input_embeddings().weight, cli_lora_pti.py:596-606 / train_lora_w_ti.py:1052):
 * ids int64 [n_tok] (n_tok = B*S <= 2048), grad [n_tok, D] of grad_dtype (LB_F32/LB_BF16/LB_F16).
 * For every distinct token, the gradient rows of its positions are summed in position order (fp32,
 * no atomics: bitwise deterministic) and ADDED to slot_grad[slot]. A token without a slot claims the
 * next one, in first-occurrence order, and its master becomes table[tok] * decay (table_dtype).
 * Reads state[0], writes state[1] (lb_embed_rows_write_back commits it). Past capacity, flag bit 0 is
 * set and that token's gradient is dropped; nothing is written out of bounds. */
int lb_embed_rows_scatter(const long long* ids, const void* grad, int grad_dtype, int n_tok, int D, int V,
                          int* slot_of, int* slot_tok, int capacity, int* state, const void* table,
                          int table_dtype, const double* decay, float* master, float* slot_grad, void* stream);

/* lb_embed_rows_scatter for `world` data-parallel replicas (1 <= world <= 16, 0 <= rank < world), one
 * launch. ids_by_rank: HOST array of `world` device pointers, rank r's ids int64 [n_per_rank]
 * (world * n_per_rank <= 2048); grad [n_per_rank, D] holds this rank's positions only. Slots are
 * claimed over the concatenation [ids of rank 0; ids of rank 1; ...] -- the order of one process
 * running the concatenated batch -- so every rank claims the same slots for the same tokens, tokens
 * seen only on other ranks included (master = table[tok] * decay, no local gradient); only this
 * rank's positions add into slot_grad (the arena's all-reduce sums the ranks). Flag bits are raised
 * identically on every rank (the union is what overflows the capacity).
 * Handshake, for ids that peers write while this launch runs (the other ranks' entries of
 * ids_by_rank are CUDA-IPC mappings): flags_by_rank, a HOST array of `world` device pointers to each
 * rank's one-word uint32 flag (zeroed once; this rank's own entry included), and epoch_dev, two
 * zero-initialised uint32 {epoch, ticket} of this rank. The launch publishes epoch + 1 in its own
 * flag (system-scope release) and waits for every peer's flag to reach it before reading that peer's
 * ids; every rank must launch it the same number of times. Waits are bounded (~20 s) and trap.
 * flags_by_rank = epoch_dev = NULL: the ids are stable for the launch (e.g. all-gathered by NCCL
 * into one buffer beforehand). world = 1 without flags is lb_embed_rows_scatter. */
int lb_embed_rows_scatter_dp(const long long* const* ids_by_rank, int world, int rank, int n_per_rank,
                             const void* grad, int grad_dtype, int D, int V, int* slot_of, int* slot_tok,
                             int capacity, int* state, const void* table, int table_dtype, const double* decay,
                             float* master, float* slot_grad, const unsigned int* const* flags_by_rank,
                             unsigned int* epoch_dev, void* stream);

/* After the optimizer launch, one launch: table[slot_tok[s]] = master[s] (cast to table_dtype) for the
 * first n_write claimed slots (n_write < 0: every claimed slot), state[0] = state[1], and, when decay
 * and lr_dev are given, decay *= (double) fl32(1 - lr_dev[lr_index] * weight_decay) -- the factor the
 * optimizer applied to every row this step. Writing back only the placeholder slots (claimed first)
 * leaves every other row bit-identical, which is train_lora_w_ti.py:1070-1075's restore. */
int lb_embed_rows_write_back(const float* master, const int* slot_tok, int capacity, int* state, int n_write,
                             void* table, int table_dtype, int D, int V, double* decay, const float* lr_dev,
                             int lr_index, float weight_decay, void* stream);

/* One launch over the table: table[row] *= decay for every unclaimed row, then decay = 1. Makes the
 * whole table what dense AdamW (cli_lora_pti.py:958-997, every row decays every step) would hold. */
int lb_embed_rows_flush(void* table, int table_dtype, int V, int D, const int* slot_of, double* decay, int* state,
                        void* stream);

/* Fold a LoRA into its frozen weight: out[n,k] = W[n,k] + alpha * sum_j up[n,j]*down[j,k]
 * (W, out: LB_F32/LB_BF16/LB_F16 [N,K]; conv weights flattened to [Cout, Cin*kh*kw]; out may alias W;
 * 1 <= r <= 64).
 * Replaces the up@down GEMM + add of collapse_lora, lora_diffusion/lora.py:635-669. */
int lb_lora_merge(const void* W, int w_dtype, const float* up, const float* down, float alpha, void* out,
                  int N, int K, int r, void* stream);

/* fp32-faithful mode ("split-bf16"): dst16 [R, 3C] bf16 = three bf16 terms of src [R,C] fp32 side
 * by side along K; pattern 0 (activations) [hi|lo|hi], pattern 1 (weights, factors) [hi|hi|lo], so
 * an ordinary K-major bf16 GEMM over 3C columns evaluates hi*hi + lo*hi + hi*lo (error 2^-16).
 * The fused kernels are then called with K := 3K; nothing else changes. */
int lb_split_bf16x3(const float* src, long long src_rs, void* dst16, int R, int C, int pattern,
                    void* stream);

/* Frozen-weight preparation for LB_W_TILED: the logical [N, K] operand, element (n, k) read from
 * src[n*src_rs + k*src_cs] (W itself: src_rs = K, src_cs = 1; the dX operand W^T of a [N_out, K_in]
 * weight: N = K_in, K = N_out, src_rs = 1, src_cs = K_in), cast to 16 bits and written as 64 x 64 blocks
 * (see LB_W_TILED), zero padded. dst16 holds lb_tiled_weight_elems(N, K) elements, 16-byte aligned. */
long long lb_tiled_weight_elems(int N, int K);
int lb_tile_weight(const void* src, int src_dtype, long long src_rs, long long src_cs, int N, int K,
                   void* dst16, int out_dtype, void* stream);

/* Frozen-weight preparation: src [R,C] (LB_F32/LB_BF16/LB_F16) -> dst16 [R,C] and/or
 * dstT16 [C,R] (either may be NULL). One-time cost per frozen weight. */
int lb_cast_weight(const void* src, int src_dtype, void* dst16, void* dstT16, int R, int C,
                   int out_dtype, void* stream);

/* Global-norm clip + AdamW over one flat fp32 arena, two launches, no host sync.
 *   total = inv_world * ||g||_2 ; coef = min(1, max_norm / (total + 1e-6))  (max_norm <= 0: no clip)
 *   g' = g * inv_world * coef ; decoupled weight decay ; Adam moments ; bias correction with
 *   t = ++(*step_dev) ; g is zeroed for the next step ; *gnorm_out = total.
 * Elements [group_off[i], group_off[i+1]) use lr_dev[i]; group_off is a HOST array of
 * n_groups+1 offsets (n_groups <= 8), lr_dev a DEVICE array (so a captured graph sees scheduler
 * updates), step_dev a DEVICE int. partials: device scratch of >= 1024 floats.
 * Replaces clip_grad_norm_ + torch.optim.AdamW.step + zero_grad,
 * training_scripts/train_lora_dreambooth.py:878-888 and lora_diffusion/cli_lora_pti.py:606-609.
 */
int lb_adamw_clip_step(float* p, float* g, float* m, float* v, long long n,
                       const long long* group_off, int n_groups, const float* lr_dev, float beta1,
                       float beta2, float eps, float weight_decay, float max_norm, float inv_world,
                       int* step_dev, float* partials, float* gnorm_out, void* stream);

/* The whole optimizer step in ONE cooperative launch: lb_adamw_clip_step's two passes plus
 * lb_refresh_shadows (the re-cast of every LoRA factor into the 16-bit [rows, C] operands of the
 * fused kernels; `table` = the rows lb_refresh_shadows walks, n_entries may be 0), separated by
 * grid barriers on `barrier2` (2 x uint32 of device memory, zero-initialised once by the caller).
 * train_lora_dreambooth.py:878-888 (clip_grad_norm_, optimizer.step, zero_grad). */
int lb_optim_step_fused(float* p, float* g, float* m, float* v, long long n,
                        const long long* group_off, int n_groups, const float* lr_dev, float beta1,
                        float beta2, float eps, float weight_decay, float max_norm, float inv_world,
                        int* step_dev, float* partials, float* gnorm_out, const long long* table,
                        int n_entries, int max_C, void* shadow16, int shadow_dtype,
                        unsigned int* barrier2, void* stream);

/* lb_optim_step_fused for `world` data-parallel replicas on one NVLink/NVSwitch node, with the
 * gradient all-reduce INSIDE the launch (no NCCL call; replaces DDP's bucketed all-reduce implied by
 * accelerator.prepare/backward, train_lora_dreambooth.py:744-757,877): after a flag barrier over
 * NVLink every rank sums the flat gradient buffers of all ranks by direct peer reads (fixed rank
 * order => identical sums everywhere), clips on the averaged gradient (DDP order), runs AdamW on its
 * replica, and zeroes its own gradients once every peer has finished reading them.
 * peer_g / peer_flags: HOST arrays of `world` device pointers in rank order (the entries of the
 * other ranks are CUDA-IPC mappings of their `g` / flag buffers; flags = 2*world uint32, zeroed
 * once); gsum: n floats of scratch; epoch_dev: one zero-initialised uint32. Must be launched by
 * every rank the same number of times. Waits are bounded (~20 s) and trap. */
int lb_optim_step_dp(float* p, float* g, float* gsum, float* m, float* v, long long n,
                     const long long* group_off, int n_groups, const float* lr_dev, float beta1,
                     float beta2, float eps, float weight_decay, float max_norm, int* step_dev,
                     float* partials, float* gnorm_out, const long long* table, int n_entries,
                     int max_C, void* shadow16, int shadow_dtype, unsigned int* barrier2,
                     const void* const* peer_g, void* const* peer_flags, int world, int rank,
                     unsigned int* epoch_dev, void* stream);

/* CUDA-IPC helpers for the peer mappings of lb_optim_step_dp. lb_ipc_export: `ptr` (anywhere inside
 * a cudaMalloc'ed block) -> 64-byte IPC handle of the block + byte offset of ptr inside it.
 * lb_ipc_open (in another process of the node, once per distinct handle): -> the block's base address
 * in this process; enables peer access from the current device to the exporter's. */
int lb_ipc_export(const void* ptr, void* handle64, long long* offset);
int lb_ipc_open(const void* handle64, void** base_out);

/* Batched 16-bit shadow refresh after an optimizer step: for every table entry e, j < e.rows, c < e.C
 *   dst16_base[e.dst_off + j*e.dst_rs + c] = (j < e.r) ? p[e.src_off + j*e.src_rs + c*e.src_cs] : 0
 * table: DEVICE array of n_entries x 8 long long {src_off, src_rs, src_cs, r, C, dst_off, dst_rs, rows}
 * (conv down factors use one entry per filter tap so that K is ordered tap-major, channel-minor).
 * The table is not checked: `rows` must be 16, 32 or 64, r <= rows, and the destination slot must
 * hold `rows` rows of pitch dst_rs (rows * dst_rs elements from dst_off) -- a larger `rows` writes
 * past the slot. lb_optim_step_fused and lb_optim_step_dp walk the same table. */
int lb_refresh_shadows(const float* p, const long long* table, int n_entries, int max_C,
                       void* dst16_base, int out_dtype, void* stream);

/* ---- batched truncated SVD for LoRA distillation (replaces the serial torch.linalg.svd loop of
 * lora_diffusion/cli_svd.py:24-92). Randomized range finder with 32 probe vectors on
 * dW[b] = Wt[b] - Wb[b] (N x K, row-major, LB_F32/LB_BF16/LB_F16). Wt/Wb are DEVICE arrays of `batch` device pointers to same-shape
 * matrices. Tall-skinny operands are fp32 row-major [batch, rows, 32]. See lora_b200/svd.py for
 * the driver (probe -> power iterations with CholeskyQR2 -> 32x32 Jacobi -> factors). */
/* SVD distillation of cli_svd.py:24-92 (`overwrite_base`) for ALL sites of a model in one call,
 * ragged over shapes: for b < batch,
 *   dW = Wt[b] - Wb[b]  ([N[b], K[b]] row-major, w_dtype in {LB_F32, LB_BF16, LB_F16}; Wb NULL or
 *   Wb[b] ignored when the array is NULL: dW = Wt[b]) -> top-`rank` singular triplets by a
 *   randomized range finder (32 probes, `power_iters` power iterations = 2*power_iters+2 streaming
 *   passes over both weights, contraction on the tensor cores in 3-term split-bf16) ->
 *   out[off_b ...] = [ up = U_r diag(S_r) as [N, rank] | down = Vh_r as [rank, K] ] fp32, with
 *   off_b = rank * sum_{c<b} (N[c] + K[c]); sigma_out[b, 0..31] (descending; may be NULL);
 *   clamp_q > 0: both factors clamped to +-torch.quantile(cat(up, down), clamp_q) (exact order
 *   statistics, cli_svd.py:43-47), the threshold reported in hi_out[b] (may be NULL).
 * All array arguments are HOST arrays; workspace is device memory of at least
 * lb_svd_workspace_bytes(N, K, batch, w_dtype) bytes. K[b] must keep rows 16-byte aligned. */
long long lb_svd_workspace_bytes(const int* N, const int* K, int batch, int w_dtype);
int lb_svd_truncated_batched(const void* const* Wt, const void* const* Wb, const int* N, const int* K,
                             int batch, int w_dtype, int rank, int power_iters, float clamp_q,
                             unsigned long long seed, float* out, float* sigma_out, float* hi_out,
                             void* workspace, long long workspace_bytes, void* stream);

/* transpose = 0: out[b] (N x 32) = dW[b] . in[b] (K x 32);  1: out[b] (K x 32) = dW[b]^T . in[b] (N x 32) */
int lb_svd_mul(const void* const* Wt, const void* const* Wb, int w_dtype, const float* in, float* out,
               int N, int K, int batch, int transpose, void* stream);
/* G[b] (32x32) = Y[b]^T Y[b] */
int lb_svd_gram(const float* Y, float* G, int rows, int batch, void* stream);
/* G = R^T R (upper R, tiny ridge) -> Rinv[b] = R^-1 (32x32) */
int lb_svd_chol_inv(const float* G, float* Rinv, int batch, void* stream);
/* out[b] = Y[b] (rows x 32) . M[b] (32x32), first out_cols columns, optionally column-scaled
 * (scale_mode 1: * colscale[b][j], 2: / colscale[b][j]); out may alias Y; transposed = 1 writes
 * out[b][j*out_pitch + row]. */
int lb_svd_apply(const float* Y, const float* M, const float* colscale, int scale_mode, float* out,
                 int rows, int out_cols, long long out_pitch, int transposed,
                 long long out_batch_stride, int batch, void* stream);
/* symmetric 32x32 eigen-decomposition (cyclic Jacobi): V columns sorted by descending eigenvalue,
 * sigma = sqrt(max(eig, 0)) */
int lb_svd_jacobi(const float* G, float* V, float* sigma, int batch, int sweeps, void* stream);
/* standard-normal probes from a counter hash */
int lb_svd_randn(float* out, long long n, unsigned long long seed, void* stream);

/* Step prologue, one launch (cli_lora_pti.py:295-313, train_lora_dreambooth.py:822-840):
 *   out[b, h, w, c] = sqrt_acp[t_b] * latents[b, c, h, w] + sqrt_one_minus_acp[t_b] * noise[b, c, h, w]
 * latents / noise fp32 NCHW, timesteps int64 [B], out NHWC (a channels_last [B, C', H, W] tensor) of
 * out_dtype. With inpaint_mask [B,1,H,W] and masked_latents [B,C,H,W] (both or neither): C' = 2C + 1,
 * out = cat([noisy, mask, masked_latents], channel) -- the 9-channel inpainting input. */
int lb_step_prologue(const float* latents, const float* noise, const long long* timesteps,
                     const float* sqrt_acp, const float* sqrt_one_minus_acp, int n_timesteps,
                     const float* inpaint_mask, const float* masked_latents, void* out, int out_dtype,
                     int B, int C, int H, int W, void* stream);

/* lb_step_prologue plus the v-prediction target of the same timesteps (cli_lora_pti.py:333-338,
 * diffusers' DDPMScheduler.get_velocity), in the same launch:
 *   velocity[b, c, h, w] = sqrt_acp[t_b] * noise[b, c, h, w] - sqrt_one_minus_acp[t_b] * latents[b, c, h, w]
 * fp32 NCHW (the target layout lb_masked_mse_fwd_bwd reads), two rounded products and one rounded
 * difference: equal to torch's evaluation bit for bit. velocity NULL: LB_ERR_SHAPE. */
int lb_step_prologue_v(const float* latents, const float* noise, const long long* timesteps,
                       const float* sqrt_acp, const float* sqrt_one_minus_acp, int n_timesteps,
                       const float* inpaint_mask, const float* masked_latents, void* out, int out_dtype,
                       float* velocity, int B, int C, int H, int W, void* stream);

/* Loss epilogue, one launch (cli_lora_pti.py:340-370, train_lora_dreambooth.py:855-875):
 *   loss = sum_b weights[b] * mean_{c,h,w} (mask[b,h,w] * (pred - target))^2      (weights NULL: 1/B)
 *   grad = d loss / d pred = 2 weights[b] mask^2 (pred - target) / (C H W)        (pred's dtype/layout)
 * pred element (b, c, pixel) at b*stride_b + c*stride_c + pixel*stride_p (NCHW or channels_last);
 * target fp32 NCHW; mask [B,1,H,W] fp32 (already normalised as in cli_lora_pti.py:356-364) or NULL.
 * partials64: >= 64 floats of scratch; counter: one zero-initialised uint32 (self-resetting). */
int lb_masked_mse_fwd_bwd(const void* pred, int pred_dtype, long long stride_b, long long stride_c,
                          long long stride_p, const float* target, const float* mask,
                          const float* weights, void* grad, float* loss, float* partials64,
                          unsigned int* counter, int B, int C, int H, int W, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LORA_B200_H */
