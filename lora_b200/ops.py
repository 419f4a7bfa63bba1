"""Tensor-level wrappers over the C-ABI (lora_b200._C) and the autograd glue.

torch is used for device memory, streams and autograd bookkeeping only; all arithmetic of the
LoRA path happens in liblora_b200.so. There is deliberately no eager fallback in this module.
"""
from typing import Optional, Tuple

import os

import torch

from . import _C
from ._C import check, dtype_code, ptr, stream_ptr

R_PAD = 16
MAX_RANK = 64      # widest rank the fused kernels run natively (rank pads 16, 32, 64)
LAUNCH_COUNT = 0  # kernels of liblora_b200.so enqueued through this process (bench.py reads it)


def rank_pad(r: int) -> int:
    """Rows of the zero-padded rank operands for a rank-r site: 16, 32 or 64 (r <= 64)."""
    if not 1 <= r <= MAX_RANK:
        raise _C.LoraB200Error(f"LoRA rank {r} outside 1..{MAX_RANK} of the fused kernels")
    return 16 if r <= 16 else (32 if r <= 32 else 64)


def _count(n: int = 1):
    global LAUNCH_COUNT
    LAUNCH_COUNT += n


# Deferred factor gradients: dA / dB feed only the optimizer, so (when they accumulate straight into
# an arena) a step engine can QUEUE every linear-site reduction of the backward pass and run them
# all in ceil(n/24) launches at its end (lb_lora_wgrad_batch) instead of one small launch per site.
# The queue keeps the operand tensors alive until the flush; under gradient checkpointing it is also
# flushed when the next segment's recompute starts (wgrad_segment_boundary).
import ctypes as _ct


class _WgProblemC(_ct.Structure):
    _fields_ = [("S", _ct.c_void_p), ("V", _ct.c_void_p), ("out", _ct.c_void_p),
                ("out_js", _ct.c_longlong), ("out_cs", _ct.c_longlong),
                ("M", _ct.c_int), ("C", _ct.c_int), ("r", _ct.c_int), ("scale", _ct.c_float),
                ("diag", _ct.c_void_p), ("drop_p", _ct.c_float), ("seed_dev", _ct.c_void_p),
                ("conv_H", _ct.c_int), ("conv_W", _ct.c_int), ("kh", _ct.c_int), ("kw", _ct.c_int),
                ("pad_h", _ct.c_int), ("pad_w", _ct.c_int), ("r_pad", _ct.c_int)]


_WG_QUEUE = None      # None: launch immediately; dict dtype -> [(_WgProblemC fields, keepalive)]
WG_BATCH = 24


def wgrad_defer_begin():
    global _WG_QUEUE
    _WG_QUEUE = {}


def wgrad_defer_cancel():
    global _WG_QUEUE
    _WG_QUEUE = None


def _wgrad_launch(dtype, items):
    arr = (_WgProblemC * len(items))(*[_WgProblemC(*it[0]) for it in items])
    check(_C.lib.lb_lora_wgrad_batch(arr, len(items), dtype_code(dtype), stream_ptr()), "lb_lora_wgrad_batch")
    n =(len(items) + WG_BATCH - 1) // WG_BATCH
    _count(n)
    return n


def _wgrad_enqueue(S, V, out, out_js, out_cs, M, C, r, scale, diag, drop_p=0.0, seed=None, conv=None):
    dp = lambda t: None if t is None else t.data_ptr()
    item = (dp(S), dp(V), dp(out), int(out_js), int(out_cs), int(M), int(C), int(r), float(scale), dp(diag),
            float(drop_p), dp(seed)) + (tuple(int(v) for v in conv) if conv is not None else (0, 0, 0, 0, 0, 0)) + (
            int(V.shape[1]),)
    _WG_QUEUE.setdefault(S.dtype, []).append((item, (S, V, out, diag, seed)))


def _wgrad_launch_all(q) -> int:
    n_launch = 0
    for dtype, items in q.items():
        if items:
            n_launch += _wgrad_launch(dtype, items)
    return n_launch


def wgrad_flush():
    """Run every queued reduction (lb_lora_wgrad_batch) and leave deferral mode."""
    global _WG_QUEUE
    q, _WG_QUEUE = _WG_QUEUE, None
    if not q:
        return 0
    return _wgrad_launch_all(q)


def wgrad_segment_boundary() -> int:
    """Called by every LoRA site's forward. A forward that runs inside the backward pass is a
    gradient-checkpointing recompute, so the backward of the segment checkpointed before it (later
    in the forward order) has finished: run what the queue holds now and keep deferring. The queue
    then never keeps one segment's recomputed activations alive while the next one is recomputed;
    the step takes about one batched launch per checkpointed segment with LoRA sites instead of
    ceil(n/24). Without checkpointing no site forward runs during backward and nothing changes."""
    global _WG_QUEUE
    if not _WG_QUEUE or torch._C._current_graph_task_id() == -1:
        return 0
    q, _WG_QUEUE = _WG_QUEUE, {}
    return _wgrad_launch_all(q)


def _req_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _C.LoraB200Error("lora_b200 kernels need CUDA tensors (no CPU path)")


def cast_rows_pad16(src: torch.Tensor, rs: int, cs: int, r: int, C: int, dtype,
                    out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 factor -> zero-padded 16-bit [rank_pad(r), C] operand (see lb_cast_rows_pad); `out`: re-cast
    into that existing operand in place."""
    _req_cuda(src)
    if out is None:
        out = torch.empty((rank_pad(r) if r >= 1 else R_PAD, C), device=src.device, dtype=dtype)
    check(_C.lib.lb_cast_rows_pad(ptr(src), rs, cs, ptr(out), r, out.shape[0], C, dtype_code(dtype), stream_ptr()),
          "lb_cast_rows_pad")
    _count()
    return out


def cast_weight(w: torch.Tensor, dtype, want_plain: bool, want_t: bool):
    """Frozen weight [R,C] -> (16-bit copy or None, 16-bit transpose [C,R] or None)."""
    _req_cuda(w)
    if not want_plain and not want_t:
        return None, None
    w = w.detach()
    if not w.is_contiguous():
        w = w.contiguous()
    R, C = w.shape
    plain = torch.empty((R, C), device=w.device, dtype=dtype) if want_plain else None
    wt = torch.empty((C, R), device=w.device, dtype=dtype) if want_t else None
    check(_C.lib.lb_cast_weight(ptr(w), dtype_code(w.dtype), ptr(plain), ptr(wt), R, C,
                                dtype_code(dtype), stream_ptr()), "lb_cast_weight")
    _count()
    return plain, wt


LB_W_TILED = 0x100
# LB_TILED_W=1: the module layer (modules._SiteState.frozen) keeps its frozen-weight copies in the
# 64x64-block layout. OFF by default: it costs a second copy of every 16-bit frozen weight, and DRAM
# page locality of the weight stream is not what limits these kernels.
TILED_WEIGHTS = os.environ.get("LB_TILED_W", "0") == "1"

class TiledWeight:
    """A frozen weight's 16-bit copy in the 64 x 64-block layout (include/lora_b200.h, LB_W_TILED):
    logical operand [N, K]; accepted wherever the fused linear entries take `w16` / `wt16`."""
    __slots__ = ("buf", "N", "K", "dtype")

    def __init__(self, buf, N, K, dtype):
        self.buf, self.N, self.K, self.dtype = buf, N, K, dtype

    @property
    def shape(self):
        return (self.N, self.K)

    def data_ptr(self):
        return self.buf.data_ptr()


def tile_weight(w: torch.Tensor, dtype, transpose: bool = False) -> TiledWeight:
    """lb_tile_weight: w [R, C] (fp32/bf16/fp16, CUDA, contiguous) -> TiledWeight of w (logical [R, C]) or,
    transpose=True, of w^T (logical [C, R]: the dX operand)."""
    _req_cuda(w)
    assert w.dim() == 2 and w.is_contiguous()
    R, C = w.shape
    N, K = (C, R) if transpose else (R, C)
    rs, cs = (1, C) if transpose else (C, 1)
    n = int(_C.lib.lb_tiled_weight_elems(N, K))
    buf = torch.empty(n, device=w.device, dtype=dtype)
    check(_C.lib.lb_tile_weight(ptr(w), dtype_code(w.dtype), rs, cs, N, K, ptr(buf), dtype_code(dtype), stream_ptr()),
          "lb_tile_weight")
    _count()
    return TiledWeight(buf, N, K, dtype)


def _w_arg(w16, K):
    """(pointer, N, in_dtype flag) of a frozen-weight argument: row-major tensor or TiledWeight."""
    if isinstance(w16, TiledWeight):
        assert w16.K == K
        return ptr(w16.buf), w16.N, LB_W_TILED
    assert w16.shape[1] == K and w16.is_contiguous()
    return ptr(w16), w16.shape[0], 0


def _coef_args(coef_rows, r: int):
    """(table, ld, rows_per_sample, S) of a per-sample coefficient argument, checked."""
    table, ld, rps, S = coef_rows
    _req_cuda(table)
    ld, rps, S = int(ld), int(rps), int(S)
    assert table.dtype == torch.float32 and ld >= r and rps >= 1 and S >= 1
    # row b of the table starts b * ld elements in: a 2-D table must have that row pitch
    assert table.dim() in (1, 2) and table.stride(-1) == 1 and (table.dim() == 1 or table.stride(0) == ld)
    assert table.numel() >= (S - 1) * ld + r
    return table, ld, rps, S


def fused_linear(x2d: torch.Tensor, w16: torch.Tensor, bias: Optional[torch.Tensor],
                 down16: torch.Tensor, up: torch.Tensor, up_rs: int, up_cs: int,
                 diag: Optional[torch.Tensor], scale: float, r: int, out_dtype,
                 want_t: bool, t_in: Optional[torch.Tensor] = None, drop_p: float = 0.0,
                 seed: Optional[torch.Tensor] = None, coef_rows=None
                 ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """Y = x2d.w16^T + bias + ((x2d.down16^T) * scale*diag) . up^T ; returns (Y, T or None).
    down16: [RP, K] with RP = 16, 32 or 64 rows (the rank pad); T is [M, RP].
    t_in: use these rank-r activations [M,RP] instead of x2d.down16^T (dropout backward).
    drop_p > 0 (+ seed: int64[1] on the device): nn.Dropout on the branch, masked in the drain.
    coef_rows = (table fp32 [S, ld] on the device, ld, rows_per_sample, S): per-sample coefficients in
    place of scale*diag (lb_lora_linear_fwd_ps; row m takes table row (m // rows_per_sample) % S).
    Forward only: no T, t_in or dropout; diag and scale are ignored."""
    _req_cuda(x2d, down16, up)
    M, K = x2d.shape
    wp, N, wflag = _w_arg(w16, K)
    rp = down16.shape[0]
    assert down16.shape == (rp, K) and rp in (16, 32, 64)
    assert x2d.is_contiguous() and down16.is_contiguous()
    if coef_rows is not None:
        assert not want_t and t_in is None and drop_p == 0.0, "per-sample coefficients: forward only"
        table, ld, rps, S = _coef_args(coef_rows, r)
        y = torch.empty((M, N), device=x2d.device, dtype=out_dtype)
        check(_C.lib.lb_lora_linear_fwd_ps(ptr(x2d), wp, ptr(bias), ptr(down16), ptr(up), up_rs, up_cs,
                                           ptr(table), ld, rps, S, ptr(y), M, K, N, r, rp,
                                           dtype_code(x2d.dtype) | wflag, dtype_code(out_dtype), stream_ptr()),
              "lb_lora_linear_fwd_ps")
        _count()
        return y, None
    y = torch.empty((M, N), device=x2d.device, dtype=out_dtype)
    t = torch.empty((M, rp), device=x2d.device, dtype=torch.float32) if want_t else None
    assert t_in is None or t_in.shape == (M, rp)
    if drop_p > 0.0:
        assert t_in is None and seed is not None and seed.dtype == torch.int64 and seed.is_cuda
        check(_C.lib.lb_lora_linear_fwd_dropout(ptr(x2d), wp, ptr(bias), ptr(down16), ptr(up),
                                                up_rs, up_cs, ptr(diag), float(scale), ptr(y), ptr(t),
                                                M, K, N, r, rp, dtype_code(x2d.dtype) | wflag,
                                                dtype_code(out_dtype), float(drop_p), ptr(seed), stream_ptr()),
              "lb_lora_linear_fwd_dropout")
    else:
        check(_C.lib.lb_lora_linear_fwd(ptr(x2d), wp, ptr(bias), ptr(down16), ptr(up),
                                        up_rs, up_cs, ptr(diag), float(scale), ptr(y), ptr(t), ptr(t_in),
                                        M, K, N, r, rp, dtype_code(x2d.dtype) | wflag, dtype_code(out_dtype),
                                        stream_ptr()), "lb_lora_linear_fwd")
    _count()
    return y, t


def wgrad(S: torch.Tensor, V: torch.Tensor, diag: Optional[torch.Tensor], scale: float,
          out: torch.Tensor, out_js: int, out_cs: int, r: int, deferrable: bool = False):
    """out[j*out_js + c*out_cs] += scale*diag[j] * sum_m V[m,j]*S[m,c]."""
    _req_cuda(S, V, out)
    M, C = S.shape
    rp = V.shape[1]
    assert S.is_contiguous() and V.shape == (M, rp) and V.dtype == torch.float32
    assert out.dtype == torch.float32
    if _WG_QUEUE is not None and deferrable:
        _wgrad_enqueue(S, V, out, out_js, out_cs, M, C, r, scale, diag)
        return
    check(_C.lib.lb_lora_wgrad(ptr(S), ptr(V), ptr(diag), float(scale), ptr(out), out_js, out_cs,
                               M, C, r, rp, dtype_code(S.dtype), stream_ptr()), "lb_lora_wgrad")
    _count()


# ------------------------------------------------------------------------------------ conv path
def cast_conv_weight(w: torch.Tensor, dtype, want_fwd: bool, want_bwd: bool):
    """Frozen conv weight [Cout,Cin,kh,kw] -> (forward operand [Cout, kh*kw*Cin] or None,
    flipped+transposed input-gradient operand [Cin, kh*kw*Cout] or None)."""
    _req_cuda(w)
    if not want_fwd and not want_bwd:
        return None, None
    w = w.detach().contiguous()
    cout, cin, kh, kw = w.shape
    f = torch.empty((cout, kh * kw * cin), device=w.device, dtype=dtype) if want_fwd else None
    b = torch.empty((cin, kh * kw * cout), device=w.device, dtype=dtype) if want_bwd else None
    check(_C.lib.lb_cast_conv_weight(ptr(w), dtype_code(w.dtype), ptr(f), ptr(b), cout, cin, kh, kw,
                                     dtype_code(dtype), stream_ptr()), "lb_cast_conv_weight")
    _count()
    return f, b


def conv_tap_rows(src_off: int, dst_off: int, r: int, cin: int, taps: int, rp: int):
    """lb_refresh_shadows rows that re-cast a conv down factor A [r,Cin,kh,kw] (fp32, `src_off` elements
    into the source) to its [rp, taps*Cin] 16-bit operand (`dst_off` into the destination), whose K
    index is tap-major, channel-minor: one row per tap."""
    return [(src_off + t, cin * taps, taps, r, cin, dst_off + t * cin, taps * cin, rp) for t in range(taps)]


def conv_tap_table(a4d: torch.Tensor, table_cache: dict) -> torch.Tensor:
    """conv_down16's row table for a down factor shaped like a4d, built once per shape and device
    into `table_cache` (an upload: build it before a graph capture that re-casts through it)."""
    r, cin, kh, kw = a4d.shape
    key = (r, cin, kh * kw, a4d.device)
    tab = table_cache.get(key)
    if tab is None:
        tab = torch.tensor(conv_tap_rows(0, 0, r, cin, kh * kw, rank_pad(r)), device=a4d.device, dtype=torch.int64)
        table_cache[key] = tab
    return tab


def conv_down16(a4d: torch.Tensor, dtype, table_cache: dict, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """A [r,Cin,kh,kw] fp32 -> [rank_pad(r), kh*kw*Cin] 16-bit with K ordered tap-major, channel-minor;
    `out`: re-cast into that existing operand in place."""
    _req_cuda(a4d)
    r, cin, kh, kw = a4d.shape
    tab = conv_tap_table(a4d, table_cache)
    src = a4d.detach()
    if src.dtype != torch.float32 or not src.is_contiguous():
        src = src.float().contiguous()
    if out is None:
        out = torch.empty((rank_pad(r), kh * kw * cin), device=a4d.device, dtype=dtype)
    check(_C.lib.lb_refresh_shadows(ptr(src), ptr(tab), kh * kw, cin, ptr(out), dtype_code(dtype), stream_ptr()),
          "lb_refresh_shadows")
    _count()
    return out


def fused_conv2d(x_nhwc: torch.Tensor, w16: torch.Tensor, bias: Optional[torch.Tensor],
                 down16: torch.Tensor, up: torch.Tensor, up_off: int, up_rs: int, up_cs: int,
                 up_gs: int, diag: Optional[torch.Tensor], scale: float, r: int, cout: int,
                 kh: int, kw: int, pad_h: int, pad_w: int, per_tap: bool, out_dtype,
                 want_t: bool, t_in: Optional[torch.Tensor] = None, drop_p: float = 0.0,
                 seed: Optional[torch.Tensor] = None, coef_rows=None
                 ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """x_nhwc: a [N,C,H,W] tensor in channels_last memory format (NHWC bytes). Returns
    (Y as [N,cout,H,W] channels_last, T [N*H*W,RP] or None); RP = down16.shape[0] (16, 32 or 64).
    coef_rows: per-sample coefficients as in fused_linear, pixel rows (img*H + h)*W + w
    (lb_lora_conv2d_fwd_ps; forward direction only: no T, t_in, dropout or per-tap form)."""
    _req_cuda(x_nhwc, w16, down16, up)
    n, cin, h, w = x_nhwc.shape
    rp = down16.shape[0]
    assert x_nhwc.is_contiguous(memory_format=torch.channels_last) and rp in (16, 32, 64)
    y = torch.empty((n, cout, h, w), device=x_nhwc.device, dtype=out_dtype,
                    memory_format=torch.channels_last)
    t = torch.empty((n * h * w, rp), device=x_nhwc.device, dtype=torch.float32) if want_t else None
    import ctypes
    up_ptr = ctypes.c_void_p(up.data_ptr() + 4 * up_off)
    if coef_rows is not None:
        assert not want_t and t_in is None and drop_p == 0.0 and not per_tap and up_gs == 0
        table, ld, rps, S = _coef_args(coef_rows, r)
        check(_C.lib.lb_lora_conv2d_fwd_ps(ptr(x_nhwc), ptr(w16), ptr(bias), ptr(down16), up_ptr, up_rs, up_cs,
                                           ptr(table), ld, rps, S, ptr(y), n, h, w, cin, cout, kh, kw, pad_h, pad_w,
                                           r, rp, dtype_code(x_nhwc.dtype), dtype_code(out_dtype), stream_ptr()),
              "lb_lora_conv2d_fwd_ps")
    elif drop_p > 0.0:     # forward with nn.Dropout on the branch: masked in the drain, one launch
        assert t_in is None and not per_tap and up_gs == 0 and seed is not None and seed.dtype == torch.int64
        check(_C.lib.lb_lora_conv2d_fwd_dropout(ptr(x_nhwc), ptr(w16), ptr(bias), ptr(down16), up_ptr, up_rs,
                                                up_cs, ptr(diag), float(scale), ptr(y), ptr(t), n, h, w,
                                                cin, cout, kh, kw, pad_h, pad_w, r, rp, dtype_code(x_nhwc.dtype),
                                                dtype_code(out_dtype), float(drop_p), ptr(seed), stream_ptr()),
              "lb_lora_conv2d_fwd_dropout")
    else:
        check(_C.lib.lb_lora_conv2d_fwd(ptr(x_nhwc), ptr(w16), ptr(bias), ptr(down16), up_ptr, up_rs,
                                        up_cs, up_gs, ptr(diag), float(scale), ptr(y), ptr(t), ptr(t_in),
                                        n, h, w, cin, cout, kh, kw, pad_h, pad_w, r, rp, 1 if per_tap else 0,
                                        dtype_code(x_nhwc.dtype), dtype_code(out_dtype), stream_ptr()),
              "lb_lora_conv2d_fwd")
    _count()
    return y, t


# ------------------------------------------------------------------------------------ dropout
def up_dropout_(y2d: torch.Tensor, T: torch.Tensor, up: torch.Tensor, up_rs: int, up_cs: int,
                diag, scale: float, p: float, seed: torch.Tensor, r: int):
    """y2d[m,n] += scale/(1-p) * keep(m,n) * sum_j T[m,j] diag[j] up[n,j]   (in place)."""
    _req_cuda(y2d, T, up, seed)
    M, N = y2d.shape
    rp = T.shape[1]
    assert y2d.is_contiguous() and seed.dtype == torch.int64
    check(_C.lib.lb_lora_up_dropout(ptr(y2d), dtype_code(y2d.dtype), ptr(T), ptr(up), up_rs, up_cs,
                                    ptr(diag), float(scale), float(p), ptr(seed), M, N, r, rp,
                                    stream_ptr()), "lb_lora_up_dropout")
    _count()


def dropout_dt(gy2d: torch.Tensor, up: torch.Tensor, up_rs: int, up_cs: int, p: float,
               seed: torch.Tensor, r: int) -> torch.Tensor:
    """dTs[m,j] = sum_n keep(m,n)/(1-p) * gY[m,n] * up[n,j]  (fp32 [M,rank_pad(r)])."""
    _req_cuda(gy2d, up, seed)
    M, N = gy2d.shape
    rp = rank_pad(r)
    out = torch.empty((M, rp), device=gy2d.device, dtype=torch.float32)
    check(_C.lib.lb_lora_dropout_dt(ptr(gy2d), dtype_code(gy2d.dtype), ptr(up), up_rs, up_cs,
                                    float(p), ptr(seed), ptr(out), M, N, r, rp, stream_ptr()),
          "lb_lora_dropout_dt")
    _count()
    return out


def wgrad_masked(S: torch.Tensor, V: torch.Tensor, diag, scale: float, out: torch.Tensor,
                 out_js: int, out_cs: int, r: int, p: float, seed: torch.Tensor, deferrable: bool = False):
    _req_cuda(S, V, out, seed)
    M, C = S.shape
    if _WG_QUEUE is not None and deferrable:
        _wgrad_enqueue(S, V, out, out_js, out_cs, M, C, r, scale, diag, p, seed)
        return
    rp = V.shape[1]
    check(_C.lib.lb_lora_wgrad_masked(ptr(S), ptr(V), ptr(diag), float(scale), ptr(out), out_js,
                                      out_cs, M, C, r, rp, float(p), ptr(seed), dtype_code(S.dtype),
                                      stream_ptr()), "lb_lora_wgrad_masked")
    _count()


def wgrad_pair(x2d: torch.Tensor, dTs: torch.Tensor, dA: torch.Tensor, gy2d: torch.Tensor,
               T: torch.Tensor, dB: torch.Tensor, diag, scale: float, r: int, p: float = 0.0,
               seed: Optional[torch.Tensor] = None, deferrable: bool = False):
    """dA [r,K] += s*d * dTs^T x2d  and  dB [N,r] += s*d * (mask o gy2d)^T T  in one launch."""
    _req_cuda(x2d, dTs, dA, gy2d, T, dB)
    M, K = x2d.shape
    N = gy2d.shape[1]
    assert gy2d.shape[0] == M and dA.dtype == torch.float32 and dB.dtype == torch.float32
    if _WG_QUEUE is not None and deferrable:
        _wgrad_enqueue(x2d, dTs, dA, K, 1, M, K, r, scale, diag)
        _wgrad_enqueue(gy2d, T, dB, 1, r, M, N, r, scale, diag, p, seed)
        return
    rp = dTs.shape[1]
    assert T.shape[1] == rp
    check(_C.lib.lb_lora_wgrad_pair(ptr(x2d), ptr(dTs), ptr(dA), K, 1, K, ptr(gy2d), ptr(T), ptr(dB),
                                    1, r, N, ptr(diag), float(scale), M, r, rp, float(p), ptr(seed),
                                    dtype_code(x2d.dtype), stream_ptr()), "lb_lora_wgrad_pair")
    _count()


def merge_lora(W: torch.Tensor, up: torch.Tensor, down: torch.Tensor, alpha: float) -> torch.Tensor:
    """W + alpha * up.flatten(1) @ down.flatten(1), same shape/dtype as W (new tensor)."""
    _req_cuda(W, up, down)
    w2 = W.detach().contiguous()
    N = w2.shape[0]
    K = w2.numel() // N
    r = down.shape[0]
    u = up.detach().reshape(N, r).float().contiguous()
    d = down.detach().reshape(r, K).float().contiguous()
    out = torch.empty_like(w2)
    check(_C.lib.lb_lora_merge(ptr(w2), dtype_code(w2.dtype), ptr(u), ptr(d), float(alpha), ptr(out), N, K, r,
                               stream_ptr()), "lb_lora_merge")
    _count()
    return out


def fused_linear_grouped(problems, out_dtype, want_t: bool, coef_rows=None):
    """problems: list (<= 4) of (x2d, w16, bias32|None, down16, up32, up_rs, up_cs, diag|None, scale, r).
    One launch; returns ([Y_i], [T_i or None]). coef_rows: one (table, ld, rows_per_sample, S) per
    problem, per-sample coefficients as in fused_linear (lb_lora_linear_fwd_grouped_ps; forward only)."""
    import ctypes
    n = len(problems)
    assert 1 <= n <= 4
    assert coef_rows is None or (len(coef_rows) == n and not want_t)
    if any(p[3].shape[0] != R_PAD for p in problems):
        # the grouped kernel is built for rank pad 16 only (grouping.py groups only r <= 16 sites);
        # other callers with wider problems (bench.py's kernel sweep at --rank 32) get one launch each
        outs = [fused_linear(x, w, b, d, up, rs, cs, diag, sc, r, out_dtype, want_t,
                             coef_rows=None if coef_rows is None else coef_rows[i])
                for i, (x, w, b, d, up, rs, cs, diag, sc, r) in enumerate(problems)]
        return [o[0] for o in outs], [o[1] for o in outs]
    VP, LL, I, F = ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_float
    ys, ts = [], []
    tiled = isinstance(problems[0][1], TiledWeight)
    for (x, w, b, d, up, rs, cs, diag, sc, r) in problems:
        _req_cuda(x, d, up)
        assert isinstance(w, TiledWeight) == tiled, "a grouped launch takes one weight layout"
        assert x.is_contiguous() and (tiled or w.is_contiguous()) and d.is_contiguous() and w.shape[1] == x.shape[1]
        ys.append(torch.empty((x.shape[0], w.shape[0]), device=x.device, dtype=out_dtype))
        ts.append(torch.empty((x.shape[0], R_PAD), device=x.device, dtype=torch.float32) if want_t else None)
    dp = lambda t: None if t is None else t.data_ptr()
    arr = lambda ty, vals: (ty * n)(*vals)
    X = arr(VP, [p[0].data_ptr() for p in problems])
    W = arr(VP, [p[1].data_ptr() for p in problems])
    B = arr(VP, [dp(p[2]) for p in problems])
    D = arr(VP, [p[3].data_ptr() for p in problems])
    U = arr(VP, [p[4].data_ptr() for p in problems])
    RS = arr(LL, [p[5] for p in problems])
    CS = arr(LL, [p[6] for p in problems])
    DG = arr(VP, [dp(p[7]) for p in problems])
    SC = arr(F, [float(p[8]) for p in problems])
    Y = arr(VP, [y.data_ptr() for y in ys])
    T = arr(VP, [dp(t) for t in ts])
    M = arr(I, [p[0].shape[0] for p in problems])
    K = arr(I, [p[0].shape[1] for p in problems])
    N = arr(I, [p[1].shape[0] for p in problems])
    R = arr(I, [p[9] for p in problems])
    if coef_rows is not None:
        cargs = [_coef_args(c, p[9]) for c, p in zip(coef_rows, problems)]
        check(_C.lib.lb_lora_linear_fwd_grouped_ps(
            n, X, W, B, D, U, RS, CS, arr(VP, [c[0].data_ptr() for c in cargs]), arr(I, [c[1] for c in cargs]),
            arr(I, [c[2] for c in cargs]), arr(I, [c[3] for c in cargs]), Y, M, K, N, R,
            dtype_code(problems[0][0].dtype) | (LB_W_TILED if tiled else 0), dtype_code(out_dtype), stream_ptr()),
            "lb_lora_linear_fwd_grouped_ps")
        _count()
        return ys, ts
    check(_C.lib.lb_lora_linear_fwd_grouped(n, X, W, B, D, U, RS, CS, DG, SC, Y, T, M, K, N, R,
                                            dtype_code(problems[0][0].dtype) | (LB_W_TILED if tiled else 0),
                                            dtype_code(out_dtype), stream_ptr()), "lb_lora_linear_fwd_grouped")
    _count()
    return ys, ts


def wgrad_multi(x2d: torch.Tensor, items, deferrable: bool = False):
    """items: list (<= 4) of (dTs, dA [r,K] fp32, gy2d [M,N], T, dB [N,r] fp32, diag|None, scale, r):
    all dA/dB of a family that shares x2d in one launch."""
    import ctypes
    n = len(items)
    VP, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    M, K = x2d.shape
    if _WG_QUEUE is not None and deferrable:
        for (dTs, dA, gy2d, T, dB, diag, scale, r) in items:
            _wgrad_enqueue(x2d, dTs, dA, K, 1, M, K, r, scale, diag)
            _wgrad_enqueue(gy2d, T, dB, 1, r, M, gy2d.shape[1], r, scale, diag)
        return
    dp = lambda t: None if t is None else t.data_ptr()
    arr = lambda ty, vals: (ty * n)(*vals)
    a = (arr(VP, [it[0].data_ptr() for it in items]), arr(VP, [it[1].data_ptr() for it in items]),
         arr(VP, [it[2].data_ptr() for it in items]), arr(VP, [it[3].data_ptr() for it in items]),
         arr(VP, [it[4].data_ptr() for it in items]), arr(I, [it[2].shape[1] for it in items]),
         arr(VP, [dp(it[5]) for it in items]), arr(F, [float(it[6]) for it in items]),
         arr(I, [it[7] for it in items]))
    check(_C.lib.lb_lora_wgrad_multi(n, ptr(x2d), a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7], a[8], M, K,
                                     dtype_code(x2d.dtype), stream_ptr()), "lb_lora_wgrad_multi")
    _count()


def wgrad_conv(x_nhwc_rows: torch.Tensor, V: torch.Tensor, diag, scale: float, out: torch.Tensor, r: int,
               C: int, H: int, W: int, kh: int, kw: int, pad_h: int, pad_w: int, deferrable: bool = False):
    """dA [r, C*kh*kw] (flat [r,Cin,kh,kw]) += all taps, one launch (see lb_lora_wgrad_conv)."""
    _req_cuda(x_nhwc_rows, V, out)
    M = V.shape[0]
    if _WG_QUEUE is not None and deferrable:
        _wgrad_enqueue(x_nhwc_rows, V, out, C * kh * kw, kh * kw, M, C, r, scale, diag,
                       conv=(H, W, kh, kw, pad_h, pad_w))
        return
    rp = V.shape[1]
    check(_C.lib.lb_lora_wgrad_conv(ptr(x_nhwc_rows), ptr(V), ptr(diag), float(scale), ptr(out), M, C, r,
                                    rp, H, W, kh, kw, pad_h, pad_w, dtype_code(x_nhwc_rows.dtype), stream_ptr()),
          "lb_lora_wgrad_conv")
    _count()
