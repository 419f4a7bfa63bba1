"""LoRA operator modules whose forward/backward run in liblora_b200.so (sm_90a).

Drop-in for the two operator classes of the reference (same class NAMES -- three reference call
sites match on ``__class__.__name__``, lora_diffusion/lora.py:879,885,1030 -- same constructor
signatures, same child names ``linear|conv``, ``lora_down``, ``dropout``, ``lora_up``,
``selector``, same attributes ``r`` and ``scale``):

    LoraInjectedLinear   <- /root/reference/lora_diffusion/lora.py:32-70
    LoraInjectedConv2d   <- /root/reference/lora_diffusion/lora.py:73-156

What differs is only *how* ``forward`` is computed: one fused wgmma kernel
(include/lora_b200.h: lb_lora_linear_fwd / lb_lora_conv2d_fwd) instead of three library GEMMs
and four elementwise passes; backward = the same fused kernel on the pre-transposed frozen weight
plus one skinny reduction per LoRA factor. The children stay ordinary nn.Linear / nn.Conv2d
objects so that every external ``.weight = ...`` assignment, ``state_dict`` key and ``.to()`` call
made by the reference's own inject/patch code keeps working; they are containers, never called.

There is no eager fallback: a CPU tensor or a missing library raises LoraB200Error.
"""
import math
import weakref
from typing import Optional

import torch
import torch.nn as nn

from . import dropout_path, ops
from ._C import LoraB200Error

_LOW = (torch.bfloat16, torch.float16)
_FP32_MODE = "bf16"   # fp32 activations outside autocast: "bf16" operands, or "split" (precise_path.py)


def set_fp32_mode(mode: str):
    """Policy for fp32 activations outside autocast: "bf16" (default: bf16 operands, fp32
    accumulate and output) or "split" (3-term split-bf16 operands, fp32-faithful; 3x tensor work)."""
    global _FP32_MODE
    if mode not in ("bf16", "split"):
        raise ValueError("fp32 mode must be 'bf16' or 'split'")
    _FP32_MODE = mode


def get_fp32_mode() -> str:
    return _FP32_MODE


def _compute_dtype(x: torch.Tensor) -> torch.dtype:
    """16-bit operand type for this call: the activation's own 16-bit type, else the autocast
    type, else bf16 (fp32 activations outside autocast: bf16 operands, fp32 accumulate/output)."""
    if x.dtype in _LOW:
        return x.dtype
    if x.dtype != torch.float32:
        raise LoraB200Error(f"lora_b200: unsupported activation dtype {x.dtype} (fp32, bf16, fp16 only)")
    if torch.is_autocast_enabled("cuda"):
        dt = torch.get_autocast_dtype("cuda")
        if dt in _LOW:
            return dt
    return torch.bfloat16


def _out_dtype(x: torch.Tensor, cdt: torch.dtype) -> torch.dtype:
    if x.dtype in _LOW:
        return x.dtype
    if torch.is_autocast_enabled("cuda"):
        return cdt  # like F.linear under autocast
    return torch.float32


class _Key:
    """Identity of a cached operand's source tensor: the tensor OBJECT (held weakly -- `id()` values
    are recycled after garbage collection, a weak reference is not), its version counter, storage
    address, dtype and device. Two keys are equal only while the original object is alive."""
    __slots__ = ("ref", "ver", "ptr", "dtype", "device", "tag")

    def __init__(self, t: torch.Tensor, tag=None):
        self.ref = weakref.ref(t)
        self.ver, self.ptr, self.dtype, self.device, self.tag = t._version, t.data_ptr(), t.dtype, t.device, tag

    def __eq__(self, o):
        if not isinstance(o, _Key):
            return False
        a = self.ref()
        return (a is not None and a is o.ref() and self.ver == o.ver and self.ptr == o.ptr
                and self.dtype == o.dtype and self.device == o.device and self.tag == o.tag)

    def __ne__(self, o):
        return not self.__eq__(o)

    __hash__ = None


def _key(t: Optional[torch.Tensor], tag=None):
    return None if t is None else _Key(t, tag)


def invalidate_caches(model: nn.Module):
    """Drop every cached 16-bit operand of the LoRA sites under `model`. The caches follow
    re-assignment (`.weight = ...`, `.weight.data = ...`) and version-counted in-place edits on
    their own; an in-place edit made THROUGH `.data` (`p.data.copy_()`, `p.data.mul_()`, an EMA or
    a hand-written weight loader) bumps no counter and moves no pointer -- call this afterwards.
    Sites owned by a LoraArena re-publish their factor shadows at the next `arena.step()`."""
    for m in model.modules():
        st = m.__dict__.get("_lb")
        if isinstance(st, _SiteState):
            st.w.clear()
            st.down.clear()
            st.upT.clear()
            st.bias = None
            st.w3 = None


class _SiteState:
    """Per-module device caches: 16-bit frozen weight (+ transpose), fp32 bias, 16-bit padded
    copies of the LoRA factors. Re-validated on every call against (object id, version counter,
    data_ptr), because the reference's API re-assigns ``.weight`` from outside at will
    (lora.py:290,302-303,706-711; cli_svd.py:52-53)."""

    def __init__(self):
        self.w = {}        # dtype -> (key, w16, wt16); a conv site: (key, forward operand, dX operand)
        self.bias = None   # (key, bias fp32)
        self.down = {}     # dtype -> (key, down16 [RP,K]), RP = ops.rank_pad(r); a conv site: K = taps*Cin
        self.upT = {}      # dtype -> (key, upT16 [RP,N])
        self.w3 = None     # (key, W, W^T or None) as split-bf16 [.., 3K] (precise_path.py)
        self.conv_tables = {}  # ops.conv_tap_table's tables: they follow the factor's shape, never its values
        self.grad_sink = None  # (gA view, gB view) when the arena owns the gradients
        self.parent = None     # weakref to the module this site was injected into (grouping.py)
        self.ps = None         # (coefficient table [S, r] fp32, S) bound by per_sample.py, or None

    # caches and the parent back-reference are per-process runtime state: a copied / pickled module
    # starts with an empty one (copy.deepcopy(model), torch.save(model) keep working)
    def __getstate__(self):
        return {}

    def __setstate__(self, state):
        self.__init__()

    def __deepcopy__(self, memo):
        return _SiteState()

    def frozen(self, weight2d: torch.Tensor, dtype, need_t: bool, tiled: Optional[bool] = None):
        """16-bit copies of the frozen weight: (W [N,K], W^T [K,N] or None), row-major tensors -- or, with
        ops.TILED_WEIGHTS (opt-in, LB_TILED_W=1), ops.TiledWeight in contiguous
        64 x 64 blocks. tiled=False forces row-major (row slicing: the rank > 64 chunks)."""
        tiled = ops.TILED_WEIGHTS if tiled is None else tiled
        k = _key(weight2d)
        slot = (dtype, "tiled") if tiled else dtype
        ent = self.w.get(slot)
        if ent is not None and ent[0] != k:
            ent = None
        have_plain = ent is not None
        have_t = ent is not None and ent[2] is not None
        if not have_plain or (need_t and not have_t):
            if tiled:
                src = weight2d.detach()
                if not src.is_contiguous():
                    src = src.contiguous()
                w16 = ent[1] if have_plain else ops.tile_weight(src, dtype)
                wt16 = ops.tile_weight(src, dtype, transpose=True) if need_t else None
            else:
                reuse = weight2d.dtype == dtype and weight2d.is_contiguous()
                make_plain = not have_plain and not reuse
                w16, wt16 = ops.cast_weight(weight2d, dtype, make_plain, need_t)
                if have_plain:
                    w16 = ent[1]
                elif reuse:
                    w16 = weight2d.detach()
            ent = (k, w16, wt16 if need_t else None)
            self.w[slot] = ent
        return ent[1], ent[2]

    def frozen_conv(self, weight: torch.Tensor, dtype, need_bwd: bool):
        """16-bit operands of a frozen conv weight (ops.cast_conv_weight): (forward [Cout, taps*Cin],
        input-gradient [Cin, taps*Cout] or None)."""
        k = _key(weight, tag="conv")
        ent = self.w.get(dtype)
        if ent is not None and ent[0] != k:
            ent = None
        have_f = ent is not None
        have_b = ent is not None and ent[2] is not None
        if not have_f or (need_bwd and not have_b):
            f, b = ops.cast_conv_weight(weight, dtype, not have_f, need_bwd)
            ent = (k, ent[1] if have_f else f, b if need_bwd else None)
            self.w[dtype] = ent
        return ent[1], ent[2]

    def bias32(self, bias: Optional[torch.Tensor]):
        if bias is None:
            return None
        k = _key(bias)
        if self.bias is None or self.bias[0] != k:
            self.bias = (k, bias.detach().to(torch.float32).contiguous())
        return self.bias[1]

    def down16(self, a2d: torch.Tensor, dtype):
        """A [r,K] fp32 master -> [RP,K] 16-bit, rows r.. zero (RP = ops.rank_pad(r))."""
        k = _key(a2d)
        ent = self.down.get(dtype)
        if ent is None or ent[0] != k:
            r, K = a2d.shape
            ent = (k, ops.cast_rows_pad16(_fp32_master(a2d), K, 1, r, K, dtype))
            self.down[dtype] = ent
        return ent[1]

    def conv_down16(self, a4d: torch.Tensor, dtype):
        """A [r,Cin,kh,kw] fp32 master -> [RP, taps*Cin] 16-bit, tap-major (ops.conv_down16)."""
        k = _key(a4d)
        ent = self.down.get(dtype)
        if ent is None or ent[0] != k:
            ent = (k, ops.conv_down16(a4d, dtype, self.conv_tables))
            self.down[dtype] = ent
        return ent[1]

    def upT16(self, b: torch.Tensor, dtype):
        """B [N,r] (a conv site: [Cout,r,1,1]) fp32 master -> B^T [RP,N] 16-bit, rows r.. zero."""
        k = _key(b)
        ent = self.upT.get(dtype)
        if ent is None or ent[0] != k:
            N, r = b.shape[0], b.shape[1]
            ent = (k, ops.cast_rows_pad16(_fp32_master(b), 1, r, r, N, dtype))
            self.upT[dtype] = ent
        return ent[1]


def _fp32_master(w: torch.Tensor) -> torch.Tensor:
    d = w.detach()
    if d.dtype != torch.float32 or not d.is_contiguous():
        d = d.float().contiguous()
    return d


# ---- what every site's autograd function shares (fused linear / conv, precise, rank chunks, grouped)
def _rows(t: torch.Tensor, C: int, cdt) -> torch.Tensor:
    """t as contiguous [M, C] rows of dtype cdt (the x2d / gy2d operands)."""
    t2d = t.reshape(-1, C)
    if t2d.dtype != cdt or not t2d.is_contiguous():
        t2d = t2d.to(cdt).contiguous()
    return t2d


def _dx_dtype(x_dtype: torch.dtype) -> torch.dtype:
    """dX is computed in the activation's own 16-bit type, else in fp32."""
    return x_dtype if x_dtype in _LOW else torch.float32


def _grad_targets(st: _SiteState, need_a: bool, need_b: bool, a_shape, b_shape, device):
    """(tA, tB, deferrable): where dA / dB accumulate. With an arena these are its gradient views,
    which feed only the optimizer, so their reductions may be deferred (ops.wgrad_defer_begin);
    otherwise fresh fp32 zeros. A target is None when its factor needs no gradient."""
    sink = st.grad_sink
    if sink is not None:
        return (sink[0] if need_a else None), (sink[1] if need_b else None), True
    z = lambda shape: torch.zeros(shape, device=device, dtype=torch.float32)
    return (z(a_shape) if need_a else None), (z(b_shape) if need_b else None), False


def _factor_grads(tA, tB, deferrable: bool, A: torch.Tensor, B: torch.Tensor):
    """(dA, dB) for autograd: None when the targets are the arena's (the gradients are in place)."""
    if deferrable:
        return None, None
    return (None if tA is None else tA.to(A.dtype).view_as(A)), (None if tB is None else tB.to(B.dtype).view_as(B))


def _active_dropout(mod) -> float:
    """p of the site's nn.Dropout when it acts (training mode and p > 0), else 0."""
    p = float(mod.dropout.p)
    return p if mod.training and p > 0.0 else 0.0


def _split_mode(x: torch.Tensor) -> bool:
    """Whether the fp32-faithful split-bf16 policy (set_fp32_mode("split")) applies to this input."""
    return _FP32_MODE == "split" and x.dtype == torch.float32 and not torch.is_autocast_enabled("cuda")


class _FusedLoraLinearFn(torch.autograd.Function):
    """autograd node for one LoRA linear site. Inputs A, B are passed so that autograd knows the
    factors are used; W and bias are frozen (train_lora_dreambooth.py:595) and never get grads.
    With an active nn.Dropout the forward masks the branch in the kernel's drain and the backward
    recomputes the same mask from the saved seed (dropout_path.py)."""

    @staticmethod
    def forward(ctx, x, A, B, mod):
        st: _SiteState = mod._lb
        lin = mod.linear
        if not x.is_cuda:
            raise LoraB200Error("LoraInjectedLinear.forward: lora_b200 runs on CUDA tensors only")
        cdt = _compute_dtype(x)
        odt = _out_dtype(x, cdt)
        K, N, r = lin.in_features, lin.out_features, mod.r
        x2d = _rows(x, K, cdt)
        w16, _ = st.frozen(lin.weight, cdt, need_t=False)
        b32 = st.bias32(lin.bias)
        down16 = st.down16(A, cdt)
        diag = mod._selector_diag()
        scale = float(mod.scale)
        p = _active_dropout(mod)
        seed = dropout_path._fresh_seed(mod, x.device) if p > 0.0 else None
        want_t = p > 0.0 or any(ctx.needs_input_grad[:3])
        y, T = ops.fused_linear(x2d, w16, b32, down16, _fp32_master(B), r, 1, diag, scale, r, odt, want_t,
                                drop_p=p, seed=seed)
        ctx.mod, ctx.cdt, ctx.scale, ctx.p, ctx.diag = mod, cdt, scale, p, diag
        ctx.x_shape, ctx.x_dtype = x.shape, x.dtype
        ctx.save_for_backward(x2d, T, A, B, *([] if seed is None else [seed]))
        return y.view(*x.shape[:-1], N)

    @staticmethod
    def backward(ctx, gy):
        mod = ctx.mod
        st: _SiteState = mod._lb
        x2d, T, A, B, *seed = ctx.saved_tensors
        lin = mod.linear
        K, N, r, p = lin.in_features, lin.out_features, mod.r, ctx.p
        cdt = ctx.cdt
        gy2d = _rows(gy, N, cdt)
        _, wt16 = st.frozen(lin.weight, cdt, need_t=True)
        upT16 = st.upT16(B, cdt)
        A32 = _fp32_master(A)
        # dX = gY.W + (dTs * s*d).A, dTs = gY.B   (same fused kernel, transposed operands); with dropout
        # one masked pass gives dTs = (mask o gY / (1-p)) . B first and the dX kernel takes it (T_in)
        t_in = ops.dropout_dt(gy2d, _fp32_master(B), r, 1, p, seed[0], r) if p > 0.0 else None
        dX, dTs = ops.fused_linear(gy2d, wt16, None, upT16, A32, 1, K, ctx.diag, ctx.scale, r,
                                   _dx_dtype(ctx.x_dtype), t_in is None, t_in=t_in)
        dTs = dTs if t_in is None else t_in
        need_x, need_a, need_b = ctx.needs_input_grad[:3]
        tA, tB, deferrable = _grad_targets(st, need_a, need_b, (r, K), (N, r), gy.device)
        if need_a and need_b and p == 0.0:
            ops.wgrad_pair(x2d, dTs, tA, gy2d, T, tB, ctx.diag, ctx.scale, r, deferrable=deferrable)
        else:
            if need_a:
                ops.wgrad(x2d, dTs, ctx.diag, ctx.scale, tA, K, 1, r, deferrable=deferrable)
            if need_b and p > 0.0:      # dB reduces the masked gY
                ops.wgrad_masked(gy2d, T, ctx.diag, ctx.scale, tB, 1, r, r, p, seed[0], deferrable=deferrable)
            elif need_b:
                ops.wgrad(gy2d, T, ctx.diag, ctx.scale, tB, 1, r, r, deferrable=deferrable)
        dA, dB = _factor_grads(tA, tB, deferrable, A, B)
        dx = dX.view(ctx.x_shape).to(ctx.x_dtype) if need_x else None
        return dx, dA, dB, None


def _selector_diag(self) -> Optional[torch.Tensor]:
    sel = self.selector
    if isinstance(sel, nn.Identity):
        return None
    w = sel.weight.detach()
    return torch.diagonal(w.reshape(self.r, self.r)).to(torch.float32).contiguous()


def realize_as_lora(self):
    return self.lora_up.weight.data * self.scale, self.lora_down.weight.data


class LoraInjectedLinear(nn.Module):
    """y = linear(x) + dropout(lora_up(selector(lora_down(x)))) * scale   (lora.py:53-58)."""

    def __init__(self, in_features, out_features, bias=False, r=4, dropout_p=0.1, scale=1.0):
        super().__init__()
        if r > min(in_features, out_features):
            raise ValueError(
                f"LoRA rank {r} must be less or equal than {min(in_features, out_features)}"
            )
        self.r = r
        # Construction order mirrors the reference so the torch RNG stream is consumed
        # identically (three kaiming draws, then normal_ on the down factor) -- seed parity.
        self.linear = nn.Linear(in_features, out_features, bias)
        self.lora_down = nn.Linear(in_features, r, bias=False)
        self.dropout = nn.Dropout(dropout_p)
        self.lora_up = nn.Linear(r, out_features, bias=False)
        self.scale = scale
        self.selector = nn.Identity()
        nn.init.normal_(self.lora_down.weight, std=1 / r)
        nn.init.zeros_(self.lora_up.weight)
        self._lb = _SiteState()

    _selector_diag = _selector_diag
    realize_as_lora = realize_as_lora

    def forward(self, input):
        ops.wgrad_segment_boundary()
        if self._lb.ps is not None:   # per-image coefficients (per_sample.py)
            from .per_sample import linear_forward
            return linear_forward(self, input)
        if self.r > ops.MAX_RANK:   # joined LoRAs above rank 64 (lora_manager.py:13-71): rank chunks of 64
            from .rank_chunks import lora_linear_chunked
            return lora_linear_chunked(self, input)
        if not _active_dropout(self):
            if _split_mode(input) and self.linear.weight.dtype == torch.float32:
                from .precise_path import lora_linear_precise
                return lora_linear_precise(self, input)
            from . import grouping
            if grouping._ENABLED and self._lb.parent is not None:
                out = grouping.forward_maybe_grouped(self, input)
                if out is not None:
                    return out
        return _FusedLoraLinearFn.apply(input, self.lora_down.weight, self.lora_up.weight, self)

    def set_selector_from_diag(self, diag: torch.Tensor):
        assert diag.shape == (self.r,)
        self.selector = nn.Linear(self.r, self.r, bias=False)
        self.selector.weight.data = torch.diag(diag)
        self.selector.weight.data = self.selector.weight.data.to(
            self.lora_up.weight.device
        ).to(self.lora_up.weight.dtype)


class LoraInjectedConv2d(nn.Module):
    """y = conv(x) + dropout(lora_up(selector(lora_down(x)))) * scale   (lora.py:130-135);
    lora_down has the base conv's kernel/stride/padding/dilation/groups, lora_up is 1x1."""

    def __init__(self, in_channels: int, out_channels: int, kernel_size, stride=1, padding=0,
                 dilation=1, groups: int = 1, bias: bool = True, r: int = 4,
                 dropout_p: float = 0.1, scale: float = 1.0):
        super().__init__()
        if r > min(in_channels, out_channels):
            raise ValueError(
                f"LoRA rank {r} must be less or equal than {min(in_channels, out_channels)}"
            )
        self.r = r
        self.conv = nn.Conv2d(in_channels=in_channels, out_channels=out_channels,
                              kernel_size=kernel_size, stride=stride, padding=padding,
                              dilation=dilation, groups=groups, bias=bias)
        self.lora_down = nn.Conv2d(in_channels=in_channels, out_channels=r,
                                   kernel_size=kernel_size, stride=stride, padding=padding,
                                   dilation=dilation, groups=groups, bias=False)
        self.dropout = nn.Dropout(dropout_p)
        self.lora_up = nn.Conv2d(in_channels=r, out_channels=out_channels, kernel_size=1,
                                 stride=1, padding=0, bias=False)
        self.selector = nn.Identity()
        self.scale = scale
        nn.init.normal_(self.lora_down.weight, std=1 / r)
        nn.init.zeros_(self.lora_up.weight)
        self._lb = _SiteState()

    _selector_diag = _selector_diag
    realize_as_lora = realize_as_lora

    def forward(self, input):
        ops.wgrad_segment_boundary()
        if self._lb.ps is not None:   # per-image coefficients (per_sample.py)
            from .per_sample import conv_forward
            return conv_forward(self, input)
        from .conv_path import lora_conv2d
        return lora_conv2d(self, input)

    def set_selector_from_diag(self, diag: torch.Tensor):
        assert diag.shape == (self.r,)
        self.selector = nn.Conv2d(in_channels=self.r, out_channels=self.r, kernel_size=1,
                                  stride=1, padding=0, bias=False)
        self.selector.weight.data = torch.diag(diag)
        self.selector.weight.data = self.selector.weight.data.to(
            self.lora_up.weight.device
        ).to(self.lora_up.weight.dtype)
