"""Per-image LoRA scale and selector mix: every image of a batch with its own `scale` and selector
diagonal, in the same fused launches (lb_lora_linear_fwd_ps, lb_lora_linear_fwd_grouped_ps,
lb_lora_conv2d_fwd_ps).

    with lora_b200.per_sample_lora(pipe.unet, scale=[0.0, 0.3, 0.7, 1.0], samples=4):
        images = pipe([prompt] * 4).images

Each LoRA site under the model gets a coefficient table [S, r] fp32 on its device (a view of one
buffer per call): row b is fl32(fl32(scale_b) * fl32(diag_bj)), computed in fp32, which is what the
scalar path's `scale * diag` gives for that image. A site's forward scales output row m by row
(m // rows_per_sample) % S, with rows_per_sample = the rows of one batch element (tokens or pixels),
so the [uncond B ; cond B] halves of classifier-free guidance and a text encoder's [negative ; prompt]
batch map both copies to the same image. A table whose rows are all equal gives the default forward
bit for bit.

Forward only: a site forward under grad, with an active dropout, under the split-fp32 policy or at a
rank above 64 raises LoraB200Error.
"""
import contextlib
from typing import List, Optional, Sequence

import torch

from . import ops
from ._C import LoraB200Error

_SITE_NAMES = ("LoraInjectedLinear", "LoraInjectedConv2d")


def sites_of(*models) -> List[torch.nn.Module]:
    return [m for model in models for m in model.modules() if type(m).__name__ in _SITE_NAMES]


def _as_scales(scale, S: int) -> Optional[torch.Tensor]:
    """scale: None, a float or S floats -> None or fp32 [S]."""
    if scale is None:
        return None
    t = torch.as_tensor(scale, dtype=torch.float32).detach().cpu()
    if t.dim() == 0:
        return t.expand(S)
    if t.dim() != 1 or t.shape[0] != S:
        raise ValueError(f"scale: a float or {S} values (one per image), got shape {tuple(t.shape)}")
    return t


def _as_diag(diag, S: int, r: int) -> Optional[torch.Tensor]:
    """diag: None, [r] or [S, r] -> None or fp32 [S, r]."""
    if diag is None:
        return None
    t = torch.as_tensor(diag, dtype=torch.float32).detach().cpu()
    if t.dim() == 1:
        t = t.unsqueeze(0).expand(S, -1)
    if t.dim() != 2 or t.shape[0] != S:
        raise ValueError(f"diag: [r] or [{S}, r] (one row per image), got shape {tuple(t.shape)}")
    if t.shape[1] != r:
        raise ValueError(f"diag of width {t.shape[1]}: the LoRA sites have rank {r}")
    return t


def samples_of(scale, diag, samples: Optional[int]) -> int:
    """The number of per-image rows S: `samples`, else the length of scale / diag."""
    if samples is not None:
        S = int(samples)
    else:
        S = None
        for v, dim in ((scale, 1), (diag, 2)):
            t = None if v is None else torch.as_tensor(v)
            if t is not None and t.dim() == dim:
                S = int(t.shape[0])
                break
        if S is None:
            raise ValueError("per_sample_lora: give samples=S (or per-image scale / diag rows)")
    if S < 1:
        raise ValueError(f"samples must be >= 1, got {S}")
    return S


def selector_diags(sites) -> dict:
    """{id(site): fp32 CPU [r]} of the sites that have a selector (set_lora_diag), read with one
    device-to-host copy per device instead of one per site."""
    by_dev = {}
    for m in sites:
        if not isinstance(m.selector, torch.nn.Identity):
            w = m.selector.weight.detach()
            by_dev.setdefault(w.device, []).append((m, torch.diagonal(w.reshape(m.r, m.r))))
    out = {}
    for items in by_dev.values():
        flat = torch.cat([d.float() for _, d in items]).cpu()
        off = 0
        for m, d in items:
            out[id(m)] = flat[off:off + m.r]
            off += m.r
    return out


def site_rows(m, scale: Optional[torch.Tensor], diag: Optional[torch.Tensor], S: int, sel=None) -> torch.Tensor:
    """One site's [S, r] fp32 table: fl32(fl32(scale_b) * fl32(diag_bj)). Missing parts come from the
    site's current `scale` and selector (identity: ones); `sel` = selector_diags' dict, when the
    caller has read the selectors already."""
    s = scale if scale is not None else torch.tensor(float(m.scale), dtype=torch.float32).expand(S)
    if diag is None:
        d = (selector_diags([m]) if sel is None else sel).get(id(m))
        d = torch.ones(m.r, dtype=torch.float32) if d is None else d
        diag = d.unsqueeze(0).expand(S, -1)
    return (s.unsqueeze(1) * diag).contiguous()


def check_args(sites, scale, diag, S: int):
    """(scale [S] | None, diag [S, r] | None), validated against the sites (ValueError)."""
    if not sites:
        raise ValueError("the model has no LoRA sites")
    sc = _as_scales(scale, S)
    dg = None
    if diag is not None:
        ranks = sorted({m.r for m in sites})
        if len(ranks) != 1:
            raise ValueError(f"diag needs every LoRA site at one rank, the sites have ranks {ranks}")
        dg = _as_diag(diag, S, ranks[0])
    return sc, dg


def host_table(sites, scale, diag, S: int) -> torch.Tensor:
    """Every site's [S, r] table, concatenated (fp32, CPU), in `sites` order."""
    sel = selector_diags(sites) if diag is None else {}
    return torch.cat([site_rows(m, scale, diag, S, sel).reshape(-1) for m in sites])


def table_views(buf: torch.Tensor, sites, S: int):
    """The per-site [S, r] views of a flat table laid out by host_table."""
    views, off = [], 0
    for m in sites:
        n = S * m.r
        views.append(buf[off:off + n].view(S, m.r))
        off += n
    return views


@contextlib.contextmanager
def bound(sites, views, S: int):
    """Bind each site to its table view for the body (restores the previous binding on exit)."""
    prev = [m._lb.ps for m in sites]
    try:
        for m, v in zip(sites, views):
            m._lb.ps = (v, S)
        yield
    finally:
        for m, p in zip(sites, prev):
            m._lb.ps = p


@contextlib.contextmanager
def per_sample_lora(model, scale=None, diag=None, samples: Optional[int] = None):
    """Run every LoRA site under `model` with per-image coefficients for the body of the `with`.

    scale: a float or [S] values -- each image's `scale`, as tune_lora_scale would set it;
    diag: [r] or [S, r] -- each image's selector diagonal, as set_lora_diag would set it (every site
          must have rank r); samples: S, the images of the batch (a batch of k * S rows is k copies).
    What is not given comes from each site's current scale and selector. The tables are built and
    uploaded once, on entry."""
    S = samples_of(scale, diag, samples)
    sites = sites_of(model)
    sc, dg = check_args(sites, scale, diag, S)
    flat = host_table(sites, sc, dg, S)
    dev = sites[0].lora_up.weight.device
    buf = flat.to(dev)
    by_dev = {dev: buf}
    views = []
    for m, v in zip(sites, table_views(flat, sites, S)):   # sites on other devices: their own copy
        d = m.lora_up.weight.device
        if d not in by_dev:
            by_dev[d] = flat.to(d)
        off = v.storage_offset()
        views.append(by_dev[d][off:off + v.numel()].view(v.shape))
    with bound(sites, views, S):
        yield


# ---------------------------------------------------------------------------- site forwards
def coef_rows(m, x: torch.Tensor, K: int):
    """(table, ld, rows_per_sample, S) of a bound site for input x (K = input features / channels),
    or LoraB200Error for a call the per-sample kernels do not cover."""
    from .modules import _active_dropout, _split_mode
    table, S = m._lb.ps
    name = type(m).__name__
    if m.r > ops.MAX_RANK:
        raise LoraB200Error(f"{name}: per-sample LoRA coefficients cover ranks up to {ops.MAX_RANK}, not {m.r}")
    if torch.is_grad_enabled() and (x.requires_grad or m.lora_down.weight.requires_grad
                                    or m.lora_up.weight.requires_grad):
        raise LoraB200Error(f"{name}: per-sample LoRA coefficients are forward only (run under torch.no_grad())")
    if _active_dropout(m):
        raise LoraB200Error(f"{name}: per-sample LoRA coefficients do not run with an active dropout (eval())")
    if _split_mode(x):
        raise LoraB200Error(f"{name}: per-sample LoRA coefficients do not run under the split-fp32 policy")
    if x.dim() < 2 or x.shape[0] % S != 0:
        raise LoraB200Error(f"{name}: a batch of {x.shape[0] if x.dim() else 0} is not a multiple of the "
                            f"{S} per-sample coefficient rows")
    if table.device != x.device:
        raise LoraB200Error(f"{name}: coefficient table on {table.device}, input on {x.device}")
    rps = x.numel() // (K * x.shape[0])
    return table, m.r, rps, S


def linear_forward(m, x: torch.Tensor) -> torch.Tensor:
    """LoraInjectedLinear.forward with the bound per-sample table (lb_lora_linear_fwd_ps; a grouped
    family launches lb_lora_linear_fwd_grouped_ps)."""
    from . import grouping
    from .modules import _compute_dtype, _fp32_master, _out_dtype, _rows
    if not x.is_cuda:
        raise LoraB200Error("LoraInjectedLinear.forward: lora_b200 runs on CUDA tensors only")
    lin = m.linear
    K, N, r = lin.in_features, lin.out_features, m.r
    rows = coef_rows(m, x, K)
    if grouping._ENABLED and m._lb.parent is not None:
        out = grouping.forward_maybe_grouped(m, x)
        if out is not None:
            return out
    st = m._lb
    cdt = _compute_dtype(x)
    x2d = _rows(x, K, cdt)
    w16, _ = st.frozen(lin.weight, cdt, need_t=False)
    y, _ = ops.fused_linear(x2d, w16, st.bias32(lin.bias), st.down16(m.lora_down.weight, cdt),
                            _fp32_master(m.lora_up.weight), r, 1, None, 1.0, r, _out_dtype(x, cdt), False,
                            coef_rows=rows)
    return y.view(*x.shape[:-1], N)


def conv_forward(m, x: torch.Tensor) -> torch.Tensor:
    """LoraInjectedConv2d.forward with the bound per-sample table (lb_lora_conv2d_fwd_ps)."""
    from .conv_path import _geometry, _nhwc16
    from .modules import _compute_dtype, _fp32_master, _out_dtype
    if not x.is_cuda or x.dim() != 4:
        raise LoraB200Error("LoraInjectedConv2d.forward: lora_b200 runs on 4-D NCHW CUDA tensors only")
    conv = m.conv
    kh, kw, ph, pw = _geometry(conv)
    rows = coef_rows(m, x, conv.in_channels)
    st = m._lb
    cdt = _compute_dtype(x)
    w_f, _ = st.frozen_conv(conv.weight, cdt, False)
    y, _ = ops.fused_conv2d(_nhwc16(x, cdt), w_f, st.bias32(conv.bias), st.conv_down16(m.lora_down.weight, cdt),
                            _fp32_master(m.lora_up.weight), 0, m.r, 1, 0, None, 1.0, m.r, conv.out_channels,
                            kh, kw, ph, pw, False, _out_dtype(x, cdt), False, coef_rows=rows)
    return y


def ps_sig(m):
    """What of a site's binding a parked grouped result depends on (grouping._site_sig)."""
    ps = m._lb.ps
    if ps is None:
        return None
    t = ps[0]
    return (id(t), t.data_ptr(), t._version, tuple(t.shape), ps[1])
