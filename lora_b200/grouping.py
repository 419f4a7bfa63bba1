"""Grouped launches for LoRA linear sites that share an input (q/k/v of a self-attention, k/v of a
cross-attention, CLIP's k/v/q projections).

At bs = 1 those sites are 12-40 output tiles each: alone they leave most of the 132 SMs idle, and
the host model calls them back to back on the same tensor. With `lora_b200.set_grouping(True)`
the first site of such a family to be called launches ONE kernel (`lb_lora_linear_fwd_grouped`)
that computes the outputs of the whole family; the siblings' outputs are parked on the parent
module and handed out when the host model calls them with THE SAME input (same storage, shape,
strides, dtype and version counter; the parked entry keeps the input alive, so the allocator
cannot recycle its address). A sibling called with anything else simply computes on its own.
Families are learned from the first forward pass per parent module (sites that received an
identical input), never guessed from names. Backward of a family is likewise one grouped dX launch.

Semantics are unchanged: every site still returns exactly what its own forward would have
returned, gradients land in the same places; only the number of launches changes.
"""
import weakref
from typing import List, Optional

import torch

from . import ops, per_sample
from .modules import (_SiteState, _active_dropout, _compute_dtype, _dx_dtype, _factor_grads, _fp32_master,
                      _grad_targets, _out_dtype, _rows, _split_mode)

_ENABLED = False


def set_grouping(flag: bool):
    global _ENABLED
    _ENABLED = bool(flag)


def get_grouping() -> bool:
    return _ENABLED


def link_sites(*models) -> int:
    """(Re)attach every LoRA site of `models` to the module that holds it. Injection does this
    itself; a `copy.deepcopy`'d or unpickled model starts without the back-references (and hence
    runs ungrouped) until this is called. Returns the number of sites linked."""
    import weakref
    n = 0
    for model in models:
        for parent in model.modules():
            for child in parent._modules.values():
                if child is not None and type(child).__name__ in ("LoraInjectedLinear", "LoraInjectedConv2d") \
                        and hasattr(child, "_lb"):
                    child._lb.parent = weakref.ref(parent)
                    n += 1
    return n


class _ParentState:
    __slots__ = ("trace", "groups", "cache", "learned")

    def __init__(self):
        self.trace = []      # [(site, key)] of the learning pass
        self.groups = {}     # id(site) -> tuple(sites) | None
        self.cache = {}      # id(site) -> (key, x kept alive, y)
        self.learned = False

    def __reduce__(self):          # runtime state: copies / pickles start empty
        return (_ParentState, ())

    def __deepcopy__(self, memo):
        return _ParentState()

    def finalize(self):
        by_key = {}
        for s, k in self.trace:
            by_key.setdefault(k, []).append(s)
        self.groups = {}
        for sites in by_key.values():
            fam = tuple(sites) if 2 <= len(sites) <= 4 else None
            for s in sites:
                self.groups[id(s)] = fam
        self.trace = []
        self.learned = True


def _key(x: torch.Tensor):
    return (x.data_ptr(), x._version, tuple(x.shape), tuple(x.stride()), x.dtype, x.requires_grad,
            torch.is_grad_enabled(), torch.is_autocast_enabled("cuda"))


def _plain(site, x) -> bool:
    if _active_dropout(site) or _split_mode(x):
        return False
    return x.is_cuda and site.linear.in_features == x.shape[-1]


class _GroupedLoraLinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, members, *factors):
        cdt = _compute_dtype(x)
        odt = _out_dtype(x, cdt)
        K = x.shape[-1]
        x2d = _rows(x, K, cdt)
        need_bwd = any(ctx.needs_input_grad)
        # per-image coefficients (per_sample.py): every member is bound, one table per problem. The table
        # replaces scale and selector, so neither is read: a graph captured here holds no copy of a
        # selector weight that set_lora_diag may free (per-sample graphs outlive selector changes)
        bound = members[0]._lb.ps is not None
        probs, meta = [], []
        for i, m in enumerate(members):
            A, B = factors[2 * i], factors[2 * i + 1]
            st: _SiteState = m._lb
            w16, _ = st.frozen(m.linear.weight, cdt, need_t=False)
            diag = None if bound else m._selector_diag()
            scale = 1.0 if bound else float(m.scale)
            probs.append((x2d, w16, st.bias32(m.linear.bias), st.down16(A, cdt), _fp32_master(B), m.r, 1,
                          diag, scale, m.r))
            meta.append((diag, scale))
        if not bound:
            ys, Ts = ops.fused_linear_grouped(probs, odt, need_bwd)
        else:
            ys, Ts = ops.fused_linear_grouped(probs, odt, False,
                                              coef_rows=[per_sample.coef_rows(m, x, K) for m in members])
        ctx.members, ctx.meta, ctx.cdt = members, meta, cdt
        ctx.x_shape, ctx.x_dtype = x.shape, x.dtype
        ctx.save_for_backward(x2d, *[t for t in Ts if t is not None], *factors)
        ctx.n_T = sum(t is not None for t in Ts)
        return tuple(y.view(*x.shape[:-1], y.shape[-1]) for y in ys)

    @staticmethod
    def backward(ctx, *gys):
        members, cdt = ctx.members, ctx.cdt
        saved = ctx.saved_tensors
        x2d = saved[0]
        Ts = saved[1:1 + ctx.n_T]
        factors = saved[1 + ctx.n_T:]
        K = x2d.shape[1]
        dx_dtype = _dx_dtype(ctx.x_dtype)
        live = [i for i, g in enumerate(gys) if g is not None]
        probs, g2ds = [], {}
        for i in live:
            m = members[i]
            A, B = factors[2 * i], factors[2 * i + 1]
            st: _SiteState = m._lb
            N = m.linear.out_features
            g2d = g2ds[i] = _rows(gys[i], N, cdt)
            _, wt16 = st.frozen(m.linear.weight, cdt, need_t=True)
            diag, scale = ctx.meta[i]
            probs.append((g2d, wt16, None, st.upT16(B, cdt), _fp32_master(A), 1, K, diag, scale, m.r))
        grads: List[Optional[torch.Tensor]] = [None] * (2 * len(members))
        dx = None
        if probs:
            dXs, dTs = ops.fused_linear_grouped(probs, dx_dtype, True)
            multi, temps = [], []
            all_sink = all(members[i]._lb.grad_sink is not None for i in live)
            for j, i in enumerate(live):
                m = members[i]
                A, B = factors[2 * i], factors[2 * i + 1]
                st: _SiteState = m._lb
                N, r = m.linear.out_features, m.r
                diag, scale = ctx.meta[i]
                need_a, need_b = ctx.needs_input_grad[2 + 2 * i], ctx.needs_input_grad[3 + 2 * i]
                tA, tB, deferrable = _grad_targets(st, need_a, need_b, (r, K), (N, r), x2d.device)
                if need_a and need_b:
                    multi.append((dTs[j], tA, g2ds[i], Ts[i], tB, diag, scale, r))
                elif need_a:
                    ops.wgrad(x2d, dTs[j], diag, scale, tA, K, 1, r, deferrable=deferrable)
                elif need_b:
                    ops.wgrad(g2ds[i], Ts[i], diag, scale, tB, 1, r, r, deferrable=deferrable)
                temps.append((i, tA, tB, deferrable, A, B))
            if multi:
                ops.wgrad_multi(x2d, multi, deferrable=all_sink)   # every dA/dB of the family: one launch
            for (i, tA, tB, deferrable, A, B) in temps:
                grads[2 * i], grads[2 * i + 1] = _factor_grads(tA, tB, deferrable, A, B)
            if ctx.needs_input_grad[0]:
                acc = dXs[0]
                for extra in dXs[1:]:
                    acc = acc + extra
                dx = acc.view(ctx.x_shape).to(ctx.x_dtype)
        return (dx, None, *grads)


def _site_sig(m):
    """Everything of a site that the parked output depends on besides the input: if any of it is
    edited between the family's launch and the sibling's own call (an external `.weight = ...`,
    an in-place update, tune_lora_scale, set_lora_diag, another per-sample table), the parked result is
    stale."""
    from .modules import _key as mkey
    sel = m.selector
    return (mkey(m.linear.weight), mkey(m.linear.bias), mkey(m.lora_down.weight), mkey(m.lora_up.weight),
            float(m.scale), mkey(getattr(sel, "weight", None)), m.training, m.dropout.p, per_sample.ps_sig(m))


def forward_maybe_grouped(site, x):
    """Returns the site's output if it was served by / started a grouped launch, else None."""
    ref = site._lb.parent
    par = ref() if ref is not None else None
    if par is None or not _plain(site, x):
        return None
    st = par.__dict__.get("_lb_groups")
    if st is None:
        st = _ParentState()
        par.__dict__["_lb_groups"] = st
    k = _key(x)
    ent = st.cache.pop(id(site), None)
    if ent is not None and ent[0] == k and ent[3] == _site_sig(site):
        return ent[2]
    # a forward inside the backward pass is a gradient-checkpointing recompute: it must launch exactly
    # what the pass it recomputes launched (torch.utils.checkpoint matches the saved tensors one by
    # one), so it never learns, finalizes or relearns families -- it only reuses what is learned
    recompute = torch._C._current_graph_task_id() != -1
    if not st.learned:
        if recompute:
            return None
        if any(s is site for s, _ in st.trace):
            st.finalize()               # the same site again: the previous pass is complete
        else:
            st.trace.append((site, k))
            return None
    if id(site) not in st.groups:       # a site this parent has never seen (re-patched model): relearn
        if recompute:
            return None
        st.__init__()
        st.trace.append((site, k))
        return None
    fam = st.groups[id(site)]
    if fam is None:
        return None
    bound = site._lb.ps is not None      # per-sample members launch together, apart from unbound ones
    members = tuple(m for m in fam if _plain(m, x) and m.r <= 16 and (m._lb.ps is not None) == bound)
    if len(members) < 2 or not any(m is site for m in members):
        return None
    factors = []
    for m in members:
        factors += [m.lora_down.weight, m.lora_up.weight]
    outs = _GroupedLoraLinearFn.apply(x, members, *factors)
    st.cache.clear()
    ret = None
    for m, y in zip(members, outs):
        if m is site:
            ret = y
        else:
            st.cache[id(m)] = (k, x, y, _site_sig(m))
    return ret
