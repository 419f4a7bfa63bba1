"""The exact C launches of every LoRA site form, against a recorded golden (GPU).

Every module forward / backward reaches liblora_b200.so through `lora_b200._C.lib`. This test puts a
recording proxy in its place and compares, call by call, the entry name and every argument with
tests/golden/site_launches.json: a NULL pointer as "NULL", any other pointer (the stream included)
as "P", integers exactly, floats by repr, ctypes arrays as lists of the same and
`lb_wgrad_problem` arrays field by field. Device addresses are the only thing it leaves out.

Forms covered, each on small shapes: the fused linear at ranks 4 and 24, plain and with active
dropout; the split-bf16 fp32 mode; rank chunks (r = 80, eval mode); a grouped q/k/v family
(learning pass, then the grouped pass); the fused conv 1x1 / 3x3 at ranks 4 and 40, plain and with
dropout; a selector diagonal; sites where only one factor takes a gradient. Each case runs twice:
alone (fresh fp32 gradients, immediate reductions) and inside a LoraArena with deferred reductions
(the arena's gradient views, its published 16-bit factor copies and the batched flush). Each run
is two forwards (the second hits the operand caches) and one backward.

A change that means to alter launches re-records the golden on purpose:

    python tests/test_site_launches_gpu.py --record [path]
"""
import ctypes
import json
import os
import sys

import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLDEN = os.path.join(ROOT, "tests", "golden", "site_launches.json")


# ------------------------------------------------------------------------------------ recording
def _val(v, pointer=False):
    if pointer:
        return "NULL" if v is None or v == 0 else "P"
    if v is None:
        return "NULL"
    if isinstance(v, ctypes.c_void_p):
        return "NULL" if v.value is None else "P"
    if isinstance(v, ctypes.Array):
        t = v._type_
        if isinstance(t, type) and issubclass(t, ctypes.Structure):
            return [[_val(getattr(s, f), ft is ctypes.c_void_p) for f, ft in t._fields_] for s in v]
        return [_val(e, t is ctypes.c_void_p) for e in v]
    if isinstance(v, ctypes._SimpleCData):
        return _val(v.value)
    if isinstance(v, bool):
        return int(v)
    if isinstance(v, int):
        return v
    if isinstance(v, float):
        return repr(v)
    return "P"          # byref / pointer objects


class _Recorder:
    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)

        def call(*args):
            self.calls.append([name] + [_val(a) for a in args])
            return fn(*args)
        return call


class _recording:
    """Swaps `lora_b200._C.lib` for a _Recorder for the duration of the block."""

    def __enter__(self):
        from lora_b200 import _C
        self.mp = pytest.MonkeyPatch()
        self.rec = _Recorder(_C.lib)
        self.mp.setattr(_C, "lib", self.rec)
        return self.rec

    def __exit__(self, *exc):
        self.mp.undo()


# ------------------------------------------------------------------------------------ cases
# name -> (kind, r, dropout p, geometry / option, which factors take a gradient)
CASES = {
    "lin_r4": ("lin", 4, 0.0, None, "AB"),
    "lin_r4_drop": ("lin", 4, 0.1, None, "AB"),
    "lin_r24": ("lin", 24, 0.0, None, "AB"),
    "lin_r24_drop": ("lin", 24, 0.1, None, "AB"),
    "lin_r4_only_B": ("lin", 4, 0.0, None, "B"),
    "lin_r4_drop_only_A": ("lin", 4, 0.1, None, "A"),
    "lin_r4_diag": ("lin", 4, 0.0, "diag", "AB"),
    "lin_split_fp32": ("lin", 4, 0.0, "split", "AB"),
    "lin_split_fp32_only_A": ("lin", 4, 0.0, "split", "A"),
    "lin_r80_chunks": ("lin", 80, 0.1, "eval", "AB"),
    "group_qkv": ("group", 4, 0.0, None, "AB"),
    "conv1_r4": ("conv", 4, 0.0, 1, "AB"),
    "conv1_r4_drop": ("conv", 4, 0.1, 1, "AB"),
    "conv3_r4": ("conv", 4, 0.0, 3, "AB"),
    "conv3_r4_drop": ("conv", 4, 0.1, 3, "AB"),
    "conv1_r40": ("conv", 40, 0.0, 1, "AB"),
    "conv1_r40_drop": ("conv", 40, 0.1, 1, "AB"),
    "conv3_r40": ("conv", 40, 0.0, 3, "AB"),
    "conv3_r40_drop": ("conv", 40, 0.1, 3, "AB"),
    "conv3_r4_only_B": ("conv", 4, 0.0, 3, "B"),
    "conv3_r4_drop_only_A": ("conv", 4, 0.1, 3, "A"),
}
K, N, CIN, COUT = 128, 96, 64, 96


class _QKV(nn.Module):
    def __init__(self):
        super().__init__()
        import lora_b200 as L
        self.to_q = L.LoraInjectedLinear(K, K, r=4, dropout_p=0.0)
        self.to_k = L.LoraInjectedLinear(K, K, r=4, dropout_p=0.0)
        self.to_v = L.LoraInjectedLinear(K, N, r=4, dropout_p=0.0)

    def forward(self, x):
        return self.to_q(x).float().sum() + self.to_k(x).float().sum() + self.to_v(x).float().sum()


def _model(kind, r, p, opt):
    import lora_b200 as L
    torch.manual_seed(0)
    if kind == "lin":
        m = L.LoraInjectedLinear(K, N, bias=True, r=r, dropout_p=p, scale=0.75)
        if opt == "diag":
            m.set_selector_from_diag(torch.linspace(0.5, 1.5, r))
    elif kind == "conv":
        m = L.LoraInjectedConv2d(CIN, COUT, opt, padding=opt // 2, r=r, dropout_p=p, scale=0.75)
    else:
        m = _QKV()
        L.link_sites(m)
    m = m.to(DEV)
    for s in m.modules():
        if type(s).__name__ in ("LoraInjectedLinear", "LoraInjectedConv2d"):
            s.lora_up.weight.data.normal_(0, 0.05)
            (s.linear if hasattr(s, "linear") else s.conv).requires_grad_(False)
    m.train(opt != "eval")
    return m


def _sites(m):
    return [s for s in m.modules() if type(s).__name__ in ("LoraInjectedLinear", "LoraInjectedConv2d")]


def _run(name, arena):
    """One run of a case: {"calls": [...]} (+ the arena's refresh table with `arena`)."""
    import lora_b200 as L
    from lora_b200 import ops
    from lora_b200.arena import LoraArena
    kind, r, p, opt, grads = CASES[name]
    m = _model(kind, r, p, opt)
    out = {}
    if arena:
        if r > ops.MAX_RANK:
            # the arena holds ranks up to 64; wider sites still accumulate into caller-owned targets
            for s in _sites(m):
                s._lb.grad_sink = (torch.zeros(r, K, device=DEV), torch.zeros(N, r, device=DEV))
        else:
            a = LoraArena([(m, 1e-3)])
            out["arena_table"] = a.table.tolist()
    for s in _sites(m):
        s.lora_down.weight.requires_grad_("A" in grads)
        s.lora_up.weight.requires_grad_("B" in grads)
    g = torch.Generator(device=DEV).manual_seed(1)
    if kind == "conv":
        x = torch.randn(2, CIN, 8, 8, device=DEV, generator=g).to(torch.bfloat16)
    elif opt == "split":
        x = torch.randn(2, 37, K, device=DEV, generator=g)
    else:
        x = torch.randn(2, 37, K, device=DEV, generator=g).to(torch.bfloat16)
    x.requires_grad_(True)
    try:
        if opt == "split":
            L.set_fp32_mode("split")
        if kind == "group":
            L.set_grouping(True)
        torch.cuda.synchronize()
        with _recording() as rec:
            if arena:
                ops.wgrad_defer_begin()
            try:
                m(x)
                y = m(x)
                y = y if kind == "group" else y.float().square().sum()
                y.backward()
                if arena:
                    ops.wgrad_flush()
            finally:
                ops.wgrad_defer_cancel()
        torch.cuda.synchronize()
    finally:
        L.set_fp32_mode("bf16")
        L.set_grouping(False)
    out["calls"] = rec.calls
    return out


def _trace(name):
    return {"alone": _run(name, False), "arena": _run(name, True)}


def _dumps(golden) -> str:
    """JSON with one launch per line, so that a re-recorded golden diffs launch by launch."""
    cases = []
    for name in sorted(golden):
        runs = []
        for run in ("alone", "arena"):
            t = golden[name][run]
            items = ['   "calls": [\n' + ",\n".join("    " + json.dumps(c) for c in t["calls"]) + "]"]
            if "arena_table" in t:
                items.insert(0, '   "arena_table": ' + json.dumps(t["arena_table"]))
            runs.append(f'  "{run}": {{\n' + ",\n".join(items) + "}")
        cases.append(f' "{name}": {{\n' + ",\n".join(runs) + "}")
    return "{\n" + ",\n".join(cases) + "\n}\n"


@pytest.mark.parametrize("name", list(CASES))
def test_site_launches_match_golden(name):
    with open(GOLDEN) as f:
        want = json.load(f)[name]
    got = json.loads(json.dumps(_trace(name)))
    for run in ("alone", "arena"):
        g, w = got[run], want[run]
        assert g.get("arena_table") == w.get("arena_table"), run
        for i, (gc, wc) in enumerate(zip(g["calls"], w["calls"])):
            assert gc == wc, f"{run}: call {i} differs"
        assert len(g["calls"]) == len(w["calls"]), run


if __name__ == "__main__":
    if "--record" not in sys.argv:
        sys.exit("usage: python tests/test_site_launches_gpu.py --record [path]")
    i = sys.argv.index("--record")
    path = sys.argv[i + 1] if len(sys.argv) > i + 1 else GOLDEN
    golden = {name: _trace(name) for name in CASES}
    with open(path, "w") as f:
        f.write(_dumps(golden))
    print(f"recorded {len(golden)} cases, {sum(len(v[k]['calls']) for v in golden.values() for k in v)} calls "
          f"-> {path}")
