"""The C-ABI shared library loads and exports every symbol include/lora_b200.h declares; argument
validation returns status codes without touching a GPU (no compute call is made here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    text = open(os.path.join(ROOT, "include", "lora_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\bint\s+(lb_[a-z0-9_]+)\s*\(", text)))


def test_build_and_load():
    import __graft_entry__ as g
    g.build()
    from lora_b200 import _C
    assert os.path.exists(_C.LIB_PATH)
    assert _C.lib.lb_abi_version() >= 1


def test_every_declared_symbol_is_exported():
    from lora_b200 import _C
    names = _declared()
    assert "lb_lora_linear_fwd" in names and "lb_optim_step_fused" in names and len(names) >= 13
    lib = ctypes.CDLL(_C.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/lora_b200.h but not exported"


def test_rank_padded_argument_validation_without_gpu():
    from lora_b200 import _C
    L = _C.lib
    buf = ctypes.create_string_buffer(4096)
    base = (ctypes.addressof(buf) + 255) & ~255
    p = ctypes.c_void_p(base)
    # rank out of range, bad dtype, misaligned K / pointer: refused before any CUDA call
    assert L.lb_lora_linear_fwd(p, p, None, p, p, 4, 1, None, 1.0, p, None, None, 8, 64, 64, 17, 16, 0, 0, None) == -2
    assert L.lb_lora_linear_fwd(p, p, None, p, p, 4, 1, None, 1.0, p, None, None, 8, 64, 64, 4, 16, 2, 0, None) == -3
    assert L.lb_lora_linear_fwd(p, p, None, p, p, 4, 1, None, 1.0, p, None, None, 8, 60, 64, 4, 16, 0, 0, None) == -1
    assert L.lb_lora_linear_fwd(ctypes.c_void_p(base + 2), p, None, p, p, 4, 1, None, 1.0, p, None, None,
                                8, 64, 64, 4, 16, 0, 0, None) == -4
    assert L.lb_lora_wgrad(p, p, None, 1.0, p, 1, 1, 8, 60, 4, 16, 0, None) == -1
    assert L.lb_lora_wgrad(p, p, None, 1.0, p, 1, 1, 8, 64, 0, 16, 0, None) == -2
    assert L.lb_cast_rows_pad(p, 1, 1, p, 4, 16, 64, 2, None) == -3
    # frozen-weight block layout: host-side size query and refusals of the tiler
    assert L.lb_tiled_weight_elems(320, 768) == 5 * 12 * 64 * 64
    assert L.lb_tiled_weight_elems(1000, 136) == 16 * 3 * 64 * 64
    assert L.lb_tiled_weight_elems(0, 64) == 0
    assert L.lb_tile_weight(p, 0, 64, 1, 0, 64, p, 0, None) == -1          # N = 0
    assert L.lb_tile_weight(p, 0, 64, 1, 64, 64, p, 2, None) == -3         # fp32 is not a 16-bit operand type
    assert L.lb_tile_weight(p, 0, 64, 1, 64, 64, ctypes.c_void_p(base + 2), 0, None) == -4
    # the LB_W_TILED flag does not hide a bad dtype
    assert L.lb_lora_linear_fwd(p, p, None, p, p, 4, 1, None, 1.0, p, None, None, 8, 64, 64, 4, 16, 0x100 | 2, 0, None) == -3


def test_missing_library_fails_loudly(tmp_path, monkeypatch):
    """No silent fallback: importing the binding without the .so raises."""
    import importlib
    from lora_b200 import _C
    monkeypatch.setattr(_C, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_C.LoraB200Error):
        _C._load()
