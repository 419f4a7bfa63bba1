"""Argument validation of the rank-pad (`r_pad`) arguments: refused before any CUDA call."""
import ctypes

import pytest


@pytest.fixture(scope="module")
def L():
    import __graft_entry__ as g
    g.build()
    from lora_b200 import _C
    return _C.lib


def test_r_pad_argument_of_every_entry_point_validates_without_gpu(L):
    buf = ctypes.create_string_buffer(4096)
    base = (ctypes.addressof(buf) + 255) & ~255
    p = ctypes.c_void_p(base)
    fwd = lambda r, rp, K=64, dt=0: L.lb_lora_linear_fwd(p, p, None, p, p, 4, 1, None, 1.0, p, None, None,
                                                         8, K, 64, r, rp, dt, 0, None)
    assert fwd(4, 24) == -1 and fwd(4, 0) == -1 and fwd(4, 128) == -1      # pad not in {16, 32, 64}
    assert fwd(17, 16) == -2 and fwd(33, 32) == -2 and fwd(65, 64) == -2    # r > r_pad
    assert fwd(0, 32) == -2
    assert fwd(20, 32, dt=2) == -3 and fwd(20, 32, K=60) == -1
    fwd_drop = lambda r, rp: L.lb_lora_linear_fwd_dropout(p, p, None, p, p, 4, 1, None, 1.0, p, None, 8, 64, 64, r,
                                                          rp, 0, 0, 0.1, p, None)
    assert fwd_drop(40, 32) == -2 and fwd_drop(20, 24) == -1
    conv = lambda r, rp, per_tap=0, t_in=None: L.lb_lora_conv2d_fwd(
        p, p, None, p, p, 4, 1, 0, None, 1.0, p, None, t_in, 1, 8, 8, 64, 64, 3, 3, 1, 1, r, rp, per_tap, 0, 0, None)
    assert conv(20, 48) == -1 and conv(20, 24) == -1 and conv(40, 32) == -2
    assert conv(20, 32, per_tap=1) == -1          # the wide 3x3 input gradient needs T_in
    conv_drop = lambda r, rp: L.lb_lora_conv2d_fwd_dropout(p, p, None, p, p, 4, 1, None, 1.0, p, None, 1, 8, 8, 64,
                                                           64, 1, 1, 0, 0, r, rp, 0, 0, 0.1, p, None)
    assert conv_drop(70, 64) == -2 and conv_drop(20, 24) == -1
    assert L.lb_lora_wgrad(p, p, None, 1.0, p, 1, 1, 8, 64, 20, 48, 0, None) == -1
    assert L.lb_lora_wgrad(p, p, None, 1.0, p, 1, 1, 8, 64, 20, 24, 0, None) == -1
    assert L.lb_lora_wgrad(p, p, None, 1.0, p, 1, 1, 8, 64, 40, 32, 0, None) == -2
    assert L.lb_lora_wgrad(p, p, None, 1.0, p, 1, 1, 8, 60, 20, 32, 0, None) == -1
    assert L.lb_lora_wgrad_masked(p, p, None, 1.0, p, 1, 1, 8, 64, 65, 64, 0.1, p, 0, None) == -2
    assert L.lb_lora_wgrad_masked(p, p, None, 1.0, p, 1, 1, 8, 64, 20, 24, 0.1, p, 0, None) == -1
    assert L.lb_lora_wgrad_conv(p, p, None, 1.0, p, 64, 64, 33, 32, 8, 8, 3, 3, 1, 1, 0, None) == -2
    assert L.lb_lora_wgrad_conv(p, p, None, 1.0, p, 64, 64, 20, 24, 8, 8, 3, 3, 1, 1, 0, None) == -1
    assert L.lb_lora_wgrad_pair(p, p, p, 64, 1, 64, p, p, p, 1, 20, 64, None, 1.0, 8, 20, 20, 0.0, None, 0,
                                None) == -1
    assert L.lb_lora_wgrad_pair(p, p, p, 64, 1, 64, p, p, p, 1, 20, 64, None, 1.0, 8, 20, 24, 0.0, None, 0,
                                None) == -1
    assert L.lb_lora_wgrad_pair(p, p, p, 64, 1, 64, p, p, p, 1, 40, 64, None, 1.0, 8, 40, 32, 0.0, None, 0,
                                None) == -2
    from lora_b200.ops import _WgProblemC
    batch = lambda r, rp: L.lb_lora_wgrad_batch(
        (_WgProblemC * 1)(_WgProblemC(base, base, base, 64, 1, 8, 64, r, 1.0, None, 0.0, None, 0, 0, 0, 0, 0, 0, rp)),
        1, 0, None)
    assert batch(20, 24) == -1 and batch(40, 32) == -2
    assert L.lb_lora_up_dropout(p, 0, p, p, 1, 1, None, 1.0, 0.0, p, 8, 64, 40, 32, None) == -2
    assert L.lb_lora_up_dropout(p, 0, p, p, 1, 1, None, 1.0, 0.0, p, 8, 64, 20, 8, None) == -1
    assert L.lb_lora_up_dropout(p, 0, p, p, 1, 1, None, 1.0, 0.0, p, 8, 64, 20, 24, None) == -1
    assert L.lb_lora_dropout_dt(p, 0, p, 1, 1, 0.0, p, p, 8, 64, 65, 64, None) == -2
    assert L.lb_lora_dropout_dt(p, 0, p, 1, 1, 0.0, p, p, 8, 64, 20, 40, None) == -1
    assert L.lb_lora_dropout_dt(p, 0, p, 1, 1, 0.0, p, p, 8, 64, 20, 24, None) == -1
    assert L.lb_cast_rows_pad(p, 1, 1, p, 20, 32, 64, 2, None) == -3
    assert L.lb_cast_rows_pad(p, 1, 1, p, 40, 32, 64, 0, None) == -2
    assert L.lb_cast_rows_pad(p, 1, 1, p, 20, 20, 64, 0, None) == -1
    assert L.lb_cast_rows_pad(p, 1, 1, p, 20, 24, 64, 0, None) == -1
    assert L.lb_refresh_shadows(p, p, 0, 64, p, 0, None) == -1
    assert L.lb_lora_merge(p, 0, p, p, 1.0, p, 8, 64, 65, None) == -2
    # a pad of 16 keeps the rank limit of 16
    assert L.lb_cast_rows_pad(p, 1, 1, p, 17, 16, 64, 0, None) == -2
    assert L.lb_lora_wgrad(p, p, None, 1.0, p, 1, 1, 8, 64, 17, 16, 0, None) == -2
    assert L.lb_abi_version() == 6


def test_rank_pad():
    from lora_b200 import ops
    from lora_b200._C import LoraB200Error
    assert [ops.rank_pad(r) for r in (1, 16, 17, 32, 33, 64)] == [16, 16, 32, 32, 64, 64]
    for r in (0, 65):
        with pytest.raises(LoraB200Error):
            ops.rank_pad(r)
