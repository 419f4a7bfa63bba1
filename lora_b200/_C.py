"""ctypes binding of the C-ABI in include/lora_b200.h.

The library is the product: there is no CPU or eager fallback behind these calls. The first call
without a built liblora_b200.so raises, and every wrapper raises on a non-zero status.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblora_b200.so")

LB_BF16, LB_F16, LB_F32 = 0, 1, 2

_STATUS = {
    0: "LB_OK", -1: "LB_ERR_SHAPE", -2: "LB_ERR_RANK", -3: "LB_ERR_DTYPE",
    -4: "LB_ERR_ALIGN", -5: "LB_ERR_TMAP", -6: "LB_ERR_CUDA",
}


class LoraB200Error(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH) and LIB_PATH == os.path.join(_HERE, "liblora_b200.so"):
        # fresh checkout: the library is a build artefact (git-ignored). Build it once, in-tree.
        try:
            from .build import build
            build()
        except Exception as e:  # nvcc missing or compile error: there is nothing to fall back to
            raise LoraB200Error(
                f"{LIB_PATH} is missing and building it failed ({e}); run `python -m lora_b200.build` "
                "(nvcc, sm_90a). lora_b200 has no fallback path.") from e
    if not os.path.exists(LIB_PATH):
        raise LoraB200Error(
            f"{LIB_PATH} is missing: build it with `python -m lora_b200.build` "
            "(nvcc, sm_90a). lora_b200 has no fallback path."
        )
    lib = ctypes.CDLL(LIB_PATH)
    vp, ll, i32, f32 = ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_float
    sig = {
        "lb_abi_version": ([], i32),
        "lb_lora_linear_fwd": ([vp, vp, vp, vp, vp, ll, ll, vp, f32, vp, vp, vp,
                                i32, i32, i32, i32, i32, i32, i32, vp], i32),
        "lb_lora_linear_fwd_dropout": ([vp, vp, vp, vp, vp, ll, ll, vp, f32, vp, vp,
                                        i32, i32, i32, i32, i32, i32, i32, f32, vp, vp], i32),
        "lb_lora_conv2d_fwd_dropout": ([vp, vp, vp, vp, vp, ll, ll, vp, f32, vp, vp,
                                        i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32,
                                        f32, vp, vp], i32),
        "lb_tiled_weight_elems": ([i32, i32], ll),
        "lb_tile_weight": ([vp, i32, ll, ll, i32, i32, vp, i32, vp], i32),
        "lb_lora_wgrad": ([vp, vp, vp, f32, vp, ll, ll, i32, i32, i32, i32, i32, vp], i32),
        "lb_cast_rows_pad": ([vp, ll, ll, vp, i32, i32, i32, i32, vp], i32),
        "lb_cast_weight": ([vp, i32, vp, vp, i32, i32, i32, vp], i32),
        "lb_adamw_clip_step": ([vp, vp, vp, vp, ll, ctypes.POINTER(ll), i32, vp, f32, f32, f32,
                                f32, f32, f32, vp, vp, vp, vp], i32),
        "lb_optim_step_fused": ([vp, vp, vp, vp, ll, ctypes.POINTER(ll), i32, vp, f32, f32, f32,
                                 f32, f32, f32, vp, vp, vp, vp, i32, i32, vp, i32, vp, vp], i32),
        "lb_step_prologue": ([vp, vp, vp, vp, vp, i32, vp, vp, vp, i32, i32, i32, i32, i32, vp], i32),
        "lb_step_prologue_v": ([vp, vp, vp, vp, vp, i32, vp, vp, vp, i32, vp, i32, i32, i32, i32, vp], i32),
        "lb_masked_mse_fwd_bwd": ([vp, i32, ll, ll, ll, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, vp], i32),
        "lb_optim_step_dp": ([vp, vp, vp, vp, vp, ll, ctypes.POINTER(ll), i32, vp, f32, f32, f32, f32, f32,
                              vp, vp, vp, vp, i32, i32, vp, i32, vp, vp, vp, i32, i32, vp, vp], i32),
        "lb_ipc_export": ([vp, vp, ctypes.POINTER(ll)], i32),
        "lb_ipc_open": ([vp, ctypes.POINTER(vp)], i32),
        "lb_lora_wgrad_batch": ([vp, i32, i32, vp], i32),
        "lb_refresh_shadows": ([vp, vp, i32, i32, vp, i32, vp], i32),
        "lb_debug_set_linear_mode": ([i32], i32),
        "lb_lora_wgrad_conv": ([vp, vp, vp, f32, vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32,
                                vp], i32),
        "lb_lora_wgrad_multi": ([i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, vp], i32),
        "lb_lora_linear_fwd_grouped": ([i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp,
                                        i32, i32, vp], i32),
        "lb_ti_embed_step": ([vp, vp, vp, vp, vp, vp, i32, i32, i32, vp, f32, f32, f32, f32, vp, i32, f32, vp], i32),
        "lb_embed_rows_scatter": ([vp, vp, i32, i32, i32, i32, vp, vp, i32, vp, vp, i32, vp, vp, vp, vp], i32),
        "lb_embed_rows_scatter_dp": ([vp, i32, i32, i32, vp, i32, i32, i32, vp, vp, i32, vp, vp, i32, vp, vp, vp,
                                      vp, vp, vp], i32),
        "lb_embed_rows_write_back": ([vp, vp, i32, vp, i32, vp, i32, i32, i32, vp, vp, i32, f32, vp], i32),
        "lb_embed_rows_flush": ([vp, i32, i32, i32, vp, vp, vp, vp], i32),
        "lb_lora_merge": ([vp, i32, vp, vp, f32, vp, i32, i32, i32, vp], i32),
        "lb_split_bf16x3": ([vp, ll, vp, i32, i32, i32, vp], i32),
        "lb_debug_set_stamp_buffer": ([vp], i32),
        "lb_debug_set_pdl": ([i32], i32),
        "lb_lora_wgrad_pair": ([vp, vp, vp, ll, ll, i32, vp, vp, vp, ll, ll, i32, vp, f32, i32, i32, i32,
                                f32, vp, i32, vp], i32),
        "lb_svd_workspace_bytes": ([ctypes.POINTER(i32), ctypes.POINTER(i32), i32, i32], ll),
        "lb_svd_truncated_batched": ([vp, vp, ctypes.POINTER(i32), ctypes.POINTER(i32), i32, i32, i32, i32, f32,
                                      ctypes.c_ulonglong, vp, vp, vp, vp, ll, vp], i32),
        "lb_svd_mul": ([vp, vp, i32, vp, vp, i32, i32, i32, i32, vp], i32),
        "lb_svd_gram": ([vp, vp, i32, i32, vp], i32),
        "lb_svd_chol_inv": ([vp, vp, i32, vp], i32),
        "lb_svd_apply": ([vp, vp, vp, i32, vp, i32, i32, ll, i32, ll, i32, vp], i32),
        "lb_svd_jacobi": ([vp, vp, vp, i32, i32, vp], i32),
        "lb_svd_randn": ([vp, ll, ctypes.c_ulonglong, vp], i32),
        "lb_lora_conv2d_fwd": ([vp, vp, vp, vp, vp, ll, ll, ll, vp, f32, vp, vp, vp,
                                i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32,
                                vp], i32),
        "lb_cast_conv_weight": ([vp, i32, vp, vp, i32, i32, i32, i32, i32, vp], i32),
        "lb_lora_up_dropout": ([vp, i32, vp, vp, ll, ll, vp, f32, f32, vp, i32, i32, i32, i32, vp], i32),
        "lb_lora_dropout_dt": ([vp, i32, vp, ll, ll, f32, vp, vp, i32, i32, i32, i32, vp], i32),
        "lb_lora_wgrad_masked": ([vp, vp, vp, f32, vp, ll, ll, i32, i32, i32, i32, f32, vp, i32, vp], i32),
    }
    for name, s in sig.items():
        if s is None or not hasattr(lib, name):
            continue
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = s
    return lib


class _LazyLib:
    """The library is mapped on first use (first kernel call, `build()`'s symbol check), not at
    `import lora_b200`: the host-side file tools (persist, lora_add, join, to_ckpt,
    pt_to_safetensors) and anything that only needs the host models import without a CUDA
    toolchain or runtime, like the reference's package. There is still no fallback: the first
    kernel call without a loadable library raises LoraB200Error."""
    _lib = None

    def __getattr__(self, name):
        lib = _LazyLib._lib
        if lib is None:
            lib = _LazyLib._lib = _load()
        return getattr(lib, name)


lib = _LazyLib()


def is_loaded() -> bool:
    return _LazyLib._lib is not None
EXPORTED = [n for n in ("lb_abi_version", "lb_lora_linear_fwd", "lb_lora_wgrad",
                        "lb_cast_rows_pad", "lb_cast_weight", "lb_adamw_clip_step",
                        "lb_refresh_shadows", "lb_lora_conv2d_fwd",
                        "lb_cast_conv_weight", "lb_lora_up_dropout", "lb_lora_dropout_dt",
                        "lb_lora_wgrad_masked", "lb_lora_wgrad_pair", "lb_svd_mul", "lb_svd_gram",
                        "lb_svd_chol_inv", "lb_svd_apply", "lb_svd_jacobi", "lb_svd_randn", "lb_split_bf16x3", "lb_lora_merge", "lb_ti_embed_step",
                        "lb_embed_rows_scatter", "lb_embed_rows_scatter_dp", "lb_embed_rows_write_back", "lb_embed_rows_flush", "lb_lora_linear_fwd_grouped", "lb_lora_wgrad_multi", "lb_lora_wgrad_conv",
                        "lb_lora_linear_fwd_dropout", "lb_lora_conv2d_fwd_dropout", "lb_debug_set_pdl", "lb_svd_workspace_bytes", "lb_svd_truncated_batched",
                        "lb_optim_step_fused", "lb_step_prologue", "lb_step_prologue_v", "lb_masked_mse_fwd_bwd",
                        "lb_optim_step_dp", "lb_ipc_export", "lb_ipc_open", "lb_lora_wgrad_batch", "lb_tiled_weight_elems", "lb_tile_weight")]


def check(status: int, what: str):
    if status != 0:
        raise LoraB200Error(f"{what} failed: {_STATUS.get(status, status)}")


def dtype_code(torch_dtype):
    import torch
    if torch_dtype == torch.bfloat16:
        return LB_BF16
    if torch_dtype == torch.float16:
        return LB_F16
    if torch_dtype == torch.float32:
        return LB_F32
    raise LoraB200Error(f"unsupported dtype {torch_dtype}")


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
