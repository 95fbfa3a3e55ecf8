"""ctypes binding of libdinov3_b200.so (the C ABI declared in include/dinov3_b200.h).

There is deliberately no fallback: if the shared library is missing, or the process has no sm_90 GPU, every
entry point raises.  PyTorch tensors are only containers for device memory here (``tensor.data_ptr()``).
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import torch

_LIB = None
_INIT_DEVICE = None

PKG_ROOT = Path(__file__).resolve().parent.parent  # .../dinov3-jax_b200
LIB_PATH = PKG_ROOT / "libdinov3_b200.so"

# epilogue flags (include/dinov3_b200.h)
EP_BIAS, EP_GELU, EP_STORE_PRE, EP_MUL_DGELU, EP_GAMMA, EP_RESID, EP_OUT_F32, EP_ACCUM = 1, 2, 4, 8, 16, 32, 64, 128
EP_SCATTER = 256


class NativeError(RuntimeError):
    pass


class GemmEpilogue(C.Structure):
    _fields_ = [
        ("bias", C.c_void_p), ("gamma", C.c_void_p), ("resid", C.c_void_p), ("aux_in", C.c_void_p),
        ("aux_out", C.c_void_p), ("out", C.c_void_p),
        ("ld_out", C.c_int), ("ld_aux", C.c_int), ("ld_resid", C.c_int), ("flags", C.c_int), ("alpha", C.c_float),
        ("sc_peer", C.c_void_p * 8), ("sc_off", C.c_longlong), ("sc_shard", C.c_int), ("sc_world", C.c_int),
    ]


P, I, LL, F = C.c_void_p, C.c_int, C.c_longlong, C.c_float
# name -> argtypes, mirrors include/dinov3_b200.h (tests/test_abi.py checks every declared symbol is exported)
SIGNATURES = {
    "d3_init": [I],
    "d3_set_sm_limit": [I],
    "d3_gemm_bf16": [P, I, I, P, I, I, I, I, I, C.POINTER(GemmEpilogue), I, I, P],
    "d3_scatter_add_peers": [P, LL, P, I, LL, I, F, P],
    "d3_allreduce_peers": [P, I, P, LL, I, P],
    "d3_set_scatter_mode": [I],
    "d3_im2col": [P, P, I, I, I, I, I, P],
    "d3_assemble_tokens": [P, P, P, P, P, P, I, I, I, I, P],
    "d3_assemble_tokens_bwd": [P, P, P, P, P, P, I, I, I, I, P],
    "d3_layernorm_fwd": [P, P, P, P, I, P, P, I, I, F, P],
    "d3_layernorm_bwd_ls": [P, I, P, P, P, P, P, P, P, P, I, I, P, P, I, P, P, P, P],
    "d3_ls_gamma_from_wgrad": [P, P, P, P, P, P, I, I, P],
    "d3_rope": [P, P, P, LL, I, I, I, I, I, P],
    "d3_attn_fwd": [P, P, P, I, I, I, I, P],
    "d3_debug_attn_trace": [P],
    "d3_attn_bwd": [P, P, P, P, P, P, I, I, I, I, P, P, I, P],
    "d3_token_rows": [P, P, I, I, I, I, P],
    "d3_gather_rows": [P, P, P, P, I, I, P],
    "d3_scatter_add_rows": [P, I, P, P, I, I, P],
    "d3_l2norm_fwd": [P, P, P, I, I, F, P],
    "d3_l2norm_bwd": [P, P, P, P, I, I, F, P],
    "d3_ls_act_bwd": [P, P, P, P, P, P, I, I, I, P],
    "d3_colsum_bf16": [P, P, LL, I, I, P],
    "d3_cast_f32_bf16": [P, P, LL, P],
    "d3_swiglu_fwd": [P, P, LL, I, P],
    "d3_swiglu_bwd": [P, P, P, LL, I, P],
    "d3_absmax": [P, LL, P, P],
    "d3_colmax": [P, P, I, I, P],
    "d3_sinkhorn_colsum": [P, P, F, P, P, I, I, P],
    "d3_sinkhorn_rowsum": [P, P, F, P, P, P, I, I, P],
    "d3_sinkhorn_probs": [P, P, F, P, P, P, P, I, I, P],
    "d3_colsum_f32": [P, P, I, I, P],
    "d3_center_update": [P, P, P, F, F, P, I, P],
    "d3_ce_fwd_bwd": [P, F, P, P, F, P, P, P, P, P, P, P, P, P, P, I, I, P],
    "d3_gram_diff": [P, P, P, LL, I, F, P, I, I, P],
    "d3_resize_tokens_bicubic": [P, P, I, I, I, I, I, I, I, P],
    "d3_koleo_fwd_bwd": [P, P, P, P, P, P, P, I, I, F, F, F, P],
    "d3_koleo_fwd_bwd_rows": [P, P, P, P, P, P, P, I, I, I, I, F, F, F, P],
    "d3_aug_resized_crop": [P, I, I, I, P, I, P, I, P],
    "d3_aug_color": [P, P, I, I, P, P],
    "d3_aug_blur": [P, P, P, P, I, I, P],
    "d3_aug_finish": [P, P, P, I, I, C.POINTER(C.c_float), C.POINTER(C.c_float), P],
    "d3_sumsq": [P, LL, P, P],
    "d3_ema": [P, P, P, LL, LL, F, P],
    "d3_adamw_ema": [P, P, P, P, P, P, P, LL, P, I, LL, P, F, F, F, F, F, F, F, I, F, P],
}
NO_ARG_SYMBOLS = ["d3_last_error", "d3_abi_version", "d3_launch_count", "d3_reset_launch_count"]


def lib() -> C.CDLL:
    """Load the shared library (no GPU needed for loading / symbol checks)."""
    global _LIB
    if _LIB is None:
        path = os.environ.get("DINOV3_B200_LIB", str(LIB_PATH))
        if not os.path.exists(path):
            raise NativeError(
                f"{path} not found: build it with `python __graft_entry__.py` (nvcc, sm_90a). "
                "There is no CPU / PyTorch fallback for the training hot path.")
        _LIB = C.CDLL(path)
        _LIB.d3_last_error.restype = C.c_char_p
        _LIB.d3_launch_count.restype = C.c_longlong
        for name, args in SIGNATURES.items():
            fn = getattr(_LIB, name)
            fn.argtypes = args
            fn.restype = C.c_int
    return _LIB


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        raise NativeError(f"{what} failed ({rc}): {lib().d3_last_error().decode()}")


def init(device: int | None = None) -> C.CDLL:
    """Bind the library to a CUDA device; raises if it is not a Hopper (sm_90) part."""
    global _INIT_DEVICE
    l = lib()
    if not torch.cuda.is_available():
        raise NativeError("no CUDA device: the dinov3 GPU engine has no CPU fallback")
    if device is None:
        device = torch.cuda.current_device()
    if _INIT_DEVICE != device:
        check(l.d3_init(int(device)), "d3_init")
        _INIT_DEVICE = device
    return l


def stream_ptr() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t: torch.Tensor | None) -> C.c_void_p:
    return C.c_void_p(0 if t is None else t.data_ptr())


def launch_count() -> int:
    return int(lib().d3_launch_count())


def reset_launch_count() -> None:
    lib().d3_reset_launch_count()
