"""ctypes binding of libfresco_b200.so (the C ABI declared in include/fresco_b200.h).

There is deliberately no fallback: if the shared library is missing or a call
fails, the caller gets an exception.  torch is used only for device memory and
streams (``tensor.data_ptr()``, ``torch.cuda.current_stream()``).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_int64, c_longlong, c_size_t, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# FRESCO_B200_LIB: measurement tools only (A/B builds made with FRESCO_BUILD_TAG); the product is libfresco_b200.so
LIB_PATH = os.environ.get("FRESCO_B200_LIB") or os.path.join(_HERE, "libfresco_b200.so")

_P = c_void_p
_SIGNATURES = {
    "fresco_abi_version": (c_int, []),
    "fresco_last_error": (c_char_p, []),
    "fresco_launch_count": (c_longlong, []),
    "fresco_last_kernel": (c_char_p, []),
    "fresco_set_option": (c_int, [c_char_p, c_int]),
    "fresco_attn_variant": (c_char_p, [c_int]),
    "fresco_kv_compact": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    "fresco_attn_fwd": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_float, _P]),
    "fresco_attn_fwd_kv_strided": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_longlong, c_longlong,
                                           c_float, c_float, _P]),
    "fresco_kv_compact_packed": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "fresco_rows_gather": (c_int, [_P, _P, _P, c_longlong, c_int, c_int, c_int, _P]),
    "fresco_rows_scatter": (c_int, [_P, _P, _P, c_longlong, c_int, _P]),
    "fresco_temporal_attn_fwd_strided": (c_int, [_P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_float, _P]),
    "fresco_temporal_attn_fwd": (c_int, [_P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float, _P]),
    "fresco_flow_warp": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "fresco_warp_fuse_chain": (c_int, [_P, _P, c_int, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "fresco_warp_taps": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P]),
    "fresco_warp_loss_fwd_bwd": (c_int, [_P] * 8 + [c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "fresco_warp_loss_fwd_bwd_halo": (c_int, [_P] * 8 + [c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P,
                                              c_int, _P]),
    "fresco_gram_normalize": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P]),
    "fresco_gram_sign": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_float, _P]),
    "fresco_gram_grad": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_float, _P, c_size_t, _P]),
    "fresco_gram_grad_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "fresco_gram_sign_ref": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_float, _P]),
    "fresco_gram_tx": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_float, _P]),
    "fresco_gram_sign_scaled": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_double, _P]),
    "fresco_gram_sign_ref_scaled": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_double, _P]),
    "fresco_gram_grad_scaled": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_double, _P, c_size_t, _P]),
    "fresco_adam_step": (c_int, [_P, _P, _P, _P, c_longlong, c_int, c_double, c_double, c_double, c_double, _P]),
    "fresco_adain": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P]),
    "gmflow_global_corr_softmax": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P, c_size_t, _P]),
    "fresco_gmflow_corr_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "gmflow_flow_attention": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_float, _P]),
    "fresco_dilate": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    "fresco_cfg_pred_x0": (c_int, [_P, _P, _P, _P, c_int, c_longlong, c_float, c_float, _P]),
    "fresco_ddpm_prev": (c_int, [_P, _P, _P, _P, c_int, c_longlong, c_longlong, c_int, c_float, c_float, c_float, _P]),
    "fresco_mapping_single": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P, _P, _P, c_size_t, _P]),
    "fresco_mapping_workspace_bytes": (c_size_t, [c_int]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


class FrescoError(RuntimeError):
    pass


_lib = None


def lib() -> ctypes.CDLL:
    """Load the shared library (once).  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FrescoError(
                f"{LIB_PATH} is missing: build it with `python -m fresco_b200.build` "
                "(there is no CPU / PyTorch fallback for the FRESCO kernels)")
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        if l.fresco_abi_version() != 1:
            raise FrescoError("libfresco_b200.so ABI version mismatch")
        _lib = l
    return _lib


def last_error() -> str:
    return (lib().fresco_last_error() or b"").decode()


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise FrescoError(f"{what} failed ({rc}): {last_error()}")


def ptr(t: torch.Tensor) -> int:
    if not t.is_cuda:
        raise FrescoError("fresco_b200 kernels need CUDA tensors (no CPU fallback)")
    if not t.is_contiguous():
        raise FrescoError("fresco_b200 kernels need contiguous tensors")
    return t.data_ptr()


def stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def set_option(name: str, value: int) -> None:
    """Override a tuning option (named like its environment variable); value < 0 restores the default."""
    check(lib().fresco_set_option(name.encode(), int(value)), "fresco_set_option")


def launch_count() -> int:
    return int(lib().fresco_launch_count())


def last_kernel() -> str:
    """Name of the last kernel the library launched on this thread, template arguments included."""
    return (lib().fresco_last_kernel() or b"").decode()
