"""ctypes binding of libvidtome_b200.so (the C-ABI declared in include/vidtome_b200.h).

There is no fallback of any kind: if the shared library has not been built, or a compute entry point
reports an error, a RuntimeError is raised.  Build with `python -m vidtome_b200._build` (or
`__graft_entry__.build()`).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
# VIDTOME_B200_LIB: load another build of the SAME library (e.g. for an A/B comparison of two builds); never a fallback
LIB_PATH = os.environ.get("VIDTOME_B200_LIB") or os.path.join(_HERE, "libvidtome_b200.so")


class VtmSplit(C.Structure):
    """struct vtm_split (include/vidtome_b200.h)."""
    _fields_ = [(n, C.c_int32) for n in
                ("mode", "N", "unm_pre", "F", "tnum", "stride", "randf", "src_len")] + [
                    ("randf_dev", C.c_void_p), ("coin_dev", C.c_void_p), ("coin_threshold", C.c_double)]

    @classmethod
    def local(cls, N: int, unm_pre: int, F: int, target_stride: int, randf) -> "VtmSplit":
        """`randf`: the drawn int, or a 1-element int32 CUDA tensor holding it (kept alive on the descriptor) when
        the draw stays on the device (CUDA-graph capture; needs F % stride == 0)."""
        tnum = (N - unm_pre) // F                      # merge.py:43
        stride = min(target_stride, F)                 # merge.py:55
        if isinstance(randf, int):
            return cls(0, N, unm_pre, F, tnum, stride, randf, 0, None)
        import torch
        if not (isinstance(randf, torch.Tensor) and randf.is_cuda and randf.dtype == torch.int32 and randf.numel() == 1):
            raise RuntimeError("VtmSplit.local: randf must be an int or a 1-element int32 CUDA tensor")
        sp = cls(0, N, unm_pre, F, tnum, stride, 0, 0, randf.data_ptr())
        sp._keepalive = randf
        return sp

    @classmethod
    def prefix(cls, N: int, src_len: int) -> "VtmSplit":
        return cls(1, N, 0, 0, 0, 0, 0, src_len, None)

    @classmethod
    def prefix_coin(cls, L: int, coin, global_rand: float) -> "VtmSplit":
        """The global stage's split with its coin left on the device: the sequence is stored as [local (L rows) |
        global (L rows)], and the kernels read `coin` (a 1-element fp32 CUDA tensor, kept alive on the descriptor)
        to pick the roles.  coin > global_rand: src = local, dst = global; otherwise src = global, dst = local."""
        import torch
        if not (isinstance(coin, torch.Tensor) and coin.is_cuda and coin.dtype == torch.float32 and coin.numel() == 1):
            raise RuntimeError("VtmSplit.prefix_coin: coin must be a 1-element float32 CUDA tensor")
        if not isinstance(L, int) or L <= 0:
            raise RuntimeError(f"VtmSplit.prefix_coin: L must be a positive int, got {L!r}")
        sp = cls(1, 2 * L, 0, 0, 0, 0, 0, L, None, coin.data_ptr(), float(global_rand))
        sp._keepalive = coin
        return sp


    @classmethod
    def prefix_coin_dev(cls, L: int, glob_len_dev, glob_cap: int, coin, global_rand: float) -> "VtmSplitDev":
        """The global stage's split when the two token sets may differ in length (mode 2): the sequence is stored as
        [local (L rows) | global (*glob_len_dev rows, at most glob_cap)], and the coin picks the src half as in
        prefix_coin.  The counts that follow from the draw (Ns, Nd, r, the merged length) stay on the device
        (ops.split_counts_dev); `glob_len_dev` is a 1-element int32 CUDA tensor, kept alive on the descriptor with
        the coin."""
        import torch
        if not (isinstance(coin, torch.Tensor) and coin.is_cuda and coin.dtype == torch.float32 and coin.numel() == 1):
            raise RuntimeError("VtmSplit.prefix_coin_dev: coin must be a 1-element float32 CUDA tensor")
        if not (isinstance(glob_len_dev, torch.Tensor) and glob_len_dev.is_cuda and glob_len_dev.dtype == torch.int32
                and glob_len_dev.numel() == 1):
            raise RuntimeError("VtmSplit.prefix_coin_dev: glob_len_dev must be a 1-element int32 CUDA tensor")
        if not isinstance(L, int) or L <= 0 or not isinstance(glob_cap, int) or glob_cap <= 0:
            raise RuntimeError(f"VtmSplit.prefix_coin_dev: L and glob_cap must be positive ints, got {L!r}, {glob_cap!r}")
        sp = VtmSplitDev(2, L + glob_cap, 0, 0, 0, 0, 0, L, None, coin.data_ptr(), float(global_rand),
                         glob_len_dev.data_ptr(), glob_cap)
        sp._keepalive = (coin, glob_len_dev)
        return sp


class VtmSplitDev(VtmSplit):
    """struct vtm_split with its mode-2 tail (glob_len_dev, glob_cap): the full C layout.  The library reads the tail
    only for mode 2, so VtmSplit itself keeps the shorter layout for modes 0 and 1."""
    _fields_ = [("glob_len_dev", C.c_void_p), ("glob_cap", C.c_int32)]


class VtmLora(C.Structure):
    """struct vtm_lora_t (include/vidtome_b200.h): a GEMM's stacked LoRA adapters, down D [R, K] and up U [N, R]."""
    _fields_ = [("down_dev", C.c_void_p), ("up_dev", C.c_void_p), ("R", C.c_int32)]


_vp, _i32, _i64, _sz = C.c_void_p, C.c_int32, C.c_int64, C.c_size_t
_SPL = C.POINTER(VtmSplit)
_LORA = C.POINTER(VtmLora)

# name -> (restype, argtypes); mirrors include/vidtome_b200.h one to one
SIGNATURES = {
    "vtm_version": (C.c_int, []),
    "vtm_error_string": (C.c_char_p, [C.c_int]),
    "vtm_split_counts": (C.c_int, [_SPL, C.POINTER(_i32), C.POINTER(_i32)]),
    "vtm_merge_count": (_i32, [_i32, C.c_double]),
    "vtm_normalize_split": (C.c_int, [_vp, _i64, _vp, _i64, _SPL, _i32, _i32, _vp, _vp, _vp]),
    "vtm_normalize_split_ln": (C.c_int, [_vp, _i64, _vp, _i64, _SPL, _i32, _i32, _vp, _vp, C.c_float, _vp, _vp, _vp]),
    "vtm_gather_rows_ln": (C.c_int, [_vp, _i64, _vp, _i64, _i32, _i32, _i32, _vp, _vp, C.c_float, _vp, _i64, _vp]),
    "vtm_gather_rows_peers": (C.c_int, [_vp, _i64, _vp, _i64, _i32, _i32, _i32, _vp, _vp, C.c_float, _vp, _i64,
                                        C.POINTER(C.c_void_p), _i32, _vp]),
    "vtm_sim_argmax": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp]),
    "vtm_sim_argmax_simt": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp]),
    "vtm_key_score_half_bits": (C.c_uint16, [C.c_uint64]),
    "vtm_key_arg": (C.c_uint32, [C.c_uint64]),
    "vtm_topr_workspace_bytes": (_sz, [_i32, _i32]),
    "vtm_topr_sort": (C.c_int, [_vp, _i32, _i32, _vp, _vp, _vp, _sz, _vp]),
    "vtm_compose_maps": (C.c_int, [_SPL, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _i32, _i32,
                                   _vp, _vp, _vp]),
    "vtm_decode_match": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vtm_gather_rows": (C.c_int, [_vp, _i64, _vp, _i64, _i32, _i32, _i32, _vp, _i64, _vp]),
    "vtm_merge_reduce_workspace_bytes": (_sz, [_i32, _i32, _i32]),
    "vtm_merge_reduce": (C.c_int, [_vp, _i64, _SPL, _i32, _i32, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _sz, _vp]),
    "vtm_unmerge_add": (C.c_int, [_vp, _i64, _vp, _i64, _vp, _i32, _i32, _i32, _vp, _vp]),
    "vtm_attention_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32]),
    "vtm_attention": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, C.c_float, _vp, _vp, _sz, _vp]),
    "vtm_attention_ex": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, C.c_float, _i32, _vp, _vp, _sz, _vp]),
    "vtm_cross_attention_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32, _i32]),
    "vtm_cross_attention": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, C.c_float,
                                      _vp, _vp, _sz, _vp]),
    "vtm_split_counts_dev": (C.c_int, [_SPL, C.c_double, _vp, _vp]),
    "vtm_sim_argmax_dev": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "vtm_topr_sort_dev": (C.c_int, [_vp, _i32, _i32, _vp, _vp, _vp, _vp, _sz, _vp]),
    "vtm_compose_maps_dev": (C.c_int, [_SPL, _vp, _i32, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp]),
    "vtm_gather_rows_dev": (C.c_int, [_vp, _i64, _vp, _i64, _i32, _i32, _i32, _vp, _vp, _i64, _vp]),
    "vtm_attention_dev": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, C.c_float, _i32, _vp, _vp, _vp, _sz,
                                    _vp]),
    "vtm_linear_f16": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _vp, _i64, _vp]),
    "vtm_linear_geglu_f16": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _vp, _i64, _vp]),
    "vtm_linear_residual_f16": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _vp, _i64, _vp]),
    "vtm_linear_lora_workspace_bytes": (_sz, [_i32, _i32]),
    "vtm_linear_lora_f16": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _LORA, _i32, _i32, _i32, _vp, _i64, _vp, _sz, _vp]),
    "vtm_linear_geglu_lora_f16": (C.c_int, [_vp, _vp, _vp, _LORA, _i32, _i32, _i32, _vp, _i64, _vp, _sz, _vp]),
    "vtm_attention_lora_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32, _i32, _i32]),
    "vtm_attention_lora": (C.c_int, [_vp, _vp, _vp, _vp, _LORA, _LORA, _i32, _i32, _i32, _i32, C.c_float, _i32, _vp,
                                     _vp, _vp, _sz, _vp]),
    "vtm_cross_attention_lora_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32]),
    "vtm_cross_attention_lora": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _LORA, _LORA, _LORA, _i32, _i32, _i32,
                                           _i32, _i32, _i32, C.c_float, _vp, _vp, _sz, _vp]),
    "vtm_resnet_tail_f16": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i64, C.c_float, _i32, _vp]),
    "vtm_attention_residual": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _LORA, _LORA, _i32, _i32, _i32, _i32, C.c_float, _vp,
                                         _vp, _sz, _vp]),
    "vtm_attention_residual_ex": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _LORA, _LORA, _i32, _i32, _i32, _i32, C.c_float,
                                            _i32, _i32, _vp, _vp, _sz, _vp]),
    "vtm_ddim_update_f16": (C.c_int, [_vp, _vp, _i64, _vp, _vp, _vp, _i32, _vp, _i32, _vp]),
    "vtm_cfg_ddim_update_f16": (C.c_int, [_vp, _vp, _i64, _i32, C.c_float, _vp, _vp, _i32, _vp, _vp]),
    "vtm_group_norm_stats_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32]),
    "vtm_group_norm_stats_f16": (C.c_int, [_vp, _i32, _i32, _i32, _i32, C.c_float, _vp, _vp, _sz, _vp]),
    "vtm_group_norm_tokens_f16": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "vtm_linear_nchw_residual_f16": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
}

_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """Load the library once and attach the declared signatures.  Raises if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"vidtome_b200: {LIB_PATH} is missing. The CUDA extension is the only implementation of "
            "this path (no CPU/PyTorch fallback); build it with `python -m vidtome_b200._build`.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)      # AttributeError here = header/library mismatch: fail loudly
        fn.restype, fn.argtypes = res, args
    if lib.vtm_version() != 100:
        raise RuntimeError(f"vidtome_b200: library version {lib.vtm_version()} != 100")
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().vtm_error_string(rc).decode()
        raise RuntimeError(f"vidtome_b200: {what} failed with code {rc}: {msg}")
