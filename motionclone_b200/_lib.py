"""ctypes binding of the C ABI in include/motionclone_b200.h (libmotionclone_b200.so, built in-tree by
__graft_entry__.build()). There is NO fallback: a missing library or a failing kernel raises."""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_int64, c_uint8, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
# The one library this package loads (A/B scripts may point this attribute at a side-by-side build of the same sources
# BEFORE the first call; nothing in the package or in the environment selects a library).
LIB_PATH = os.path.join(_HERE, "libmotionclone_b200.so")


class TemporalLayout(Structure):
    """mc_temporal_layout: element strides of (batch, frame, position); channels are contiguous."""
    _fields_ = [("stride_b", c_int64), ("stride_f", c_int64), ("stride_p", c_int64)]


class MotionCloneKernelError(RuntimeError):
    pass


_lib = None

EXPORTS = ("mc_abi_version", "mc_last_error", "mc_launch_count", "mc_reset_launch_count", "mc_add_launch_count", "mc_temporal_attn_fwd",
           "mc_temporal_attn_bwd", "mc_top1_rows", "mc_motion_loss_fwd", "mc_motion_loss_bwd", "mc_cfg_ddim_step", "mc_ddim_step_ex",
           "mc_add_noise", "mc_groupnorm_workspace_bytes", "mc_groupnorm_nhwc", "mc_layernorm", "mc_geglu", "mc_groupnorm_nhwc_stats", "mc_groupnorm_nhwc_bwd", "mc_layernorm_bwd",
           "mc_groupnorm_nhwc_batched", "mc_groupnorm_nhwc_bwd_batched", "mc_groupnorm_nhwc_pooled",
           "mc_groupnorm_nhwc_bwd_pooled",
           "mc_geglu_bwd", "mc_bias_residual_add", "mc_cross_attn_fwd", "mc_cross_attn_bwd_dq",
           "mc_spatial_attn_fwd", "mc_spatial_attn_bwd", "mc_spatial_attn_bwd_workspace_bytes")


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MotionCloneKernelError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). motionclone_b200 has no CPU or eager fallback.")
    L = ctypes.CDLL(LIB_PATH)
    P = c_void_p
    L.mc_abi_version.restype = c_int
    L.mc_last_error.restype = c_char_p
    L.mc_launch_count.restype = c_uint64
    L.mc_reset_launch_count.restype = None
    L.mc_add_launch_count.restype = None
    L.mc_add_launch_count.argtypes = [c_uint64]
    L.mc_temporal_attn_fwd.restype = c_int
    L.mc_temporal_attn_fwd.argtypes = [P, P, P, TemporalLayout, P, TemporalLayout, P, P, P, P, P,
                                       c_int, c_int, c_int, c_int, c_int, c_float, P]
    L.mc_temporal_attn_bwd.restype = c_int
    L.mc_temporal_attn_bwd.argtypes = [P, P, P, TemporalLayout, P, TemporalLayout, P, P, P, P, P, P, TemporalLayout,
                                       c_int, c_int, c_int, c_int, c_int, c_float, P]
    L.mc_top1_rows.restype = c_int
    L.mc_top1_rows.argtypes = [P, c_int64, c_int, P, P, P]
    L.mc_motion_loss_fwd.restype = c_int
    L.mc_motion_loss_fwd.argtypes = [c_int, POINTER(P), POINTER(P), POINTER(c_int64), P, P, P]
    L.mc_motion_loss_bwd.restype = c_int
    L.mc_motion_loss_bwd.argtypes = [c_int, POINTER(P), POINTER(P), POINTER(c_int64), P, POINTER(P), P]
    L.mc_cfg_ddim_step.restype = c_int
    L.mc_cfg_ddim_step.argtypes = [P, P, P, P, P, c_int64] + [c_float] * 6 + [P]
    L.mc_ddim_step_ex.restype = c_int
    L.mc_ddim_step_ex.argtypes = [P, P, P, P, P, P, P, c_int64, c_int, c_int] + [c_float] * 10 + [P]
    L.mc_add_noise.restype = c_int
    L.mc_add_noise.argtypes = [P, P, P, c_int64, c_float, c_float, P]
    L.mc_groupnorm_workspace_bytes.restype = c_int64
    L.mc_groupnorm_workspace_bytes.argtypes = [c_int, c_int]
    L.mc_groupnorm_nhwc.restype = c_int
    L.mc_groupnorm_nhwc.argtypes = [P, P, c_int, P, P, P, P, c_int64, c_int, c_int, c_int, c_int, c_float, c_int, P]
    L.mc_layernorm.restype = c_int
    L.mc_layernorm.argtypes = [P, P, P, P, P, P, c_int, c_int, c_int64, c_int, c_float, P]
    L.mc_geglu.restype = c_int
    L.mc_geglu.argtypes = [P, P, c_int64, c_int, P]
    L.mc_groupnorm_nhwc_stats.restype = c_int
    L.mc_groupnorm_nhwc_stats.argtypes = [P, P, c_int, c_int, c_int, c_float, P]
    L.mc_groupnorm_nhwc_bwd.restype = c_int
    L.mc_groupnorm_nhwc_bwd.argtypes = [P, P, c_int, P, P, P, P, P, P, c_int64, c_int, c_int, c_int, c_int, c_int, P]
    L.mc_groupnorm_nhwc_batched.restype = c_int
    L.mc_groupnorm_nhwc_batched.argtypes = [P, P, c_int, P, P, P, P, c_int64, c_int, c_int, c_int, c_int, c_int, c_float,
                                            c_int, P]
    L.mc_groupnorm_nhwc_bwd_batched.restype = c_int
    L.mc_groupnorm_nhwc_bwd_batched.argtypes = [P, P, c_int, P, P, P, P, P, P, c_int64, c_int, c_int, c_int, c_int, c_int,
                                                c_int, P]
    L.mc_groupnorm_nhwc_pooled.restype = c_int
    L.mc_groupnorm_nhwc_pooled.argtypes = [P, P, c_int, P, P, P, P, c_int64, c_int, c_int, c_int, c_int, c_int, c_int,
                                           c_float, c_int, P]
    L.mc_groupnorm_nhwc_bwd_pooled.restype = c_int
    L.mc_groupnorm_nhwc_bwd_pooled.argtypes = [P, P, c_int, P, P, P, P, P, P, c_int64, c_int, c_int, c_int, c_int, c_int,
                                               c_int, c_int, P]
    L.mc_layernorm_bwd.restype = c_int
    L.mc_layernorm_bwd.argtypes = [P, P, P, P, P, c_int64, c_int, c_float, P]
    L.mc_geglu_bwd.restype = c_int
    L.mc_geglu_bwd.argtypes = [P, P, P, c_int64, c_int, P]
    L.mc_bias_residual_add.restype = c_int
    L.mc_bias_residual_add.argtypes = [P, P, P, P, c_int64, c_int, P]
    L.mc_cross_attn_fwd.restype = c_int
    L.mc_cross_attn_fwd.argtypes = [P, P, P, P, c_int, c_int, c_int, c_int, c_int] + [c_int64] * 6 + [c_float, P]
    L.mc_cross_attn_bwd_dq.restype = c_int
    L.mc_cross_attn_bwd_dq.argtypes = [P, P, P, P, P, c_int, c_int, c_int, c_int, c_int] + [c_int64] * 8 + [c_float, P]
    L.mc_spatial_attn_fwd.restype = c_int
    L.mc_spatial_attn_fwd.argtypes = [P, P, P, P, P, c_int, c_int, c_int, c_int] + [c_int64] * 8 + [c_float, P]
    L.mc_spatial_attn_bwd_workspace_bytes.restype = c_int64
    L.mc_spatial_attn_bwd_workspace_bytes.argtypes = [c_int, c_int, c_int]
    L.mc_spatial_attn_bwd.restype = c_int
    L.mc_spatial_attn_bwd.argtypes = [P] * 10 + [c_int, c_int, c_int, c_int] + [c_int64] * 12 + [c_float, P]
    if L.mc_abi_version() != 2:
        raise MotionCloneKernelError(f"ABI version mismatch: library {L.mc_abi_version()}, binding 2")
    _lib = L
    return L


def check(status: int, what: str) -> None:
    if status != 0:
        msg = lib().mc_last_error().decode(errors="replace")
        if status == -2:
            raise NotImplementedError(f"{what}: {msg}")  # mirrors the reference's NotImplementedError (motion_module.py:286)
        raise MotionCloneKernelError(f"{what} failed (status {status}): {msg}")


def launch_count() -> int:
    return int(lib().mc_launch_count())


def reset_launch_count() -> None:
    lib().mc_reset_launch_count()


def add_launch_count(n: int) -> None:
    lib().mc_add_launch_count(int(n))
