"""ctypes binding of libpcl_b200.so (the C ABI declared in include/pcl.h).

There is no fallback: if the library is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

from . import build as _build

c_i32, c_i64, c_u64, c_f32, c_vp = C.c_int32, C.c_int64, C.c_uint64, C.c_float, C.c_void_p

PLAN_HEADER = 16
PLAN_TC, PLAN_V, PLAN_A, PLAN_FLAGS = 0, 1, 2, 3
FLAG_NO_CLASS, FLAG_ZERO_VIEWS, FLAG_SPLIT_ERROR = 1, 2, 4
CHUNK = 1024
MAX_CLASSES = 256
DT_F32, DT_BF16, DT_F16 = 0, 1, 2          # element types of embed / seg / bank keys (pcl_step_desc.embed_dtype, ...)


class PclError(RuntimeError):
    pass


class Geom(C.Structure):
    _fields_ = [("B", c_i32), ("D", c_i32), ("h", c_i32), ("w", c_i32), ("Himg", c_i32), ("Wimg", c_i32),
                ("K", c_i32), ("max_samples", c_i32), ("max_views", c_i32), ("ignore_label", c_i32)]


class SelectSizes(C.Structure):
    _fields_ = [("keys_u16", c_i64), ("chunk_pref_i32", c_i64), ("counts_i32", c_i64), ("plan_i32", c_i64),
                ("anchor_meta_i32", c_i64), ("nchunk", c_i32), ("max_pairs", c_i32)]


class SweepDesc(C.Structure):
    _fields_ = [("anchors", c_vp), ("anchor_cls", c_vp), ("diag_col", c_vp), ("plan", c_vp),
                ("a_rows", c_i32), ("D", c_i32), ("mode", c_i32),
                ("segment_queue", c_vp), ("pixel_queue", c_vp),
                ("bank_K", c_i32), ("bank_M0", c_i32), ("bank_M1", c_i32),
                ("contrast", c_vp), ("contrast_cls", c_vp), ("n_cols", c_i32),
                ("temperature", c_f32), ("base_temperature", c_f32), ("nan_safe", c_i32)]


class SweepSizes(C.Structure):
    _fields_ = [("n_real_cols", c_i64), ("row_tiles", c_i32), ("splits", c_i32), ("partial_f32", c_i64),
                ("rowstat_f32", c_i64), ("dpartial_f32", c_i64)]


class BankGeom(C.Structure):
    _fields_ = [("B", c_i32), ("D", c_i32), ("h", c_i32), ("w", c_i32), ("Himg", c_i32), ("Wimg", c_i32),
                ("K", c_i32), ("M", c_i32), ("network_stride", c_i32), ("pixel_update_freq", c_i32)]


class TcDesc(C.Structure):
    _fields_ = [("anchors_f32", c_vp), ("anchors_bf16", c_vp), ("anchor_cls", c_vp), ("diag_col", c_vp), ("plan", c_vp),
                ("a_rows", c_i32), ("D", c_i32), ("mode", c_i32),
                ("contrast_bf16", c_vp), ("contrast_cls", c_vp), ("n_cols", c_i64), ("contrast_rows_alloc", c_i64),
                ("bank_K", c_i32), ("bank_R", c_i32), ("sorted", c_i32), ("contrast_norm_bound", c_f32),
                ("temperature", c_f32), ("base_temperature", c_f32), ("nan_safe", c_i32), ("neg_only", c_i32)]


class StepDesc(C.Structure):
    _fields_ = [("g", Geom),
                ("embed", c_vp), ("labels", c_vp), ("seg", c_vp), ("predict", c_vp), ("ranks", c_vp),
                ("seed", c_u64), ("normalize", c_i32),
                ("mode", c_i32), ("segment_queue", c_vp), ("pixel_queue", c_vp),
                ("bank_K", c_i32), ("bank_M0", c_i32), ("bank_M1", c_i32),
                ("temperature", c_f32), ("base_temperature", c_f32), ("nan_safe", c_i32),
                ("keys", c_vp), ("chunk_pref", c_vp), ("counts", c_vp), ("plan", c_vp), ("anchor_meta", c_vp),
                ("anchors_f32", c_vp), ("anchors_bf16", c_vp), ("inv_norm", c_vp), ("norm_max", c_vp),
                ("partials", c_vp), ("rowstats", c_vp), ("dpartials", c_vp), ("dA", c_vp),
                ("precision", c_i32), ("shadow_bf16", c_vp), ("shadow_rows", c_i64), ("contrast_norm_bound", c_f32),
                ("row_m2", c_vp),
                ("loss", c_vp), ("grad_embed", c_vp), ("sync", c_vp),
                ("embed_dtype", c_i32), ("seg_dtype", c_i32),
                ("topk_negatives", c_i32), ("topk_scratch", c_vp)]


ABI_STRUCTS = (Geom, SelectSizes, SweepDesc, SweepSizes, BankGeom, TcDesc, StepDesc)   # pcl_abi_sizeof ids 0..6

# name -> (restype, argtypes); every symbol declared in include/pcl.h
SIGNATURES = {
    "pcl_version": (c_i32, []),
    "pcl_strerror": (C.c_char_p, [c_i32]),
    "pcl_last_cuda_error": (C.c_char_p, []),
    "pcl_device_count": (c_i32, []),
    "pcl_abi_sizeof": (c_i64, [c_i32]),
    "pcl_launch_count": (c_u64, []),
    "pcl_select_sizes": (c_i32, [C.POINTER(Geom), C.POINTER(SelectSizes)]),
    "pcl_class_stats": (c_i32, [C.POINTER(Geom), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_plan_anchors": (c_i32, [C.POINTER(Geom), c_vp, c_vp, c_vp]),
    "pcl_select_gather": (c_i32, [C.POINTER(Geom), c_vp, c_vp, c_vp, c_vp, c_vp, c_u64, c_i32, c_vp, c_vp, c_vp,
                                  c_vp, c_vp, c_vp]),
    "pcl_sweep_sizes": (c_i32, [C.POINTER(SweepDesc), C.POINTER(SweepSizes)]),
    "pcl_infonce_fwd": (c_i32, [C.POINTER(SweepDesc), c_vp, c_vp, c_vp, c_vp]),
    "pcl_infonce_bwd": (c_i32, [C.POINTER(SweepDesc), c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_topk_scratch_u32": (c_i64, [C.POINTER(SweepDesc)]),
    "pcl_infonce_topk_fwd": (c_i32, [C.POINTER(SweepDesc), c_i32, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_infonce_topk_bwd": (c_i32, [C.POINTER(SweepDesc), c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_scatter_grad": (c_i32, [C.POINTER(Geom), c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_vp, c_vp]),
    "pcl_l2norm_fwd": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_i64, c_vp]),
    "pcl_l2norm_bwd": (c_i32, [c_vp, c_vp, c_vp, c_i32, c_i32, c_i64, c_vp]),
    "pcl_proj_workspace_bytes": (c_i64, [c_i32, c_i32, c_i64, c_i32]),
    "pcl_proj_pack": (c_i32, [c_vp, c_i32, c_vp, c_vp]),
    "pcl_proj_fwd": (c_i32, [c_vp, c_vp, c_vp, c_i32, c_i32, c_i64, c_vp, c_vp, c_vp]),
    "pcl_proj_bwd": (c_i32, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_proj_fwd_dt": (c_i32, [c_vp, c_i32, c_vp, c_vp, c_i32, c_i32, c_i64, c_vp, c_vp, c_vp]),
    "pcl_proj_bwd_dt": (c_i32, [c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_proj_bn_workspace_bytes": (c_i64, [c_i32, c_i32, c_i64, c_i32]),
    "pcl_proj_bn_stats_dt": (c_i32, [c_vp, c_i32, c_i32, c_i32, c_i64, c_vp, c_vp]),
    "pcl_proj_bn_finalize": (c_i32, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_f32, c_f32, c_i32, c_vp, c_vp]),
    "pcl_proj_bn_fwd_dt": (c_i32, [c_vp, c_i32, c_vp, c_vp, c_vp, c_i32, c_i32, c_i64, c_vp, c_vp, c_vp]),
    "pcl_proj_bn_bwd_dt": (c_i32, [c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_i64, c_vp, c_vp, c_vp,
                                   c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_proj_bn_input_grad_dt": (c_i32, [c_vp, c_i32, c_vp, c_vp, c_i32, c_i32, c_i64, c_i32, c_vp, c_vp]),
    "pcl_proj_bn_cols_workspace_bytes": (c_i64, [c_i32, c_i32]),
    "pcl_proj_bn_bwd_cols_dt": (c_i32, [c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_vp, c_i32, c_i32, c_i64,
                                        c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_proj_bn_input_grad_cols_dt": (c_i32, [c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i64, c_i32,
                                               c_vp, c_vp]),
    "pcl_proj_conv1_workspace_bytes": (c_i64, [c_i32, c_i32, c_i64, c_i32]),
    "pcl_proj_conv1_pack": (c_i32, [c_vp, c_i32, c_vp, c_vp]),
    "pcl_proj_conv1_fwd_dt": (c_i32, [c_vp, c_i32, c_vp, c_vp, c_i32, c_i32, c_i64, c_vp, c_vp, c_vp, c_vp]),
    "pcl_proj_conv1_bwd_dt": (c_i32, [c_vp, c_i32, c_vp, c_vp, c_i32, c_i32, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_seg_ce_scratch_floats":(c_i64, [c_i32, c_i32, c_i32]),
    "pcl_seg_ce_fwd": (c_i32, [c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp]),
    "pcl_seg_ce_bwd": (c_i32, [c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp,
                               c_vp]),
    "pcl_seg_ce_fwd_bwd_scratch_floats": (c_i64, [c_i32] * 4),
    "pcl_seg_ce_fwd_bwd": (c_i32, [c_vp, c_vp, c_vp] + [c_i32] * 7 + [c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_rmi_scratch_bytes": (c_i64, [c_i32] * 9),
    "pcl_rmi_fwd": (c_i32, [c_vp, c_vp] + [c_i32] * 9 + [c_f32, c_i32, c_f32, c_vp, c_vp, c_vp]),
    "pcl_rmi_bwd": (c_i32, [c_vp, c_vp] + [c_i32] * 9 + [c_f32, c_i32, c_f32, c_vp, c_vp, c_vp, c_vp]),
    "pcl_lovasz_scratch_bytes": (c_i64, [c_i32] * 6),
    "pcl_lovasz_fwd": (c_i32, [c_vp, c_vp] + [c_i32] * 7 + [c_vp, c_vp, c_vp]),
    "pcl_lovasz_bwd": (c_i32, [c_vp, c_vp] + [c_i32] * 7 + [c_vp, c_vp, c_vp, c_vp]),
    "pcl_ohem_ce_scratch_bytes": (c_i64, [c_i32] * 6),
    "pcl_ohem_ce_fwd": (c_i32, [c_vp, c_vp, c_vp] + [c_i32] * 7 + [c_f32, c_i64, c_i32, c_vp, c_vp, c_vp]),
    "pcl_ohem_ce_bwd": (c_i32, [c_vp, c_vp, c_vp] + [c_i32] * 7 + [c_vp, c_vp, c_vp, c_vp]),
    "pcl_bank_packet_floats": (c_i64, [C.POINTER(BankGeom)]),
    "pcl_bank_scratch_floats": (c_i64, [C.POINTER(BankGeom)]),
    "pcl_bank_packet": (c_i32, [C.POINTER(BankGeom), c_vp, c_vp, c_vp, c_u64, c_vp, c_vp, c_vp]),
    "pcl_bank_packet_dev": (c_i32, [C.POINTER(BankGeom), c_vp, c_vp, c_u64, c_vp, c_vp, c_vp, c_vp]),
    "pcl_bank_packet_dt": (c_i32, [C.POINTER(BankGeom), c_vp, c_i32, c_vp, c_vp, c_u64, c_vp, c_vp, c_vp]),
    "pcl_bank_packet_dev_dt": (c_i32, [C.POINTER(BankGeom), c_vp, c_i32, c_vp, c_u64, c_vp, c_vp, c_vp, c_vp]),
    "pcl_bank_apply": (c_i32, [C.POINTER(BankGeom), c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_bank_apply_ctr": (c_i32, [C.POINTER(BankGeom), c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_bank_shadow_rebuild": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_i32, c_vp, c_vp]),
    "pcl_tc_sizes": (c_i32, [C.POINTER(TcDesc), C.POINTER(SweepSizes)]),
    "pcl_to_bf16": (c_i32, [c_vp, c_vp, c_i64, c_i64, c_vp]),
    "pcl_infonce_tc_fwd": (c_i32, [C.POINTER(TcDesc), c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_infonce_tc_bwd": (c_i32, [C.POINTER(TcDesc), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_tc_topk_scratch_u32": (c_i64, [C.POINTER(TcDesc)]),
    "pcl_infonce_tc_topk_fwd": (c_i32, [C.POINTER(TcDesc), c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_infonce_tc_topk_bwd": (c_i32, [C.POINTER(TcDesc), c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_tc_dump_logits": (c_i32, [C.POINTER(TcDesc), c_vp, c_vp, c_vp]),
    "pcl_step_stats": (c_i32, [C.POINTER(StepDesc), c_vp]),
    "pcl_step_forward": (c_i32, [C.POINTER(StepDesc), c_vp]),
    "pcl_step_backward": (c_i32, [C.POINTER(StepDesc), c_vp, c_vp]),
    "pcl_step_backward_prezeroed": (c_i32, [C.POINTER(StepDesc), c_vp, c_vp]),
    "pcl_step_backward_cols": (c_i32, [C.POINTER(StepDesc), c_vp, c_vp, c_vp, c_vp]),
    "pcl_step_ranks": (c_i32, [C.POINTER(StepDesc), c_vp, c_vp, c_vp]),
    "pcl_step_forward_ctr": (c_i32, [C.POINTER(StepDesc), c_vp, c_vp]),
    "pcl_step_fused_supported": (c_i32, [C.POINTER(StepDesc)]),
    "pcl_step_fused_select": (c_i32, [C.POINTER(StepDesc), c_vp, c_vp, c_vp]),
    "pcl_step_fused_loss": (c_i32, [C.POINTER(StepDesc), c_vp]),
    "pcl_step_fused_scatter": (c_i32, [C.POINTER(StepDesc), c_vp, c_vp, c_vp, c_vp]),
    "pcl_step_fused_cols": (c_i32, [C.POINTER(StepDesc), c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pcl_step_fused_fill": (c_i32, [C.POINTER(StepDesc), c_vp]),
    "pcl_fill_zero": (c_i32, [c_vp, c_u64, c_vp]),
}

_lib = None
_lock = threading.Lock()


def library_path() -> str:
    return os.environ.get("PCL_B200_LIB") or _build.library_path()


def load(build_if_missing: bool = False):
    """Load the shared library (once).  Raises PclError when it is absent — there is no CPU fallback."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        path = library_path()
        if not os.path.exists(path):
            if build_if_missing:
                _build.build_library()
            else:
                raise PclError(f"{path} not found: build it with `python -m contrastiveseg_b200.build` "
                               "(the engine has no CPU / PyTorch fallback)")
        lib = C.CDLL(path)
        if hasattr(lib, "pcl_emulated"):
            # tests/emu builds the SIMT kernel sources for host threads so that CPU-only test runs execute kernel logic;
            # that build is test infrastructure and must never serve the product (there is no CPU path)
            raise PclError(f"{path} is the host-thread emulation build of the test suite, not the sm_90a library")
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)            # AttributeError here = ABI mismatch: fail loudly
            fn.restype = res
            fn.argtypes = args
        if lib.pcl_version() // 100 != 1:
            raise PclError(f"ABI version mismatch: library reports {lib.pcl_version()}")
        for sid, st in enumerate(ABI_STRUCTS):       # struct layouts as compiled vs as declared here
            if lib.pcl_abi_sizeof(sid) != C.sizeof(st):
                raise PclError(f"ABI layout mismatch: {st.__name__} is {C.sizeof(st)} bytes here, "
                               f"{lib.pcl_abi_sizeof(sid)} in {path}")
        _lib = lib
    return _lib


def check(status: int, what: str = "") -> None:
    if status == 0:
        return
    lib = load()
    msg = lib.pcl_strerror(status).decode()
    if status == -2:
        msg += ": " + lib.pcl_last_cuda_error().decode()
    raise PclError(f"{what or 'pcl call'} failed ({status}): {msg}")


def ptr(t) -> int:
    """Device (or host) address of a torch tensor, None -> NULL."""
    return None if t is None else t.data_ptr()
