"""ctypes binding of include/powerpaint_b200.h (the C-ABI boundary).

The product path has no CPU fallback: if the shared library is missing or cannot be
loaded, `lib()` raises, and every op raises `RuntimeError` with `pp_last_error()` on a
non-zero status.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import os

# PP_B200_LIB points at an alternative build of the same library (kernel experiments)
_LIB_PATH = Path(os.environ.get("PP_B200_LIB") or Path(__file__).resolve().parent / "libpowerpaint_b200.so")
_lib = None

# enums (mirror include/powerpaint_b200.h)
PP_A_MATRIX, PP_A_CONV3X3, PP_A_CONV3X3_S2, PP_A_CONV3X3_S2P0 = 0, 1, 2, 3
PP_EPI_PLAIN, PP_EPI_GEGLU, PP_EPI_TRANSPOSED, PP_EPI_ROWS_THEN_TRANSPOSED = 0, 1, 2, 3
PP_ACT_NONE, PP_ACT_SILU, PP_ACT_QUICK_GELU = 0, 1, 2
PP_BLEND_LUMA, PP_BLEND_HOLE_FILL, PP_BLEND_RED_OVERLAY, PP_BLEND_PASTE = 0, 1, 2, 3
ABI_VERSION = 5

vp = C.c_void_p
i32 = C.c_int32
i64 = C.c_int64
f32 = C.c_float
u64 = C.c_uint64


class StatsGeom(C.Structure):
    _fields_ = [
        ("supported", i32), ("channels", i32), ("segs", i32), ("seg_rows", i32), ("tiles_per_group", i32),
        ("tiles_x", i32), ("tiles_y", i32), ("bw", i32), ("bh", i32), ("wo", i32), ("ho", i32),
        ("bytes", i64),
    ]


class GemmDesc(C.Structure):
    _fields_ = [
        ("a_mode", i32), ("epilogue", i32),
        ("a0", vp), ("a1", vp),
        ("c0", i32), ("c1", i32),
        ("lda0", i64), ("lda1", i64),
        ("nb", i32), ("h", i32), ("w", i32),
        ("M", i32), ("N", i32),
        ("b", vp), ("ldb", i64),
        ("bias", vp), ("rowvec", vp), ("rows_per_group", i32), ("rowvec_ld", i64),
        ("res1", vp), ("ldr1", i64),
        ("res2", vp), ("ldr2", i64),
        ("alpha", f32), ("act", i32),
        ("out", vp), ("ldc", i64),
        ("out_fp32", i32), ("t_rows", i32), ("t_ld", i64),
        ("block_n", i32), ("t_fp16", i32),
        ("alpha_dev", vp), ("alpha_step", vp), ("alpha_stride", i32),
        ("chan_stats", vp),
        ("row_stats", vp), ("row_stats_ld", i64), ("row_final", vp), ("row_ticket", vp),
        ("ln_stats", vp), ("ln_u", vp), ("ln_eps", f32),
        ("out_t", vp), ("trans_from_col", i32),
        ("splitk_ws", vp), ("splitk_flags", vp),
    ]


class AttnDesc(C.Structure):
    _fields_ = [
        ("q", vp), ("k", vp), ("vt", vp), ("out", vp),
        ("batch", i32), ("heads", i32), ("d", i32), ("nq", i32), ("nk", i32),
        ("q_ld", i64), ("k_ld", i64), ("vt_ld", i64), ("o_ld", i64),
        ("q_batch_stride", i64), ("k_batch_stride", i64),
        ("scale", f32), ("vt_fp16", i32),
    ]


class GnDesc(C.Structure):
    _fields_ = [
        ("x0", vp), ("x1", vp), ("c0", i32), ("c1", i32),
        ("batch", i32), ("hw", i32), ("groups", i32),
        ("gamma", vp), ("beta", vp), ("eps", f32), ("silu", i32),
        ("stats", vp), ("y", vp), ("stats_prezeroed", i32),
        ("from_partials", i32), ("part0", vp), ("part1", vp), ("geom0", StatsGeom), ("geom1", StatsGeom),
    ]


class RandnDraw(C.Structure):
    """pp_randn_draw: one draw of torch's CUDA randn, computed inside the step kernels"""
    _fields_ = [("seed", u64), ("offset0", u64), ("offset_per_step", u64), ("threads", i64),
                ("first_row", i32), ("rows", i32)]


class CfgDdimDesc(C.Structure):
    _fields_ = [
        ("eps", vp), ("eps_fp32", i32), ("eps_ld", i32),
        ("latents", vp), ("coef", vp), ("step_idx", vp), ("advance_step", i32),
        ("noise", vp), ("guidance_scale", f32), ("do_cfg", i32),
        ("batch", i32), ("hw", i32),
        ("next_in", vp), ("next_c", i32), ("n_copies", i32),
        ("extra", vp), ("extra_c", i32), ("guidance_from_coef", i32), ("extra_per_copy", i32),
        ("blend_x0", vp), ("blend_mask", vp), ("blend_noise", vp),
        ("draws", vp), ("n_draws", i32),
    ]


class UniPCDesc(C.Structure):
    _fields_ = [
        ("eps", vp), ("eps_fp32", i32), ("eps_ld", i32),
        ("latents", vp), ("last_sample", vp), ("m1", vp), ("m2", vp),
        ("coef", vp), ("ucoef", vp), ("step_idx", vp), ("advance_step", i32), ("do_cfg", i32),
        ("batch", i32), ("hw", i32),
        ("next_in", vp), ("next_c", i32), ("n_copies", i32),
    ]


class SolverDesc(C.Structure):
    _fields_ = [
        ("eps", vp), ("eps_fp32", i32), ("eps_ld", i32),
        ("latents", vp), ("m1", vp), ("noise", vp),
        ("coef", vp), ("scoef", vp), ("step_idx", vp), ("advance_step", i32), ("do_cfg", i32),
        ("batch", i32), ("hw", i32),
        ("next_in", vp), ("next_c", i32), ("n_copies", i32),
        ("draws", vp), ("n_draws", i32),
    ]


class PlmsDesc(C.Structure):
    _fields_ = [
        ("eps", vp), ("eps_fp32", i32), ("eps_ld", i32),
        ("latents", vp), ("cur_sample", vp), ("ets", vp),
        ("coef", vp), ("pcoef", vp), ("step_idx", vp), ("advance_step", i32), ("do_cfg", i32),
        ("batch", i32), ("hw", i32),
        ("next_in", vp), ("next_c", i32), ("n_copies", i32),
        ("blend_x0", vp), ("blend_mask", vp), ("blend_noise", vp),
    ]


class Window(C.Structure):
    _fields_ = [("src_off", i64), ("dst_off", i64), ("src_row", i64), ("dst_row", i64), ("rows", i32), ("cols", i32)]


class TileBlendDesc(C.Structure):
    _fields_ = [
        ("b", vp), ("av", vp), ("ah", vp),
        ("b_stride", i64), ("av_stride", i64), ("ah_stride", i64),
        ("batch", i32), ("channels", i32),
        ("b_h", i32), ("b_w", i32),
        ("av_h", i32), ("ah_w", i32),
        ("e_v", i32), ("e_h", i32),
    ]


class PoolBroadcastDesc(C.Structure):
    _fields_ = [("x", vp), ("prev", vp), ("out", vp), ("batch", i32), ("hw", i32), ("channels", i32)]


# every exported symbol of include/powerpaint_b200.h with (restype, argtypes)
_SIGNATURES = {
    "pp_last_error": (C.c_char_p, []),
    "pp_abi_version": (C.c_int, []),
    "pp_device_supported": (C.c_int, []),
    "pp_gemm_conv": (C.c_int, [C.POINTER(GemmDesc), vp]),
    "pp_gemm_stats_geometry": (C.c_int, [C.POINTER(GemmDesc), C.POINTER(StatsGeom)]),
    "pp_gemm_row_stats_records": (i32, [C.POINTER(GemmDesc)]),
    "pp_gemm_splitk_bytes": (i64, [C.POINTER(GemmDesc), C.POINTER(i32)]),
    "pp_gemm_variant": (C.c_int, [C.POINTER(GemmDesc), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]),
    "pp_gemm_staging": (C.c_int, [C.POINTER(GemmDesc), C.POINTER(i32), C.POINTER(i32)]),
    "pp_attention": (C.c_int, [C.POINTER(AttnDesc), vp]),
    "pp_attention_variant": (C.c_int, [C.POINTER(AttnDesc), C.POINTER(i32), C.POINTER(i32)]),
    "pp_group_norm": (C.c_int, [C.POINTER(GnDesc), vp]),
    "pp_group_norm_scratch_bytes": (i64, [i32, i32, i32, i32]),
    "pp_layer_norm": (C.c_int, [vp, vp, vp, vp, i32, i32, f32, vp]),
    "pp_upsample2x": (C.c_int, [vp, vp, i32, i32, i32, i32, vp]),
    "pp_upsample_nearest": (C.c_int, [vp, vp, i32, i32, i32, i32, i32, i32, vp]),
    "pp_add": (C.c_int, [vp, vp, vp, i64, vp]),
    "pp_time_embed": (C.c_int, [vp, vp, vp, i32, i32, vp]),
    "pp_nchw_to_nhwc": (C.c_int, [vp, vp, i32, i32, i32, i32, vp]),
    "pp_nhwc_to_nchw": (C.c_int, [vp, i32, vp, i32, i32, i32, i32, vp]),
    "pp_cfg_ddim_step": (C.c_int, [C.POINTER(CfgDdimDesc), vp]),
    "pp_unipc_step": (C.c_int, [C.POINTER(UniPCDesc), vp]),
    "pp_program_add_unipc": (C.c_int, [vp, C.POINTER(UniPCDesc)]),
    "pp_solver_step": (C.c_int, [C.POINTER(SolverDesc), vp]),
    "pp_program_add_solver_step": (C.c_int, [vp, C.POINTER(SolverDesc)]),
    "pp_plms_step": (C.c_int, [C.POINTER(PlmsDesc), vp]),
    "pp_program_add_plms_step": (C.c_int, [vp, C.POINTER(PlmsDesc)]),
    "pp_softmax_rows": (C.c_int, [vp, vp, i64, i32, i64, i64, vp]),
    "pp_embed_gather": (C.c_int, [vp, vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "pp_causal_attention_small": (C.c_int, [vp, vp, i32, i32, i32, i32, f32, vp]),
    "pp_program_add_embed_gather": (C.c_int, [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32]),
    "pp_program_add_causal_attention_small": (C.c_int, [vp, vp, vp, i32, i32, i32, i32, f32]),
    "pp_image_preprocess_u8": (C.c_int, [vp, vp, i32, vp, i32, i32, i32, f32, f32, vp]),
    "pp_image_postprocess": (C.c_int, [vp, i32, i32, vp, vp, i32, i32, vp]),
    "pp_resample_u8": (C.c_int, [vp, vp, vp, i32, i32, i32, i32, i32, vp, vp, i32, vp, vp, i32, vp]),
    "pp_gaussian_box_radius": (f32, [f32, i32]),
    "pp_box_blur_u8": (C.c_int, [vp, vp, vp, i32, i32, i32, f32, i32, vp]),
    "pp_canny_workspace_bytes": (i64, [i32, i32]),
    "pp_canny_u8": (C.c_int, [vp, vp, vp, i64, i32, i32, i32, C.c_double, C.c_double, vp]),
    "pp_outpaint_canvas_u8": (C.c_int, [vp, i32, i32, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, vp]),
    "pp_app_blend_u8": (C.c_int, [i32, vp, vp, vp, vp, i32, i32, i32, vp]),
    "pp_program_add_softmax_rows": (C.c_int, [vp, vp, vp, i64, i32, i64, i64]),
    "pp_window_copy": (C.c_int, [vp, vp, i32, i32, i64, i64, vp, i32, i32, vp]),
    "pp_program_add_window_copy": (C.c_int, [vp, vp, vp, i32, i32, i64, i64, vp, i32, i32]),
    "pp_tile_blend": (C.c_int, [C.POINTER(TileBlendDesc), vp]),
    "pp_program_add_tile_blend": (C.c_int, [vp, C.POINTER(TileBlendDesc)]),
    "pp_pool_broadcast": (C.c_int, [C.POINTER(PoolBroadcastDesc), vp]),
    "pp_program_add_pool_broadcast": (C.c_int, [vp, C.POINTER(PoolBroadcastDesc)]),
    "pp_program_create": (C.c_int, [C.POINTER(vp)]),
    "pp_program_run_range": (C.c_int, [vp, i32, i32, vp]),
    "pp_program_destroy": (None, [vp]),
    "pp_program_add_gemm": (C.c_int, [vp, C.POINTER(GemmDesc)]),
    "pp_program_add_attention": (C.c_int, [vp, C.POINTER(AttnDesc)]),
    "pp_program_add_group_norm": (C.c_int, [vp, C.POINTER(GnDesc)]),
    "pp_program_add_layer_norm": (C.c_int, [vp, vp, vp, vp, vp, i32, i32, f32]),
    "pp_program_add_upsample2x": (C.c_int, [vp, vp, vp, i32, i32, i32, i32]),
    "pp_program_add_upsample_nearest": (C.c_int, [vp, vp, vp, i32, i32, i32, i32, i32, i32]),
    "pp_program_add_add": (C.c_int, [vp, vp, vp, vp, i64]),
    "pp_program_add_time_embed": (C.c_int, [vp, vp, vp, vp, i32, i32]),
    "pp_program_add_cfg_ddim": (C.c_int, [vp, C.POINTER(CfgDdimDesc)]),
    "pp_program_add_memset": (C.c_int, [vp, vp, i64]),
    "pp_program_num_ops": (i32, [vp]),
    "pp_program_num_launches": (i32, [vp]),
    "pp_program_run": (C.c_int, [vp, vp]),
    "pp_program_graph_build": (C.c_int, [vp, vp]),
    "pp_program_graph_launch": (C.c_int, [vp, vp]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def lib_path() -> Path:
    return _LIB_PATH


def lib():
    """Load (once) and return the C-ABI library; raises if it is not built."""
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            raise RuntimeError(
                f"{_LIB_PATH} is not built: run `python -m powerpaint_b200.build` "
                "(there is no CPU fallback for the hot path)"
            )
        L = C.CDLL(str(_LIB_PATH))
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        if L.pp_abi_version() != ABI_VERSION:
            raise RuntimeError(f"{_LIB_PATH} has ABI version {L.pp_abi_version()}, this binding needs {ABI_VERSION}: "
                               "rebuild with `python -m powerpaint_b200.build`")
        _lib = L
    return _lib


def check(status: int, what: str = "") -> None:
    if status != 0:
        msg = lib().pp_last_error()
        raise RuntimeError(f"powerpaint_b200 native call failed ({what} status {status}): "
                           f"{msg.decode() if msg else '?'}")


def ptr(t) -> int | None:
    """data_ptr of a torch tensor (or None)."""
    return None if t is None else t.data_ptr()


def current_stream(device=None) -> int:
    """raw handle of torch's current stream on `device` (default: the current device)"""
    import torch

    return torch.cuda.current_stream(device).cuda_stream
