"""ctypes binding of libv3d_b200.so (the C ABI declared in include/v3d_b200.h).

There is no CPU fallback: if the shared library is missing the import of any compute op fails
loudly with instructions to build it (`python -m v3d_b200.build` or `__graft_entry__.build()`).
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

_LIB_PATH = Path(__file__).resolve().parent / "_lib" / "libv3d_b200.so"
_lib = None


class V3DLibraryError(RuntimeError):
    pass


class GemmArgs(C.Structure):
    """Mirror of `v3d_gemm_args` (include/v3d_b200.h)."""

    _fields_ = [
        ("A", C.c_void_p), ("B", C.c_void_p), ("D", C.c_void_p),
        ("bias", C.c_void_p), ("fbias", C.c_void_p), ("R1", C.c_void_p), ("R2", C.c_void_p),
        ("lda", C.c_int64), ("ldb", C.c_int64), ("ldd", C.c_int64), ("ldr1", C.c_int64), ("ldr2", C.c_int64),
        ("ldfb", C.c_int64),
        ("a_batch_stride", C.c_int64), ("b_batch_stride", C.c_int64),
        ("batch", C.c_int32), ("rows_per_batch", C.c_int32),
        ("N", C.c_int32), ("K", C.c_int32),
        ("ntaps", C.c_int32), ("tap_shift", C.c_int32),
        ("rows_per_frame", C.c_int32), ("act", C.c_int32), ("out_fp32", C.c_int32),
        ("conv_n", C.c_int32), ("conv_h", C.c_int32), ("conv_w", C.c_int32),
        ("block_n", C.c_int32),
        ("out_transposed", C.c_int32), ("valid_cols", C.c_int32), ("accumulate", C.c_int32),
        ("s0", C.c_float), ("s1", C.c_float), ("s2", C.c_float),
        ("a_rows", C.c_int32), ("a_row0", C.c_int32),
        ("kv_col0", C.c_int32), ("kv_n", C.c_int32), ("kv_ld", C.c_int64), ("kv_dst", C.c_void_p * 8),
    ]


# name -> (restype, argtypes); kept in one table so tests can check every declared symbol exports.
_i32, _i64, _f32, _vp = C.c_int32, C.c_int64, C.c_float, C.c_void_p
SIGNATURES = {
    "v3d_abi_version": (C.c_int, []),
    "v3d_last_error": (C.c_char_p, []),
    "v3d_launch_count": (C.c_int64, []),
    "v3d_gemm_bf16": (C.c_int, [C.POINTER(GemmArgs), _vp]),
    "v3d_gemm_args_size": (C.c_int, []),
    "v3d_geglu_pack_rows": (C.c_int, [_i32, _i32, C.POINTER(C.c_int32)]),
    "v3d_gemm_pick_block_n": (C.c_int, [_i32, _i32]),
    "v3d_debug_set_trace": (C.c_int, [_vp]),
    # norm.cu
    "v3d_groupnorm_stats": (C.c_int, [_vp, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _vp]),
    "v3d_groupnorm_apply": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _f32, _i32, _vp]),
    "v3d_groupnorm_workspace_bytes": (C.c_int64, []),
    "v3d_groupnorm": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _f32, _i32, _vp, _i64, _vp]),
    "v3d_groupnorm_det_blocks": (C.c_int64, [_i64, _i64]),
    "v3d_groupnorm_det_workspace_bytes": (C.c_int64, [_i64, _i64, _i32, _i32]),
    "v3d_groupnorm_partials": (C.c_int, [_vp, _vp, _i64, _i64, _i32, _i32, _i32, _i32, _i64, _vp]),
    "v3d_groupnorm_fold_apply": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _i64, _i64, _f32,
                                           _i32, _vp]),
    "v3d_groupnorm_det": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, _i32, _i32, _i32, _i32, _f32, _i32, _vp, _i64,
                                    _vp]),
    "v3d_layernorm": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _f32, _vp]),
    "v3d_softmax_rows": (C.c_int, [_vp, _i64, _i32, _f32, _vp]),
    "v3d_softmax_rows_f32": (C.c_int, [_vp, _vp, _i64, _i32, _f32, _vp]),
    # peer.cu
    "v3d_peer_alloc": (C.c_int, [_i64, C.POINTER(_vp)]),
    "v3d_peer_free": (C.c_int, [_vp]),
    "v3d_peer_export": (C.c_int, [_vp, _vp]),
    "v3d_peer_import": (C.c_int, [_vp, C.POINTER(_vp)]),
    "v3d_peer_close": (C.c_int, [_vp]),
    "v3d_peer_epoch_bump": (C.c_int, [_vp, _vp]),
    "v3d_peer_put": (C.c_int, [_i32, C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_i64), _i32, C.POINTER(_vp), _vp, _vp, _vp]),
    "v3d_peer_wait": (C.c_int, [_i32, C.POINTER(_vp), _vp, _vp, _i32, _vp]),
    "v3d_peer_allreduce_f64": (C.c_int, [_vp, _i32, C.c_double, _i32, _i32, C.POINTER(_vp), C.POINTER(_vp), _vp, _vp, _i32, _vp]),
    # attention.cu
    "v3d_attention_spatial": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, _i32, _i32, _i32, _f32, _vp]),
    "v3d_attention_spatial_mma": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, _i32, _i32, _i32, _f32, _vp]),
    "v3d_attention_temporal": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, _i32, _i32, _i32, _i32, _f32, _vp]),
    "v3d_attention_temporal_kv": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _i32, _i32, _i32, _i32,
                                            C.POINTER(C.c_int32), C.POINTER(C.c_int32), _f32, _vp]),
    "v3d_attention_cross": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _i32, _i32, _i64, _i32, _f32, _vp]),
    # elementwise.cu
    "v3d_upsample_nearest2x": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "v3d_copy_channels": (C.c_int, [_vp, _i64, _vp, _i64, _i64, _i32, _vp]),
    "v3d_im2col3x3": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "v3d_nchw_f32_to_nhwc_bf16": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp]),
    "v3d_nhwc_to_nchw_f32": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i64, _i32, _f32, _vp]),
    "v3d_small_linear": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i64, _i64, _vp]),
    "v3d_prep_small_x": (C.c_int, [_vp, _i64, _vp, _i32, _i32, _i32, _vp]),
    "v3d_timestep_embedding": (C.c_int, [_vp, _vp, _i32, _i32, _f32, _vp]),
    "v3d_add_rows": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _vp]),
    "v3d_time_mix_conv": (C.c_int, [_vp, _i64, _vp, _vp, _vp, _i32, _i32, _i64, _i32, _vp]),
    # sampler.cu
    "v3d_edm_scale_input": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i64, _vp]),
    "v3d_edm_denoise_combine": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i64, _vp]),
    "v3d_cfg_combine": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i64, _vp]),
    "v3d_euler_step": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i32, _i64, _vp]),
    "v3d_heun_step": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i64, _vp]),
    "v3d_ancestral_euler_step": (C.c_int, [_vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _f32, _i32, _i64, _vp]),
    "v3d_dpmpp2s_stage": (C.c_int, [_vp, _vp, _vp, _f32, _f32, _i32, _i64, _vp]),
    "v3d_dpmpp2s_step": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _f32, _f32, _f32, _i32, _i64,
                                   _vp]),
    "v3d_dpmpp2m_step": (C.c_int, [_vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _i32, _i32, _i64, _vp]),
    "v3d_lms_step": (C.c_int, [_vp, _vp, _vp, _vp, _f32, C.POINTER(C.c_float), C.POINTER(C.c_int32), _i32, _i32,
                               _i32, _i64, _vp]),
    "v3d_decode_to_u8": (C.c_int, [_vp, _i64, _i32, _vp, _i64, _vp]),
    "v3d_frames_nchw_to_u8": (C.c_int, [_vp, _vp, _i32, _i64, _vp]),
    # pixelnerf.cu
    "v3d_pixelnerf_rays": (C.c_int, [_vp, _i32, _i32, _f32, _i32, _vp, _vp, _vp]),
    "v3d_pixelnerf_render": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i32, _i32, _i32, _i32, _i32, _i32,
                                       _f32, _f32, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "v3d_pixelnerf_decode": (C.c_int, [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
}


def lib_path() -> Path:
    return _LIB_PATH


def load():
    """Load the shared library once and attach prototypes for every symbol the header declares."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise V3DLibraryError(
            f"{_LIB_PATH} is missing: the sm_90a kernels were not built. "
            "Run `python -m v3d_b200.build` (needs nvcc); there is no CPU fallback for the product path."
        )
    lib = C.CDLL(str(_LIB_PATH))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here means header/library drift: fail loudly
        fn.restype = res
        fn.argtypes = args
    if lib.v3d_abi_version() != 1:
        raise V3DLibraryError("libv3d_b200.so ABI version mismatch; rebuild")
    if lib.v3d_gemm_args_size() != C.sizeof(GemmArgs):
        raise V3DLibraryError(f"v3d_gemm_args is {lib.v3d_gemm_args_size()} bytes in libv3d_b200.so but "
                              f"{C.sizeof(GemmArgs)} in the ctypes mirror; rebuild (python -m v3d_b200.build)")
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().v3d_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"{what} failed (code {rc}): {msg}")
