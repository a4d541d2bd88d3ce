"""ctypes binding of the C-ABI kernel library (``include/frl_b200.h``).

There is no fallback: if ``csrc/libfrl_b200.so`` is missing or a launch fails this module
raises.  ``python __graft_entry__.py build`` (or ``make -C csrc``) produces the library in-tree.
"""
import ctypes as C
import os
import subprocess
from typing import Optional, Sequence

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC_DIR = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(CSRC_DIR, "libfrl_b200.so")

F32, BF16, U8, I64 = 0, 1, 2, 3
LOSS_MSE, LOSS_CE, LOSS_CE_PROB = 0, 1, 2
FP8_E4M3, FP8_E5M2 = 0, 1
FP8_DTYPE = {FP8_E4M3: torch.float8_e4m3fn, FP8_E5M2: torch.float8_e5m2}
MAX_TASKS = 8

_DTYPE_CODE = {torch.float32: F32, torch.bfloat16: BF16, torch.uint8: U8, torch.bool: U8,
               torch.int64: I64}


class NativeLibraryError(RuntimeError):
    pass


class TaskDesc(C.Structure):
    """Mirror of ``frl_task_desc``."""
    _fields_ = [
        ("kind", C.c_int32), ("out_dtype", C.c_int32), ("tgt_dtype", C.c_int32),
        ("ignore_index", C.c_int32),
        ("out", C.c_void_p), ("tgt", C.c_void_p), ("mask", C.c_void_p), ("dout", C.c_void_p),
        ("rows", C.c_int64), ("cols", C.c_int64), ("mask_inner", C.c_int64),
        ("weight", C.c_float), ("label_smoothing", C.c_float),
    ]


class GradSeg(C.Structure):
    """Mirror of ``frl_grad_seg``."""
    _fields_ = [("g", C.c_void_p), ("arena_off", C.c_int64), ("numel", C.c_int64),
                ("g_dtype", C.c_int32), ("_pad", C.c_int32)]


# name -> (restype, argtypes); every name here must be declared in include/frl_b200.h
_vp, _i, _i64, _f, _d = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_double
_u64 = C.c_uint64
SIGNATURES = {
    "frl_abi_version": (_i, []),
    "frl_last_error": (C.c_char_p, []),
    "frl_launch_count": (C.c_uint64, []),
    "frl_launch_count_reset": (None, []),
    "frl_device_sm_count": (_i, []),
    "frl_device_arch": (_i, []),
    "frl_sgd_momentum": (_i, [_vp, _vp, _vp, _vp, _i64, _d, _d, _d, _d, _d, _vp, _vp, _i, _i, _vp]),
    "frl_adam": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _d, _d, _d, _d, _d, _i64, _d, _vp, _vp, _i, _vp]),
    "frl_adamw": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _d, _d, _d, _d, _d, _i64, _d, _vp, _vp, _i, _vp]),
    "frl_lion": (_i, [_vp, _vp, _vp, _vp, _i64, _d, _d, _d, _d, _d, _vp, _vp, _i, _vp]),
    "frl_rmsprop": (_i, [_vp, _vp, _vp, _vp, _vp, _i64, _d, _d, _d, _d, _d, _d, _vp, _vp, _i, _vp]),
    "frl_dw_gemm": (_i, [_vp, _i64, _vp, _i64, _i64, _i64, _i64, _vp, _vp]),
    "frl_dw_gemm_sgd": (_i, [_vp, _i64, _vp, _i64, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _d, _d, _d, _d, _d,
                             _vp, _i, _vp]),
    "frl_dw_gemm_sgd_sr": (_i, [_vp, _i64, _vp, _i64, _i64, _i64, _i64, _vp, _vp, _vp, _i64, _u64, _i64, _d, _d,
                                _d, _d, _d, _vp, _i, _vp]),
    "frl_dw_gemm_lion": (_i, [_vp, _i64, _vp, _i64, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _d, _d, _d, _d, _d,
                              _vp, _vp]),
    "frl_dw_gemm_lion_sr": (_i, [_vp, _i64, _vp, _i64, _i64, _i64, _i64, _vp, _vp, _vp, _i64, _u64, _i64, _d, _d,
                                 _d, _d, _d, _vp, _vp]),
    "frl_dx_drelu_scratch_bytes": (_i64, [_i64, _i64]),
    "frl_dx_gemm_drelu": (_i, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i64, _i64, _i, _vp, _vp]),
    "frl_mt_tile_elems": (_i64, []),
    "frl_flatten_grads": (_i, [_vp, _vp, _vp, _i64, _vp, _i, _d, _vp]),
    "frl_sgd_momentum_mt": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _d, _d, _d, _d, _d, _vp, _vp, _i, _vp]),
    "frl_adam_mt": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _d, _d, _d, _d, _d, _i64, _d, _vp, _vp, _vp]),
    "frl_adamw_mt": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _d, _d, _d, _d, _d, _i64, _d, _vp, _vp, _vp]),
    "frl_lion_mt": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _d, _d, _d, _d, _d, _vp, _vp, _vp]),
    "frl_rmsprop_mt": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _d, _d, _d, _d, _d, _d, _vp, _vp, _vp]),
    "frl_sgd_momentum_sr": (_i, [_vp, _vp, _vp, _i64, _i64, _u64, _i64, _d, _d, _d, _d, _d, _vp, _vp, _i, _i, _vp]),
    "frl_adam_sr": (_i, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _u64, _d, _d, _d, _d, _d, _i64, _d, _vp, _vp, _i, _vp]),
    "frl_adamw_sr": (_i, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _u64, _d, _d, _d, _d, _d, _i64, _d, _vp, _vp, _i, _vp]),
    "frl_lion_sr": (_i, [_vp, _vp, _vp, _i64, _i64, _u64, _i64, _d, _d, _d, _d, _d, _vp, _vp, _i, _vp]),
    "frl_rmsprop_sr": (_i, [_vp, _vp, _vp, _vp, _i64, _i64, _u64, _i64, _d, _d, _d, _d, _d, _d, _vp, _vp, _i, _vp]),
    "frl_sgd_momentum_mt_sr": (_i, [_vp, _vp, _vp, _vp, _vp, _i64, _u64, _i64, _d, _d, _d, _d, _d, _vp, _vp, _i,
                                    _vp]),
    "frl_adam_mt_sr": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _u64, _d, _d, _d, _d, _d, _i64, _d, _vp, _vp,
                            _vp]),
    "frl_adamw_mt_sr": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _u64, _d, _d, _d, _d, _d, _i64, _d, _vp, _vp,
                             _vp]),
    "frl_lion_mt_sr": (_i, [_vp, _vp, _vp, _vp, _vp, _i64, _u64, _i64, _d, _d, _d, _d, _d, _vp, _vp, _vp]),
    "frl_rmsprop_mt_sr": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _u64, _i64, _d, _d, _d, _d, _d, _d, _vp, _vp,
                               _vp]),
    "frl_weight_ema_bf16": (_i, [_vp, _vp, _i64, _d, _vp]),
    "frl_sgd_momentum_mt_grouped": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i, _d, _d, _d, _vp, _i,
                                         _vp]),
    "frl_adam_mt_grouped": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i, _d, _d, _d, _d, _vp,
                                 _vp]),
    "frl_adamw_mt_grouped": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i, _d, _d, _d, _d,
                                  _vp, _vp]),
    "frl_lion_mt_grouped": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i, _d, _d, _d, _vp, _vp]),
    "frl_rmsprop_mt_grouped": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i, _d, _d, _d, _d, _vp,
                                    _vp]),
    "frl_sgd_momentum_mt_grouped_sr": (_i, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i, _u64, _d, _d, _d, _vp,
                                            _i, _vp]),
    "frl_adam_mt_grouped_sr": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i, _u64, _d, _d, _d, _d,
                                    _vp, _vp]),
    "frl_adamw_mt_grouped_sr": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i, _u64, _d, _d, _d,
                                     _d, _vp, _vp]),
    "frl_lion_mt_grouped_sr": (_i, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i, _u64, _d, _d, _d, _vp, _vp]),
    "frl_rmsprop_mt_grouped_sr": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i, _u64, _d, _d, _d, _d,
                                       _vp, _vp]),
    "frl_layerwise_scratch_bytes": (_i64, [_i64, _i64]),
    "frl_lars_mt": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _d, _d, _d, _d, _vp, _vp, _i, _vp]),
    "frl_lamb_mt": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _d, _d, _d, _d, _d, _i64,
                         _d, _vp, _vp, _vp]),
    "frl_q8_tables": (None, [_vp, _vp]),
    "frl_adam8_mt": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _d, _d, _d, _d, _d,
                          _i64, _d, _vp, _vp, _vp]),
    "frl_adamw8_mt": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _d, _d, _d, _d, _d,
                           _i64, _d, _vp, _vp, _vp]),
    "frl_q8_encode_mt": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _i64, _i64, _vp, _vp]),
    "frl_q8_decode_mt": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _i64, _i64, _vp, _vp]),
    "frl_adafactor_plan": (_i64, [_vp, _i64, _vp, _vp]),
    "frl_adafactor_scratch_bytes": (_i64, [_vp, _i64]),
    "frl_adafactor_mt": (_i, [_vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _d, _d, _d, _d, _d, _d,
                              _i64, _d, _vp, _vp, _vp]),
    "frl_muon_plan_bytes": (_i64, [_vp, _i64, _vp, _vp]),
    "frl_muon_plan": (_i, [_vp, _i64, _vp, _vp, _vp]),
    "frl_muon_mt": (_i, [_vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _d, _d, _d, _i, _d, _d, _d, _i, _d, _i, _d, _vp,
                         _vp, _vp]),
    "frl_grad_accumulate_mt": (_i, [_vp, _vp, _vp, _vp, _i64, _d, _i, _vp, _vp]),
    "frl_weight_ema": (_i, [_vp, _vp, _i64, _d, _vp]),
    "frl_reduce_scratch_bytes": (_i64, []),
    "frl_grad_sumsq_clip": (_i, [_vp, _i64, _i, _f, _f, _vp, _vp, _vp]),
    "frl_criteria_scratch_bytes": (_i64, [_i]),
    "frl_criteria_forward": (_i, [C.POINTER(TaskDesc), _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "frl_criteria_backward": (_i, [C.POINTER(TaskDesc), _i, _vp, _vp, _vp, _vp]),
    "frl_preproc_affine": (_i, [_vp, _i, _vp, _i, _i64, _i64, _i64, _vp, _vp, _vp]),
    "frl_preproc_affine_nhwc": (_i, [_vp, _i, _vp, _i, _i64, _i, _i64, _vp, _vp, _vp]),
    "frl_cast_scale": (_i, [_vp, _i, _vp, _i, _i64, _f, _vp]),
    "frl_augment_images": (_i, [_vp, _i64, _i, _i, _i, _vp, C.c_uint64, _i, _i, _d, _d, _d, _d, _d, _i, _i,
                                _vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "frl_augment_mix_images": (_i, [_vp, _i64, _i, _i, _i, _vp, C.c_uint64, _i, _i, _d, _d, _d, _d, _d, _i, _i,
                                    _vp, _vp, _vp, _i, _i, _i, _vp, _i, _f, _i, _i, _i, _i, _vp]),
    "frl_augment_images_nhwc": (_i, [_vp, _i64, _i, _i, _i, _vp, C.c_uint64, _i, _i, _d, _d, _d, _d, _d, _i, _i,
                                     _vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "frl_augment_mix_images_nhwc": (_i, [_vp, _i64, _i, _i, _i, _vp, C.c_uint64, _i, _i, _d, _d, _d, _d, _d, _i,
                                         _i, _vp, _vp, _vp, _i, _i, _i, _vp, _i, _f, _i, _i, _i, _i, _vp]),
    "frl_mix_targets": (_i, [_vp, _i, _i64, _i64, _i, _f, _vp, _vp]),
    "frl_augment_policy_images": (_i, [_vp, _i64, _i, _i, _i, _vp, C.c_uint64, _i, _i, _d, _d, _d, _d, _i, _i, _i,
                                       _i, _i, _i, _vp, _d, _d, _d, _d, _d, _i, _vp, _vp, _vp, _vp, _i, _i, _i,
                                       _vp, _vp, _vp]),
    "frl_augment_policy_images_nhwc": (_i, [_vp, _i64, _i, _i, _i, _vp, C.c_uint64, _i, _i, _d, _d, _d, _d, _i, _i,
                                            _i, _i, _i, _i, _vp, _d, _d, _d, _d, _d, _i, _vp, _vp, _vp, _vp, _i, _i,
                                            _i, _vp, _vp, _vp]),
    "frl_mix_images": (_i, [_vp, _i, _i64, _i, _i, _i, _i, _f, _i, _i, _i, _i, _vp]),
    "frl_mix_images_nhwc": (_i, [_vp, _i, _i64, _i, _i, _i, _i, _f, _i, _i, _i, _i, _vp]),
    "frl_colsum_scratch_bytes": (_i64, [_i64, _i64]),
    "frl_colsum": (_i, [_vp, _i, _i64, _i64, _vp, _i, _i, _vp, _vp]),
    "frl_drelu_colsum": (_i, [_vp, _vp, _vp, _i, _i64, _i64, _vp, _i, _i, _vp, _vp]),
    "frl_gather_rows": (_i, [_vp, _i64, _vp, _vp, _i64, _i64, _i, _vp]),
    "frl_gather_rows_tma": (_i, [_vp, _i64, _vp, _vp, _i64, _i64, _i, _vp]),
    "frl_gather_window_rows": (_i, [_vp, _vp, _i, _vp, _vp, _i64, _i64, _vp]),
    "frl_gather_lines": (_i, [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _i64, _i64, _i, _i, _vp]),
    "frl_gather_pool_create": (_vp, [_i]),
    "frl_gather_pool_destroy": (None, [_vp]),
    "frl_gather_pool_threads": (_i, [_vp]),
    "frl_gather_pool_submit": (_i64, [_vp, _vp, _i64, _vp, _vp, _i64, _i64]),
    "frl_gather_pool_submit_f32_to_bf16": (_i64, [_vp, _vp, _i64, _vp, _vp, _i64, _i64]),
    "frl_gather_pool_wait": (_i, [_vp, _i64]),
    "frl_nvls_sgd": (_i, [_vp, _vp, _vp, _vp, _i64, _i, _i, _vp, _i, _vp, _i, _d, _d, _d, _d, _d, _vp, _i, _i, _i, _vp]),
    "frl_nvls_adam": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _vp, _i, _vp, _i, _d, _d, _d, _d, _d,
                           _i64, _d, _vp, _i, _i, _vp]),
    "frl_nvls_adamw": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _vp, _i, _vp, _i, _d, _d, _d, _d, _d,
                            _i64, _d, _vp, _i, _i, _vp]),
    "frl_nvls_lion": (_i, [_vp, _vp, _vp, _vp, _i64, _i, _i, _vp, _i, _vp, _i, _d, _d, _d, _d, _d, _vp, _i, _i,
                           _vp]),
    "frl_nvls_rmsprop": (_i, [_vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _vp, _i, _vp, _i, _d, _d, _d, _d, _d, _d,
                              _vp, _i, _i, _vp]),
    "frl_nvls_barrier": (_i, [_vp, _i, _i, _i, _vp]),
    "frl_fp8_amax": (_i, [_vp, _i64, _i, _vp, _vp]),
    "frl_fp8_quantize": (_i, [_vp, _i64, _i64, _i, _vp, _i, _vp, _vp, _vp, _vp]),
}

_lib: Optional[C.CDLL] = None


def build(verbose: bool = False) -> str:
    """Compile the library in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
    cmd = ["make", "-C", CSRC_DIR, "-j8"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        print(res.stdout)
        print(res.stderr)
    if res.returncode != 0:
        raise NativeLibraryError("building libfrl_b200.so failed:\n" + res.stderr[-4000:])
    return LIB_PATH


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeLibraryError(
                f"{LIB_PATH} is missing: the sm_90a kernel library has not been built "
                "(run `python __graft_entry__.py build` or `make -C <pkg>/csrc`). "
                "There is no fallback path.")
        handle = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(handle, name)        # AttributeError if the .so is stale
            fn.restype = restype
            fn.argtypes = argtypes
        if handle.frl_abi_version() != 1:
            raise NativeLibraryError("libfrl_b200.so ABI version mismatch; rebuild")
        _lib = handle
    return _lib


def is_available() -> bool:
    return os.path.exists(LIB_PATH)


def _check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().frl_last_error().decode("utf-8", "replace")
        raise NativeLibraryError(f"{what} failed (rc={rc}): {msg}")


def dtype_code(dt: torch.dtype) -> int:
    try:
        return _DTYPE_CODE[dt]
    except KeyError:
        raise NativeLibraryError(f"dtype {dt} has no kernel path") from None


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def launch_count() -> int:
    return int(lib().frl_launch_count())


def launch_count_reset() -> None:
    lib().frl_launch_count_reset()


# ---- K2 -------------------------------------------------------------------------------------

def sgd_momentum(p, g, buf, p_lp, n, *, lr, mu, dampening, wd, grad_scale=1.0,
                 grad_scale_dev=None, first_step=False, dyn=None) -> None:
    _check(lib().frl_sgd_momentum(_ptr(p), _ptr(g), _ptr(buf), _ptr(p_lp), n, lr, mu, dampening,
                                  wd, grad_scale, _ptr(grad_scale_dev), _ptr(dyn), int(first_step),
                                  dtype_code(g.dtype), _stream()), "frl_sgd_momentum")


def adam(p, g, m, v, vmax, p_lp, n, *, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
         grad_scale_dev=None, dyn=None) -> None:
    _check(lib().frl_adam(_ptr(p), _ptr(g), _ptr(m), _ptr(v), _ptr(vmax), _ptr(p_lp), n, lr,
                          beta1, beta2, eps, wd, step, grad_scale, _ptr(grad_scale_dev), _ptr(dyn),
                          dtype_code(g.dtype), _stream()), "frl_adam")


def adamw(p, g, m, v, vmax, p_lp, n, *, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
          grad_scale_dev=None, dyn=None) -> None:
    """K2 AdamW: ``adam``'s arguments, ``wd`` decoupled (see frl_adamw in include/frl_b200.h)."""
    _check(lib().frl_adamw(_ptr(p), _ptr(g), _ptr(m), _ptr(v), _ptr(vmax), _ptr(p_lp), n, lr,
                           beta1, beta2, eps, wd, step, grad_scale, _ptr(grad_scale_dev), _ptr(dyn),
                           dtype_code(g.dtype), _stream()), "frl_adamw")


def lion(p, g, m, p_lp, n, *, lr, beta1, beta2, wd, grad_scale=1.0, grad_scale_dev=None, dyn=None) -> None:
    """K2 Lion: ``sgd_momentum``'s arguments with (beta1, beta2) for (mu, dampening), m = exp_avg, ``wd``
    decoupled (see frl_lion in include/frl_b200.h)."""
    _check(lib().frl_lion(_ptr(p), _ptr(g), _ptr(m), _ptr(p_lp), n, lr, beta1, beta2, wd, grad_scale,
                          _ptr(grad_scale_dev), _ptr(dyn), dtype_code(g.dtype), _stream()), "frl_lion")


def rmsprop(p, g, sq, buf, p_lp, n, *, lr, alpha, eps, wd, mu, grad_scale=1.0,
            grad_scale_dev=None, dyn=None) -> None:
    _check(lib().frl_rmsprop(_ptr(p), _ptr(g), _ptr(sq), _ptr(buf), _ptr(p_lp), n, lr, alpha,
                             eps, wd, mu, grad_scale, _ptr(grad_scale_dev), _ptr(dyn),
                             dtype_code(g.dtype), _stream()), "frl_rmsprop")


# ---- K12: weight-gradient GEMM, optionally with the SGD update in its epilogue ----------------------

DW_TILE = (128, 256, 64)      # (out, in, rows) multiples K12 needs


def dw_gemm_fits(dz, x, gw) -> bool:
    """Whether K12 can compute gw = dz^T x: bf16 operands with unit column stride, rows 16-byte
    aligned, a contiguous bf16 output and shapes that are multiples of ``DW_TILE``."""
    tm, tn, tk = DW_TILE
    return (dz.dim() == 2 and x.dim() == 2 and dz.dtype == x.dtype == gw.dtype == torch.bfloat16
            and dz.stride(1) == 1 and x.stride(1) == 1 and dz.stride(0) % 8 == 0 and x.stride(0) % 8 == 0
            and dz.data_ptr() % 16 == 0 and x.data_ptr() % 16 == 0 and gw.data_ptr() % 16 == 0
            and gw.is_contiguous() and dz.shape[0] == x.shape[0] and tuple(gw.shape) == (dz.shape[1], x.shape[1])
            and dz.shape[1] % tm == 0 and x.shape[1] % tn == 0 and dz.shape[0] % tk == 0 and dz.shape[0] > 0)


def dw_gemm(dz, x, gw) -> None:
    """gw = dz^T x (bf16, fp32 accumulation) for dz [rows, out], x [rows, in]."""
    _check(lib().frl_dw_gemm(_ptr(dz), dz.stride(0), _ptr(x), x.stride(0), dz.shape[0], dz.shape[1], x.shape[1],
                             _ptr(gw), _stream()), "frl_dw_gemm")


def dw_gemm_sgd(dz, x, gw, p, buf, p_lp, *, lr, mu, dampening, wd, grad_scale=1.0, first_step=False,
                dyn=None) -> None:
    """gw = dz^T x, then ``sgd_momentum``'s update of the [out, in] slices p / buf / p_lp from it."""
    _check(lib().frl_dw_gemm_sgd(_ptr(dz), dz.stride(0), _ptr(x), x.stride(0), dz.shape[0], dz.shape[1],
                                 x.shape[1], _ptr(gw), _ptr(p), _ptr(buf), _ptr(p_lp), lr, mu, dampening, wd,
                                 grad_scale, _ptr(dyn), int(first_step), _stream()), "frl_dw_gemm_sgd")


def dw_gemm_sgd_sr(dz, x, gw, p, buf, *, arena_off, seed, t, lr, mu, dampening, wd, grad_scale=1.0,
                   first_step=False, dyn=None) -> None:
    """gw = dz^T x, then ``sgd_momentum_sr``'s update of the bf16 [out, in] weights p (arena elements
    from ``arena_off``) and buf from it."""
    if p.dtype != torch.bfloat16:
        raise NativeLibraryError("dw_gemm_sgd_sr: p must be the bf16 weights, got %s" % p.dtype)
    _check(lib().frl_dw_gemm_sgd_sr(_ptr(dz), dz.stride(0), _ptr(x), x.stride(0), dz.shape[0], dz.shape[1],
                                    x.shape[1], _ptr(gw), _ptr(p), _ptr(buf), arena_off, seed, t, lr, mu, dampening,
                                    wd, grad_scale, _ptr(dyn), int(first_step), _stream()), "frl_dw_gemm_sgd_sr")


def dw_gemm_lion(dz, x, gw, p, m, p_lp, *, lr, beta1, beta2, wd, grad_scale=1.0, dyn=None) -> None:
    """gw = dz^T x, then ``lion``'s update of the [out, in] slices p / m / p_lp from it."""
    _check(lib().frl_dw_gemm_lion(_ptr(dz), dz.stride(0), _ptr(x), x.stride(0), dz.shape[0], dz.shape[1],
                                  x.shape[1], _ptr(gw), _ptr(p), _ptr(m), _ptr(p_lp), lr, beta1, beta2, wd,
                                  grad_scale, _ptr(dyn), _stream()), "frl_dw_gemm_lion")


def dw_gemm_lion_sr(dz, x, gw, p, m, *, arena_off, seed, t, lr, beta1, beta2, wd, grad_scale=1.0,
                    dyn=None) -> None:
    """gw = dz^T x, then ``lion_sr``'s update of the bf16 [out, in] weights p (arena elements from
    ``arena_off``) and m from it."""
    if p.dtype != torch.bfloat16:
        raise NativeLibraryError("dw_gemm_lion_sr: p must be the bf16 weights, got %s" % p.dtype)
    _check(lib().frl_dw_gemm_lion_sr(_ptr(dz), dz.stride(0), _ptr(x), x.stride(0), dz.shape[0], dz.shape[1],
                                     x.shape[1], _ptr(gw), _ptr(p), _ptr(m), arena_off, seed, t, lr, beta1, beta2,
                                     wd, grad_scale, _ptr(dyn), _stream()), "frl_dw_gemm_lion_sr")


# ---- K13: data-gradient GEMM with the lower unit's ReLU backward and bias gradient in its epilogue --

def dx_drelu_fits(dz_up, w_up, act, db) -> bool:
    """Whether K13 can form dZ = [act > 0] * (dz_up w_up) and db from it: bf16 operands with unit
    column stride and rows 16-byte aligned, a bf16 bias gradient, rows a multiple of 128, columns a
    multiple of 256 and the contraction width a multiple of 8."""
    return (dz_up.dim() == 2 and w_up.dim() == 2 and act.dim() == 2 and db.dim() == 1
            and dz_up.dtype == w_up.dtype == act.dtype == db.dtype == torch.bfloat16
            and dz_up.stride(1) == 1 and w_up.stride(1) == 1 and act.stride(1) == 1
            and dz_up.stride(0) % 8 == 0 and w_up.stride(0) % 8 == 0 and act.stride(0) % 8 == 0
            and dz_up.data_ptr() % 16 == 0 and w_up.data_ptr() % 16 == 0 and act.data_ptr() % 16 == 0
            and dz_up.shape[1] == w_up.shape[0] and tuple(act.shape) == (dz_up.shape[0], w_up.shape[1])
            and db.shape[0] == act.shape[1] and db.stride(0) == 1
            and act.shape[0] % 128 == 0 and act.shape[0] > 0 and act.shape[1] % 256 == 0
            and dz_up.shape[1] % 8 == 0 and dz_up.shape[1] > 0)


_dx_drelu_scratch = {}

#: K13 reads dZ_up in 64-byte rows; when dZ_up's rows start on 128-byte boundaries (a row stride that
#: is a multiple of 64 bf16) no row straddles a cache line, and at the heads' K = 1064 the GEMM
#: measured 30 % faster on H100 than with the unpadded stride of 1064
DX_DRELU_ROW_ALIGN = 64


def dx_gemm_drelu(dz_up, w_up, act, dz_out, db_out, accumulate: bool = False) -> None:
    """dz_out = threshold_backward(bf16(dz_up @ w_up), act, 0); db_out (+)= its column sums (K13)."""
    rows, cols = act.shape
    key = (act.device.index, cols)
    need = int(lib().frl_dx_drelu_scratch_bytes(rows, cols))
    buf = _dx_drelu_scratch.get(key)
    if buf is None or buf.numel() * 4 < need:
        buf = _dx_drelu_scratch[key] = torch.zeros((need + 3) // 4, dtype=torch.int32, device=act.device)
    _check(lib().frl_dx_gemm_drelu(_ptr(dz_up), dz_up.stride(0), _ptr(w_up), w_up.stride(0), _ptr(act),
                                   act.stride(0), _ptr(dz_out), dz_out.stride(0), _ptr(db_out), rows,
                                   dz_up.shape[1], cols, int(accumulate), _ptr(buf), _stream()),
           "frl_dx_gemm_drelu")


# ---- K2-mt / K1: multi-tensor forms (gradients read where autograd left them) ---------------------

def mt_tile_elems() -> int:
    return int(lib().frl_mt_tile_elems())


def flatten_grads(table, arena_grad, *, scale: float = 1.0) -> None:
    """arena_grad[seg.arena_off + i] = cast(seg.g[i] * scale) for every segment of ``table``
    (a ``multi_tensor.GradSegTable`` whose device copy is current): one launch."""
    _check(lib().frl_flatten_grads(table.segs_dev_ptr, table.prefix_dev_ptr, table.tile_seg_dev_ptr, table.n_tiles,
                                   _ptr(arena_grad), dtype_code(arena_grad.dtype), scale, _stream()),
           "frl_flatten_grads")


def sgd_momentum_mt(p, buf, p_lp, table, *, lr, mu, dampening, wd, grad_scale=1.0, grad_scale_dev=None,
                    first_step=False, dyn=None) -> None:
    _check(lib().frl_sgd_momentum_mt(_ptr(p), _ptr(buf), _ptr(p_lp), table.segs_dev_ptr, table.prefix_dev_ptr,
                                     table.tile_seg_dev_ptr, table.n_tiles, lr, mu, dampening, wd, grad_scale,
                                     _ptr(grad_scale_dev), _ptr(dyn), int(first_step), _stream()),
           "frl_sgd_momentum_mt")


def adam_mt(p, m, v, vmax, p_lp, table, *, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
            grad_scale_dev=None, dyn=None) -> None:
    _check(lib().frl_adam_mt(_ptr(p), _ptr(m), _ptr(v), _ptr(vmax), _ptr(p_lp), table.segs_dev_ptr,
                             table.prefix_dev_ptr, table.tile_seg_dev_ptr, table.n_tiles, lr, beta1, beta2, eps, wd,
                             step, grad_scale, _ptr(grad_scale_dev), _ptr(dyn), _stream()), "frl_adam_mt")


def adamw_mt(p, m, v, vmax, p_lp, table, *, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
             grad_scale_dev=None, dyn=None) -> None:
    """K2-mt AdamW: ``adam_mt``'s arguments, ``wd`` decoupled."""
    _check(lib().frl_adamw_mt(_ptr(p), _ptr(m), _ptr(v), _ptr(vmax), _ptr(p_lp), table.segs_dev_ptr,
                              table.prefix_dev_ptr, table.tile_seg_dev_ptr, table.n_tiles, lr, beta1, beta2, eps, wd,
                              step, grad_scale, _ptr(grad_scale_dev), _ptr(dyn), _stream()), "frl_adamw_mt")


def lion_mt(p, m, p_lp, table, *, lr, beta1, beta2, wd, grad_scale=1.0, grad_scale_dev=None, dyn=None) -> None:
    """K2-mt Lion: ``lion``'s rule over a segment table (see frl_lion_mt)."""
    _check(lib().frl_lion_mt(_ptr(p), _ptr(m), _ptr(p_lp), table.segs_dev_ptr, table.prefix_dev_ptr,
                             table.tile_seg_dev_ptr, table.n_tiles, lr, beta1, beta2, wd, grad_scale,
                             _ptr(grad_scale_dev), _ptr(dyn), _stream()), "frl_lion_mt")


def rmsprop_mt(p, sq, buf, p_lp, table, *, lr, alpha, eps, wd, mu, grad_scale=1.0, grad_scale_dev=None,
               dyn=None) -> None:
    _check(lib().frl_rmsprop_mt(_ptr(p), _ptr(sq), _ptr(buf), _ptr(p_lp), table.segs_dev_ptr,
                                table.prefix_dev_ptr, table.tile_seg_dev_ptr, table.n_tiles, lr, alpha, eps, wd, mu,
                                grad_scale, _ptr(grad_scale_dev), _ptr(dyn), _stream()), "frl_rmsprop_mt")


# ---- K2-sr / K2-mt-sr: updates of bf16 master weights with stochastic rounding --------------------

def _check_sr(p, seed: int) -> None:
    if p.dtype != torch.bfloat16:
        raise NativeLibraryError("stochastic-rounding update: p must be the bf16 weights, got %s" % p.dtype)
    if not 0 <= seed < 1 << 64:
        raise NativeLibraryError("stochastic-rounding update: seed %r is not a uint64" % (seed,))


def sgd_momentum_sr(p, g, buf, n, *, arena_off, seed, t, lr, mu, dampening, wd, grad_scale=1.0,
                    grad_scale_dev=None, first_step=False, dyn=None) -> None:
    """K2 SGD on bf16 weights ``p`` (arena elements ``[arena_off, arena_off + n)``), rounded
    stochastically with the draws of update ``t`` (see frl_sgd_momentum_sr in include/frl_b200.h)."""
    _check_sr(p, seed)
    _check(lib().frl_sgd_momentum_sr(_ptr(p), _ptr(g), _ptr(buf), n, arena_off, seed, t, lr, mu, dampening, wd,
                                     grad_scale, _ptr(grad_scale_dev), _ptr(dyn), int(first_step),
                                     dtype_code(g.dtype), _stream()), "frl_sgd_momentum_sr")


def adam_sr(p, g, m, v, vmax, n, *, arena_off, seed, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
            grad_scale_dev=None, dyn=None) -> None:
    _check_sr(p, seed)
    _check(lib().frl_adam_sr(_ptr(p), _ptr(g), _ptr(m), _ptr(v), _ptr(vmax), n, arena_off, seed, lr, beta1, beta2,
                             eps, wd, step, grad_scale, _ptr(grad_scale_dev), _ptr(dyn), dtype_code(g.dtype),
                             _stream()), "frl_adam_sr")


def adamw_sr(p, g, m, v, vmax, n, *, arena_off, seed, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
             grad_scale_dev=None, dyn=None) -> None:
    _check_sr(p, seed)
    _check(lib().frl_adamw_sr(_ptr(p), _ptr(g), _ptr(m), _ptr(v), _ptr(vmax), n, arena_off, seed, lr, beta1, beta2,
                              eps, wd, step, grad_scale, _ptr(grad_scale_dev), _ptr(dyn), dtype_code(g.dtype),
                              _stream()), "frl_adamw_sr")


def lion_sr(p, g, m, n, *, arena_off, seed, t, lr, beta1, beta2, wd, grad_scale=1.0, grad_scale_dev=None,
            dyn=None) -> None:
    """K2-sr Lion: ``lion`` on bf16 weights p (arena elements from ``arena_off``), stored rounded
    stochastically with the draws of update ``t`` (see frl_lion_sr)."""
    _check_sr(p, seed)
    _check(lib().frl_lion_sr(_ptr(p), _ptr(g), _ptr(m), n, arena_off, seed, t, lr, beta1, beta2, wd, grad_scale,
                             _ptr(grad_scale_dev), _ptr(dyn), dtype_code(g.dtype), _stream()), "frl_lion_sr")


def rmsprop_sr(p, g, sq, buf, n, *, arena_off, seed, t, lr, alpha, eps, wd, mu, grad_scale=1.0,
               grad_scale_dev=None, dyn=None) -> None:
    _check_sr(p, seed)
    _check(lib().frl_rmsprop_sr(_ptr(p), _ptr(g), _ptr(sq), _ptr(buf), n, arena_off, seed, t, lr, alpha, eps, wd,
                                mu, grad_scale, _ptr(grad_scale_dev), _ptr(dyn), dtype_code(g.dtype), _stream()),
           "frl_rmsprop_sr")


def sgd_momentum_mt_sr(p, buf, table, *, seed, t, lr, mu, dampening, wd, grad_scale=1.0, grad_scale_dev=None,
                       first_step=False, dyn=None) -> None:
    """K2-mt SGD on the bf16 weights ``p`` (arena base) over the model slots of ``table``."""
    _check_sr(p, seed)
    _check(lib().frl_sgd_momentum_mt_sr(_ptr(p), _ptr(buf), table.segs_dev_ptr, table.prefix_dev_ptr,
                                        table.tile_seg_dev_ptr, table.n_tiles, seed, t, lr, mu, dampening, wd,
                                        grad_scale, _ptr(grad_scale_dev), _ptr(dyn), int(first_step), _stream()),
           "frl_sgd_momentum_mt_sr")


def adam_mt_sr(p, m, v, vmax, table, *, seed, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
               grad_scale_dev=None, dyn=None) -> None:
    _check_sr(p, seed)
    _check(lib().frl_adam_mt_sr(_ptr(p), _ptr(m), _ptr(v), _ptr(vmax), table.segs_dev_ptr, table.prefix_dev_ptr,
                                table.tile_seg_dev_ptr, table.n_tiles, seed, lr, beta1, beta2, eps, wd, step,
                                grad_scale, _ptr(grad_scale_dev), _ptr(dyn), _stream()), "frl_adam_mt_sr")


def adamw_mt_sr(p, m, v, vmax, table, *, seed, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
                grad_scale_dev=None, dyn=None) -> None:
    _check_sr(p, seed)
    _check(lib().frl_adamw_mt_sr(_ptr(p), _ptr(m), _ptr(v), _ptr(vmax), table.segs_dev_ptr, table.prefix_dev_ptr,
                                 table.tile_seg_dev_ptr, table.n_tiles, seed, lr, beta1, beta2, eps, wd, step,
                                 grad_scale, _ptr(grad_scale_dev), _ptr(dyn), _stream()), "frl_adamw_mt_sr")


def lion_mt_sr(p, m, table, *, seed, t, lr, beta1, beta2, wd, grad_scale=1.0, grad_scale_dev=None,
               dyn=None) -> None:
    """K2-mt-sr Lion: ``lion_mt`` on the bf16 weights' arena base p (see frl_lion_mt_sr)."""
    _check_sr(p, seed)
    _check(lib().frl_lion_mt_sr(_ptr(p), _ptr(m), table.segs_dev_ptr, table.prefix_dev_ptr, table.tile_seg_dev_ptr,
                                table.n_tiles, seed, t, lr, beta1, beta2, wd, grad_scale, _ptr(grad_scale_dev),
                                _ptr(dyn), _stream()), "frl_lion_mt_sr")


def rmsprop_mt_sr(p, sq, buf, table, *, seed, t, lr, alpha, eps, wd, mu, grad_scale=1.0, grad_scale_dev=None,
                  dyn=None) -> None:
    _check_sr(p, seed)
    _check(lib().frl_rmsprop_mt_sr(_ptr(p), _ptr(sq), _ptr(buf), table.segs_dev_ptr, table.prefix_dev_ptr,
                                   table.tile_seg_dev_ptr, table.n_tiles, seed, t, lr, alpha, eps, wd, mu,
                                   grad_scale, _ptr(grad_scale_dev), _ptr(dyn), _stream()), "frl_rmsprop_mt_sr")


# ---- K2-mt grouped / K2-mt-sr grouped: parameter groups over a segment table --------------------

GROUP_DYN_COLS = 8       # FRL_GROUP_DYN_COLS: floats per row of the group_dyn table


class SegGroups:
    """The group arrays of one segment table (see frl_*_mt_grouped in include/frl_b200.h): the
    device int32 ``seg_group`` / ``seg_flags`` of its segments and the fp32 ``[n_groups, 8]`` row
    table ``group_dyn`` (shared, not owned: the optimizer rewrites its rows).  The group indices are
    validated here, on the host, because the kernels do not read them back before launching."""

    def __init__(self, seg_group: Sequence[int], seg_flags: Sequence[int], group_dyn: torch.Tensor) -> None:
        if group_dyn.dtype != torch.float32 or group_dyn.dim() != 2 or group_dyn.shape[1] != GROUP_DYN_COLS \
                or not group_dyn.is_contiguous() or group_dyn.shape[0] < 1:
            raise NativeLibraryError("grouped update: group_dyn must be contiguous fp32 [n_groups >= 1, %d], got %s %s"
                                     % (GROUP_DYN_COLS, group_dyn.dtype, tuple(group_dyn.shape)))
        n_groups = group_dyn.shape[0]
        if len(seg_group) != len(seg_flags):
            raise NativeLibraryError("grouped update: %d segment groups for %d segment flags"
                                     % (len(seg_group), len(seg_flags)))
        bad = [g for g in seg_group if not 0 <= int(g) < n_groups]
        if bad:
            raise NativeLibraryError("grouped update: group indices %s outside [0, %d)" % (sorted(set(bad)), n_groups))
        dev = group_dyn.device
        self.n_segs = len(seg_group)
        self.n_groups = n_groups
        self.seg_group = torch.tensor([int(g) for g in seg_group] or [0], dtype=torch.int32).to(dev)
        self.seg_flags = torch.tensor([int(f) for f in seg_flags] or [0], dtype=torch.int32).to(dev)
        self.group_dyn = group_dyn


def _grouped(table, groups: "SegGroups"):
    if groups.n_segs != table.n_segs:
        raise NativeLibraryError("grouped update: group arrays of %d segments for a table of %d"
                                 % (groups.n_segs, table.n_segs))
    return (table.segs_dev_ptr, table.prefix_dev_ptr, table.tile_seg_dev_ptr, table.n_tiles,
            _ptr(groups.seg_group), _ptr(groups.seg_flags), _ptr(groups.group_dyn), groups.n_groups)


def sgd_momentum_mt_grouped(p, buf, p_lp, table, groups, *, mu, dampening, grad_scale=1.0, grad_scale_dev=None,
                            first_step=False) -> None:
    """K2-mt SGD with each segment's lr / wd from its group's row (see frl_sgd_momentum_mt_grouped)."""
    _check(lib().frl_sgd_momentum_mt_grouped(_ptr(p), _ptr(buf), _ptr(p_lp), *_grouped(table, groups), mu, dampening,
                                             grad_scale, _ptr(grad_scale_dev), int(first_step), _stream()),
           "frl_sgd_momentum_mt_grouped")


def adam_mt_grouped(p, m, v, vmax, p_lp, table, groups, *, beta1, beta2, eps, grad_scale=1.0,
                    grad_scale_dev=None) -> None:
    _check(lib().frl_adam_mt_grouped(_ptr(p), _ptr(m), _ptr(v), _ptr(vmax), _ptr(p_lp), *_grouped(table, groups),
                                     beta1, beta2, eps, grad_scale, _ptr(grad_scale_dev), _stream()),
           "frl_adam_mt_grouped")


def adamw_mt_grouped(p, m, v, vmax, p_lp, table, groups, *, beta1, beta2, eps, grad_scale=1.0,
                     grad_scale_dev=None) -> None:
    _check(lib().frl_adamw_mt_grouped(_ptr(p), _ptr(m), _ptr(v), _ptr(vmax), _ptr(p_lp), *_grouped(table, groups),
                                      beta1, beta2, eps, grad_scale, _ptr(grad_scale_dev), _stream()),
           "frl_adamw_mt_grouped")


def lion_mt_grouped(p, m, p_lp, table, groups, *, beta1, beta2, grad_scale=1.0, grad_scale_dev=None) -> None:
    _check(lib().frl_lion_mt_grouped(_ptr(p), _ptr(m), _ptr(p_lp), *_grouped(table, groups), beta1, beta2,
                                     grad_scale, _ptr(grad_scale_dev), _stream()), "frl_lion_mt_grouped")


def rmsprop_mt_grouped(p, sq, buf, p_lp, table, groups, *, alpha, eps, mu, grad_scale=1.0,
                       grad_scale_dev=None) -> None:
    _check(lib().frl_rmsprop_mt_grouped(_ptr(p), _ptr(sq), _ptr(buf), _ptr(p_lp), *_grouped(table, groups), alpha,
                                        eps, mu, grad_scale, _ptr(grad_scale_dev), _stream()),
           "frl_rmsprop_mt_grouped")


def sgd_momentum_mt_grouped_sr(p, buf, table, groups, *, seed, mu, dampening, grad_scale=1.0, grad_scale_dev=None,
                               first_step=False) -> None:
    """K2-mt-sr SGD with each segment's lr / wd and the update count from its group's row."""
    _check_sr(p, seed)
    _check(lib().frl_sgd_momentum_mt_grouped_sr(_ptr(p), _ptr(buf), *_grouped(table, groups), seed, mu, dampening,
                                                grad_scale, _ptr(grad_scale_dev), int(first_step), _stream()),
           "frl_sgd_momentum_mt_grouped_sr")


def adam_mt_grouped_sr(p, m, v, vmax, table, groups, *, seed, beta1, beta2, eps, grad_scale=1.0,
                       grad_scale_dev=None) -> None:
    _check_sr(p, seed)
    _check(lib().frl_adam_mt_grouped_sr(_ptr(p), _ptr(m), _ptr(v), _ptr(vmax), *_grouped(table, groups), seed, beta1,
                                        beta2, eps, grad_scale, _ptr(grad_scale_dev), _stream()),
           "frl_adam_mt_grouped_sr")


def adamw_mt_grouped_sr(p, m, v, vmax, table, groups, *, seed, beta1, beta2, eps, grad_scale=1.0,
                        grad_scale_dev=None) -> None:
    _check_sr(p, seed)
    _check(lib().frl_adamw_mt_grouped_sr(_ptr(p), _ptr(m), _ptr(v), _ptr(vmax), *_grouped(table, groups), seed,
                                         beta1, beta2, eps, grad_scale, _ptr(grad_scale_dev), _stream()),
           "frl_adamw_mt_grouped_sr")


def lion_mt_grouped_sr(p, m, table, groups, *, seed, beta1, beta2, grad_scale=1.0, grad_scale_dev=None) -> None:
    _check_sr(p, seed)
    _check(lib().frl_lion_mt_grouped_sr(_ptr(p), _ptr(m), *_grouped(table, groups), seed, beta1, beta2, grad_scale,
                                        _ptr(grad_scale_dev), _stream()), "frl_lion_mt_grouped_sr")


def rmsprop_mt_grouped_sr(p, sq, buf, table, groups, *, seed, alpha, eps, mu, grad_scale=1.0,
                          grad_scale_dev=None) -> None:
    _check_sr(p, seed)
    _check(lib().frl_rmsprop_mt_grouped_sr(_ptr(p), _ptr(sq), _ptr(buf), *_grouped(table, groups), seed, alpha, eps,
                                           mu, grad_scale, _ptr(grad_scale_dev), _stream()),
           "frl_rmsprop_mt_grouped_sr")


# ---- K2-lw: layer-wise adaptive updates (LARS, LAMB) over a segment table -------------------------

LW_ADAPTED, LW_CLIPPED = 1, 2


def layerwise_scratch_bytes(n_tiles: int, n_segs: int) -> int:
    return int(lib().frl_layerwise_scratch_bytes(n_tiles, n_segs))


def _check_layerwise(table, flags, ratio, scratch, *vecs) -> None:
    for t in vecs:
        if t is not None and not (t.dtype == torch.float32 and t.is_contiguous()):
            raise NativeLibraryError("layer-wise update: master weights and state must be contiguous fp32")
    if flags.dtype != torch.int32 or flags.numel() < table.n_segs:
        raise NativeLibraryError("layer-wise update: seg_flags must be int32 [n_segs]")
    if ratio.dtype != torch.float32 or ratio.numel() < table.n_segs:
        raise NativeLibraryError("layer-wise update: ratio must be fp32 [n_segs]")
    if scratch.numel() * scratch.element_size() < layerwise_scratch_bytes(table.n_tiles, table.n_segs):
        raise NativeLibraryError("layer-wise update: scratch too small")


def lars_mt(p, buf, p_lp, table, flags, ratio, scratch, *, lr, mu, wd, grad_scale=1.0,
            grad_scale_dev=None, first_step=False, dyn=None) -> None:
    """K2-lw LARS over the segments of ``table``; ``ratio`` receives each tensor's trust ratio.
    See frl_lars_mt in include/frl_b200.h."""
    _check_layerwise(table, flags, ratio, scratch, p, buf)
    _check(lib().frl_lars_mt(_ptr(p), _ptr(buf), _ptr(p_lp), table.segs_dev_ptr, table.prefix_dev_ptr,
                             table.tile_seg_dev_ptr, table.n_tiles, table.n_segs, _ptr(flags), _ptr(ratio),
                             _ptr(scratch), lr, mu, wd, grad_scale, _ptr(grad_scale_dev), _ptr(dyn),
                             int(first_step), _stream()), "frl_lars_mt")


def lamb_mt(p, m, v, p_lp, table, flags, ratio, scratch, *, lr, beta1, beta2, eps, wd, step,
            grad_scale=1.0, grad_scale_dev=None, dyn=None) -> None:
    """K2-lw LAMB over the segments of ``table``.  See frl_lamb_mt in include/frl_b200.h."""
    _check_layerwise(table, flags, ratio, scratch, p, m, v)
    _check(lib().frl_lamb_mt(_ptr(p), _ptr(m), _ptr(v), _ptr(p_lp), table.segs_dev_ptr, table.prefix_dev_ptr,
                             table.tile_seg_dev_ptr, table.n_tiles, table.n_segs, _ptr(flags), _ptr(ratio),
                             _ptr(scratch), lr, beta1, beta2, eps, wd, step, grad_scale, _ptr(grad_scale_dev),
                             _ptr(dyn), _stream()), "frl_lamb_mt")


# ---- K2-q8: Adam with 8-bit block-wise state over a segment table ---------------------------------

Q8_BLOCK = 256                        # elements per quantisation block (FRL_Q8_BLOCK)
Q8_EXP_AVG, Q8_EXP_AVG_SQ = 0, 1


def q8_device_tables():
    """The library's (MAG7, MAG8) tables as fp32 CPU tensors of 128 and 256 entries."""
    mag7, mag8 = torch.zeros(128, dtype=torch.float32), torch.zeros(256, dtype=torch.float32)
    lib().frl_q8_tables(_ptr(mag7), _ptr(mag8))
    return mag7, mag8


def _check_q8(table, qbase, flags=None, codes=(), absmax=(), fp32=()) -> None:
    for t in fp32:
        if t is not None and not (t.dtype == torch.float32 and t.is_contiguous()):
            raise NativeLibraryError("8-bit state: master weights and fp32 state must be contiguous fp32")
    for q in codes:
        if not (q.dtype == torch.uint8 and q.is_contiguous()):
            raise NativeLibraryError("8-bit state: codes must be contiguous uint8 (one byte per arena element)")
    for a in absmax:
        if not (a.dtype == torch.float32 and a.is_contiguous()):
            raise NativeLibraryError("8-bit state: absmax must be contiguous fp32")
    if qbase.dtype != torch.int64 or qbase.numel() < table.n_segs:
        raise NativeLibraryError("8-bit state: qbase must be int64 [n_segs]")
    if flags is not None and (flags.dtype != torch.int32 or flags.numel() < table.n_segs):
        raise NativeLibraryError("8-bit state: seg_flags must be int32 [n_segs]")


def adam8_mt(p, m_q, v_q, m_absmax, v_absmax, p_lp, table, qbase, flags, *, lr, beta1, beta2, eps, wd, step,
             grad_scale=1.0, grad_scale_dev=None, dyn=None) -> None:
    """K2-q8 Adam over the segments of ``table`` with 8-bit block-wise ``exp_avg`` / ``exp_avg_sq``.
    See frl_adam8_mt in include/frl_b200.h."""
    _check_q8(table, qbase, flags, codes=(m_q, v_q), absmax=(m_absmax, v_absmax), fp32=(p,))
    _check(lib().frl_adam8_mt(_ptr(p), _ptr(m_q), _ptr(v_q), _ptr(m_absmax), _ptr(v_absmax), _ptr(p_lp),
                              table.segs_dev_ptr, table.prefix_dev_ptr, table.tile_seg_dev_ptr, table.n_tiles,
                              table.n_segs, _ptr(qbase), _ptr(flags), lr, beta1, beta2, eps, wd, step, grad_scale,
                              _ptr(grad_scale_dev), _ptr(dyn), _stream()), "frl_adam8_mt")


def adamw8_mt(p, m_q, v_q, m_absmax, v_absmax, p_lp, table, qbase, flags, *, lr, beta1, beta2, eps, wd, step,
              grad_scale=1.0, grad_scale_dev=None, dyn=None) -> None:
    """K2-q8 AdamW: ``adam8_mt``'s arguments, ``wd`` decoupled.  See frl_adamw8_mt in include/frl_b200.h."""
    _check_q8(table, qbase, flags, codes=(m_q, v_q), absmax=(m_absmax, v_absmax), fp32=(p,))
    _check(lib().frl_adamw8_mt(_ptr(p), _ptr(m_q), _ptr(v_q), _ptr(m_absmax), _ptr(v_absmax), _ptr(p_lp),
                               table.segs_dev_ptr, table.prefix_dev_ptr, table.tile_seg_dev_ptr, table.n_tiles,
                               table.n_segs, _ptr(qbase), _ptr(flags), lr, beta1, beta2, eps, wd, step, grad_scale,
                               _ptr(grad_scale_dev), _ptr(dyn), _stream()), "frl_adamw8_mt")


def q8_encode_mt(x, q, absmax, state: int, table, qbase) -> None:
    """Codes and absmax of the fp32 arena-shaped ``x`` over the segments of ``table`` (``state``:
    ``Q8_EXP_AVG`` or ``Q8_EXP_AVG_SQ``).  See frl_q8_encode_mt in include/frl_b200.h."""
    _check_q8(table, qbase, codes=(q,), absmax=(absmax,), fp32=(x,))
    _check(lib().frl_q8_encode_mt(_ptr(x), _ptr(q), _ptr(absmax), int(state), table.segs_dev_ptr,
                                  table.prefix_dev_ptr, table.tile_seg_dev_ptr, table.n_tiles, table.n_segs,
                                  _ptr(qbase), _stream()), "frl_q8_encode_mt")


def q8_decode_mt(q, absmax, x, state: int, table, qbase) -> None:
    """fp32 values of the codes over the segments of ``table`` into the arena-shaped ``x``.  See
    frl_q8_decode_mt in include/frl_b200.h."""
    _check_q8(table, qbase, codes=(q,), absmax=(absmax,), fp32=(x,))
    _check(lib().frl_q8_decode_mt(_ptr(q), _ptr(absmax), _ptr(x), int(state), table.segs_dev_ptr,
                                  table.prefix_dev_ptr, table.tile_seg_dev_ptr, table.n_tiles, table.n_segs,
                                  _ptr(qbase), _stream()), "frl_q8_decode_mt")


# ---- K2-af: Adafactor over a segment table ----------------------------------------------------------

def _host_shape(shape: torch.Tensor) -> torch.Tensor:
    if shape.dtype != torch.int64 or shape.dim() != 2 or shape.shape[1] != 3 or shape.device.type != "cpu":
        raise NativeLibraryError("Adafactor: shape must be a CPU int64 [n_segs, 3] tensor of (B, R, C)")
    return shape.contiguous()


def adafactor_plan(shape: torch.Tensor):
    """Band table of the segments' (B, R, C) shapes: (work int64 [n_work, 4], seg_info int64
    [n_segs, 3]) on the CPU.  See frl_adafactor_plan in include/frl_b200.h."""
    shape = _host_shape(shape)
    n_segs = shape.shape[0]
    n = int(lib().frl_adafactor_plan(_ptr(shape), n_segs, None, None))
    if n < 0:
        raise NativeLibraryError("Adafactor: bad segment shape")
    work = torch.zeros(n, 4, dtype=torch.int64)
    seg_info = torch.zeros(n_segs, 3, dtype=torch.int64)
    lib().frl_adafactor_plan(_ptr(shape), n_segs, _ptr(work), _ptr(seg_info))
    return work, seg_info


def adafactor_scratch_bytes(shape: torch.Tensor) -> int:
    shape = _host_shape(shape)
    n = int(lib().frl_adafactor_scratch_bytes(_ptr(shape), shape.shape[0]))
    if n < 0:
        raise NativeLibraryError("Adafactor: bad segment shape")
    return n


def adafactor_mt(p, state, p_lp, table, plan, *, lr, beta2_decay, eps1, eps2, d, wd, step, grad_scale=1.0,
                 grad_scale_dev=None, dyn=None) -> None:
    """K2-af Adafactor over the segments of ``table``.  ``plan``: the device arrays (shape,
    state_off, seg_flags, work, seg_info, scratch) and the host shape they were built from.  See
    frl_adafactor_mt in include/frl_b200.h."""
    shape_dev, state_off, flags, work, seg_info, scratch, shape_host = plan
    for t in (p, state):
        if not (t.dtype == torch.float32 and t.is_contiguous()):
            raise NativeLibraryError("Adafactor: master weights and state must be contiguous fp32")
    n = table.n_segs
    if (shape_dev.dtype != torch.int64 or shape_dev.numel() < 3 * n or state_off.dtype != torch.int64
            or state_off.numel() < n or flags.dtype != torch.int32 or flags.numel() < n
            or work.dtype != torch.int64 or seg_info.dtype != torch.int64 or seg_info.numel() < 3 * n):
        raise NativeLibraryError("Adafactor: shape/state_off/work/seg_info must be int64, seg_flags int32, "
                                 "each covering the table's segments")
    if n and scratch.numel() * scratch.element_size() < adafactor_scratch_bytes(shape_host):
        raise NativeLibraryError("Adafactor: scratch too small")
    _check(lib().frl_adafactor_mt(_ptr(p), _ptr(state), _ptr(p_lp), table.segs_dev_ptr, n, _ptr(shape_dev),
                                  _ptr(state_off), _ptr(flags), _ptr(work), work.shape[0] if n else 0,
                                  _ptr(seg_info), _ptr(scratch), lr, beta2_decay, eps1, eps2, d, wd, step,
                                  grad_scale, _ptr(grad_scale_dev), _ptr(dyn), _stream()), "frl_adafactor_mt")


# ---- K14: Muon over a segment table -----------------------------------------------------------------

class MuonPlan:
    """K14's plan for one segment table: the host and device copies of the tile tables and tensor
    maps, its scratch (tickets, norms, partials), the matrices' (segment, arena offset, R, C) rows,
    and the workspace and exp_avg_sq vector the plan points into."""

    def __init__(self, shape, host, dev, scratch, workspace, state):
        self.shape, self.host, self.dev, self.scratch = shape, host, dev, scratch
        self.workspace, self.state = workspace, state
        self.n_mat = shape.shape[0]


def _muon_shape(shape: torch.Tensor) -> torch.Tensor:
    if shape.dtype != torch.int64 or shape.dim() != 2 or shape.shape[1] != 4 or shape.device.type != "cpu":
        raise NativeLibraryError("Muon: shape must be a CPU int64 [n_mat, 4] tensor of (segment, arena offset, R, C)")
    return shape.contiguous()


def muon_plan_bytes(shape: torch.Tensor):
    """(plan bytes, scratch bytes, workspace bytes) of the matrices in ``shape``; host only."""
    shape = _muon_shape(shape)
    scratch, ws = C.c_int64(0), C.c_int64(0)
    n = int(lib().frl_muon_plan_bytes(_ptr(shape), shape.shape[0], C.byref(scratch), C.byref(ws)))
    if n < 0:
        raise NativeLibraryError("Muon: bad matrix shape")
    return n, int(scratch.value), int(ws.value)


def muon_plan(shape: torch.Tensor, exp_avg_sq: torch.Tensor, workspace: torch.Tensor) -> MuonPlan:
    """Plan K14 over the matrices of ``shape`` (see frl_muon_plan in include/frl_b200.h), with the
    iterates in ``exp_avg_sq`` (fp32, arena-shaped), the Gram buffers in ``workspace`` (which plans
    over subsets of the same matrices may share) and a fresh zeroed scratch."""
    shape = _muon_shape(shape)
    if exp_avg_sq.dtype != torch.float32 or not exp_avg_sq.is_contiguous():
        raise NativeLibraryError("Muon: exp_avg_sq must be contiguous fp32")
    nbytes, scratch_bytes, ws_bytes = muon_plan_bytes(shape)
    if workspace.numel() * workspace.element_size() < ws_bytes or workspace.data_ptr() % 128:
        raise NativeLibraryError("Muon: workspace needs %d bytes, 128-byte aligned" % ws_bytes)
    dev = exp_avg_sq.device
    scratch = torch.zeros((scratch_bytes + 15) // 16 * 4, dtype=torch.int32, device=dev)
    host = torch.zeros((nbytes + 63) // 64 * 64, dtype=torch.uint8)
    _check(lib().frl_muon_plan(_ptr(shape), shape.shape[0], _ptr(exp_avg_sq), _ptr(workspace), _ptr(host)),
           "frl_muon_plan")
    return MuonPlan(shape, host, host.to(dev), scratch, workspace, exp_avg_sq)


def check_muon_hyper(*, lr, wd, momentum, ns_steps, eps, adjust_lr_fn) -> None:
    """The argument checks of frl_muon_mt, for a caller that must refuse before launching anything."""
    if not (float(lr) >= 0.0 and float(wd) >= 0.0 and float(momentum) >= 0.0 and float(eps) >= 0.0):
        raise NativeLibraryError("Muon: lr, weight_decay, momentum and eps must be >= 0")
    if int(ns_steps) != ns_steps or not 1 <= int(ns_steps) < 100:
        raise NativeLibraryError("Muon: ns_steps must be an integer in [1, 100), got %r" % (ns_steps,))
    if adjust_lr_fn not in (None, "original", "match_rms_adamw"):
        raise NativeLibraryError("Muon: adjust_lr_fn must be None, 'original' or 'match_rms_adamw'")


def muon_mt(p, exp_avg, p_lp, table, plan: MuonPlan, *, lr, wd, momentum, nesterov, ns_coefficients, ns_steps, eps,
            adjust_lr_fn, grad_scale=1.0, grad_scale_dev=None, dyn=None) -> None:
    """K14 Muon over the matrices of ``plan``, gradients read through ``table`` (the plan's segment
    indices refer to it).  See frl_muon_mt in include/frl_b200.h."""
    for t in (p, exp_avg):
        if not (t.dtype == torch.float32 and t.is_contiguous()):
            raise NativeLibraryError("Muon: master weights and exp_avg must be contiguous fp32")
    check_muon_hyper(lr=lr, wd=wd, momentum=momentum, ns_steps=ns_steps, eps=eps, adjust_lr_fn=adjust_lr_fn)
    if dyn is not None and (dyn.dtype != torch.float32 or dyn.numel() < 3):
        raise NativeLibraryError("Muon: dyn must be fp32 with at least 3 elements")
    for seg, _, r, c in plan.shape.tolist():
        if not (0 <= seg < table.n_segs and table.slots[seg].numel == r * c):
            raise NativeLibraryError("Muon: the plan's matrix [%d, %d] does not match segment %d of the table"
                                     % (r, c, seg))
    a, b, c = (float(x) for x in ns_coefficients)
    _check(lib().frl_muon_mt(_ptr(p), _ptr(exp_avg), _ptr(p_lp), table.segs_dev_ptr, table.n_segs, _ptr(plan.host),
                             _ptr(plan.dev), _ptr(plan.scratch), float(lr), float(wd), float(momentum),
                             int(bool(nesterov)), a, b, c, int(ns_steps), float(eps),
                             int(adjust_lr_fn == "match_rms_adamw"), float(grad_scale), _ptr(grad_scale_dev),
                             _ptr(dyn), _stream()), "frl_muon_mt")


# ---- K10: gradient accumulation over a segment table ----------------------------------------------

def grad_accumulate_mt(acc, table, *, w: float = 1.0, first: bool = False, dyn=None) -> None:
    """acc[slot] = (first ? 0 : acc[slot]) + w * g for every slot of ``table`` (a
    ``multi_tensor.GradSegTable`` whose device copy is current; a slot pointed at address 0
    contributes nothing).  ``dyn``: optional device fp32 [2] = (w, first) overriding the
    arguments.  See frl_grad_accumulate_mt in include/frl_b200.h."""
    if acc.dtype != torch.float32 or not acc.is_contiguous():
        raise NativeLibraryError("gradient accumulation: the accumulator must be contiguous fp32")
    if dyn is not None and (dyn.dtype != torch.float32 or dyn.numel() < 2):
        raise NativeLibraryError("gradient accumulation: dyn must be fp32 [2]")
    _check(lib().frl_grad_accumulate_mt(_ptr(acc), table.segs_dev_ptr, table.prefix_dev_ptr, table.tile_seg_dev_ptr,
                                        table.n_tiles, float(w), int(bool(first)), _ptr(dyn), _stream()),
           "frl_grad_accumulate_mt")


# ---- K11: weight EMA ------------------------------------------------------------------------------

def weight_ema(ema, p, w: float) -> None:
    """ema = lerp(ema, p, w) in fp32, torch's formula, over ``ema.numel()`` elements of two
    contiguous fp32 device vectors (``p`` at least as long).  See frl_weight_ema in
    include/frl_b200.h."""
    if ema.dtype != torch.float32 or p.dtype != torch.float32 or not (ema.is_contiguous() and p.is_contiguous()):
        raise NativeLibraryError("weight EMA: ema and p must be contiguous fp32")
    if p.numel() < ema.numel():
        raise NativeLibraryError("weight EMA: p has %d elements, ema %d" % (p.numel(), ema.numel()))
    _check(lib().frl_weight_ema(_ptr(ema), _ptr(p), ema.numel(), float(w), _stream()), "frl_weight_ema")


def weight_ema_bf16(ema, p, w: float) -> None:
    """``weight_ema`` with ``p`` the contiguous bf16 weights (frl_weight_ema_bf16)."""
    if ema.dtype != torch.float32 or p.dtype != torch.bfloat16 or not (ema.is_contiguous() and p.is_contiguous()):
        raise NativeLibraryError("weight EMA (bf16): ema must be contiguous fp32 and p contiguous bf16")
    if p.numel() < ema.numel():
        raise NativeLibraryError("weight EMA (bf16): p has %d elements, ema %d" % (p.numel(), ema.numel()))
    _check(lib().frl_weight_ema_bf16(_ptr(ema), _ptr(p), ema.numel(), float(w), _stream()), "frl_weight_ema_bf16")


# ---- K3 -------------------------------------------------------------------------------------

def reduce_scratch_bytes() -> int:
    return int(lib().frl_reduce_scratch_bytes())


def grad_sumsq_clip(g, n, *, pre_scale, max_norm, out3, scratch) -> None:
    _check(lib().frl_grad_sumsq_clip(_ptr(g), n, dtype_code(g.dtype), pre_scale, max_norm,
                                     _ptr(out3), _ptr(scratch), _stream()), "frl_grad_sumsq_clip")


# ---- K4 -------------------------------------------------------------------------------------

def criteria_scratch_bytes(n_tasks: int) -> int:
    return int(lib().frl_criteria_scratch_bytes(n_tasks))


def make_task_array(descs: Sequence[TaskDesc]):
    arr = (TaskDesc * len(descs))()
    for i, d in enumerate(descs):
        arr[i] = d
    return arr


def criteria_forward(task_array, n_tasks, losses, aux, lse, sink, nan_flag, scratch) -> None:
    _check(lib().frl_criteria_forward(task_array, n_tasks, _ptr(losses), _ptr(aux), _ptr(lse),
                                      _ptr(sink), _ptr(nan_flag), _ptr(scratch), _stream()),
           "frl_criteria_forward")


def criteria_backward(task_array, n_tasks, grad_losses, aux, lse) -> None:
    _check(lib().frl_criteria_backward(task_array, n_tasks, _ptr(grad_losses), _ptr(aux),
                                       _ptr(lse), _stream()), "frl_criteria_backward")


# ---- K5 -------------------------------------------------------------------------------------

def preproc_affine(src, dst, *, inner=1, channels=1, scale=None, bias=None) -> None:
    n = src.numel()
    assert dst.numel() == n and src.is_contiguous() and dst.is_contiguous()
    _check(lib().frl_preproc_affine(_ptr(src), dtype_code(src.dtype), _ptr(dst),
                                    dtype_code(dst.dtype), n, inner, channels, _ptr(scale),
                                    _ptr(bias), _stream()), "frl_preproc_affine")


def is_nhwc(t) -> bool:
    """A 4-D tensor stored channels_last whose NCHW order differs (C, H and W not all trivial)."""
    return t.dim() == 4 and not t.is_contiguous() and t.is_contiguous(memory_format=torch.channels_last)


def preproc_affine_nhwc(src, dst, *, scale=None, bias=None) -> None:
    """K5 into channels_last: ``src`` contiguous [B, C, H, W] (1 <= C <= 4) -> ``dst`` [B, C, H, W]
    stored channels_last, the values of ``preproc_affine(src, ..., inner=H*W, channels=C)``."""
    B, Cc, H, W = src.shape
    assert src.is_contiguous() and dst.shape == src.shape
    assert dst.is_contiguous(memory_format=torch.channels_last)
    _check(lib().frl_preproc_affine_nhwc(_ptr(src), dtype_code(src.dtype), _ptr(dst), dtype_code(dst.dtype),
                                         B, Cc, H * W, _ptr(scale), _ptr(bias), _stream()),
           "frl_preproc_affine_nhwc")


AUG_RRC, AUG_PAD_CROP, AUG_CENTER_RESIZE, AUG_CENTER_CROP = 0, 1, 2, 3


MIX_MIXUP, MIX_CUTMIX = 1, 2


def _augment_args(src, idx, dst, seed, epoch, mode, scale_range, ratio_range, eval_crop, pad, flip, scale, bias,
                  params_out):
    B, Cc, H, W = src.shape
    assert src.dtype == torch.uint8 and src.is_contiguous() and (dst.is_contiguous() or is_nhwc(dst))
    assert dst.dim() == 4 and tuple(dst.shape[:2]) == (B, Cc)
    assert idx.dtype == torch.int64 and idx.is_contiguous() and idx.numel() == B
    assert params_out is None or (params_out.dtype == torch.int32 and params_out.is_contiguous()
                                  and tuple(params_out.shape) == (B, 5))
    return [_ptr(src), B, Cc, H, W, _ptr(idx), int(seed) & (2 ** 64 - 1), int(epoch),
            int(mode), float(scale_range[0]), float(scale_range[1]),
            float(ratio_range[0]), float(ratio_range[1]), float(eval_crop), int(pad),
            int(bool(flip)), _ptr(scale), _ptr(bias), _ptr(dst), dtype_code(dst.dtype),
            dst.shape[2], dst.shape[3], _ptr(params_out)]


def augment_images(src, idx, dst, *, seed: int, epoch: int, mode: int, scale_range=(0.08, 1.0),
                   ratio_range=(3.0 / 4.0, 4.0 / 3.0), eval_crop: float = 0.875, pad: int = 0,
                   flip: bool = True, scale=None, bias=None, params_out=None) -> None:
    """K5a: crop box drawn per (seed, epoch, idx[b]), bilinear resize to ``dst``'s [out_h, out_w],
    optional flip, then ``x * scale[c] + bias[c]``.  ``src`` uint8 [B, C, H, W], ``idx`` device
    int64 [B], ``dst`` fp32/bf16 [B, C, out_h, out_w] (contiguous, or channels_last: then
    ``frl_augment_images_nhwc`` writes it), ``params_out`` optional int32 [B, 5]
    (top, left, h, w, flipped).  See frl_augment_images in include/frl_b200.h."""
    args = _augment_args(src, idx, dst, seed, epoch, mode, scale_range, ratio_range, eval_crop, pad, flip, scale,
                         bias, params_out)
    name = "frl_augment_images_nhwc" if is_nhwc(dst) else "frl_augment_images"
    _check(getattr(lib(), name)(*args, _stream()), name)


def augment_mix_images(src, idx, dst, *, mix_mode: int, lam: float, box=(0, 0, 0, 0), seed: int, epoch: int,
                       mode: int, scale_range=(0.08, 1.0), ratio_range=(3.0 / 4.0, 4.0 / 3.0),
                       eval_crop: float = 0.875, pad: int = 0, flip: bool = True, scale=None, bias=None,
                       params_out=None) -> None:
    """K5a with Mixup (``mix_mode=MIX_MIXUP``) or CutMix (``MIX_CUTMIX``, ``box`` = (y0, y1, x0, x1)
    on the output image) of sample p with sample B-1-p, in the same pass.  Other arguments as
    ``augment_images``.  See frl_augment_mix_images in include/frl_b200.h."""
    args = _augment_args(src, idx, dst, seed, epoch, mode, scale_range, ratio_range, eval_crop, pad, flip, scale,
                         bias, params_out)
    y0, y1, x0, x1 = (int(v) for v in box)
    name = "frl_augment_mix_images_nhwc" if is_nhwc(dst) else "frl_augment_mix_images"
    _check(getattr(lib(), name)(*args, int(mix_mode), float(lam), y0, y1, x0, x1, _stream()), name)


def mix_targets(src, dst, lam: float, n_classes: int = 0) -> None:
    """The batch's target field mixed with partner B-1-i: int64 labels [B] -> fp32 ``dst`` [B,
    n_classes] (lam at y_i plus 1-lam at y_j, NaN rows for labels outside [0, n_classes)), or a
    floating field [B, ...] -> ``dst`` of its dtype and shape.  See frl_mix_targets in
    include/frl_b200.h."""
    assert src.is_contiguous() and dst.is_contiguous() and src.dim() >= 1
    B = src.shape[0]
    if src.dtype == torch.int64:
        assert src.dim() == 1 and dst.dtype == torch.float32 and tuple(dst.shape) == (B, n_classes)
        inner = 1
    else:
        assert dst.dtype == src.dtype and dst.shape == src.shape
        inner = src[0].numel() if B else 1
    _check(lib().frl_mix_targets(_ptr(src), dtype_code(src.dtype), B, inner, int(n_classes), float(lam), _ptr(dst),
                                 _stream()), "frl_mix_targets")


POLICY_NONE, POLICY_TRIVIAL_AUGMENT, POLICY_RAND_AUGMENT = 0, 1, 2
#: bytes of shared memory K5p stages a sample's uint8 crop in (FRL_AUGMENT_POLICY_SMEM_BYTES)
POLICY_SMEM_BYTES = 224256


def augment_policy_images(src, idx, dst, *, seed: int, epoch: int, mode: int, scale_range=(0.08, 1.0),
                          ratio_range=(3.0 / 4.0, 4.0 / 3.0), pad: int = 0, flip: bool = True,
                          policy: int = POLICY_NONE, num_ops: int = 1, magnitude: int = 0, mags=None,
                          erase_p: float = 0.0, erase_scale=(0.02, 0.33), erase_ratio=(0.3, 3.3),
                          erase_random: bool = False, erase_value=None, scale=None, bias=None, params_out=None,
                          policy_out=None) -> None:
    """K5p: K5a's training crop and flip, then the policy (``POLICY_TRIVIAL_AUGMENT`` /
    ``POLICY_RAND_AUGMENT``, magnitude table ``mags`` device fp32 [14, num_bins]), the affine and
    random erasing (``erase_p`` > 0; ``erase_random`` or ``erase_value`` device fp32 [C]).
    ``policy_out`` optional int32 [B, 3*num_ops + 5] (num_ops 0 without a policy).  Other
    arguments as ``augment_images``.  See frl_augment_policy_images in include/frl_b200.h."""
    B, Cc, H, W = src.shape
    assert src.dtype == torch.uint8 and src.is_contiguous() and (dst.is_contiguous() or is_nhwc(dst))
    assert dst.dim() == 4 and tuple(dst.shape[:2]) == (B, Cc)
    assert idx.dtype == torch.int64 and idx.is_contiguous() and idx.numel() == B
    assert params_out is None or (params_out.dtype == torch.int32 and params_out.is_contiguous()
                                  and tuple(params_out.shape) == (B, 5))
    n_ops = num_ops if policy != POLICY_NONE else 0
    assert policy_out is None or (policy_out.dtype == torch.int32 and policy_out.is_contiguous()
                                  and tuple(policy_out.shape) == (B, 3 * n_ops + 5))
    num_bins = 0
    if mags is not None:
        assert mags.dtype == torch.float32 and mags.is_contiguous() and mags.dim() == 2 and mags.shape[0] == 14
        num_bins = mags.shape[1]
    assert erase_value is None or (erase_value.dtype == torch.float32 and erase_value.numel() == Cc)
    name = "frl_augment_policy_images_nhwc" if is_nhwc(dst) else "frl_augment_policy_images"
    _check(getattr(lib(), name)(
        _ptr(src), B, Cc, H, W, _ptr(idx), int(seed) & (2 ** 64 - 1), int(epoch), int(mode),
        float(scale_range[0]), float(scale_range[1]), float(ratio_range[0]), float(ratio_range[1]), int(pad),
        int(bool(flip)), int(policy), int(num_ops), int(magnitude), int(num_bins), _ptr(mags), float(erase_p),
        float(erase_scale[0]), float(erase_scale[1]), float(erase_ratio[0]), float(erase_ratio[1]),
        int(bool(erase_random)), _ptr(erase_value), _ptr(scale), _ptr(bias), _ptr(dst), dtype_code(dst.dtype),
        dst.shape[2], dst.shape[3], _ptr(params_out), _ptr(policy_out), _stream()), name)


def mix_images(dst, *, mix_mode: int, lam: float, box=(0, 0, 0, 0)) -> None:
    """Mixup (``MIX_MIXUP``) or CutMix (``MIX_CUTMIX``, ``box`` = (y0, y1, x0, x1)) of the finished
    images ``dst`` [B, C, H, W] (contiguous or channels_last, fp32 / bf16) in place, sample p with
    B-1-p.  See frl_mix_images in include/frl_b200.h."""
    assert dst.dim() == 4 and (dst.is_contiguous() or is_nhwc(dst))
    B, Cc, H, W = dst.shape
    y0, y1, x0, x1 = (int(v) for v in box)
    name = "frl_mix_images_nhwc" if is_nhwc(dst) else "frl_mix_images"
    _check(getattr(lib(), name)(_ptr(dst), dtype_code(dst.dtype), B, Cc, H, W, int(mix_mode), float(lam), y0, y1,
                                x0, x1, _stream()), name)


def cast_scale(src, dst, scale: float = 1.0) -> None:
    """dst = src * scale element by element: both contiguous, or both channels_last (cast as the
    [B, H, W, C] arrays they store)."""
    if is_nhwc(src) and is_nhwc(dst):
        src, dst = src.permute(0, 2, 3, 1), dst.permute(0, 2, 3, 1)
    n = src.numel()
    assert dst.numel() == n and src.is_contiguous() and dst.is_contiguous()
    _check(lib().frl_cast_scale(_ptr(src), dtype_code(src.dtype), _ptr(dst),
                                dtype_code(dst.dtype), n, scale, _stream()), "frl_cast_scale")


# ---- K6 -------------------------------------------------------------------------------------

_colsum_scratch = {}


def colsum(x, out, accumulate: bool = False) -> None:
    """out[c] (+)= sum_r x[r, c] for a contiguous 2-D ``x``; ``out`` may be an arena view."""
    rows, cols = x.shape
    key = (x.device.index, cols)
    need = int(lib().frl_colsum_scratch_bytes(rows, cols))
    buf = _colsum_scratch.get(key)
    if buf is None or buf.numel() * 4 < need:
        buf = _colsum_scratch[key] = torch.zeros((need + 3) // 4, dtype=torch.int32, device=x.device)
    _check(lib().frl_colsum(_ptr(x), dtype_code(x.dtype), rows, cols, _ptr(out),
                            dtype_code(out.dtype), int(accumulate), _ptr(buf), _stream()),
           "frl_colsum")


def drelu_colsum(dy, act, dz, out, accumulate: bool = False) -> None:
    """dz = threshold_backward(dy, act, 0) (dy unless act <= 0); out[c] (+)= sum_r dz[r, c] — one
    pass (contiguous 2-D inputs)."""
    rows, cols = dy.shape
    assert act.shape == dy.shape == dz.shape and act.dtype == dy.dtype == dz.dtype
    assert dy.is_contiguous() and act.is_contiguous() and dz.is_contiguous()
    key = (dy.device.index, cols)
    need = int(lib().frl_colsum_scratch_bytes(rows, cols))
    buf = _colsum_scratch.get(key)
    if buf is None or buf.numel() * 4 < need:
        buf = _colsum_scratch[key] = torch.zeros((need + 3) // 4, dtype=torch.int32, device=dy.device)
    _check(lib().frl_drelu_colsum(_ptr(dy), _ptr(act), _ptr(dz), dtype_code(dy.dtype), rows, cols,
                                  _ptr(out), dtype_code(out.dtype), int(accumulate), _ptr(buf), _stream()),
           "frl_drelu_colsum")


# ---- K7 -------------------------------------------------------------------------------------
# mc_g / mc_out / pads are raw addresses (ints): multicast mappings have no torch tensor.

def nvls_sgd(p, buf, mc_g, mc_out, n, link, *, lr, mu, dampening, wd, grad_scale, first_step,
             g_dtype, dyn=None) -> None:
    _check(lib().frl_nvls_sgd(_ptr(p), _ptr(buf), mc_g, mc_out, n, link.rank, link.world,
                              link.pads_dev, link.pad_base, _ptr(link.scratch), link.max_blocks, lr, mu, dampening, wd,
                              grad_scale, _ptr(dyn), int(first_step), g_dtype, link.flags, _stream()),
           "frl_nvls_sgd")


def nvls_adam(p, m, v, vmax, mc_g, mc_out, n, link, *, lr, beta1, beta2, eps, wd, step, grad_scale,
              g_dtype, dyn=None) -> None:
    _check(lib().frl_nvls_adam(_ptr(p), _ptr(m), _ptr(v), _ptr(vmax), mc_g, mc_out, n, link.rank,
                               link.world, link.pads_dev, link.pad_base, _ptr(link.scratch), link.max_blocks, lr, beta1,
                               beta2, eps, wd, step, grad_scale, _ptr(dyn), g_dtype, link.flags, _stream()),
           "frl_nvls_adam")


def nvls_adamw(p, m, v, vmax, mc_g, mc_out, n, link, *, lr, beta1, beta2, eps, wd, step, grad_scale,
               g_dtype, dyn=None) -> None:
    """K7 AdamW: ``nvls_adam``'s arguments, ``wd`` decoupled."""
    _check(lib().frl_nvls_adamw(_ptr(p), _ptr(m), _ptr(v), _ptr(vmax), mc_g, mc_out, n, link.rank,
                                link.world, link.pads_dev, link.pad_base, _ptr(link.scratch), link.max_blocks, lr,
                                beta1, beta2, eps, wd, step, grad_scale, _ptr(dyn), g_dtype, link.flags, _stream()),
           "frl_nvls_adamw")


def nvls_lion(p, m, mc_g, mc_out, n, link, *, lr, beta1, beta2, wd, grad_scale, g_dtype, dyn=None) -> None:
    """K7 Lion: ``nvls_sgd``'s arguments with (beta1, beta2) for (mu, dampening), m = exp_avg."""
    _check(lib().frl_nvls_lion(_ptr(p), _ptr(m), mc_g, mc_out, n, link.rank, link.world, link.pads_dev,
                               link.pad_base, _ptr(link.scratch), link.max_blocks, lr, beta1, beta2, wd, grad_scale,
                               _ptr(dyn), g_dtype, link.flags, _stream()), "frl_nvls_lion")


def nvls_rmsprop(p, sq, buf, mc_g, mc_out, n, link, *, lr, alpha, eps, wd, mu, grad_scale, g_dtype,
                 dyn=None) -> None:
    _check(lib().frl_nvls_rmsprop(_ptr(p), _ptr(sq), _ptr(buf), mc_g, mc_out, n, link.rank,
                                  link.world, link.pads_dev, link.pad_base, _ptr(link.scratch), link.max_blocks, lr,
                                  alpha, eps, wd, mu, grad_scale, _ptr(dyn), g_dtype, link.flags, _stream()),
           "frl_nvls_rmsprop")


NVLS_EXTERNAL_SYNC = 1


def nvls_barrier(link, slot: int) -> None:
    _check(lib().frl_nvls_barrier(link.pads_dev, link.rank, link.world, slot, _stream()),
           "frl_nvls_barrier")


# ---- K9 -------------------------------------------------------------------------------------

def fp8_amax(src, amax_out) -> None:
    """amax_out[0] = max |src| (NaN if src holds one) for a contiguous bf16/fp32 device tensor;
    ``amax_out``: device fp32 scalar, zeroed by the call itself."""
    assert src.is_contiguous() and amax_out.dtype == torch.float32
    _check(lib().frl_fp8_amax(_ptr(src), src.numel(), dtype_code(src.dtype), _ptr(amax_out), _stream()),
           "frl_fp8_amax")


def fp8_quantize(src, amax, fmt: int, dst=None, dst_t=None, inv_scale_out=None) -> None:
    """Codes of the 2-D ``src`` [rows, cols] at the power-of-two scale ``amax`` implies: ``dst``
    [rows, cols] and/or ``dst_t`` [cols, rows] of the ``fmt`` float8 dtype; ``inv_scale_out``
    (device fp32 scalar) receives 1 / scale.  See frl_fp8_quantize in include/frl_b200.h."""
    rows, cols = src.shape
    want = FP8_DTYPE[fmt]
    assert src.is_contiguous() and amax.dtype == torch.float32 and inv_scale_out.dtype == torch.float32
    assert dst is None or (dst.shape == (rows, cols) and dst.dtype == want and dst.is_contiguous())
    assert dst_t is None or (dst_t.shape == (cols, rows) and dst_t.dtype == want and dst_t.is_contiguous())
    _check(lib().frl_fp8_quantize(_ptr(src), rows, cols, dtype_code(src.dtype), _ptr(amax), fmt, _ptr(dst),
                                  _ptr(dst_t), _ptr(inv_scale_out), _stream()), "frl_fp8_quantize")


# ---- K8 -------------------------------------------------------------------------------------

def gather_rows(src_pinned, idx_dev, dst, max_blocks: int = 64) -> None:
    """dst[i] = src_pinned[idx[i]] — ``src_pinned`` is a pinned HOST tensor [rows, ...], ``dst`` a
    device tensor [len(idx), ...]; the kernel reads host memory over PCIe."""
    assert src_pinned.is_pinned() and src_pinned.is_contiguous() and dst.is_contiguous()
    row_bytes = src_pinned[0].numel() * src_pinned.element_size() if src_pinned.shape[0] else 0
    _check(lib().frl_gather_rows(_ptr(src_pinned), src_pinned.shape[0], _ptr(idx_dev), _ptr(dst),
                                 idx_dev.numel(), row_bytes, max_blocks, _stream()),
           "frl_gather_rows")


def _row_bytes(src) -> int:
    return src[0].numel() * src.element_size() if src.shape[0] else 0


def gather_rows_tma(src_pinned, idx_dev, dst, max_blocks: int = 0) -> None:
    """``gather_rows`` through the SMs' bulk-copy engine (rows must be multiples of 16 bytes)."""
    assert src_pinned.is_pinned() and src_pinned.is_contiguous() and dst.is_contiguous()
    _check(lib().frl_gather_rows_tma(_ptr(src_pinned), src_pinned.shape[0], _ptr(idx_dev), _ptr(dst),
                                     idx_dev.numel(), _row_bytes(src_pinned), max_blocks, _stream()),
           "frl_gather_rows_tma")


def gather_lines(corpus_ptr: int, corpus_bytes: int, corpus_alloc_bytes: int, starts_dev, idx_dev, dst,
                 pad: int = 0, max_blocks: int = 0) -> None:
    """dst[r] = line idx[r] of a text corpus, cut or padded with ``pad`` to ``dst.shape[1]`` bytes.
    ``corpus_ptr``: address of the pinned, device-mapped corpus (16-byte aligned, allocation of
    ``corpus_alloc_bytes``); ``starts_dev``: device int64 line-start table [n_lines + 1];
    ``dst``: contiguous device uint8 [len(idx), row_len], any alignment."""
    assert starts_dev.dtype == torch.int64 and starts_dev.is_cuda and starts_dev.is_contiguous()
    assert idx_dev.dtype == torch.int64 and dst.dtype == torch.uint8 and dst.dim() == 2
    assert dst.is_contiguous() and dst.shape[0] == idx_dev.numel()
    _check(lib().frl_gather_lines(corpus_ptr, corpus_bytes, corpus_alloc_bytes, _ptr(starts_dev),
                                  starts_dev.numel() - 1, _ptr(idx_dev), _ptr(dst), dst.shape[0], dst.shape[1],
                                  pad, max_blocks, _stream()), "frl_gather_lines")


def gather_window_rows(batches, idx_dev, dst=None):
    """Rows ``idx_dev`` (device int64, numbered through the concatenation of ``batches``) of a
    list of separate device tensors [rows_b, ...] with one row shape, without concatenating them."""
    first = batches[0]
    assert all(b.is_cuda and b.is_contiguous() and b.shape[1:] == first.shape[1:] and b.dtype == first.dtype
               for b in batches) and idx_dev.dtype == torch.int64 and idx_dev.is_cuda
    if dst is None:
        dst = torch.zeros((idx_dev.numel(),) + tuple(first.shape[1:]), dtype=first.dtype, device=first.device)
    n = len(batches)
    ptrs = (C.c_void_p * n)(*[b.data_ptr() for b in batches])
    rows = (C.c_int64 * n)(*[b.shape[0] for b in batches])
    row_bytes = first[0].numel() * first.element_size() if first.shape[0] else \
        (int(torch.tensor(first.shape[1:]).prod()) * first.element_size())
    _check(lib().frl_gather_window_rows(ptrs, rows, n, _ptr(idx_dev), _ptr(dst), idx_dev.numel(), row_bytes,
                                        _stream()), "frl_gather_window_rows")
    return dst


class HostGatherPool:
    """Persistent native worker threads assembling minibatch rows into pinned staging buffers."""

    def __init__(self, n_threads: int) -> None:
        self._h = lib().frl_gather_pool_create(int(n_threads))
        if not self._h:
            raise NativeLibraryError("frl_gather_pool_create failed: "
                                     + lib().frl_last_error().decode("utf-8", "replace"))
        self.n_threads = int(lib().frl_gather_pool_threads(self._h))

    def submit(self, src, idx_host, dst_host) -> int:
        """Queue dst_host[i] = src[idx_host[i]]; returns a ticket for ``wait``."""
        assert src.is_contiguous() and dst_host.is_contiguous()
        assert not src.is_cuda and not dst_host.is_cuda and not idx_host.is_cuda
        assert idx_host.dtype == torch.int64 and idx_host.is_contiguous()
        assert dst_host.shape[0] >= idx_host.numel()
        t = int(lib().frl_gather_pool_submit(self._h, _ptr(src), src.shape[0], _ptr(idx_host),
                                             _ptr(dst_host), idx_host.numel(), _row_bytes(src)))
        if t < 1:
            _check(t if t != 0 else -1, "frl_gather_pool_submit")
        return t

    def submit_f32_to_bf16(self, src, idx_host, dst_host) -> int:
        """Queue dst_host[i] = bfloat16(src[idx_host[i]]) (round to nearest even) for fp32 ``src``."""
        assert src.dtype == torch.float32 and dst_host.dtype == torch.bfloat16
        assert src.is_contiguous() and dst_host.is_contiguous()
        assert not src.is_cuda and not dst_host.is_cuda and not idx_host.is_cuda
        assert idx_host.dtype == torch.int64 and idx_host.is_contiguous()
        assert dst_host.shape[0] >= idx_host.numel() and dst_host.shape[1:] == src.shape[1:]
        row_elems = src[0].numel() if src.shape[0] else 0
        t = int(lib().frl_gather_pool_submit_f32_to_bf16(self._h, _ptr(src), src.shape[0], _ptr(idx_host),
                                                         _ptr(dst_host), idx_host.numel(), row_elems))
        if t < 1:
            _check(t if t != 0 else -1, "frl_gather_pool_submit_f32_to_bf16")
        return t

    def wait(self, ticket: int) -> None:
        _check(lib().frl_gather_pool_wait(self._h, ticket), "frl_gather_pool_wait")

    def close(self) -> None:
        if self._h:
            lib().frl_gather_pool_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:                 # noqa: BLE001  (interpreter shutdown)
            pass
