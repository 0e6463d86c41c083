"""ctypes loader for libb200dsp.so (the C-ABI declared in include/b200dsp.h).

The library is built in-tree by `__graft_entry__.build()` / `cyberether_b200/build.py`. There is
no fallback: if the shared object is missing, importing the product path raises.
"""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200dsp.so")

c_u64 = ctypes.c_uint64
c_vp = ctypes.c_void_p
c_int = ctypes.c_int
c_f32 = ctypes.c_float
c_f64 = ctypes.c_double
P = ctypes.POINTER

# name -> (restype, argtypes); mirrors include/b200dsp.h one to one.
SIGNATURES = {
    "b200_version": (ctypes.c_char_p, []),
    "b200_last_error": (ctypes.c_char_p, []),
    "b200_device_count": (c_int, [P(c_int)]),
    "b200_ctx_create": (c_int, [c_int, P(c_vp)]),
    "b200_ctx_destroy": (c_int, [c_vp]),
    "b200_ctx_device": (c_int, [c_vp, P(c_int)]),
    "b200_ctx_sm_count": (c_int, [c_vp, P(c_int)]),
    "b200_ctx_info": (c_int, [c_vp, c_vp]),
    "b200_malloc": (c_int, [c_vp, c_u64, P(c_vp)]),
    "b200_free": (c_int, [c_vp, c_vp]),
    "b200_host_alloc": (c_int, [c_vp, c_u64, P(c_vp)]),
    "b200_host_free": (c_int, [c_vp, c_vp]),
    "b200_memcpy": (c_int, [c_vp, c_vp, c_vp, c_u64, c_int, c_vp]),
    "b200_memset": (c_int, [c_vp, c_vp, c_int, c_u64, c_vp]),
    "b200_stream_create": (c_int, [c_vp, P(c_vp)]),
    "b200_stream_destroy": (c_int, [c_vp, c_vp]),
    "b200_stream_synchronize": (c_int, [c_vp, c_vp]),
    "b200_malloc_managed": (c_int, [c_vp, c_u64, P(c_vp)]),
    "b200_host_register": (c_int, [c_vp, c_vp, c_u64, P(c_int)]),
    "b200_host_unregister": (c_int, [c_vp, c_vp]),
    "b200_event_create": (c_int, [c_vp, P(c_vp)]),
    "b200_event_record": (c_int, [c_vp, c_vp, c_vp]),
    "b200_event_elapsed_ms": (c_int, [c_vp, c_vp, c_vp, P(c_f32)]),
    "b200_event_destroy": (c_int, [c_vp, c_vp]),
    "b200_check_async_error": (c_int, [c_vp]),
    "b200_window_blackman_cf32": (c_int, [c_vp, c_vp, c_u64, c_vp]),
    "b200_invert_cf32": (c_int, [c_vp, c_vp, c_vp, c_u64, c_u64, c_u64, c_vp]),
    "b200_multiply_cf32": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, P(c_u64), P(c_u64), P(c_u64), c_vp]),
    "b200_multiply_f32": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, P(c_u64), P(c_u64), P(c_u64), c_vp]),
    "b200_multiply_constant_cf32": (c_int, [c_vp, c_vp, c_vp, c_u64, c_f32, c_vp]),
    "b200_multiply_constant_f32": (c_int, [c_vp, c_vp, c_vp, c_u64, c_f32, c_vp]),
    "b200_fft_plan_c2c": (c_int, [c_vp, c_u64, c_u64, P(c_vp)]),
    "b200_fft_exec": (c_int, [c_vp, c_vp, c_vp, c_int, c_vp]),
    "b200_fft_plan_destroy": (c_int, [c_vp]),
    "b200_fft_exec_real": (c_int, [c_vp, c_vp, c_vp, c_int, c_vp]),
    "b200_fft_real_helper": (c_int, [c_vp, c_int, c_vp, c_vp, c_u64, c_u64, c_vp]),
    "b200_amplitude_cf32": (c_int, [c_vp, c_vp, c_vp, c_u64, c_f32, c_vp]),
    "b200_amplitude_f32": (c_int, [c_vp, c_vp, c_vp, c_u64, c_f32, c_vp]),
    "b200_range_f32": (c_int, [c_vp, c_vp, c_vp, c_u64, c_f32, c_f32, c_vp]),
    "b200_amplitude_scaling_coeff": (c_int, [c_u64, P(c_f32)]),
    "b200_range_coefficients": (c_int, [c_f32, c_f32, P(c_f32), P(c_f32)]),
    "b200_cast_f32_cf32": (c_int, [c_vp, c_vp, c_vp, c_u64, c_vp]),
    "b200_cast_int": (c_int, [c_vp, c_vp, c_int, c_vp, c_u64, c_vp]),
    "b200_agc_scratch_bytes": (c_int, [c_u64, c_u64, c_u64, c_vp]),
    "b200_agc": (c_int, [c_vp, c_vp, c_vp, c_int, c_u64, c_u64, c_u64, c_f64, c_f64, c_f64, c_f64, c_f64, c_vp, c_vp]),
    "b200_copy_strided": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, P(c_u64), P(c_u64), P(c_u64), c_vp]),
    "b200_chain_plan_create": (c_int, [c_vp, c_u64, c_u64, c_vp, P(c_vp)]),
    "b200_chain_exec": (c_int, [c_vp, c_vp, c_vp, c_u64, c_f32, c_int, c_f32, c_f32, c_vp]),
    "b200_chain_exec_typed": (c_int, [c_vp, c_vp, c_int, c_vp, c_u64, c_f32, c_int, c_f32, c_f32, c_vp]),
    "b200_chain_exec_agc": (c_int, [c_vp, c_vp, c_int, c_vp, c_u64, c_f32, c_int, c_f32, c_f32, c_f64, c_f64, c_f64, c_f64,
                                    c_vp]),
    "b200_chain_exec_colsum": (c_int, [c_vp, c_vp, c_int, c_vp, c_u64, c_f32, c_int, c_f32, c_f32, c_vp, c_vp]),
    "b200_lineplot_scratch_bytes": (c_int, [c_u64, c_u64, c_u64, P(c_u64)]),
    "b200_lineplot_init": (c_int, [c_vp, c_vp, c_vp, c_u64, c_vp]),
    "b200_lineplot_update": (c_int, [c_vp, c_vp, c_u64, c_u64, c_u64, c_u64, c_u64, c_f32, c_u64, c_vp, c_vp, c_vp, c_vp]),
    "b200_lineplot_update_from_colsum": (c_int, [c_vp, c_vp, c_u64, c_u64, c_f32, c_u64, c_vp, c_vp, c_vp]),
    "b200_waterfall_update": (c_int, [c_vp, c_vp, c_u64, c_u64, c_u64, c_u64, c_vp, c_u64, c_u64, c_vp]),
    "b200_waterfall_advance": (c_int, [P(c_u64), c_u64, c_u64]),
    "b200_chain_exec_host": (c_int, [c_vp, c_vp, c_vp, c_u64, c_f32, c_int, c_f32, c_f32, c_u64]),
    "b200_chain_exec_host_typed": (c_int, [c_vp, c_vp, c_int, c_vp, c_u64, c_f32, c_int, c_f32, c_f32, c_u64]),
    "b200_chain_plan_destroy": (c_int, [c_vp]),
    "b200_chain_plan_variant": (ctypes.c_char_p, [c_vp]),
    "b200_filter_taps_host": (c_int, [ctypes.c_double, ctypes.c_double, P(ctypes.c_double), c_u64, c_u64, c_vp]),
    "b200_fir_plan_create": (c_int, [c_vp, c_vp, c_u64, c_u64, c_u64, P(c_vp)]),
    "b200_fir_plan_variant": (ctypes.c_char_p, [c_vp]),
    "b200_fir_plan_set_translation": (c_int, [c_vp, c_u64, P(ctypes.c_int64)]),
    "b200_fir_exec": (c_int, [c_vp, c_vp, c_vp, c_u64, c_u64, c_vp]),
    "b200_fir_reset": (c_int, [c_vp, c_vp]),
    "b200_fir_set_history": (c_int, [c_vp, c_vp, c_u64, c_u64, c_vp]),
    "b200_fir_plan_destroy": (c_int, [c_vp]),
    "b200_fold": (c_int, [c_vp, c_vp, c_vp, c_int, c_u64, c_u64, c_u64, c_u64, c_u64, c_vp, c_u64, c_u64, c_vp]),
    "b200_overlap_add": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_u64, c_u64, c_u64, c_u64, c_u64, c_u64, c_vp]),
    "b200_phase_correction": (c_int, [c_vp, c_vp, c_vp, c_u64, c_u64, c_u64, c_u64, c_u64, P(c_f64), P(c_f64), c_vp]),
    "b200_fm_plan_create": (c_int, [c_vp, c_u64, c_f32, c_int, c_int, P(c_vp)]),
    "b200_fm_exec": (c_int, [c_vp, c_vp, c_vp, c_u64, c_u64, c_vp]),
    "b200_fm_reset": (c_int, [c_vp, c_vp]),
    "b200_fm_plan_destroy": (c_int, [c_vp]),
    "b200_fm_nco_phases_host": (c_int, [c_f32, c_u64, c_u64, c_vp, P(c_u64), P(c_u64)]),
    "b200_fm_nco_phases": (c_int, [c_vp, c_u64, c_u64, c_vp, c_vp]),
}

_lib = None


class B200Error(RuntimeError):
    """A libb200dsp call returned a non-SUCCESS Result code."""

    def __init__(self, code: int, message: str):
        super().__init__(f"libb200dsp Result={code}: {message}")
        self.code = code


def load():
    """Load the shared library and attach signatures. Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback for the product path)")
        lib = ctypes.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
    return _lib


def check(rc: int):
    if rc != 0:
        raise B200Error(rc, load().b200_last_error().decode(errors="replace"))
