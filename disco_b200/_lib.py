"""ctypes binding of libdisco_b200.so (the C ABI declared in include/disco_b200.h).

The library is built in-tree by ``python -m disco_b200.build`` (nvcc, sm_90a).  There is no
fallback: if the shared object is missing this module raises, and every compute call needs a
CUDA device.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# DISCO_B200_LIB loads another build of the same ABI instead (an instrumented variant, or an older build to compare
# against); unset, the library built in-tree is used.
LIB_PATH = os.environ.get("DISCO_B200_LIB") or os.path.join(_HERE, "libdisco_b200.so")

c_int, c_void_p, c_size_t, c_float, c_double = (ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                                                ctypes.c_float, ctypes.c_double)
c_int_p = ctypes.POINTER(ctypes.c_int)

# name -> (restype, argtypes); mirrors include/disco_b200.h one to one
SIGNATURES = {
    "disco_abi_version": (c_int, []),
    "disco_last_error": (ctypes.c_char_p, []),
    "disco_n_frames": (c_int, [c_int, c_int]),
    "disco_init": (c_int, [c_int]),
    "disco_set_reserved_sms": (c_int, [c_int]),
    "disco_stft": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "disco_stft_scm_workspace": (c_size_t, [c_int, c_int, c_int, c_int]),
    "disco_stft_scm": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                               c_void_p, c_size_t, c_void_p]),
    "disco_stft_scm_supported": (c_int, [c_int, c_int, c_int]),
    "disco_stft_scm2_workspace": (c_size_t, [c_int, c_int, c_int, c_int]),
    "disco_stft_scm2": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                c_size_t, c_void_p]),
    "disco_stft_filter_dual": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                       c_int, c_int, c_int, c_void_p]),
    "disco_scm_from_workspace": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                         c_void_p]),
    "disco_mwf_solve_workspace2": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                           c_double, c_void_p]),
    "disco_filter_dual": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                  c_int, c_int, c_int, c_void_p]),
    "disco_tf_mask": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_int, c_float, c_void_p]),
    "disco_masked_scm": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                 c_int, c_int_p, c_int, c_int, c_void_p]),
    "disco_filter_sum_scm": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                     c_int, c_int, c_int, c_int, c_void_p]),
    "disco_tango_mid_supported": (c_int, [c_int, c_int]),
    "disco_tango_mid": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int,
                                c_int, c_int, c_int, c_void_p]),
    "disco_mwf_solve_workspace": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                          c_int, c_int, c_double, c_void_p]),
    "disco_mwf_solve": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_double,
                                c_void_p]),
    "disco_filter_sum": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                 c_int, c_int, c_int, c_int_p, c_int, c_int, c_void_p]),
    "disco_istft": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "disco_stft_lengths": (c_int, [c_void_p, c_void_p, c_int_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "disco_istft_lengths": (c_int, [c_void_p, c_void_p, c_int_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "disco_scm_recursive": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_double,
                                    c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int_p, c_int, c_void_p]),
    "disco_filter_sum_blocks": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                        c_int, c_int, c_int, c_int, c_int, c_int_p, c_int, c_void_p]),
    "disco_scm_recursive_lengths": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                            ctypes.c_double, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int_p,
                                            c_int, c_void_p, c_int_p, c_void_p]),
    "disco_filter_sum_blocks_lengths": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                                c_int, c_int, c_int, c_int, c_int, c_int, c_int_p, c_int, c_void_p,
                                                c_int_p, c_void_p]),
    "disco_stream_stft": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                  c_int, c_int, c_int, c_int, c_void_p]),
    "disco_stream_istft": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                   c_void_p]),
    "disco_stream_stft_slots": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int_p, c_int, c_int, c_int,
                                        c_int, c_int, c_int, c_void_p]),
    "disco_stream_istft_slots": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int_p, c_int, c_int, c_int, c_int,
                                         c_int, c_void_p]),
    "disco_band_stats": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, ctypes.c_longlong, c_int, c_int,
                                 c_void_p]),
    "disco_bss_eval_workspace": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "disco_bss_eval": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_size_t,
                               c_void_p]),
    "disco_resample_poly": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "disco_resample_poly_lengths": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                            c_int_p, c_void_p]),
    "disco_stoi_lengths": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                   c_int, c_void_p, c_int_p, c_void_p, c_size_t, c_void_p]),
    "disco_stoi_workspace": (c_size_t, [c_int, c_int, c_int]),
    "disco_stoi": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                           c_void_p, c_size_t, c_void_p]),
    "disco_transpose_c64":(c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "disco_transpose_f32": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "disco_apply_mask": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_void_p]),
    "disco_apply_mask_channels": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_size_t, c_int, c_void_p]),
}

_lib = None


def load():
    """Load the shared library (once) and attach the prototypes.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "disco_b200: %s not found -- build the CUDA library first (python -m disco_b200.build). "
            "There is no CPU or PyTorch fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)     # AttributeError if the ABI symbol is missing
        fn.restype = res
        fn.argtypes = args
    if lib.disco_abi_version() != 2:
        raise ImportError("disco_b200: ABI version mismatch")
    _lib = lib
    return lib


class DiscoError(RuntimeError):
    pass


def check(rc):
    if rc != 0:
        msg = load().disco_last_error()
        raise DiscoError("libdisco_b200 error %d: %s" % (rc, msg.decode() if msg else "?"))
