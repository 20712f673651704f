"""ctypes binding of ``libffc_b200.so`` (C ABI: include/ffc_b200.h).

The library is the product; there is no fallback.  ``get_lib()`` raises if the shared object
is missing or does not export every symbol the header declares, and every wrapper raises on a
non-zero return code with the library's own message.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libffc_b200.so")

# enums (mirror include/ffc_b200.h)
OK, EINVAL, EARCH, ECUDA, ENOMEM = 0, -1, -2, -3, -4
F32, BF16X2 = 0, 1
ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_TANH = 0, 1, 2, 3
BORDER_ZERO, BORDER_REFLECT = 0, 1
MATH_FP32, MATH_BF16X3 = 0, 1
MAX_KSEG = 64
PLAN_FLAT, PLAN_SPATIAL, PLAN_ROWS, PLAN_HALO = 0, 1, 2, 3
VERSION = 117


class Tensor(C.Structure):
    """``ffcb_tensor``"""
    _fields_ = [("ptr", C.c_void_p), ("sb", C.c_int64), ("sy", C.c_int64), ("sx", C.c_int64),
                ("lo_off", C.c_int64), ("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("C", C.c_int32),
                ("fmt", C.c_int32), ("pad", C.c_int32), ("reflect_border", C.c_int32), ("window", C.c_int32),
                ("cg", C.c_int32), ("tile", C.c_int32), ("sg", C.c_int64)]


class KSeg(C.Structure):
    """``ffcb_kseg``"""
    _fields_ = [("src", C.c_int32), ("dy", C.c_int32), ("dx", C.c_int32), ("c0", C.c_int32), ("nch", C.c_int32)]


class ConvDesc(C.Structure):
    """``ffcb_conv_desc``"""
    _fields_ = [("inp", Tensor * 2), ("out", Tensor), ("addend", Tensor), ("weight", C.c_void_p),
                ("shift", C.c_void_p), ("n_out", C.c_int32), ("stride", C.c_int32), ("border", C.c_int32),
                ("act", C.c_int32), ("nseg", C.c_int32), ("math", C.c_int32), ("addend_post", C.c_int32),
                ("_reserved", C.c_int32), ("seg", KSeg * MAX_KSEG)]


class ConvPlanInfo(C.Structure):
    """``ffcb_conv_plan_info``"""
    _fields_ = [("kind", C.c_int32), ("il", C.c_int32), ("po", C.c_int32), ("ring", C.c_int32), ("bn", C.c_int32),
                ("tw", C.c_int32), ("th", C.c_int32), ("stages", C.c_int32), ("m_tiles", C.c_int64),
                ("n_tiles", C.c_int32), ("_reserved", C.c_int32)]


_PT = C.POINTER(Tensor)
# name -> (restype, argtypes): every symbol include/ffc_b200.h declares
SIGNATURES = {
    "ffcb_version": (C.c_int, []),
    "ffcb_last_error": (C.c_char_p, []),
    "ffcb_check_device": (C.c_int, [C.c_int]),
    "ffcb_shutdown": (None, []),
    "ffcb_conv": (C.c_int, [C.POINTER(ConvDesc), C.c_void_p]),
    "ffcb_conv_plan": (C.c_int, [C.POINTER(ConvDesc), C.POINTER(ConvPlanInfo)]),
    "ffcb_stem_conv7": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                  _PT, C.c_void_p]),
    "ffcb_stem_pack": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, _PT, C.c_void_p]),
    "ffcb_head_gather7": (C.c_int, [_PT, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ffcb_stem_pack_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, _PT, C.c_void_p]),
    "ffcb_head_gather7_blend_u8": (C.c_int, [_PT, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                             C.c_void_p, C.c_void_p]),
    "ffcb_head_conv7": (C.c_int, [_PT, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ffcb_fft2_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "ffcb_rfft2": (C.c_int, [_PT, _PT, C.c_void_p, C.c_size_t, C.c_void_p]),
    "ffcb_irfft2": (C.c_int, [_PT, _PT, _PT, C.c_void_p, C.c_size_t, C.c_void_p]),
    "ffcb_nchw_to_nhwc": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, _PT, C.c_void_p]),
    "ffcb_nhwc_to_nchw": (C.c_int, [_PT, C.c_void_p, C.c_void_p]),
    "ffcb_fill_reflect_border": (C.c_int, [_PT, C.c_void_p]),
    "ffcb_relu_bwd": (C.c_int, [_PT, _PT, _PT, C.c_void_p]),
    "ffcb_relu_mask_pack": (C.c_int, [_PT, C.c_void_p, C.c_void_p]),
    "ffcb_relu_bwd_bits": (C.c_int, [_PT, C.c_void_p, _PT, C.c_void_p]),
    "ffcb_fold_reflect_border": (C.c_int, [_PT, _PT, C.c_int, _PT, C.c_int, _PT, C.c_void_p]),
    "ffcb_add": (C.c_int, [_PT, _PT, _PT, C.c_void_p]),
    "ffcb_head_bwd7": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                 _PT, _PT, C.c_void_p]),
    "ffcb_head_bwd7_bits": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                      C.c_int, C.c_void_p, C.c_int, _PT, C.c_void_p]),
    "ffcb_relu_mask_pack_rows": (C.c_int, [_PT, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "ffcb_relu_bwd_bits_rows": (C.c_int, [_PT, C.c_void_p, C.c_int, C.c_int, _PT, C.c_void_p]),
    "ffcb_head_gather7_rows": (C.c_int, [_PT, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                         C.c_void_p]),
    "ffcb_stem_bwd7": (C.c_int, [_PT, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "ffcb_refine_l1_grad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_int] * 6 + [C.c_void_p] * 7
                            + [C.c_void_p]),
    "ffcb_launch_count": (C.c_longlong, []),
    "ffcb_reset_launch_count": (None, []),
}

_lib = None


class FFCBError(RuntimeError):
    pass


def get_lib():
    """Load the shared library (once).  Raises if it is missing or incomplete — never falls back."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise FFCBError(f"{LIB_PATH} not found: build it with `python -m lama_b200.build` "
                        f"(or __graft_entry__.build()); lama_b200 has no CPU/PyTorch fallback")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise FFCBError(f"{LIB_PATH} does not export {name}") from e
        fn.restype = res
        fn.argtypes = args
    if lib.ffcb_version() != VERSION:
        raise FFCBError(f"libffc_b200.so version {lib.ffcb_version()} != binding {VERSION}; rebuild")
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != OK:
        msg = get_lib().ffcb_last_error().decode("utf-8", "replace")
        exc = ValueError if rc == EINVAL else FFCBError
        raise exc(f"libffc_b200 {what} failed ({rc}): {msg}")
