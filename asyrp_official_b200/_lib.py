"""ctypes binding of libasyrp_b200.so (the C-ABI in include/asyrp_b200.h).

The library is the only compute path of this package: if it is missing or fails to load, importing the
engine raises — there is no PyTorch / CPU fallback.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# ASYRP_LIB_SUFFIX selects a diagnostic build made with the same suffix (asyrp_official_b200/build.py); default: the product
LIB_PATH = os.path.join(_HERE, f"libasyrp_b200{os.environ.get('ASYRP_LIB_SUFFIX', '')}.so")

c_void_p, c_int, c_float = C.c_void_p, C.c_int, C.c_float


class AsyrpConvSeg(C.Structure):
    _fields_ = [("src", c_void_p), ("C", c_int), ("mode", c_int), ("affine", c_void_p), ("affine_stride", c_int),
                ("act", c_int), ("ld", c_int),
                ("gn_sums_a", c_void_p), ("gn_Ca", c_int), ("gn_sums_b", c_void_p), ("gn_Cb", c_int),
                ("gn_gamma", c_void_p), ("gn_beta", c_void_p), ("gn_scale_shift", c_void_p), ("gn_ss_stride", c_int),
                ("gn_eps", c_float), ("gn_hw", c_int), ("gn_off", c_int)]


class AsyrpConvDesc(C.Structure):
    _fields_ = [
        ("N", c_int), ("H", c_int), ("W", c_int), ("Cout", c_int),
        ("nseg", c_int),
        ("seg", AsyrpConvSeg * 3),
        ("weight", c_void_p),
        ("weight_batched", c_int),
        ("weight_ld", c_int),
        ("weight_batch_stride", C.c_longlong),
        ("a_heads", c_int), ("b_heads", c_int), ("out_heads", c_int), ("out_f32", c_int),
        ("ebias", c_void_p),
        ("ebias_stride", c_int),
        ("residual", c_void_p),
        ("res_scale", c_float), ("acc_scale", c_float),
        ("out", c_void_p),
        ("stats", c_void_p),
        ("out_planar", c_void_p),
        ("planar_c", c_int),
        ("up2", c_int),
        ("scales", c_void_p),
        ("res_mode", c_int),
        ("sums_out", c_void_p),
    ]


# name -> (restype, argtypes); every symbol include/asyrp_b200.h declares
SIGNATURES = {
    "asyrp_last_error": (C.c_char_p, []),
    "asyrp_set_pdl": (c_int, [c_int]),
    "asyrp_get_pdl": (c_int, []),
    "asyrp_conv_stats_tiles": (c_int, [c_int, c_int, c_int, c_int]),
    "asyrp_conv_stats_tiles_up2": (c_int, [c_int, c_int, c_int]),
    "asyrp_conv_tile_config": (c_int, [c_int, c_int, c_int, c_int]),
    "asyrp_set_silu_tanh": (c_int, [c_int]),
    "asyrp_conv_create": (c_int, [C.POINTER(AsyrpConvDesc), C.POINTER(c_void_p)]),
    "asyrp_conv_launch": (c_int, [c_void_p, c_void_p]),
    "asyrp_conv_set_scales": (c_int, [c_void_p, c_float, c_float]),
    "asyrp_conv_destroy": (None, [c_void_p]),
    "asyrp_gn_finalize": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_float,
                                  c_int, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "asyrp_apply": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int,
                            c_int, c_void_p]),
    "asyrp_pack_input": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "asyrp_timestep_embedding": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "asyrp_linear": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                             c_int, c_void_p]),
    "asyrp_ddim_update": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                  c_int, c_float, c_float, c_float, c_float, c_void_p]),
    "asyrp_ddpm_update": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_float,
                                  c_float, c_int, c_float, c_void_p]),
    "asyrp_axpby": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_float, C.c_longlong, c_void_p]),
    "asyrp_unpack_nchw": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "asyrp_slerp_h": (c_int, [c_void_p, c_void_p, C.c_longlong, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                              c_float, c_int, c_void_p]),
    "asyrp_transpose_tc": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "asyrp_softmax_rows": (c_int, [c_void_p, c_void_p, C.c_longlong, c_int, c_float, c_void_p]),
    "asyrp_attention": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p]),
}

_lib = None


class AsyrpError(RuntimeError):
    pass


def load():
    """Load the shared library (once) and attach prototypes.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise AsyrpError(
            f"{LIB_PATH} not found: build it with `python -m asyrp_official_b200.build` "
            "(this package has no fallback path)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().asyrp_last_error().decode(errors="replace")
        raise AsyrpError(f"{what} failed (rc={rc}): {msg}")
