"""ctypes binding of libpika_b200.so (the C ABI declared in include/pika_b200.h).

There is no CPU fallback: importing this module without the built library raises, and every
entry point raises ``PikaError`` on a non-zero return code.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpika_b200.so")

PK_F32, PK_BF16 = 0, 1
SEL_ZERO, SEL_ZB0, SEL_ZB1, SEL_KZ = 0, 1, 2, 3
ACT_NONE, ACT_RELU = 0, 1
AUX_NONE, AUX_ADD, AUX_MASK_NZ = 0, 1, 2
MAX_PAIRS = 9


class PikaError(RuntimeError):
    pass


class View4(ctypes.Structure):
    _fields_ = [("ptr", ctypes.c_void_p), ("dim", ctypes.c_int64 * 4), ("stride", ctypes.c_int64 * 3)]


class GemmDesc(ctypes.Structure):
    _fields_ = [
        ("n_pairs", ctypes.c_int),
        ("a", View4 * MAX_PAIRS),
        ("b", View4 * MAX_PAIRS),
        ("a_row_off", ctypes.c_int * MAX_PAIRS),
        ("b_row_off", ctypes.c_int * MAX_PAIRS),
        ("a_mn_major", ctypes.c_int), ("b_mn_major", ctypes.c_int),
        ("a_sel2", ctypes.c_int), ("a_sel3", ctypes.c_int), ("b_sel2", ctypes.c_int), ("b_sel3", ctypes.c_int),
        ("kz_count", ctypes.c_int),
        ("c", View4),
        ("c_dtype", ctypes.c_int),
        ("c_accumulate", ctypes.c_int),
        ("alpha", ctypes.c_float),
        ("bias", ctypes.c_void_p),
        ("act", ctypes.c_int),
        ("drop_p", ctypes.c_float),
        ("drop_seed", ctypes.c_uint32),
        ("aux_mode", ctypes.c_int),
        ("aux", ctypes.c_void_p),
        ("aux_dtype", ctypes.c_int),
        ("aux_stride", ctypes.c_int64 * 3),
        ("aux_scale", ctypes.c_float),
        ("block_n", ctypes.c_int),
        ("k_splits", ctypes.c_int),
        ("row_lse", ctypes.c_void_p),
    ]


if not os.path.exists(LIB_PATH):
    raise ImportError(
        "pika_b200: %s is missing -- build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(there is no CPU fallback)" % LIB_PATH)

lib = ctypes.CDLL(LIB_PATH)
lib.pk_last_error.restype = ctypes.c_char_p
lib.pk_launch_count.restype = ctypes.c_longlong
lib.pk_rnnt_loss_workspace_bytes.restype = ctypes.c_longlong

_vp, _i, _ll, _f, _u32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_uint32


def _sig(name, argtypes, restype=ctypes.c_int):
    fn = getattr(lib, name)
    fn.argtypes = argtypes
    fn.restype = restype
    return fn


_sig("pk_gemm_bf16", [ctypes.POINTER(GemmDesc), _vp])
_sig("pk_gemm_row_lse_parts", [_ll, _ll, _i])
_sig("pk_rnnt_loss_workspace_bytes", [_i, _i, _i], ctypes.c_longlong)
_sig("pk_attention_keep_bits_bytes", [_i, _i, _i], ctypes.c_longlong)
_sig("pk_rnnt_loss_colsum_workspace_bytes", [_i, _i, _i, _i], ctypes.c_longlong)
_sig("pk_rnnt_loss_fwd_bwd", [_vp, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _ll, _vp])
_sig("pk_rnnt_loss_fwd_bwd_lse", [_vp, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _ll, _vp, _i, _vp])
_sig("pk_frontend_noise_rir_workspace_bytes", [_i, _i, _i, _i, _i, _i], ctypes.c_longlong)
_sig("pk_conv_same_f64_workspace_bytes", [_i, _i, _i], ctypes.c_longlong)
_sig("pk_conv_same_f64", [_vp, _ll, _vp, _vp, _ll, _vp, _i, _i, _i, _vp, _ll, _vp, _ll, _vp])
_d = ctypes.c_double
_sig("pk_adam_clip", [_vp, _vp, _vp, _vp, _vp, _ll, _d, _d, _d, _d, _d, _d, _f, _vp, _vp, _vp])
_sig("pk_bmuf_adam_update", [_vp, _vp, _vp, _vp, _vp, _vp, _ll, _i, _d, _d, _d, _d, _d, _d, _vp])


def check(rc, what=""):
    if rc != 0:
        raise PikaError("%s failed (rc=%d): %s" % (what, rc, lib.pk_last_error().decode()))


def launch_count():
    return int(lib.pk_launch_count())
