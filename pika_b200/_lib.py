"""ctypes binding of libpika_b200.so (the C ABI declared in include/pika_b200.h).

The header is the only statement of the ABI's types: at import every ``pk_*`` prototype it declares gets its ``argtypes`` and
``restype`` from it, and the integer constants below are its ``#define``s.  Callers pass plain Python values: ints, floats and
bools for numbers, an address (``t.data_ptr()``) or ``None`` for a pointer, an instance of the mirror class below for a struct
pointer (ctypes passes its address).  A call with the wrong number of arguments or a float for an integer parameter raises
before anything runs.

There is no CPU fallback: importing this module without the built library raises, and every
entry point raises ``PikaError`` on a non-zero return code.
"""
import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpika_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "pika_b200.h")


class PikaError(RuntimeError):
    pass


def _read_header(path):
    """-> ({name: value} of the integer #defines, [(return type, name, [parameter declarations])] of the prototypes)"""
    with open(path) as f:
        src = re.sub(r"/\*.*?\*/", " ", f.read(), flags=re.S)
    defines = {k: int(v) for k, v in re.findall(r"^\s*#define\s+(\w+)\s+(-?\d+)\s*$", src, flags=re.M)}
    src = re.sub(r"^\s*#.*$", " ", src, flags=re.M)
    src = re.sub(r"typedef\s+struct\s*\{.*?\}\s*\w+\s*;", " ", src, flags=re.S)       # mirrored by the classes below
    src = re.sub(r'extern\s+"C"\s*\{|\}', " ", src)
    protos = []
    for decl in filter(None, (" ".join(d.split()) for d in src.split(";"))):
        m = re.fullmatch(r"(.+?)\s*\b(pk_\w+)\s*\((.*)\)", decl)
        if m is None:
            raise ImportError("pika_b200: %s: cannot read the declaration %r" % (path, decl))
        params = m.group(3).strip()
        protos.append((m.group(1), m.group(2), [] if params in ("", "void") else [p.strip() for p in params.split(",")]))
    return defines, protos


_DEFINES, _PROTOTYPES = _read_header(HEADER_PATH)
PK_F32, PK_BF16 = _DEFINES["PK_F32"], _DEFINES["PK_BF16"]
SEL_ZERO, SEL_ZB0, SEL_ZB1, SEL_KZ = (_DEFINES["PK_SEL_" + s] for s in ("ZERO", "ZB0", "ZB1", "KZ"))
ACT_NONE, ACT_RELU = _DEFINES["PK_ACT_NONE"], _DEFINES["PK_ACT_RELU"]
AUX_NONE, AUX_ADD, AUX_MASK_NZ = _DEFINES["PK_AUX_NONE"], _DEFINES["PK_AUX_ADD"], _DEFINES["PK_AUX_MASK_NZ"]
MAX_PAIRS = _DEFINES["PK_GEMM_MAX_PAIRS"]


class View4(ctypes.Structure):
    """pk_view4"""
    _fields_ = [("ptr", ctypes.c_void_p), ("dim", ctypes.c_int64 * 4), ("stride", ctypes.c_int64 * 3)]


class GemmDesc(ctypes.Structure):
    """pk_gemm_desc"""
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
        ("a_rows_dev", ctypes.c_void_p),
    ]


class LmFst(ctypes.Structure):
    """pk_lm_fst: the flattened arc table of an FST language model for shallow fusion in the beam step"""
    _fields_ = [("arc_off", ctypes.c_void_p), ("arc_ilabel", ctypes.c_void_p), ("arc_weight", ctypes.c_void_p),
                ("arc_next", ctypes.c_void_p), ("finals", ctypes.c_void_p), ("backoff_id", ctypes.c_int),
                ("n_disambig", ctypes.c_int), ("disambig_ids", ctypes.c_int * 4)]


class BeamXfState(ctypes.Structure):
    """pk_beam_xf_state: the device buffers of the transformer prediction net's incremental beam step"""
    _fields_ = [("next_ys", ctypes.c_void_p), ("step_ctx", ctypes.c_void_p), ("hyp_tok", ctypes.c_void_p), ("hyp_len", ctypes.c_void_p),
                ("slot", ctypes.c_void_p), ("pool", ctypes.c_void_p), ("n_entries", ctypes.c_longlong), ("blk", ctypes.c_int),
                ("rows", ctypes.c_int), ("S1", ctypes.c_int), ("layers", ctypes.c_int), ("D", ctypes.c_int), ("dtype", ctypes.c_int),
                ("init", ctypes.c_int)]


STRUCTS = {"pk_view4": View4, "pk_gemm_desc": GemmDesc, "pk_lm_fst": LmFst, "pk_beam_xf_state": BeamXfState}
_SCALARS = {"int": ctypes.c_int, "long long": ctypes.c_longlong, "float": ctypes.c_float, "double": ctypes.c_double,
            "uint32_t": ctypes.c_uint32, "unsigned int": ctypes.c_uint32}
_RESULTS = {"int": ctypes.c_int, "long long": ctypes.c_longlong, "const char*": ctypes.c_char_p}


def _param_type(decl, fn):
    """'const float* w' -> c_void_p, 'const pk_gemm_desc* desc' -> POINTER(GemmDesc), 'long long n' -> c_longlong, ..."""
    words = re.findall(r"\w+|\*", decl)[:-1]                  # the type: drop the parameter's name
    if "*" in words:
        base = " ".join(w for w in words if w not in ("const", "*"))
        if base in STRUCTS:
            return ctypes.POINTER(STRUCTS[base])
        if not base.startswith("pk_"):
            return ctypes.c_void_p
    elif " ".join(words) in _SCALARS:
        return _SCALARS[" ".join(words)]
    raise ImportError("pika_b200: %s: no ctypes type for the parameter %r of %s" % (HEADER_PATH, decl, fn))


class _CDLL(ctypes.CDLL):
    # ctypes lets a function flagged cdecl take more arguments than its argtypes list; without the flag the count must match
    # exactly.  On Linux the flag has no other effect: the calling convention is the platform's either way.
    _func_flags_ = 0


def _bind(lib):
    for ret, name, params in _PROTOTYPES:
        if not hasattr(lib, name):
            raise ImportError("pika_b200: %s declares %s, which %s does not export" % (HEADER_PATH, name, LIB_PATH))
        ret = re.sub(r"\s*\*", "*", ret)
        if ret not in _RESULTS:
            raise ImportError("pika_b200: %s: no ctypes type for the return type %r of %s" % (HEADER_PATH, ret, name))
        fn = getattr(lib, name)
        fn.restype = _RESULTS[ret]
        fn.argtypes = [_param_type(p, name) for p in params]
    return lib


if not os.path.exists(LIB_PATH):
    raise ImportError(
        "pika_b200: %s is missing -- build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(there is no CPU fallback)" % LIB_PATH)

lib = _bind(_CDLL(LIB_PATH))


def check(rc, what=""):
    if rc != 0:
        raise PikaError("%s failed (rc=%d): %s" % (what, rc, lib.pk_last_error().decode()))


def launch_count():
    return int(lib.pk_launch_count())
