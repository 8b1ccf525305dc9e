"""ctypes binding of libb200sql.so.  Prototypes are derived from include/b200sql.h so the Python
side can never drift from the C ABI.  There is NO CPU fallback: if the library is missing the
import fails loudly, and every call fails loudly when no CUDA device is present."""
import ctypes
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "b200sql.h")
LIB_PATH = os.path.join(HERE, "lib", "libb200sql.so")

_CTYPES = {
    "int": ctypes.c_int, "int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64, "size_t": ctypes.c_size_t,
    "b2_handle": ctypes.c_int64, "float": ctypes.c_float, "void": None,
}


class B2ColumnInfo(ctypes.Structure):
    _fields_ = [("dtype", ctypes.c_int32), ("scale", ctypes.c_int32), ("size", ctypes.c_int64),
                ("null_count", ctypes.c_int64), ("data", ctypes.c_void_p), ("validity", ctypes.c_void_p),
                ("offsets", ctypes.c_void_p), ("data_bytes", ctypes.c_int64)]


class B2AggSpec(ctypes.Structure):
    _fields_ = [("kind", ctypes.c_int32), ("column", ctypes.c_int32), ("out_dtype", ctypes.c_int32),
                ("out_scale", ctypes.c_int32), ("out_precision", ctypes.c_int32)]


class B2HostColumn(ctypes.Structure):
    _fields_ = [("dtype", ctypes.c_int32), ("scale", ctypes.c_int32), ("rows", ctypes.c_int64), ("data", ctypes.c_void_p),
                ("validity_bits", ctypes.c_void_p), ("offsets", ctypes.c_void_p)]


class B2OrderByArg(ctypes.Structure):
    _fields_ = [("column", ctypes.c_int32), ("ascending", ctypes.c_int32), ("nulls_first", ctypes.c_int32)]


class B2WindowSpec(ctypes.Structure):
    _fields_ = [("kind", ctypes.c_int32), ("column", ctypes.c_int32), ("frame", ctypes.c_int32), ("offset", ctypes.c_int32),
                ("lower", ctypes.c_int64), ("upper", ctypes.c_int64), ("default_value", ctypes.c_uint8 * 16),
                ("default_is_null", ctypes.c_int32), ("out_dtype", ctypes.c_int32), ("out_precision", ctypes.c_int32),
                ("out_scale", ctypes.c_int32), ("ignore_nulls", ctypes.c_int32)]


def _arg_type(decl):
    decl = decl.strip()
    if "*" in decl:
        return ctypes.c_void_p  # every pointer is passed as an address (buffers, arrays, out-params)
    base = decl.replace("const", "").split()
    return _CTYPES[base[0]]


def parse_header(path=HEADER):
    """-> {name: (restype_str, [arg decls])} for every function declared in the header."""
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    out = {}
    for m in re.finditer(r"\b(int|void\s*\*|const\s+char\s*\*)\s*(b2_\w+)\s*\(([^;{}]*?)\)\s*;", src, flags=re.S):
        ret, name, args = m.group(1), m.group(2), m.group(3)
        args = [a for a in (x.strip() for x in args.split(",")) if a and a != "void"]
        out[name] = (ret, args)
    return out


class B2Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("b200sql error %d: %s" % (code, msg))
        self.code = code


def load():
    if not os.path.exists(LIB_PATH):
        raise ImportError("libb200sql.so is not built (%s); run `python -c 'import __graft_entry__ as g; g.build()'`. "
                          "There is no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
    for name, (ret, args) in parse_header().items():
        if not hasattr(lib, name) and os.environ.get("B2_ALLOW_MISSING"):
            continue  # development only
        fn = getattr(lib, name)  # AttributeError here = header/library drift
        fn.argtypes = [_arg_type(a) for a in args]
        if ret == "int":
            fn.restype = ctypes.c_int
        elif "char" in ret:
            fn.restype = ctypes.c_char_p
        else:
            fn.restype = ctypes.c_void_p
    return lib


lib = load()


def check(rc):
    if rc != 0:
        raise B2Error(rc, (lib.b2_last_error() or b"").decode())
