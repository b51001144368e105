"""ctypes binding of libevk_sm90.so.  Prototypes are parsed from include/evk.h so the header stays the
single source of truth for the C ABI."""
import ctypes
import os
import re
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(HERE), "include", "evk.h")
LIB_PATH = os.environ.get("EVK_LIB_PATH") or os.path.join(HERE, "libevk_sm90.so")   # override: instrumented developer builds (tools/exp)
MAX_TAPS = 48


class GconvDesc(ctypes.Structure):
    _fields_ = (
        [(n, ctypes.c_void_p) for n in ("x", "w", "y", "res", "bias", "in_len", "out_len")]
        + [(n, ctypes.c_int64) for n in ("x_sb", "x_sh", "w_sb", "w_sh", "w_sq", "y_sb", "y_sh", "r_sb", "r_sh")]
        + [(n, ctypes.c_int32) for n in ("ldx", "ldw", "ldy", "ldr", "b_sh", "Z", "H", "C", "N", "Q", "G", "Tin", "J", "P",
                                         "is_", "os_", "o0", "Tout", "act")]
        + [("slope", ctypes.c_float), ("off", ctypes.c_int32 * MAX_TAPS)]
        + [("drop_rng", ctypes.c_void_p), ("drop_sid", ctypes.c_uint64), ("drop_p", ctypes.c_float)]
    )


_CTYPE = {
    "int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64, "uint64_t": ctypes.c_uint64, "float": ctypes.c_float,
    "int": ctypes.c_int, "evk_stream_t": ctypes.c_void_p,
}


def parse_header(path=HEADER):
    """-> {name: (restype, [argtypes])} for every function declared in evk.h."""
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(int|const char\*)\s+(evk_\w+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S):
        ret, name, args = m.group(1), m.group(2), m.group(3).strip()
        argtypes = []
        if args and args != "void":
            for a in args.split(","):
                a = a.strip()
                if "*" in a:
                    argtypes.append(ctypes.POINTER(GconvDesc) if "evk_gconv_desc" in a else ctypes.c_void_p)
                else:
                    ty = a.replace("const ", "").split()[0]
                    argtypes.append(_CTYPE[ty])
        protos[name] = (ctypes.c_char_p if "char" in ret else ctypes.c_int, argtypes)
    return protos


_lib = None
_lock = threading.Lock()
_inited = False


def load():
    """dlopen the library and attach prototypes (no CUDA call; safe on a CPU-only host)."""
    global _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                                   "(there is no CPU fallback)")
            lib = ctypes.CDLL(LIB_PATH)
            for name, (ret, argtypes) in parse_header().items():
                fn = getattr(lib, name)      # AttributeError => header/library mismatch: fail loudly
                fn.restype, fn.argtypes = ret, argtypes
            _lib = lib
    return _lib


def last_error():
    return load().evk_last_error().decode()


def init():
    """Load + evk_init() (requires an H100)."""
    global _inited
    lib = load()
    if not _inited:
        rc = lib.evk_init()
        if rc != 0:
            raise RuntimeError(f"evk_init failed ({rc}): {last_error()}")
        _inited = True
    return lib


def check(rc):
    if rc != 0:
        raise RuntimeError(f"libevk_sm90 error {rc}: {last_error()}")
