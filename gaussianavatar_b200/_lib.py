"""ctypes binding of libgavatar_sm90.so, derived at import from the C ABI declared in include/gavatar.h.

Each ``typedef struct`` of the header becomes a ``ctypes.Structure`` of the same name here, each integer ``#define GA_*`` a
module constant, and each ``ga_*`` prototype the restype / argtypes of the library function, so that an entry point is
declared once, in the header, and the compiler checks it against its definition.

There is no CPU fallback and no alternative backend: if the library is missing or a call fails, a RuntimeError is
raised.  The library is built in-tree by ``gaussianavatar_b200.build.build_library()`` (``__graft_entry__.build()``).
"""
from __future__ import annotations

import ctypes
import os
import re

from .build import LIB_PATH

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "gavatar.h")

# developer override: load an experiment build of the same library (same C ABI) instead of the in-tree one
LIB_PATH = os.environ.get("GA_LIB_PATH", LIB_PATH)

# the C types the ABI passes by value; every pointer is mapped in _ctype
_SCALARS = {"int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64, "size_t": ctypes.c_size_t, "float": ctypes.c_float,
            "int": ctypes.c_int, "long long": ctypes.c_longlong, "void": None}


def _ctype(ctype: str, structs: dict, what: str):
    """ctypes type of a C type without its name: char * -> c_char_p, a header struct's pointer -> POINTER(struct), any
    other pointer -> c_void_p, a value -> _SCALARS.  Anything else raises, naming the declaration `what`."""
    base = " ".join(w for w in ctype.replace("*", " ").split() if w != "const")
    stars = ctype.count("*")
    if stars == 1 and base == "char":
        return ctypes.c_char_p
    if stars == 1 and base in structs:
        return ctypes.POINTER(structs[base])
    if stars:
        return ctypes.c_void_p
    if base not in _SCALARS:
        raise RuntimeError(f"gavatar.h: no ctypes type for `{base}` in `{what}`")
    return _SCALARS[base]


def _declarator(decl: str):
    """'const float *Y[5]' -> ('const float *', 'Y', 5); the length is None for a declaration without [N]."""
    m = re.fullmatch(r"(.*\W)?(\w+)\s*(?:\[\s*(\d+)\s*\])?", decl.strip(), re.S)
    if not m:
        raise RuntimeError(f"gavatar.h: cannot read the declaration `{' '.join(decl.split())}`")
    return m.group(1) or "", m.group(2), None if m.group(3) is None else int(m.group(3))


def parse_header(text: str):
    """(structs, functions, constants) of a header written as include/gavatar.h is: {name: ctypes.Structure},
    {name: (restype, argtypes)} and {name: int} of its integer #define GA_* lines.  Enums are skipped; a statement that is
    neither a struct typedef nor a ga_* prototype, or a type outside _ctype's table, raises."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    constants = {k: int(v) for k, v in re.findall(r"^\s*#\s*define\s+(GA_\w+)\s+(-?\d+)\s*$", text, re.M)}
    text = re.sub(r"^\s*#.*$", "", text, flags=re.M)
    text = re.sub(r'extern\s+"C"\s*\{|\}\s*$', "", text)
    structs, functions = {}, {}

    def typedef(m):
        kind, body, name = m.groups()
        if kind == "struct":
            fields = []
            for stmt in filter(str.strip, body.split(";")):
                first, *more = stmt.split(",")        # `const float *Fp, *dFp`: the `*` and [N] belong to each name
                base = _declarator(first)[0].replace("*", " ")
                for decl in [first] + [base + d for d in more]:
                    ctype, field, n = _declarator(decl)
                    t = _ctype(ctype, structs, f"{name}.{field}")
                    fields.append((field, t if n is None else t * n))
            structs[name] = type(name, (ctypes.Structure,), {"_fields_": fields})
        return ""

    text = re.sub(r"typedef\s+(struct|enum)\s+\w+\s*\{(.*?)\}\s*(\w+)\s*;", typedef, text, flags=re.S)
    for stmt in filter(str.strip, text.split(";")):
        m = re.fullmatch(r"\s*(.*?)\b(ga_\w+)\s*\((.*)\)\s*", stmt, re.S)
        if not m:
            raise RuntimeError(f"gavatar.h: cannot read `{' '.join(stmt.split())}`")
        ret, name, params = m.groups()
        args = [] if params.strip() == "void" else \
            [_ctype(_declarator(p)[0], structs, f"{name}({' '.join(p.split())})") for p in params.split(",")]
        functions[name] = (_ctype(ret, structs, name), args)
    return structs, functions, constants


with open(HEADER) as _f:
    _STRUCTS, _SIGNATURES, _CONSTANTS = parse_header(_f.read())
globals().update(_STRUCTS)      # GaRasterSettings, GaRasterBatchDesc, ... (positional, in the header's field order)
globals().update(_CONSTANTS)    # GA_DECODER_TENSOR_CORES, ...

_lib = None


def lib() -> ctypes.CDLL:
    """Load the shared library (once).  Raises RuntimeError if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: the sm_90a CUDA library has not been built. Run "
                "`python -c 'import __graft_entry__ as g; g.build()'` (needs nvcc). There is no CPU fallback.")
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)     # AttributeError if the .so is stale -> loud
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().ga_last_error()
        raise RuntimeError(f"libgavatar {what} failed (status {rc}): {msg.decode() if msg else ''}")


def ptr(t) -> int | None:
    """Device pointer of a torch tensor (None -> NULL)."""
    if t is None:
        return None
    return t.data_ptr()


def profile(on: bool) -> None:
    lib().ga_profile_enable(1 if on else 0)


def profile_report() -> dict:
    """{kernel name: (launches, total_ms)} since the last report; synchronises the device."""
    buf = ctypes.create_string_buffer(1 << 16)
    check(lib().ga_profile_report(buf, len(buf)), "ga_profile_report")
    out = {}
    for line in buf.value.decode().splitlines():
        name, n, ms = line.rsplit(" ", 2)
        out[name] = (int(n), float(ms))
    return out


def launch_count() -> int:
    return int(lib().ga_launch_count())
