"""CPU: the C-ABI library loads and exports what include/gavatar.h declares, the bindings _lib.py derives from the header
have each prototype's arity and each struct's C layout, and the header parser reads every construct it supports (no compute
calls here)."""
import ctypes
import os
import re
import subprocess

import pytest

from gaussianavatar_b200 import _lib
from gaussianavatar_b200.build import LIB_PATH

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    """{name: parameter count} of every ga_* prototype, read without _lib's parser."""
    txt = open(os.path.join(ROOT, "include", "gavatar.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return {name: 0 if params.strip() == "void" else params.count(",") + 1
            for name, params in re.findall(r"\b(ga_[a-z0-9_]+)\s*\(([^)]*)\)", txt)}


def test_library_exists_and_loads():
    assert os.path.exists(LIB_PATH), "run __graft_entry__.build() first"
    L = _lib.lib()
    assert L.ga_version() >= 100
    assert L.ga_last_error() is not None


def test_header_and_binding_agree():
    declared = _declared()
    assert declared, "no declarations parsed"
    L = _lib.lib()
    for name, nparams in declared.items():
        assert hasattr(L, name), f"{name} declared in gavatar.h but not exported"
        assert name in _lib._SIGNATURES, f"{name} declared in gavatar.h but not bound by _lib.py"
        argtypes = getattr(L, name).argtypes
        assert argtypes is not None and len(argtypes) == nparams, \
            f"{name}: {nparams} parameters in gavatar.h, bound with {None if argtypes is None else len(argtypes)} argtypes"
    for name in _lib._SIGNATURES:
        assert name in declared, f"{name} bound by _lib.py but not declared in gavatar.h"


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _lib.lib()


def test_struct_layouts_match_c(tmp_path):
    """sizeof, and each field's offsetof and sizeof, of every header struct as the host C compiler lays it out, and the value of
    every #define GA_* constant, against the ctypes bindings."""
    lines = [f'printf("{k} %lld\\n", (long long)({k}));' for k in _lib._CONSTANTS]
    for name, S in _lib._STRUCTS.items():
        lines.append(f'printf("{name} %zu\\n", sizeof({name}));')
        lines += [f'printf("{name}.{f} %zu %zu\\n", offsetof({name}, {f}), sizeof((({name} *)0)->{f}));' for f, _ in S._fields_]
    src = tmp_path / "layout.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"gavatar.h\"\nint main(void) {\n    "
                   + "\n    ".join(lines) + "\n    return 0;\n}\n")
    exe = tmp_path / "layout"
    r = subprocess.run(["cc", "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    c = dict(line.split(" ", 1) for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())

    got = {k: str(v) for k, v in _lib._CONSTANTS.items()}
    for name, S in _lib._STRUCTS.items():
        got[name] = str(ctypes.sizeof(S))
        got.update({f"{name}.{f}": f"{getattr(S, f).offset} {getattr(S, f).size}" for f, _ in S._fields_})
    assert len(_lib._STRUCTS) >= 11 and "GA_DECODER_TENSOR_CORES" in got
    assert got == c


SNIPPET = r"""
/* a comment naming ga_not_a_prototype(int x); and a typedef struct GaNo { double d; } GaNo; */
#ifndef SNIPPET_H_
#define SNIPPET_H_
#define GA_ANSWER 42
#define GA_BELOW -3
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif
typedef enum GaStatus { GA_OK = 0, GA_ERR = -1 } GaStatus;
typedef struct GaT {
    int32_t n, first[9];         /* a value and an array in one line */
    const float *Fp, *dFp;
    const float *Y[5], *Y6, *Y7;
    int64_t big; size_t sz; float f; int i; long long ll;
    uint8_t *bytes;
    const double *stat;
} GaT;
typedef struct GaU {
    const GaT *t;
    float origin[3];
} GaU;
void ga_a(void);
const char *ga_b(char *buf, const char *name, size_t cap);
long long ga_c(const GaT *t, GaU *u, const void *v, double *w, int32_t **pp);
const int32_t *ga_d(int64_t n,
                    float x);  // a line comment
#ifdef __cplusplus
}
#endif
#endif
"""


def test_parse_header_snippet():
    structs, functions, constants = _lib.parse_header(SNIPPET)
    c = ctypes
    assert constants == {"GA_ANSWER": 42, "GA_BELOW": -3}
    assert list(structs) == ["GaT", "GaU"]
    GaT, GaU = structs["GaT"], structs["GaU"]
    assert GaT._fields_ == [("n", c.c_int32), ("first", c.c_int32 * 9), ("Fp", c.c_void_p), ("dFp", c.c_void_p),
                            ("Y", c.c_void_p * 5), ("Y6", c.c_void_p), ("Y7", c.c_void_p), ("big", c.c_int64),
                            ("sz", c.c_size_t), ("f", c.c_float), ("i", c.c_int), ("ll", c.c_longlong), ("bytes", c.c_void_p),
                            ("stat", c.c_void_p)]
    assert GaU._fields_ == [("t", c.POINTER(GaT)), ("origin", c.c_float * 3)]
    assert functions == {
        "ga_a": (None, []),
        "ga_b": (c.c_char_p, [c.c_char_p, c.c_char_p, c.c_size_t]),
        "ga_c": (c.c_longlong, [c.POINTER(GaT), c.POINTER(GaU), c.c_void_p, c.c_void_p, c.c_void_p]),
        "ga_d": (c.c_void_p, [c.c_int64, c.c_float]),
    }


@pytest.mark.parametrize("decl, error", [
    ("int ga_e(int32_t n, double x);", r"no ctypes type for `double` in `ga_e\(double x\)`"),
    ("uint32_t ga_e(int32_t n);", r"no ctypes type for `uint32_t` in `ga_e`"),
    ("typedef struct GaV { int32_t n; uint8_t b[4]; } GaV;", r"no ctypes type for `uint8_t` in `GaV.b`"),
    ("typedef struct GaV { int32_t n; } GaV;\nint ga_e(GaV v);", r"no ctypes type for `GaV` in `ga_e\(GaV v\)`"),
    ("int other_e(int32_t n);", r"cannot read `int other_e\(int32_t n\)`"),
])
def test_parse_header_refuses_unmapped(decl, error):
    with pytest.raises(RuntimeError, match=error):
        _lib.parse_header("#include <stdint.h>\n" + decl + "\n")
