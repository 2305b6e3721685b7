"""CPU check of the ctypes view of the C ABI: hover_net_b200._lib.PROTOTYPES declares exactly the functions of
include/hvn.h, with their parameter counts and types (every pointer as c_void_p, `const char *` as c_char_p).  The
table is read without loading libhvn.so."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_prototypes():
    """name -> (return type, [parameter types]) of every function include/hvn.h declares, as C text."""
    src = open(os.path.join(ROOT, "include", "hvn.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for ret, name, params in re.findall(r"^([A-Za-z_][\w \*]*?)\s*\b(hvn_[a-z0-9_]+)\s*\(([^)]*)\);", src, flags=re.M):
        ps = [] if params.strip() == "void" else [p.strip() for p in params.split(",")]
        # a parameter's type is its text without the trailing name; an array parameter decays to a pointer
        out[name] = (ret.strip(), [re.sub(r"\s*\b\w+\s*(\[\d*\])?$", lambda m: " *" if m.group(1) else "", p)
                                   for p in ps])
    # every hvn_ function the header names is one of the parsed declarations
    assert sorted(out) == sorted(set(re.findall(r"\b(hvn_[a-z0-9_]+)\s*\(", src)))
    return out


def _ctype(c):
    c = re.sub(r"\s+", " ", c.replace("*", " * ")).strip()
    if c == "const char *":
        return ctypes.c_char_p
    if "*" in c:
        return ctypes.c_void_p
    return {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "size_t": ctypes.c_size_t, "void": None}[c]


def test_prototype_table_matches_header():
    from hover_net_b200 import _lib
    declared = _declared_prototypes()
    assert len(declared) >= 25
    assert sorted(_lib.PROTOTYPES) == sorted(declared)
    for name, (ret, params) in declared.items():
        restype, argtypes = _lib.PROTOTYPES[name]
        assert restype is _ctype(ret), (name, ret, restype)
        assert len(argtypes) == len(params), (name, params, argtypes)
        for i, (c, t) in enumerate(zip(params, argtypes)):
            assert t is _ctype(c), (name, i, c, t)
