"""ctypes binding of libssp_b200.so, read from include/ssp_b200.h itself: the argument and return types of every entry point,
the SSP_* integer macros and the structs that cross the boundary are parsed from the header, so there is no second copy of them
to keep in step.  There is NO fallback: if the library is missing or a call fails, an exception is raised -- the product path
never routes through the CPU oracle."""
from __future__ import annotations

import ctypes as C
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SSP_LIB") or os.path.join(_HERE, "csrc", "libssp_b200.so")   # SSP_LIB: A/B experiments only


class SspError(RuntimeError):
    pass


_CTYPES = {"int": C.c_int, "unsigned": C.c_uint, "long long": C.c_longlong, "float": C.c_float, "double": C.c_double}


def _ctype(decl, where):
    """the ctypes type of a C type as the header spells it; every pointer is a c_void_p (callers pass ptr(t), None or byref)"""
    decl = " ".join(decl.split()).removeprefix("const ")
    if decl.endswith("*"):
        return C.c_void_p
    if decl not in _CTYPES:
        raise SspError("ssp_b200.h: unknown type '%s' in: %s" % (decl, " ".join(where.split())))
    return _CTYPES[decl]


def _decls(text, sep, where):
    """[(name, ctype)] of a parameter list (sep ',') or a struct body (sep ';', where 'int ow, oh' declares two fields)"""
    out = []
    for decl in filter(None, map(str.strip, text.split(sep))):
        first, *names = decl.split(",")
        m = re.fullmatch(r"(.*[\s*])(\w+)", first.strip(), re.S)
        if not m:
            raise SspError("ssp_b200.h: no 'type name' in '%s' of: %s" % (decl, " ".join(where.split())))
        out += [(n.strip(), _ctype(m.group(1), where)) for n in [m.group(2)] + names]
    return out


def parse_header(text):
    """The binding the header text declares: ({symbol: argtypes}, {symbol: restype}, {macro: int}, {struct name: Structure class}).
    Reads the constructs include/ssp_b200.h uses and nothing else of C; anything it cannot read is an SspError, never a guess."""
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    text = re.sub(r"#ifdef __cplusplus.*?#endif", "", text, flags=re.S)            # the extern "C" braces
    constants = {}
    for name, value in re.findall(r"^#define[ \t]+(\w+)[ \t]+(\S.*?)[ \t]*$", text, re.M):
        if not re.fullmatch(r"-?\d+|\(-?\d+\)", value):
            raise SspError("ssp_b200.h: #define %s %s is not an integer literal" % (name, value))
        constants[name] = int(value.strip("()"))
    text = re.sub(r"^#.*$", "", text, flags=re.M)
    structs = {}

    def struct(m):
        structs[m.group(1)] = type(m.group(1), (C.Structure,), {"_fields_": _decls(m.group(2), ";", m.group(0))})
        return ""
    text = re.sub(r"typedef struct (\w+) \{(.*?)\} \1;", struct, text, flags=re.S)
    signatures, returns = {}, {}
    for stmt in filter(None, map(str.strip, text.split(";"))):
        m = re.fullmatch(r"(.*?[\s*])(ssp_\w+)\s*\((.*)\)", stmt, re.S)
        if not m:
            raise SspError("ssp_b200.h: neither a prototype nor a struct: %s" % " ".join(stmt.split()))
        ret, name, args = m.groups()
        returns[name] = C.c_char_p if ret.split() == ["const", "char*"] else _ctype(ret, stmt)
        signatures[name] = [] if args.strip() == "void" else [t for _, t in _decls(args, ",", stmt)]
    return signatures, returns, constants, structs


# Parsed once at import (the constants are read by importers at their import); the library itself is opened lazily by load().
with open(os.path.join(_HERE, "..", "include", "ssp_b200.h")) as _f:
    SIGNATURES, RETURNS, CONSTANTS, STRUCTS = parse_header(_f.read())
# FMT_F16, IMPL_BANDT, EPI_STATS, ROUTE_POOL, ...: the header's SSP_FMT_* / SSP_IMPL_* / SSP_EPI_* / SSP_ROUTE_* without the prefix
globals().update((k[4:], v) for k, v in CONSTANTS.items() if k.startswith(("SSP_FMT_", "SSP_IMPL_", "SSP_EPI_", "SSP_ROUTE_")))

_lib = None


def load():
    """Load the CUDA library (building is __graft_entry__.build()'s job).  Raises if it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SspError("libssp_b200.so not built (%s): run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "-- singleshotpose_b200 has no CPU fallback" % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        for name, args in SIGNATURES.items():
            fn = getattr(lib, name)            # AttributeError if the .so lacks a declared symbol
            fn.argtypes = args
            fn.restype = RETURNS[name]
        _lib = lib
    return _lib


def call(name, *args):
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise SspError("%s failed (%d): %s" % (name, rc, lib.ssp_last_error().decode()))
    return rc


def ptr(t):
    """device (or host) pointer of a torch tensor / None."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def flat_alloc_rows(N, H, W):
    return int(load().ssp_flat_alloc_rows(N, H, W))
