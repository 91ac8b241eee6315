"""include/simon_gpu.h against its one Python copy, simon_b200/abi.py: the value of every constant and the layout of every struct as
a small C program built from the header prints them, and every prototype as the header text states it.  CPU only; the library test
loads the built library without a device call."""
import ctypes as C
import os
import re
import subprocess
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest

from simon_b200 import abi, engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# header constants Python does not use: a call's status is only compared with 0, its text comes from simon_last_error
UNUSED = {"SIMON_OK", "SIMON_ERR_INVALID", "SIMON_ERR_CUDA", "SIMON_ERR_STATE", "SIMON_ERR_LIMIT", "SIMON_ERR_NOMEM"}
# structs passed as numpy arrays: simon_plan_step as abi.PLAN_STEP_DTYPE, simon_move / simon_move_rank as the rows of the [n, 2]
# uint32 array of Engine.moves_upload / int32 array of Engine.moves_run's top-k
DTYPES = {"simon_plan_step": abi.PLAN_STEP_DTYPE}
ROWS = {"simon_move": np.dtype(np.uint32), "simon_move_rank": np.dtype(np.int32)}
CTYPES = {"char": C.c_char, "int": C.c_int, "float": C.c_float, "double": C.c_double, "uint8_t": C.c_uint8, "int32_t": C.c_int32,
          "uint32_t": C.c_uint32, "int64_t": C.c_int64, "uint64_t": C.c_uint64}


def _decl(text):
    """One C declaration -> (base type, pointer depth, name, array length or None): 'const simon_ctx_opts *opts' ->
    ('simon_ctx_opts', 1, 'opts', None), 'char kernel[48]' -> ('char', 0, 'kernel', 48)."""
    m = re.fullmatch(r"\s*(?:const\s+)?(\w+)\s*((?:\*\s*)*)(\w+)\s*(?:\[(\d+)\])?\s*", text)
    assert m, text
    return m[1], m[2].count("*"), m[3], int(m[4]) if m[4] else None


def _parse(code):
    """Constant names, {struct: [(field, base type, pointer depth, array length)]} and {function: ((return type, pointer depth),
    [(parameter type, pointer depth)])} of the header text without comments."""
    consts = re.findall(r"^#define\s+(SIMON_\w+)[ \t]+\S", code, re.M)
    for body in re.findall(r"enum\s+\w+\s*\{(.*?)\}", code, re.S):
        consts += [m.split("=")[0].strip() for m in body.split(",") if m.strip()]
    structs = {}
    for name, body in re.findall(r"typedef\s+struct\s+(\w+)\s*\{(.*?)\}\s*\1\s*;", code, re.S):
        structs[name] = []
        for d in filter(str.strip, body.split(";")):
            first, *more = d.split(",")
            ty, ptr, f, n = _decl(first)
            structs[name] += [(f, ty, ptr, n)] + [(_decl(f"{ty} {m}")[2], ty, ptr, n) for m in more]
    protos = {}
    for head, params in re.findall(r"^([^;{}()#]*?\bsimon_\w+)\s*\(([^)]*)\)\s*;", code, re.M):
        ty, ptr, name, _ = _decl(head)
        protos[name] = ((ty, ptr), [_decl(p)[:2] for p in params.split(",") if p.strip() != "void"])
    return consts, structs, protos


@pytest.fixture(scope="module")
def header():
    """The header parsed, and what the compiler says of it: the value of every constant, sizeof of every struct and (offset, size) of
    every field."""
    with open(os.path.join(ROOT, "include", "simon_gpu.h")) as fh:
        consts, structs, protos = _parse(re.sub(r"/\*.*?\*/|//[^\n]*", " ", fh.read(), flags=re.S))
    out = [f'printf("const {n} %lld\\n", (long long)({n}));' for n in consts]
    for s, fields in structs.items():
        out.append(f'printf("size {s} %zu\\n", sizeof({s}));')
        out += [f'printf("field {s}.{f} %zu %zu\\n", offsetof({s}, {f}), sizeof((({s} *)0)->{f}));' for f, *_ in fields]
    src = "#include <stdio.h>\n#include <stddef.h>\n#include \"simon_gpu.h\"\nint main(void) {\n" + "\n".join(out) + "\nreturn 0;\n}\n"
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "abi.c"), "w") as fh:
            fh.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "abi.c"), "-o", os.path.join(d, "abi")])
        lines = [ln.split() for ln in subprocess.check_output([os.path.join(d, "abi")]).decode().splitlines()]
    return SimpleNamespace(structs=structs, protos=protos, values={k: int(v) for t, k, v in (x for x in lines if x[0] == "const")},
                           sizes={k: int(v) for t, k, v in (x for x in lines if x[0] == "size")},
                           fields={k: (int(o), int(n)) for t, k, o, n in (x for x in lines if x[0] == "field")})


def _check_type(t, ty, ptr, where):
    """ctypes type t stands for C type `ty` behind `ptr` pointers: the same scalar type, c_char_p for char *, c_void_p for any pointer,
    POINTER(T) for a pointer to what T stands for; None for void."""
    if ty == "void" and ptr == 0:
        assert t is None, where
    elif ptr == 0:
        assert t is CTYPES[ty], where
    elif t is C.c_char_p:
        assert (ty, ptr) == ("char", 1), where
    elif t is not C.c_void_p:
        assert isinstance(t, type) and issubclass(t, C._Pointer), where
        _check_type(t._type_, ty, ptr - 1, where)


def test_constants_match_header(header):
    """Every constant of abi.py has the header's value; every header constant has a counterpart in abi.py unless it is on UNUSED."""
    mine = {k: v for k, v in vars(abi).items() if k.isupper() and type(v) is int}
    for k, v in mine.items():
        h = k if k in header.values else "SIMON_" + k
        assert header.values.get(h) == v, k
    for h in header.values:
        assert h in UNUSED or h.removeprefix("SIMON_") in mine, f"{h} has no counterpart in abi.py"
    assert UNUSED <= set(header.values)


def test_ctypes_layouts_match_header(header):
    """Every struct of the header against its Python mirror (the ctypes class named after it, or the numpy layout it is passed as): the
    same size, the same fields in the same order at the same offsets with the same sizes and types."""
    classes = set()
    for s, fields in header.structs.items():
        want = [(f, *header.fields[f"{s}.{f}"]) for f, *_ in fields]
        if s in ROWS:
            it = ROWS[s].itemsize
            assert header.sizes[s] == len(fields) * it and [w[1:] for w in want] == [(i * it, it) for i in range(len(fields))], s
        elif s in DTYPES:
            dt = DTYPES[s]
            assert dt.itemsize == header.sizes[s], s
            assert [(f, dt.fields[f][1], dt.fields[f][0].itemsize) for f in dt.names] == want, s
            for f, ty, ptr, n in fields:
                assert ptr == 0 and n is None and dt.fields[f][0] == np.dtype(CTYPES[ty]), f"{s}.{f}"
        else:
            cls = getattr(abi, "".join(w.capitalize() for w in s.split("_")))
            classes.add(cls)
            assert C.sizeof(cls) == header.sizes[s], s
            assert [(f, getattr(cls, f).offset, getattr(cls, f).size) for f, _ in cls._fields_] == want, s
            for (f, ty, ptr, n), (_, t) in zip(fields, cls._fields_):
                if n is not None:
                    assert issubclass(t, C.Array) and t._length_ == n, f"{s}.{f}"
                    t = t._type_
                _check_type(t, ty, ptr, f"{s}.{f}")
    assert classes == {v for v in vars(abi).values() if isinstance(v, type) and issubclass(v, C.Structure)}


def test_signatures_match_prototypes(header):
    """SIGNATURES and the header's prototypes name the same functions, and each entry has the prototype's arity, return type and, per
    parameter, its scalar type or a ctypes pointer type to what it points to."""
    assert set(abi.SIGNATURES) == set(header.protos)
    for name, (ret, params) in header.protos.items():
        restype, argtypes = abi.SIGNATURES[name]
        assert len(argtypes) == len(params), name
        _check_type(restype, *ret, f"{name} return type")
        for i, (t, p) in enumerate(zip(argtypes, params)):
            _check_type(t, *p, f"{name} parameter {i}")


def test_abi_library_exports(header):
    """The C-ABI library loads, exports every symbol include/simon_gpu.h declares, and reports the header's ABI version (no compute
    calls)."""
    L = engine.lib()
    for name in header.protos:
        assert hasattr(L, name), name
    assert set(engine.EXPORTS) == set(header.protos)
    assert L.simon_gpu_version() == abi.ABI_VERSION == 3
