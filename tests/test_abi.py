"""The C-ABI shared library loads on a CPU-only box, exports every symbol include/bke.h declares, the ctypes
binding agrees with the header (prototypes, struct layouts, constants), the library validates arguments, and it
refuses to compute without a GPU (no CPU fallback)."""
import ctypes
import os
import re
import subprocess
from ctypes import c_char_p, c_double, c_int, c_int32, c_int64, c_size_t, c_uint32, c_uint64, c_void_p

import numpy as np
import pytest

from filterpy_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


_SCALARS = {"int64_t": c_int64, "int32_t": c_int32, "uint32_t": c_uint32, "uint64_t": c_uint64, "double": c_double,
            "size_t": c_size_t}
_RETURNS = {"int": c_int, "size_t": c_size_t, "const char *": c_char_p, "void": None}


def _header():
    """include/bke.h with comments stripped: its numeric #defines, struct typedefs {name: body} and prototypes
    [(return type, name, [(type, parameter name)])]."""
    src = open(os.path.join(ROOT, "include", "bke.h")).read()
    src = re.sub(r"/\*.*?\*/|//[^\n]*", " ", src, flags=re.S)
    defines = {k: int(v) for k, v in re.findall(r"^#define (BKE_\w+) (\d+)u?[ \t]*$", src, re.M)}
    code = re.sub(r"^[ \t]*#.*$", "", src, flags=re.M)
    structs = {name: body for body, name in re.findall(r"typedef struct (?:\w+ )?\{([^{}]*)\}\s*(bke_\w+);", code)}
    protos = []
    for ret, name, params in re.findall(r"([\w\s*]+?)\b(bke_\w+)\s*\(([^()]*)\)\s*;", code):
        params = [] if params.strip() == "void" else [re.fullmatch(r"(.*?)\s*(\w+)", p.strip()).groups()
                                                      for p in params.split(",")]
        protos.append((" ".join(ret.split()), name, params))
    return defines, structs, protos


def _members(body):
    """The member names of a struct body, in order."""
    names = []
    for decl in body.split(";"):
        decl = re.sub(r"\[\w+\]", "", decl)
        names += [re.findall(r"\w+", d)[-1] for d in decl.split(",") if d.strip()]
    return names


def _structs_by_signature(lib):
    """{C struct: ctypes class} wherever a prototype takes `bke_X *` and the binding passes POINTER(cls)."""
    _, structs, protos = _header()
    pairs = {}
    for _, name, params in protos:
        for (ctype, _), argtype in zip(params, getattr(lib, name).argtypes or ()):
            base = ctype.replace("const", "").replace("*", "").strip()
            if base in structs and ctype.count("*") == 1 and argtype is not c_void_p:
                pairs.setdefault(base, set()).add(argtype._type_)
    assert set(pairs) == set(structs), set(structs) ^ set(pairs)
    assert all(len(classes) == 1 for classes in pairs.values()), pairs
    return structs, {c: classes.pop() for c, classes in pairs.items()}


def _accepts(argtype, ctype, structs):
    """Whether the ctypes argument type passes a C parameter of type `ctype` correctly."""
    base, stars = ctype.replace("const", "").replace("*", "").strip(), ctype.count("*")
    if stars == 0:
        return argtype is _SCALARS[base]
    if stars == 2:                                   # T ** and const void *const *
        return argtype is ctypes.POINTER(c_void_p)
    if base == "char":
        return argtype is c_char_p
    if argtype is c_void_p:                          # any other pointer, a struct in device memory included
        return True
    if not (isinstance(argtype, type) and issubclass(argtype, ctypes._Pointer)):
        return False
    if base in structs:
        return issubclass(argtype._type_, ctypes.Structure)
    return argtype._type_ is _SCALARS.get(base)


def test_header_symbols_are_exported():
    """The library exports every prototype of include/bke.h, and the binding types each one as declared."""
    lib = _lib.load()
    _, structs, protos = _header()
    assert {name for _, name, _ in protos} == set(_lib.EXPORTED_SYMBOLS), \
        {name for _, name, _ in protos} ^ set(_lib.EXPORTED_SYMBOLS)
    for ret, name, params in protos:
        f = getattr(lib, name)
        assert f.restype is _RETURNS[ret], name
        assert len(f.argtypes) == len(params), name
        for i, ((ctype, pname), argtype) in enumerate(zip(params, f.argtypes)):
            assert _accepts(argtype, ctype, structs), (name, i, pname, ctype, argtype)
    assert lib.bke_abi_version() == 1


def test_struct_layout_matches_header(tmp_path):
    """Every struct of include/bke.h has the ctypes class the prototypes pass it as, with the C compiler's layout:
    the same members in the same order, and by name the same offset and size of each, and the same sizeof."""
    structs, classes = _structs_by_signature(_lib.load())
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "bke.h"',
             '#define MEMBER(T, f) printf(#T " " #f " %zu %zu\\n", offsetof(T, f), sizeof(((T *)0)->f))',
             'int main(void) {']
    for cname, cls in classes.items():
        assert [f for f, _ in cls._fields_] == _members(structs[cname]), cname
        lines.append('printf("%s sizeof %%zu\\n", sizeof(%s));' % (cname, cname))
        lines += ['MEMBER(%s, %s);' % (cname, f) for f, _ in cls._fields_]
    lines += ['return 0; }']
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = {}
    for ln in subprocess.check_output([str(exe)]).decode().split("\n"):
        if ln.strip():
            cname, fname, *values = ln.split()
            got[cname, fname] = tuple(int(v) for v in values)
    for cname, cls in classes.items():
        assert got[cname, "sizeof"] == (ctypes.sizeof(cls),), cname
        for fname, _ in cls._fields_:
            field = getattr(cls, fname)
            assert (field.offset, field.size) == got[cname, fname], (cname, fname)
    assert _lib.KfArgs.alpha_sq.offset == 32 and _lib.KfArgs.x.offset == 40


def test_constants_match_the_header():
    defines, _, _ = _header()
    assert defines
    for name, value in defines.items():
        assert getattr(_lib, name, None) == value, name


def test_argument_validation_without_gpu():
    lib = _lib.load()
    a = _lib.KfArgs()
    a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags = 4, 0, 1, _lib.BKE_F64, 3
    assert lib.bke_kf_step(a, None) == _lib.BKE_ERR_BAD_ARG
    assert b"dim_x must be 1 or greater" in lib.bke_last_error()
    a.dim_x = 2
    a.flags = 0
    assert lib.bke_kf_step(a, None) == _lib.BKE_ERR_BAD_ARG
    with pytest.raises(ValueError):
        _lib.check(_lib.BKE_ERR_BAD_ARG)
    assert lib.bke_resample_workspace_bytes(1 << 20) > (1 << 20) // 2048 * 8
    assert lib.bke_systematic_resample(-1, None, 0.5, None, None, 0, None, None, None) == _lib.BKE_ERR_BAD_ARG


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = _lib.load()
    assert lib.bke_device_count() == 0
    x = np.zeros((1, 2)); P = np.eye(2)[None].copy(); F = np.eye(2); Q = np.eye(2)
    a = _lib.KfArgs()
    a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags, a.alpha_sq = 1, 2, 1, _lib.BKE_F64, _lib.BKE_DO_PREDICT, 1.0
    a.x = a.x_out = x.ctypes.data; a.P = a.P_out = P.ctypes.data; a.F = F.ctypes.data; a.Q = Q.ctypes.data
    assert lib.bke_kf_step(a, None) == _lib.BKE_ERR_CUDA
    assert b"no CPU fallback" in lib.bke_last_error()
    from filterpy_b200.kalman import KalmanFilter
    from filterpy_b200.monte_carlo import systematic_resample
    with pytest.raises(_lib.BkeError):
        KalmanFilter(2, 1)
    with pytest.raises(_lib.BkeError):
        systematic_resample([.5, .5])
    from filterpy_b200.monte_carlo import residual_resample, multinomial_resample
    for fn in (residual_resample, multinomial_resample):
        with pytest.raises(_lib.BkeError):
            fn([.5, .5])
    # the filter whose steps run on the tensor-core tile has no CPU path either
    with pytest.raises(_lib.BkeError):
        KalmanFilter(16, 4, n_filters=8, dtype=np.float32)


def test_product_never_imports_oracle():
    """The product path must not route through the oracle (only tests/, smoke() and bench.py may)."""
    pkg = os.path.join(ROOT, "filterpy_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), f
                assert "liboracle" not in src, f
