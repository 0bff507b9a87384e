"""The ctypes signature table of engine.py against the prototypes of include/cosmo_b200.h: the same entry points, the
same number of parameters, the same return types, and scalar parameters of the same width (no library needed)."""
import ctypes as C
import os
import re

from cosmo_b200 import engine as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_RESTYPES = {"int": C.c_int, "void": None, "const char*": C.c_char_p}
_SCALARS = {"int32_t": C.c_int32, "int64_t": C.c_int64, "double": C.c_double}


def _prototypes():
    """{name: (return type, [parameter declarations])} of every function the header declares."""
    src = re.sub(r"/\*.*?\*/", " ", open(os.path.join(ROOT, "include", "cosmo_b200.h")).read(), flags=re.S)
    protos = {}
    pattern = r"^([A-Za-z_][\w ]*?\*?)\s*(cosmo_b200_\w+)\s*\(([^)]*)\)\s*;"
    for ret, name, params in re.findall(pattern, src, flags=re.M):
        params = " ".join(params.split())
        protos[name] = (ret.strip(), [] if params == "void" else [p.strip() for p in params.split(",")])
    return protos


def test_the_table_names_every_entry_point_of_the_header():
    protos = _prototypes()
    assert len(protos) >= 40
    assert set(E.SIGNATURES) == set(protos)
    assert E.EXPORTS == list(E.SIGNATURES)


def test_arity_and_return_type_of_every_entry_point():
    protos = _prototypes()
    for name, (restype, argtypes) in E.SIGNATURES.items():
        ret, params = protos[name]
        assert len(argtypes) == len(params), name
        assert restype is _RESTYPES[ret], name
    assert {n for n, (ret, _) in protos.items() if ret != "int"} == {"cosmo_b200_destroy", "cosmo_b200_last_error"}


def test_scalar_parameters_keep_their_width_and_pointers_stay_pointers():
    for name, (_, params) in _prototypes().items():
        for decl, t in zip(params, E.SIGNATURES[name][1]):
            if "*" in decl or "[" in decl:
                assert t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer), (name, decl)
            else:
                assert t is _SCALARS[decl.split()[0]], (name, decl)
