"""CPU tests: magma_b200/_lib.py::SIGNATURES states every prototype of include/magma_b200.h in ctypes terms (same names,
same parameter count, the ctypes type of each parameter and return value), and a handle configured with it converts
plain Python values and rejects a wrong call before it reaches C."""
import ctypes
import os
import re

import pytest
import torch

from conftest import ROOT

_SCALARS = {"int": ctypes.c_int32, "int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64, "uint64_t": ctypes.c_uint64,
            "size_t": ctypes.c_size_t, "float": ctypes.c_float, "long long": ctypes.c_longlong}


def _struct_mirrors():
    from magma_b200 import _lib

    return {"mb200_gemm_args": _lib.GemmArgs, "mb200_vit_model": _lib.VitModelC, "mb200_vit_grads": _lib.VitGradsC,
            "mb200_gptj_model_ex": _lib.GptjModelExC}


def _ctype(c_type, is_return=False):
    """The ctypes type a C parameter or return type maps to."""
    t = " ".join(c_type.replace("*", " * ").split())
    if is_return and t == "const char *":
        return ctypes.c_char_p
    if t == "void * const *":
        return ctypes.POINTER(ctypes.c_void_p)
    if t.endswith("*"):
        base = t.removeprefix("const ").removesuffix(" *")
        return ctypes.POINTER(_struct_mirrors()[base]) if base.startswith("mb200_") else ctypes.c_void_p
    return _SCALARS[t]


def _header():
    return re.sub(r"/\*.*?\*/", " ", open(os.path.join(ROOT, "include", "magma_b200.h")).read(), flags=re.S)


def _prototypes():
    """{name: (return type, [parameter types])} of every function the header declares, as C type strings."""
    hdr = _header()
    out = {}
    for m in re.finditer(r"^((?:const\s+)?\w+(?:\s+\w+)?\s*\**)\s*(mb200_\w+)\s*\(([^)]*)\)\s*;", hdr, flags=re.M):
        params = [p.strip() for p in m.group(3).split(",")]
        params = [] if params == ["void"] else [re.match(r"(.*?)\s*\b\w+$", p, flags=re.S).group(1) for p in params]
        out[m.group(2)] = (m.group(1), params)
    return out


def test_signature_table_mirrors_the_header():
    from magma_b200._lib import EXPORTED_SYMBOLS, SIGNATURES

    protos = _prototypes()
    assert len(protos) == len(set(re.findall(r"\b(mb200_\w+)\s*\(", _header())))  # no prototype missed by the parser
    assert sorted(SIGNATURES) == sorted(protos)
    assert EXPORTED_SYMBOLS == list(SIGNATURES)
    for name, (ret, params) in protos.items():
        restype, argtypes = SIGNATURES[name]
        assert restype is _ctype(ret, is_return=True), f"{name} returns {ret}"
        assert len(argtypes) == len(params), f"{name} takes {len(params)} parameters"
        for i, (have, c_type) in enumerate(zip(argtypes, params)):
            assert have is _ctype(c_type), f"{name} parameter {i} is {c_type}, not {have.__name__}"


@pytest.fixture
def emul(monkeypatch):
    """The CPU emulation library installed as the loaded handle, as the emul_ops fixture installs it."""
    from magma_b200 import _lib
    from oracle import build_emul

    L = ctypes.CDLL(build_emul.build())
    monkeypatch.setattr(_lib, "_lib", L)
    return L


def test_lib_configures_an_installed_handle(emul):
    from magma_b200 import _lib

    assert _lib.lib() is emul
    assert not hasattr(emul, "mb200_gemm_last_plan")  # the emulation exports a subset: missing names are skipped
    assert list(emul.mb200_add.argtypes) == _lib.SIGNATURES["mb200_add"][1]
    assert emul.mb200_gptj_sched_workspace_bytes.restype is ctypes.c_size_t
    # plain values are converted; wrapped values, byref for pointers and struct pointers still pass
    a = torch.full((8,), 1.5, dtype=torch.bfloat16)
    y = torch.empty_like(a)
    assert emul.mb200_add(a.data_ptr(), a.data_ptr(), None, y.data_ptr(), 8, None) == 0
    assert torch.equal(y, torch.full_like(a, 3.0))
    assert emul.mb200_add(ctypes.c_void_p(a.data_ptr()), a.data_ptr(), None, y.data_ptr(), ctypes.c_int64(8), None) == 0
    ms, n = ctypes.c_double(-1.0), ctypes.c_longlong(-1)
    assert emul.mb200_prof_read(ctypes.byref(ms), ctypes.byref(ms), ctypes.byref(ms), ctypes.byref(n)) == 0
    assert ms.value == 0.0 and n.value == 0 and emul.mb200_launch_count() == 0


def test_wrong_calls_are_rejected_before_c(emul):
    from magma_b200 import _lib

    L = _lib.configure(emul)
    assert L.mb200_add.argtypes  # without argtypes the calls below would reach C with garbage in n and the stream
    a = torch.zeros(8, dtype=torch.bfloat16)
    p = a.data_ptr()
    with pytest.raises((ctypes.ArgumentError, TypeError)):
        L.mb200_add(p, p, None, p, 8)  # one argument too few
    with pytest.raises((ctypes.ArgumentError, TypeError)):
        L.mb200_add(p, p, None, p, 8.0, None)  # a float where int64_t n is declared
    with pytest.raises((ctypes.ArgumentError, TypeError)):
        L.mb200_vit_workspace_bytes(ctypes.byref(_lib.GptjModelExC()), 1)  # the wrong struct
