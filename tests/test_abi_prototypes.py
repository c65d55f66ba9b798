"""CPU: every ctypes signature in xuance_b200/_lib.py matches its prototype in include/xb200.h, parameter by parameter,
including the trailing ``void *stream`` that ``_lib.call`` appends.  A missing argtype is not an error to ctypes: the
extra Python int is passed as a 32-bit C int, so a stream handle would arrive truncated."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _prototypes():
    src = open(os.path.join(ROOT, "include", "xb200.h")).read()
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    out = {}
    for m in re.finditer(r"\b(?:int|int64_t|const char\s*\*)\s*\b(xb_\w+)\s*\(([^;]*?)\)\s*;", src):
        params = " ".join(m.group(2).split())
        out[m.group(1)] = [] if params in ("", "void") else [p.strip() for p in params.split(",")]
    return out


def _kind(param):
    """The ctypes class a C parameter declaration maps to."""
    decl = re.sub(r"\b(const|restrict|__restrict__)\b", " ", param)
    if "*" in decl or "[" in decl:
        return "pointer"
    words = decl.split()
    base = " ".join(words[:-1]) if len(words) > 1 else words[0]
    return {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "float": ctypes.c_float, "double": ctypes.c_double,
            "uint32_t": ctypes.c_uint32}[base]


def test_every_signature_matches_its_header_prototype():
    from xuance_b200 import _lib
    protos = _prototypes()
    checked = 0
    for name, sig in _lib._SIGNATURES.items():
        if sig is None:
            continue
        assert name in protos, f"{name} has a ctypes signature but no prototype in include/xb200.h"
        params, argtypes = protos[name], sig[1]
        assert len(argtypes) == len(params), (name, len(argtypes), len(params))
        for i, (p, t) in enumerate(zip(params, argtypes)):
            k = _kind(p)
            if k == "pointer":
                assert t is ctypes.c_void_p or issubclass(t, (ctypes._Pointer, ctypes.c_void_p)), (name, i, p, t)
            else:
                assert t is k, (name, i, p, t)
        checked += 1
    assert checked == len([k for k, v in _lib._SIGNATURES.items() if v is not None])


def test_the_distributional_entry_points_take_the_stream_last():
    protos = _prototypes()
    for name in ("xb_dist_greedy", "xb_c51_loss_fwd_bwd", "xb_qrdqn_loss_fwd_bwd"):
        assert protos[name][-1].replace(" ", "") == "void*stream", name
