"""CPU: the snapshot-capture calls (docs/SPEC.md S.2d) are declared in include/fi_epp.h, bound by _abi.py with their
types, exported by the library, and the Python wrapper's argument checks need no device."""
import ctypes as C
import os
import re

import pytest

import fusioninfer_b200
from fusioninfer_b200 import _abi as abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = {
    "fi_epp_snapshot_capture": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]),
    "fi_epp_snapshot_read": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64]),
    "fi_epp_snapshot_free": (None, [C.c_void_p]),
}


def test_capture_calls_are_declared_bound_and_exported():
    src = open(os.path.join(ROOT, "include", "fi_epp.h")).read()
    assert "typedef struct fi_epp_capture fi_epp_capture;" in src
    for name in CALLS:
        assert re.search(r"\b" + name + r"\s*\(", re.sub(r"/\*.*?\*/", "", src, flags=re.S)), name
    bound = {name: (res, args) for name, res, args in abi.SYMBOLS}
    lib = abi.load()
    for name, (res, args) in CALLS.items():
        assert bound[name] == (res, args), name
        assert getattr(lib, name) is not None


def test_null_arguments_need_no_device():
    lib = abi.load()
    out, n = C.c_void_p(), C.c_uint64(0)
    assert lib.fi_epp_snapshot_capture(None, C.byref(out), C.byref(n)) == abi.FI_ERR_INVALID
    assert out.value is None
    assert lib.fi_epp_snapshot_read(None, None, 0) == abi.FI_ERR_INVALID
    lib.fi_epp_snapshot_free(None)  # a no-op


def test_closed_capture_refuses_to_read():
    c = fusioninfer_b200.SnapshotCapture(abi.load(), C.c_void_p(), 0)
    c.close()
    with pytest.raises(ValueError):
        c.read()
    with c:
        pass
