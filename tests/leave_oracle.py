"""ctypes front end of tests/leave_oracle.c, the CPU oracle's graceful leaves (DESIGN.md 2.8). TEST INFRASTRUCTURE ONLY.
The library is compiled with the oracle's own flags into the temporary directory, under a name derived from its sources,
so the repository tree is never written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRCS = [os.path.join(_HERE, "leave_oracle.c"), os.path.join(_ROOT, "oracle", "swim_oracle.c"),
         os.path.join(_ROOT, "include", "swim.h")]
_CFLAGS = ["-O2", "-march=x86-64-v3", "-fPIC", "-Wall", "-Wextra", "-fvisibility=hidden", "-fopenmp", "-shared"]
_lib = None


def build():
    h = hashlib.sha256()
    for p in _SRCS:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(_CFLAGS).encode())
    so = os.path.join(tempfile.gettempdir(), f"swim_leave_oracle_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.check_call(["gcc"] + _CFLAGS + ["-o", tmp, _SRCS[0]])
        os.replace(tmp, so)
    return so


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        u64p, u32p = C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)
        L.oracle_leave.restype = C.c_int
        L.oracle_leave.argtypes = [C.c_void_p, u32p, C.c_size_t, u64p, u64p]
        _lib = L
    return _lib


def leave(orc, nodes):
    """Graceful leaves on an oracle.oracle.Oracle at its current round. Returns (left, delivered)."""
    from oracle.oracle import OracleError
    u32p = C.POINTER(C.c_uint32)
    ids = np.ascontiguousarray(np.atleast_1d(nodes), dtype=np.uint32)
    lv, dl = C.c_uint64(), C.c_uint64()
    rc = lib().oracle_leave(orc._h, ids.ctypes.data_as(u32p), len(ids), C.byref(lv), C.byref(dl))
    if rc:
        raise OracleError(rc, "leave")
    return lv.value, dl.value
