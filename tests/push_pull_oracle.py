"""ctypes front end of tests/push_pull_oracle.c, the CPU oracle's push-pull state exchange (DESIGN.md 2.6). TEST
INFRASTRUCTURE ONLY. The library is compiled with the oracle's own flags (oracle/Makefile) into the temporary directory,
under a name derived from its sources, so the repository tree is never written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRCS = [os.path.join(_HERE, "push_pull_oracle.c"), os.path.join(_ROOT, "oracle", "swim_oracle.c"),
         os.path.join(_ROOT, "include", "swim.h")]
_CFLAGS = ["-O2", "-march=x86-64-v3", "-fPIC", "-Wall", "-Wextra", "-fvisibility=hidden", "-fopenmp", "-shared"]
_lib = None


def build():
    h = hashlib.sha256()
    for p in _SRCS:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(_CFLAGS).encode())
    so = os.path.join(tempfile.gettempdir(), f"swim_push_pull_oracle_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.check_call(["gcc"] + _CFLAGS + ["-o", tmp, _SRCS[0]])
        os.replace(tmp, so)
    return so


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        u64p = C.POINTER(C.c_uint64)
        L.oracle_push_pull.restype = C.c_int
        L.oracle_push_pull.argtypes = [C.c_void_p, u64p, u64p, u64p]
        _lib = L
    return _lib


def push_pull(orc):
    """The exchange on an oracle.oracle.Oracle at its current round. Returns (exchanges, inserted, full)."""
    from oracle.oracle import OracleError
    e, i, f = C.c_uint64(), C.c_uint64(), C.c_uint64()
    rc = lib().oracle_push_pull(orc._h, C.byref(e), C.byref(i), C.byref(f))
    if rc:
        raise OracleError(rc, "push_pull")
    return e.value, i.value, f.value
