"""ctypes front end of tests/join_oracle.c, the CPU oracle's seed joins (DESIGN.md 2.7). TEST INFRASTRUCTURE ONLY. The
library is compiled with the oracle's own flags into the temporary directory, under a name derived from its sources, so
the repository tree is never written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRCS = [os.path.join(_HERE, "join_oracle.c"), os.path.join(_HERE, "push_pull_oracle.c"),
         os.path.join(_ROOT, "oracle", "swim_oracle.c"), os.path.join(_ROOT, "include", "swim.h")]
_CFLAGS = ["-O2", "-march=x86-64-v3", "-fPIC", "-Wall", "-Wextra", "-fvisibility=hidden", "-fopenmp", "-shared"]
_lib = None


def build():
    h = hashlib.sha256()
    for p in _SRCS:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(_CFLAGS).encode())
    so = os.path.join(tempfile.gettempdir(), f"swim_join_oracle_{h.hexdigest()[:16]}.so")
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
        L.oracle_join.restype = C.c_int
        L.oracle_join.argtypes = [C.c_void_p, u32p, u32p, C.c_size_t, C.c_uint32, u64p, u64p, u64p]
        _lib = L
    return _lib


def join(orc, nodes, seeds, fresh=False):
    """Seed joins on an oracle.oracle.Oracle at its current round: pair k is (nodes[k], seeds[k]). Returns (exchanges,
    inserted, full)."""
    from oracle.oracle import OracleError
    u32p = C.POINTER(C.c_uint32)
    nodes = np.ascontiguousarray(np.atleast_1d(nodes), dtype=np.uint32)
    seeds = np.ascontiguousarray(np.atleast_1d(seeds), dtype=np.uint32)
    assert len(nodes) == len(seeds)
    e, i, f = C.c_uint64(), C.c_uint64(), C.c_uint64()
    rc = lib().oracle_join(orc._h, nodes.ctypes.data_as(u32p), seeds.ctypes.data_as(u32p), len(nodes), 1 if fresh else 0,
                           C.byref(e), C.byref(i), C.byref(f))
    if rc:
        raise OracleError(rc, "join")
    return e.value, i.value, f.value
