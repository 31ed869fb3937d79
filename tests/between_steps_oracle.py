"""ctypes front end of tests/between_steps_oracle.c, the CPU oracle's calls between steps: push-pull (DESIGN.md 2.6),
seed joins (2.7) and graceful leaves (2.8). TEST INFRASTRUCTURE ONLY. The library is compiled with the oracle's own
flags (oracle/Makefile) into the temporary directory, under a name derived from its sources, so the repository tree is
never written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRCS = [os.path.join(_HERE, "between_steps_oracle.c"), os.path.join(_ROOT, "oracle", "swim_oracle.c"),
         os.path.join(_ROOT, "include", "swim.h")]
_CFLAGS = ["-O2", "-march=x86-64-v3", "-fPIC", "-Wall", "-Wextra", "-fvisibility=hidden", "-fopenmp", "-shared"]
_lib = None
_u32p, _u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)


def build():
    h = hashlib.sha256()
    for p in _SRCS:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(_CFLAGS).encode())
    so = os.path.join(tempfile.gettempdir(), f"swim_between_steps_oracle_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.check_call(["gcc"] + _CFLAGS + ["-o", tmp, _SRCS[0]])
        os.replace(tmp, so)
    return so


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        for f, args in ((L.oracle_push_pull, [C.c_void_p, _u64p, _u64p, _u64p]),
                        (L.oracle_join, [C.c_void_p, _u32p, _u32p, C.c_size_t, C.c_uint32, _u64p, _u64p, _u64p]),
                        (L.oracle_leave, [C.c_void_p, _u32p, C.c_size_t, _u64p, _u64p])):
            f.restype, f.argtypes = C.c_int, args
        _lib = L
    return _lib


def _ids(a):
    a = np.ascontiguousarray(np.atleast_1d(a), dtype=np.uint32)
    return a, a.ctypes.data_as(_u32p)


def _call(name, *args, outs):
    from oracle.oracle import OracleError
    res = [C.c_uint64() for _ in range(outs)]
    rc = getattr(lib(), "oracle_" + name)(*args, *map(C.byref, res))
    if rc:
        raise OracleError(rc, name)
    return tuple(r.value for r in res)


def push_pull(orc):
    """The exchange on an oracle.oracle.Oracle at its current round. Returns (exchanges, inserted, full)."""
    return _call("push_pull", orc._h, outs=3)


def join(orc, nodes, seeds, fresh=False):
    """Seed joins on an oracle.oracle.Oracle at its current round: pair k is (nodes[k], seeds[k]). Returns (exchanges,
    inserted, full)."""
    nodes, pn = _ids(nodes)
    seeds, ps = _ids(seeds)
    assert len(nodes) == len(seeds)
    return _call("join", orc._h, pn, ps, len(nodes), 1 if fresh else 0, outs=3)


def leave(orc, nodes):
    """Graceful leaves on an oracle.oracle.Oracle at its current round. Returns (left, delivered)."""
    ids, p = _ids(nodes)
    return _call("leave", orc._h, p, len(ids), outs=2)
