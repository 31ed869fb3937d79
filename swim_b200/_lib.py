"""Loader of the in-tree CUDA library (libswim_b200.so). There is no CPU fallback: if the
library is missing, import fails; if there is no GPU, swim_sim_create fails with ENODEV."""
import ctypes as C
import os

from . import _abi as A

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "libswim_b200.so")


class SwimError(RuntimeError):
    """`Left err` of the reference's `Either Error a` (Types.hs:33)."""

    def __init__(self, code, what, detail=""):
        super().__init__(f"{what}: {strerror(code)}" + (f" — {detail}" if detail else ""))
        self.code = code


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise ImportError(f"{SO_PATH} is missing: build it with `python -m swim_b200.build` "
                          "(nvcc, sm_90a). swim_b200 has no CPU fallback.")
    L = C.CDLL(SO_PATH)
    vp, u8p, u32, u64, sz, i = C.c_void_p, C.POINTER(C.c_uint8), C.c_uint32, C.c_uint64, C.c_size_t, C.c_int
    P = C.POINTER

    def sig(name, res, *args):
        f = getattr(L, name)
        f.restype = res
        f.argtypes = list(args)

    sig("swim_abi_version", u32)
    sig("swim_strerror", C.c_char_p, i)
    sig("swim_last_error", C.c_char_p, vp)
    sig("swim_config_default", i, P(A.Config))
    sig("swim_sim_create", i, P(A.Config), P(vp))
    sig("swim_sim_destroy", None, vp)
    sig("swim_sim_local_range", i, vp, P(u32), P(u32))
    sig("swim_sim_set_view", i, vp, vp)
    sig("swim_sim_set_view_device", i, vp, vp)
    sig("swim_sim_remove_dead_nodes", i, vp, u32, P(u64))
    sig("swim_sim_add_members", i, vp, vp, sz, P(u64), P(u64))
    sig("swim_topology_generate", i, i, u32, u32, u32, u64, vp)
    sig("swim_sim_set_round", i, vp, u32)
    sig("swim_sim_save", i, vp)
    sig("swim_sim_set_params", i, vp, P(A.Config))
    sig("swim_sim_calibrate", i, vp, vp, sz)
    sig("swim_sim_set_timeline", i, vp, u32)
    sig("swim_sim_get_timeline", i, vp, vp, sz)
    sig("swim_sim_load", i, vp)
    sig("swim_sim_step", i, vp, u32)
    sig("swim_sim_step_async", i, vp, u32)
    sig("swim_sim_sync", i, vp)
    sig("swim_sim_set_stream", i, vp, vp)
    sig("swim_sim_inject", i, vp, vp, sz)
    sig("swim_sim_round", i, vp, P(u32))
    sig("swim_sim_get_array", i, vp, i, vp, sz)
    sig("swim_sim_set_array", i, vp, i, vp, sz)
    sig("swim_sim_array_bytes", i, vp, i, P(sz))
    sig("swim_sim_digest", i, vp, P(u64))
    sig("swim_sim_counters", i, vp, vp, sz)
    sig("swim_sim_mismatches", i, vp, P(u64))
    sig("swim_sim_observe", i, vp, vp, sz, P(u64), P(u64))
    sig("swim_sim_step_observe", i, vp, u32, vp, sz, P(u64))
    sig("swim_sim_last_step_ms", i, vp, P(C.c_float))
    sig("swim_sim_launch_count", i, vp, P(u64))
    sig("swim_sim_set_profile", i, vp, i)
    sig("swim_sim_profile_ms", i, vp, vp, sz)
    sig("swim_sim_export_round", i, vp, vp, sz, vp, sz, P(sz), P(sz))
    sig("swim_sim_inject_datagram", i, vp, u32, u32, vp, sz)
    sig("swim_nccl_unique_id", i, vp)
    sig("swim_sim_connect", i, vp, vp)
    sig("swim_sim_ipc_export", i, vp, vp)
    sig("swim_sim_ipc_connect", i, vp, vp)
    for name, args in {
        "swim_get_members": (vp, u32, vp, sz, P(sz)),
        "swim_set_members": (vp, u32, vp, sz),
        "swim_k_random_members": (vp, u32, u32, vp, sz, vp, sz, P(sz)),
        "swim_remove_dead_nodes": (vp, u32),
        "swim_next_seqno": (vp, u32, P(u32)),
        "swim_next_incarnation": (vp, u32, P(u32)),
        "swim_suspect_node": (vp, u32, P(A.Message), P(A.Message), P(i)),
        "swim_dead_node": (vp, u32, P(A.Message), P(A.Message), P(i)),
        "swim_alive_node": (vp, u32, P(A.Message), P(A.Message), P(i)),
        "swim_handle_message": (vp, u32, u32, C.c_uint16, P(A.Message), vp, sz, P(sz)),
        "swim_broadcast": (vp, u32, P(A.Message)),
        "swim_get_broadcasts": (vp, u32, vp, sz, P(sz)),
        "swim_take_broadcasts": (vp, u32, vp, sz, P(sz)),
        "swim_tick_timers": (vp, u32, P(u32)),
        "swim_envelope_encode": (vp, sz, vp, sz, P(sz)),
        "swim_envelope_decode": (vp, sz, vp, sz, P(sz)),
    }.items():
        if hasattr(L, name):
            sig(name, i, *args)
    if L.swim_abi_version() != A.ABI_VERSION:
        raise ImportError("libswim_b200.so ABI version mismatch; rebuild it")
    _lib = L
    return L


def strerror(code):
    return lib().swim_strerror(code).decode()


def check(rc, what, handle=None):
    if rc != 0:
        detail = lib().swim_last_error(handle).decode(errors="replace")
        raise SwimError(rc, what, detail)
