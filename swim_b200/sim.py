"""Bulk simulator front end: N simulated `Store`s (reference Types.hs:53-60) stepped on the GPU.

Replaces the process wiring of `Core.main` (Core.hs:272-287): `Simulator.step(r)` runs r
protocol periods (failureDetector Core.hs:233-241 + handleUDPMessage Core.hs:79-121 +
disseminate Core.hs:127-138) for every node."""
import ctypes as C

import numpy as np

from . import _abi as A
from ._lib import SwimError, check, lib


def default_config(**kw) -> A.Config:
    """parseConfig (Util.hs:44-50) + the simulator knobs; keyword overrides."""
    cfg = A.Config()
    check(lib().swim_config_default(C.byref(cfg)), "swim_config_default")
    for k, v in kw.items():
        if not hasattr(cfg, k):
            raise AttributeError(f"swim_config_t has no field {k}")
        setattr(cfg, k, v)
    return cfg


TOPOLOGIES = {"complete": A.TOPO_COMPLETE, "random": A.TOPO_RANDOM, "ring": A.TOPO_RING, "symmetric": A.TOPO_SYMMETRIC}


def generate_topology(kind, n_nodes, view_cap=32, degree=32, seed=1):
    """Synthetic view graph [N, view_cap] (ids ascending, NO_MEMBER padded). Host only. kind: "complete", "random",
    "ring", "symmetric" (the union of degree / 2 random Hamiltonian cycles: j lists i exactly when i lists j) or a
    SWIM_TOPO_* number."""
    out = np.empty((n_nodes, view_cap), dtype=np.uint32)
    check(lib().swim_topology_generate(TOPOLOGIES.get(kind, kind), n_nodes, view_cap, degree, seed, out.ctypes.data),
          "swim_topology_generate")
    return out


def make_events(rounds, nodes, kinds, msg_kind=None, msg_node=None, msg_inc=None, msg_from=None):
    """Pack an event trace into the swim_event_t layout."""
    n = len(nodes)
    ev = np.zeros(n, dtype=A.EVENT_DTYPE)
    ev["round"] = rounds
    ev["node"] = nodes
    ev["kind"] = kinds
    if msg_kind is not None:
        ev["msg_kind"] = msg_kind
        ev["msg_node"] = msg_node
        ev["msg_incarnation"] = msg_inc
        ev["msg_dead_from"] = 0 if msg_from is None else msg_from
    return ev


def concat_events(parts):
    """np.concatenate drops the padding of the swim_event_t layout; this keeps it."""
    parts = [np.asarray(p) for p in parts]
    out = np.zeros(sum(len(p) for p in parts), dtype=A.EVENT_DTYPE)
    pos = 0
    for p in parts:
        for name in A.EVENT_DTYPE.names:
            out[name][pos:pos + len(p)] = p[name]
        pos += len(p)
    return out


def crash_events(round_, nodes):
    nodes = np.asarray(nodes, dtype=np.uint32)
    return make_events(np.full(len(nodes), round_, np.uint32), nodes, np.full(len(nodes), A.EV_CRASH, np.uint8))


def churn_events(n_nodes, rounds, crash_ppm, rejoin_min=10, rejoin_max=50, seed=1, first_round=1):
    """Seeded churn trace (BASELINE config C5): every round each up node crashes with probability
    crash_ppm/1e6 and rejoins after U[rejoin_min, rejoin_max] rounds (with incarnation + 1 and an Alive
    broadcast — that is what SWIM_EV_REJOIN does). Returns events for rounds first_round..first_round+rounds-1."""
    rng = np.random.default_rng(seed)
    up = np.ones(n_nodes, dtype=bool)
    back_at = np.zeros(n_nodes, dtype=np.int64)
    parts = []
    for r in range(first_round, first_round + rounds):
        rejoin = np.flatnonzero(~up & (back_at == r))
        crash = np.flatnonzero(up & (rng.random(n_nodes) < crash_ppm * 1e-6))
        if len(rejoin):
            parts.append(make_events(np.full(len(rejoin), r, np.uint32), rejoin.astype(np.uint32),
                                     np.full(len(rejoin), A.EV_REJOIN, np.uint8)))
            up[rejoin] = True
        if len(crash):
            parts.append(make_events(np.full(len(crash), r, np.uint32), crash.astype(np.uint32),
                                     np.full(len(crash), A.EV_CRASH, np.uint8)))
            up[crash] = False
            back_at[crash] = r + rng.integers(rejoin_min, rejoin_max + 1, size=len(crash))
    return concat_events(parts) if parts else np.zeros(0, dtype=A.EVENT_DTYPE)


class Simulator:
    def __init__(self, cfg: A.Config = None, **kw):
        self.cfg = cfg if cfg is not None else default_config(**kw)
        h = C.c_void_p()
        self._lib = lib()  # the library that owns the handle also destroys it
        check(self._lib.swim_sim_create(C.byref(self.cfg), C.byref(h)), "swim_sim_create")
        self._h = h
        f, n = C.c_uint32(), C.c_uint32()
        check(lib().swim_sim_local_range(h, C.byref(f), C.byref(n)), "swim_sim_local_range", h)
        self.first, self.n_local = f.value, n.value

    def close(self):
        if getattr(self, "_h", None):
            self._lib.swim_sim_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # ---- bulk path
    def set_view(self, nbr):
        """Install the view graph: the global [N, view_cap] id matrix, as a NumPy array or as a torch CUDA tensor (int32 or
        uint32, contiguous, on the handle's device), which is read in place (swim_sim_set_view_device)."""
        if getattr(nbr, "is_cuda", False):
            import torch
            if nbr.dtype not in (torch.int32, torch.uint32) or not nbr.is_contiguous():
                raise ValueError("a CUDA view matrix must be a contiguous int32 or uint32 tensor")
            if nbr.numel() != self.cfg.n_nodes * self.cfg.view_cap:
                raise ValueError("nbr must be the global [N, view_cap] id matrix")
            if self.cfg.device >= 0 and nbr.device.index != self.cfg.device:
                raise ValueError(f"the view matrix is on {nbr.device}, the handle on cuda:{self.cfg.device}")
            torch.cuda.current_stream(nbr.device).synchronize()  # the handle reads it on its own stream
            check(lib().swim_sim_set_view_device(self._h, nbr.data_ptr()), "swim_sim_set_view_device", self._h)
            return
        nbr = np.ascontiguousarray(nbr, dtype=np.uint32)
        if nbr.size != self.cfg.n_nodes * self.cfg.view_cap:
            raise ValueError("nbr must be the global [N, view_cap] id matrix")
        check(lib().swim_sim_set_view(self._h, nbr.ctypes.data), "swim_sim_set_view", self._h)

    def generate_view(self, kind, degree=32, seed=1):
        """Generate the view graph on the device and install it as set_view does (swim_sim_generate_view): the matrix
        generate_topology(kind, N, view_cap, degree, seed) returns, bit for bit, without a host copy. On a sharded handle
        every rank generates the whole global matrix itself."""
        check(lib().swim_sim_generate_view(self._h, TOPOLOGIES.get(kind, kind), degree, seed), "swim_sim_generate_view",
              self._h)

    def remove_dead_nodes(self, min_age=0):
        """removeDeadNodes (Core.hs:65-67) on every local store: Dead entries at least `min_age` rounds old leave.
        Returns the number removed on this shard; the next step rebuilds the mail graph. On a sharded handle a
        collective: every rank makes the call (the rebuild in the next step is done by all ranks together)."""
        n = C.c_uint64()
        check(lib().swim_sim_remove_dead_nodes(self._h, min_age, C.byref(n)), "swim_sim_remove_dead_nodes", self._h)
        return n.value

    def add_members(self, observers, members, incarnations=0):
        """addNewMember (Core.hs:206-216) for many stores, in the order given: an unlisted member is inserted Alive with
        its incarnation, a listed one is left alone, an add to a full row is dropped. Returns (added, full) of this shard.
        On a sharded handle a collective: every rank is given the same global list and applies its own observers' adds."""
        observers = np.atleast_1d(np.asarray(observers))
        adds = np.zeros(len(observers), dtype=A.MEMBER_ADD_DTYPE)
        adds["observer"] = observers
        adds["member"] = members
        adds["incarnation"] = incarnations
        added, full = C.c_uint64(), C.c_uint64()
        check(lib().swim_sim_add_members(self._h, adds.ctypes.data, len(adds), C.byref(added), C.byref(full)),
              "swim_sim_add_members", self._h)
        return added.value, full.value

    def push_pull(self):
        """Push-pull state exchange (DESIGN.md 2.6) at the current round: every up node swaps its full member state with
        one random Alive member, and each side merges what it receives, inserting the Alive members it did not list.
        Returns (exchanges, inserted, full) of this shard. On a sharded handle a collective: every rank makes the call,
        each on its own host thread or process."""
        e, n, f = C.c_uint64(), C.c_uint64(), C.c_uint64()
        check(lib().swim_sim_push_pull(self._h, C.byref(e), C.byref(n), C.byref(f)), "swim_sim_push_pull", self._h)
        return e.value, n.value, f.value

    def join(self, nodes, seeds, fresh=False):
        """Seed joins (DESIGN.md 2.7) at the current round, memberlist's Join(joinHosts): pair k is one full-state
        exchange between joiner nodes[k] and its join host seeds[k] when both are up, whether or not either lists the
        other; each side merges what it receives as push_pull does. With `fresh` every listed joiner that is up first
        loses its view and piggyback buffer (a restart that lost its state). Returns (exchanges, inserted, full) of this
        shard. On a sharded handle a collective: every rank is given the same global list."""
        nodes = np.atleast_1d(np.asarray(nodes))
        pairs = np.zeros(len(nodes), dtype=A.JOIN_DTYPE)
        pairs["node"] = nodes
        pairs["seed"] = seeds
        e, n, f = C.c_uint64(), C.c_uint64(), C.c_uint64()
        check(lib().swim_sim_join(self._h, pairs.ctypes.data, len(pairs), A.JOIN_FRESH if fresh else 0, C.byref(e),
                                  C.byref(n), C.byref(f)), "swim_sim_join", self._h)
        return e.value, n.value, f.value

    def leave(self, nodes):
        """Graceful leaves (DESIGN.md 2.8) at the current round, memberlist's Leave: every listed process that is up goes
        down as a crash does (and the seeded churn never brings it back), and each member it holds Alive or Suspect that
        is up receives Dead about it, from it, as an injected datagram. Returns (left, delivered) of this shard. On a
        sharded handle a collective: every rank is given the same global list."""
        ids = np.ascontiguousarray(np.atleast_1d(np.asarray(nodes)), dtype=np.uint32)
        lv, dl = C.c_uint64(), C.c_uint64()
        check(lib().swim_sim_leave(self._h, ids.ctypes.data, len(ids), C.byref(lv), C.byref(dl)), "swim_sim_leave",
              self._h)
        return lv.value, dl.value

    def inject(self, events):
        events = np.ascontiguousarray(events, dtype=A.EVENT_DTYPE)
        check(lib().swim_sim_inject(self._h, events.ctypes.data, len(events)), "swim_sim_inject", self._h)

    def step(self, rounds=1):
        check(lib().swim_sim_step(self._h, rounds), "swim_sim_step", self._h)

    def step_async(self, rounds=1):
        check(lib().swim_sim_step_async(self._h, rounds), "swim_sim_step_async", self._h)

    def sync(self):
        check(lib().swim_sim_sync(self._h), "swim_sim_sync", self._h)

    def set_stream(self, cuda_stream):
        check(lib().swim_sim_set_stream(self._h, C.c_void_p(cuda_stream)), "swim_sim_set_stream", self._h)

    def last_step_ms(self):
        ms = C.c_float()
        check(lib().swim_sim_last_step_ms(self._h, C.byref(ms)), "swim_sim_last_step_ms", self._h)
        return ms.value

    @property
    def round(self):
        r = C.c_uint32()
        check(lib().swim_sim_round(self._h, C.byref(r)), "swim_sim_round", self._h)
        return r.value

    def get_array(self, arr):
        nb = C.c_size_t()
        check(lib().swim_sim_array_bytes(self._h, arr, C.byref(nb)), "swim_sim_array_bytes", self._h)
        dt = A.ARRAY_DTYPES[arr]
        out = np.zeros(nb.value // dt.itemsize, dtype=dt)
        check(lib().swim_sim_get_array(self._h, arr, out.ctypes.data, nb.value), "swim_sim_get_array", self._h)
        return out

    def set_array(self, arr, data):
        data = np.ascontiguousarray(data, dtype=A.ARRAY_DTYPES[arr])
        check(lib().swim_sim_set_array(self._h, arr, data.ctypes.data, data.nbytes), "swim_sim_set_array",
              self._h)

    def digest(self):
        d = C.c_uint64()
        check(lib().swim_sim_digest(self._h, C.byref(d)), "swim_sim_digest", self._h)
        return d.value

    def mismatches(self):
        d = C.c_uint64()
        check(lib().swim_sim_mismatches(self._h, C.byref(d)), "swim_sim_mismatches", self._h)
        return d.value

    def counters(self):
        out = np.zeros(A.CTR_COUNT, dtype=np.uint64)
        check(lib().swim_sim_counters(self._h, out.ctypes.data, A.CTR_COUNT), "swim_sim_counters", self._h)
        return out

    def launch_count(self):
        d = C.c_uint64()
        check(lib().swim_sim_launch_count(self._h, C.byref(d)), "swim_sim_launch_count", self._h)
        return d.value

    def set_profile(self, enable=True):
        check(lib().swim_sim_set_profile(self._h, int(enable)), "swim_sim_set_profile", self._h)

    def profile_ms(self):
        """Cumulative per-phase device ms since set_profile(True)."""
        out = (C.c_double * 6)()
        check(lib().swim_sim_profile_ms(self._h, out, 6), "swim_sim_profile_ms", self._h)
        return dict(zip(["events", "tick_scan", "exchange", "recv", "tick_work", "rounds"], list(out)))

    def calibrate(self):
        """Latency calibration of this GPU (swim_sim_calibrate), nanoseconds."""
        out = (C.c_double * 4)()
        check(lib().swim_sim_calibrate(self._h, out, 4), "swim_sim_calibrate", self._h)
        return {"grid_barrier_ns": out[0], "hbm_load_ns": out[1], "l2_load_ns": out[2], "resident_warps": int(out[3])}

    def set_timeline(self, rounds):
        """Record the phase boundaries of the next `rounds` rounds of the fused kernel (0 = off)."""
        check(lib().swim_sim_set_timeline(self._h, rounds), "swim_sim_set_timeline", self._h)

    def timeline(self, rounds):
        """[rounds, 8] uint64 nanosecond stamps (swim_sim_get_timeline); 0 = phase not run."""
        out = np.zeros((rounds, 8), dtype=np.uint64)
        check(lib().swim_sim_get_timeline(self._h, out.ctypes.data, rounds), "swim_sim_get_timeline", self._h)
        return out

    def observe(self, digest=True, mismatches=True):
        """(counters, digest, mismatches) with one device synchronisation; a part that is switched off is not
        computed (its kernel is not launched) and comes back as None."""
        out = np.zeros(A.CTR_COUNT, dtype=np.uint64)
        dg, mm = C.c_uint64(), C.c_uint64()
        check(lib().swim_sim_observe(self._h, out.ctypes.data, A.CTR_COUNT, C.byref(dg) if digest else None,
                                     C.byref(mm) if mismatches else None), "swim_sim_observe", self._h)
        return out, dg.value if digest else None, mm.value if mismatches else None

    def step_observe(self, rounds=1):
        """`rounds` rounds, then (counters, mismatches) — one call, no stream synchronisation (swim_sim_step_observe)."""
        so = getattr(self, "_so", None)
        if so is None:  # the per-round call of a study loop: its argument objects are made once
            buf = (C.c_uint64 * A.CTR_COUNT)()
            mm = C.c_uint64()
            so = self._so = (buf, mm, C.byref(mm), lib().swim_sim_step_observe)
        buf, mm, mm_ref, fn = so
        rc = fn(self._h, rounds, buf, A.CTR_COUNT, mm_ref)
        if rc:
            check(rc, "swim_sim_step_observe", self._h)
        return np.frombuffer(buf, dtype=np.uint64).copy(), mm.value

    def export_round(self):
        """The last round's piggyback envelopes as real datagrams in the reference's wire format:
        [(src, dst, bytes)] — node i is called "n<i>" on the wire (swim_sim_export_round)."""
        nd, nb = C.c_size_t(), C.c_size_t()
        rc = lib().swim_sim_export_round(self._h, None, 0, None, 0, C.byref(nd), C.byref(nb))
        if rc not in (0, A.ECAP):
            check(rc, "swim_sim_export_round", self._h)
        if nd.value == 0:
            return []
        buf = (C.c_uint8 * max(1, nb.value))()
        idx = (A.Datagram * nd.value)()
        check(lib().swim_sim_export_round(self._h, buf, nb.value, idx, nd.value, C.byref(nd), C.byref(nb)),
              "swim_sim_export_round", self._h)
        raw = bytes(buf)
        return [(d.src, d.dst, raw[d.offset:d.offset + d.length]) for d in idx]

    def inject_datagram(self, round_, node, data: bytes):
        """Queue a captured datagram (names "n<id>") for delivery to `node` at `round_`."""
        buf = (C.c_uint8 * max(1, len(data))).from_buffer_copy(data if data else b"\0")
        check(lib().swim_sim_inject_datagram(self._h, round_, node, buf, len(data)), "swim_sim_inject_datagram", self._h)

    def state(self):
        """All bulk arrays as a dict (the checkable form of dumpStore, Util.hs:64-74)."""
        return {A.ARRAY_NAMES[a]: self.get_array(a) for a in range(A.ARR_COUNT)}

    def set_round(self, r):
        check(lib().swim_sim_set_round(self._h, r), "swim_sim_set_round", self._h)

    def save(self):
        """Device-resident checkpoint (swim_sim_save): state, counters, round and pending events, no host traffic."""
        check(lib().swim_sim_save(self._h), "swim_sim_save", self._h)

    def load(self):
        """Back to the last save() (swim_sim_load)."""
        check(lib().swim_sim_load(self._h), "swim_sim_load", self._h)

    def set_params(self, **kw):
        """Change protocol scalars of the live handle between steps (swim_sim_set_params): suspicion_rounds, suspicion_max,
        retransmit, loss_ppm, flags, churn_ppm, rejoin_min, rejoin_max, seed."""
        cfg = A.Config.from_buffer_copy(self.cfg)
        for k, v in kw.items():
            setattr(cfg, k, v)
        check(lib().swim_sim_set_params(self._h, C.byref(cfg)), "swim_sim_set_params", self._h)
        self.cfg = cfg

    def checkpoint(self):
        """Everything a single-shard run needs to be resumed bit for bit: the state arrays and the round (the counter of
        every Philox draw). Pending events and the config are the caller's (they are inputs, not state)."""
        ck = self.state()
        ck["round"] = self.round
        return ck

    def restore(self, ck):
        """Put a FRESH single-shard handle (same config) into a checkpointed state."""
        if self.cfg.world != 1:
            raise ValueError("restore() takes the global view matrix: single-shard handles only")
        by_name = {v: k for k, v in A.ARRAY_NAMES.items()}
        self.set_view(ck["nbr"].reshape(self.cfg.n_nodes, self.cfg.view_cap))
        for name, data in ck.items():
            if name not in ("nbr", "round"):
                self.set_array(by_name[name], data)
        self.set_round(int(ck["round"]))

    # ---- multi-GPU
    def connect(self, unique_id: bytes):
        """Staged exchange: join the NCCL communicator (swim_sim_connect)."""
        buf = (C.c_uint8 * A.NCCL_ID_BYTES).from_buffer_copy(unique_id)
        check(lib().swim_sim_connect(self._h, buf), "swim_sim_connect", self._h)

    def ipc_export(self) -> bytes:
        buf = (C.c_uint8 * A.IPC_BLOB_BYTES)()
        check(lib().swim_sim_ipc_export(self._h, buf), "swim_sim_ipc_export", self._h)
        return bytes(buf)

    def ipc_connect(self, blobs):
        """Fused exchange over peer memory: blobs = every rank's ipc_export(), in rank order."""
        raw = b"".join(blobs)
        buf = (C.c_uint8 * len(raw)).from_buffer_copy(raw)
        check(lib().swim_sim_ipc_connect(self._h, buf), "swim_sim_ipc_connect", self._h)


def nccl_unique_id() -> bytes:
    buf = (C.c_uint8 * A.NCCL_ID_BYTES)()
    check(lib().swim_nccl_unique_id(buf), "swim_nccl_unique_id")
    return bytes(buf)
