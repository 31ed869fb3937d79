"""ctypes mirror of include/swim.h (the C ABI). Field order and widths must match the header;
tests/test_abi.py checks sizeof/offsets against a compiled probe."""
import ctypes as C

ABI_VERSION = 2

# error codes
OK, EINVAL, ENOMEM, ECUDA, ERANGE, EDECODE, ENODEV, ENCCL, ECAP, ESTATE = 0, -1, -2, -3, -4, -5, -6, -7, -8, -9

# Liveness (Types.hs:76-77)
ALIVE, SUSPECT, DEAD, VACANT = 0, 1, 2, 3
# MsgType (Types.hs:159-167)
MSG_PING, MSG_INDIRECT_PING, MSG_ACK, MSG_SUSPECT, MSG_ALIVE, MSG_DEAD, MSG_COMPOUND = range(7)
NO_MEMBER = 0xFFFFFFFF
MAX_K, MAX_PB, MAX_TIMER, MAX_VIEW = 7, 32, 63, 256
ACK_PAYLOAD_MAX = 16
NAME_MAX = 255
NCCL_ID_BYTES = 128
IPC_BLOB_BYTES = 1024

EV_CRASH, EV_REJOIN, EV_INJECT = 0, 1, 2
F_NONE, F_STRICT_OVERRIDE, F_ROUND_ROBIN = 0, 1, 2  # SWIM_F_*: protocol variants
TOPO_COMPLETE, TOPO_RANDOM, TOPO_RING, TOPO_SYMMETRIC = 0, 1, 2, 3
JOIN_FRESH = 1  # SWIM_JOIN_FRESH: swim_sim_join empties the joiners first

(ARR_ALIVE, ARR_SELF_INC, ARR_SEQNO, ARR_NBR, ARR_VST, ARR_VINC, ARR_VLAST, ARR_PB, ARR_PB_CNT, ARR_BACK_AT,
 ARR_LAST_CRASH, ARR_LAST_REJOIN) = range(12)
ARR_COUNT = 12
REPLICATED_ARRAYS = (ARR_ALIVE, ARR_BACK_AT, ARR_LAST_CRASH, ARR_LAST_REJOIN)  # [N] on every rank; the others are per shard
(CTR_PINGS, CTR_DIRECT_FAIL, CTR_INDIRECT_PINGS, CTR_SUSPECT_LOCAL, CTR_DEAD_TIMEOUT, CTR_MSGS,
 CTR_RECS_SENT, CTR_RECS_APPLIED, CTR_REFUTES, CTR_PB_DROPPED, CTR_MSGS_RECV) = range(11)
CTR_COUNT = 11
CTR_NAMES = ["pings", "direct_fail", "indirect_pings", "suspect_local", "dead_timeout", "msgs",
             "recs_sent", "recs_applied", "refutes", "pb_dropped", "msgs_recv"]


class Config(C.Structure):
    _fields_ = [("abi_version", C.c_uint32), ("n_nodes", C.c_uint32), ("view_cap", C.c_uint32),
                ("k_indirect", C.c_uint32), ("fanout", C.c_uint32), ("pb_cap", C.c_uint32),
                ("suspicion_rounds", C.c_uint32), ("retransmit", C.c_uint32), ("loss_ppm", C.c_uint32),
                ("flags", C.c_uint32), ("seed", C.c_uint64), ("rank", C.c_uint32), ("world", C.c_uint32),
                ("device", C.c_int32), ("base_port", C.c_uint32), ("churn_ppm", C.c_uint32),
                ("rejoin_min", C.c_uint32), ("rejoin_max", C.c_uint32), ("probes_per_round", C.c_uint32),
                ("suspicion_max", C.c_uint32), ("_reserved", C.c_uint32)]


class Member(C.Structure):
    _fields_ = [("id", C.c_uint32), ("addr", C.c_uint32), ("port", C.c_uint16), ("liveness", C.c_uint8),
                ("timer", C.c_uint8), ("incarnation", C.c_uint32), ("last_change", C.c_uint64)]


class Message(C.Structure):
    _fields_ = [("kind", C.c_uint8), ("payload_len", C.c_uint8), ("port", C.c_uint16), ("seq_no", C.c_uint32),
                ("node", C.c_uint32), ("target", C.c_uint32), ("incarnation", C.c_int64),
                ("dead_from", C.c_uint32), ("payload", C.c_uint8 * ACK_PAYLOAD_MAX), ("_pad", C.c_uint32)]


class Gossip(C.Structure):
    _fields_ = [("is_direct", C.c_uint8), ("_pad", C.c_uint8), ("dest_port", C.c_uint16),
                ("dest_addr", C.c_uint32), ("msg", Message)]


class Record(C.Structure):
    _fields_ = [("member", C.c_uint32), ("incarnation", C.c_uint32), ("from_", C.c_uint32),
                ("kind", C.c_uint8), ("ttl", C.c_uint8), ("_pad", C.c_uint16)]


class Event(C.Structure):
    _fields_ = [("round", C.c_uint32), ("node", C.c_uint32), ("kind", C.c_uint8), ("_pad", C.c_uint8 * 7),
                ("msg", Message)]


class MemberAdd(C.Structure):
    _fields_ = [("observer", C.c_uint32), ("member", C.c_uint32), ("incarnation", C.c_uint32), ("_pad", C.c_uint32)]


class Join(C.Structure):
    _fields_ = [("node", C.c_uint32), ("seed", C.c_uint32)]


class Datagram(C.Structure):
    _fields_ = [("src", C.c_uint32), ("dst", C.c_uint32), ("length", C.c_uint32), ("n_messages", C.c_uint32),
                ("offset", C.c_uint64)]


class WireMessage(C.Structure):
    _fields_ = [("kind", C.c_uint8), ("payload_len", C.c_uint8), ("port", C.c_uint16), ("seq_no", C.c_uint32),
                ("target", C.c_uint32), ("incarnation", C.c_int64), ("payload", C.c_uint8 * ACK_PAYLOAD_MAX),
                ("node", C.c_char * (NAME_MAX + 1)), ("dead_from", C.c_char * (NAME_MAX + 1))]


# numpy dtypes of the bulk arrays (SWIM_ARR_*): (dtype, elements per node as f(cap, B))
import numpy as _np

RECORD_DTYPE = _np.dtype([("member", "<u4"), ("incarnation", "<u4"), ("from", "<u4"), ("kind", "u1"),
                          ("ttl", "u1"), ("_pad", "<u2")])
EVENT_DTYPE = _np.dtype({"names": ["round", "node", "kind", "msg_kind", "msg_node", "msg_incarnation",
                                   "msg_dead_from"],
                         "formats": ["<u4", "<u4", "u1", "u1", "<u4", "<i8", "<u4"],
                         "offsets": [0, 4, 8, 16, 24, 32, 40],
                         "itemsize": C.sizeof(Event)})
MEMBER_ADD_DTYPE = _np.dtype([("observer", "<u4"), ("member", "<u4"), ("incarnation", "<u4"), ("_pad", "<u4")])
JOIN_DTYPE = _np.dtype([("node", "<u4"), ("seed", "<u4")])
ARRAY_DTYPES = {
    ARR_ALIVE: _np.dtype("u1"), ARR_SELF_INC: _np.dtype("<u4"), ARR_SEQNO: _np.dtype("<u4"),
    ARR_NBR: _np.dtype("<u4"), ARR_VST: _np.dtype("u1"), ARR_VINC: _np.dtype("<u4"),
    ARR_VLAST: _np.dtype("<u4"), ARR_PB: RECORD_DTYPE, ARR_PB_CNT: _np.dtype("u1"), ARR_BACK_AT: _np.dtype("<u4"),
    ARR_LAST_CRASH: _np.dtype("<u4"), ARR_LAST_REJOIN: _np.dtype("<u4"),
}
ARRAY_NAMES = {ARR_ALIVE: "alive", ARR_SELF_INC: "self_inc", ARR_SEQNO: "seqno", ARR_NBR: "nbr",
               ARR_VST: "vst", ARR_VINC: "vinc", ARR_VLAST: "vlast", ARR_PB: "pb", ARR_PB_CNT: "pb_cnt",
               ARR_BACK_AT: "back_at", ARR_LAST_CRASH: "last_crash", ARR_LAST_REJOIN: "last_rejoin"}
