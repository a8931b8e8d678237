"""ctypes binding of include/mrq.h (the C-ABI of libmrq.so).

This is exactly the binding a non-Python host would write (see INTEGRATION.md for the cgo form):
plain pointers and sizes, no torch types.  The library is built in-tree by `make` /
`__graft_entry__.build()`; if it is missing the import fails loudly — there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MRQ_LIB_PATH") or os.path.join(_HERE, "libmrq.so")  # (MRQ_LIB_PATH: development builds of the same ABI)

MRQ_ABI_VERSION = 1
MRQ_MAX_REPLICAS = 8
MRQ_COMM_ID_BYTES = 128
MRQ_IPC_HANDLE_BYTES = 64

# error codes
MRQ_OK, MRQ_E_INVAL, MRQ_E_CUDA, MRQ_E_NOMEM, MRQ_E_STATE, MRQ_E_NCCL, MRQ_E_NODEVICE = 0, -1, -2, -3, -4, -5, -6

ROLE_FOLLOWER, ROLE_CANDIDATE, ROLE_LEADER = 0, 1, 2

MSG_NONE, MSG_APP, MSG_APP_RESP, MSG_VOTE, MSG_VOTE_RESP, MSG_HEARTBEAT, MSG_HEARTBEAT_RESP = 0, 3, 4, 5, 6, 8, 9
MSG_TYPE_MASK, MSG_REJECT = 0x0F, 0x80

OUT_CAMPAIGN, OUT_BECAME_LEADER, OUT_BCAST_APPEND, OUT_BCAST_HEARTBEAT = 0x01, 0x02, 0x04, 0x08
OUT_STEPPED_DOWN, OUT_PROP_DROPPED, OUT_PROP_FORWARD, OUT_COMMIT_ADVANCED = 0x10, 0x20, 0x40, 0x80
OUT_VOTE_REPLY_SHIFT, OUT_ACK_REPLY_SHIFT = 8, 24

PTR_TERM, PTR_META, PTR_LAST_INDEX, PTR_LAST_TERM, PTR_COMMITTED, PTR_TERM_START, PTR_MATCH, PTR_OUT, PTR_GATHERED = range(9)

u8p = C.POINTER(C.c_uint8)
u16p = C.POINTER(C.c_uint16)
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)


class Config(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32),
        ("n_replicas", C.c_uint32),
        ("n_groups", C.c_uint64),
        ("group_base", C.c_uint64),
        ("election_tick", C.c_uint32),
        ("heartbeat_tick", C.c_uint32),
        ("seed", C.c_uint64),
        ("self_id", C.c_uint32),
        ("device", C.c_int32),
        ("stream", C.c_void_p),
        ("inbox_slots", C.c_uint32),
        ("flags", C.c_uint32),
    ]


class State(C.Structure):
    _fields_ = [
        ("term", u64p), ("vote", u64p), ("committed", u64p), ("last_index", u64p), ("last_term", u64p),
        ("term_start", u64p), ("match", u64p), ("role", u8p), ("lead", u8p), ("self_id", u8p), ("votes", u8p),
        ("election_elapsed", u16p), ("heartbeat_elapsed", u16p), ("randomized_timeout", u16p),
    ]


class Inbox(C.Structure):
    _fields_ = [("type", u8p), ("term", u64p), ("index", u64p), ("logterm", u64p), ("commit", u64p),
                ("prop_count", u32p)]


class InboxOut(C.Structure):
    _fields_ = Inbox._fields_


class Msg(C.Structure):
    _fields_ = [("group", C.c_uint64), ("term", C.c_uint64), ("index", C.c_uint64), ("logterm", C.c_uint64),
                ("commit", C.c_uint64), ("type", C.c_uint8), ("from_", C.c_uint8), ("pad", C.c_uint8 * 6)]


class InboxPacked(C.Structure):
    _fields_ = [("word", C.c_void_p), ("prop_count8", u8p), ("wide", C.POINTER(Msg)), ("n_wide", C.c_size_t),
                ("word_bits", C.c_uint32), ("reserved", C.c_uint32)]


class TraceParams(C.Structure):
    """include/mrq_trace.h `mrq_trace_params`."""

    _fields_ = [("seed", C.c_uint64), ("p_ack_256", C.c_uint32), ("p_grant_256", C.c_uint32),
                ("p_reject_256", C.c_uint32), ("p_heartbeat_256", C.c_uint32), ("churn_65536", C.c_uint32),
                ("lagging_pct", C.c_uint32), ("max_prop", C.c_uint32), ("lag_kind", C.c_uint32)]


CHANGE_TERM, CHANGE_VOTE, CHANGE_ROLE, CHANGE_LEAD = 0x01, 0x02, 0x04, 0x08


class Change(C.Structure):
    """include/mrq.h `mrq_change`: one change-feed record (32 bytes)."""

    _fields_ = [("tick", C.c_uint64), ("term", C.c_uint64), ("term_start", C.c_uint64), ("group", C.c_uint32),
                ("vote", C.c_uint8), ("role", C.c_uint8), ("lead", C.c_uint8), ("what", C.c_uint8)]


class Counters(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("ticks", "kernel_launches", "campaigns", "elections_won", "step_downs",
                                          "commits_advanced", "votes_granted", "errors")]


# name -> (restype, argtypes); every function include/mrq.h declares
_EP = C.c_void_p
SIGNATURES = {
    "mrq_version": (C.c_uint32, [u32p]),
    "mrq_config_default": (None, [C.POINTER(Config)]),
    "mrq_create": (C.c_int, [C.POINTER(Config), C.POINTER(_EP)]),
    "mrq_destroy": (None, [_EP]),
    "mrq_last_error": (C.c_char_p, [_EP]),
    "mrq_export_state": (C.c_int, [_EP, C.POINTER(State)]),
    "mrq_import_state": (C.c_int, [_EP, C.POINTER(State)]),
    "mrq_export_groups": (C.c_int, [_EP, u64p, C.c_uint64, C.POINTER(State)]),
    "mrq_import_groups": (C.c_int, [_EP, u64p, C.c_uint64, C.POINTER(State)]),
    "mrq_export_next": (C.c_int, [_EP, u64p]),
    "mrq_tick_count": (C.c_uint64, [_EP]),
    "mrq_set_tick_count": (C.c_int, [_EP, C.c_uint64]),
    "mrq_post_inbox_dense": (C.c_int, [_EP, C.c_uint32, C.POINTER(Inbox)]),
    "mrq_post_inbox_delta": (C.c_int, [_EP, C.c_uint32, C.POINTER(Msg), C.c_size_t, C.c_int]),
    "mrq_post_inbox_packed": (C.c_int, [_EP, C.c_uint32, C.POINTER(InboxPacked)]),
    "mrq_set_packed_base": (C.c_int, [_EP, u64p, u64p]),
    "mrq_pack8": (C.c_int, [C.POINTER(Inbox), u8p, C.c_uint64, C.c_uint32, u64p, u64p, u8p, u8p, C.POINTER(Msg), C.c_size_t,
                            C.POINTER(C.c_size_t)]),
    "mrq_unpack8": (C.c_int, [u8p, u8p, C.c_uint64, C.c_uint32, u64p, u64p, C.POINTER(InboxOut)]),
    "mrq_propose": (C.c_int, [_EP, C.c_uint32, u64p, u32p, C.c_size_t]),
    "mrq_clear_inbox": (C.c_int, [_EP, C.c_uint32]),
    "mrq_tick": (C.c_int, [_EP, C.c_uint32]),
    "mrq_tick_many": (C.c_int, [_EP, u32p, C.c_uint32]),
    "mrq_set_graph_mode": (C.c_int, [_EP, C.c_int]),
    "mrq_set_l2_policy": (C.c_int, [_EP, C.c_int]),
    "mrq_tick_idle": (C.c_int, [_EP, C.c_uint32]),
    "mrq_set_tick_mode": (C.c_int, [_EP, C.c_int]),
    "mrq_quorum_commit": (C.c_int, [_EP]),
    "mrq_set_quorum_variant": (C.c_int, [_EP, C.c_int]),
    "mrq_quorum_commit_ext": (C.c_int, [_EP, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_int]),
    "mrq_match_update": (C.c_int, [_EP, u64p, u8p, u64p, C.c_size_t]),
    "mrq_sync_commits": (C.c_int, [_EP, u64p, u8p, u64p]),
    "mrq_sync_out": (C.c_int, [_EP, u32p]),
    "mrq_sync_commit_deltas": (C.c_int, [_EP, u8p]),
    "mrq_drain_commit_deltas": (C.c_int, [_EP, u8p]),
    "mrq_drain_wait": (C.c_int, [_EP]),
    "mrq_drain_tick_deltas": (C.c_int, [_EP, u8p]),
    "mrq_set_write_through": (C.c_int, [_EP, C.c_int]),
    "mrq_sync_slot_outputs": (C.c_int, [_EP, C.c_uint32, u32p, u8p]),
    "mrq_synchronize": (C.c_int, [_EP]),
    "mrq_set_change_capacity": (C.c_int, [_EP, C.c_uint64]),
    "mrq_sync_changes": (C.c_int, [_EP, C.POINTER(Change), C.c_uint64, u64p, u64p]),
    "mrq_gen_trace": (C.c_int, [_EP, C.c_uint32, C.POINTER(TraceParams), C.c_uint64]),
    "mrq_read_inbox": (C.c_int, [_EP, C.c_uint32, C.POINTER(InboxOut)]),
    "mrq_get_counters": (C.c_int, [_EP, C.POINTER(Counters)]),
    "mrq_timer_start": (C.c_int, [_EP]),
    "mrq_timer_stop": (C.c_int, [_EP, C.POINTER(C.c_float)]),
    "mrq_comm_unique_id": (C.c_int, [u8p]),
    "mrq_comm_init": (C.c_int, [_EP, u8p, C.c_uint32, C.c_uint32]),
    "mrq_comm_set_mode": (C.c_int, [_EP, C.c_uint32]),
    "mrq_sync_gathered": (C.c_int, [_EP, u64p]),
    "mrq_ipc_prepare": (C.c_int, [_EP, C.c_uint32]),
    "mrq_ipc_export": (C.c_int, [_EP, u8p]),
    "mrq_ipc_attach": (C.c_int, [_EP, u8p, C.c_uint32, C.c_uint32]),
    "mrq_device_ptr": (C.c_void_p, [_EP, C.c_int]),
    "mrq_stream": (C.c_void_p, [_EP]),
    "mrq_group_stride": (C.c_uint64, [_EP]),
    "mrq_alloc_pinned": (C.c_void_p, [C.c_size_t]),
    "mrq_free_pinned": (None, [C.c_void_p]),
}

_lib = None


class MrqLibraryMissing(ImportError):
    pass


def load() -> C.CDLL:
    """dlopen raftsql_b200/libmrq.so and type every entry point.  Fails loudly if it was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MrqLibraryMissing(
            f"{LIB_PATH} not found: build it with `make` (or `python -c 'import __graft_entry__ as g; g.build()'`). "
            "raftsql_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(L, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L
