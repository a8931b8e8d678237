"""Engine — numpy-facing wrapper over the C-ABI (include/mrq.h) for tests, bench.py and the host shim.

One Engine is this node's replica of G raft groups, as one reference process is this node's replica of
one group (reference raft.go:62-78).  Every method maps 1:1 onto an `mrq_*` entry point; nothing here
computes raft arithmetic — that happens in the sm_90a kernels behind the ABI.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _ffi as F


class MrqError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"mrq error {code}: {msg}")
        self.code = code


def _p(a, ty):
    if a is None:
        return None
    assert isinstance(a, np.ndarray) and a.flags["C_CONTIGUOUS"], "need a C-contiguous numpy array"
    return a.ctypes.data_as(ty)


def preset_trace(config_no: int) -> F.TraceParams:
    """Python mirror of include/mrq_trace.h mrq_trace_preset()."""
    p = F.TraceParams()
    p.seed = 0x5EED0000 + config_no
    p.p_ack_256, p.p_grant_256, p.p_reject_256, p.p_heartbeat_256 = 256, 230, 0, 0
    p.churn_65536, p.lagging_pct, p.max_prop, p.lag_kind = 0, 0, 3, 0
    if config_no in (3, 4):
        p.lag_kind = 1
    elif config_no == 5:
        p.p_grant_256, p.p_reject_256, p.churn_65536, p.lagging_pct, p.lag_kind = 205, 26, 43, 20, 1
    return p


STATE_COLUMNS = ("term", "vote", "committed", "last_index", "last_term", "term_start", "match", "role", "lead",
                 "self_id", "votes", "election_elapsed", "heartbeat_elapsed", "randomized_timeout")
_STATE_TYPES = dict(term=F.u64p, vote=F.u64p, committed=F.u64p, last_index=F.u64p, last_term=F.u64p,
                    term_start=F.u64p, match=F.u64p, role=F.u8p, lead=F.u8p, self_id=F.u8p, votes=F.u8p,
                    election_elapsed=F.u16p, heartbeat_elapsed=F.u16p, randomized_timeout=F.u16p)


def empty_state(G: int, R: int) -> dict:
    z64 = lambda *s: np.zeros(s, dtype=np.uint64)
    return dict(term=z64(G), vote=z64(G), committed=z64(G), last_index=z64(G), last_term=z64(G),
                term_start=z64(G), match=z64(R, G), role=np.zeros(G, np.uint8), lead=np.zeros(G, np.uint8),
                self_id=np.zeros(G, np.uint8), votes=np.zeros((R, G), np.uint8),
                election_elapsed=np.zeros(G, np.uint16), heartbeat_elapsed=np.zeros(G, np.uint16),
                randomized_timeout=np.zeros(G, np.uint16))


CHANGE_DTYPE = np.dtype([("tick", np.uint64), ("term", np.uint64), ("term_start", np.uint64), ("group", np.uint32),
                         ("vote", np.uint8), ("role", np.uint8), ("lead", np.uint8), ("what", np.uint8)])  # mrq_change


def empty_inbox(G: int, R: int) -> dict:
    return dict(type=np.zeros((R, G), np.uint8), term=np.zeros((R, G), np.uint64), index=np.zeros((R, G), np.uint64),
                logterm=np.zeros((R, G), np.uint64), commit=np.zeros((R, G), np.uint64),
                prop_count=np.zeros(G, np.uint32))


class Engine:
    def __init__(self, G: int, R: int, *, group_base: int = 0, election_tick: int = 10, heartbeat_tick: int = 1,
                 seed: int = 0, self_id: int = 0, device: int = 0, stream: int | None = None, inbox_slots: int = 2):
        self.L = F.load()
        cfg = F.Config()
        self.L.mrq_config_default(C.byref(cfg))
        cfg.n_replicas, cfg.n_groups, cfg.group_base = R, G, group_base
        cfg.election_tick, cfg.heartbeat_tick, cfg.seed, cfg.self_id = election_tick, heartbeat_tick, seed, self_id
        cfg.device, cfg.stream, cfg.inbox_slots = device, stream, inbox_slots
        h = C.c_void_p()
        rc = self.L.mrq_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise MrqError(rc, (self.L.mrq_last_error(None) or b"").decode())
        self.h = h
        self.G, self.R = int(G), int(R)
        self.cfg = cfg

    # -- lifecycle ---------------------------------------------------------------------------
    def close(self):
        if getattr(self, "h", None):
            self.L.mrq_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _ck(self, rc: int):
        if rc != 0:
            raise MrqError(rc, (self.L.mrq_last_error(self.h) or b"").decode())

    # -- state -----------------------------------------------------------------------------
    def export_state(self, columns=STATE_COLUMNS) -> dict:
        full = empty_state(self.G, self.R)
        st = F.State()
        out = {}
        for k in columns:
            setattr(st, k, _p(full[k], _STATE_TYPES[k]))
            out[k] = full[k]
        self._ck(self.L.mrq_export_state(self.h, C.byref(st)))
        return out

    def import_state(self, s: dict):
        st = F.State()
        keep = []
        for k, ty in _STATE_TYPES.items():
            a = s.get(k)
            if a is not None:
                a = np.ascontiguousarray(a)
                keep.append(a)
                setattr(st, k, _p(a, ty))
        self._ck(self.L.mrq_import_state(self.h, C.byref(st)))

    def export_groups(self, groups, columns=STATE_COLUMNS) -> dict:
        """Rows of the listed local groups (duplicates allowed): arrays of shape [n], and [R, n] for match / votes.
        Row k equals column groups[k] of export_state(); nothing in the engine changes or converts."""
        g = np.ascontiguousarray(groups, dtype=np.uint64).reshape(-1)
        rows = empty_state(len(g), self.R)
        st = F.State()
        out = {}
        for k in columns:
            setattr(st, k, _p(rows[k], _STATE_TYPES[k]))
            out[k] = rows[k]
        self._ck(self.L.mrq_export_groups(self.h, _p(g, F.u64p), len(g), C.byref(st)))
        return out

    def import_groups(self, groups, s: dict):
        """Overwrite the given columns of the listed local groups (no duplicates) with rows shaped as export_groups
        returns them; every other group, including its compact state in tick mode 4, is untouched."""
        g = np.ascontiguousarray(groups, dtype=np.uint64).reshape(-1)
        st = F.State()
        keep = []
        for k, ty in _STATE_TYPES.items():
            a = s.get(k)
            if a is not None:
                dt = np.dtype(ty._type_)
                a = np.ascontiguousarray(a, dtype=dt)
                want = (self.R, len(g)) if k in ("match", "votes") else (len(g),)
                if a.shape != want:
                    raise ValueError(f"{k}: shape {a.shape}, want {want}")
                keep.append(a)
                setattr(st, k, _p(a, ty))
        self._ck(self.L.mrq_import_groups(self.h, _p(g, F.u64p), len(g), C.byref(st)))

    def export_next(self) -> np.ndarray:
        nx = np.zeros((self.R, self.G), np.uint64)
        self._ck(self.L.mrq_export_next(self.h, _p(nx, F.u64p)))
        return nx

    @property
    def tick_count(self) -> int:
        return int(self.L.mrq_tick_count(self.h))

    @tick_count.setter
    def tick_count(self, t: int):
        self._ck(self.L.mrq_set_tick_count(self.h, t))

    # -- inbox -----------------------------------------------------------------------------
    def post_inbox_dense(self, ib: dict, slot: int = 0):
        v = F.Inbox()
        v.type, v.term, v.index = _p(ib.get("type"), F.u8p), _p(ib.get("term"), F.u64p), _p(ib.get("index"), F.u64p)
        v.logterm, v.commit = _p(ib.get("logterm"), F.u64p), _p(ib.get("commit"), F.u64p)
        v.prop_count = _p(ib.get("prop_count"), F.u32p)
        self._ck(self.L.mrq_post_inbox_dense(self.h, slot, C.byref(v)))

    def post_inbox_delta(self, msgs, slot: int = 0, accumulate: bool = False):
        """msgs: iterable of dicts/tuples (group, from, type, term, index, logterm, commit)."""
        arr = (F.Msg * len(msgs))()
        for i, m in enumerate(msgs):
            g, frm, ty, term, index, logterm, commit = m
            arr[i].group, arr[i].from_, arr[i].type = g, frm, ty
            arr[i].term, arr[i].index, arr[i].logterm, arr[i].commit = term, index, logterm, commit
        self._ck(self.L.mrq_post_inbox_delta(self.h, slot, arr, len(msgs), int(accumulate)))

    def post_inbox_packed(self, word: np.ndarray, prop8: np.ndarray | None = None, wide=(), slot: int = 0, keep: bool = False):
        """word: uint32 or uint16 [R][G] (raftsql_b200.packed.pack_inbox / pack_inbox16), or uint8 [R-1][G] (the
        byte form, raftsql_b200.packed.Pack8).  The copy is asynchronous: this convenience wrapper synchronises
        before returning so numpy temporaries are safe; hosts that pipeline call mrq_post_inbox_packed directly
        with pinned buffers (see bench.py)."""
        assert word.dtype in (np.uint32, np.uint16, np.uint8) and word.flags["C_CONTIGUOUS"]
        rows = self.R - 1 if word.dtype == np.uint8 else self.R
        assert word.shape == (rows, self.G), f"word must be [{rows}][{self.G}]"
        v = F.InboxPacked()
        buf = word if word.size else np.zeros(1, np.uint8)  # R = 1 in the byte form: no sender rows at all
        v.word, v.prop_count8 = buf.ctypes.data, _p(prop8, F.u8p)
        v.word_bits = 8 * word.dtype.itemsize
        v.reserved = 1 if bool(keep) else 0  # MRQ_PACKED_KEEP (tick mode 3: the frame stays in its slot after its tick)
        arr = (F.Msg * max(1, len(wide)))()
        for i, m in enumerate(wide):
            g, frm, ty, term, index, logterm, commit = m
            arr[i].group, arr[i].from_, arr[i].type = g, frm, ty
            arr[i].term, arr[i].index, arr[i].logterm, arr[i].commit = term, index, logterm, commit
        v.wide, v.n_wide = arr, len(wide)
        self._ck(self.L.mrq_post_inbox_packed(self.h, slot, C.byref(v)))
        self.synchronize()

    def set_packed_base(self, base_index: np.ndarray | None, base_term: np.ndarray | None):
        self._ck(self.L.mrq_set_packed_base(self.h, _p(base_index, F.u64p), _p(base_term, F.u64p)))

    def propose(self, groups, counts, slot: int = 0):
        g = np.ascontiguousarray(groups, dtype=np.uint64)
        c = np.ascontiguousarray(counts, dtype=np.uint32)
        self._ck(self.L.mrq_propose(self.h, slot, _p(g, F.u64p), _p(c, F.u32p), len(g)))

    def clear_inbox(self, slot: int = 0):
        self._ck(self.L.mrq_clear_inbox(self.h, slot))

    def gen_trace(self, params: F.TraceParams, tick: int, slot: int = 0):
        self._ck(self.L.mrq_gen_trace(self.h, slot, C.byref(params), tick))

    def read_inbox(self, slot: int = 0) -> dict:
        ib = empty_inbox(self.G, self.R)
        v = F.InboxOut()
        v.type, v.term, v.index = _p(ib["type"], F.u8p), _p(ib["term"], F.u64p), _p(ib["index"], F.u64p)
        v.logterm, v.commit, v.prop_count = _p(ib["logterm"], F.u64p), _p(ib["commit"], F.u64p), _p(ib["prop_count"], F.u32p)
        self._ck(self.L.mrq_read_inbox(self.h, slot, C.byref(v)))
        return ib

    # -- hot path --------------------------------------------------------------------------
    def tick(self, slot: int = 0):
        self._ck(self.L.mrq_tick(self.h, slot))

    def tick_many(self, slots):
        s = np.ascontiguousarray(slots, dtype=np.uint32)
        self._ck(self.L.mrq_tick_many(self.h, _p(s, F.u32p), len(s)))

    def set_l2_policy(self, on: int):
        self._ck(self.L.mrq_set_l2_policy(self.h, on))

    def set_graph_mode(self, mode: int):
        self._ck(self.L.mrq_set_graph_mode(self.h, mode))

    def tick_idle(self, n: int = 1):
        self._ck(self.L.mrq_tick_idle(self.h, n))

    def set_tick_mode(self, mode: int):
        self._ck(self.L.mrq_set_tick_mode(self.h, mode))

    def set_write_through(self, on: int):
        self._ck(self.L.mrq_set_write_through(self.h, on))

    def quorum_commit(self):
        self._ck(self.L.mrq_quorum_commit(self.h))

    def set_quorum_variant(self, variant: int):
        self._ck(self.L.mrq_set_quorum_variant(self.h, variant))

    def quorum_commit_ext(self, d_match: int, d_committed: int, d_term_start: int, n_groups: int, stride: int,
                          variant: int = 0):
        self._ck(self.L.mrq_quorum_commit_ext(self.h, d_match, d_committed, d_term_start, n_groups, stride, variant))

    def match_update(self, groups, frm, index):
        g = np.ascontiguousarray(groups, dtype=np.uint64)
        f = np.ascontiguousarray(frm, dtype=np.uint8)
        i = np.ascontiguousarray(index, dtype=np.uint64)
        self._ck(self.L.mrq_match_update(self.h, _p(g, F.u64p), _p(f, F.u8p), _p(i, F.u64p), len(g)))

    # -- outputs ---------------------------------------------------------------------------
    def synchronize(self):
        self._ck(self.L.mrq_synchronize(self.h))

    def sync_commits(self, want_role: bool = False, want_term: bool = False):
        c = np.zeros(self.G, np.uint64)
        r = np.zeros(self.G, np.uint8) if want_role else None
        t = np.zeros(self.G, np.uint64) if want_term else None
        self._ck(self.L.mrq_sync_commits(self.h, _p(c, F.u64p), _p(r, F.u8p), _p(t, F.u64p)))
        return (c, r, t) if (want_role or want_term) else c

    def sync_out(self) -> np.ndarray:
        o = np.zeros(self.G, np.uint32)
        self._ck(self.L.mrq_sync_out(self.h, _p(o, F.u32p)))
        return o

    def sync_commit_deltas(self) -> np.ndarray:
        d = np.zeros(self.G, np.uint8)
        self._ck(self.L.mrq_sync_commit_deltas(self.h, _p(d, F.u8p)))
        return d

    def sync_tick_deltas(self) -> np.ndarray:
        """mode 4: the commit advances of the last tick, as the tick kernels wrote them (1 B per group)"""
        d = np.zeros(self.G, np.uint8)
        self._ck(self.L.mrq_drain_tick_deltas(self.h, _p(d, F.u8p)))
        self._ck(self.L.mrq_drain_wait(self.h))
        self.synchronize()
        return d

    def sync_slot_outputs(self, slot: int):
        """mode 4, after tick_many: (out words, commit advances) of the tick that consumed `slot`"""
        o, d = np.zeros(self.G, np.uint32), np.zeros(self.G, np.uint8)
        self._ck(self.L.mrq_sync_slot_outputs(self.h, slot, _p(o, F.u32p), _p(d, F.u8p)))
        return o, d

    def set_change_capacity(self, n: int):
        """Change feed: record up to n changes of term / vote / role / lead between drains (0 = off).  Discards
        pending records."""
        self._ck(self.L.mrq_set_change_capacity(self.h, n))
        self._change_room = min(int(n), 1 << 16)

    def sync_changes(self):
        """Drain the change feed: (records sorted by (tick, group) as a CHANGE_DTYPE array, lost).  lost > 0 means
        the list is incomplete and the host must read state in full."""
        room = max(1, getattr(self, "_change_room", 1))
        n, lost = C.c_uint64(), C.c_uint64()
        while True:
            buf = np.zeros(room, CHANGE_DTYPE)
            rc = self.L.mrq_sync_changes(self.h, buf.ctypes.data_as(C.POINTER(F.Change)), room, C.byref(n), C.byref(lost))
            if rc == F.MRQ_E_INVAL and n.value > room:  # more records than room: nothing was consumed, retry with enough
                room = int(n.value)
                continue
            self._ck(rc)
            self._change_room = room
            return buf[: n.value], int(lost.value)

    def counters(self) -> dict:
        c = F.Counters()
        self._ck(self.L.mrq_get_counters(self.h, C.byref(c)))
        return {n: int(getattr(c, n)) for n, _ in F.Counters._fields_}

    def timer_start(self):
        self._ck(self.L.mrq_timer_start(self.h))

    def timer_stop(self) -> float:
        ms = C.c_float()
        self._ck(self.L.mrq_timer_stop(self.h, C.byref(ms)))
        return float(ms.value)

    # -- multi-GPU -------------------------------------------------------------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        L = F.load()
        buf = (C.c_uint8 * F.MRQ_COMM_ID_BYTES)()
        rc = L.mrq_comm_unique_id(buf)
        if rc != 0:
            raise MrqError(rc, (L.mrq_last_error(None) or b"").decode())
        return bytes(buf)

    def comm_init(self, uid: bytes, rank: int, world: int):
        buf = (C.c_uint8 * F.MRQ_COMM_ID_BYTES).from_buffer_copy(uid)
        self._ck(self.L.mrq_comm_init(self.h, buf, rank, world))
        self.world, self.rank = world, rank

    def comm_set_mode(self, mode: int):
        self._ck(self.L.mrq_comm_set_mode(self.h, mode))

    def ipc_prepare(self, world: int):
        self._ck(self.L.mrq_ipc_prepare(self.h, world))

    def ipc_export(self) -> bytes:
        buf = (C.c_uint8 * F.MRQ_IPC_HANDLE_BYTES)()
        self._ck(self.L.mrq_ipc_export(self.h, buf))
        return bytes(buf)

    def ipc_attach(self, handles: bytes, rank: int, world: int):
        buf = (C.c_uint8 * len(handles)).from_buffer_copy(handles)
        self._ck(self.L.mrq_ipc_attach(self.h, buf, rank, world))
        self.world, self.rank = world, rank

    def sync_gathered(self) -> np.ndarray:
        w = getattr(self, "world", 1)
        g = np.zeros(w * self.G, np.uint64)
        self._ck(self.L.mrq_sync_gathered(self.h, _p(g, F.u64p)))
        return g

    def device_ptr(self, which: int) -> int:
        return int(self.L.mrq_device_ptr(self.h, which) or 0)

    @property
    def stream(self) -> int:
        return int(self.L.mrq_stream(self.h) or 0)

    @property
    def group_stride(self) -> int:
        return int(self.L.mrq_group_stride(self.h))
