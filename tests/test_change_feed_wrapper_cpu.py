"""Engine.set_change_capacity / Engine.sync_changes against a stub of libmrq (no GPU, no library call): the record
layout, the numpy dtype, `lost`, and the retry when more records are pending than the buffer holds."""
import ctypes as C

import numpy as np
import pytest

from raftsql_b200 import _ffi as F
from raftsql_b200.engine import CHANGE_DTYPE, Engine, MrqError


class FeedStub:
    """mrq_set_change_capacity / mrq_sync_changes over a host list of pending records"""

    def __init__(self, pending, lost=0, rc=0):
        self.pending, self.lost, self.rc, self.calls = list(pending), lost, rc, []

    def mrq_set_change_capacity(self, h, n):
        self.calls.append(("set", n))
        return self.rc

    def mrq_sync_changes(self, h, out, cap, n_out, lost):
        self.calls.append(("sync", cap))
        if self.rc:
            return self.rc
        n_out._obj.value = len(self.pending)
        if cap < len(self.pending):
            return F.MRQ_E_INVAL
        for k, rec in enumerate(self.pending):
            out[k] = rec
        lost._obj.value = self.lost
        self.pending = []
        return F.MRQ_OK

    def mrq_last_error(self, h):
        return b"stub error"


def rec(tick, group, what, term=3, term_start=2**64 - 1, vote=2, role=0, lead=2):
    c = F.Change()
    c.tick, c.group, c.what, c.term, c.term_start, c.vote, c.role, c.lead = tick, group, what, term, term_start, vote, role, lead
    return c


def make(stub):
    e = Engine.__new__(Engine)
    e.L, e.h, e.G, e.R = stub, C.c_void_p(0x1234), 64, 5
    return e


def test_record_layout_matches_the_header():
    assert C.sizeof(F.Change) == 32
    assert CHANGE_DTYPE.itemsize == 32
    for name, _ in F.Change._fields_:
        assert CHANGE_DTYPE.fields[name][1] == getattr(F.Change, name).offset, name
    assert (F.CHANGE_TERM, F.CHANGE_VOTE, F.CHANGE_ROLE, F.CHANGE_LEAD) == (1, 2, 4, 8)
    assert "mrq_set_change_capacity" in F.SIGNATURES and "mrq_sync_changes" in F.SIGNATURES


def test_sync_changes_returns_the_records_as_a_structured_array():
    pending = [rec(7, 3, F.CHANGE_TERM | F.CHANGE_VOTE, term=9, vote=4),
               rec(7, 40, F.CHANGE_ROLE | F.CHANGE_LEAD, role=2, lead=1, term_start=123)]
    stub = FeedStub(pending, lost=5)
    e = make(stub)
    e.set_change_capacity(1000)
    assert stub.calls[-1] == ("set", 1000)
    recs, lost = e.sync_changes()
    assert recs.dtype == CHANGE_DTYPE and len(recs) == 2 and lost == 5
    assert (int(recs[0]["tick"]), int(recs[0]["group"]), int(recs[0]["term"]), int(recs[0]["vote"])) == (7, 3, 9, 4)
    assert int(recs[0]["what"]) == F.CHANGE_TERM | F.CHANGE_VOTE and int(recs[0]["term_start"]) == 2**64 - 1
    assert (int(recs[1]["role"]), int(recs[1]["lead"]), int(recs[1]["term_start"])) == (2, 1, 123)


def test_sync_changes_retries_with_room_for_every_pending_record():
    pending = [rec(t, g, F.CHANGE_TERM) for t in range(3) for g in range(9)]
    stub = FeedStub(pending)
    e = make(stub)
    e._change_room = 4  # smaller than what is pending: the first call consumes nothing and says how much is needed
    recs, lost = e.sync_changes()
    assert [c for c in stub.calls if c[0] == "sync"] == [("sync", 4), ("sync", 27)]
    assert len(recs) == 27 and lost == 0
    assert [(int(r["tick"]), int(r["group"])) for r in recs] == [(t, g) for t in range(3) for g in range(9)]
    recs, lost = e.sync_changes()  # drained: nothing left
    assert len(recs) == 0 and lost == 0


def test_feed_off_raises_the_library_error():
    e = make(FeedStub([], rc=F.MRQ_E_STATE))
    with pytest.raises(MrqError) as ei:
        e.sync_changes()
    assert ei.value.code == F.MRQ_E_STATE and "stub error" in str(ei.value)
