"""Engine.resize_groups against a stub of libmrq (no GPU, no library call): the handle and count the wrapper hands over,
the new G it keeps, the [G] / [R, G] shapes of every array it sizes by G afterwards, and the MrqError mapping (a refused
resize leaves G as it was)."""
import ctypes as C

import numpy as np
import pytest

from raftsql_b200 import _ffi as F
from raftsql_b200.engine import STATE_COLUMNS, Engine, MrqError

G, R = 64, 5


def _count(ptr, dtype, n):
    """a view of n elements behind a ctypes pointer (byref() hands the stub a CArgObject, whose _obj is the struct)"""
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(np.ctypeslib.as_ctypes_type(dtype))), shape=(n,))


class ResizeStub:
    """mrq_resize_groups plus the calls whose host arrays the wrapper sizes by G: each fills exactly G (or R x G) elements,
    so an array of the wrong size shows up as a wrong shape or a short fill"""

    def __init__(self, rc=0):
        self.G, self.rc, self.calls = G, rc, []

    def mrq_resize_groups(self, h, n):
        self.calls.append(("resize", h.value, n))
        if self.rc:
            return self.rc
        self.G = n
        return F.MRQ_OK

    def mrq_export_state(self, h, st):
        st = st._obj
        for k in STATE_COLUMNS:
            p = getattr(st, k)
            if p:
                n = self.G * (R if k in ("match", "votes") else 1)
                _count(p, np.dtype(p._type_), n)[:] = 7
        return F.MRQ_OK

    def mrq_export_next(self, h, p):
        _count(p, np.uint64, R * self.G)[:] = 7
        return F.MRQ_OK

    def mrq_sync_out(self, h, p):
        _count(p, np.uint32, self.G)[:] = 7
        return F.MRQ_OK

    def mrq_sync_commits(self, h, c, r, t):
        for p, dt in ((c, np.uint64), (r, np.uint8), (t, np.uint64)):
            if p:
                _count(p, dt, self.G)[:] = 7
        return F.MRQ_OK

    def mrq_sync_commit_deltas(self, h, p):
        _count(p, np.uint8, self.G)[:] = 7
        return F.MRQ_OK

    def mrq_sync_slot_outputs(self, h, slot, o, d):
        _count(o, np.uint32, self.G)[:] = 7
        _count(d, np.uint8, self.G)[:] = 7
        return F.MRQ_OK

    def mrq_read_inbox(self, h, slot, ib):
        ib = ib._obj
        for k, dt, rows in (("type", np.uint8, R), ("term", np.uint64, R), ("index", np.uint64, R), ("logterm", np.uint64, R),
                            ("commit", np.uint64, R), ("prop_count", np.uint32, 1)):
            _count(getattr(ib, k), dt, rows * self.G)[:] = 7
        return F.MRQ_OK

    def mrq_last_error(self, h):
        return b"stub error"


def make(stub):
    e = Engine.__new__(Engine)
    e.L, e.h, e.G, e.R = stub, C.c_void_p(0x1234), G, R
    e.cfg = F.Config()
    e.cfg.n_groups = G
    return e


def test_the_entry_point_is_declared():
    res, args = F.SIGNATURES["mrq_resize_groups"]
    assert res is C.c_int and args == [C.c_void_p, C.c_uint64]


@pytest.mark.parametrize("n", [G + 1, G + 200, G - 1, 0, 3000])
def test_arrays_follow_the_new_group_count(n):
    stub = ResizeStub()
    e = make(stub)
    e.resize_groups(n)
    assert stub.calls == [("resize", 0x1234, n)]
    assert e.G == n and e.cfg.n_groups == n
    st = e.export_state()
    for k, a in st.items():
        assert a.shape == ((R, n) if k in ("match", "votes") else (n,)), k
        assert (a == 7).all(), k
    assert e.export_next().shape == (R, n)
    assert e.sync_out().shape == (n,)
    c, r, t = e.sync_commits(want_role=True, want_term=True)
    assert c.shape == r.shape == t.shape == (n,)
    assert e.sync_commit_deltas().shape == (n,)
    o, d = e.sync_slot_outputs(1)
    assert o.shape == d.shape == (n,)
    ib = e.read_inbox(0)
    assert ib["type"].shape == (R, n) and ib["prop_count"].shape == (n,)
    for a in (c, r, t, o, d, ib["commit"]):
        assert (a == 7).all()


def test_a_refused_resize_keeps_the_group_count():
    stub = ResizeStub(rc=F.MRQ_E_STATE)
    e = make(stub)
    with pytest.raises(MrqError) as ei:
        e.resize_groups(G * 2)
    assert ei.value.code == F.MRQ_E_STATE and "stub error" in str(ei.value)
    assert e.G == G and e.cfg.n_groups == G
    assert e.sync_out().shape == (G,)
