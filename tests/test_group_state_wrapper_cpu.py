"""Engine.export_groups / Engine.import_groups against a stub of libmrq (no GPU, no library call): the group list and
row arrays the wrapper hands over, the [n] / [R, n] shapes and dtypes, column subsets, n == 0, and the MrqError
mapping."""
import ctypes as C

import numpy as np
import pytest

from raftsql_b200 import _ffi as F
from raftsql_b200.engine import STATE_COLUMNS, Engine, MrqError

G, R = 64, 5
_DT = dict(term=np.uint64, vote=np.uint64, committed=np.uint64, last_index=np.uint64, last_term=np.uint64,
           term_start=np.uint64, match=np.uint64, role=np.uint8, lead=np.uint8, self_id=np.uint8, votes=np.uint8,
           election_elapsed=np.uint16, heartbeat_elapsed=np.uint16, randomized_timeout=np.uint16)
_PER_REPLICA = ("match", "votes")


def _view(ptr, dtype, count):
    if not ptr or count == 0:
        return None
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(np.ctypeslib.as_ctypes_type(dtype))), shape=(count,))


class GroupsStub:
    """mrq_export_groups / mrq_import_groups over a host copy of G groups' state (engine column layout [R][G])"""

    def __init__(self, rc=0):
        rng = np.random.default_rng(7)
        self.state = {k: rng.integers(0, 200, size=(R, G) if k in _PER_REPLICA else (G,)).astype(dt) for k, dt in _DT.items()}
        self.rc, self.calls = rc, []

    def _rows(self, k):
        return R if k in _PER_REPLICA else 1

    def mrq_export_groups(self, h, groups, n, st):
        st = st._obj
        got = [k for k in _DT if getattr(st, k)]
        self.calls.append(("export", n, got))
        if self.rc or n == 0:
            return self.rc
        g = _view(groups, np.uint64, n)
        for k in got:
            dst = _view(getattr(st, k), _DT[k], n * self._rows(k)).reshape(self._rows(k), n)
            src = self.state[k].reshape(self._rows(k), G)
            dst[:] = src[:, g.astype(np.int64)]
        return F.MRQ_OK

    def mrq_import_groups(self, h, groups, n, st):
        st = st._obj
        got = [k for k in _DT if getattr(st, k)]
        self.calls.append(("import", n, got))
        if self.rc or n == 0:
            return self.rc
        g = _view(groups, np.uint64, n)
        for k in got:
            src = _view(getattr(st, k), _DT[k], n * self._rows(k)).reshape(self._rows(k), n)
            self.state[k].reshape(self._rows(k), G)[:, g.astype(np.int64)] = src
        return F.MRQ_OK

    def mrq_last_error(self, h):
        return b"stub error"


def make(stub):
    e = Engine.__new__(Engine)
    e.L, e.h, e.G, e.R = stub, C.c_void_p(0x1234), G, R
    return e


def test_the_entry_points_are_declared():
    for name in ("mrq_export_groups", "mrq_import_groups"):
        res, args = F.SIGNATURES[name]
        assert res is C.c_int and args[1] is F.u64p and args[2] is C.c_uint64 and args[3] is C.POINTER(F.State)


def test_export_groups_returns_rows_of_the_listed_groups():
    stub = GroupsStub()
    e = make(stub)
    groups = [0, 63, 5, 5, 17]  # first, last, a duplicate
    rows = e.export_groups(groups)
    assert set(rows) == set(STATE_COLUMNS)
    for k, a in rows.items():
        assert a.dtype == _DT[k], k
        assert a.shape == ((R, len(groups)) if k in _PER_REPLICA else (len(groups),)), k
        want = stub.state[k][..., groups]
        np.testing.assert_array_equal(a, want, err_msg=k)
    assert stub.calls == [("export", 5, list(_DT))]


def test_export_groups_column_subset_passes_null_for_the_others():
    stub = GroupsStub()
    e = make(stub)
    rows = e.export_groups(np.array([3, 9], np.int64), columns=("committed", "match"))
    assert set(rows) == {"committed", "match"}
    assert rows["match"].shape == (R, 2)
    assert stub.calls[-1] == ("export", 2, ["committed", "match"])


def test_import_groups_writes_rows_and_converts_dtypes():
    stub = GroupsStub()
    e = make(stub)
    groups = [2, 40, 63]
    before = {k: v.copy() for k, v in stub.state.items()}
    e.import_groups(groups, dict(term=[11, 12, 13], match=np.full((R, 3), 99, np.int64), role=np.array([2, 0, 1])))
    assert stub.calls[-1] == ("import", 3, ["term", "match", "role"])
    np.testing.assert_array_equal(stub.state["term"][groups], [11, 12, 13])
    np.testing.assert_array_equal(stub.state["match"][:, groups], np.full((R, 3), 99))
    np.testing.assert_array_equal(stub.state["role"][groups], [2, 0, 1])
    others = [g for g in range(G) if g not in groups]
    for k in _DT:
        np.testing.assert_array_equal(stub.state[k][..., others], before[k][..., others], err_msg=k)
    np.testing.assert_array_equal(stub.state["vote"], before["vote"])


def test_import_groups_round_trips_export_groups():
    stub = GroupsStub()
    e = make(stub)
    rows = e.export_groups([4, 8])
    for k in rows:
        rows[k] = rows[k] + 1
    e.import_groups([8, 4], {k: v[..., ::-1] for k, v in rows.items()})
    again = e.export_groups([4, 8])
    for k in rows:
        np.testing.assert_array_equal(again[k], rows[k], err_msg=k)


def test_import_groups_rejects_a_wrong_shape_before_the_call():
    stub = GroupsStub()
    e = make(stub)
    with pytest.raises(ValueError):
        e.import_groups([1, 2], dict(match=np.zeros((R, 3), np.uint64)))
    with pytest.raises(ValueError):
        e.import_groups([1, 2], dict(term=np.zeros(3, np.uint64)))
    assert stub.calls == []


def test_empty_list():
    stub = GroupsStub()
    e = make(stub)
    rows = e.export_groups([])
    assert rows["term"].shape == (0,) and rows["votes"].shape == (R, 0)
    e.import_groups([], dict(term=np.zeros(0, np.uint64)))
    assert [c[:2] for c in stub.calls] == [("export", 0), ("import", 0)]


@pytest.mark.parametrize("call", ["export", "import"])
def test_errors_raise_mrq_error(call):
    e = make(GroupsStub(rc=F.MRQ_E_INVAL))
    with pytest.raises(MrqError) as ei:
        if call == "export":
            e.export_groups([G])
        else:
            e.import_groups([1, 1], dict(term=[1, 2]))
    assert ei.value.code == F.MRQ_E_INVAL and "stub error" in str(ei.value)
