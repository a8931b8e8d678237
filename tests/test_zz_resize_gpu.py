"""Resizing a running engine's group count on hardware: mrq_resize_groups.

Twin equivalence: engine A runs, resizes and runs on; at every resize a twin B is created fresh at the new size and
given A's surviving rows (every column, timers, votes and self ids included), its own fresh rows, A's tick count and
packed bases.  After every tick A equals B (state, out words, commit advances, mode-4 per-slot outputs, change-feed
records) and the oracle (resized the same way).  In tick modes 0-4 at R = 3, 5, 7 (mode 4 also R = 1 and 8, both
kernel shapes, write-through on and off, per-tick and batched ticks), over 1000 -> 900 -> 1000 (a shrink and a grow
back that keep the stride: no buffer moves, and the grow re-initialises rows that still hold dropped groups), grows
and a shrink that move the stride (-> 1100 -> 3000 -> 1000), 0 -> 500 -> 0, and 130 single-group grows across a
stride boundary.  Also: fresh rows equal a fresh engine's, a
resize adds one launch for a grow and none for a shrink and the next mode-4 batch re-compacts nothing, pending feed
records survive, graph replay after a resize equals the oracle, a 1,048,576 x 5 mode-4 engine grown by 131,072 and shrunk
back equals a mode-0 engine, and refused resizes change nothing."""
import itertools
import os
import socket
import sys

import numpy as np
import pytest

from oracle import Oracle, TraceParams
from raftsql_b200 import Engine, preset_trace
from raftsql_b200 import _ffi as F
from raftsql_b200.engine import CHANGE_DTYPE, STATE_COLUMNS, MrqError
from raftsql_b200.packed import Pack8

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from util import assert_state_equal  # noqa: E402

pytestmark = [pytest.mark.gpu]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_GATE = np.uint64(2**64 - 1)
BATCHES = (3, 1, 20, 7, 13, 5, 4, 11)
FEED_CAP = 1 << 18


def oracle_params(cfg):
    p = TraceParams()
    for n, _ in F.TraceParams._fields_:
        setattr(p, n, getattr(preset_trace(cfg), n))
    return p


def stride(n):
    return max(128, -(-n // 128) * 128)


def diff(b: dict, a: dict, tick: int) -> np.ndarray:
    """the change-feed records one tick must produce, from the oracle's exports before (b) and after (a) it"""
    what = ((a["term"] != b["term"]) * F.CHANGE_TERM | (a["vote"] != b["vote"]) * F.CHANGE_VOTE |
            (a["role"] != b["role"]) * F.CHANGE_ROLE | (a["lead"] != b["lead"]) * F.CHANGE_LEAD)
    g = np.nonzero(what)[0]
    r = np.zeros(len(g), CHANGE_DTYPE)
    r["tick"], r["group"], r["what"] = tick, g, what[g]
    r["term"], r["vote"], r["role"], r["lead"] = a["term"][g], a["vote"][g], a["role"][g], a["lead"][g]
    r["term_start"] = np.where(a["role"][g] == F.ROLE_LEADER, a["term_start"][g], NO_GATE)
    return r


def assert_records_equal(got, want, where):
    assert len(got) == len(want), f"{where}: {len(got)} records, want {len(want)}"
    for name in CHANGE_DTYPE.names:
        np.testing.assert_array_equal(got[name], want[name], err_msg=f"{where}: field {name}")


def assert_all_columns_equal(x: dict, y: dict, where):
    for k in STATE_COLUMNS:
        np.testing.assert_array_equal(x[k], y[k], err_msg=f"{where}: column {k}")


class Twins:
    """Engine A under test and the oracle in lockstep with it; from A's first resize on, twin B (created fresh at the
    new size at every resize) gets the same posts"""

    def __init__(self, G, R, mode, wt=1, seed=0x5E51, graph_mode=2, cfg=5):
        self.G, self.R, self.mode, self.wt, self.seed, self.graph_mode = G, R, mode, wt, seed, graph_mode
        self.p = oracle_params(cfg)
        self.t = 0
        self.a, self.b = self.engine(G), None
        self.orc = Oracle(G, R, seed=seed) if G else None
        self.pk = None
        if mode in (3, 4):
            self.pk = Pack8(self.a.export_state(("self_id",))["self_id"], np.zeros(G, np.uint64), np.zeros(G, np.uint64), R)
        self.want = []  # oracle records A has not drained yet
        self.b_since = 0  # the first tick B ran
        self.compact_live = False  # mode 4: A's compact state exists (its next batch converts nothing)
        self.launches_ok = 0
        self.in_place = []  # resizes that kept the stride (and every buffer) with groups on both sides

    def engine(self, G):
        e = Engine(G, self.R, seed=self.seed, inbox_slots=20)
        e.set_tick_mode(self.mode)
        e.set_write_through(self.wt)
        e.set_graph_mode(self.graph_mode)
        e.set_change_capacity(FEED_CAP)
        return e

    def close(self):
        for x in (self.a, self.b, self.orc):
            if x is not None:
                x.close()

    def run(self, n, batches=(1,), drain=True):
        if self.G == 0:  # nothing to post: the ticks only count
            self.a.tick_idle(n)
            if self.b is not None:
                self.b.tick_idle(n)
            self.t += n
            return
        it = itertools.cycle(batches)
        end = self.t + n
        while self.t < end:
            self.batch(min(next(it), end - self.t), drain)

    def batch(self, K, drain=True):
        mode, orc = self.mode, self.orc
        before = orc.export()
        ibs, want_out, want_adv = [], [], []
        for k in range(K):
            ib = orc.gen_trace(self.p, self.t + k, nthreads=8)
            orc.tick(ib, nthreads=8)
            after = orc.export()
            ibs.append(ib)
            self.want.append(diff(before, after, self.t + k))
            want_out.append(after["out"])
            want_adv.append(np.minimum(after["committed"] - before["committed"], np.uint64(255)).astype(np.uint8))
            before = after
        engines = [e for e in (self.a, self.b) if e is not None]
        for k, ib in enumerate(ibs):
            frame = self.pk.frame(ib) if self.pk is not None else None
            for e in engines:
                if frame is not None:
                    e.post_inbox_packed(*frame, slot=k)
                else:
                    e.post_inbox_dense(ib, slot=k)
        outs = []
        for e in engines:
            l0 = e.counters()["kernel_launches"]
            if K == 1:
                e.tick(0)
            else:
                e.tick_many(list(range(K)))
            dl = e.counters()["kernel_launches"] - l0
            if e is self.a and mode == 4:
                assert dl == (2 if self.compact_live else 3), f"tick {self.t}: a mode-4 batch launched {dl} kernels"
                self.compact_live = True
                self.launches_ok += 1
            if K == 1:
                outs.append([(e.sync_out(), e.sync_tick_deltas() if mode == 4 else None)])
            else:
                outs.append([e.sync_slot_outputs(k) for k in range(K)] if mode == 4 else [(e.sync_out(), None)])
        self.t += K
        w = f"mode {mode} R {self.R} G {self.G} tick {self.t}"
        oa = outs[0]
        if len(oa) == K:
            for k, (o, d) in enumerate(oa):
                np.testing.assert_array_equal(o, want_out[k], err_msg=f"{w}: out words of tick {self.t - K + k}")
                if d is not None:
                    np.testing.assert_array_equal(d, want_adv[k], err_msg=f"{w}: commit advances of tick {self.t - K + k}")
        else:
            np.testing.assert_array_equal(oa[-1][0], want_out[-1], err_msg=f"{w}: out words")
        sa = self.a.export_state()
        assert_state_equal(sa, before, w)
        if self.b is not None:
            for k, ((o, d), (ob, db)) in enumerate(zip(oa, outs[1])):
                np.testing.assert_array_equal(o, ob, err_msg=f"{w}: A and B out words, tick {k} of the batch")
                if d is not None:
                    np.testing.assert_array_equal(d, db, err_msg=f"{w}: A and B commit advances, tick {k} of the batch")
            assert_all_columns_equal(sa, self.b.export_state(), f"{w}: A and B")
            np.testing.assert_array_equal(self.a.sync_commit_deltas(), self.b.sync_commit_deltas(), err_msg=f"{w}: drained deltas")
        if drain:
            want = np.concatenate(self.want)
            ra, lost = self.a.sync_changes()
            assert lost == 0
            assert_records_equal(ra, want, f"{w}: A's records")
            if self.b is not None:
                rb, lost = self.b.sync_changes()
                assert lost == 0
                assert_records_equal(rb, want[want["tick"] >= self.b_since], f"{w}: B's records")
            self.want = []

    def resize(self, n, twin=True):
        a, R, old = self.a, self.R, self.G
        keep = min(old, n)
        pre = a.export_state()
        a.sync_commits()  # rebase A's commit-delta drain: B's is rebased after its import
        l0 = a.counters()["kernel_launches"]
        ptrs = [a.device_ptr(w) for w in (F.PTR_TERM, F.PTR_META, F.PTR_MATCH, F.PTR_OUT)]
        a.resize_groups(n)
        assert a.counters()["kernel_launches"] == l0 + (1 if n > old else 0), "one launch for a grow, none for a shrink"
        assert a.G == n and a.group_stride == stride(n)
        in_place = stride(n) == stride(old)
        moved = [a.device_ptr(w) for w in (F.PTR_TERM, F.PTR_META, F.PTR_MATCH, F.PTR_OUT)] != ptrs
        assert moved != in_place, f"{old} -> {n}: the buffers {'moved' if moved else 'stayed'}"
        if in_place and old:
            self.in_place.append("grow" if n > old else "shrink")
        assert (a.sync_out() == 0).all(), "out words read as right after mrq_create"
        if self.mode == 4 and n:
            with pytest.raises(MrqError) as ei:
                a.sync_tick_deltas()
            assert ei.value.code == F.MRQ_E_STATE
            with pytest.raises(MrqError) as ei:
                a.sync_slot_outputs(0)
            assert ei.value.code == F.MRQ_E_STATE
        now = a.export_state()
        # the oracle: the survivors' rows, fresh rows for the rest, A's tick count
        orc = None
        if n:
            orc = Oracle(n, R, seed=self.seed)
            full = orc.export()
            if keep:
                prev = self.orc.export()
                for k in STATE_COLUMNS:
                    full[k][..., :keep] = prev[k][..., :keep]
            orc.import_state(full)
            orc.tick_count = a.tick_count
        if self.orc is not None:
            self.orc.close()
        self.orc = orc
        if self.b is not None:
            self.b.close()
            self.b = None
        if twin and n:
            b = self.engine(n)
            st = b.export_state()
            for k in STATE_COLUMNS:
                st[k][..., :keep] = pre[k][..., :keep]
            assert_all_columns_equal(now, st, f"right after {old} -> {n}: survivors kept, new rows those of a fresh engine")
            b.import_state(st)
            b.tick_count = a.tick_count
            b.sync_commits()
            self.b, self.b_since = b, a.tick_count
        if self.pk is not None:
            base, term = np.zeros(n, np.uint64), np.zeros(n, np.uint64)  # the host's bases, extended with zeros
            base[:keep], term[:keep] = self.pk.base_index[:keep], self.pk.base_term[:keep]
            self.pk = Pack8(now["self_id"], base, term, R)
            if self.b is not None:
                self.b.set_packed_base(base, term)
        self.G = n


TWIN_CASES = [(m, R, None, 1, (1,)) for m in range(4) for R in (3, 5, 7)]
TWIN_CASES += [(4, R, gpt, wt, b) for R in (3, 5, 7) for gpt, wt, b in (("4", 1, BATCHES), ("4", 0, BATCHES), ("1", 1, BATCHES),
                                                                           ("1", 0, (1,)))]
TWIN_CASES += [(4, R, gpt, wt, BATCHES) for R in (1, 8) for gpt, wt in (("4", 1), ("1", 0))]


@pytest.mark.parametrize("mode,R,gpt,wt,batches", TWIN_CASES,
                         ids=[f"mode {c[0]} R {c[1]} gpt {c[2]} wt {c[3]} K {'1' if len(c[4]) == 1 else 'many'}" for c in TWIN_CASES])
def test_resized_engine_equals_a_fresh_twin_and_the_oracle(mode, R, gpt, wt, batches, monkeypatch):
    if gpt:
        monkeypatch.setenv("MRQ_T4_GPT", gpt)
    tw = Twins(1000, R, mode, wt, seed=0x5E51 + 16 * mode + R)
    try:
        tw.run(30, batches)
        # a shrink that keeps the stride (1024), a grow back over the rows that still hold the dropped groups (compact
        # flags set in mode 4), then a grow, a grow and a shrink that each move it (1152, 3072, 1024)
        for n in (900, 1000, 1100, 3000, 1000):
            tw.resize(n)
            tw.run(24, batches)
        assert tw.in_place == ["shrink", "grow"]
        assert (tw.a.export_state()["role"] == F.ROLE_LEADER).mean() > 0.3, "the run should have elected leaders"
    finally:
        tw.close()
    tw = Twins(0, R, mode, wt, seed=0x5E52 + 16 * mode + R)
    try:
        tw.run(5)
        tw.resize(500)
        tw.run(30, batches)
        tw.resize(0)
        tw.run(3)
        tw.resize(300)
        tw.run(24, batches)
        if mode == 4:
            assert tw.launches_ok > 0
    finally:
        tw.close()


@pytest.mark.parametrize("mode,gpt", [(0, None), (4, "4"), (4, "1")])
def test_single_group_grows_across_a_stride_boundary(mode, gpt, monkeypatch):
    if gpt:
        monkeypatch.setenv("MRQ_T4_GPT", gpt)
    tw = Twins(1000, 5, mode, seed=0x51461E + mode)
    try:
        tw.run(25)
        for n in range(1001, 1131):  # 1024 -> 1152: the stride moves at 1025
            tw.resize(n, twin=n % 8 == 0 or n in (1024, 1025))
            tw.run(1)
        assert tw.a.group_stride == 1152
        tw.run(20)
    finally:
        tw.close()


@pytest.mark.parametrize("mode", [0, 4])
def test_pending_records_survive_a_resize(mode):
    """records of ticks before a resize come back with the first drain after it, groups since dropped included; the
    later ones name the new groups"""
    tw = Twins(2000, 5, mode, seed=0xFEED5)
    try:
        tw.run(20)
        tw.run(15, drain=False)
        assert any((w["group"] >= 1500).any() for w in tw.want), "the trace should have changed groups that the shrink drops"
        tw.resize(1500, twin=False)
        tw.resize(2600, twin=False)
        tw.run(1)  # drains: every pending record plus this tick's, against the oracle's
        tw.run(25)
    finally:
        tw.close()


@pytest.mark.parametrize("mode", [0, 2])
def test_graph_replay_after_a_resize_equals_the_oracle(mode):
    """graph mode 1: sequences captured before a resize hold the old G; after it they are captured anew"""
    for gm in (1, 0):
        tw = Twins(1000, 5, mode, seed=0x6A9, graph_mode=gm)
        try:
            tw.run(24, (4,))
            for n in (900, 1000, 1100, 3000, 1000):
                tw.resize(n)
                tw.run(24, (4,))
        finally:
            tw.close()


def test_full_size_mode_4_grow_and_shrink_equal_mode_0():
    import bench

    G, R, extra = bench.G_TOTAL, bench.R, 131072
    st0 = bench.steady_state(G, R, 0, bench.SEED)
    ref = Engine(G, R, seed=bench.SEED, inbox_slots=1)
    eng = Engine(G, R, seed=bench.SEED, inbox_slots=20)
    for e in (ref, eng):
        e.import_state(st0)
        e.set_change_capacity(G)
    eng.set_tick_mode(4)
    base0 = (st0["last_index"] - np.uint64(40)).astype(np.uint64)
    eng.set_packed_base(base0, st0["term"])
    pk = Pack8(st0["self_id"], base0, st0["term"], R)
    t, compacted = 0, False

    def batch(cfg):
        nonlocal t, compacted
        p = preset_trace(cfg)
        for k in range(20):
            ref.gen_trace(p, t, slot=0)
            ib = ref.read_inbox(0)
            ref.tick(0)
            eng.post_inbox_packed(*pk.frame(ib), slot=k)
            t += 1
        l0 = eng.counters()["kernel_launches"]
        eng.tick_many(list(range(20)))
        assert eng.counters()["kernel_launches"] == l0 + (2 if compacted else 3), "only the first batch compacts"
        compacted = True
        assert_records_equal(eng.sync_changes()[0], ref.sync_changes()[0], f"full size, tick {t}")

    def resize(n):
        nonlocal pk
        keep = min(eng.G, n)
        l0 = eng.counters()["kernel_launches"]
        for e in (ref, eng):
            e.resize_groups(n)
        assert eng.counters()["kernel_launches"] == l0 + (1 if n > keep else 0)
        self_id = eng.export_state(("self_id",))["self_id"]
        base, term = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
        base[:keep], term[:keep] = pk.base_index[:keep], pk.base_term[:keep]
        pk = Pack8(self_id, base, term, R)

    batch(3)
    batch(3)
    resize(G + extra)
    assert eng.group_stride == G + extra
    for cfg in (3, 5, 5, 3):  # the new groups elect leaders
        batch(cfg)
    s_ref, s_eng = ref.export_state(), eng.export_state()
    assert_state_equal(s_eng, s_ref, "full size after the grow")
    assert (s_eng["role"][G:] == F.ROLE_LEADER).any()
    resize(G)
    batch(3)
    batch(5)
    assert_state_equal(eng.export_state(), ref.export_state(), "full size after the shrink")
    assert eng.counters()["errors"] == 0
    ref.close()
    eng.close()


def test_refused_resizes_change_nothing():
    G, R = 1000, 5
    with Engine(G, R, seed=3) as eng:
        eng.set_tick_mode(4)
        eng.tick_idle(25)
        before, gs, l0 = eng.export_state(), eng.group_stride, eng.counters()["kernel_launches"]
        for n in (1 << 32, (1 << 64) - 1):
            with pytest.raises(MrqError) as ei:
                eng.resize_groups(n)
            assert ei.value.code == F.MRQ_E_INVAL
        eng.resize_groups(G)  # no-op
        assert eng.counters()["kernel_launches"] == l0
        assert eng.G == G and eng.group_stride == gs
        assert_all_columns_equal(eng.export_state(), before, "after refused resizes")
    with Engine(G, R, seed=3) as eng:
        eng.tick_idle(25)
        before = eng.export_state()
        eng.ipc_prepare(2)
        with pytest.raises(MrqError) as ei:
            eng.resize_groups(G + 500)
        assert ei.value.code == F.MRQ_E_STATE
        assert eng.G == G
        assert_all_columns_equal(eng.export_state(), before, "after a refused resize (CUDA-IPC gather)")


def _ngpu():
    import torch

    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _comm_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist

    from raftsql_b200 import multi

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        eng = Engine(4096, 5, seed=11, group_base=4096 * rank, device=rank)
        multi.attach(eng, dist, "nccl")
        try:
            eng.resize_groups(5000)
            code = 0
        except MrqError as ex:
            code = ex.code
        codes = [None] * world
        dist.all_gather_object(codes, (code, eng.G))
        if rank == 0:
            q.put(codes)
        dist.barrier()
        eng.close()
    finally:
        dist.destroy_process_group()


def test_a_communicator_refuses_a_resize():
    if _ngpu() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_comm_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    codes = q.get(timeout=600)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert codes == [(F.MRQ_E_STATE, 4096)] * 2, codes
