"""State of a list of groups on hardware: mrq_export_groups / mrq_import_groups.

Export: in tick modes 0 to 4 (mode 4 with both kernel shapes, write-through on and off) at 16,384 x 7 on lag + churn, the
rows export_groups returns mid-run for random lists (first and last group, duplicates, a ragged G) equal the rows of
export_state, and a twin engine that did not export gives identical later state, out words, per-slot outputs and
change-feed records.  Import: mid-run in every mode, import_groups of perturbed rows (another group's row, leaders with
out-of-range timers, acks beyond lastIndex, lastIndex beyond the 16-bit span) followed by 64 more ticks equals the oracle
given the same rows, on every column, out word, commit advance and feed record.  In mode 4 neither call converts the
whole engine (kernel_launches), and at 1,048,576 x 5 an import into 1,000 groups equals a mode-0 engine given the same
import.  Also: argument errors change nothing, and the fused gather republishes imported indices (two or more GPUs)."""
import functools
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
BATCHES = (3, 20, 7, 13, 5, 20, 4, 11, 17, 3, 9, 20)
ET = 10


def oracle_params(cfg):
    p = TraceParams()
    for n, _ in F.TraceParams._fields_:
        setattr(p, n, getattr(preset_trace(cfg), n))
    return p


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


def assert_rows_equal(rows: dict, full: dict, groups, where):
    for k, a in rows.items():
        np.testing.assert_array_equal(a, full[k][..., groups], err_msg=f"{where}: column {k}")


@functools.lru_cache(maxsize=2)
def trace(G, R, cfg, T, seed):
    """the inboxes of trace preset `cfg` from a cold start (the trace depends on state: the oracle generates it)"""
    orc = Oracle(G, R, seed=seed)
    p = oracle_params(cfg)
    ibs = []
    for t in range(T):
        ib = orc.gen_trace(p, t, nthreads=8)
        orc.tick(ib, nthreads=8)
        ibs.append(ib)
    assert orc.errors == 0
    orc.close()
    return ibs


def new_engine(G, R, seed, mode, wt=1):
    eng = Engine(G, R, seed=seed, inbox_slots=20)
    eng.set_tick_mode(mode)
    eng.set_write_through(wt)
    eng.set_change_capacity(8 * G)
    pk = None
    if mode in (3, 4):
        st = eng.export_state(("self_id", "last_index", "term"))
        base = st["last_index"].copy()
        eng.set_packed_base(base, st["term"])
        pk = Pack8(st["self_id"], base, st["term"], R)
    return eng, pk


def run_batch(eng, pk, mode, ibs):
    """post and tick one batch; returns (per-tick out words, per-tick commit advances or None, feed records)"""
    K = len(ibs)
    for k, ib in enumerate(ibs):
        if pk is not None:
            eng.post_inbox_packed(*pk.frame(ib), slot=k)
        else:
            eng.post_inbox_dense(ib, slot=k)
    if K == 1:
        eng.tick(0)
        outs = [(eng.sync_out(), eng.sync_tick_deltas() if mode == 4 else None)]
    else:
        eng.tick_many(list(range(K)))
        outs = [eng.sync_slot_outputs(k) for k in range(K)] if mode == 4 else [(eng.sync_out(), None)]
    recs, lost = eng.sync_changes()
    assert lost == 0
    return outs, recs


def random_list(rng, G, n, unique):
    """n random groups and the first and last one, in random order; with duplicates unless `unique`"""
    if unique:
        g = np.unique(np.concatenate([[0, G - 1], rng.choice(G, size=n, replace=False)]))
    else:
        g = np.concatenate([[0, G - 1, 0, G - 1], rng.integers(0, G, size=n)])
    return rng.permutation(g).astype(np.uint64)


EXPORT_CASES = [
    # (mode, batches, MRQ_T4_GPT, write-through, G)
    (0, (1,), None, 1, 16384),
    (0, BATCHES, None, 1, 16381),
    (1, (1,), None, 1, 16384),
    (2, (1, 4, 9), None, 1, 16384),
    (3, (1,), None, 1, 16384),
    (4, (1,), "4", 1, 16384),
    (4, BATCHES, "4", 1, 16384),
    (4, BATCHES, "4", 0, 16381),
    (4, BATCHES, "1", 1, 16384),
    (4, BATCHES, "1", 0, 16384),
]


@pytest.mark.parametrize("mode,batches,gpt,wt,G", EXPORT_CASES,
                         ids=[f"mode {c[0]} K {'1' if len(c[1]) == 1 else 'many'} gpt {c[2]} wt {c[3]} G {c[4]}" for c in EXPORT_CASES])
def test_export_groups_equals_export_state_rows_and_changes_nothing(mode, batches, gpt, wt, G, monkeypatch):
    if gpt:
        monkeypatch.setenv("MRQ_T4_GPT", gpt)
    R, seed, T = 7, 0x6E0E0000 + G, 100
    ibs = trace(G, R, 5, T, seed)
    rng = np.random.default_rng(G + mode)
    (a, pa), (b, pb) = new_engine(G, R, seed, mode, wt), new_engine(G, R, seed, mode, wt)
    t, nb, n_checked = 0, 0, 0
    it = itertools.cycle(batches)
    while t < T:
        K = min(next(it), T - t)
        oa, ra = run_batch(a, pa, mode, ibs[t:t + K])
        ob, rb = run_batch(b, pb, mode, ibs[t:t + K])
        t += K
        for (wa, da), (wb, db) in zip(oa, ob):
            np.testing.assert_array_equal(wa, wb)
            if da is not None:
                np.testing.assert_array_equal(da, db)
        assert_records_equal(ra, rb, f"tick {t}")
        nb += 1
        if nb % 2 == 0 or t == T:
            groups = random_list(rng, G, int(rng.integers(1, 3000)), unique=False)
            l0 = a.counters()["kernel_launches"]
            rows = a.export_groups(groups)
            sub = a.export_groups(groups[::-1], columns=("committed", "match", "heartbeat_elapsed"))
            assert a.counters()["kernel_launches"] == l0 + 2, "one launch per export, and no conversion"
            full = a.export_state()
            b.export_state()  # the twin makes the same whole-engine calls, not the group-list ones
            assert_rows_equal(rows, full, groups, f"mode {mode} tick {t}")
            assert_rows_equal(sub, full, groups[::-1], f"mode {mode} tick {t} (column subset)")
            n_checked += 1
    assert n_checked >= 3
    sa, sb = a.export_state(), b.export_state()
    for k in STATE_COLUMNS:
        np.testing.assert_array_equal(sa[k], sb[k], err_msg=k)
    if mode == 4:
        assert (sa["role"] == F.ROLE_LEADER).mean() > 0.3, "the run should have elected leaders (compact clock leaders)"
    a.close()
    b.close()


def perturb(rows: dict, donor: dict, rng, R) -> dict:
    """what a host might import: another group's row (a slot reused for another range: its self id too), leaders with
    out-of-range timers, acks beyond lastIndex, lastIndex beyond the 16-bit span of the compact offsets"""
    rows = {k: v.copy() for k, v in rows.items()}
    n = len(rows["term"])
    sel = rng.integers(0, 5, size=n)
    for k in rows:
        rows[k][..., sel == 0] = donor[k][..., sel == 0]
    lead = rows["role"] == F.ROLE_LEADER
    cols = np.arange(n)
    m = (sel == 1) & lead
    rows["election_elapsed"][m] = ET + 5
    rows["heartbeat_elapsed"][m] = 3
    m = (sel == 2) & lead
    other = rows["self_id"].astype(np.int64) % R  # a replica slot other than the group's own
    rows["match"][other[m], cols[m]] = rows["last_index"][m] + np.uint64(3)
    m = sel == 3  # (the entries keep the last entry's term: only a leader's own entries carry its term)
    rows["last_index"][m] += np.uint64(70000)
    ml = m & lead
    rows["match"][rows["self_id"][ml].astype(np.int64) - 1, cols[ml]] = rows["last_index"][ml]
    return rows


IMPORT_CASES = [
    (0, (1,), None, 1),
    (1, (1,), None, 1),
    (2, (1,), None, 1),
    (3, (1,), None, 1),
    (4, (1,), "4", 1),
    (4, BATCHES, "4", 1),
    (4, BATCHES, "1", 0),
]


@pytest.mark.parametrize("mode,batches,gpt,wt", IMPORT_CASES,
                         ids=[f"mode {c[0]} K {'1' if len(c[1]) == 1 else 'many'} gpt {c[2]} wt {c[3]}" for c in IMPORT_CASES])
def test_import_groups_then_ticks_equal_the_oracle(mode, batches, gpt, wt, monkeypatch):
    if gpt:
        monkeypatch.setenv("MRQ_T4_GPT", gpt)
    G, R, seed = 16384, 7, 0x1A90000 + mode
    orc = Oracle(G, R, seed=seed)
    eng, pk = new_engine(G, R, seed, mode, wt)
    p = oracle_params(5)
    rng = np.random.default_rng(seed)
    t = 0
    it = itertools.cycle(batches)

    def lockstep(n_ticks, where):
        nonlocal t
        end = t + n_ticks
        while t < end:
            K = min(next(it), end - t)
            before = orc.export()
            ibs, want_recs, want_out, want_adv = [], [], [], []
            for k in range(K):
                ib = orc.gen_trace(p, t + k, nthreads=8)
                orc.tick(ib, nthreads=8)
                after = orc.export()
                ibs.append(ib)
                want_recs.append(diff(before, after, t + k))
                want_out.append(after["out"])
                want_adv.append(np.minimum(after["committed"] - before["committed"], np.uint64(255)).astype(np.uint8))
                before = after
            outs, recs = run_batch(eng, pk, mode, ibs)
            t += K
            w = f"{where}, mode {mode}, tick {t}"
            assert_state_equal(eng.export_state(), before, w)
            if len(outs) == K:
                for k, (o, d) in enumerate(outs):
                    np.testing.assert_array_equal(o, want_out[k], err_msg=f"{w}: out words of tick {t - K + k}")
                    if d is not None:
                        np.testing.assert_array_equal(d, want_adv[k], err_msg=f"{w}: commit advances of tick {t - K + k}")
            else:
                np.testing.assert_array_equal(outs[-1][0], want_out[-1], err_msg=f"{w}: out words")
            assert_records_equal(recs, np.concatenate(want_recs), w)

    lockstep(40, "before the import")
    groups = random_list(rng, G, 600, unique=True)
    donors = rng.integers(0, G, size=len(groups)).astype(np.uint64)
    rows = perturb(eng.export_groups(groups), eng.export_groups(donors), rng, R)
    l0 = eng.counters()["kernel_launches"]
    eng.import_groups(groups, rows)
    assert eng.counters()["kernel_launches"] == l0 + 1
    full = orc.export()
    for k in STATE_COLUMNS:
        full[k][..., groups.astype(np.int64)] = rows[k]
    orc.import_state(full)
    if pk is not None:
        pk.self_id[groups.astype(np.int64)] = rows["self_id"]
    assert_rows_equal(eng.export_groups(groups), rows, np.arange(len(groups)), "right after the import")
    lockstep(64, "after the import")
    assert eng.counters()["errors"] == 0 and orc.errors == 0
    eng.close()
    orc.close()


def test_mode_4_calls_convert_nothing():
    """kernel_launches: an export adds one launch at any G; after import_groups the next batch launches no
    compact_all_kernel, after import_state it does"""
    R, seed = 5, 0x1A9C0C0
    for G in (1000, 16384):
        eng, _ = new_engine(G, R, seed, 4)
        eng.tick_idle(30)  # elections: compact leaders on the clock
        l0 = eng.counters()["kernel_launches"]
        eng.export_groups(np.arange(0, G, 7, dtype=np.uint64))
        assert eng.counters()["kernel_launches"] == l0 + 1, G
        eng.close()
    G = 16384
    ibs = trace(G, R, 5, 60, seed)
    (x, px), (y, py) = new_engine(G, R, seed, 4), new_engine(G, R, seed, 4)
    for e, pk in ((x, px), (y, py)):
        run_batch(e, pk, 4, ibs[0:20])
        run_batch(e, pk, 4, ibs[20:40])
    rng = np.random.default_rng(1)
    groups = random_list(rng, G, 500, unique=True)
    rows = perturb(x.export_groups(groups), x.export_groups(rng.integers(0, G, len(groups)).astype(np.uint64)), rng, R)
    x.import_groups(groups, rows)
    full = y.export_state()
    for k in STATE_COLUMNS:
        full[k][..., groups.astype(np.int64)] = rows[k]
    y.import_state(full)
    for pk in (px, py):
        pk.self_id[groups.astype(np.int64)] = rows["self_id"]
    lx, ly = x.counters()["kernel_launches"], y.counters()["kernel_launches"]
    ox, rx = run_batch(x, px, 4, ibs[40:60])
    oy, ry = run_batch(y, py, 4, ibs[40:60])
    dx, dy = x.counters()["kernel_launches"] - lx, y.counters()["kernel_launches"] - ly
    assert dy == dx + 1, f"after import_state the batch re-compacts every group ({dy} launches), after import_groups not ({dx})"
    for (wa, da), (wb, db) in zip(ox, oy):
        np.testing.assert_array_equal(wa, wb)
        np.testing.assert_array_equal(da, db)
    assert_records_equal(rx, ry, "import_groups vs import_state")
    sx, sy = x.export_state(), y.export_state()
    for k in STATE_COLUMNS:
        np.testing.assert_array_equal(sx[k], sy[k], err_msg=k)
    x.close()
    y.close()


def test_full_size_mode_4_import_equals_mode_0():
    import bench

    G, R = bench.G_TOTAL, bench.R
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
    rng = np.random.default_rng(5)
    groups = np.sort(rng.choice(G, size=1000, replace=False)).astype(np.uint64)
    t = 0
    for cfg, nbatches in ((3, 1), (3, 1), (5, 2)):  # the steady trace, the import, the steady trace, then churn
        p = preset_trace(cfg)
        for _ in range(nbatches):
            for k in range(20):
                ref.gen_trace(p, t, slot=0)
                ib = ref.read_inbox(0)
                ref.tick(0)
                eng.post_inbox_packed(*pk.frame(ib), slot=k)
                t += 1
            eng.tick_many(list(range(20)))
            assert_records_equal(eng.sync_changes()[0], ref.sync_changes()[0], f"full size, tick {t}")
        if t == 20:  # re-created replicas: fresh followers at their log position, from their WAL's HardState
            now = ref.export_groups(groups)
            rows = dict(term=now["term"] + np.uint64(1), vote=np.zeros(1000, np.uint64), committed=now["committed"],
                        last_index=now["last_index"], last_term=now["last_term"], term_start=np.full(1000, NO_GATE),
                        match=np.zeros((R, 1000), np.uint64), role=np.zeros(1000, np.uint8), lead=np.zeros(1000, np.uint8),
                        votes=np.zeros((R, 1000), np.uint8), election_elapsed=np.zeros(1000, np.uint16),
                        heartbeat_elapsed=np.zeros(1000, np.uint16))
            l0 = eng.counters()["kernel_launches"]
            mine = eng.export_groups(groups)
            assert eng.counters()["kernel_launches"] == l0 + 1
            assert_rows_equal(mine, ref.export_state(), groups, "full size export")
            for e in (ref, eng):
                e.import_groups(groups, rows)
    s_ref, s_eng = ref.export_state(), eng.export_state()
    assert_state_equal(s_eng, s_ref, "full size after the import")
    assert (s_eng["role"][groups.astype(np.int64)] != F.ROLE_LEADER).any()
    ref.close()
    eng.close()


def test_argument_errors_change_nothing():
    G, R = 1000, 5
    with Engine(G, R, seed=3) as eng:
        eng.set_tick_mode(4)
        eng.tick_idle(25)
        before = eng.export_state()
        rows = dict(term=np.full(3, 99, np.uint64), committed=np.zeros(3, np.uint64))
        for groups in ([1, 2, G], [5, 6, 5]):
            with pytest.raises(MrqError) as ei:
                eng.import_groups(groups, rows)
            assert ei.value.code == F.MRQ_E_INVAL
        with pytest.raises(MrqError) as ei:
            eng.export_groups([0, G + 3])
        assert ei.value.code == F.MRQ_E_INVAL
        st = F.State()
        term = np.zeros(3, np.uint64)
        st.term = term.ctypes.data_as(F.u64p)
        assert eng.L.mrq_import_groups(eng.h, None, 3, st) == F.MRQ_E_INVAL
        assert eng.L.mrq_export_groups(eng.h, None, 3, st) == F.MRQ_E_INVAL
        assert eng.L.mrq_import_groups(eng.h, None, 0, st) == F.MRQ_OK  # n == 0: no-op
        after = eng.export_state()
        for k in STATE_COLUMNS:
            np.testing.assert_array_equal(after[k], before[k], err_msg=k)
    with Engine(0, 3) as empty:
        assert empty.export_groups([])["term"].shape == (0,)
        assert empty.L.mrq_export_groups(empty.h, np.zeros(2, np.uint64).ctypes.data_as(F.u64p), 2, F.State()) == F.MRQ_OK


def _ngpu():
    import torch

    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gather_worker(rank, world, port, G_total, R, q):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist

    from raftsql_b200 import multi

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        base, G = multi.shard_range(G_total, rank, world)
        eng = Engine(G, R, seed=11, group_base=base, device=rank)
        multi.attach(eng, dist, "fused")
        p = preset_trace(3)
        for t in range(30):
            eng.gen_trace(p, t)
            eng.tick()
        groups = np.arange(rank, G, 97, dtype=np.uint64)
        now = eng.export_groups(groups, ("committed", "last_index"))
        jump = np.uint64(1 << 20)  # above the low byte: the peers must see the new high bits
        eng.import_groups(groups, dict(committed=now["committed"] + jump, last_index=now["last_index"] + jump))
        eng.gen_trace(p, 30)
        eng.tick()
        eng.synchronize()
        dist.barrier()
        torch.cuda.synchronize()
        ok = bool(np.array_equal(eng.sync_gathered(), multi.gather_reference(dist, eng.sync_commits())))
        oks = [None] * world
        dist.all_gather_object(oks, ok)
        if rank == 0:
            q.put(oks)
        dist.barrier()
        eng.close()
    finally:
        dist.destroy_process_group()


def test_fused_gather_republishes_imported_indices():
    if _ngpu() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp

    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gather_worker, args=(r, world, port, 1 << 14, 5, q)) for r in range(world)]
    for p in procs:
        p.start()
    oks = q.get(timeout=600)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert all(oks), f"the gather shows stale high bits of an imported index on some rank: {oks}"
