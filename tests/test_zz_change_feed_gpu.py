"""The change feed on hardware: the records mrq_sync_changes drains against the oracle.

Every tick, the groups whose term, vote, role or lead moved must come back exactly once, with the values after the
tick, sorted by (tick, group): the diff of consecutive oracle exports.  Tick modes 0 to 4 run lag + churn from a cold
start (elections first) at 16,384 groups x 7 replicas; mode 4 with both kernel shapes, per-tick and mrq_tick_many
batches of 3 to 20 ticks, write-through on and off.  Also: idle-tick elections, a CUDA graph captured with the feed off
and replayed with it on, a capacity below the change count, the feed changing nothing else, and the full
1,048,576 x 5 shape in mode 4 against the mode-0 engine's feed."""
import functools

import numpy as np
import pytest

from oracle import Oracle, TraceParams
from raftsql_b200 import Engine, preset_trace
from raftsql_b200 import _ffi as F
from raftsql_b200.engine import CHANGE_DTYPE, MrqError
from raftsql_b200.packed import Pack8

pytestmark = [pytest.mark.gpu]

NO_GATE = np.uint64(2**64 - 1)
BATCHES = (3, 20, 7, 13, 5, 20, 4, 11, 17, 3, 9, 20)


def diff(b: dict, a: dict, tick: int) -> np.ndarray:
    """the records one tick must produce, from the oracle's exports before (b) and after (a) it"""
    what = ((a["term"] != b["term"]) * F.CHANGE_TERM | (a["vote"] != b["vote"]) * F.CHANGE_VOTE |
            (a["role"] != b["role"]) * F.CHANGE_ROLE | (a["lead"] != b["lead"]) * F.CHANGE_LEAD)
    g = np.nonzero(what)[0]
    r = np.zeros(len(g), CHANGE_DTYPE)
    r["tick"], r["group"], r["what"] = tick, g, what[g]
    r["term"], r["vote"], r["role"], r["lead"] = a["term"][g], a["vote"][g], a["role"][g], a["lead"][g]
    r["term_start"] = np.where(a["role"][g] == F.ROLE_LEADER, a["term_start"][g], NO_GATE)
    return r


def assert_records_equal(got: np.ndarray, want: np.ndarray, where: str):
    assert len(got) == len(want), f"{where}: {len(got)} records, want {len(want)}"
    for name in CHANGE_DTYPE.names:
        np.testing.assert_array_equal(got[name], want[name], err_msg=f"{where}: field {name}")


@functools.lru_cache(maxsize=4)
def oracle_trace(G, R, cfg, T, seed):
    """(inboxes, expected records per tick) of trace preset `cfg` from a cold start"""
    orc = Oracle(G, R, seed=seed)
    p = TraceParams()
    for n, _ in F.TraceParams._fields_:
        setattr(p, n, getattr(preset_trace(cfg), n))
    before = orc.export()
    inboxes, want = [], []
    for t in range(T):
        ib = orc.gen_trace(p, t, nthreads=8)
        orc.tick(ib, nthreads=8)
        after = orc.export()
        inboxes.append(ib)
        want.append(diff(before, after, t))
        before = after
    assert orc.errors == 0
    orc.close()
    return inboxes, want


def run_engine(eng, inboxes, mode, batches, G, R):
    """drive `eng` through the inboxes in tick mode `mode`; a drain after every batch"""
    got = []
    packed = mode in (3, 4)
    if packed:
        st = eng.export_state(("self_id", "last_index", "term"))
        base = st["last_index"].copy()
        eng.set_packed_base(base, st["term"])
        pk = Pack8(st["self_id"], base, st["term"], R)
    t = 0
    it = iter(batches)
    while t < len(inboxes):
        K = min(next(it, 1), len(inboxes) - t)
        for k in range(K):
            ib = inboxes[t + k]
            if packed:
                word, prop8, wide = pk.frame(ib)
                eng.post_inbox_packed(word, prop8, wide, slot=k)
            else:
                eng.post_inbox_dense(ib, slot=k)
        if K == 1:
            eng.tick(0)
        else:
            eng.tick_many(list(range(K)))
        t += K
        recs, lost = eng.sync_changes()
        assert lost == 0
        got.append(recs)
    return np.concatenate(got)


CASES = [
    # (mode, batches, graph mode, MRQ_T4_GPT, write-through)
    (0, (1,), 2, None, 1),
    (0, BATCHES, 1, None, 1),  # graph replay of slot sequences
    (1, (1,), 2, None, 1),
    (2, (1, 4, 9), 1, None, 1),
    (3, (1,), 2, None, 1),
    (4, (1,), 2, "4", 1),
    (4, BATCHES, 2, "4", 1),
    (4, BATCHES, 2, "4", 0),
    (4, BATCHES, 2, "1", 1),
    (4, BATCHES, 2, "1", 0),
]


@pytest.mark.parametrize("mode,batches,graph,gpt,wt", CASES,
                         ids=[f"mode {c[0]} K {'1' if len(c[1]) == 1 else 'many'} graph {c[2]} gpt {c[3]} wt {c[4]}" for c in CASES])
@pytest.mark.parametrize("cfg,T", [(5, 140), (2, 60)], ids=["lag+churn", "cold-start election"])
def test_feed_equals_the_oracle_diff_in_every_mode(mode, batches, graph, gpt, wt, cfg, T, monkeypatch):
    if gpt:
        monkeypatch.setenv("MRQ_T4_GPT", gpt)
    G, R, seed = 16384, 7, 0xFEED0000 + cfg
    inboxes, want = oracle_trace(G, R, cfg, T, seed)
    want = np.concatenate(want)
    assert len(want) > G, "the trace should change many groups"
    with Engine(G, R, seed=seed, inbox_slots=20) as eng:
        eng.set_graph_mode(graph)
        eng.set_tick_mode(mode)
        eng.set_write_through(wt)
        eng.set_change_capacity(8 * G)
        got = run_engine(eng, inboxes, mode, batches * 100, G, R)
        assert eng.counters()["errors"] == 0
    assert_records_equal(got, want, f"mode {mode}")


@pytest.mark.parametrize("mode", [0, 4])
def test_idle_tick_elections_from_term_0(mode):
    G, R, seed = 4096, 5, 0xFEED1D1E
    orc = Oracle(G, R, seed=seed)
    before, want = orc.export(), []
    for t in range(30):
        orc.tick(None)
        after = orc.export()
        want.append(diff(before, after, t))
        before = after
    want = np.concatenate(want)
    with Engine(G, R, seed=seed) as eng:
        eng.set_tick_mode(mode)
        eng.set_change_capacity(4 * G)
        eng.tick_idle(30)
        got, lost = eng.sync_changes()
    assert lost == 0 and (got["what"] & F.CHANGE_ROLE).any(), "the timers should have started campaigns"
    assert_records_equal(got, want, "tick_idle")


def test_graph_captured_with_the_feed_off_then_replayed_with_it_on():
    G, R, seed = 8192, 5, 0xFEED6A9F
    inboxes, want = oracle_trace(G, R, 2, 60, seed)
    with Engine(G, R, seed=seed, inbox_slots=4) as eng:
        eng.set_graph_mode(1)
        got = []
        for t in range(0, 60, 4):
            for k in range(4):
                eng.post_inbox_dense(inboxes[t + k], slot=k)
            eng.tick_many([0, 1, 2, 3])
            if t == 8:  # the graph of this sequence was captured (and replayed once) with the feed off
                eng.set_change_capacity(4 * G)
            elif t > 8:
                recs, lost = eng.sync_changes()
                assert lost == 0
                got.append(recs)
    assert_records_equal(np.concatenate(got), np.concatenate(want[12:]), "replay")


@pytest.mark.parametrize("mode", [0, 4])
def test_capacity_below_the_change_count(mode):
    G, R, seed, cap = 16384, 5, 0xFEED0F10, 1000
    inboxes, want = oracle_trace(G, R, 2, 40, seed)
    want = np.concatenate(want)
    assert len(want) > cap
    with Engine(G, R, seed=seed, inbox_slots=1) as eng:
        eng.set_tick_mode(mode)
        eng.set_change_capacity(cap)
        if mode == 4:
            st = eng.export_state(("self_id", "last_index", "term"))
            eng.set_packed_base(st["last_index"], st["term"])
            pk = Pack8(st["self_id"], st["last_index"].copy(), st["term"], R)
        for ib in inboxes:
            if mode == 4:
                word, prop8, wide = pk.frame(ib)
                eng.post_inbox_packed(word, prop8, wide, slot=0)
            else:
                eng.post_inbox_dense(ib, slot=0)
            eng.tick(0)
        got, lost = eng.sync_changes()
        assert len(got) == cap and lost == len(want) - cap
        key = lambda r: tuple(int(r[n]) for n in CHANGE_DTYPE.names)
        assert {key(r) for r in got} <= {key(r) for r in want}, "every record returned must be genuine"
        got, lost = eng.sync_changes()  # the drain reset the feed
        assert len(got) == 0 and lost == 0


def test_feed_off_changes_nothing():
    G, R, seed = 16384, 5, 0xFEED0FF0
    inboxes, _ = oracle_trace(G, R, 5, 60, seed)
    results = []
    for on in (False, True):
        with Engine(G, R, seed=seed, inbox_slots=20) as eng:
            if not on:
                with pytest.raises(MrqError) as ei:
                    eng.sync_changes()
                assert ei.value.code == F.MRQ_E_STATE
            else:
                eng.set_change_capacity(G)
            eng.set_tick_mode(4)
            st = eng.export_state(("self_id", "last_index", "term"))
            eng.set_packed_base(st["last_index"], st["term"])
            pk = Pack8(st["self_id"], st["last_index"].copy(), st["term"], R)
            outs = []
            for t0 in range(0, 60, 20):
                for k in range(20):
                    word, prop8, wide = pk.frame(inboxes[t0 + k])
                    eng.post_inbox_packed(word, prop8, wide, slot=k)
                eng.tick_many(list(range(20)))
                outs.append([eng.sync_slot_outputs(k) for k in range(20)])
            results.append((eng.export_state(), outs))
    (s0, o0), (s1, o1) = results
    for c in s0:
        np.testing.assert_array_equal(s1[c], s0[c], err_msg=c)
    for b0, b1 in zip(o0, o1):
        for (w0, d0), (w1, d1) in zip(b0, b1):
            np.testing.assert_array_equal(w1, w0)
            np.testing.assert_array_equal(d1, d0)


def test_full_size_mode_4_equals_mode_0():
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
    t = 0
    for cfg, nbatches in ((3, 1), (5, 2)):  # the steady trace, then churn (preset 5's churn and vote parameters)
        p = preset_trace(cfg)
        for _ in range(nbatches):
            for k in range(20):
                ref.gen_trace(p, t, slot=0)
                ib = ref.read_inbox(0)
                ref.tick(0)
                word, prop8, wide = pk.frame(ib)
                eng.post_inbox_packed(word, prop8, wide, slot=k)
                t += 1
            eng.tick_many(list(range(20)))
            want, lw = ref.sync_changes()
            got, lg = eng.sync_changes()
            assert lw == 0 and lg == 0
            if cfg == 3:
                assert len(got) == 0 and len(want) == 0, "the steady trace changes no term, vote, role or lead"
            assert_records_equal(got, want, f"full size, preset {cfg}, tick {t}")
    assert len(want) > 0, "the churn trace should change some groups"
    ref.close()
    eng.close()
