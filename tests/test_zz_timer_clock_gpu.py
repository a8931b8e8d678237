"""Tick mode 4's clock-relative leader timers on hardware.

A compact leader's electionElapsed and heartbeatElapsed are kept as phases against the engine's tick number, so the
batched tick neither computes nor stores them, and they are written into the meta word only when the wide columns are
made exact (an export, the general path).  Here mode-4 mrq_tick_many batches of 3 to 20 ticks run the steady trace
against tick mode 0 fed the same messages from the wide inbox: every tick's out words (heartbeat bits included) and
commit advances, and after every batch every exported column, the timers and the randomized timeout included, must be
equal bit for bit.  The cases cover HeartbeatTick 1 and 3 with a non-default ElectionTick, leaders imported with timers
at or above ElectionTick / HeartbeatTick, both kernel shapes, write-through on and off, and a tick-count change in the
middle of the run."""
import numpy as np
import pytest

from raftsql_b200 import Engine, preset_trace
from raftsql_b200.packed import Pack8

pytestmark = [pytest.mark.gpu]

COLUMNS = ("term", "vote", "committed", "last_index", "last_term", "term_start", "match", "role", "lead", "votes",
           "election_elapsed", "heartbeat_elapsed", "randomized_timeout")
BATCHES = (3, 20, 7, 13, 5, 20, 4, 11, 17, 3, 9, 20)


def _run(et, ht, wt, reset_at=None, tick0=0, rounds=2):
    import bench

    G, R = 4096, 5
    st0 = bench.steady_state(G, R, 0, bench.SEED)
    rng = np.random.default_rng(7)
    # timers anywhere in range, and for some leaders at or above ElectionTick / HeartbeatTick (they stay wide for a tick)
    st0["election_elapsed"][:] = rng.integers(0, et + 4, size=G).astype(np.uint16)
    st0["heartbeat_elapsed"][:] = rng.integers(0, ht + 2, size=G).astype(np.uint16)
    p = preset_trace(3)
    ref = Engine(G, R, seed=bench.SEED, inbox_slots=1, election_tick=et, heartbeat_tick=ht)
    eng = Engine(G, R, seed=bench.SEED, inbox_slots=max(BATCHES), election_tick=et, heartbeat_tick=ht)
    for e in (ref, eng):
        e.import_state(st0)
        e.tick_count = tick0
    eng.set_tick_mode(4)
    eng.set_write_through(wt)
    base0 = (st0["last_index"] - np.uint64(40)).astype(np.uint64)
    eng.set_packed_base(base0, st0["term"])
    pk = Pack8(st0["self_id"], base0, st0["term"], R)
    t = 0
    for batch, K in enumerate(BATCHES * rounds):
        if batch == reset_at:  # with compact state live: both engines move to another tick number
            np.testing.assert_array_equal(eng.export_state()["election_elapsed"], ref.export_state()["election_elapsed"])
            for e in (ref, eng):
                e.tick_count = (1 << 32) + 5
        want_out, want_adv = [], []
        for k in range(K):
            before = ref.sync_commits().copy()
            ref.gen_trace(p, t, slot=0)
            ib = ref.read_inbox(0)
            ref.tick(0)
            word, prop8, wide = pk.frame(ib)
            eng.post_inbox_packed(word, prop8, wide, slot=k)
            want_out.append(ref.sync_out().copy())
            want_adv.append(np.minimum(ref.sync_commits() - before, 255).astype(np.uint8))
            t += 1
        eng.tick_many(list(range(K)))
        assert eng.tick_count == ref.tick_count
        for k in range(K):
            o, d = eng.sync_slot_outputs(k)
            np.testing.assert_array_equal(o, want_out[k], err_msg=f"out words of tick {k} of batch {batch} (K = {K})")
            np.testing.assert_array_equal(d, want_adv[k], err_msg=f"commit advances of tick {k} of batch {batch} (K = {K})")
        want, got = ref.export_state(), eng.export_state()
        for c in COLUMNS:
            np.testing.assert_array_equal(got[c], want[c], err_msg=f"column {c} after batch {batch} (K = {K})")
    assert (ref.export_state()["role"] == 2).mean() > 0.99, "the leaders should have stayed leaders: the case misses its point"
    assert eng.counters()["errors"] == 0 and ref.counters()["errors"] == 0
    ref.close()
    eng.close()


@pytest.mark.parametrize("gpt", ["4", "1"], ids=["4 groups per thread", "1 group per thread"])
@pytest.mark.parametrize("wt", [1, 0], ids=["write-through", "write-back at end"])
@pytest.mark.parametrize("et,ht", [(10, 1), (7, 3)], ids=["ET 10 HT 1", "ET 7 HT 3"])
def test_mode_4_clock_timers_equal_mode_0(et, ht, wt, gpt, monkeypatch):
    monkeypatch.setenv("MRQ_T4_GPT", gpt)
    _run(et, ht, wt)


@pytest.mark.parametrize("gpt", ["4", "1"], ids=["4 groups per thread", "1 group per thread"])
def test_mode_4_clock_timers_across_a_tick_count_change(gpt, monkeypatch):
    monkeypatch.setenv("MRQ_T4_GPT", gpt)
    _run(13, 4, 1, reset_at=7, tick0=(1 << 40) + 11, rounds=1)
