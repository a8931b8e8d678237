"""The quad kernel's lane-pair hot step on hardware, across its guards and the 16-bit re-base.

tick_fast4_kernel steps two settled leaders at once in the 16-bit lanes of its pair words (compact_hot_pair) and
falls back to the scalar steps for a pair whose lanes leave its guards: a lastIndex above 0xFEFF or a window base above
0xFFBF.  Here the logs grow by up to 32 entries a tick, so over 5,000 mode-4 ticks in batches of 20 every pair crosses
those bounds, reaches the end of the 16-bit span and is re-based by the general path.  With
HeartbeatTick 1 and 3 and write-through on and off, every tick's out words and commit advances, and every exported
column, must equal tick mode 0 fed the same messages from the wide inbox, bit for bit."""
import numpy as np
import pytest

from raftsql_b200 import Engine, preset_trace
from raftsql_b200.packed import Pack8

pytestmark = [pytest.mark.gpu]

COLUMNS = ("term", "vote", "committed", "last_index", "last_term", "term_start", "match", "role", "lead", "election_elapsed",
           "heartbeat_elapsed")


@pytest.mark.parametrize("wt", [1, 0], ids=["write-through", "write-back at end"])
@pytest.mark.parametrize("ht", [1, 3], ids=["HT 1", "HT 3"])
def test_mode_4_pair_step_across_the_guards_equals_mode_0(ht, wt, monkeypatch):
    import bench

    monkeypatch.setenv("MRQ_T4_GPT", "4")
    G, R, K, batches = 4096, 5, 20, 250
    st0 = bench.steady_state(G, R, 0, bench.SEED)
    p = preset_trace(3)
    p.max_prop = 32
    ref = Engine(G, R, seed=bench.SEED, inbox_slots=1, heartbeat_tick=ht)
    ref.import_state(st0)
    eng = Engine(G, R, seed=bench.SEED, inbox_slots=K, heartbeat_tick=ht)
    eng.import_state(st0)
    eng.set_tick_mode(4)
    eng.set_write_through(wt)
    base0 = (st0["last_index"] - np.uint64(40)).astype(np.uint64)
    eng.set_packed_base(base0, st0["term"])
    pk = Pack8(st0["self_id"], base0, st0["term"], R)
    t = 0
    for batch in range(batches):
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
        for k in range(K):
            o, d = eng.sync_slot_outputs(k)
            np.testing.assert_array_equal(o, want_out[k], err_msg=f"out words of tick {k} of batch {batch}")
            np.testing.assert_array_equal(d, want_adv[k], err_msg=f"commit advances of tick {k} of batch {batch}")
        if batch % 25 == 24 or batch == batches - 1:
            want, got = ref.export_state(), eng.export_state()
            for c in COLUMNS:
                np.testing.assert_array_equal(got[c], want[c], err_msg=f"column {c} after batch {batch}")
    grown = ref.export_state()["last_index"] - st0["last_index"]
    assert (grown > 0xFFFE).mean() > 0.95, "the logs did not outgrow the 16-bit span: the case misses its point"
    assert (ref.export_state()["role"] == 2).mean() > 0.99, "the leaders should have stayed leaders"
    assert eng.counters()["errors"] == 0 and ref.counters()["errors"] == 0
    ref.close()
    eng.close()
