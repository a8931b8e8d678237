"""Tick mode 4 on hardware with logs that outgrow the 16-bit offset columns.

The compact columns hold offsets from a per-group base in 16 bits; a group whose log reaches the end of that span is
handed to the general path, which materialises it and re-compacts it on a fresh base (or leaves it wide when it no
longer fits).  The steady trace proposes 1.5 entries a tick and takes ~43k ticks to get there, so this trace proposes
up to 32 a tick: every leader's log grows past 2^16 entries from its first base within a few thousand ticks.  Run in
mrq_tick_many batches, with write-through on and off and under both kernel shapes, every tick's out words and commit
advances and every state column must equal tick mode 0 fed the same messages from the wide inbox, bit for bit."""
import numpy as np
import pytest

from raftsql_b200 import Engine, preset_trace
from raftsql_b200.packed import Pack8

pytestmark = [pytest.mark.gpu]

SPAN16 = 0xFFFE
COLUMNS = ("term", "vote", "committed", "last_index", "last_term", "term_start", "match", "role", "lead", "election_elapsed",
           "heartbeat_elapsed")


@pytest.mark.parametrize("gpt", ["4", "1"], ids=["4 groups per thread", "1 group per thread"])
@pytest.mark.parametrize("wt", [1, 0], ids=["write-through", "write-back at end"])
def test_mode_4_logs_past_the_16_bit_span_equal_mode_0(gpt, wt, monkeypatch):
    import bench

    monkeypatch.setenv("MRQ_T4_GPT", gpt)
    G, R, K, batches = 4096, 5, 20, 250
    st0 = bench.steady_state(G, R, 0, bench.SEED)
    p = preset_trace(3)
    p.max_prop = 32  # about as many as the 64-entry ack window keeps up with: the groups stay on the fast path
    ref = Engine(G, R, seed=bench.SEED, inbox_slots=1)
    ref.import_state(st0)
    eng = Engine(G, R, seed=bench.SEED, inbox_slots=K)
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
    np.testing.assert_array_equal(eng.sync_out(), ref.sync_out())
    grown = ref.export_state()["last_index"] - st0["last_index"]
    assert (grown > SPAN16).mean() > 0.95, "the logs did not outgrow the 16-bit span: the case misses its point"
    # (not commits_advanced: the general path of a multi-tick launch counts a group's events once per launch, and
    # these groups take it often)
    assert eng.counters()["errors"] == 0 and ref.counters()["errors"] == 0
    ref.close()
    eng.close()
