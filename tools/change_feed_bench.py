"""What the change feed costs, and what it saves, at 1,048,576 groups x 5 replicas in tick mode 4.

Three things are timed with mrq_tick_many batches of K = 20 ticks on pre-encoded byte frames (bench.py's steady state and
frame builder, by import):

  1. the steady trace (preset 3), feed off vs on: CUDA-event time of the K ticks (no group changes term, vote, role or
     lead there, so the feed must be free);
  2. a churn trace (preset 5's churn and vote parameters) from the same state, feed off vs on, plus the host time of one
     mrq_sync_changes per K ticks;
  3. what a host pays without the feed to learn the same: export_state(term, vote, role, lead) after every K ticks.

Runs alternate five times per trace (off, on, export; then on, off, export).  Prints one JSON line with the GPU's name and power limit.

    python tools/change_feed_bench.py [--reps 5] [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from raftsql_b200 import Engine, preset_trace  # noqa: E402
from raftsql_b200.packed import Pack8  # noqa: E402

HARD_SOFT = ("term", "vote", "role", "lead")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "runs": [round(x, 3) for x in xs]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    G, R, K, W = bench.G_TOTAL, bench.R, args.steps, args.warmup
    N = W + K
    st0 = bench.steady_state(G, R, 0, bench.SEED)
    base0 = (st0["last_index"] - np.uint64(40)).astype(np.uint64)
    eng = Engine(G, R, seed=bench.SEED, inbox_slots=2 * N)
    traces = {"steady": (preset_trace(3), 0), "churn": (preset_trace(5), N)}

    # dry runs in tick mode 0: each trace's inboxes tick by tick from the steady state, encoded as byte frames kept in
    # their slots (slots [0, N) steady, [N, 2N) churn)
    ibs = {}
    for name, (p, s0) in traces.items():
        eng.set_tick_mode(0)
        eng.import_state(st0)
        eng.tick_count = 0
        ibs[name] = []
        for t in range(N):
            eng.gen_trace(p, t, slot=s0 + t)
            eng.tick(s0 + t)
            ibs[name].append(eng.read_inbox(s0 + t))
    eng.set_tick_mode(4)  # (a byte frame posted in tick mode 4 stays a frame; in modes 0-2 it is unpacked)
    n_escapes = {}
    for name, (_, s0) in traces.items():
        pk = Pack8(st0["self_id"], base0, st0["term"], R)
        n_escapes[name] = 0
        for t, ib in enumerate(ibs[name]):
            w8, p8, wide = pk.frame(ib)
            n_escapes[name] += len(wide)
            eng.post_inbox_packed(w8, p8, wide, slot=s0 + t, keep=True)

    def rewind(cap):
        eng.set_tick_mode(0)
        eng.import_state(st0)
        eng.tick_count = 0
        eng.set_tick_mode(4)
        eng.set_packed_base(base0, st0["term"])
        eng.set_change_capacity(cap)

    def leg(s0, how):
        """one run: W warm-up ticks, then K timed ticks; how = off / on / export"""
        rewind(G if how == "on" else 0)
        eng.tick_many(list(range(s0, s0 + W)))
        if how == "on":
            eng.sync_changes()
        eng.synchronize()
        t0 = time.perf_counter()
        eng.timer_start()
        eng.tick_many(list(range(s0 + W, s0 + N)))
        ms = eng.timer_stop()
        t1 = time.perf_counter()
        n_rec, drain_ms = 0, 0.0
        if how == "on":
            recs, lost = eng.sync_changes()
            assert lost == 0
            n_rec = len(recs)
        elif how == "export":
            eng.export_state(HARD_SOFT)
        t2 = time.perf_counter()
        drain_ms = (t2 - t1) * 1e3
        return ms, drain_ms, (t2 - t0) * 1e3, n_rec

    # rehearsal: module loads, descriptor tables
    for name, (_, s0) in traces.items():
        for how in ("off", "on", "export"):
            leg(s0, how)
    res = {}
    for name, (_, s0) in traces.items():
        r = {how: {"tick_ms": [], "drain_ms": [], "round_ms": [], "records": []} for how in ("off", "on", "export")}
        for rep in range(args.reps):
            for how in (("off", "on", "export") if rep % 2 == 0 else ("on", "off", "export")):
                ms, dms, rms, n = leg(s0, how)
                r[how]["tick_ms"].append(ms)
                r[how]["drain_ms"].append(dms)
                r[how]["round_ms"].append(rms)
                r[how]["records"].append(n)
        res[name] = {
            "escaped_messages": n_escapes[name],
            "us_per_tick_feed_off": stats([x / K * 1e3 for x in r["off"]["tick_ms"]]),
            "us_per_tick_feed_on": stats([x / K * 1e3 for x in r["on"]["tick_ms"]]),
            "records_per_K_ticks": r["on"]["records"],
            "sync_changes_ms_per_K_ticks": stats(r["on"]["drain_ms"]),
            "export_hard_soft_state_ms_per_K_ticks": stats(r["export"]["drain_ms"]),
            "round_ms_ticks_plus_drain": stats(r["on"]["round_ms"]),
            "round_ms_ticks_plus_export": stats(r["export"]["round_ms"]),
        }
    eng.close()
    print(json.dumps({"gpu": gpu_info(), "groups": G, "replicas": R, "K": K, "tick_mode": 4, "results": res}))


if __name__ == "__main__":
    main()
