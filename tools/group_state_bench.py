"""What reading or writing the state of n groups costs, against the whole-engine calls, at 1,048,576 groups x 5 replicas in
tick mode 4.

The engine runs bench.py's steady state on the steady trace (preset 3) with pre-encoded byte frames, in mrq_tick_many
batches of K = 20 ticks after W warm-up ticks (as tools/change_feed_bench.py does).  For n in {1, 256, 16,384, 262,144}
random distinct groups it times, on the host clock around the blocking call:

  1. mrq_export_groups of the status columns against mrq_export_state of the same columns;
  2. mrq_import_groups of those columns (the groups' current rows) against mrq_import_state of them;
  3. with CUDA events, the first mrq_tick_many batch after each call (and after no call): a whole-engine import leaves
     every group to be re-compacted by that batch.

Every run starts from the same state.  Runs alternate five times (the order reverses every other run).  Prints one JSON
line with the GPU's name and power limit.

    python tools/group_state_bench.py [--reps 5] [--steps 20] [--warmup 3]
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

STATUS = ("term", "vote", "committed", "last_index", "role", "lead", "match")  # what a status lookup reads
SIZES = (1, 256, 16384, 262144)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "runs": [round(x, 4) for x in xs]}


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
    eng = Engine(G, R, seed=bench.SEED, inbox_slots=N)
    p = preset_trace(3)

    # a dry run in tick mode 0 gives the trace's inboxes from the steady state; they are encoded as byte frames that stay
    # in their slots
    eng.import_state(st0)
    ibs = []
    for t in range(N):
        eng.gen_trace(p, t, slot=t)
        eng.tick(t)
        ibs.append(eng.read_inbox(t))
    eng.set_tick_mode(4)
    pk = Pack8(st0["self_id"], base0, st0["term"], R)
    for t, ib in enumerate(ibs):
        eng.post_inbox_packed(*pk.frame(ib), slot=t, keep=True)

    rng = np.random.default_rng(0x6E0E)
    lists = {n: np.sort(rng.choice(G, size=n, replace=False)).astype(np.uint64) for n in SIZES}

    def leg(how, n):
        """rewind, W warm-up ticks (the compact state goes live), the call, then K timed ticks"""
        eng.set_tick_mode(0)
        eng.import_state(st0)
        eng.tick_count = 0
        eng.set_tick_mode(4)
        eng.set_packed_base(base0, st0["term"])
        eng.tick_many(list(range(W)))
        eng.synchronize()
        groups = lists.get(n)
        if how == "import_groups":
            rows = eng.export_groups(groups, STATUS)
        elif how == "import_state":
            full = eng.export_state(STATUS)
        t0 = time.perf_counter()
        if how == "export_groups":
            eng.export_groups(groups, STATUS)
        elif how == "export_state":
            eng.export_state(STATUS)
        elif how == "import_groups":
            eng.import_groups(groups, rows)
        elif how == "import_state":
            eng.import_state(full)
        call_ms = (time.perf_counter() - t0) * 1e3
        eng.timer_start()
        eng.tick_many(list(range(W, N)))
        tick_ms = eng.timer_stop()
        return call_ms, tick_ms

    plan = [("none", None), ("export_state", None), ("import_state", None)]
    plan += [(how, n) for n in SIZES for how in ("export_groups", "import_groups")]
    for how, n in plan:  # rehearsal: module loads, descriptor tables, staging buffers
        leg(how, n)
    res = {f"{how}" + (f" n={n}" if n else ""): {"call_ms": [], "next_batch_ms": []} for how, n in plan}
    for rep in range(args.reps):
        for how, n in (plan if rep % 2 == 0 else plan[::-1]):
            c, t = leg(how, n)
            r = res[f"{how}" + (f" n={n}" if n else "")]
            r["call_ms"].append(c)
            r["next_batch_ms"].append(t)
    out = {k: {"call_ms": stats(v["call_ms"]), "next_batch_ms": stats(v["next_batch_ms"])} for k, v in res.items()}
    eng.close()
    print(json.dumps({"gpu": gpu_info(), "groups": G, "replicas": R, "K": K, "tick_mode": 4, "columns": STATUS, "results": out}))


if __name__ == "__main__":
    main()
