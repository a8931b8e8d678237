"""What resizing a running engine's group count costs, at 1,048,576 groups x 5 replicas in tick mode 4.

The engine runs bench.py's steady state on the steady trace (preset 3) with pre-encoded byte frames that stay in their
slots, in mrq_tick_many batches of K = 20 ticks after W warm-up ticks (as tools/group_state_bench.py does).  Every leg
starts from the same state with the compact state live, then times on the host clock around the blocking call:

  1. "within stride": a grow from 1,048,476 to 1,048,576 groups (stride 1,048,576 before and after);
  2. "1048000": a grow from 1,048,000 to 1,048,576 groups (the stride moves from 1,048,064 to 1,048,576);
  3. "grow 131072": a grow from 1,048,576 to 1,179,648 groups, and the shrink back right after the batch below;
  4. "shrink 131072": a shrink from 1,048,576 to 917,504 groups;
  5. "shrink within stride": a shrink from 1,048,576 to 1,048,476 groups: no fresh group, no buffer moves;
(the engine is first shrunk untimed where a leg starts below 1,048,576), and with CUDA events the next K-tick batch, with
its kernel launches: 2 means nothing was re-compacted.  A resize clears the inbox slots, so every leg, "none" included,
posts the frames again and synchronises (untimed) before that batch: the same frames, with the new groups' bytes 0 (no
message) and without the dropped groups' columns.  The new groups are fresh followers: those whose election timeout
falls inside the batch campaign on the general path, which a fresh engine of that size would do too.  Legs 4 and 5 have
no fresh groups; where the buffers move (legs 2-4) the batch also rebuilds its mode-4 descriptor table.

Runs alternate five times (the order reverses every other run).  Prints one JSON line with the GPU's name and power
limit.

    python tools/resize_bench.py [--reps 5] [--steps 20] [--warmup 3]
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

GROW = 131072
STARTS = {"within stride": 100, "1048000": 576}  # groups below 1,048,576 where the grow starts


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

    # a dry run in tick mode 0 gives the trace's inboxes from the steady state, encoded once as byte frames
    eng.import_state(st0)
    ibs = []
    for t in range(N):
        eng.gen_trace(p, t, slot=t)
        eng.tick(t)
        ibs.append(eng.read_inbox(t))
    pk = Pack8(st0["self_id"], base0, st0["term"], R)
    frames = [pk.frame(ib) for ib in ibs]

    def reshaped(n, silent=0):
        """the frames for n groups: groups [G, n) and the last `silent` groups below G without messages, groups >= n
        cut off"""
        quiet = min(n, G) - silent
        out = []
        for word, p8, wide in frames:
            w = np.zeros((word.shape[0], n), np.uint8)
            w[:, :quiet] = word[:, :quiet]
            q = None
            if p8 is not None:
                q = np.zeros(n, np.uint8)
                q[:quiet] = p8[:quiet]
            out.append((w, q, [m for m in wide if m[0] < quiet]))
        return out

    big, small, within = reshaped(G + GROW), reshaped(G - GROW), reshaped(G - STARTS["within stride"])
    starts = {how: reshaped(G, d) for how, d in STARTS.items()}

    def post(fs):
        for t, (w, q, wide) in enumerate(fs):
            eng.post_inbox_packed(w, q, wide, slot=t, keep=True)
        eng.synchronize()

    def rewind():
        eng.set_tick_mode(0)
        eng.resize_groups(G)
        eng.import_state(st0)
        eng.tick_count = 0
        eng.set_tick_mode(4)
        eng.set_packed_base(base0, st0["term"])
        post(frames)
        eng.tick_many(list(range(W)))  # the compact state goes live
        eng.synchronize()

    def resize(n):
        t0 = time.perf_counter()
        eng.resize_groups(n)
        return (time.perf_counter() - t0) * 1e3

    def timed_batch():
        eng.timer_start()
        eng.tick_many(list(range(W, N)))
        return eng.timer_stop()

    def batch(r, fs):
        """post the frames again, then the first batch after the resize"""
        post(fs)
        l0 = eng.counters()["kernel_launches"]
        r["next_batch_ms"] = timed_batch()
        r["next_batch_launches"] = eng.counters()["kernel_launches"] - l0

    def leg(how):
        rewind()
        r = {}
        if how == "none":
            batch(r, frames)
        elif how in STARTS:
            eng.resize_groups(G - STARTS[how])
            r["call_ms"] = resize(G)
            batch(r, starts[how])
        elif how == "grow 131072":
            r["call_ms"] = resize(G + GROW)
            batch(r, big)
            r["shrink_back_call_ms"] = resize(G)
        elif how == "shrink 131072":
            r["call_ms"] = resize(G - GROW)
            batch(r, small)
        else:
            r["call_ms"] = resize(G - STARTS["within stride"])
            batch(r, within)
        return r

    plan = ["none", "within stride", "1048000", "grow 131072", "shrink 131072", "shrink within stride"]
    for how in plan:  # rehearsal: module loads, descriptor tables, staging buffers
        leg(how)
    res = {how: {} for how in plan}
    for rep in range(args.reps):
        for how in (plan if rep % 2 == 0 else plan[::-1]):
            for k, v in leg(how).items():
                res[how].setdefault(k, []).append(v)
    out = {how: {k: stats(v) for k, v in r.items()} for how, r in res.items()}
    eng.close()
    print(json.dumps({"gpu": gpu_info(), "groups": G, "replicas": R, "K": K, "tick_mode": 4, "grow": GROW,
                      "results": out}))


if __name__ == "__main__":
    main()
