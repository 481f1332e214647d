#!/usr/bin/env python
"""cancel_bench.py -- what cancelling problems of a batch in flight (ualm_cancel_problems) buys a server.

    python tools/cancel_bench.py [--steps 6] [--warmup 2] [--out result.json]

Workload: 1024 problems per batch with the hill parameters on the synthetic terrain ("bumps", seed 0), on the parity path at depth 1
and 3 and the throughput path at precision 32 and depth 8 (the depths of tools/stream_bench.py).  `warmup + steps` batches go
through a ring of `depth` lanes; each batch is polled (wait_ms = 1) until it is drained.  Two arms:

1. Withdrawn requests: a seeded random fraction f of every batch is cancelled right after its submit.  Reported: the mean time from a
   batch's submit to the delivery of its last problem that was not withdrawn, and converged trajectories per second of wall time
   over the problems not withdrawn.  Against the same batches without cancels (the same problems counted) and against batches that
   never held the withdrawn problems.
2. Per-request deadlines: every request of a batch is due D ms after its batch's submit.  The poll loop cancels the pending requests
   of a ticket once their deadline has passed.  Reported: p50 / p99 / max latency (submit to the poll that returned the problem),
   the fraction delivered by the deadline, the fraction converged and converged trajectories per second.  Against
   ualm_wait_batch_for with the same D per batch (every problem's latency is then its batch's wait).

Prints one JSON line with the card's name, power limit and maximum SM clock, read in the same run.
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


def device():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception:
        return None


def run(opt, pb, depth, steps, warmup, withdraw=None, deadline_ms=None, wait_for=False):
    """`warmup + steps` batches of `pb` through `depth` lanes, each polled until drained (or waited with ualm_wait_batch_for when
    `wait_for`).  withdraw: problem indices cancelled right after each submit; deadline_ms: cancel a ticket's pending problems once
    that much time has passed since its submit.  Returns per timed batch (latency ms per problem, records) and the wall seconds of the
    timed batches."""
    host = [np.ascontiguousarray(a) for a in (pb.N.astype(np.int32), pb.M.astype(np.int32), pb.bnd.astype(np.float64), pb.total_time.astype(np.float64),
                                              pb.inner_xy.astype(np.float64), pb.inner_yaw.astype(np.float64))]
    outs = [opt.outputs(pb) for _ in range(depth)]
    total = warmup + steps
    inflight, done, batches = [], set(), []
    state = {"next": 0, "t_start": None, "t_end": None}

    def submit_ready():
        while state["next"] < total and len(inflight) < depth and (state["next"] < depth or state["next"] - depth in done):
            k = state["next"]
            t0 = time.perf_counter()
            t = opt.submit(pb, depth=depth, host=host)
            if withdraw is not None and withdraw.size:
                opt.cancel(t, withdraw)
            if k == warmup:
                state["t_start"] = t0
            inflight.append({"t": t, "t0": t0, "k": k, "out": outs[k % depth], "pending": pb.B, "lat": np.full(pb.B, np.nan), "cut": False})
            state["next"] += 1

    def finish(f, timeout=None):
        res, _, _ = opt.wait(f["t"], out=f["out"], timeout_ms=timeout)
        now = time.perf_counter()
        if wait_for:
            f["lat"][:] = (now - f["t0"]) * 1e3
        if f["k"] >= warmup:
            batches.append((f["lat"].copy(), [(r.ret_code, r.n_evals) for r in res]))
            state["t_end"] = now
        inflight.remove(f)
        done.add(f["k"])

    submit_ready()
    while inflight:
        if wait_for:
            f = inflight[0]
            finish(f, max(0.0, deadline_ms - (time.perf_counter() - f["t0"]) * 1e3))
        else:
            for f in list(inflight):
                idx, f["pending"] = opt.poll(f["t"], f["out"], 1.0)
                now = time.perf_counter()
                f["lat"][idx] = (now - f["t0"]) * 1e3
                if deadline_ms is not None and f["pending"] and not f["cut"] and (now - f["t0"]) * 1e3 >= deadline_ms:
                    opt.cancel(f["t"], np.flatnonzero(np.isnan(f["lat"])))
                    f["cut"] = True
                if f["pending"] == 0:
                    finish(f)
        submit_ready()
    return batches, state["t_end"] - state["t_start"]


def summary(batches, wall, keep=None, deadline_ms=None):
    """over the problems `keep` (default all) of the timed batches"""
    lat = np.concatenate([b[0] if keep is None else b[0][keep] for b in batches])
    rc = np.concatenate([np.array([r[0] for r in b[1]]) if keep is None else np.array([r[0] for r in b[1]])[keep] for b in batches])
    last = [float(np.nanmax(b[0] if keep is None else b[0][keep])) for b in batches]
    s = {"latency_ms": {q: round(float(np.percentile(lat, int(q[1:]))), 2) for q in ("p50", "p99")} | {"max": round(float(lat.max()), 2)},
         "last_delivered_ms_mean": round(float(np.mean(last)), 2), "converged_fraction": round(float((rc == 0).mean()), 4),
         "stopped_fraction": round(float((rc == 3).mean()), 4), "converged_per_s": round(float((rc == 0).sum()) / wall, 1), "wall_s": round(wall, 3)}
    if deadline_ms is not None:
        s["delivered_by_deadline"] = round(float((lat <= deadline_ms).mean()), 4)
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import torch
    from uneven_planner_b200 import api, configs, maps, problems
    if not torch.cuda.is_available():
        raise SystemExit("cancel_bench.py: no CUDA device")
    m = maps.synthetic_terrain("bumps", seed=0)
    params = configs.params_for("hill")
    pb = problems.generate(m, 1024, seed=0, **configs.gen_kwargs("hill"))
    rng = np.random.default_rng(7)
    arms = []
    for precision, depth in ((64, 1), (64, 3), (32, 8)):
        opt = api.BatchALMTrajOpt(precision=precision).init(params).set_environment(m)
        arm = {"precision": precision, "depth": depth, "withdrawn": [], "deadline": []}
        base, base_wall = run(opt, pb, depth, args.steps, args.warmup)
        arm["no_cancel"] = summary(base, base_wall)
        for f in (0.25, 0.5):
            cut = np.sort(rng.choice(pb.B, int(f * pb.B), replace=False))
            keep = np.setdiff1d(np.arange(pb.B), cut)
            b, w = run(opt, pb, depth, args.steps, args.warmup, withdraw=cut)
            kb = pb.select(keep)
            kept, kw = run(opt, kb, depth, args.steps, args.warmup)
            arm["withdrawn"].append({"fraction": f, "cancelled": summary(b, w, keep), "no_cancel_same_problems": summary(base, base_wall, keep),
                                     "never_held": summary(kept, kw)})
            print(json.dumps({"precision": precision, "depth": depth, "withdrawn": arm["withdrawn"][-1]}), file=sys.stderr)
        for D in (100.0, 200.0):
            b, w = run(opt, pb, depth, args.steps, args.warmup, deadline_ms=D)
            wb, ww = run(opt, pb, depth, args.steps, args.warmup, deadline_ms=D, wait_for=True)
            arm["deadline"].append({"D_ms": D, "poll_and_cancel": summary(b, w, deadline_ms=D), "wait_batch_for": summary(wb, ww, deadline_ms=D)})
            print(json.dumps({"precision": precision, "depth": depth, "deadline": arm["deadline"][-1]}), file=sys.stderr)
        opt.close()
        arms.append(arm)
    line = json.dumps({"device": device(), "workload": "%d problems per batch, %s, hill parameters, %d timed batches after %d" % (pb.B, m.name, args.steps, args.warmup),
                       "poll_wait_ms": 1.0, "arms": arms})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
