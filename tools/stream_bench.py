#!/usr/bin/env python
"""stream_bench.py -- when each trajectory of a submitted batch becomes available to its caller: waiting for the whole batch
(ualm_wait_batch) against collecting problems as they finish (ualm_poll_batch with wait_ms = 1 in a loop).

    python tools/stream_bench.py [--steps 8] [--warmup 3] [--out result.json]

Workload: BASELINE configs[1]'s recipe, 1024 problems per batch with the hill parameters on the hill terrain (or the labelled
synthetic stand-in tools/budget_bench.py uses without it).  Arms: the parity path at depth 1 and 3, the throughput path at
precision 32 and depth 8; each in both modes.  `warmup + steps` batches go through a ring of `depth` lanes; for the `steps` timed
batches it reports, per problem, the availability latency (host time from the submit of its batch to the return of the call that
handed it back: the wait in wait mode, the poll in poll mode) as p50 / p90 / p99 / max, and converged trajectories per second of
wall time.  Both modes return the same bits (tests/test_gpu_stream.py); this only measures when.  Prints one JSON line with the
card's name, power limit and maximum SM clock, read in the same run.
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


def run(opt, pb, depth, mode, steps, warmup):
    """`warmup + steps` batches through `depth` lanes; latencies (ms) of the timed batches' problems, converged count, wall seconds"""
    B = pb.B
    host = [np.ascontiguousarray(a) for a in (pb.N.astype(np.int32), pb.M.astype(np.int32), pb.bnd.astype(np.float64), pb.total_time.astype(np.float64),
                                              pb.inner_xy.astype(np.float64), pb.inner_yaw.astype(np.float64))]
    outs = [opt.outputs(pb) for _ in range(depth)]
    total = warmup + steps
    inflight, done = [], set()
    lat, conv = [], 0
    state = {"next": 0, "t_start": None, "t_end": None}

    def submit_ready():
        # the ring reuses the lane of batch k - depth: submit only once that batch has been waited
        while state["next"] < total and len(inflight) < depth and (state["next"] < depth or state["next"] - depth in done):
            k = state["next"]
            t0 = time.perf_counter()
            t = opt.submit(pb, depth=depth, host=host)
            if k == warmup:
                state["t_start"] = t0
            inflight.append({"t": t, "t0": t0, "k": k, "out": outs[k % depth], "pending": B})
            state["next"] += 1

    def finish(f):
        nonlocal conv
        res, _, _ = opt.wait(f["t"], out=f["out"])
        now = time.perf_counter()
        if f["k"] >= warmup:
            conv += sum(1 for r in res if r.ret_code == 0)
            if mode == "wait":
                lat.extend([(now - f["t0"]) * 1e3] * B)
            state["t_end"] = now
        inflight.remove(f)
        done.add(f["k"])

    submit_ready()
    while inflight:
        if mode == "wait":
            finish(inflight[0])
        else:
            for f in list(inflight):
                idx, f["pending"] = opt.poll(f["t"], f["out"], 1.0)
                now = time.perf_counter()
                if f["k"] >= warmup:
                    lat.extend([(now - f["t0"]) * 1e3] * idx.size)
                if f["pending"] == 0:
                    finish(f)
        submit_ready()
    return np.array(lat), conv, state["t_end"] - state["t_start"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import torch
    from uneven_planner_b200 import api, configs, maps, problems
    if not torch.cuda.is_available():
        raise SystemExit("stream_bench.py: no CUDA device")
    m = maps.get_terrain("hill") or maps.synthetic_terrain("bumps", seed=0)
    params = configs.params_for("hill")
    pb = problems.generate(m, 1024, seed=0, **configs.gen_kwargs("hill"))
    arms = []
    for precision, depth in ((64, 1), (64, 3), (32, 8)):
        opt = api.BatchALMTrajOpt(precision=precision).init(params).set_environment(m)
        arm = {"precision": precision, "depth": depth}
        for mode in ("wait", "poll"):
            lat, conv, wall = run(opt, pb, depth, mode, args.steps, args.warmup)
            arm[mode] = {"latency_ms": {q: round(float(np.percentile(lat, int(q[1:]))), 2) for q in ("p50", "p90", "p99")} | {"max": round(float(lat.max()), 2)},
                         "converged_per_s": round(conv / wall, 1), "converged_per_batch": conv / args.steps, "wall_s": round(wall, 3)}
        opt.close()
        arms.append(arm)
        print(json.dumps(arm), file=sys.stderr)
    line = json.dumps({"device": device(), "workload": "%d problems per batch, %s, hill parameters, %d timed batches after %d" % (pb.B, m.name, args.steps, args.warmup),
                       "poll_wait_ms": 1.0, "arms": arms})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
