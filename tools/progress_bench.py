#!/usr/bin/env python
"""progress_bench.py -- what a batch in flight gets done while the host does something else (DESIGN 3g).

    python tools/progress_bench.py [--steps 6] [--warmup 2] [--out result.json]

Only existing entry points are used, so the same script runs on any commit that has ualm_poll_batch.  Every arm runs on the throughput
path (precision 32, depth 8) and on the parity path (precision 64, depth 3) as the reference, with the hill parameters on the hill
terrain or its stand-in ("bumps", seed 0):

1. host-busy server loop: batch k+1 is planned with ualm_front_end_batch (256 random (start, goal) pairs, every host thread) while
   batch k is in flight; after each plan every ticket in flight is polled once (wait_ms = 0) and a ticket is waited once it has
   returned every problem (or when its lane is needed).  Reported: converged trajectories per second of wall time and the p50 / p99
   latency from a problem's submit to the poll or wait that returned it.
2. sleep-then-wait: 1024 generated problems, submit, sleep S ms (S = 50, 200), wait.  Reported: the median time from submit to the
   return of wait, and the same without the sleep.
3. sleeping poller: 1024 generated problems per batch through `depth` lanes from one thread that polls (wait_ms = 1) every ticket in
   turn and sleeps 1 ms between rounds of polls.  Reported: converged per second and p50 / p99 latency.

Every lane takes a batch before the timed region of arms 1 and 3.  Every arm also reports the p50 / max time of the timed submit calls.  Prints one JSON line with the card's name, power limit and
maximum SM clock, read in the same run.
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


def pct(a, q):
    return round(float(np.percentile(a, q)), 2) if len(a) else None


class Ring:
    """tickets in flight: submit time, outputs, per-problem delivery times"""

    def __init__(self, opt, depth):
        self.opt, self.depth, self.live, self.lat, self.conv, self.sub_ms, self.n = opt, depth, [], [], 0, [], 0

    def submit(self, pb, timed):
        # the library's ring: this submit takes the lane of the ticket submitted `depth` submits ago, which must be waited first
        if self.live and self.live[0]["n"] == self.n - self.depth:
            self.finish(self.live[0])
        t0 = time.perf_counter()
        t = self.opt.submit(pb, depth=self.depth)
        if timed:
            self.sub_ms.append(1e3 * (time.perf_counter() - t0))
        self.n += 1
        self.live.append({"n": self.n - 1, "t": t, "pb": pb, "t0": t0, "out": self.opt.outputs(pb), "got": np.full(pb.B, np.nan), "timed": timed})

    def poll(self, k, wait_ms):
        idx, pending = self.opt.poll(k["t"], k["out"], wait_ms)
        k["got"][idx] = time.perf_counter()
        return pending

    def finish(self, k):
        self.opt.wait(k["t"], out=k["out"])
        now = time.perf_counter()
        k["got"][np.isnan(k["got"])] = now
        self.live.remove(k)
        if k["timed"]:
            self.lat.extend((1e3 * (k["got"] - k["t0"])).tolist())
            self.conv += sum(1 for r in k["out"][0] if r.ret_code == 0)

    def poll_all(self, wait_ms):
        for k in list(self.live):
            if self.poll(k, wait_ms) == 0:
                self.finish(k)

    def drain(self, wait_ms=1.0):
        while self.live:
            self.poll_all(wait_ms)

    def report(self, wall):
        return {"converged_per_s": round(self.conv / wall, 1), "latency_ms": {"p50": pct(self.lat, 50), "p99": pct(self.lat, 99)},
                "submit_ms": {"p50": pct(self.sub_ms, 50), "max": round(max(self.sub_ms), 2)}, "wall_s": round(wall, 3)}


def host_busy(opt, view, depth, steps, warmup, front_end):
    rng = np.random.default_rng(0)

    def plan():
        s = np.column_stack([rng.uniform(-4.3, 4.3, 256), rng.uniform(-4.3, 4.3, 256), rng.uniform(-np.pi, np.pi, 256)])
        g = np.column_stack([rng.uniform(-4.3, 4.3, 256), rng.uniform(-4.3, 4.3, 256), rng.uniform(-np.pi, np.pi, 256)])
        return front_end.plan_batch(view, s, g)[0]
    ring, nxt, plan_ms = Ring(opt, depth), plan(), []
    warmup = max(warmup, depth)            # every lane once: the first batch on a lane sets its group loops up
    for k in range(warmup + steps):
        if k == warmup:
            ring.drain()
            wall0 = time.perf_counter()
        ring.submit(nxt, k >= warmup)
        t0 = time.perf_counter()
        nxt = plan()
        plan_ms.append(1e3 * (time.perf_counter() - t0))
        ring.poll_all(0.0)
    ring.drain()
    r = ring.report(time.perf_counter() - wall0)
    r["plan_ms_p50"] = pct(plan_ms, 50)
    return r


def sleep_then_wait(opt, pb, reps=3):
    out = {}
    opt.wait(opt.submit(pb, depth=1))
    for S in (0, 50, 200):
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            t = opt.submit(pb, depth=1)
            time.sleep(S / 1e3)
            opt.wait(t)
            ts.append(1e3 * (time.perf_counter() - t0))
        out["sleep_%d_ms" % S] = round(float(np.median(ts)), 2)
    return out


def sleeping_poller(opt, pb, depth, steps, warmup):
    ring = Ring(opt, depth)
    for k in range(max(warmup, depth)):
        ring.submit(pb, False)
    ring.drain()
    wall0 = time.perf_counter()
    k = 0
    while k < steps or ring.live:
        while k < steps and len(ring.live) < depth:
            ring.submit(pb, True)
            k += 1
        ring.poll_all(1.0)
        time.sleep(1e-3)
    return ring.report(time.perf_counter() - wall0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import torch
    from uneven_planner_b200 import api, configs, front_end, maps, problems
    if not torch.cuda.is_available():
        raise SystemExit("progress_bench.py: no CUDA device")
    m = maps.get_terrain("hill") or maps.synthetic_terrain("bumps", seed=0)
    params = configs.params_for("hill")
    pb = problems.generate(m, 1024, seed=0, **configs.gen_kwargs("hill"))
    view = front_end.MapView(m)
    arms = []
    for precision, depth in ((32, 8), (64, 3)):
        opt = api.BatchALMTrajOpt(precision=precision).init(params).set_environment(m)
        arm = {"precision": precision, "depth": depth,
               "host_busy": host_busy(opt, view, depth, args.steps, args.warmup, front_end),
               "sleep_then_wait": sleep_then_wait(opt, pb),
               "sleeping_poller": sleeping_poller(opt, pb, depth, 2 * args.steps, args.warmup)}
        opt.close()
        arms.append(arm)
        print(json.dumps(arm), file=sys.stderr)
    line = json.dumps({"device": device(), "workload": "hill parameters on %s; host-busy: 256 front-end pairs per batch; other arms: %d generated problems per batch"
                       % (m.name, pb.B), "arms": arms})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
