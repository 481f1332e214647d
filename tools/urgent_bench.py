#!/usr/bin/env python
"""urgent_bench.py -- the check and replan of tools/replan_bench.py made urgent (include/ualm.h, ualm_set_urgent) against not urgent,
alternated in one run, on both paths.

    python tools/urgent_bench.py [--batches 12] [--warmup 2] [--rounds 2] [--period-ms 250] [--precisions 64,32] [--margin 0.8]
                                 [--horizon 1.0] [--max-rows 32]

Workload: that of tools/replan_bench.py (four environments, 1024 problems per batch, pipelined at depth 3 on the parity path and 8 on the
throughput path, environment 0's 2 m x 2 m window written every `period-ms`; after each update the last delivered batch is checked from
half its duration with the limits at `margin`, and the `max-rows` rows with the earliest first violation within `horizon` s are
replanned on the same lane ring).  Per precision, `rounds` pairs of arms, not urgent then urgent, each on a fresh context after `warmup`
batches.  Reported per arm and per mode over its arms: the check call's and the replan call's p50 / max, the replanned tickets'
submit-to-delivery p50 / p99 (polled every 2 ms), converged traj/s of the main stream.  Prints one JSON line with the card's name and
power limit read in the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from check_bench import BOXES, mid_t_from  # noqa: E402
from map_update_bench import NAMES, device  # noqa: E402
from replan_bench import NX, NY, Server, flagged, margin_limits, ms_stats  # noqa: E402


class UrgentServer(Server):
    """replan_bench's server with its check and replan made urgent or not, and the check call timed too"""

    def __init__(self, *a, urgent=False, **k):
        super().__init__(*a, **k)
        self.urgent, self.check_call = urgent, []

    def update(self):
        ix0, iy0 = BOXES[self.k % len(BOXES)]
        self.opt.update_environment_window(ix0, iy0, self.windows[self.k % 2][self.k % len(BOXES)], env=0)
        self.k += 1
        if not self.replan or self.last is None:
            return
        last = self.last
        tf = mid_t_from(self.mixed, last[0])
        t = time.perf_counter()
        chk = self.opt.check_results(self.mixed, last, t_from=tf, limits=self.limits, urgent=self.urgent)
        self.check_call.append(time.perf_counter() - t)
        rows = flagged(chk, tf, self.horizon)
        self.flagged.append(int(rows.size))
        if self.max_rows > 0:
            rows = np.sort(rows[:self.max_rows])
        self.rows.append(int(rows.size))
        if rows.size == 0:
            return
        if len(self.flight) == self.depth:
            self._wait_oldest()
        t = time.perf_counter()
        ticket, new = self.opt.submit_replan(self.mixed, last, rows, tf[rows], depth=self.depth, urgent=self.urgent)
        self.call.append(time.perf_counter() - t)
        self.flight.append((ticket, new, t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--period-ms", type=float, default=250.0)
    ap.add_argument("--precisions", default="64,32")
    ap.add_argument("--margin", type=float, default=0.8)
    ap.add_argument("--horizon", type=float, default=1.0)
    ap.add_argument("--max-rows", type=int, default=32, dest="max_rows")
    args = ap.parse_args()

    import torch
    from uneven_planner_b200 import api, configs, maps, problems
    if not torch.cuda.is_available():
        raise SystemExit("urgent_bench.py: no CUDA device")
    ms_, params, pbs, src = [], [], [], {}
    for name in NAMES:
        m = maps.get_terrain(name)
        src[name] = "reference" if m is not None else "stand-in"
        m = m or maps.stand_in_terrain(name)
        ms_.append(m); params.append(configs.params_for(name, overrides=False))
        pbs.append(problems.generate(m, 256, seed=0, **configs.gen_kwargs(name)))
    cat = problems.concat(pbs, range(len(NAMES)))
    mixed = cat.select(np.arange(cat.B).reshape(len(NAMES), -1).T.reshape(-1))     # interleaved
    other = maps.stand_in_terrain("mountain")
    windows = [[np.ascontiguousarray(g.cells[b[0]:b[0] + NX, b[1]:b[1] + NY]) for b in BOXES] for g in (other, ms_[0])]
    limits = margin_limits(params[0], args.margin)

    def context(prec):
        opt = api.BatchALMTrajOpt(precision=prec)
        for e in range(len(NAMES)):
            opt.init(params[e], env=e).set_environment(ms_[e], env=e)
        return opt

    out = {"device": device(), "grids": src, "problems_per_batch": int(mixed.B), "batches": args.batches, "rounds": args.rounds,
           "period_ms": args.period_ms, "margin": args.margin, "horizon_s": args.horizon, "max_rows": args.max_rows}
    for prec in [int(p) for p in args.precisions.split(",")]:
        depth = 3 if prec == 64 else 8
        res = {"depth": depth, "arms": []}
        pooled = {False: {"check": [], "replan": [], "deliver": [], "tps": []}, True: {"check": [], "replan": [], "deliver": [], "tps": []}}
        for rnd in range(args.rounds):
            for urgent in (False, True):
                opt = context(prec)
                Server(opt, mixed, depth, windows, limits, args.horizon, False).run(args.warmup, 0.0)
                torch.cuda.synchronize()
                s = UrgentServer(opt, mixed, depth, windows, limits, args.horizon, True, args.max_rows, urgent=urgent)
                tps = s.run(args.batches, args.period_ms / 1e3)
                opt.close()
                r = {"round": rnd, "urgent": urgent, "converged_traj_per_s": tps, "rows_per_update": s.rows, "check_call": ms_stats(s.check_call),
                     "replan_call": ms_stats(s.call), "submit_to_delivery": ms_stats(s.deliver, (50, 99))}
                res["arms"].append(r)
                p = pooled[urgent]
                p["check"] += s.check_call; p["replan"] += s.call; p["deliver"] += s.deliver; p["tps"].append(tps)
                print(prec, json.dumps(r), file=sys.stderr, flush=True)
        for urgent in (False, True):
            p = pooled[urgent]
            res["urgent" if urgent else "not_urgent"] = {"check_call": ms_stats(p["check"]), "replan_call": ms_stats(p["replan"]),
                                                         "submit_to_delivery": ms_stats(p["deliver"], (50, 99)),
                                                         "converged_traj_per_s": [float(x) for x in p["tps"]]}
        out["precision_%d" % prec] = res
        print(prec, json.dumps({k: v for k, v in res.items() if k != "arms"}), file=sys.stderr, flush=True)
    out["device_after"] = device()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
