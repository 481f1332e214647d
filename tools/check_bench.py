#!/usr/bin/env python
"""check_bench.py -- checking the trajectories a server handed out against the current grid after each window update (include/ualm.h,
ualm_check_trajectories), idle and while batches are in flight.

    python tools/check_bench.py [--batches 12] [--warmup 2] [--period-ms 250] [--precisions 64,32] [--idle-reps 10]

Workload: that of tools/map_window_bench.py (four environments, 1024 problems per batch, pipelined at depth 3 on the parity path and 8
on the throughput path).  Every `period-ms` environment 0's 2 m x 2 m window is written from host cells (ualm_update_map_window), and
after each update the 1024 trajectories of the last delivered batch are checked from the middle of each trajectory on.  Arms per
precision: none (no update, no check), updates (updates only), checks (updates and checks).  Before them the check runs `idle-reps`
times with nothing in flight.  The check kernel's time comes from torch.profiler runs (idle and in flight) made after every timed
arm, so the timed runs carry no tracing.  Prints one JSON line with the card's name and power limit read in the same run.
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
from map_update_bench import NAMES, device  # noqa: E402

BOXES = [(80, 80), (90, 80), (90, 90), (80, 90)]      # (ix0, iy0) of the 40 x 40 window
NX = NY = 40


def mid_t_from(pb, res):
    """half of each trajectory's duration: a robot halfway along"""
    return np.array([0.5 * min(int(pb.N[i]) * r.piece_T_xy, int(pb.M[i]) * r.piece_T_yaw) for i, r in enumerate(res)])


class Updater:
    """one window update of environment 0 and, if `check`, the check of the last delivered batch"""

    def __init__(self, opt, windows, mixed, check):
        self.opt, self.windows, self.mixed, self.check = opt, windows, mixed, check
        self.k, self.call, self.last = 0, [], None

    def __call__(self):
        ix0, iy0 = BOXES[self.k % len(BOXES)]
        self.opt.update_environment_window(ix0, iy0, self.windows[self.k % 2][self.k % len(BOXES)], env=0)
        if self.check and self.last is not None:
            t = time.perf_counter()
            self.opt.check_results(self.mixed, self.last, t_from=mid_t_from(self.mixed, self.last[0]))
            self.call.append(time.perf_counter() - t)
        self.k += 1


def run(opt, mixed, depth, batches, update, period):
    """submit `batches` batches at most `depth` in flight, calling update() every `period` s; returns converged traj/s"""
    flight, converged = [], 0
    t0 = time.perf_counter()
    due = t0 + period
    for _ in range(batches):
        if update is not None and time.perf_counter() >= due:
            update()
            due += period
        if len(flight) == depth:
            out = opt.wait(flight.pop(0))
            converged += sum(r.ret_code == 0 for r in out[0])
            if update is not None:
                update.last = out
        flight.append(opt.submit(mixed, depth=depth))
    while flight:
        converged += sum(r.ret_code == 0 for r in opt.wait(flight.pop(0))[0])
    return converged / (time.perf_counter() - t0)


def ms_stats(a):
    a = np.asarray(a) * 1e3
    return {"calls": int(a.size), "call_ms_p50": float(np.percentile(a, 50)) if a.size else None, "call_ms_max": float(a.max()) if a.size else None}


def kernel_ms_per_call(prof, calls):
    """summed device time of check_kernel over the profiled calls, per call (ms)"""
    tot = 0.0
    for e in prof.key_averages():
        if "check_kernel" in e.key:
            tot += getattr(e, "device_time_total", None) or e.cuda_time_total
    return tot / 1e3 / max(calls, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--period-ms", type=float, default=250.0)
    ap.add_argument("--precisions", default="64,32")
    ap.add_argument("--idle-reps", type=int, default=10)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from uneven_planner_b200 import api, configs, maps, problems
    if not torch.cuda.is_available():
        raise SystemExit("check_bench.py: no CUDA device")
    ms_, params, pbs, src = [], [], [], {}
    for name in NAMES:
        m = maps.get_terrain(name)
        src[name] = "reference" if m is not None else "stand-in"
        m = m or maps.stand_in_terrain(name)
        ms_.append(m); params.append(configs.params_for(name, overrides=False))
        pbs.append(problems.generate(m, 256, seed=0, **configs.gen_kwargs(name)))
    cat = problems.concat(pbs, range(len(NAMES)))
    mixed = cat.select(np.arange(cat.B).reshape(len(NAMES), -1).T.reshape(-1))     # interleaved
    # window cells alternate between another terrain's box and environment 0's own
    other = maps.stand_in_terrain("mountain")
    windows = [[np.ascontiguousarray(g.cells[b[0]:b[0] + NX, b[1]:b[1] + NY]) for b in BOXES] for g in (other, ms_[0])]

    def context(prec):
        opt = api.BatchALMTrajOpt(precision=prec)
        for e in range(len(NAMES)):
            opt.init(params[e], env=e).set_environment(ms_[e], env=e)
        return opt

    out = {"device": device(), "grids": src, "problems_per_batch": int(mixed.B), "batches": args.batches, "period_ms": args.period_ms,
           "window": [NX, NY]}
    precs = [int(p) for p in args.precisions.split(",")]
    for prec in precs:
        depth = 3 if prec == 64 else 8
        res = {"depth": depth}
        opt = context(prec)
        last = opt.optimize(mixed)
        tf = mid_t_from(mixed, last[0])
        calls = []
        for k in range(args.idle_reps + 1):
            t = time.perf_counter()
            chk = opt.check_results(mixed, last, t_from=tf)
            calls.append(time.perf_counter() - t)
        res["idle"] = ms_stats(calls[1:])                    # the first call warms up
        res["kept_samples_mean"] = float(chk[:, 7].mean())
        res["rows_with_a_violation"] = int(np.any(chk[:, 10:] >= 0.0, axis=1).sum())
        opt.close()
        for arm in ("none", "updates", "checks"):
            opt = context(prec)
            run(opt, mixed, depth, args.warmup, None, 1.0)
            torch.cuda.synchronize()
            u = None if arm == "none" else Updater(opt, windows, mixed, arm == "checks")
            r = {"converged_traj_per_s": run(opt, mixed, depth, args.batches, u, args.period_ms / 1e3)}
            if arm == "checks":
                r.update(ms_stats(u.call))
            opt.close()
            res[arm] = r
            print(prec, arm, json.dumps(r), file=sys.stderr, flush=True)
        out["precision_%d" % prec] = res
    # kernel times last: a profiler session slows the throughput path's later launches, so no timed arm runs after one
    for prec in precs:
        depth, res = (3 if prec == 64 else 8), out["precision_%d" % prec]
        opt = context(prec)
        last = opt.optimize(mixed)
        tf = mid_t_from(mixed, last[0])
        opt.check_results(mixed, last, t_from=tf)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.idle_reps):
                opt.check_results(mixed, last, t_from=tf)
            torch.cuda.synchronize()
        res["idle"]["kernel_ms"] = kernel_ms_per_call(prof, args.idle_reps)
        run(opt, mixed, depth, args.warmup, None, 1.0)
        u = Updater(opt, windows, mixed, True)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(opt, mixed, depth, args.batches, u, args.period_ms / 1e3)
            torch.cuda.synchronize()
        res["checks"]["kernel_ms_in_flight"] = kernel_ms_per_call(prof, len(u.call))
        opt.close()
        print(prec, json.dumps(res), file=sys.stderr, flush=True)
    out["device_after"] = device()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
