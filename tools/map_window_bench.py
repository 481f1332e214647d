#!/usr/bin/env python
"""map_window_bench.py -- rebuilding one 2 m x 2 m window of an environment's grid from a local scan (include/ualm.h,
ualm_update_map_window_from_cloud), or writing it from host cells (ualm_update_map_window), against rebuilding the whole grid from the
whole cloud (ualm_update_map_from_cloud), while batches are in flight.

    python tools/map_window_bench.py [--batches 12] [--warmup 2] [--period-ms 250] [--precisions 64,32] [--idle-reps 5]

Workload: that of tools/map_update_bench.py (four environments, 1024 problems per batch, pipelined at depth 3 on the parity path and
8 on the throughput path).  Every `period-ms`, environment 0's grid (200x200x64, 10 m) is updated:
  whole_cloud:  ualm_update_map_from_cloud with one of two seeded 400k-point clouds;
  window_cloud: ualm_update_map_window_from_cloud of a 40x40-column box (2 m x 2 m, at one of four places) from the points of one of
                those clouds within the box plus 0.5 m (the ellipsoid's reach is 0.32 m);
  window_cells: ualm_update_map_window with that box's cells from the host (copy engines only);
  none:         no updates.
Before the pipelined runs, each update kind runs `idle-reps` times with nothing in flight.  Prints one JSON line: local cloud size,
idle update call time and kernel time, and per precision and arm converged traj/s, update call time p50 / max (ms), the cell kernel's
CUDA-event time p50 (ms) and the number of updates, with the card's name and power limit read in the same run.
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
from map_update_bench import NAMES, cloud, device  # noqa: E402

BOXES = [(80, 80), (90, 80), (90, 90), (80, 90)]      # (ix0, iy0) of the 40 x 40 window, a robot's moving scan
NX = NY = 40
MARGIN = 0.5


def local(pts, geom, ix0, iy0):
    """the points of `pts` within the window plus MARGIN"""
    r = geom.xy_resolution
    x0, y0 = geom.origin[0] + ix0 * r - MARGIN, geom.origin[1] + iy0 * r - MARGIN
    x1, y1 = x0 + NX * r + 2 * MARGIN, y0 + NY * r + 2 * MARGIN
    return np.ascontiguousarray(pts[(pts[:, 0] >= x0) & (pts[:, 0] <= x1) & (pts[:, 1] >= y0) & (pts[:, 1] <= y1)])


class Updater:
    def __init__(self, opt, kind, clouds, windows, geom):
        self.opt, self.kind, self.clouds, self.windows, self.geom = opt, kind, clouds, windows, geom
        self.k, self.call, self.kernel = 0, [], []

    def __call__(self):
        k, opt = self.k, self.opt
        ix0, iy0 = BOXES[k % len(BOXES)]
        t = time.perf_counter()
        if self.kind == "whole_cloud":
            ms = opt.update_environment_from_cloud(self.clouds[k % 2], self.geom, env=0)[1]
        elif self.kind == "window_cloud":
            ms = opt.update_environment_window_from_cloud(self.windows[k % 2][k % len(BOXES)], ix0, iy0, NX, NY, env=0)[1]
        else:
            opt.update_environment_window(ix0, iy0, self.windows[2 + k % 2][k % len(BOXES)], env=0)
            ms = None
        self.call.append(time.perf_counter() - t)
        if ms is not None:
            self.kernel.append(ms)
        self.k += 1


def run(opt, mixed, depth, batches, update, period):
    """submit `batches` batches at most `depth` in flight, calling update() every `period` s"""
    flight, converged = [], 0
    t0 = time.perf_counter()
    due = t0 + period
    for _ in range(batches):
        if update is not None and time.perf_counter() >= due:
            update()
            due += period
        if len(flight) == depth:
            converged += sum(r.ret_code == 0 for r in opt.wait(flight.pop(0))[0])
        flight.append(opt.submit(mixed, depth=depth))
    while flight:
        converged += sum(r.ret_code == 0 for r in opt.wait(flight.pop(0))[0])
    return converged / (time.perf_counter() - t0)


def stats(u):
    ms = lambda a, q: float(np.percentile(np.asarray(a), q)) if len(a) else None
    return {"updates": len(u.call), "update_ms_p50": ms(np.array(u.call) * 1e3, 50), "update_ms_max": max(u.call) * 1e3 if u.call else None,
            "kernel_ms_p50": ms(u.kernel, 50)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--period-ms", type=float, default=250.0)
    ap.add_argument("--precisions", default="64,32")
    ap.add_argument("--idle-reps", type=int, default=5)
    args = ap.parse_args()

    import torch
    from uneven_planner_b200 import _lib, api, configs, maps, problems
    if not torch.cuda.is_available():
        raise SystemExit("map_window_bench.py: no CUDA device")
    ms_, params, pbs, src = [], [], [], {}
    for name in NAMES:
        m = maps.get_terrain(name)
        src[name] = "reference" if m is not None else "stand-in"
        m = m or maps.stand_in_terrain(name)
        ms_.append(m); params.append(configs.params_for(name, overrides=False))
        pbs.append(problems.generate(m, 256, seed=0, **configs.gen_kwargs(name)))
    cat = problems.concat(pbs, range(len(NAMES)))
    mixed = cat.select(np.arange(cat.B).reshape(len(NAMES), -1).T.reshape(-1))     # interleaved
    geom = _lib.map_geometry()
    clouds = [cloud(1), cloud(2)]
    # window sources per update parity: local clouds (0, 1), and host cells of the grids those clouds build (2, 3)
    o = api.BatchALMTrajOpt()
    built = [o.build_map(c, geom)[0] for c in clouds]
    o.close()
    windows = [[local(c, geom, *b) for b in BOXES] for c in clouds] + \
              [[np.ascontiguousarray(g.cells[b[0]:b[0] + NX, b[1]:b[1] + NY]) for b in BOXES] for g in built]

    def context(prec):
        opt = api.BatchALMTrajOpt(precision=prec)
        for e in range(len(NAMES)):
            opt.init(params[e], env=e).set_environment(ms_[e], env=e)
        return opt

    out = {"device": device(), "grids": src, "problems_per_batch": int(mixed.B), "batches": args.batches, "period_ms": args.period_ms,
           "cloud_points": int(len(clouds[0])), "local_cloud_points": int(np.mean([len(w) for w in windows[0]])),
           "window": [NX, NY], "kinds": ["whole_cloud", "window_cloud", "window_cells"]}
    opt = context(64)
    idle = {}
    for kind in out["kinds"]:
        u = Updater(opt, kind, clouds, windows, geom)
        for _ in range(args.idle_reps + 1):
            u()
        u.call, u.kernel = u.call[1:], u.kernel[1:]        # the first call of a kind warms up
        idle[kind] = stats(u)
        print("idle", kind, json.dumps(idle[kind]), file=sys.stderr, flush=True)
    opt.close()
    out["idle"] = idle
    for prec in [int(p) for p in args.precisions.split(",")]:
        depth = 3 if prec == 64 else 8
        res = {"depth": depth}
        for kind in ["none"] + out["kinds"]:
            opt = context(prec)
            run(opt, mixed, depth, args.warmup, None, 1.0)
            torch.cuda.synchronize()
            u = None if kind == "none" else Updater(opt, kind, clouds, windows, geom)
            r = {"converged_traj_per_s": run(opt, mixed, depth, args.batches, u, args.period_ms / 1e3)}
            if u is not None:
                r.update(stats(u))
            opt.close()
            res[kind] = r
            print(prec, kind, json.dumps(r), file=sys.stderr, flush=True)
        out["precision_%d" % prec] = res
    out["device_after"] = device()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
