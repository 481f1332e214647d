#!/usr/bin/env python
"""map_shift_bench.py -- keeping environment 0's grid around a robot that drives across a larger world, by moving it whole cells
(include/ualm.h, ualm_shift_map with host cells of the strips, ualm_shift_map_from_cloud with a local scan of the strips) against
replacing the whole moved grid (ualm_update_map from host cells, ualm_update_map_from_cloud from the cloud around it), while batches
are in flight.

    python tools/map_shift_bench.py [--batches 12] [--warmup 2] [--period-ms 250] [--precisions 64,32] [--idle-reps 5]

Workload: that of tools/map_window_bench.py (four environments, 1024 problems per batch, pipelined at depth 3 on the parity path and
8 on the throughput path).  Environment 0's 200x200x64 grid (10 m, 0.05 m cells) follows a robot driving at 0.5 m/s along x with a
slow drift in y: every `period-ms` (250 ms, 0.125 m) it moves by 2 or 3 cells in x, alternately, and by 1 cell in y every fourth time.
The world is the analytic surface of tools/map_update_bench.py's clouds extended along the drive (a seeded cloud at that density), and
its host cells are the grid a whole-grid device build of that cloud gives:
  shift_cells:  ualm_shift_map with the strips' cells from the host (copy engines only);
  shift_cloud:  ualm_shift_map_from_cloud with the points of the strips plus 0.5 m (the ellipsoid's reach is 0.32 m);
  update_cells: ualm_update_map of the whole moved grid from the host;
  update_cloud: ualm_update_map_from_cloud of the whole moved grid from the points of the grid plus 0.5 m;
  none:         no updates.
Before the pipelined runs, each arm runs `idle-reps` times with nothing in flight.  Prints one JSON line: per arm the idle call time
and kernel time, and per precision and arm converged traj/s, call time p50 / max (ms), the cell kernel's CUDA-event time p50 (ms) and
the number of updates, with the card's name and power limit read in the same run.
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
from map_window_bench import run, stats  # noqa: E402

MARGIN = 0.5
DRIVE_CELLS = 480             # how far the world reaches past the first grid in x (24 m at 0.05 m): more than any run drives


def world_cloud(seed, x0=-5.5, x1=5.5 + DRIVE_CELLS * 0.05, y0=-5.5, y1=8.0, density=3560.0):
    """tools/map_update_bench.py's surface (400k points over 10.6 m x 10.6 m) over the whole drive, at the same density"""
    rng = np.random.default_rng(seed)
    n = int(density * (x1 - x0) * (y1 - y0))
    xy = np.column_stack([rng.uniform(x0, x1, n), rng.uniform(y0, y1, n)])
    z = 0.4 * np.exp(-((xy[:, 0] - 0.5) ** 2 + (xy[:, 1] + 0.3) ** 2) / 0.8) + 0.15 * np.sin(2.0 * xy[:, 0]) * np.cos(1.5 * xy[:, 1]) + 0.3
    z += rng.normal(0.0, 0.004, n)
    return np.column_stack([xy, z]).astype(np.float32)


def crop(pts, x0, y0, x1, y1):
    return np.ascontiguousarray(pts[(pts[:, 0] >= x0 - MARGIN) & (pts[:, 0] <= x1 + MARGIN) & (pts[:, 1] >= y0 - MARGIN) & (pts[:, 1] <= y1 + MARGIN)])


def step(k):
    """the k-th move of the robot's grid in cells"""
    return (2 if k % 2 == 0 else 3), (1 if k % 4 == 3 else 0)


class Mover:
    """moves environment 0's grid one step per call as `kind` says; grid k's cells are world[ox:ox + 200, oy:oy + 200]"""

    def __init__(self, opt, kind, world, pts, geom0):
        from uneven_planner_b200 import maps
        self.maps = maps
        self.opt, self.kind, self.world, self.pts, self.geom = opt, kind, world, pts, geom0
        self.k, self.ox, self.oy, self.call, self.kernel = 0, 0, 0, [], []

    def __call__(self):
        maps, opt = self.maps, self.opt
        dx, dy = step(self.k)
        g2 = maps.shift_geometry(self.geom, dx, dy)
        ox, oy = self.ox + dx, self.oy + dy
        r = g2.xy_resolution
        if self.kind == "shift_cells":
            arg = [np.ascontiguousarray(self.world[ox + a:ox + a + nx, oy + b:oy + b + ny]) for a, b, nx, ny in maps.shift_boxes(self.geom, dx, dy)]
        elif self.kind == "shift_cloud":
            arg = np.vstack([crop(self.pts, g2.origin[0] + a * r, g2.origin[1] + b * r, g2.origin[0] + (a + nx) * r, g2.origin[1] + (b + ny) * r)
                             for a, b, nx, ny in maps.shift_boxes(self.geom, dx, dy)])
        elif self.kind == "update_cells":
            arg = maps.UnevenMapData(g2, self.world[ox:ox + 200, oy:oy + 200], "moved")
        else:
            arg = crop(self.pts, g2.origin[0], g2.origin[1], g2.max_boundary[0], g2.max_boundary[1])
        ms = None
        t = time.perf_counter()
        if self.kind == "shift_cells":
            opt.shift_environment(dx, dy, arg, env=0)
        elif self.kind == "shift_cloud":
            ms = opt.shift_environment_from_cloud(arg, dx, dy, env=0)[2]
        elif self.kind == "update_cells":
            opt.update_environment(arg, env=0)
        else:
            ms = opt.update_environment_from_cloud(arg, g2, env=0)[1]
        self.call.append(time.perf_counter() - t)
        if ms is not None:
            self.kernel.append(ms)
        self.geom, self.ox, self.oy, self.k = g2, ox, oy, self.k + 1


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
        raise SystemExit("map_shift_bench.py: no CUDA device")
    pts = world_cloud(1)
    # the world's host cells: the whole drive built once on the device (the crop box keeps 20 m about a grid's centre, so in pieces)
    W = _lib.map_geometry().voxel_num[2]
    world = np.zeros((200 + DRIVE_CELLS, 240, W, 4), np.float32)
    o = api.BatchALMTrajOpt()
    for x in range(0, world.shape[0], 200):
        nx = min(200, world.shape[0] - x)
        g = _lib.map_geometry(nx / 20.0, 12.0, 0.05, 0.1)
        assert tuple(g.voxel_num) == (nx, 240, W)
        g.origin[0], g.max_boundary[0] = -5.0 + x * 0.05, -5.0 + (x + nx) * 0.05
        g.origin[1], g.max_boundary[1] = -5.0, 7.0
        world[x:x + nx] = o.build_map(crop(pts, g.origin[0], g.origin[1], g.max_boundary[0], g.max_boundary[1]), g)[0].cells
    o.close()
    ms_, params, pbs, src = [], [], [], {}
    for name in NAMES:
        m = maps.get_terrain(name)
        src[name] = "reference" if m is not None else "stand-in"
        m = m or maps.stand_in_terrain(name)
        ms_.append(m); params.append(configs.params_for(name, overrides=False))
        pbs.append(problems.generate(m, 256, seed=0, **configs.gen_kwargs(name)))
    cat = problems.concat(pbs, range(len(NAMES)))
    mixed = cat.select(np.arange(cat.B).reshape(len(NAMES), -1).T.reshape(-1))     # interleaved
    geom0 = _lib.map_geometry()
    grid0 = maps.UnevenMapData(geom0, world[:200, :200], "world0")

    def context(prec):
        opt = api.BatchALMTrajOpt(precision=prec)
        for e in range(len(NAMES)):
            opt.init(params[e], env=e).set_environment(grid0 if e == 0 else ms_[e], env=e)
        return opt

    kinds = ["shift_cells", "shift_cloud", "update_cells", "update_cloud"]
    out = {"device": device(), "grids": src, "problems_per_batch": int(mixed.B), "batches": args.batches, "period_ms": args.period_ms,
           "world_cloud_points": int(len(pts)), "steps": "2,3 cells in x alternately, 1 in y every 4th", "kinds": kinds}
    idle = {}
    for kind in kinds:
        opt = context(64)
        u = Mover(opt, kind, world, pts, geom0)
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
        for kind in ["none"] + kinds:
            opt = context(prec)
            run(opt, mixed, depth, args.warmup, None, 1.0)
            torch.cuda.synchronize()
            u = None if kind == "none" else Mover(opt, kind, world, pts, geom0)
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
