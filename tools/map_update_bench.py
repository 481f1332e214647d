#!/usr/bin/env python
"""map_update_bench.py -- replacing one environment's grid while batches are in flight (include/ualm.h, ualm_update_map /
ualm_update_map_from_cloud) against draining the pipeline around ualm_set_map.

    python tools/map_update_bench.py [--batches 12] [--warmup 2] [--period-ms 250] [--precisions 64,32]

Workload: four environments (hill, desert, volcano, forest; run_<terrain>.yaml parameters; the reference's grid where maps_built/ has
it, else the labelled stand-in), one batch of 1024 problems (256 per terrain, interleaved) per submit, pipelined at depth 3 on the
parity path and 8 on the throughput path.  Every `period-ms`, environment 0's grid is replaced:
  grid source "prebuilt": alternately two prebuilt 200x200x64 grids (the hill and mountain stand-ins);
  grid source "cloud":    rebuilt on the device from one of two seeded 400k-point clouds.
Arms:
  inflight: ualm_update_map / ualm_update_map_from_cloud with the batches in flight;
  drain:    wait for every batch in flight, then ualm_set_map (for "cloud": ualm_map_build_device to the host first), then resume;
  none:     no updates.
Prints one JSON line: per precision and arm, converged traj/s, submit-to-delivery p50 / p99 (ms, from ualm_submit_batch to the return
of its ualm_wait_batch), update call time p50 / max (ms) and the number of updates, with the card's name and power limit read in the
same run.
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
NAMES = ["hill", "desert", "volcano", "forest"]


def device():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def cloud(seed, n=400000, half=5.3):
    """a seeded analytic surface with noise (tests/test_gpu_map_update.py)"""
    rng = np.random.default_rng(seed)
    xy = rng.uniform(-half, half, (n, 2))
    z = 0.4 * np.exp(-((xy[:, 0] - 0.5) ** 2 + (xy[:, 1] + 0.3) ** 2) / 0.8) + 0.15 * np.sin(2.0 * xy[:, 0]) * np.cos(1.5 * xy[:, 1]) + 0.3
    z += rng.normal(0.0, 0.004, n)
    return np.column_stack([xy, z]).astype(np.float32)


def run(opt, mixed, depth, batches, arm, source, grids, clouds, period):
    """submit `batches` batches at most `depth` in flight, replacing environment 0's grid every `period` s as `arm` says"""
    from uneven_planner_b200 import _lib
    flight, lat, upd, converged = [], [], [], 0

    def deliver():
        nonlocal converged
        t, ts = flight.pop(0)
        res = opt.wait(t)[0]
        lat.append(time.perf_counter() - ts)
        converged += sum(r.ret_code == 0 for r in res)

    t0 = time.perf_counter()
    due, k = t0 + period, 0
    for _ in range(batches):
        if arm != "none" and time.perf_counter() >= due:
            if arm == "drain":
                while flight:
                    deliver()
            tu = time.perf_counter()
            if source == "prebuilt":
                g = grids[k % 2]
                (opt.update_environment if arm == "inflight" else opt.set_environment)(g, env=0)
            elif arm == "inflight":
                opt.update_environment_from_cloud(clouds[k % 2], _lib.map_geometry(), env=0)
            else:
                m, _ = opt.build_map(clouds[k % 2], _lib.map_geometry())
                opt.set_environment(m, env=0)
            upd.append(time.perf_counter() - tu)
            k += 1
            due += period
        if len(flight) == depth:
            deliver()
        flight.append((opt.submit(mixed, depth=depth), time.perf_counter()))
    while flight:
        deliver()
    wall = time.perf_counter() - t0
    ms = lambda a, q: float(np.percentile(np.array(a) * 1e3, q)) if a else None
    return {"converged_traj_per_s": converged / wall, "wall_s": wall, "delivery_ms_p50": ms(lat, 50), "delivery_ms_p99": ms(lat, 99),
            "updates": len(upd), "update_ms_p50": ms(upd, 50), "update_ms_max": max(upd) * 1e3 if upd else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--period-ms", type=float, default=250.0)
    ap.add_argument("--precisions", default="64,32")
    args = ap.parse_args()

    import torch
    from uneven_planner_b200 import api, configs, maps, problems
    if not torch.cuda.is_available():
        raise SystemExit("map_update_bench.py: no CUDA device")
    ms_, params, pbs, src = [], [], [], {}
    for name in NAMES:
        m = maps.get_terrain(name)
        src[name] = "reference" if m is not None else "stand-in"
        m = m or maps.stand_in_terrain(name)
        ms_.append(m); params.append(configs.params_for(name, overrides=False))
        pbs.append(problems.generate(m, 256, seed=0, **configs.gen_kwargs(name)))
    cat = problems.concat(pbs, range(len(NAMES)))
    mixed = cat.select(np.arange(cat.B).reshape(len(NAMES), -1).T.reshape(-1))     # interleaved
    grids = [maps.stand_in_terrain("hill"), maps.stand_in_terrain("mountain")]
    clouds = [cloud(1), cloud(2)]

    out = {"device": device(), "grids": src, "problems_per_batch": int(mixed.B), "batches": args.batches, "period_ms": args.period_ms}
    for prec in [int(p) for p in args.precisions.split(",")]:
        depth = 3 if prec == 64 else 8
        res = {"depth": depth}
        for arm, source in [("none", None), ("inflight", "prebuilt"), ("drain", "prebuilt"), ("inflight", "cloud"), ("drain", "cloud")]:
            opt = api.BatchALMTrajOpt(precision=prec)
            for e in range(len(NAMES)):
                opt.init(params[e], env=e).set_environment(ms_[e], env=e)
            run(opt, mixed, depth, args.warmup, "none", None, grids, clouds, 1.0)
            torch.cuda.synchronize()
            r = run(opt, mixed, depth, args.batches, arm, source, grids, clouds, args.period_ms / 1e3)
            opt.close()
            res[arm if source is None else "%s_%s" % (arm, source)] = r
            print(prec, arm, source, json.dumps(r), file=sys.stderr, flush=True)
        out["precision_%d" % prec] = res
    out["device_after"] = device()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
