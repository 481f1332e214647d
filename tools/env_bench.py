#!/usr/bin/env python
"""env_bench.py -- batches that mix terrains on one context (include/ualm.h, ualm_select_env) against what a caller without
environments does: rebind one context terrain by terrain.

    python tools/env_bench.py [--steps 4] [--warmup 1] [--precisions 64,32]

Workload per step: 1024 problems, 256 from each of hill, desert, volcano and forest, each with its run_<terrain>.yaml parameter set
(configs.params_for(name, overrides=False)) on the reference's grid where maps_built/ has it, else the labelled stand-in.
  mixed:     four environments, one batch of the 1024 problems per step, `steps` batches pipelined at the default depth (3 on the
             parity path, 8 on the throughput path);
  by_terrain: environment 0 only; per terrain: rebind parameters and grid, pipeline that terrain's `steps` batches of 256, drain.
Prints one JSON line: ms per step, converged traj/s and converged counts per terrain for both arms and precisions, with the card's
name, power limit and L2 size.
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
    out = {"l2_bytes": torch.cuda.get_device_properties(0).L2_cache_size}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        out["name_power_limit"] = q.stdout.strip().splitlines()[0]
    except Exception:
        out["name_power_limit"] = torch.cuda.get_device_name(0)
    return out


def pipeline(opt, batches, depth):
    """submit every batch, at most `depth` in flight; results of each batch in order"""
    out, flight = [], []
    for pb in batches:
        if len(flight) == depth:
            out.append(opt.wait(flight.pop(0)))
        flight.append(opt.submit(pb, depth=depth))
    out += [opt.wait(t) for t in flight]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--precisions", default="64,32")
    args = ap.parse_args()

    import torch
    from uneven_planner_b200 import api, configs, maps, problems
    if not torch.cuda.is_available():
        raise SystemExit("env_bench.py: no CUDA device")
    ms_, params, pbs, grids = [], [], [], {}
    for name in NAMES:
        m = maps.get_terrain(name)
        grids[name] = "reference" if m is not None else "stand-in"
        m = m or maps.stand_in_terrain(name)
        ms_.append(m); params.append(configs.params_for(name, overrides=False))
        pbs.append(problems.generate(m, 256, seed=0, **configs.gen_kwargs(name)))
    cat = problems.concat(pbs, range(len(NAMES)))
    mixed = cat.select(np.arange(cat.B).reshape(len(NAMES), -1).T.reshape(-1))     # interleaved

    def count(res, env):
        rc = np.array([r.ret_code for r in res])
        return {NAMES[e]: int((rc[env == e] == 0).sum()) for e in range(len(NAMES))}

    out = {"device": device(), "grids": grids, "problems_per_step": int(mixed.B), "steps": args.steps}
    for prec in [int(p) for p in args.precisions.split(",")]:
        depth = 3 if prec == 64 else 8
        opt = api.BatchALMTrajOpt(precision=prec)
        for e in range(len(NAMES)):
            opt.init(params[e], env=e).set_environment(ms_[e], env=e)
        pipeline(opt, [mixed] * args.warmup, depth)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = pipeline(opt, [mixed] * args.steps, depth)
        t_mixed = time.perf_counter() - t0
        opt.close()
        c_mixed = count(res[-1][0], mixed.env)

        opt = api.BatchALMTrajOpt(precision=prec)
        opt.init(params[0]).set_environment(ms_[0])
        pipeline(opt, [pbs[0]] * args.warmup, depth)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        c_by = {}
        for e in range(len(NAMES)):
            opt.init(params[e]).set_environment(ms_[e])
            r = pipeline(opt, [pbs[e]] * args.steps, depth)
            c_by[NAMES[e]] = int(sum(q.ret_code == 0 for q in r[-1][0]))
        t_by = time.perf_counter() - t0
        opt.close()
        arm = lambda t, c: {"ms_per_step": t * 1e3 / args.steps, "converged_traj_per_s": sum(c.values()) * args.steps / t, "converged": c}
        out["precision_%d" % prec] = {"depth": depth, "mixed": arm(t_mixed, c_mixed), "by_terrain": arm(t_by, c_by)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
