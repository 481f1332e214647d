#!/usr/bin/env python
"""problem_params_bench.py -- per-problem vehicle limits and cost weights (include/ualm.h, ualm_problem_params_t and the *_pp entry
points): what the rows cost, and a mixed fleet as rows against what a caller without them does.

    python tools/problem_params_bench.py [--steps 4] [--warmup 1] [--rounds 2] [--precisions 64,32]

Workload per step: bench.py's 1024 problems (hill, seed 0, run_hill.yaml parameters) on the reference's hill grid where maps_built/
has it, else the labelled stand-in.  Every arm pipelines its batches at the default depth (3 on the parity path, 8 on the throughput
path) and is timed from its first submit to its last wait.
  (a) cost of the rows:  `steps` batches with rows equal to the environment's values against the same batches without rows,
                         alternated `rounds` times in one context;
  (b) a fleet mix:       eight vehicle classes (seeded rows: rho_T in {1e3, 1e4, 1e5, 3e5}, rho_ter in [1, 20], max_vel in [0.3, 1.2],
                         max_acc_lon in [2, 8], max_acc_lat in [4, 12], max_kap in [1, 3], min_cxi in [0.7, 0.9], max_sig in
                         [0.03, 0.1]), problem b in class b mod 8.
      rows:              one ticket stream, every step one batch of the 1024 problems, each with its class's row;
      rebind:            environment 0 only; per class: rebind its parameters (ualm_set_params, which needs the lanes drained),
                         pipeline that class's `steps` batches of 128, drain.
Prints one JSON line: ms per step, converged traj/s and converged counts (per class for (b), of the last batch of each class) for
every arm and precision, with the card's name and power limit.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NCLASS = 8


def device():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def pipeline(opt, batches, depth):
    """submit every batch, at most `depth` in flight; results of each batch in order"""
    out, flight = [], []
    for pb in batches:
        if len(flight) == depth:
            out.append(opt.wait(flight.pop(0)))
        flight.append(opt.submit(pb, depth=depth))
    out += [opt.wait(t) for t in flight]
    return out


def timed(opt, batches, depth):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = pipeline(opt, batches, depth)
    return time.perf_counter() - t0, res


def class_rows(seed=0):
    r = np.random.default_rng(seed)
    return np.column_stack([r.choice([1e3, 1e4, 1e5, 3e5], NCLASS), r.uniform(1, 20, NCLASS), r.uniform(0.3, 1.2, NCLASS), r.uniform(2, 8, NCLASS),
                            r.uniform(4, 12, NCLASS), r.uniform(1, 3, NCLASS), r.uniform(0.7, 0.9, NCLASS), r.uniform(0.03, 0.1, NCLASS)])


def with_row(params, row):
    from uneven_planner_b200 import _lib
    p = _lib.Params()
    C.memmove(C.byref(p), C.byref(params), C.sizeof(p))
    for (f, _), v in zip(_lib.ProblemParams._fields_, row):
        setattr(p, f, float(v))
    return p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--precisions", default="64,32")
    args = ap.parse_args()

    import torch
    from uneven_planner_b200 import _lib, api, configs, maps, problems
    if not torch.cuda.is_available():
        raise SystemExit("problem_params_bench.py: no CUDA device")
    m = maps.get_terrain("hill")
    grid = "reference" if m is not None else "stand-in"
    m = m or maps.stand_in_terrain("hill")
    params = configs.params_for("hill")
    pb = problems.generate(m, 1024, seed=0, **configs.gen_kwargs("hill"))
    same = problems.concat([pb], [0])
    same.env, same.params = None, np.tile(_lib.problem_params(params), (pb.B, 1))
    rows = class_rows()
    cls = np.arange(pb.B) % NCLASS
    fleet = problems.concat([pb], [0])
    fleet.env, fleet.params = None, rows[cls]
    per_class = [pb.select(np.flatnonzero(cls == c)) for c in range(NCLASS)]

    def arm(t, conv, steps):
        n = sum(conv.values()) if isinstance(conv, dict) else conv
        return {"ms_per_step": t * 1e3 / steps, "converged_traj_per_s": n * steps / t, "converged": conv}

    def converged(res, idx=None):
        rc = np.array([r.ret_code for r in res])
        return int((rc == 0).sum()) if idx is None else {str(c): int((rc[idx == c] == 0).sum()) for c in range(NCLASS)}

    out = {"device": device(), "grid": grid, "problems_per_step": int(pb.B), "steps": args.steps, "classes": rows.tolist()}
    for prec in [int(p) for p in args.precisions.split(",")]:
        depth = 3 if prec == 64 else 8
        res_p = {}
        opt = api.BatchALMTrajOpt(precision=prec).init(params).set_environment(m)
        pipeline(opt, [pb, same] * args.warmup, depth)
        a = {"no_rows": [], "rows_equal": []}
        for _ in range(args.rounds):
            for name, b in (("no_rows", pb), ("rows_equal", same)):
                t, r = timed(opt, [b] * args.steps, depth)
                a[name].append(arm(t, converged(r[-1][0]), args.steps))
        res_p["a_cost_of_rows"] = a
        pipeline(opt, [fleet] * args.warmup, depth)
        t, r = timed(opt, [fleet] * args.steps, depth)
        res_p["b_rows"] = arm(t, converged(r[-1][0], cls), args.steps)
        opt.close()

        opt = api.BatchALMTrajOpt(precision=prec).init(with_row(params, rows[0])).set_environment(m)
        pipeline(opt, per_class[:1] * args.warmup, depth)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        conv = {}
        for c in range(NCLASS):
            opt.init(with_row(params, rows[c]))
            r = pipeline(opt, [per_class[c]] * args.steps, depth)
            conv[str(c)] = converged(r[-1][0])
        res_p["b_rebind"] = arm(time.perf_counter() - t0, conv, args.steps)
        opt.close()
        res_p["depth"] = depth
        out["precision_%d" % prec] = res_p
    print(json.dumps(out))


if __name__ == "__main__":
    main()
