#!/usr/bin/env python
"""budget_bench.py -- what the cost bounds of include/ualm.h (ualm_set_budget, ualm_wait_batch_for) do on the bench workload
(BASELINE config 2: 1024 problems on the hill terrain, or the labelled synthetic stand-in bench.py uses without it), parity path.

    python tools/budget_bench.py --max-evals 300 --deadline-ms 50 [--steps 8] [--warmup 3] [--depth 3]

Prints one JSON line:
  unbudgeted:  evaluations per problem by ret_code of one unbudgeted batch (what the non-converging problems cost);
  max_evals:   `steps` batches pipelined over `depth` lanes with ualm_set_budget(K): step time, converged traj/s, stopped fraction
               (and the same without a budget, measured in the same run, for comparison);
  deadline:    batches one at a time, ualm_submit_batch then ualm_wait_batch_for(D): wall time of the wait, converged / stopped per batch.
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
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-evals", type=int, default=300, dest="max_evals")
    ap.add_argument("--deadline-ms", type=float, default=50.0, dest="deadline_ms")
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--depth", type=int, default=3)
    args = ap.parse_args()

    import torch
    from uneven_planner_b200 import api, configs, maps, problems
    if not torch.cuda.is_available():
        raise SystemExit("budget_bench.py: no CUDA device")
    m = maps.get_terrain("hill") or maps.synthetic_terrain("bumps", seed=0)
    params = configs.params_for("hill")
    pb = problems.generate(m, 1024, seed=0, **configs.gen_kwargs("hill"))

    def pipelined(max_evals):
        opt = api.BatchALMTrajOpt(precision=64).init(params).set_environment(m).set_budget(max_evals)
        for lane in range(args.depth):
            opt.select_lane(lane); opt.upload(pb)

        def run(nsteps):
            for s in range(nsteps):
                lane = s % args.depth
                opt.select_lane(lane)
                if s >= args.depth:
                    opt.sync()
                opt.solve_resident()
            for lane in range(args.depth):
                opt.select_lane(lane); opt.sync()
        run(args.warmup)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run(args.steps)
        ms = (time.perf_counter() - t0) * 1e3
        opt.select_lane((args.steps - 1) % args.depth)
        res, _, _ = opt.download()
        opt.close()
        rc = np.array([r.ret_code for r in res]); ev = np.array([r.n_evals for r in res])
        conv = int((rc == 0).sum())
        return {"ms_per_step": ms / args.steps, "converged_per_step": conv, "converged_per_s": conv * args.steps / (ms * 1e-3),
                "stopped_fraction": float((rc == 3).mean()), "evals_per_step": int(ev.sum())}, rc, ev

    free, rc0, ev0 = pipelined(0)
    budget, _, _ = pipelined(args.max_evals)
    by_rc = {str(int(c)): {"problems": int((rc0 == c).sum()), "evals": int(ev0[rc0 == c].sum()), "share_of_evals": float(ev0[rc0 == c].sum() / ev0.sum()),
                           "p50": float(np.percentile(ev0[rc0 == c], 50)), "max": int(ev0[rc0 == c].max())} for c in np.unique(rc0)}

    od = api.BatchALMTrajOpt(precision=64).init(params).set_environment(m)
    waits, conv_b, stop_b = [], [], []
    for s in range(args.warmup + args.steps):
        t = od.submit(pb, depth=1)
        t0 = time.perf_counter()
        r, _, _ = od.wait(t, timeout_ms=args.deadline_ms)
        if s >= args.warmup:
            waits.append((time.perf_counter() - t0) * 1e3)
            conv_b.append(sum(1 for q in r if q.ret_code == 0)); stop_b.append(sum(1 for q in r if q.ret_code == 3))
    od.close()

    print(json.dumps({"device": device(), "workload": "1024 problems, %s, hill parameters, parity path" % m.name,
                      "unbudgeted": {"n_evals_by_ret_code": by_rc, **free},
                      "max_evals": {"max_evals": args.max_evals, "batches_in_flight": args.depth, **budget},
                      "deadline": {"deadline_ms": args.deadline_ms, "batches": len(waits), "wait_ms_p50": float(np.percentile(waits, 50)),
                                   "wait_ms_max": float(max(waits)), "converged_per_batch": conv_b, "stopped_per_batch": stop_b}}))


if __name__ == "__main__":
    main()
