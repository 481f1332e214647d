#!/usr/bin/env python
"""mpc_handover_bench.py -- the hand-over to the MPC (include/ualm.h: ualm_mpc_export_trajectories, ualm_mpc_export_batch).

    python tools/mpc_handover_bench.py [--reps 5] [--calls 10] [--precisions 64,32]

Workload: the bench's 1024 problems on the hill terrain with its parameters (the reference grid when present, else its stand-in).
  (a) time to hand-over of a lone batch on the parity path: from submit until each problem's hand-over arrays are on the host, for
      poll + held export of each poll's new rows against wait + lane export; p50 / p90 / max over the problems, the median of `reps`
      runs, the two arms alternated;
  (b) one held export of all 1024 rows: idle; in flight on the parity path at depth 3 without and with ualm_set_urgent; in flight on
      the throughput path at depth 8; and the mpc_export_kernel time of an idle call from torch.profiler (a run of its own, last).
Prints one JSON line with the card's name and power limit read in the same run.
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
from map_update_bench import device  # noqa: E402


def pct(a):
    a = np.asarray(a) * 1e3
    return {"p50": float(np.percentile(a, 50)), "p90": float(np.percentile(a, 90)), "max": float(a.max())}


def handover_poll(opt, pb):
    """seconds from submit until each problem's held export is on the host"""
    t0 = time.perf_counter()
    t = opt.submit(pb, depth=2)
    out = opt.outputs(pb)
    when, pending = np.zeros(pb.B), pb.B
    while pending:
        new, pending = opt.poll(t, out, wait_ms=1.0)
        if new.size:
            opt.mpc_export_results(pb, out, rows=new)
            when[new] = time.perf_counter() - t0
    opt.wait(t)
    return when


def handover_wait(opt, pb):
    t0 = time.perf_counter()
    t = opt.submit(pb, depth=2)
    opt.wait(t)
    opt.select_lane(t)
    opt.mpc_export(pb.N, pb.M)
    return np.full(pb.B, time.perf_counter() - t0)


def in_flight_calls(opt, pb, out, depth, calls, urgent):
    """held exports of `out`, one after each submit while `depth` batches are in flight: seconds per call"""
    flight, took = [], []
    for _ in range(depth):
        flight.append(opt.submit(pb, depth=depth))
    for _ in range(calls):
        opt.wait(flight.pop(0))
        flight.append(opt.submit(pb, depth=depth))
        t = time.perf_counter()
        opt.mpc_export_results(pb, out, urgent=urgent)
        took.append(time.perf_counter() - t)
    while flight:
        opt.wait(flight.pop(0))
    return took


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--precisions", default="64,32")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from uneven_planner_b200 import api, configs, maps, problems
    if not torch.cuda.is_available():
        raise SystemExit("mpc_handover_bench.py: no CUDA device")
    m = maps.get_terrain("hill")
    src = "reference" if m is not None else "stand-in"
    m = m or maps.stand_in_terrain("hill")
    params = configs.params_for("hill")
    pb = problems.generate(m, 1024, seed=0, **configs.gen_kwargs("hill"))

    def context(prec):
        return api.BatchALMTrajOpt(precision=prec).init(params).set_environment(m)

    res = {"device": device(), "grid": src, "problems": int(pb.B)}
    # (a)
    opt = context(64)
    handover_poll(opt, pb); handover_wait(opt, pb)          # warm-up
    arms = {"poll_held": [], "wait_lane": []}
    for _ in range(args.reps):
        arms["poll_held"].append(pct(handover_poll(opt, pb)))
        arms["wait_lane"].append(pct(handover_wait(opt, pb)))
    opt.close()
    res["a_time_to_handover_ms"] = {k: {q: float(np.median([r[q] for r in v])) for q in ("p50", "p90", "max")} for k, v in arms.items()}
    print(json.dumps(res["a_time_to_handover_ms"]), file=sys.stderr, flush=True)
    # (b)
    b = {}
    for prec in [int(p) for p in args.precisions.split(",")]:
        opt = context(prec)
        out = opt.optimize(pb)
        idle = []
        for _ in range(args.calls + 1):
            t = time.perf_counter()
            opt.mpc_export_results(pb, out)
            idle.append(time.perf_counter() - t)
        r = {"idle_ms": pct(idle[1:])}
        if prec == 64:
            r["in_flight_depth3_ms"] = pct(in_flight_calls(opt, pb, out, 3, args.calls, False))
            r["in_flight_depth3_urgent_ms"] = pct(in_flight_calls(opt, pb, out, 3, args.calls, True))
        else:
            r["in_flight_depth8_ms"] = pct(in_flight_calls(opt, pb, out, 8, args.calls, False))
        opt.close()
        b["precision_%d" % prec] = r
        print(prec, json.dumps(r), file=sys.stderr, flush=True)
    # kernel time last: a profiler session slows later launches
    opt = context(64)
    out = opt.optimize(pb)
    opt.mpc_export_results(pb, out)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.calls):
            opt.mpc_export_results(pb, out)
        torch.cuda.synchronize()
    tot = sum((getattr(e, "device_time_total", None) or e.cuda_time_total) for e in prof.key_averages() if "mpc_export_kernel" in e.key)
    b["mpc_export_kernel_ms"] = tot / 1e3 / args.calls
    opt.close()
    res["b_one_call_1024_rows"] = b
    res["device_after"] = device()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
