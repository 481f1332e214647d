#!/usr/bin/env python
"""replan_bench.py -- replanning the trajectories a server handed out, after each window update, from where each robot is to its goal
(include/ualm.h, ualm_submit_replan), idle and while batches are in flight.

    python tools/replan_bench.py [--batches 12] [--warmup 2] [--period-ms 250] [--precisions 64,32] [--idle-reps 10] [--margin 0.8]
                                 [--horizon 1.0] [--max-rows 32]

Workload: that of tools/check_bench.py (four environments, 1024 problems per batch, pipelined at depth 3 on the parity path and 8 on the
throughput path, environment 0's 2 m x 2 m window written every `period-ms`).  After each update the last delivered batch is checked from
half of each trajectory's duration with every limit scaled by `margin` (ualm_check_trajectories), and the rows whose first violation
falls within `horizon` s of that time are flagged.  Of those, the `max-rows` with the earliest first violation are replanned from there
(ualm_submit_replan on the same lane ring), as a server that triages its fleet would; 0 replans every flagged row.  Arms per precision: none (no
update), replans.  Reported: rows replanned per update; the replan call's time, idle (the same 256 rows `idle-reps` times) and in flight;
replan_kernel's time from torch.profiler runs made after every timed arm; the host time to build the same problems as a caller would
without the call (the oracle's evaluation of the trajectory + ualm_resample_path, per row); for the replanned tickets, submit-to-delivery
(polled every 2 ms), converged fraction and mean evaluations; converged traj/s of the main stream.  Prints one JSON line with the card's
name and power limit read in the same run.
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
from check_bench import BOXES, NX, NY, mid_t_from  # noqa: E402
from map_update_bench import NAMES, device  # noqa: E402


def margin_limits(p, margin):
    """the environment's six limits tightened by `margin` (min_cxi, a lower bound on cos xi, raised toward 1)"""
    return (margin * p.max_vel, margin * p.max_acc_lon, margin * p.max_acc_lat, margin * p.max_kap, 1.0 - margin * (1.0 - p.min_cxi), margin * p.max_sig)


def flagged(chk, tf, horizon):
    """rows with a first violation within `horizon` s of t_from, earliest violation first"""
    first = np.where(chk[:, 10:] >= 0.0, chk[:, 10:], np.inf).min(axis=1) - tf
    rows = np.nonzero(np.isfinite(first) & (first <= horizon))[0]
    return rows[np.argsort(first[rows], kind="stable")]


class Server:
    """the main stream of batches at `depth`, with replans on the same lane ring after each window update"""

    def __init__(self, opt, mixed, depth, windows, limits, horizon, replan, max_rows=0):
        self.opt, self.mixed, self.depth, self.windows, self.limits, self.horizon, self.replan = opt, mixed, depth, windows, limits, horizon, replan
        self.max_rows, self.flagged = max_rows, []
        self.flight = []            # (ticket, pb, replan submit time or None)
        self.k, self.last = 0, None
        self.converged = 0
        self.rows, self.call, self.deliver, self.rconv, self.revals = [], [], [], [], []

    def _settle_replans(self):
        """poll the replan tickets in flight until they are complete; their delivery times"""
        for i, (t, pb, t0) in enumerate(self.flight):
            if t0 is None or t0 < 0:
                continue
            buf = self.opt.outputs(pb)
            while self.opt.poll(t, buf, 2.0)[1] > 0:
                pass
            self.deliver.append(time.perf_counter() - t0)
            self.flight[i] = (t, pb, -1.0)

    def _wait_oldest(self):
        self._settle_replans()
        t, pb, t0 = self.flight.pop(0)
        out = self.opt.wait(t)
        if t0 is None:
            self.converged += sum(r.ret_code == 0 for r in out[0])
            self.last = out
        else:
            self.rconv.extend(r.ret_code == 0 for r in out[0])
            self.revals.extend(r.n_evals for r in out[0])

    def update(self):
        ix0, iy0 = BOXES[self.k % len(BOXES)]
        self.opt.update_environment_window(ix0, iy0, self.windows[self.k % 2][self.k % len(BOXES)], env=0)
        self.k += 1
        if not self.replan or self.last is None:
            return
        last = self.last            # waiting for a lane below may deliver a newer batch
        tf = mid_t_from(self.mixed, last[0])
        chk = self.opt.check_results(self.mixed, last, t_from=tf, limits=self.limits)
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
        ticket, new = self.opt.submit_replan(self.mixed, last, rows, tf[rows], depth=self.depth)
        self.call.append(time.perf_counter() - t)
        self.flight.append((ticket, new, t))

    def run(self, batches, period):
        t0 = time.perf_counter()
        due = t0 + period
        for _ in range(batches):
            if period and time.perf_counter() >= due:
                self.update()
                due += period
            if len(self.flight) == self.depth:
                self._wait_oldest()
            self.flight.append((self.opt.submit(self.mixed, depth=self.depth), self.mixed, None))
        while self.flight:
            self._wait_oldest()
        return self.converged / (time.perf_counter() - t0)


def ms_stats(a, pct=(50,)):
    a = np.asarray(a) * 1e3
    out = {"calls": int(a.size)}
    for q in pct:
        out["ms_p%d" % q] = float(np.percentile(a, q)) if a.size else None
    out["ms_max"] = float(a.max()) if a.size else None
    return out


def kernel_ms_per_call(prof, calls):
    tot = 0.0
    for e in prof.key_averages():
        if "replan_kernel" in e.key:
            tot += getattr(e, "device_time_total", None) or e.cuda_time_total
    return tot / 1e3 / max(calls, 1)


def host_build_ms(pb, out, rows, tf, dt=0.01):
    """the caller's own build without the call, per row: the oracle's evaluation of the polyline (tests/replan_oracle.cpp) and
    ualm_resample_path on it (ms per row)"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import replan_oracle as ro
    from uneven_planner_b200 import problems
    res, cxy, cyaw = out
    _, _, ocx, ocy = pb.offsets()
    ro.lib()
    t = time.perf_counter()
    for k, i in enumerate(rows):
        pts, _, _ = ro.polyline(pb.N[i], pb.M[i], cxy[ocx[i]:ocx[i + 1]], cyaw[ocy[i]:ocy[i + 1]], res[i].piece_T_xy, res[i].piece_T_yaw, pb.bnd[i], tf[k], dt)
        try:
            problems.resample(pts)
        except RuntimeError:
            pass
    return (time.perf_counter() - t) * 1e3 / max(len(rows), 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--period-ms", type=float, default=250.0)
    ap.add_argument("--precisions", default="64,32")
    ap.add_argument("--idle-reps", type=int, default=10)
    ap.add_argument("--margin", type=float, default=0.8)
    ap.add_argument("--horizon", type=float, default=1.0)
    ap.add_argument("--max-rows", type=int, default=32, dest="max_rows")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from uneven_planner_b200 import api, configs, maps, problems
    if not torch.cuda.is_available():
        raise SystemExit("replan_bench.py: no CUDA device")
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

    out = {"device": device(), "grids": src, "problems_per_batch": int(mixed.B), "batches": args.batches, "period_ms": args.period_ms,
           "window": [NX, NY], "margin": args.margin, "horizon_s": args.horizon,
           "max_rows": args.max_rows}
    precs = [int(p) for p in args.precisions.split(",")]
    idle_rows = np.arange(0, mixed.B, 4)         # 256 rows
    for prec in precs:
        depth = 3 if prec == 64 else 8
        res = {"depth": depth}
        opt = context(prec)
        last = opt.optimize(mixed)
        ok = np.array([r.piece_T_xy > 0.0 and r.piece_T_yaw > 0.0 for r in last[0]])
        rows = idle_rows[ok[idle_rows]]
        tf = mid_t_from(mixed, last[0])[rows]
        calls = []
        for k in range(args.idle_reps + 1):
            t = time.perf_counter()
            ticket, new = opt.submit_replan(mixed, last, rows, tf, depth=depth)
            calls.append(time.perf_counter() - t)
            r = opt.wait(ticket)
        res["idle"] = dict(ms_stats(calls[1:]), rows=int(rows.size))
        res["idle"]["host_build_ms_per_row"] = host_build_ms(mixed, last, rows, tf)
        res["idle"]["replanned_converged_fraction"] = float(np.mean([x.ret_code == 0 for x in r[0]]))
        opt.close()
        for arm in ("none", "replans"):
            opt = context(prec)
            Server(opt, mixed, depth, windows, limits, args.horizon, False).run(args.warmup, 0.0)
            torch.cuda.synchronize()
            s = Server(opt, mixed, depth, windows, limits, args.horizon, arm == "replans", args.max_rows)
            r = {"converged_traj_per_s": s.run(args.batches, args.period_ms / 1e3)}
            if arm == "replans":
                r["flagged_per_update"] = s.flagged
                r["rows_per_update"] = s.rows
                r["call"] = ms_stats(s.call)
                r["submit_to_delivery"] = ms_stats(s.deliver, (50, 99))
                r["replanned_converged_fraction"] = float(np.mean(s.rconv)) if s.rconv else None
                r["replanned_mean_evals"] = float(np.mean(s.revals)) if s.revals else None
            opt.close()
            res[arm] = r
            print(prec, arm, json.dumps(r), file=sys.stderr, flush=True)
        out["precision_%d" % prec] = res
    # kernel times last: a profiler session slows the throughput path's later launches, so no timed arm runs after one
    for prec in precs:
        depth, res = (3 if prec == 64 else 8), out["precision_%d" % prec]
        opt = context(prec)
        last = opt.optimize(mixed)
        ok = np.array([r.piece_T_xy > 0.0 and r.piece_T_yaw > 0.0 for r in last[0]])
        rows = idle_rows[ok[idle_rows]]
        tf = mid_t_from(mixed, last[0])[rows]
        opt.wait(opt.submit_replan(mixed, last, rows, tf, depth=depth)[0])
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.idle_reps):
                opt.wait(opt.submit_replan(mixed, last, rows, tf, depth=depth)[0])
            torch.cuda.synchronize()
        res["idle"]["kernel_ms"] = kernel_ms_per_call(prof, args.idle_reps)
        Server(opt, mixed, depth, windows, limits, args.horizon, False).run(args.warmup, 0.0)
        s = Server(opt, mixed, depth, windows, limits, args.horizon, True, args.max_rows)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            s.run(args.batches, args.period_ms / 1e3)
            torch.cuda.synchronize()
        res["replans"]["kernel_ms_in_flight"] = kernel_ms_per_call(prof, len(s.call))
        opt.close()
        print(prec, json.dumps(res), file=sys.stderr, flush=True)
    out["device_after"] = device()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
