"""Both paths' post-solve scan (ualm_feasibility_batch), check (ualm_check_trajectories, _pp) and replan build (ualm_submit_replan)
held to the float64 restatement of tests/scan_ref.py, which shares no code with the kernels or their oracles, on each path's own
solved trajectories and on the hand-built trajectories of scan_ref.SCAN_CASES.  The check takes caller trajectories, so the hand-built
coefficients reach what no solve produces: one piece, the compiled limits, sums one ulp apart, pieces shorter than dt, samples on piece
boundaries, a standstill, reversing, high yaw rates, raw yaws beyond +-3 pi, samples off the map, in the clamped border cells, across
the yaw seam and on a steep cell, on the hill stand-in, `wide` centred at (31.4, -17.25), `fine_yaw` and the double grid.

Worst errors measured on an H100, relative to each quantity's scale: the lane scan 2.4e-14; the check of the paths' solves 3.4e-12
(cur; ax, ay 7.6e-13), of the table 7.5e-13 (cur); the non-holonomic sum 1e-14 of the summed speeds."""
import numpy as np
import pytest

import scan_ref as sr
from harness import ctx, gpu, split  # noqa: F401
from scan_ref import SCAN_CASES, scan_case, scan_limits, scan_t_froms
from workloads import hill_desert_world

pytestmark = pytest.mark.gpu
PRECISIONS = [64, 65, 32]
DT = 0.01
TOL = 3e-11              # the check of the paths' solves measured 3.4e-12 on cur
TOL_REPLAN = 1e-11


@pytest.fixture(scope="module")
def world(gpu, golden):
    return hill_desert_world(golden)


def _grids(precision):
    """name -> UnevenMapData of the four environments the hand-built table runs on; the fourth is the double grid of ualm_set_map_f64
    on the parity path"""
    from uneven_planner_b200 import _lib, maps
    from workloads import GRIDS, grid
    h = maps.stand_in_terrain("hill")
    out = {"hill": h, "wide_off": maps.UnevenMapData(_lib.map_geometry_at(*GRIDS["wide"][:4], 31.4, -17.25), grid("wide").cells, "wide_off"),
           "fine_yaw": grid("fine_yaw")}
    if precision != 64:
        out["hill_2"] = h                    # four environments on every path
    else:
        rng = np.random.default_rng(4)
        c64 = h.cells.astype(np.float64) * (1.0 + 1e-9 * rng.standard_normal(h.cells.shape))
        out["hill_f64"] = maps.UnevenMapData(h.geom, c64.astype(np.float32), "hill_f64", cells64=c64)
    return out


def _pp(params, lims):
    """a parameter row [rho_T, rho_ter, six limits]"""
    return [params.rho_T, params.rho_ter] + [float(v) for v in lims]


_GRID, _CASE, _FULL = {}, {}, {}       # restated once for the module: alm_ref grids, hand-built cases, restated scans


def _grid(m):
    if m.name not in _GRID:
        import alm_ref as ar
        _GRID[m.name] = ar.Grid(m)
    return _GRID[m.name]


def _case(name, m):
    if (name, m.name) not in _CASE:
        _CASE[(name, m.name)] = scan_case(name, m)
    return _CASE[(name, m.name)]


def _check_all(opt, trajs, full, dt, worst, fired, tag):
    """trajs: [(env, N, M, c_xy, c_yaw, Tx, Ty)], full: their restated scans; every window start of scan_t_froms, with the
    environment's limits, per-row limits (the _pp rows) and call-wide limits that override them"""
    B = len(trajs)
    N = np.array([t[1] for t in trajs], np.int32)
    M = np.array([t[2] for t in trajs], np.int32)
    pt = np.array([(t[5], t[6]) for t in trajs])
    cxy, cyaw = np.concatenate([t[3] for t in trajs]), np.concatenate([t[4] for t in trajs])
    env = np.array([t[0] for t in trajs], np.int32)
    totals = [sr.duration(t[1], t[2], t[5], t[6]) for t in trajs]
    params = opt.env_params
    for k in range(7):
        tf = np.array([scan_t_froms(T, dt)[k] if f["t"] is not None else 0.0 for T, f in zip(totals, full)])
        refs = [sr.window(f, t) for f, t in zip(full, tf)]
        for mode in ("env", "rows", "call"):
            kinds = [("median", "first", "last", "none")[(b + k) % 4] for b in range(B)]
            row_lims = [scan_limits(r, kd) if r["t"] is not None else (1.0,) * 6 for r, kd in zip(refs, kinds)]
            if mode == "env":
                lims = [tuple(getattr(params[e], n) for n in ("max_vel", "max_acc_lon", "max_acc_lat", "max_kap", "min_cxi", "max_sig")) for e in env]
                got = opt.check_trajectories(N, M, pt, cxy, cyaw, env=env, t_from=tf, dt=dt)
            elif mode == "rows":
                lims = row_lims
                pp = np.array([_pp(params[e], l) for e, l in zip(env, lims)])
                got = opt.check_trajectories(N, M, pt, cxy, cyaw, env=env, t_from=tf, dt=dt, params=pp)
            else:
                call = row_lims[0]
                lims = [call] * B
                pp = np.array([_pp(params[e], l) for e, l in zip(env, row_lims[::-1])])
                got = opt.check_trajectories(N, M, pt, cxy, cyaw, env=env, t_from=tf, dt=dt, limits=call, params=pp)
            for b in range(B):
                ref = sr.window(full[b], tf[b], lims[b])
                assert not ref["ambiguous"], (tag, b)
                w, bad = sr.compare(got[b], ref, lims[b], tol=TOL)
                assert not bad, (tag, dt, k, mode, b, trajs[b][1:3], bad)
                sr.worst_of(worst, w)
                if mode == "rows" and ref["t"] is not None:
                    fired |= got[b, 10:] >= 0.0


@pytest.mark.parametrize("precision", PRECISIONS)
def test_lane_scan_and_check_of_solves_match_the_restatement(gpu, world, precision):
    """the golden problems and 64 of the bench's solved on the path: ualm_feasibility_batch of the lane, then the check of the same
    trajectories at every window start and kind of limits"""
    from uneven_planner_b200 import problems
    pb = problems.concat([world["gold_pb"], world["bench"].select(np.arange(64))], [0, 0])
    p, g0 = world["params"], world["g0"]
    opt = ctx(gpu, precision, p, g0)
    out = opt.optimize(pb)
    feas = opt.feasibility(DT)
    grid, worst, fired = _grid(g0), {}, np.zeros(6, bool)
    trajs = []
    for i, (r, cx, cy) in enumerate(split(pb, out)):
        N, M = int(pb.N[i]), int(pb.M[i])
        ref = sr.scan(grid, p.gravity, N, M, cx, cy, r.piece_T_xy, r.piece_T_yaw, DT, device=True)
        w, bad = sr.compare(feas[i], ref, tol=TOL)
        assert not bad, (i, bad)
        sr.worst_of(worst, w)
        trajs.append((0, N, M, cx.copy(), cy.copy(), r.piece_T_xy, r.piece_T_yaw))
    print("feasibility %d worst: %s" % (precision, worst))
    worst = {}
    full = [sr.scan(grid, p.gravity, N, M, cx, cy, Tx, Ty, DT, device=True) for _, N, M, cx, cy, Tx, Ty in trajs]
    _check_all(opt, trajs, full, DT, worst, fired, "solves")
    opt.close()
    print("check of solves %d worst: %s" % (precision, worst))
    assert fired.all(), fired


@pytest.mark.parametrize("precision", PRECISIONS)
def test_check_of_hand_built_trajectories_matches_the_restatement(gpu, world, precision):
    """the whole table on every grid, four environments whose gravities differ, with a row over the compiled limits and a row past
    the sample guard in each call"""
    from uneven_planner_b200 import configs
    grids = _grids(precision)
    names = list(grids)
    gravs = [9.81, 3.71, 1.62, 24.79][:len(names)]
    prm = []
    for g in gravs:
        q = configs.params_for("hill")
        q.gravity = g
        prm.append(q)
    opt = ctx(gpu, precision, prm, [grids[n] for n in names])
    worst, fired = {}, np.zeros(6, bool)
    by_dt = {}
    for e, n in enumerate(names):
        for name in SCAN_CASES:
            c = _case(name, grids[n])
            for dt in c["dts"]:
                by_dt.setdefault(dt, []).append((e, c["N"], c["M"], c["c_xy"], c["c_yaw"], c["Tx"], c["Ty"], (n, gravs[e], name, dt)))
    for dt, rows in by_dt.items():
        for e, N, M, cx, cy, Tx, Ty, key in rows:
            if key not in _FULL:
                _FULL[key] = sr.scan(_grid(grids[key[0]]), key[1], N, M, cx, cy, Tx, Ty, dt, device=True)
        trajs = [r[:7] for r in rows]
        full = [_FULL[r[7]] for r in rows]
        extra = [(1, 65, 10, np.zeros(12 * 65), np.zeros(60), 0.1, 0.1),                       # over the compiled limits: not scanned
                 (2, 3, 5, np.linspace(-1.0, 1.0, 36), np.zeros(30), 2e6 * dt, 2e6 * dt)]     # past the guard
        full += [sr.scan(None, gravs[t[0]], *t[1:], dt, device=True) for t in extra]
        _check_all(opt, trajs + extra, full, dt, worst, fired, "table")
    opt.close()
    print("check of the table %d worst: %s" % (precision, worst))
    assert fired.all(), fired


def test_check_at_the_sample_guard(gpu, world):
    """total / dt one sample below the 4e6 guard (4e6 samples, restated once in chunks) and one above, on every path"""
    g0, p = world["g0"], world["params"]
    c = _case("spin", g0)
    total = sr.duration(c["N"], c["M"], c["Tx"], c["Ty"])
    lims = (1.0, 5.0, 10.0, 20.0, 0.8, 0.05)
    for side, dt in (("below", total / (sr.GUARD - 0.5)), ("above", total / (sr.GUARD + 0.5))):
        ref = sr.scan(_grid(g0), p.gravity, c["N"], c["M"], c["c_xy"], c["c_yaw"], c["Tx"], c["Ty"], dt, 0.5 * total, lims, device=True)
        for precision in PRECISIONS:
            opt = ctx(gpu, precision, p, g0)
            got = opt.check_trajectories([c["N"]], [c["M"]], [[c["Tx"], c["Ty"]]], c["c_xy"], c["c_yaw"], t_from=0.5 * total, dt=dt, limits=lims)
            opt.close()
            w, bad = sr.compare(got[0], ref, lims, tol=TOL)
            assert not bad, (side, precision, bad)
            assert (got[0, 7] > 1.9e6) if side == "below" else got[0, 7] == -1.0
        del ref


def _replan_against(opt, pb, out, rows, tf, worst):
    ticket, new = opt.submit_replan(pb, out, rows, tf, dt=DT)
    opt.wait(ticket)
    oxy, oyaw, _, _ = new.offsets()
    res, cxy, cyaw = out
    _, _, ocx, ocy = pb.offsets()
    for k, i in enumerate(rows):
        ref = sr.replan(int(pb.N[i]), int(pb.M[i]), cxy[ocx[i]:ocx[i + 1]], cyaw[ocy[i]:ocy[i + 1]], res[i].piece_T_xy, res[i].piece_T_yaw,
                        pb.bnd[i], tf[k], DT)
        w, bad = sr.compare_replan(int(new.N[k]), int(new.M[k]), new.bnd[k], new.total_time[k], new.inner_xy[oxy[k]:oxy[k + 1]],
                                   new.inner_yaw[oyaw[k]:oyaw[k + 1]], ref, tol=TOL_REPLAN)
        assert not bad, (k, i, tf[k], bad)
        sr.worst_of(worst, w)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_replan_build_matches_the_restatement(gpu, world, precision):
    """ualm_submit_replan's built problems (api.submit_replan's `new`) of the path's own solves and of the hand-built table (as records
    carrying their piece durations) from window starts before the end: 0, an exact sample time (the strict t > t_from boundary), one ulp
    below it, mid-piece, a few samples before the end"""
    from uneven_planner_b200 import _lib, problems
    pb = problems.concat([world["gold_pb"], world["bench"].select(np.arange(32))], [0, 0])
    p, g0 = world["params"], world["g0"]
    opt = ctx(gpu, precision, p, g0)
    out = opt.optimize(pb)
    opt.set_budget(1)                # only the build is compared: the replanned problems' solves stop at once
    worst = {}
    totals = [sr.duration(int(pb.N[i]), int(pb.M[i]), out[0][i].piece_T_xy, out[0][i].piece_T_yaw) for i in range(pb.B)]
    for k in range(5):
        tf = np.array([scan_t_froms(T, DT)[k] for T in totals])
        _replan_against(opt, pb, out, np.arange(pb.B), tf, worst)
    cases = [_case(n, g0) for n in SCAN_CASES if n != "standstill"]      # a robot at its goal has no polyline to resample
    hb = problems.ProblemBatch(np.array([c["N"] for c in cases], np.int32), np.array([c["M"] for c in cases], np.int32),
                               np.array([c["bnd"] for c in cases]), np.ones(len(cases)), np.zeros(sum(2 * (c["N"] - 1) for c in cases)),
                               np.zeros(sum(c["M"] - 1 for c in cases)))
    res = (_lib.Result * len(cases))()
    for i, c in enumerate(cases):
        res[i].piece_T_xy, res[i].piece_T_yaw = c["Tx"], c["Ty"]
    hout = (res, np.concatenate([c["c_xy"] for c in cases]), np.concatenate([c["c_yaw"] for c in cases]))
    htot = [sr.duration(c["N"], c["M"], c["Tx"], c["Ty"]) for c in cases]
    for k in range(5):
        tf = np.array([scan_t_froms(T, DT)[k] for T in htot])
        ok = np.nonzero(tf < np.array(htot))[0]
        _replan_against(opt, hb, hout, ok, tf[ok], worst)
    opt.close()
    print("replan %d worst: %s" % (precision, worst))
