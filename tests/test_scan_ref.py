"""The CPU references of the post-solve scan, the check and the replan build held to the float64 restatement of tests/scan_ref.py, which
shares no code with oracle/oracle.cpp: orc_feasibility (pyoracle.feasibility), tests/check_oracle.cpp with t_from and its per-sample
trace, tests/replan_oracle.cpp's rows and resampler, and ualm_resample_path on Dubins and front-end polylines.  Trajectories: oracle
solves on the hill stand-in, and the hand-built trajectories of scan_ref.SCAN_CASES on the hill stand-in, `wide` centred at
(31.4, -17.25) and `fine_yaw`.  test_case_table_reaches_the_edges fails if the table stops reaching any edge it is there for.

Worst errors measured (relative to each quantity's scale; x86-64, g++ -O3): the maxima 8e-13 (cur), the non-holonomic sum 2e-14 of
the summed speeds, the per-sample values 1.3e-12 (ax and ay on the 4 ms pieces of short_pieces, whose coefficients are large), the
replan head 1e-13, total_time 1.3e-12, the waypoints 3e-14 of the polyline's extent; the constraint columns 4e-13.  The bounds sit
about 10x above those."""
import functools

import numpy as np
import pytest

import alm_ref as ar
import check_oracle as co
import replan_oracle as ro
import scan_ref as sr
from scan_ref import SCAN_CASES, scan_case, scan_limits, scan_t_froms
from workloads import scan_times, summed

TOL = 1e-11              # maxima, sums, first-violation bands and per-sample values, relative to each quantity's scale
TOL_REPLAN = 1e-11       # the replan head, total_time and waypoints
GRIDS = ("hill", "wide_off", "fine_yaw")
LIMIT_KINDS = ("none", "median", "first", "last")


@functools.lru_cache(maxsize=None)
def _grid(name):
    from uneven_planner_b200 import _lib, configs, maps
    from workloads import GRIDS as G, grid
    if name == "hill":
        m = maps.stand_in_terrain("hill")
    elif name == "wide_off":
        m = maps.UnevenMapData(_lib.map_geometry_at(*G["wide"][:4], 31.4, -17.25), grid("wide").cells, "wide@31.4,-17.25")
    else:
        m = grid(name)
    import pyoracle as po
    return m, po.OracleMap(m), ar.Grid(m), configs.params_for("hill")


@pytest.fixture(scope="module")
def solved(built):
    """six oracle solves on the hill stand-in: (N, M, c_xy, c_yaw, T_xy, T_yaw, bnd)"""
    import pyoracle as po
    from uneven_planner_b200 import configs, problems
    m, om, _, params = _grid("hill")
    pb = problems.generate(m, 6, seed=0, **configs.gen_kwargs("hill"))
    return [(int(pb.N[i]), int(pb.M[i]), cxy, cyaw, r.total_T / int(pb.N[i]), r.total_T / int(pb.M[i]), pb.bnd[i])
            for i, (r, cxy, cyaw, _) in enumerate(po.solve_batch(po.params_from(params), om, pb, threads=6))]


def _trajs(solved):
    """(grid name, N, M, c_xy, c_yaw, T_xy, T_yaw, bnd, dts) of every solved and hand-built trajectory"""
    out = [("hill", N, M, cxy, cyaw, Tx, Ty, bnd, [0.01]) for N, M, cxy, cyaw, Tx, Ty, bnd in solved]
    for g in GRIDS:
        for name in SCAN_CASES:
            c = scan_case(name, _grid(g)[0])
            out.append((g, c["N"], c["M"], c["c_xy"], c["c_yaw"], c["Tx"], c["Ty"], c["bnd"], c["dts"]))
    return out


def _report(what, worst):
    print("%s worst: %s" % (what, ", ".join("%s %.1e" % kv for kv in sorted(worst.items()))))


# ---- the link to the cost -----------------------------------------------------------------------

def test_scanned_quantities_are_the_cost_constraints(built):
    """at the cost's own sample times, the squares minus the squared limits are alm_ref's constraint columns: the scan reports what
    the solve constrains"""
    import torch
    from uneven_planner_b200 import configs, problems
    m, _, grid, params = _grid("hill")
    pb = problems.generate(m, 4, seed=3, **configs.gen_kwargs("hill"))
    worst = 0.0
    for i in range(pb.B):
        prob = ar.Problem(pb, i)
        st = ar._Setup(prob, params, grid, prob.x0)
        with torch.no_grad():
            _, _, c_xy, c_yaw, _, con = st.samples(torch.as_tensor(prob.x0))
        s = sr.samples(grid, params.gravity, prob.N, prob.M, c_xy.numpy().T.ravel(), c_yaw.numpy().ravel(), st.Tx, st.Ty, st.tm["now"])
        con = con.numpy()
        mine = np.stack([s["term"], s["vx2"] - params.max_vel ** 2, s["ax"] ** 2 - params.max_acc_lon ** 2, s["ay"] ** 2 - params.max_acc_lat ** 2,
                         s["curv"] - params.max_kap ** 2, s["att"] + params.min_cxi, s["sig"] - params.max_sig], 1)
        con[:, 0] = np.abs(con[:, 0])
        assert np.allclose(s["vx"] ** 2, s["vx2"], rtol=1e-14, atol=0) and np.allclose(s["cur"] ** 2, s["curv"], rtol=1e-13, atol=1e-300)
        err = np.abs(mine - con).max()
        worst = max(worst, err)
        assert err <= 1e-12, (i, err)
    print("constraint columns worst: %.1e" % worst)


# ---- the scan and the check ---------------------------------------------------------------------

def test_orc_feasibility_matches_the_restatement(solved):
    import pyoracle as po
    worst = {}
    for g, N, M, cxy, cyaw, Tx, Ty, _, dts in _trajs(solved):
        _, om, grid, params = _grid(g)
        for dt in dts:
            ref = sr.scan(grid, params.gravity, N, M, cxy, cyaw, Tx, Ty, dt)
            assert not ref["ambiguous"]
            w, bad = sr.compare(po.feasibility(om, params.gravity, N, M, cxy, cyaw, Tx, Ty, dt), ref, tol=TOL)
            assert not bad, (g, N, M, dt, bad)
            sr.worst_of(worst, w)
    _report("orc_feasibility", worst)


def test_check_oracle_matches_the_restatement(solved):
    """every trajectory at every window start of scan_t_froms and four kinds of limits; the per-sample trace sample by sample"""
    worst, fired = {}, {k: np.zeros(6, bool) for k in ("start", "middle", "last")}
    for g, N, M, cxy, cyaw, Tx, Ty, _, dts in _trajs(solved):
        _, om, grid, params = _grid(g)
        for dt in dts:
            total = sr.duration(N, M, Tx, Ty)
            full = sr.scan(grid, params.gravity, N, M, cxy, cyaw, Tx, Ty, dt)
            _, tr = co.check(om, params.gravity, N, M, cxy, cyaw, Tx, Ty, dt, 0.0, trace=True)
            assert np.array_equal(tr[:, 0], full["t"])                                   # the same sequence, bit for bit
            s = full["s"]
            for j, k in enumerate(sr.QUANTITIES + ("term",)):
                scale = max(float(np.abs(s[k]).max()), 1e-3) if k != "term" else max(float(np.abs(s["vx"]).max()), 1e-3)
                e = float(np.abs(tr[:, 1 + j] - s[k]).max()) / scale
                worst["sample_" + k] = max(worst.get("sample_" + k, 0.0), e)
                assert e <= TOL, (g, N, M, dt, k, e)
            for t_from in scan_t_froms(total, dt):
                for kind in LIMIT_KINDS:
                    lim = scan_limits(sr.window(full, t_from), kind)
                    ref = sr.window(full, t_from, lim)
                    got = co.check(om, params.gravity, N, M, cxy, cyaw, Tx, Ty, dt, t_from, lim)
                    w, bad = sr.compare(got, ref, lim, tol=TOL)
                    assert not bad, (g, N, M, dt, t_from, kind, bad)
                    sr.worst_of(worst, w)
                    tk = ref["t"][ref["kept"]]
                    if tk.size > 2:
                        for j in range(6):
                            t = got[10 + j]
                            fired["start"][j] |= t == tk[0]
                            fired["last"][j] |= t == tk[-1]
                            fired["middle"][j] |= tk[0] < t < tk[-1]
    _report("check_oracle", worst)
    for k, f in fired.items():
        assert f.all(), (k, f)


@pytest.mark.parametrize("side", ["below", "above"])
def test_check_oracle_at_the_sample_guard(built, side):
    """total / dt one sample below the 4e6 guard (scanned: 4e6 samples, restated in chunks) and one above (not scanned)"""
    _, om, grid, params = _grid("hill")
    c = scan_case("spin", _grid("hill")[0])
    total = sr.duration(c["N"], c["M"], c["Tx"], c["Ty"])
    dt = total / (sr.GUARD - 0.5) if side == "below" else total / (sr.GUARD + 0.5)
    assert (total / dt < sr.GUARD) == (side == "below")
    t_from = 0.5 * total
    ref = sr.scan(grid, params.gravity, c["N"], c["M"], c["c_xy"], c["c_yaw"], c["Tx"], c["Ty"], dt, t_from, (1.0, 5.0, 10.0, 20.0, 0.8, 0.05))
    got = co.check(om, params.gravity, c["N"], c["M"], c["c_xy"], c["c_yaw"], c["Tx"], c["Ty"], dt, t_from, (1.0, 5.0, 10.0, 20.0, 0.8, 0.05))
    w, bad = sr.compare(got, ref, (1.0, 5.0, 10.0, 20.0, 0.8, 0.05), tol=TOL)
    assert not bad, bad
    assert (got[7] > 1.9e6) if side == "below" else (got[7] == -1.0 and got[8] == c["Tx"])
    _report("guard " + side, w)


# ---- the replan build and the resampler ---------------------------------------------------------

def test_replan_oracle_matches_the_restatement(solved):
    """replan rows from window starts before the end, the strict t > t_from boundary included (an exact sample time, one ulp below)"""
    worst = {}
    for g, N, M, cxy, cyaw, Tx, Ty, bnd, dts in _trajs(solved):
        for dt in dts[:1]:
            total = sr.duration(N, M, Tx, Ty)
            for t_from in [t for t in scan_t_froms(total, dt) if t < total]:
                row = ro.replan(N, M, cxy, cyaw, Tx, Ty, bnd, t_from, dt)
                ref = sr.replan(N, M, cxy, cyaw, Tx, Ty, bnd, t_from, dt)
                pts, ts, _ = ro.polyline(N, M, cxy, cyaw, Tx, Ty, bnd, t_from, dt)
                assert np.array_equal(ts[1:-1], ref["times"]), (g, N, M, t_from)          # S4: exactly the samples t_from < t
                Nn, Mn = int(row[19]), int(row[20])
                nx, ny = (Nn - 1, Mn - 1) if Nn <= 64 and Mn <= 128 else (0, 0)
                w, bad = sr.compare_replan(Nn, Mn, row[:18], row[18], row[21:21 + 2 * nx], row[21 + ro.CAP_XY * 2:21 + ro.CAP_XY * 2 + ny], ref,
                                           tol=TOL_REPLAN)
                assert not bad, (g, N, M, t_from, bad)
                sr.worst_of(worst, w)
    _report("replan_oracle", worst)


def _front_end_paths():
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "kino_astar_golden.npz"))
    ends = np.cumsum(g["lens"])
    return [g["paths"][e - n:e] for n, e in zip(g["lens"], ends)]


def _edge_paths():
    """yaw jumps just under / over pi/2 and 3 pi/2 and whole turns, a path that doubles back, and straight paths whose waypoint counts
    sit at the 64 / 128 limits, past them, at the 4095 cut (yaw waypoints) and past it"""
    out = {}
    h = 1e-6
    for name, jump in (("under_half", 0.5 * np.pi - h), ("over_half", 0.5 * np.pi + h), ("under_3half", 1.5 * np.pi - h),
                       ("over_3half", 1.5 * np.pi + h), ("turns", 6.0 * np.pi + 0.3)):
        n = 40
        x = 0.05 * np.arange(n)
        yaw = np.cumsum(np.where(np.arange(n) % 3 == 1, jump, -0.2 * jump))
        out[name] = np.stack([x, 0.01 * x, yaw], 1)
    x = np.concatenate([0.07 * np.arange(30), 0.07 * np.arange(30)[::-1]])
    out["doubles_back"] = np.stack([x, 0.02 * np.arange(60), 0.1 * np.arange(60)], 1)
    for name, L in (("at_64", 0.3 * 63 + 0.1), ("past_64", 0.3 * 64 + 0.1), ("at_128_yaw", 0.15 * 127 + 0.05), ("past_128_yaw", 0.15 * 128 + 0.05),
                    ("at_4095", 0.15 * 4095 + 0.05), ("past_4095", 0.15 * 4096 + 0.05)):
        n = int(L / 0.37) + 2
        x = np.linspace(0.0, L, n)
        out[name] = np.stack([x, np.zeros(n), 0.001 * x], 1)
    return out


def _check_resample(path, rp, got, ref, what):
    N, M, T, ixy, iyaw = got
    w, bad = sr.compare_replan(N, M, np.zeros(18), T, ixy, iyaw, dict(ref, bnd=np.zeros(18), polyline=ref["smoothed"]), tol=TOL_REPLAN, caps=None)
    assert not bad, (what, bad)
    return w


@pytest.mark.parametrize("source", ["dubins", "front_end", "wraps", "edges"])
def test_resamplers_match_the_restatement(built, golden, source):
    """ualm_resample_path (with its boundary states) and replan_oracle's resampler, unbounded and with the replan build's bound"""
    from uneven_planner_b200 import configs, maps, problems
    if source == "dubins":
        m = maps.stand_in_terrain("hill")
        gold = golden("hill", m)
        pb = problems.generate(m, int(gold["B"]), seed=int(gold["seed"]), **configs.gen_kwargs("hill"))
        paths = {i: problems.dubins(s, e) for i, (s, e) in enumerate(zip(pb.starts, pb.goals))}
    elif source == "front_end":
        paths = {k: p for k, p in enumerate(_front_end_paths()) if len(p) >= 2}
    elif source == "wraps":
        rng = np.random.default_rng(11)
        paths = {}
        for k in range(100):
            n = int(rng.integers(2, 120))
            step = rng.uniform(0.005, 0.2, n)
            head = np.cumsum(rng.normal(0.0, 0.4, n))
            xy = np.cumsum(np.stack([step * np.cos(head), step * np.sin(head)], 1), 0)
            paths[k] = np.concatenate([xy, (head + 2 * np.pi * rng.integers(-3, 4, n) + rng.normal(0.0, 0.6, n))[:, None]], 1)
    else:
        paths = _edge_paths()
    worst = {}
    for rp in (ro.DEFAULT_RP, (0.17, 3.0, 0.8, 1.5)):
        for what, path in paths.items():
            for bounded in (False, True):
                ref = sr.resample(path, rp, bounded=bounded)
                N, M, T, ixy, iyaw, sm = ro.resample(path, rp, bounded=bounded)
                sr.worst_of(worst, _check_resample(path, rp, (N, M, T, ixy, iyaw), ref, (what, rp, bounded)))
                if ref["tie_smooth"] is None:
                    assert np.max(np.abs(sm[:, 2] - ref["smoothed"][:, 2])) <= TOL_REPLAN * max(1.0, np.abs(sm[:, 2]).max()), what
                if bounded or N > 513 or M > 1025:
                    continue
                Nh, Mh, bnd, Th, ixy_h, iyaw_h = problems.resample(path, *rp)
                sr.worst_of(worst, _check_resample(path, rp, (Nh, Mh, Th, ixy_h, iyaw_h), ref, (what, rp, "ualm_resample_path")))
                p0, p1 = path[0], ref["smoothed"][-1]
                assert np.array_equal(bnd[[0, 1, 12, 6, 7]], [p0[0], p0[1], p0[2], p1[0], p1[1]]), what
                assert abs(bnd[15] - p1[2]) <= TOL_REPLAN * max(1.0, abs(p1[2])), what
                assert np.allclose(bnd[[2, 3, 8, 9]], 0.05 * np.array([np.cos(p0[2]), np.sin(p0[2]), np.cos(p1[2]), np.sin(p1[2])]), rtol=0,
                                   atol=0.05 * TOL_REPLAN * max(1.0, abs(p1[2]))), \
                    (what, bnd[[2, 3, 8, 9]] - 0.05 * np.array([np.cos(p0[2]), np.sin(p0[2]), np.cos(p1[2]), np.sin(p1[2])]))
    if source == "edges":
        cut = sr.resample(paths["past_4095"], ro.DEFAULT_RP, bounded=True)
        assert cut["cut"] and cut["N"] == 4097 and not sr.resample(paths["at_4095"], ro.DEFAULT_RP, bounded=True)["cut"]
        assert sr.resample(paths["at_64"], ro.DEFAULT_RP)["N"] == 64 and sr.resample(paths["past_64"], ro.DEFAULT_RP)["N"] == 65
        assert sr.resample(paths["at_128_yaw"], ro.DEFAULT_RP)["M"] == 128 and sr.resample(paths["past_128_yaw"], ro.DEFAULT_RP)["M"] == 129
    _report("resample " + source, worst)


# ---- the table ----------------------------------------------------------------------------------

def test_case_table_reaches_the_edges(built):
    """the hand-built table reaches: N = 1 and 64, M = 1 and 128, N != M with the smaller duration on either side one ulp apart and
    far apart,
    pieces shorter than dt, samples exactly on piece boundaries, dt 0.01 / 0.0137 / longer than the trajectory (one sample), samples off
    the map, in the clamped border cells and across the yaw seam, raw yaws beyond +-3 pi, a steep cell (cos xi < 0.9), a standstill,
    a reversal and yaw rates above 5 rad/s, on a square, an off-centre non-square and a fine-yaw grid"""
    got = set()
    for g in GRIDS:
        m, _, grid, params = _grid(g)
        for name in SCAN_CASES:
            c = scan_case(name, m)
            N, M, Tx, Ty = c["N"], c["M"], c["Tx"], c["Ty"]
            got |= {k for k, v in (("N1", N == 1), ("N64", N == 64), ("M1", M == 1), ("M128", M == 128)) if v}
            a, b = summed(Tx, N), summed(Ty, M)
            if a != b and abs(a - b) == np.spacing(min(a, b)):
                got.add("ulp_xy_min" if a < b else "ulp_yaw_min")
            if abs(a - b) > 0.1 * min(a, b):
                got.add("xy_ends_first" if a < b else "yaw_ends_first")
            for dt in c["dts"]:
                total = min(a, b)
                t = scan_times(total, dt)
                got |= {k for k, v in (("dt_0.01", dt == 0.01), ("dt_0.0137", dt == 0.0137), ("one_sample", len(t) == 1),
                                       ("short_pieces", Tx < dt)) if v}
                bounds = [summed(Tx, i) for i in range(1, N)]
                if np.isin(t, bounds).any():
                    got.add("on_boundary")
                s = sr.samples(grid, params.gravity, N, M, c["c_xy"], c["c_yaw"], Tx, Ty, t)
                yaw = sr.state(N, M, c["c_xy"], c["c_yaw"], Tx, Ty, t)[6]
                dyaw = sr.state(N, M, c["c_xy"], c["c_yaw"], Tx, Ty, t)[7]
                vx = sr.state(N, M, c["c_xy"], c["c_yaw"], Tx, Ty, t)[2]
                got |= {k for k, v in (("off_map", s["off_map"].any()), ("border", s["border"].any()), ("seam", s["seam"].any()),
                                       ("yaw_beyond_3pi", (np.abs(yaw) > 3 * np.pi).any()), ("steep", (-s["att"] < 0.9).any()),
                                       ("standstill", (np.abs(s["vx"]) < 1e-12).all() and (np.abs(dyaw) > 0.1).any()),
                                       ("reversal", (vx > 0.05).any() and (vx < -0.05).any()), ("yaw_rate", (np.abs(dyaw) > 5.0).any()))
                        if v}
                assert not s["margin"].any(), (g, name, dt)
        got.add("grid_" + g)
    want = {"N1", "N64", "M1", "M128", "ulp_xy_min", "ulp_yaw_min", "xy_ends_first", "yaw_ends_first", "dt_0.01", "dt_0.0137", "one_sample", "short_pieces", "on_boundary",
            "off_map", "border", "seam", "yaw_beyond_3pi", "steep", "standstill", "reversal", "yaw_rate"} | {"grid_" + g for g in GRIDS}
    assert want <= got, sorted(want - got)
