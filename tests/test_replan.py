"""The CPU reference of ualm_submit_replan's build (tests/replan_oracle.cpp): its restated resampler against ualm_resample_path bit for bit,
its polyline against the check's own sample sequence (tests/check_oracle.cpp), and the refusals of the Python wrapper.  Trajectories: a
few problems on the hill stand-in, solved by the oracle."""
import numpy as np
import pytest

import replan_oracle as ro

from harness import bits


def _same_resample(path, rp=ro.DEFAULT_RP):
    from uneven_planner_b200 import problems
    N, M, bnd, T, ixy, iyaw = problems.resample(path, *rp)
    N2, M2, T2, ixy2, iyaw2, sm = ro.resample(path, rp)
    assert (N, M) == (N2, M2)
    assert bits([T]) == bits([T2])
    assert np.array_equal(bits(ixy), bits(ixy2)) and np.array_equal(bits(iyaw), bits(iyaw2))
    assert bits([bnd[12], bnd[15]]).tolist() == bits([sm[0, 2], sm[-1, 2]]).tolist()   # first yaw as given, last one smoothed


@pytest.fixture(scope="module")
def gold_paths(built, golden):
    from uneven_planner_b200 import configs, maps, problems
    g = maps.stand_in_terrain("hill")
    gold = golden("hill", g)
    pb = problems.generate(g, int(gold["B"]), seed=int(gold["seed"]), **configs.gen_kwargs("hill"))
    return [problems.dubins(s, e) for s, e in zip(pb.starts, pb.goals)]


@pytest.mark.parametrize("rp", [ro.DEFAULT_RP, (0.17, 3.0, 0.8, 1.5)])
def test_restated_resampler_is_ualm_resample_path_on_dubins_paths(gold_paths, rp):
    for path in gold_paths:
        _same_resample(path, rp)


def test_restated_resampler_is_ualm_resample_path_with_yaw_wraps(built):
    rng = np.random.default_rng(11)
    wraps = 0
    for _ in range(200):
        n = int(rng.integers(2, 120))
        step = rng.uniform(0.005, 0.2, n)
        head = np.cumsum(rng.normal(0.0, 0.4, n))
        xy = np.cumsum(np.stack([step * np.cos(head), step * np.sin(head)], 1), 0)
        yaw = head + 2 * np.pi * rng.integers(-3, 4, n) + rng.normal(0.0, 0.6, n)     # whole turns and steps past +-pi/2
        path = np.concatenate([xy, yaw[:, None]], 1)
        wraps += int(np.any(np.abs(np.diff(yaw)) >= np.pi / 2))
        _same_resample(path)
    assert wraps > 100


@pytest.fixture(scope="module")
def trajs(built):
    import pyoracle as po
    from uneven_planner_b200 import configs, maps, problems
    g = maps.stand_in_terrain("hill")
    params = configs.params_for("hill")
    pb = problems.generate(g, 6, seed=0, **configs.gen_kwargs("hill"))
    om = po.OracleMap(g)
    out = []
    for i, (r, cxy, cyaw, _) in enumerate(po.solve_batch(po.params_from(params), om, pb, threads=6)):
        N, M = int(pb.N[i]), int(pb.M[i])
        out.append((N, M, cxy, cyaw, r.total_T / N, r.total_T / M, pb.bnd[i]))
    return dict(om=om, params=params, trajs=out)


def test_polyline_times_are_the_check_sequence(trajs):
    from check_oracle import check
    p = trajs["params"]
    for N, M, cxy, cyaw, Tx, Ty, bnd in trajs["trajs"]:
        for dt in (0.01, 0.037):
            _, tr = check(trajs["om"], p.gravity, N, M, cxy, cyaw, Tx, Ty, dt=dt, trace=True)
            seq = tr[:, 0]
            t_k = seq[len(seq) // 3]
            for t_from in (0.0, t_k, 0.5 * Tx, 2.0 * Tx, seq[-1], 0.37 * seq[-1] + 0.0031):
                pts, ts, head = ro.polyline(N, M, cxy, cyaw, Tx, Ty, bnd, t_from, dt)
                assert ts[0] == t_from and ts[-1] == -1.0
                assert np.array_equal(bits(ts[1:-1]), bits(seq[seq > t_from]))
                assert np.array_equal(pts[-1], [bnd[6], bnd[7], bnd[15]])
                assert bits(pts[0]).tolist() == bits(head[[0, 1, 6]]).tolist()
                row = ro.replan(N, M, cxy, cyaw, Tx, Ty, bnd, t_from, dt)
                assert np.array_equal(row[:6], head[:6]) and np.array_equal(row[12:15], head[6:9])
                assert np.array_equal(row[6:12], bnd[6:12]) and np.array_equal(row[15:18], bnd[15:18])
                N2, M2, T2, ixy, iyaw, _ = ro.resample(pts)
                assert (row[19], row[20]) == (N2, M2) and row[18] == T2
                assert np.array_equal(row[21:21 + ixy.size], ixy) and not row[21 + ixy.size:21 + 2 * ro.CAP_XY].any()


def test_rows_over_the_caps_keep_their_counts(trajs):
    N, M, cxy, cyaw, Tx, Ty, bnd = trajs["trajs"][0]
    row = ro.replan(N, M, cxy, cyaw, Tx, Ty, bnd, 0.0, 0.01, (0.01, 2.0, 0.5, 1.2))
    assert row[19] > 64 and row[20] > 128 and not row[21:].any()
    N2, M2, T2, _, _, _ = ro.resample(ro.polyline(N, M, cxy, cyaw, Tx, Ty, bnd, 0.0)[0], (0.01, 2.0, 0.5, 1.2))
    assert (row[19], row[20], row[18]) == (N2, M2, T2)


def test_wrapper_refusals(built):
    from uneven_planner_b200 import _lib, api, problems
    opt = object.__new__(api.BatchALMTrajOpt)          # the checks below come before any call into the library
    pb = problems.ProblemBatch(np.array([3, 4], np.int32), np.array([5, 6], np.int32), np.zeros((2, 18)), np.ones(2), np.zeros(10), np.zeros(9))
    out = ((_lib.Result * 2)(), np.zeros(12 * 7), np.zeros(6 * 11))
    for rows in ([2], [-1], [[0, 1]], [0.5]):
        with pytest.raises(ValueError):
            opt.submit_replan(pb, out, rows, 0.0)
    with pytest.raises(ValueError):
        opt.submit_replan(pb, ((_lib.Result * 3)(), out[1], out[2]), [0], 0.0)


def test_bounded_stream_is_the_unbounded_one_on_ordinary_paths(gold_paths):
    for path in gold_paths:
        a, b = ro.resample(path), ro.resample(path, bounded=True)
        assert a[:3] == b[:3] and np.array_equal(a[3], b[3]) and np.array_equal(a[4], b[4])


@pytest.mark.parametrize("case", ["huge_end_yaw", "far_goal", "huge_goal"])
def test_degenerate_goals_are_cut_short(trajs, case):
    """a goal no caller should send still ends the build promptly: cut short as an over-limit row (N' = M' = 4097), its total_time
    still the polyline's whole length (infinite for coordinates whose squares overflow, which the C call then refuses)"""
    import time
    N, M, cxy, cyaw, Tx, Ty, bnd = trajs["trajs"][0]
    bnd = bnd.copy()
    if case == "huge_end_yaw":
        bnd[15] = 1e300
    elif case == "far_goal":
        bnd[6] = 1e9
    else:
        bnd[6], bnd[7] = 1e300, -1e300
    t = time.perf_counter()
    row = ro.replan(N, M, cxy, cyaw, Tx, Ty, bnd, 0.5 * Tx)
    assert time.perf_counter() - t < 5.0
    assert (row[19], row[20]) == (4097, 4097) and not row[21:].any()
    pts = ro.polyline(N, M, cxy, cyaw, Tx, Ty, bnd, 0.5 * Tx)[0]
    dx, dy = np.diff(pts[:, 0]), np.diff(pts[:, 1])
    with np.errstate(over="ignore"):
        seg = np.sqrt(dx * dx + dy * dy)             # as the stream forms it: the squares overflow for the huge goal
    length = 0.0
    for s in seg:                                    # the stream's sum, in order
        length += s
    assert row[18] == length / 0.5 * 1.2
    assert np.isfinite(row[18]) == (case != "huge_goal")
