"""The CPU reference of ualm_check_trajectories (tests/check_oracle.cpp) against the oracle's own post-solve scan (orc_feasibility) and
against its own per-sample trace.  Trajectories: a few problems on the hill stand-in, solved by the oracle."""
import numpy as np
import pytest

from check_oracle import NO_LIMITS, check, limits_of


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
        out.append((N, M, cxy, cyaw, r.total_T / N, r.total_T / M))
    return dict(om=om, params=params, trajs=out)


def _window(tr, t_from, lim):
    """out16 recomputed from a full trace restricted to t >= t_from, in sample order"""
    o = [0.0, 0.0, 0.0, 0.0, -1.0, 0.0, 0.0, 0.0]
    first = [-1.0] * 6
    for t, vx, ax, ay, cur, att, sig, term, _ in tr:
        if not t >= t_from:
            continue
        for q, v in enumerate((vx, ax, ay, cur)):
            if abs(o[q]) < abs(v):
                o[q] = v
        o[4] = att if o[4] < att else o[4]
        o[5] = sig if o[5] < sig else o[5]
        o[6] += term
        o[7] += 1
        viol = (abs(vx) > lim[0], abs(ax) > lim[1], abs(ay) > lim[2], abs(cur) > lim[3], att > -lim[4], sig > lim[5])
        for q in range(6):
            if viol[q] and first[q] < 0.0:
                first[q] = t
    return o, first


def _times(tr):
    return [0.0, tr[len(tr) // 2, 0], 0.37 * tr[-1, 0] + 0.0031, tr[-1, 0], tr[-1, 0] + 0.01, 1e9]


def test_full_scan_is_orc_feasibility(trajs):
    import pyoracle as po
    p = trajs["params"]
    for N, M, cxy, cyaw, Tx, Ty in trajs["trajs"]:
        ref = po.feasibility(trajs["om"], p.gravity, N, M, cxy, cyaw, Tx, Ty, 0.01)
        out = check(trajs["om"], p.gravity, N, M, cxy, cyaw, Tx, Ty, 0.01, 0.0, NO_LIMITS)
        assert np.array_equal(out[:8], ref), (out, ref)
        assert out[8] == Tx and out[9] == Ty and np.all(out[10:] == -1.0)


@pytest.mark.parametrize("which", ["none", "env", "tight"])
def test_window_and_first_violations_follow_the_trace(trajs, which):
    p = trajs["params"]
    fired = np.zeros(6, bool)
    for N, M, cxy, cyaw, Tx, Ty in trajs["trajs"]:
        full, tr = check(trajs["om"], p.gravity, N, M, cxy, cyaw, Tx, Ty, trace=True)
        assert len(tr) == int(full[7]) and tr[0, 0] == 0.0
        lim = {"none": NO_LIMITS, "env": limits_of(p),
               "tight": (0.5 * abs(full[0]), 0.5 * abs(full[1]), 0.5 * abs(full[2]), 0.5 * abs(full[3]), -full[4] + 1e-3, 0.5 * full[5])}[which]
        for t_from in _times(tr):
            out, tr2 = check(trajs["om"], p.gravity, N, M, cxy, cyaw, Tx, Ty, 0.01, t_from, lim, trace=True)
            assert np.array_equal(tr2[:, :8], tr[:, :8])                     # the same samples, bit for bit, whatever t_from
            assert np.array_equal(tr2[:, 8], (tr[:, 0] >= t_from).astype(float))
            o, first = _window(tr, t_from, lim)
            assert np.array_equal(out[:8], np.array(o)), (t_from, out[:8], o)
            assert np.array_equal(out[10:], np.array(first)), (t_from, out[10:], first)
            assert out[8] == Tx and out[9] == Ty
            # a first violation exactly when the window's maximum breaks the limit (an empty window keeps the initial maxima, no sample)
            breaks = [out[7] > 0 and b for b in (abs(out[0]) > lim[0], abs(out[1]) > lim[1], abs(out[2]) > lim[2], abs(out[3]) > lim[3],
                                                 out[4] > -lim[4], out[5] > lim[5])]
            assert [t >= 0.0 for t in out[10:]] == breaks, (t_from, out, lim)
            fired |= np.array(breaks)
            if t_from >= tr[-1, 0] + 0.01:
                assert out[7] == 0 and np.array_equal(out[:7], [0, 0, 0, 0, -1, 0, 0])
    if which == "tight":
        assert fired.all()
    if which == "none":
        assert not fired.any()


def test_not_scanned(trajs):
    p = trajs["params"]
    N, M, cxy, cyaw, _, _ = trajs["trajs"][0]
    out = check(trajs["om"], p.gravity, N, M, cxy, cyaw, 1e6, 1e6, 0.01)
    assert out[7] == -1.0 and np.all(out[:7] == 0.0) and np.all(out[10:] == -1.0) and out[8] == 1e6
