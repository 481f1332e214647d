"""One evaluation of the parity path against the CPU oracle, bit for bit, at the MINCO system sizes where the forward sweep
L y = b, which runs inside the banded LU (lu_dual), is most likely to go wrong: the smallest systems (only the last-six pivot
types), the compiled limits, an xy system longer than the yaw system and the reverse, and right-hand sides with exact-zero
boundary rows."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu(built):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from uneven_planner_b200 import api
    return api


def _arc_problem(N, M, zero_ends=False, radius=2.5, arc=1.5 * np.pi, speed=0.5, centre=(0.0, 0.0), start=0.0):
    """One problem whose waypoints lie on a circular arc around `centre` (the map centre by default), from polar angle `start`
    counter-clockwise over `arc`: N xy pieces, M yaw pieces.  zero_ends: zero boundary velocity and acceleration, so that those
    right-hand-side rows are exact zeros."""
    from uneven_planner_b200 import problems
    length = radius * arc
    T = 1.2 * length / speed
    a = start + arc * np.linspace(0.0, 1.0, N + 1)
    rel = radius * np.stack([np.cos(a), np.sin(a)], axis=1)
    pts = rel + np.asarray(centre, np.float64)
    yaw = start + arc * np.linspace(0.0, 1.0, M + 1) + 0.5 * np.pi
    tan0, tan1 = np.array([-np.sin(a[0]), np.cos(a[0])]), np.array([-np.sin(a[-1]), np.cos(a[-1])])
    v = 0.0 if zero_ends else speed
    acc0 = np.zeros(2) if zero_ends else -speed ** 2 / radius * rel[0] / radius
    acc1 = np.zeros(2) if zero_ends else -speed ** 2 / radius * rel[-1] / radius
    dyaw = 0.0 if zero_ends else speed / radius
    bnd = np.concatenate([pts[0], v * tan0, acc0, pts[-1], v * tan1, acc1, [yaw[0], dyaw, 0.0, yaw[-1], dyaw, 0.0]])
    return problems.ProblemBatch(np.array([N], np.int32), np.array([M], np.int32), bnd.reshape(1, 18), np.array([T]),
                                 pts[1:-1].ravel().copy(), yaw[1:-1].copy())


CASES = {
    "one_piece": dict(N=1, M=1, arc=0.5 * np.pi),
    "one_xy_piece_most_yaw_pieces": dict(N=1, M=128, arc=0.5 * np.pi),
    "smallest": dict(N=2, M=1),
    "compiled_limits": dict(N=64, M=128),
    "xy_longer_than_yaw": dict(N=40, M=3),
    "yaw_longer_than_xy": dict(N=3, M=40),
    "zero_boundary_rows": dict(N=12, M=20, zero_ends=True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_minco_evaluation_bitwise(gpu, bumps_map, case):
    import pyoracle as po
    from uneven_planner_b200 import _lib
    params = _lib.default_params()
    K = params.int_K
    one = _arc_problem(**CASES[case])
    # the problem at its initial guess and at a perturbed one, in one batch
    pb = one.select([0, 0])
    offx = np.concatenate([[0], np.cumsum(pb.nvar())])
    offs = np.concatenate([[0], np.cumsum(pb.nsamples(K))])
    _, _, ocx, ocy = pb.offsets()
    rng = np.random.default_rng(7)
    S = int(offs[-1])
    lam = rng.standard_normal(S) * 0.1
    mu = np.abs(rng.standard_normal(6 * S)) * 0.1 * (rng.random(6 * S) < 0.5)
    scx = rng.uniform(0.01, 1.0, 7 * S)
    sfx = rng.uniform(1e-6, 1e-3, pb.B)
    xs = np.concatenate([pb.x0(0), pb.x0(1) * (1 + 1e-3 * rng.standard_normal(pb.nvar()[1]))])
    opt = gpu.BatchALMTrajOpt().init(params).set_environment(bumps_map)
    opt.upload(pb)
    ev = opt.eval_batch(xs, lam, mu, scx, sfx, rho=8.0)
    opt.close()
    op, om = po.params_from(params), po.OracleMap(bumps_map)
    for i in range(pb.B):
        o = po.eval_one(op, om, pb, i, xs[offx[i]:offx[i + 1]], lam[offs[i]:offs[i + 1]], mu[6 * offs[i]:6 * offs[i + 1]],
                        scx[7 * offs[i]:7 * offs[i + 1]], sfx[i], 8.0)
        assert np.all(np.isfinite(o["c_xy"])) and np.all(np.isfinite(o["c_yaw"])), i
        assert np.array_equal(ev["c_xy"][ocx[i]:ocx[i + 1]], o["c_xy"]) and np.array_equal(ev["c_yaw"][ocy[i]:ocy[i + 1]], o["c_yaw"]), i
        assert ev["f"][i] == o["f"], i
        assert np.array_equal(ev["grad"][offx[i]:offx[i + 1]], o["grad"]), i
        assert np.array_equal(ev["hx"][offs[i]:offs[i + 1]], o["hx"]) and np.array_equal(ev["gx"][6 * offs[i]:6 * offs[i + 1]], o["gx"]), i
