"""One evaluation of the parity path against the CPU oracle, bit for bit, at the MINCO system sizes where the forward sweep
L y = b, which runs inside the banded LU (lu_dual), is most likely to go wrong: the smallest systems (only the last-six pivot
types), the compiled limits, an xy system longer than the yaw system and the reverse, and right-hand sides with exact-zero
boundary rows."""
import numpy as np
import pytest

from harness import gpu  # noqa: F401
from workloads import _arc_problem


pytestmark = pytest.mark.gpu


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
