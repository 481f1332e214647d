"""Phase B of an evaluation (gradient accumulation, cost chain, adjoint sweeps) at the edges of its schedule, bit for bit against the
CPU oracle: four-warp groups, two-warp groups that join into four-warp groups (adoption), more than 32 pieces per problem (tasks take
more than one round), yaw pieces without samples, and single-warp evaluations (eval_kernel) at random duals."""
import os

import numpy as np
import pytest

from harness import gpu  # noqa: F401


pytestmark = pytest.mark.gpu


def _params(use_scaling=1, int_K=None):
    from uneven_planner_b200 import _lib
    p = _lib.default_params()
    p.use_scaling = use_scaling
    if int_K is not None:
        p.int_K = int_K
    return p


def _solve_and_compare(gpu, m, pb, params):
    import pyoracle as po
    opt = gpu.BatchALMTrajOpt().init(params).set_environment(m)
    res, cxy, cyaw = opt.optimize(pb)
    opt.close()
    ores = po.solve_batch(po.params_from(params), po.OracleMap(m), pb, threads=min(32, os.cpu_count()))
    _, _, ocx, ocy = pb.offsets()
    for i in range(pb.B):
        r, ocxy, ocyaw, _ = ores[i]
        g = res[i]
        assert (g.ret_code, g.outer_iters, g.n_evals, g.n_lbfgs_iters) == (r.ret_code, r.outer_iters, r.n_evals, r.n_lbfgs_iters), i
        assert g.inner_cost == r.inner_cost, i
        assert np.array_equal(cxy[ocx[i]:ocx[i + 1]], ocxy) and np.array_equal(cyaw[ocy[i]:ocy[i + 1]], ocyaw), i


def _long_problems(m, B, seed):
    """problems whose Dubins paths span most of the map: many of them have more than 32 xy pieces"""
    from uneven_planner_b200 import problems
    pb = problems.generate(m, B, seed=seed, min_dist=8.5)
    assert int(np.max(pb.N)) > 32
    return pb


@pytest.mark.parametrize("use_scaling", [0, 1])
def test_four_warp_groups_more_than_32_pieces(gpu, hill_map, use_scaling):
    # a batch this small gives every problem a four-warp group (the launch plan's first tier)
    pb = _long_problems(hill_map, 16, seed=7)
    _solve_and_compare(gpu, hill_map, pb, _params(use_scaling))


def test_two_warp_groups_with_adoption(gpu, bumps_map):
    # more problems than half the warp slots of an H100: two-warp groups, two per CTA; at the end of the launch the warps of a
    # finished slot join the other slot's group, which then runs phase B on four warps
    from uneven_planner_b200 import problems
    pb = problems.generate(bumps_map, 640, seed=13, n_max=40)
    _solve_and_compare(gpu, bumps_map, pb, _params(1))


def test_yaw_pieces_without_samples(gpu, bumps_map):
    # two samples per xy piece, at its ends: N + 1 distinct sample times, so a problem with more than N + 1 yaw pieces has yaw pieces
    # without a sample
    pb = _long_problems(bumps_map, 24, seed=5)
    params = _params(1, int_K=1)
    assert np.any(pb.M > pb.N + 1)
    _solve_and_compare(gpu, bumps_map, pb, params)


@pytest.mark.parametrize("use_scaling,int_K", [(0, 16), (1, 16), (1, 1), (1, 64)])
def test_single_warp_evaluation_random_duals(gpu, hill_map, use_scaling, int_K):
    import pyoracle as po
    params = _params(use_scaling, int_K)
    pb = _long_problems(hill_map, 12, seed=9)
    K = params.int_K
    offx = np.concatenate([[0], np.cumsum(pb.nvar())])
    offs = np.concatenate([[0], np.cumsum(pb.nsamples(K))])
    _, _, ocx, ocy = pb.offsets()
    rng = np.random.default_rng(int_K + 100 * use_scaling)
    S = int(offs[-1])
    lam = rng.standard_normal(S) * 0.1
    mu = np.abs(rng.standard_normal(6 * S)) * 0.1 * (rng.random(6 * S) < 0.5)
    scx = rng.uniform(0.01, 1.0, 7 * S)
    sfx = rng.uniform(1e-6, 1e-3, pb.B)
    xs = np.concatenate([pb.x0(i) * (1 + 1e-3 * rng.standard_normal(pb.nvar()[i])) for i in range(pb.B)])
    opt = gpu.BatchALMTrajOpt().init(params).set_environment(hill_map)
    opt.upload(pb)
    ev = opt.eval_batch(xs, lam, mu, scx, sfx, rho=8.0)
    opt.close()
    op, om = po.params_from(params), po.OracleMap(hill_map)
    for i in range(pb.B):
        o = po.eval_one(op, om, pb, i, xs[offx[i]:offx[i + 1]], lam[offs[i]:offs[i + 1]], mu[6 * offs[i]:6 * offs[i + 1]],
                        scx[7 * offs[i]:7 * offs[i + 1]], sfx[i], 8.0)
        assert ev["f"][i] == o["f"], i
        assert np.array_equal(ev["grad"][offx[i]:offx[i + 1]], o["grad"]), i
        assert np.array_equal(ev["c_xy"][ocx[i]:ocx[i + 1]], o["c_xy"]) and np.array_equal(ev["c_yaw"][ocy[i]:ocy[i + 1]], o["c_yaw"]), i
