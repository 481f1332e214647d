"""The throughput path (ualm_create(precision = 65 "fast64" / 32), csrc/ualm_tp*.cu) against the CPU oracle.

It is NOT bit-comparable with the oracle by construction (re-associated sums, FMA, CUDA libm, nondimensionalised prefactored MINCO
system, float penalty samples at precision 32), and the solve is chaotic with respect to last-bit differences (DESIGN.md section 2).  So:
  * one innerCallback evaluation and initScaling at fixed inputs are bounded tightly (the kernel-level gate):
        precision 65: f, gradient, constraint values, coefficients, scales within 1e-9 relative of the oracle (measured ~1e-13);
        precision 32: within 1e-4 (measured ~1e-5), the north star's fp32 kernel-level tolerance being 1e-5 .. 1e-4 on these sums;
  * whole solves are compared as POPULATIONS (converged fraction, work, cost distribution, feasibility), and as exact self-consistency
    (the same batch gives bit-identical results alone, pipelined with other batches, and with / without TMA tile staging)."""
import os

import numpy as np
import pytest

from harness import gpu  # noqa: F401
from workloads import TOL


pytestmark = pytest.mark.gpu


def _rel(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.mark.parametrize("prec", [65, 32])
@pytest.mark.parametrize("which", ["hill", "bumps"])
def test_single_evaluation_within_tolerance(gpu, prec, which, request):
    """one innerCallback (alm_traj_opt.cpp:280-347) at random duals / scales / rho, both branches of every inequality"""
    import pyoracle as po
    from uneven_planner_b200 import _lib, problems
    m = request.getfixturevalue("hill_map" if which == "hill" else "bumps_map")
    params = _lib.default_params()
    K = params.int_K
    pb = problems.generate(m, 24, seed=3)
    offx = np.concatenate([[0], np.cumsum(pb.nvar())]); offs = np.concatenate([[0], np.cumsum(pb.nsamples(K))])
    _, _, ocx, ocy = pb.offsets()
    rng = np.random.default_rng(0)
    S = int(offs[-1])
    lam = rng.standard_normal(S) * 0.1
    mu = np.abs(rng.standard_normal(6 * S)) * 0.1 * (rng.random(6 * S) < 0.5)
    scx = rng.uniform(0.01, 1.0, 7 * S)
    sfx = rng.uniform(1e-6, 1e-3, pb.B)
    xs = np.concatenate([pb.x0(i) * (1 + 1e-3 * rng.standard_normal(pb.nvar()[i])) for i in range(pb.B)])
    opt = gpu.BatchALMTrajOpt(precision=prec).init(params).set_environment(m)
    opt.upload(pb)
    ev = opt.eval_batch(xs, lam, mu, scx, sfx, rho=8.0)
    opt.close()
    op, om = po.params_from(params), po.OracleMap(m)
    t = TOL[prec]
    for i in range(pb.B):
        o = po.eval_one(op, om, pb, i, xs[offx[i]:offx[i + 1]], lam[offs[i]:offs[i + 1]], mu[6 * offs[i]:6 * offs[i + 1]], scx[7 * offs[i]:7 * offs[i + 1]], sfx[i], 8.0)
        assert abs(ev["f"][i] - o["f"]) <= t["f"] * abs(o["f"]), (i, ev["f"][i], o["f"])
        assert _rel(ev["grad"][offx[i]:offx[i + 1]], o["grad"]) <= t["grad"], i
        assert _rel(ev["hx"][offs[i]:offs[i + 1]], o["hx"]) <= t["con"] and _rel(ev["gx"][6 * offs[i]:6 * offs[i + 1]], o["gx"]) <= t["con"], i
        assert _rel(ev["c_xy"][ocx[i]:ocx[i + 1]], o["c_xy"]) <= t["coef"] and _rel(ev["c_yaw"][ocy[i]:ocy[i + 1]], o["c_yaw"]) <= t["coef"], i


@pytest.mark.parametrize("prec", [65, 32])
def test_init_scaling_within_tolerance(gpu, hill_map, prec):
    """initScaling (alm_traj_opt.cpp:349-661) through the waypoint rows of A(1)^-T and one extra forward solve instead of one adjoint
    solve per constraint: every scale_cx entry and scale_fx"""
    import pyoracle as po
    from uneven_planner_b200 import _lib, problems
    params = _lib.default_params()
    pb = problems.generate(hill_map, 8, seed=4)
    opt = gpu.BatchALMTrajOpt(precision=prec).init(params).set_environment(hill_map)
    opt.upload(pb)
    sfx, scx = opt.init_scaling_batch()
    opt.close()
    offs = np.concatenate([[0], np.cumsum(pb.nsamples(params.int_K))])
    op, om = po.params_from(params), po.OracleMap(hill_map)
    t = TOL[prec]
    for i in range(pb.B):
        osfx, oscx = po.init_scaling(op, om, pb, i)
        assert abs(sfx[i] - osfx) <= t["sfx"] * osfx, i
        assert np.max(np.abs(scx[7 * offs[i]:7 * offs[i + 1]] - oscx) / oscx) <= t["scx"], i


@pytest.mark.parametrize("prec", [65, 32])
def test_population_matches_oracle(gpu, hill_map, prec):
    """256 hill problems: the throughput path converges as often as the oracle, with the same amount of work, to trajectories that
    pass the reference's own post-solve scan, and its costs scatter around the oracle's like any bit-different implementation's."""
    import pyoracle as po
    from uneven_planner_b200 import _lib, problems
    params = _lib.default_params()
    pb = problems.generate(hill_map, 256, seed=0)
    opt = gpu.BatchALMTrajOpt(precision=prec).init(params).set_environment(hill_map)
    res, cxy, cyaw = opt.optimize(pb)
    feas = opt.feasibility(0.01)
    opt.close()
    ores = po.solve_batch(po.params_from(params), po.OracleMap(hill_map), pb, threads=len(os.sched_getaffinity(0)))
    rc = np.array([r.ret_code for r in res]); orc = np.array([r[0].ret_code for r in ores])
    ev = np.array([r.n_evals for r in res]); oev = np.array([r[0].n_evals for r in ores])
    assert set(np.unique(rc)) <= {0, 2}
    assert abs((rc == 0).mean() - (orc == 0).mean()) <= 0.06
    assert abs(np.median(ev) - np.median(oev)) <= 0.1 * np.median(oev) and abs(ev.mean() - oev.mean()) <= 0.1 * oev.mean()
    both = (rc == 0) & (orc == 0)
    assert both.mean() >= 0.55          # WHICH problems converge differs chaotically between any two implementations
    cost = np.array([r.inner_cost for r in res]); ocost = np.array([r[0].inner_cost for r in ores])
    relc = np.abs(cost[both] - ocost[both]) / np.abs(ocost[both])
    assert np.median(relc) < 5e-3 and np.percentile(relc, 90) < 5e-2
    T = np.array([r.total_T for r in res]); oT = np.array([r[0].total_T for r in ores])
    assert np.median(np.abs(T[both] - oT[both]) / oT[both]) < 5e-3
    ok = rc == 0
    tol = 1.05
    within = (np.abs(feas[:, 0]) <= params.max_vel * tol) & (np.abs(feas[:, 1]) <= params.max_acc_lon * tol) & (np.abs(feas[:, 2]) <= params.max_acc_lat * tol) & \
             (np.abs(feas[:, 3]) <= params.max_kap * tol) & (-feas[:, 4] >= params.min_cxi / tol) & (feas[:, 5] <= params.max_sig * tol)
    assert (ok & within).sum() >= 0.98 * ok.sum()
    for i in np.flatnonzero(ok)[:32]:
        assert res[i].piece_T_xy == feas[i, 8] and res[i].piece_T_yaw == feas[i, 9]


def test_results_do_not_depend_on_batching_or_tile_staging(gpu, hill_map):
    """every trajectory is advanced by deterministic per-trajectory arithmetic: alone, pipelined with other batches, split into more
    groups, and with the map tiles read directly instead of through TMA, a batch returns bit-identical results"""
    from uneven_planner_b200 import _lib, problems
    params = _lib.default_params()
    pbs = [problems.generate(hill_map, 64, seed=200 + k) for k in range(4)]

    def same(a, b):
        for x, y in zip(a[0], b[0]):
            assert (x.ret_code, x.n_evals, x.n_lbfgs_iters, x.inner_cost, x.total_T) == (y.ret_code, y.n_evals, y.n_lbfgs_iters, y.inner_cost, y.total_T)
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    opt = gpu.BatchALMTrajOpt(precision=32).init(params).set_environment(hill_map)
    alone = [opt.optimize(pb) for pb in pbs]
    tickets = [opt.submit(pb, depth=4) for pb in pbs]
    piped = [opt.wait(t) for t in tickets]
    for a, b in zip(alone, piped):
        same(a, b)
    with pytest.raises(gpu.UalmError):      # a lane in flight is not overwritten
        t = opt.submit(pbs[0], depth=1)
        opt.submit(pbs[1], depth=1)
    opt.wait(t)
    opt.close()
    for env in ({"UALM_TP_TMA": "1"}, {"UALM_TP_SUBGROUPS": "4"}):      # TMA-staged map tiles instead of the direct gather; more groups per batch
        os.environ.update(env)
        try:
            o2 = gpu.BatchALMTrajOpt(precision=32).init(params).set_environment(hill_map)
            same(alone[0], o2.optimize(pbs[0]))
            o2.close()
        finally:
            for k in env:
                os.environ.pop(k)


def test_limits_and_state_checks(gpu, bumps_map):
    """a problem over the compiled limits fails alone (UALM_ELIMIT record); calls out of order are refused"""
    from uneven_planner_b200 import _lib, problems
    from workloads import _with_oversize
    params = _lib.default_params()
    pb = problems.generate(bumps_map, 9, seed=31)
    opt = gpu.BatchALMTrajOpt(precision=32).init(params)
    with pytest.raises(gpu.UalmError):
        opt.optimize(pb)                      # no map bound
    opt.set_environment(bumps_map)
    ref = opt.optimize(pb)
    pbx = _with_oversize(pb, 4)
    res, cxy, cyaw = opt.optimize(pbx)
    _, _, ocx, _ = pbx.offsets()
    assert res[4].ret_code == _lib.UALM_ELIMIT and not cxy[ocx[4]:ocx[5]].any() and not opt.feasibility(0.01)[4].any()
    keep = [i for i in range(pbx.B) if i != 4]
    assert [(res[i].ret_code, res[i].n_evals, res[i].inner_cost) for i in keep] == [(r.ret_code, r.n_evals, r.inner_cost) for r in ref[0]]
    opt.close()
