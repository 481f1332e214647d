"""The C-ABI boundary beyond one synchronous batch (include/ualm.h): the exact bench workload against the oracle, several batches
in flight (lanes, submit / wait), the reference's double map grid, per-problem limits, state invalidation, the multi-device entry,
and the k > 1000 cancel of earlyExit (alm_traj_opt.cpp:1016) -- all through libualm.so on the GPU, bit-compared with the oracle."""
import ctypes as C
import os

import numpy as np
import pytest

from harness import gpu  # noqa: F401
from workloads import _with_oversize


pytestmark = pytest.mark.gpu


def _same(pb, a, b):
    """two (results, c_xy, c_yaw) triples of the same batch are bit-identical"""
    ra, xa, ya = a
    rb, xb, yb = b
    for i in range(pb.B):
        for f in ("ret_code", "outer_iters", "n_evals", "n_lbfgs_iters", "last_lbfgs_ret", "inner_cost", "total_T", "res_h", "res_g", "rho_final",
                  "piece_T_xy", "piece_T_yaw"):
            assert getattr(ra[i], f) == getattr(rb[i], f), (i, f)
    assert np.array_equal(xa, xb) and np.array_equal(ya, yb)


def _vs_oracle(pb, res, cxy, cyaw, ores):
    _, _, ocx, ocy = pb.offsets()
    for i in range(pb.B):
        r, ocxy, ocyaw, _ = ores[i]
        g = res[i]
        assert (g.ret_code, g.outer_iters, g.n_evals, g.n_lbfgs_iters, g.last_lbfgs_ret) == \
               (r.ret_code, r.outer_iters, r.n_evals, r.n_lbfgs_iters, r.last_lbfgs_ret), i
        assert g.inner_cost == r.inner_cost and g.total_T == r.total_T and g.res_h == r.res_h and g.res_g == r.res_g, i
        assert np.array_equal(cxy[ocx[i]:ocx[i + 1]], ocxy) and np.array_equal(cyaw[ocy[i]:ocy[i + 1]], ocyaw), i


def test_bench_workload_matches_oracle_bitwise(gpu, hill_map):
    """bench.py's default workload (BASELINE configs[1]: B = 1024, seed 0, hill, run_hill.yaml): every record and every coefficient of
    the CUDA path equals the oracle's, and so do the two numbers the bench line reports (converged count, evaluations)."""
    import pyoracle as po
    from uneven_planner_b200 import _lib, problems
    params = _lib.default_params()
    pb = problems.generate(hill_map, 1024, seed=0)
    opt = gpu.BatchALMTrajOpt().init(params).set_environment(hill_map)
    res, cxy, cyaw = opt.optimize(pb)
    opt.close()
    ores = po.solve_batch(po.params_from(params), po.OracleMap(hill_map), pb, threads=len(os.sched_getaffinity(0)))
    _vs_oracle(pb, res, cxy, cyaw, ores)
    assert sum(1 for r in res if r.ret_code == 0) == sum(1 for r in ores if r[0].ret_code == 0)
    assert sum(r.n_evals for r in res) == sum(r[0].n_evals for r in ores)


def test_piece_durations_are_the_last_evaluations(gpu, hill_map):
    """ualm_result_t.piece_T_xy / piece_T_yaw = calTfromTau of the LAST evaluated tau (alm_traj_opt.h:257-261; getTraj() carries T1(i))."""
    import pyoracle as po
    from uneven_planner_b200 import _lib, problems
    params = _lib.default_params()
    pb = problems.generate(hill_map, 8, seed=21)
    opt = gpu.BatchALMTrajOpt().init(params).set_environment(hill_map)
    res, cxy, cyaw = opt.optimize(pb)
    feas = opt.feasibility(0.01)
    opt.close()
    for i in range(pb.B):
        assert res[i].piece_T_xy == feas[i, 8] and res[i].piece_T_yaw == feas[i, 9]
        tt = 0.0
        for _ in range(int(pb.N[i])):
            tt += res[i].piece_T_xy
        assert tt == res[i].total_T
        assert abs(res[i].piece_T_xy * pb.N[i] - res[i].piece_T_yaw * pb.M[i]) < 1e-12 * res[i].total_T


def test_batches_in_flight_return_the_synchronous_results(gpu, hill_map):
    """ualm_submit_batch / ualm_wait_batch with 3 batches in flight, and ualm_select_lane + upload / solve_resident / download on
    two lanes at once: identical to one ualm_solve_batch per batch."""
    from uneven_planner_b200 import _lib, problems
    params = _lib.default_params()
    pbs = [problems.generate(hill_map, 96, seed=100 + k) for k in range(5)]
    opt = gpu.BatchALMTrajOpt().init(params).set_environment(hill_map)
    sync = [opt.optimize(pb) for pb in pbs]
    depth = 3
    tickets, got = [], []
    for k, pb in enumerate(pbs):
        if k >= depth:
            got.append(opt.wait(tickets[k - depth]))
        tickets.append(opt.submit(pb, depth=depth))
    for k in range(max(0, len(pbs) - depth), len(pbs)):
        got.append(opt.wait(tickets[k]))
    for pb, a, b in zip(pbs, sync, got):
        _same(pb, a, b)
    # a fourth submit without a wait must be refused, not overwrite a running batch
    t = [opt.submit(pbs[k], depth=2) for k in range(2)]
    with pytest.raises(gpu.UalmError):
        opt.submit(pbs[2], depth=2)
    for k in range(2):
        _same(pbs[k], sync[k], opt.wait(t[k]))
    # resident lanes
    opt.select_lane(0); opt.upload(pbs[0])
    opt.select_lane(1); opt.upload(pbs[1])
    opt.select_lane(0); opt.mark_begin(); opt.solve_resident()
    opt.select_lane(1); opt.solve_resident()
    ms = opt.mark_end()
    assert ms > 0.0
    opt.select_lane(1); _same(pbs[1], sync[1], opt.download())
    opt.select_lane(0); _same(pbs[0], sync[0], opt.download())
    opt.close()


def test_double_map_grid_is_read_without_rounding(gpu, bumps_map):
    """ualm_set_map_f64: the reference's map_buffer is double (RXS2, uneven_map.h:36-64).  A grid whose cells are NOT float32
    representable gives bit-identical results to the oracle reading the same doubles; with repack_to_float the float path's."""
    import pyoracle as po
    from uneven_planner_b200 import _lib, maps, problems
    rng = np.random.default_rng(5)
    c64 = bumps_map.cells.astype(np.float64) * (1.0 + 1e-9 * rng.standard_normal(bumps_map.cells.shape))
    m64 = maps.UnevenMapData(bumps_map.geom, c64.astype(np.float32), "bumps64", cells64=c64)
    params = _lib.default_params()
    pb = problems.generate(bumps_map, 16, seed=2)
    opt = gpu.BatchALMTrajOpt().init(params).set_environment(m64)
    res, cxy, cyaw = opt.optimize(pb)
    ores = po.solve_batch(po.params_from(params), po.OracleMap(m64), pb, threads=8)
    _vs_oracle(pb, res, cxy, cyaw, ores)
    # the float32 rounding of the same grid is a different (also valid) input: results differ from the double grid's ...
    mf = maps.UnevenMapData(bumps_map.geom, c64.astype(np.float32), "bumps32")
    opt.set_environment(m64, repack_to_float=True)
    res_r = opt.optimize(pb)
    opt.set_environment(mf)
    res_f = opt.optimize(pb)
    _same(pb, res_r, res_f)
    assert any(res_f[0][i].inner_cost != res[i].inner_cost for i in range(pb.B))
    opt.close()


def test_problem_over_the_limits_fails_alone(gpu, bumps_map):
    """N > 64 or M > 128: that record says UALM_ELIMIT, its outputs are zero, and every other problem of the batch is solved as usual"""
    from uneven_planner_b200 import _lib, problems
    params = _lib.default_params()
    pb = problems.generate(bumps_map, 9, seed=31)
    opt = gpu.BatchALMTrajOpt().init(params).set_environment(bumps_map)
    ref = opt.optimize(pb)
    at = 4
    pbx = _with_oversize(pb, at)
    res, cxy, cyaw = opt.optimize(pbx)
    feas = opt.feasibility(0.01)
    _, _, ocx, ocy = pbx.offsets()
    assert res[at].ret_code == _lib.UALM_ELIMIT and res[at].n_evals == 0
    assert not cxy[ocx[at]:ocx[at + 1]].any() and not cyaw[ocy[at]:ocy[at + 1]].any() and not feas[at].any()
    keep = [i for i in range(pbx.B) if i != at]
    _, _, rcx, rcy = pb.offsets()
    for j, i in enumerate(keep):
        assert (res[i].ret_code, res[i].n_evals, res[i].inner_cost) == (ref[0][j].ret_code, ref[0][j].n_evals, ref[0][j].inner_cost)
        assert np.array_equal(cxy[ocx[i]:ocx[i + 1]], ref[1][rcx[j]:rcx[j + 1]]) and np.array_equal(cyaw[ocy[i]:ocy[i + 1]], ref[2][rcy[j]:rcy[j + 1]])
    # the phase entry points refuse such a batch instead of indexing past their buffers
    opt.upload(pbx)
    with pytest.raises(gpu.UalmError):
        opt.eval_batch()
    opt.close()


def test_resident_batch_is_invalidated_by_its_inputs(gpu, bumps_map):
    """ualm_set_params changes int_K / mem_size, which are baked into an uploaded batch: the batch must be uploaded again.
    An upload that fails validation does not disturb the batch that is resident."""
    from uneven_planner_b200 import _lib, problems
    params = _lib.default_params()
    pb = problems.generate(bumps_map, 6, seed=41)
    opt = gpu.BatchALMTrajOpt().init(params).set_environment(bumps_map)
    opt.upload(pb)
    opt.solve_resident(); opt.sync()
    first = opt.download()
    p2 = _lib.default_params(); p2.int_K = 8; p2.mem_size = 16
    opt.init(p2)
    for call in (opt.solve_resident, opt.eval_batch, lambda: opt.feasibility(0.01), opt.download, lambda: opt.mpc_export(pb.N, pb.M)):
        with pytest.raises(gpu.UalmError):
            call()
    opt.init(params)
    opt.upload(pb)
    with pytest.raises(gpu.UalmError):
        opt.mpc_export(pb.N, pb.M)       # uploaded, not yet solved
    opt.solve_resident()
    _same(pb, first, opt.download())
    # a rejected upload (validated before anything is touched) leaves the resident batch exactly as it was
    bad = pb.select(np.arange(pb.B)); bad.total_time[2] = 0.0
    with pytest.raises(gpu.UalmError):
        opt.upload(bad)
    opt.solve_resident()
    _same(pb, first, opt.download())
    L = opt.L
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int32)
    N = np.ascontiguousarray(pb.N, np.int32); M = np.ascontiguousarray(pb.M, np.int32)
    rc = L.ualm_upload(opt.h, pb.B, N.ctypes.data_as(ip), M.ctypes.data_as(ip), pb.bnd.ctypes.data_as(dp), pb.total_time.ctypes.data_as(dp), None, None)
    assert rc == _lib.UALM_EINVAL      # NULL inner waypoint arrays with N > 1
    opt.close()


def test_inner_solve_past_1000_iterations_is_cancelled(gpu, bumps_map):
    """earlyExit (alm_traj_opt.cpp:1016): k > 1e3 cancels lbfgs_optimize.  With the stopping tests switched off (g_epsilon tiny,
    past = 0) every inner solve runs into the cancel: LBFGS_CANCELED (2) is a tolerated return code, the ALM loop goes on
    (alm_traj_opt.cpp:239-245), and the CUDA path follows the oracle bit for bit through the > 1000 iterations per problem."""
    import pyoracle as po
    from uneven_planner_b200 import _lib, problems
    LBFGS_CANCELED = 2
    pb = problems.generate(bumps_map, 64, seed=51, n_max=30).select(np.arange(6))
    for outer in (0.0, 1.0):      # one inner solve (ends in the cancel), then two (the ALM loop continues after a cancelled solve)
        params = _lib.default_params()
        params.g_epsilon = 1e-300; params.past = 0; params.max_iter = outer; params.mem_size = 1
        opt = gpu.BatchALMTrajOpt().init(params).set_environment(bumps_map)
        res, cxy, cyaw = opt.optimize(pb)
        opt.close()
        ores = po.solve_batch(po.params_from(params), po.OracleMap(bumps_map), pb, threads=6)
        _vs_oracle(pb, res, cxy, cyaw, ores)
        if outer == 0.0:
            assert all(r.last_lbfgs_ret == LBFGS_CANCELED and r.n_lbfgs_iters == 1001 for r in res), [(r.last_lbfgs_ret, r.n_lbfgs_iters) for r in res]
        else:
            assert all(r.outer_iters == 2 and r.n_lbfgs_iters > 1001 for r in res)


def test_multi_device_entry(gpu, bumps_map):
    """ualm_solve_batch_multi: contexts on different devices, one host process, results in problem order, identical to one device"""
    import torch
    from uneven_planner_b200 import _lib, problems
    nd = torch.cuda.device_count()
    params = _lib.default_params()
    pb = problems.generate(bumps_map, 33, seed=61)
    one = gpu.BatchALMTrajOpt(device=0).init(params).set_environment(bumps_map)
    ref = one.optimize(pb)
    # also with two contexts on the same device when only one GPU is visible (the sharding and scatter logic is the same)
    devs = list(range(min(nd, 4))) if nd > 1 else [0, 0]
    opts = [gpu.BatchALMTrajOpt(device=d).init(params).set_environment(bumps_map) for d in devs]
    _same(pb, ref, gpu.solve_batch_multi(opts, pb))
    for o in opts:
        o.close()
    one.close()
