"""Environments on the GPU (include/ualm.h, ualm_select_env and the *_env entry points): one batch that mixes the four terrains,
each problem in its own environment (parameter set + map grid), gives every problem exactly the result it has in a batch of its
environment alone -- on the parity path (also against the goldens, pipelined, budgeted and under a deadline), through the phase
entry points, and on the throughput path.  Workload: the golden problems of hill, desert, volcano and forest (tests/test_envs.py)."""
import struct
import subprocess

import numpy as np
import pytest

from harness import build_driver, ctx, gpu, pieces, same_values  # noqa: F401
from workloads import NAMES, mixed_golden_batch


pytestmark = pytest.mark.gpu
STOPPED = 3


@pytest.fixture(scope="module")
def work(terrain, golden):
    maps, params, golds, pbs, mixed, perm = mixed_golden_batch(terrain, golden)
    start = np.concatenate([[0], np.cumsum([p.B for p in pbs])])
    env = np.searchsorted(start, perm, side="right") - 1
    where = [(int(e), int(q - start[e])) for e, q in zip(env, perm)]        # mixed problem i = problem j of terrain e
    return dict(maps=maps, params=params, golds=golds, pbs=pbs, mixed=mixed, where=where)


@pytest.fixture(scope="module")
def single(gpu, work):
    """single-environment solves of every terrain's problems: single(precision, budget) -> [per terrain: pieces]"""
    cache = {}

    def get(precision, budget=0):
        if (precision, budget) not in cache:
            out = []
            for e in range(len(NAMES)):
                opt = gpu.BatchALMTrajOpt(precision=precision).init(work["params"][e]).set_environment(work["maps"][e]).set_budget(budget)
                out.append(pieces(work["pbs"][e], opt.optimize(work["pbs"][e])))
                opt.close()
            cache[(precision, budget)] = out
        return cache[(precision, budget)]
    return get


def _check_mixed(work, got, ref):
    for i, (e, j) in enumerate(work["where"]):
        assert same_values(got[i], ref[e][j]), (i, NAMES[e], j)


def test_parity_mixed_golden_batch(gpu, work, single):
    from uneven_planner_b200 import _lib
    mixed = work["mixed"]
    opt = ctx(gpu, 64, work["params"], work["maps"])
    out = opt.optimize(mixed)
    opt.close()
    res, cxy, cyaw = out
    _, _, ocx, ocy = mixed.offsets()
    for i, (e, j) in enumerate(work["where"]):
        g = work["golds"][e]
        gcx = np.concatenate([[0], np.cumsum(12 * work["pbs"][e].N.astype(np.int64))])
        gcy = np.concatenate([[0], np.cumsum(6 * work["pbs"][e].M.astype(np.int64))])
        r = res[i]
        assert (r.ret_code, r.n_evals, r.outer_iters, r.inner_cost) == (g["ret_code"][j], g["n_evals"][j], g["outer_iters"][j], g["inner_cost"][j]), (i, NAMES[e])
        assert np.array_equal(cxy[ocx[i]:ocx[i + 1]], g["c_xy"][gcx[j]:gcx[j + 1]]), (i, NAMES[e])
        assert np.array_equal(cyaw[ocy[i]:ocy[i + 1]], g["c_yaw"][gcy[j]:gcy[j + 1]]), (i, NAMES[e])
    _check_mixed(work, pieces(mixed, out), single(64))
    assert len(_lib.Result._fields_) == 17      # the record bytes compared cover res_h, res_g and the piece durations


def test_parity_pipelined_budget_and_deadline(gpu, work, single):
    mixed = work["mixed"]
    opt = ctx(gpu, 64, work["params"], work["maps"]).set_budget(50)
    tickets = [opt.submit(mixed, depth=3) for _ in range(3)]
    for t in tickets:
        _check_mixed(work, pieces(mixed, opt.wait(t)), single(64, 50))
    assert any(single(64, 50)[e][j][0] != single(64)[e][j][0] for e, j in work["where"])     # the budget acted
    opt.set_budget(0)
    free = single(64)
    out = opt.wait(opt.submit(mixed, depth=1), timeout_ms=5.0)
    got = pieces(mixed, out)
    for i, (e, j) in enumerate(work["where"]):
        r = out[0][i]
        assert r.ret_code in (0, 1, 2, STOPPED), i
        if r.ret_code != STOPPED:
            assert same_values(got[i], free[e][j]), i
    _check_mixed(work, pieces(mixed, opt.wait(opt.submit(mixed, depth=1))), free)     # the lane is reusable
    opt.close()


def _split(arr, sizes):
    o = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    return [arr[o[i]:o[i + 1]] for i in range(len(sizes))]


def test_other_entry_points_per_environment(gpu, work):
    mixed, pbs = work["mixed"], work["pbs"]
    K = [p.int_K for p in work["params"]]

    def run(opt, pb, Ks):
        S = pb.N.astype(np.int64) * (np.array(Ks, np.int64) + 1)
        n = pb.nvar()
        opt.upload(pb)
        ev = opt.eval_batch()
        sfx, scx = opt.init_scaling_batch()
        opt.solve_resident(); opt.sync()
        feas = opt.feasibility(0.01)
        ex = opt.mpc_export(pb.N, pb.M)
        rows = []
        for i, (g, h, gx, c_xy, c_yaw, s_cx) in enumerate(zip(_split(ev["grad"], n), _split(ev["hx"], S), _split(ev["gx"], 6 * S),
                                                            _split(ev["c_xy"], 12 * pb.N), _split(ev["c_yaw"], 6 * pb.M), _split(scx, 7 * S))):
            rows.append(dict(f=ev["f"][i], grad=g, hx=h, gx=gx, c_xy=c_xy, c_yaw=c_yaw, sfx=sfx[i], scx=s_cx, feas=feas[i],
                             c_mpc=_split(ex["c_mpc_xy"], 12 * pb.N)[i], dev=ex["dev"][i]))
        return rows

    opt = ctx(gpu, 64, work["params"], work["maps"])
    got = run(opt, mixed, [K[e] for e in mixed.env])
    opt.close()
    ref = []
    for e in range(len(NAMES)):
        o = gpu.BatchALMTrajOpt().init(work["params"][e]).set_environment(work["maps"][e])
        ref.append(run(o, pbs[e], [K[e]] * pbs[e].B))
        o.close()
    for i, (e, j) in enumerate(work["where"]):
        for k, v in got[i].items():
            assert np.array_equal(v, ref[e][j][k]), (i, NAMES[e], k)


@pytest.mark.parametrize("precision", [32, 65])
def test_throughput_mixed_alone_and_at_depth_4(gpu, work, single, precision):
    mixed = work["mixed"]
    ref = single(precision)
    opt = ctx(gpu, precision, work["params"], work["maps"])
    _check_mixed(work, pieces(mixed, opt.optimize(mixed)), ref)
    tickets = [opt.submit(mixed, depth=4) for _ in range(4)]
    for t in tickets:
        _check_mixed(work, pieces(mixed, opt.wait(t)), ref)
    feas = opt.feasibility(0.01)
    assert feas.shape == (mixed.B, 10) and (feas[:, 7] > 0).all()
    with pytest.raises(gpu.UalmError, match="mixes environments"):
        opt.upload(mixed)
        opt.time_penalty_kernel(2)
    opt.close()


@pytest.mark.parametrize("precision", [64, 32])
def test_env_argument_and_state_checks(gpu, work, precision):
    from uneven_planner_b200 import _lib, problems
    mixed = work["mixed"]
    opt = ctx(gpu, precision, work["params"], work["maps"])
    err = lambda code: pytest.raises(gpu.UalmError, match="error %d" % code)
    for bad in (4, -1):
        with err(_lib.UALM_EINVAL):
            opt.optimize(problems.concat([mixed.select([0])], [bad]))
        with err(_lib.UALM_EINVAL):
            opt.select_env(bad)
    # environment without a grid (parameters only), and one with nothing bound
    opt2 = gpu.BatchALMTrajOpt(precision=precision).init(work["params"][0]).set_environment(work["maps"][0]).init(work["params"][3], env=3)
    for e in (3, 2):
        with err(_lib.UALM_ESTATE):
            opt2.optimize(problems.concat([mixed.select([0])], [e]))
    opt2.close()
    # binding is refused while a batch is in flight
    t = opt.submit(mixed, depth=1)
    with err(_lib.UALM_ESTATE):
        opt.init(work["params"][2], env=2)
    with err(_lib.UALM_ESTATE):
        opt.set_environment(work["maps"][1], env=1)
    opt.wait(t)
    # rebinding environment 2 invalidates the resident batch
    opt.upload(mixed)
    opt.init(work["params"][2], env=2)
    with err(_lib.UALM_ESTATE):
        opt.solve_resident()
    # env = NULL is environment 0 for every problem
    one = work["pbs"][0]
    a = pieces(one, opt.optimize(one))
    zero = one.select(np.arange(one.B))
    zero.env = np.zeros(one.B, np.int32)
    b = pieces(zero, opt.optimize(zero))
    assert all(same_values(x, y) for x, y in zip(a, b))
    ref = opt.optimize(mixed)
    opt.close()
    if precision == 64:
        # ualm_solve_batch_multi_env over two contexts (on one device here) equals the single-context result
        opts = [ctx(gpu, 64, work["params"], work["maps"]) for _ in range(2)]
        got = gpu.solve_batch_multi(opts, mixed)
        for o in opts:
            o.close()
        assert all(same_values(x, y) for x, y in zip(pieces(mixed, got), pieces(mixed, ref)))


def test_cpp_adapter_environment_overloads(gpu, bumps_map, tmp_path):
    from uneven_planner_b200 import _lib, problems
    exe = build_driver("env_driver", tmp_path)
    pb = problems.generate(bumps_map, 6, seed=5)
    pb.env = np.array([0, 1, 1, 0, 1, 0], np.int32)
    case = str(tmp_path / "envs.bin")
    with open(case, "wb") as f:
        f.write(struct.pack("<4i", *bumps_map.shape, pb.B))
        f.write(bumps_map.cells.tobytes())
        for a in (pb.N, pb.M, pb.env):
            f.write(np.ascontiguousarray(a, np.int32).tobytes())
        for a in (pb.bnd, pb.total_time, pb.inner_xy, pb.inner_yaw):
            f.write(np.ascontiguousarray(a, np.float64).tobytes())
    r = subprocess.run([exe, case], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    forest = _lib.default_params()
    forest.rho_T, forest.max_sig, forest.use_scaling = 500.0, 0.001, 0
    opt = gpu.BatchALMTrajOpt().init(_lib.default_params()).set_environment(bumps_map).init(forest, env=1).set_environment(bumps_map, env=1)
    res, cxy, _ = opt.optimize(pb)
    opt.close()
    _, _, ocx, _ = pb.offsets()
    want = ["%d %d %d %d %r %r" % (p, i, res[i].ret_code, res[i].n_evals, float(res[i].inner_cost), float(cxy[ocx[i] + 1])) for p in range(2)
            for i in range(pb.B)]
    got = [" ".join(ln.split()[:4] + [repr(float(x)) for x in ln.split()[4:]]) for ln in r.stdout.strip().splitlines()]
    assert got == want


@pytest.mark.parametrize("precision", [64, 32])
def test_refused_binding_leaves_the_environment_unbound(gpu, work, precision):
    """a binding the context refuses (engine limits, a batch in flight) binds nothing: a later upload into that environment is
    UALM_ESTATE, not a solve with unset parameters or grid"""
    import copy
    from uneven_planner_b200 import _lib, problems
    err = lambda code: pytest.raises(gpu.UalmError, match="error %d" % code)
    one = work["pbs"][0].select(np.arange(2))
    if precision == 32:
        # int_K = 128 is within the parity path's range but over the throughput path's (<= 127)
        big = copy.copy(work["params"][0])
        big.int_K = 128
        opt = gpu.BatchALMTrajOpt(precision=precision)
        with err(_lib.UALM_ELIMIT):
            opt.init(big)
        opt.set_environment(work["maps"][0])
        with err(_lib.UALM_ESTATE):
            opt.optimize(one)
        opt.init(work["params"][0])
        assert opt.optimize(one)[0][0].n_evals > 0
        opt.close()
    opt = gpu.BatchALMTrajOpt(precision=precision).init(work["params"][0]).set_environment(work["maps"][0])
    t = opt.submit(work["mixed"].select(np.nonzero(work["mixed"].env == 0)[0]), depth=1)
    with err(_lib.UALM_ESTATE):
        opt.init(work["params"][2], env=2)
    with err(_lib.UALM_ESTATE):
        opt.set_environment(work["maps"][2], env=2)
    opt.wait(t)
    in2 = problems.concat([one], [2])
    with err(_lib.UALM_ESTATE):
        opt.upload(in2)
    with err(_lib.UALM_ESTATE):
        opt.optimize(in2)
    # select_env: init / set_environment without `env` bind the selected environment
    opt.select_env(2).init(work["params"][2])
    with err(_lib.UALM_ESTATE):
        opt.optimize(in2)                   # parameters, no grid yet
    opt.set_environment(work["maps"][2])
    assert opt.env == 2 and opt.env_params[2] is work["params"][2]
    assert opt.optimize(in2)[0][0].n_evals > 0
    opt.close()


def test_parity_phase_entry_points_on_mixed_parameters(gpu, work):
    """ualm_time_penalty_kernel refuses a mixed batch on the parity path too; eval_batch's default rho needs one rho over the batch"""
    import copy
    from uneven_planner_b200 import _lib, problems
    pb = problems.concat([work["pbs"][0].select([0]), work["pbs"][3].select([0])], [0, 1])
    p1 = copy.copy(work["params"][3])
    p1.rho = 2.0 * work["params"][0].rho
    opt = gpu.BatchALMTrajOpt().init(work["params"][0]).set_environment(work["maps"][0])
    opt.init(p1, env=1).set_environment(work["maps"][3])
    opt.upload(pb)
    with pytest.raises(gpu.UalmError, match="error %d.*mixes environments" % _lib.UALM_EINVAL):
        opt.time_penalty_kernel(2)
    with pytest.raises(ValueError, match="differ in rho"):
        opt.eval_batch()
    ev = opt.eval_batch(rho=p1.rho)
    assert np.isfinite(ev["f"]).all()
    opt.close()
