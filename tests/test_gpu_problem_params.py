"""Per-problem vehicle limits and cost weights on the GPU (include/ualm.h, ualm_problem_params_t and the *_pp entry points): problem b
with row pp[b] gives, bit for bit, what it gives in an environment whose parameters are its environment's with those eight fields
replaced -- against the CPU oracle at precision 64, against environments bound to the same grid on both paths, through the phase entry
points, on tickets (polls, cancels, budget, urgency, several contexts), in the check and the replan.  Workload: stand-in hill problems
with seeded rows from the ranges of a mixed fleet."""
import ctypes as C
import struct
import subprocess

import numpy as np
import pytest

import pyoracle as po
from harness import RECORD, build_driver, ctx, gpu, part, pieces, same_bytes, same_problem, solve_diff  # noqa: F401
from workloads import TOL, hill_desert_world

pytestmark = pytest.mark.gpu
STOPPED = 3
FIELDS = ("rho_T", "rho_ter", "max_vel", "max_acc_lon", "max_acc_lat", "max_kap", "min_cxi", "max_sig")


def fleet_rows(B, seed):
    """B seeded rows: rho_T in {1e3, 1e4, 1e5, 3e5}, the rest uniform over a fleet's ranges"""
    r = np.random.default_rng(seed)
    return np.column_stack([r.choice([1e3, 1e4, 1e5, 3e5], B), r.uniform(1, 20, B), r.uniform(0.3, 1.2, B), r.uniform(2, 8, B),
                            r.uniform(4, 12, B), r.uniform(1, 3, B), r.uniform(0.7, 0.9, B), r.uniform(0.03, 0.1, B)])


def with_row(params, row=None):
    """a copy of Params `params` with the eight per-problem fields replaced by `row` (None: a plain copy)"""
    from uneven_planner_b200 import _lib
    p = _lib.Params()
    C.memmove(C.byref(p), C.byref(params), C.sizeof(p))
    for f, v in zip(FIELDS, [] if row is None else row):
        setattr(p, f, float(v))
    return p


def oracle_solves(params, rows, om, pb):
    """the oracle's solve of every problem of pb with its row's parameters"""
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(16) as ex:
        return list(ex.map(lambda i: po.solve_one(po.params_from(with_row(params, rows[i])), om, pb, i), range(pb.B)))


def rows_of(params, B):
    from uneven_planner_b200 import _lib
    return np.tile(_lib.problem_params(params), (B, 1))


def with_params(pb, rows):
    from uneven_planner_b200 import problems
    out = problems.concat([pb], [0])
    out.env, out.params = pb.env, None if rows is None else np.asarray(rows, np.float64)
    return out


@pytest.fixture(scope="module")
def world(golden):
    return hill_desert_world(golden)


@pytest.mark.parametrize("use_scaling", [1, 0])
def test_oracle_parity_at_64(gpu, world, use_scaling):
    params = with_row(world["params"])
    params.use_scaling = use_scaling
    pb = world["bench"].select(range(64))
    rows = fleet_rows(pb.B, seed=11 + use_scaling)
    opt = ctx(gpu, 64, params, world["g0"])
    got = opt.optimize(with_params(pb, rows))
    plain = opt.optimize(pb)
    opt.close()
    for i, o in enumerate(oracle_solves(params, rows, po.OracleMap(world["g0"]), pb)):
        d = solve_diff(part(pb, got, i), (o[0], o[1], o[2]))
        assert not d, (i, d)
    differ = sum(not same_problem(pb, got, plain, i) for i in range(pb.B))
    assert differ > 0.9 * pb.B, differ      # the rows are read


def _classes(params):
    """four vehicle classes: (Params of the class, its row)"""
    return [(with_row(params, row), row) for row in fleet_rows(4, seed=5)]


@pytest.mark.parametrize("precision", [64, 32, 65])
def test_rows_against_environments(gpu, world, precision):
    params = world["params"]
    cls = _classes(params)
    pb = world["a64"]                           # 1090 problems: more than the resident slots of one pass on the parity path
    k = np.arange(pb.B) % 4
    env_ctx = ctx(gpu, precision, [c[0] for c in cls], [world["g0"]] * 4)
    mixed = with_params(pb, None)
    mixed.env = k.astype(np.int32)
    want = pieces(pb, env_ctx.optimize(mixed))
    env_ctx.close()
    opt = ctx(gpu, precision, params, world["g0"])
    rows = np.array([cls[q][1] for q in k])
    got = pieces(pb, opt.optimize(with_params(pb, rows)))
    opt.close()
    assert all(same_bytes(a, b) for a, b in zip(got, want))
    # a mixed-environment batch: the rows override the eight fields only (the desert grid and another int_K in environment 1)
    p1 = with_row(params)
    p1.int_K = 12
    two = ctx(gpu, precision, [params, p1], [world["g0"], world["g1"]])
    both = with_params(pb.select(range(128)), rows[:128])
    both.env = (np.arange(128) % 2).astype(np.int32)
    got = pieces(both, two.optimize(both))
    two.close()
    for e in (0, 1):
        idx = np.flatnonzero(both.env == e)
        envs = [with_row(params if e == 0 else p1, cls[q][1]) for q in range(4)]
        o = ctx(gpu, precision, envs, [world["g0"] if e == 0 else world["g1"]] * 4)
        sub = with_params(both.select(idx), None)
        sub.env = (idx % 4).astype(np.int32)
        want = pieces(sub, o.optimize(sub))
        o.close()
        assert all(same_bytes(got[i], w) for i, w in zip(idx, want)), e


@pytest.mark.parametrize("precision", [64, 32, 65])
def test_wide_groups_against_an_environment(gpu, world, precision):
    """int_K at its limit (128 on the parity path, 127 on the throughput path) with N near 64, every problem with one of four rows: on
    the parity path two- and four-warp groups and adoption read each problem's own row from its leader's slot"""
    from uneven_planner_b200 import problems, configs
    params = with_row(world["params"])
    params.int_K = 128 if precision == 64 else 127
    cls = _classes(params)
    pb = problems.generate(world["g0"], 48, seed=3, n_max=64, **configs.gen_kwargs("hill"))
    k = np.arange(pb.B) % 4
    env_ctx = ctx(gpu, precision, [c[0] for c in cls], [world["g0"]] * 4)
    by_env = with_params(pb, None)
    by_env.env = k.astype(np.int32)
    want = env_ctx.optimize(by_env)
    env_ctx.close()
    opt = ctx(gpu, precision, params, world["g0"])
    got = opt.optimize(with_params(pb, np.array([cls[q][1] for q in k])))
    opt.close()
    assert same_bytes(got, want)


@pytest.mark.parametrize("precision", [64, 32, 65])
def test_identity_rows_equal_to_the_environment(gpu, world, precision):
    pb = world["bench"]
    same = with_params(pb, rows_of(world["params"], pb.B))
    opt = ctx(gpu, precision, world["params"], world["g0"])
    ref = opt.optimize(pb)
    assert same_bytes(opt.optimize(same), ref)
    assert same_bytes(opt.wait(opt.submit(same, depth=2)), ref)
    opt.upload(same)
    opt.solve_resident(); opt.sync()
    assert same_bytes(opt.download(), ref)
    opt.close()


def _split(a, sizes):
    o = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    return [a[o[i]:o[i + 1]] for i in range(len(sizes))]


@pytest.mark.parametrize("precision", [64, 32, 65])
def test_phase_entry_points(gpu, world, precision):
    params = world["params"]
    pb = world["gold_pb"]
    rows = fleet_rows(pb.B, seed=21)
    opt = ctx(gpu, precision, params, world["g0"])
    S = pb.nsamples(params.int_K)
    x = np.concatenate([pb.x0(i) for i in range(pb.B)])
    opt.upload(with_params(pb, rows))
    ev = opt.eval_batch(x, np.zeros(S.sum()), np.zeros(6 * S.sum()), np.ones(7 * S.sum()), np.ones(pb.B), rho=8.0)
    sfx, scx = opt.init_scaling_batch()
    opt.close()
    om = po.OracleMap(world["g0"])
    tol = TOL.get(precision)
    for i, (g, h, sc) in enumerate(zip(_split(ev["grad"], pb.nvar()), _split(ev["hx"], S), _split(scx, 7 * S))):
        op = po.params_from(with_row(params, rows[i]))
        o = po.eval_one(op, om, pb, i, pb.x0(i), np.zeros(S[i]), np.zeros(6 * S[i]), np.ones(7 * S[i]), 1.0, rho=8.0)
        osfx, oscx = po.init_scaling(op, om, pb, i)
        if precision == 64:
            assert ev["f"][i] == o["f"] and np.array_equal(g, o["grad"]) and np.array_equal(h, o["hx"]), i
            assert sfx[i] == osfx and np.array_equal(sc, oscx), i
        else:
            rel = lambda a, b: np.abs(np.asarray(a) - b).max() / max(np.abs(b).max(), 1.0)
            assert abs(ev["f"][i] - o["f"]) <= tol["f"] * max(abs(o["f"]), 1.0), i
            assert rel(g, o["grad"]) <= tol["grad"] and rel(h, o["hx"]) <= tol["con"], i
            assert abs(sfx[i] - osfx) <= tol["sfx"] * max(abs(osfx), 1.0) and rel(sc, oscx) <= tol["scx"], i


@pytest.mark.parametrize("precision", [64, 32])
def test_tickets(gpu, world, precision):
    params = world["params"]
    pb = world["bench"].select(range(256))
    rows = fleet_rows(pb.B, seed=31)
    rp = with_params(pb, rows)
    opt = ctx(gpu, precision, params, world["g0"])
    ref = opt.optimize(rp)
    # polls return what the wait returns
    t = opt.submit(rp, depth=2)
    out = opt.outputs(rp)
    seen, pend = set(), rp.B
    while pend:
        idx, pend = opt.poll(t, out, 50.0)
        seen.update(int(i) for i in idx)
    assert seen == set(range(rp.B)) and same_bytes(out, ref) and same_bytes(opt.wait(t), ref)
    # cancelling half leaves the other half as it was
    t = opt.submit(rp, depth=2)
    half = np.arange(0, rp.B, 2)
    opt.cancel(t, half)
    got = opt.wait(t)
    assert all(same_problem(rp, got, ref, i) for i in range(1, rp.B, 2))
    assert all(got[0][i].ret_code in (0, 1, 2, STOPPED) for i in half)
    # a budget stops problems
    opt.set_budget(20)
    got = opt.wait(opt.submit(rp, depth=2))
    assert sum(r.ret_code == STOPPED for r in got[0]) > 0
    opt.set_budget(0)
    # urgency changes when the work runs, not its bits
    other = opt.submit(world["bench"], depth=3)
    t = opt.submit(rp, depth=3, urgent=True)
    assert same_bytes(opt.wait(t), ref)
    opt.wait(other)
    opt.close()


def test_multi_context_equals_one(gpu, world):
    params = world["params"]
    pb = world["bench"].select(range(200))
    rp = with_params(pb, fleet_rows(pb.B, seed=41))
    a, b = ctx(gpu, 64, params, world["g0"]), ctx(gpu, 64, params, world["g0"])
    got = gpu.solve_batch_multi([a, b], rp)
    assert same_bytes(got, a.optimize(rp))
    a.close(); b.close()


@pytest.mark.parametrize("precision", [64, 32])
def test_check_and_replan(gpu, world, precision):
    from uneven_planner_b200 import _lib
    params = world["params"]
    pb = world["gold_pb"]
    rows = fleet_rows(pb.B, seed=51)
    rp = with_params(pb, rows)
    opt = ctx(gpu, precision, params, world["g0"])
    out = opt.optimize(rp)
    chk = opt.check_results(rp, out, t_from=0.5)
    pt = np.array([(r.piece_T_xy, r.piece_T_yaw) for r in out[0]])
    for b in range(pb.B):
        one = opt.check_trajectories(pb.N, pb.M, pt, out[1], out[2], t_from=0.5, limits=rows[b, 2:])
        assert chk[b].tobytes() == one[b].tobytes(), b
    lim = _lib.Limits(0.4, 3.0, 5.0, 1.5, 0.85, 0.04)
    assert opt.check_results(rp, out, limits=lim).tobytes() == opt.check_results(pb, out, limits=lim).tobytes()
    # a replan ticket solves its rows with their parameters: the same as submitting the built arrays with them
    sel = np.arange(0, pb.B, 2)
    done = [i for i in sel if out[0][i].total_T > 1.0]
    t, new = opt.submit_replan(rp, out, done, t_from=0.5, depth=2)
    assert np.array_equal(new.params, rows[done])
    got = opt.wait(t)
    assert same_bytes(got, opt.wait(opt.submit(new, depth=2)))
    opt.close()


@pytest.mark.parametrize("precision", [64, 32])
def test_refusals(gpu, world, precision):
    params = world["params"]
    pb = world["gold_pb"]
    opt = ctx(gpu, precision, params, world["g0"])
    ref = opt.optimize(pb)
    for bad in (np.nan, np.inf, -np.inf):
        rows = rows_of(params, pb.B)
        rows[pb.B // 2, 3] = bad
        rp = with_params(pb, rows)
        with pytest.raises(gpu.UalmError, match="error -2"):
            opt.optimize(rp)
        with pytest.raises(gpu.UalmError, match="error -2"):
            opt.submit(rp, depth=1)
        assert not getattr(opt, "_tickets", {})             # no lane taken: a depth-1 submit goes through next
        with pytest.raises(gpu.UalmError, match="error -2"):
            opt.check_results(rp, ref)
        assert same_bytes(opt.wait(opt.submit(pb, depth=1)), ref)
    opt.close()


def test_cpp_adapter_overloads(gpu, bumps_map, tmp_path):
    """the pp overloads of include/ualm_traj_opt.hpp: optimizeBatch, submitBatch with a checkTrajectories while the ticket is in flight,
    waitBatch, submitReplan; every output byte for byte what the C ABI gives through the Python API"""
    from uneven_planner_b200 import _lib, problems
    exe = build_driver("problem_params_driver", tmp_path)
    pb = problems.generate(bumps_map, 8, seed=5)
    rows = fleet_rows(pb.B, seed=61)
    case, got = str(tmp_path / "pp.bin"), str(tmp_path / "pp.out")
    with open(case, "wb") as f:
        f.write(struct.pack("<4i", *bumps_map.shape, pb.B))
        f.write(bumps_map.cells.tobytes())
        for a in (pb.N, pb.M):
            f.write(np.ascontiguousarray(a, np.int32).tobytes())
        for a in (pb.bnd, pb.total_time, rows, pb.inner_xy, pb.inner_yaw):
            f.write(np.ascontiguousarray(a, np.float64).tobytes())
    r = subprocess.run([exe, case, got], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    rp = with_params(pb, rows)
    opt = ctx(gpu, 64, _lib.default_params(), bumps_map)
    a = opt.optimize(rp)
    t = opt.submit(rp, depth=2)
    chk = opt.check_results(rp, a, t_from=0.5)
    b = opt.wait(t)
    t, new = opt.submit_replan(rp, a, np.arange(pb.B), t_from=0.5, depth=2)
    c = opt.wait(t)
    opt.close()
    flat = lambda out: bytes(out[0]) + out[1].tobytes() + out[2].tobytes()
    want = flat(a) + flat(b) + chk.tobytes() + np.ascontiguousarray(new.N, np.int32).tobytes() + \
        np.ascontiguousarray(new.M, np.int32).tobytes() + flat(c)
    with open(got, "rb") as f:
        assert f.read() == want
