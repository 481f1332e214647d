"""The hand-over to the MPC for trajectories the caller holds, each row from its own start state (ualm_mpc_export_trajectories,
BatchALMTrajOpt.mpc_export_trajectories / mpc_export_results, ALMTrajOpt::exportToMpc).

Every row is held bit for bit to the lane form (ualm_mpc_export_batch) on the same records with the same boundary derivatives, and
to the host restatements of tests/workloads.py (message_ref, mpc_ref, dev_ref) with the row's own derivatives, at precisions 64, 65
and 32: at the piece-count edges, per-row start states, replanned rows exported from the robots' states, rows exported from polls of
a batch in flight, the sample-count guard, rows over the limits, diverged records, null outputs and every refusal."""
import ctypes as C
import struct
import subprocess

import numpy as np
import pytest

from harness import build_driver, cat, ctx, gpu, pieces, same_pieces  # noqa: F401
from test_gpu_mpc_export import OUTS, _views, check_export
from uneven_planner_b200 import _lib
from workloads import DEV_GUARD, INIT_A, INIT_V, dev_ref, message_ref, mpc_ref, orc, scan_length  # noqa: F401

pytestmark = pytest.mark.gpu
dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int32)
PRECISIONS = [64, 65, 32]


def _same(a, b):
    """two hand-over dicts, or two rows of them (_views), equal as bytes in every output"""
    return all(np.ascontiguousarray(a[k]).tobytes() == np.ascontiguousarray(b[k]).tobytes() for k in OUTS)


def _held_rows(pb, rows, ex):
    """row j of a held export of rows `rows` of pb, for every j: _views of the selected batch"""
    sub = pb.select(rows)
    return [_views(sub, ex, j) for j in range(len(rows))]


def _check_rows(orc, pb, out, rows, ex, dt, init_v, init_a):
    """every output of the held export `ex` of rows `rows` against the references with row j's own init_v[j] / init_a[j]; a record
    over the compiled limits is all zeros"""
    res, cxy, cyaw = out
    _, _, ocx, ocy = pb.offsets()
    for j, (i, got) in enumerate(zip(rows, _held_rows(pb, rows, ex))):
        if res[i].ret_code == _lib.UALM_ELIMIT:
            assert all(not np.asarray(got[k]).any() for k in OUTS), i
            continue
        N, M, Tx, Ty = int(pb.N[i]), int(pb.M[i]), res[i].piece_T_xy, res[i].piece_T_yaw
        c1, c2 = cxy[ocx[i]:ocx[i + 1]], cyaw[ocy[i]:ocy[i + 1]]
        msg = message_ref(c1, c2, N, M, Tx, Ty)
        mx, my = mpc_ref(orc, msg, Tx, Ty, init_v[j], init_a[j])
        want = dict(msg, c_mpc_xy=mx, c_mpc_yaw=my, dev=dev_ref(c1, c2, mx, my, N, M, Tx, Ty, dt))
        for k in OUTS:
            assert np.array_equal(got[k], want[k]), (j, i, k)


@pytest.fixture(scope="module")
def edge_batches(built, bumps_map):
    """test_gpu_mpc_export's edge batches (N 1 and 64, M 1 and 128, T < 1 s, partly filled CTAs, B = 1), the first with a problem
    over the compiled limits inserted"""
    from uneven_planner_b200 import problems
    from workloads import _with_oversize, case_batch
    gen = problems.generate(bumps_map, 8, seed=12)
    cases = case_batch()
    return [_with_oversize(cat([cases, gen.select([0])]), 3), gen.select(range(1, 8)), cases.select([cases.B - 1])]


@pytest.fixture(scope="module")
def solved(gpu, edge_batches, bumps_map):
    cache = {}

    def get(prec):
        if prec not in cache:
            runs = []
            for pb in edge_batches:
                opt = ctx(gpu, prec, _lib.default_params(), bumps_map)
                runs.append((pb, opt, opt.optimize(pb)))
            cache[prec] = runs
        return cache[prec]
    yield get
    for runs in cache.values():
        for _, opt, _ in runs:
            opt.close()


# ------------------------------------------------------------------ 1. the lane form's bits
@pytest.mark.parametrize("prec", PRECISIONS)
def test_same_as_the_lane_form(gpu, orc, solved, prec):
    """whole batches through both forms, with zero and with INIT_V / INIT_A on every row: every output byte-identical, and equal to the
    references"""
    runs = solved(prec)
    big = runs[0][0]
    assert {1, 64}.issubset(set(big.N.tolist())) and {1, 128}.issubset(set(big.M.tolist())) and runs[2][0].B == 1
    assert runs[0][2][0][3].ret_code == _lib.UALM_ELIMIT
    for pb, opt, out in runs:
        for v, a in ((None, None), (INIT_V, INIT_A)):
            lane = opt.mpc_export(pb.N, pb.M, init_v=v, init_a=a)
            held = opt.mpc_export_trajectories(pb.N, pb.M, _piece_T(out[0]), out[1], out[2], init_v=v, init_a=a)
            assert _same(lane, held), (pb.B, v)
            assert check_export(orc, pb, out, held, 0.01, v, a) == sum(r.ret_code != _lib.UALM_ELIMIT for r in out[0])
        assert _same(opt.mpc_export(pb.N, pb.M), opt.mpc_export_results(pb, out))


def _piece_T(res):
    return np.array([(r.piece_T_xy, r.piece_T_yaw) for r in res], np.float64).reshape(len(res), 2)


# ------------------------------------------------------------------ 2. each row its own start state
@pytest.mark.parametrize("prec", PRECISIONS)
def test_per_row_start_states(gpu, orc, solved, prec):
    """zeros, a single nonzero component of each kind, large values and seeded ones, one triple per row: every row equals the references
    with its own triple, and the head of each re-solve carries it exactly (measured error 0: rows 1 and 2 of the band are never
    eliminated, so c1 = init_v and c2 = init_a / 2, a division by two, bit for bit)"""
    pb, opt, out = solved(prec)[1]
    B = pb.B
    rng = np.random.default_rng(3)
    v, a = rng.uniform(-2.0, 2.0, (B, 3)), rng.uniform(-3.0, 3.0, (B, 3))
    v[0] = a[0] = 0.0
    v[1] = (0.0, 0.9, 0.0); a[1] = 0.0
    v[2] = 0.0; a[2] = (0.0, 0.0, -1.7)
    v[3] = (1.0e3, -2.5e3, 4.0e2); a[3] = (-7.0e4, 3.0e4, 1.0e5)
    rows = np.arange(B)
    ex = opt.mpc_export_trajectories(pb.N, pb.M, _piece_T(out[0]), out[1], out[2], init_v=v, init_a=a)
    _check_rows(orc, pb, out, rows, ex, 0.01, v, a)
    for j, got in enumerate(_held_rows(pb, rows, ex)):
        N = int(pb.N[j])
        mx, my = got["c_mpc_xy"], got["c_mpc_yaw"]
        assert (mx[1], mx[6 * N + 1], my[1]) == tuple(v[j]), j
        assert (mx[2], mx[6 * N + 2], my[2]) == tuple(a[j] / 2), j
        lane = _views(pb, opt.mpc_export(pb.N, pb.M, init_v=v[j], init_a=a[j]), j) if j < 4 else None
        assert lane is None or _same(lane, got), j


# ------------------------------------------------------------------ 3. replanned robots
@pytest.mark.parametrize("prec", PRECISIONS)
def test_replanned_rows_from_their_own_states(gpu, orc, bumps_map, prec):
    """rows 0, 3 and 5 replanned at t = 0.5, exported with start="bnd": each row matches the references with its own state.  The lane
    form can carry only one state for the whole call: with row 0's, rows 3 and 5 differ from their own messages' re-solve"""
    from uneven_planner_b200 import problems
    pb = problems.generate(bumps_map, 40, seed=77).select(range(8))
    opt = ctx(gpu, prec, _lib.default_params(), bumps_map)
    out = opt.optimize(pb)
    t, new = opt.submit_replan(pb, out, [0, 3, 5], 0.5)
    got = opt.wait(t)
    v, a = new.bnd[:, [2, 3, 13]], new.bnd[:, [4, 5, 14]]
    assert all(np.any(x != 0.0) for x in v) and all(np.any(x != 0.0) for x in a)
    held = opt.mpc_export_results(new, got, start="bnd")
    _check_rows(orc, new, got, np.arange(new.B), held, 0.01, v, a)
    rest = opt.mpc_export_results(new, got)
    _check_rows(orc, new, got, np.arange(new.B), rest, 0.01, [None] * new.B, [None] * new.B)
    opt.select_lane(t)
    lane = opt.mpc_export(new.N, new.M, init_v=v[0], init_a=a[0])
    opt.close()
    assert _same(_views(new, lane, 0), _views(new, held, 0))
    for j in (1, 2):
        assert not np.array_equal(_views(new, lane, j)["c_mpc_xy"], _views(new, held, j)["c_mpc_xy"]), j


# ------------------------------------------------------------------ 4. in flight
@pytest.fixture(scope="module")
def bench_world(built):
    from uneven_planner_b200 import configs, maps, problems
    g0 = maps.stand_in_terrain("hill")
    return dict(g0=g0, params=configs.params_for("hill"), bench=problems.generate(g0, 1024, seed=0, **configs.gen_kwargs("hill")))


@pytest.mark.parametrize("prec", PRECISIONS)
def test_export_of_polled_rows_while_the_batch_runs(gpu, bench_world, prec):
    """the 1024-problem bench batch polled, each poll's new rows exported at once (urgent on the parity path, whose solve otherwise
    keeps the SMs until its queue runs dry): some export returns while problems are still pending; after wait the lane form's rows are
    byte-identical to the held exports; the batch's records are byte-identical to a lone solve"""
    pb = bench_world["bench"]
    opt = ctx(gpu, prec, bench_world["params"], bench_world["g0"])
    t = opt.submit(pb, depth=2)
    out = opt.outputs(pb)
    exports, in_flight, n_pend = [], 0, pb.B
    while n_pend:
        new, n_pend = opt.poll(t, out, wait_ms=2.0)
        if new.size:
            ex = opt.mpc_export_results(pb, out, rows=new, urgent=prec == 64)
            exports.append((new, ex))
            new2, n_pend2 = opt.poll(t, out, 0.0)      # after the export has returned: problems still running
            in_flight += n_pend2 > 0
            if new2.size:
                exports.append((new2, opt.mpc_export_results(pb, out, rows=new2, urgent=prec == 64)))
            n_pend = n_pend2
    done = opt.wait(t)
    opt.select_lane(t)
    lane = opt.mpc_export(pb.N, pb.M)
    opt.close()
    assert in_flight > 0
    seen = np.concatenate([r for r, _ in exports])
    assert np.array_equal(np.sort(seen), np.arange(pb.B))
    for rows, ex in exports:
        for i, got in zip(rows, _held_rows(pb, rows, ex)):
            assert _same(_views(pb, lane, int(i)), got), int(i)
    o = ctx(gpu, prec, bench_world["params"], bench_world["g0"])
    alone = pieces(pb, o.optimize(pb))
    o.close()
    assert same_pieces(pieces(pb, done), alone)


# ------------------------------------------------------------------ 5. edges
@pytest.mark.parametrize("prec", PRECISIONS)
def test_row_order_dt_and_the_guard(gpu, orc, solved, prec):
    """rows in arbitrary order with a duplicate, at dt = 0.01, 0.0137, past every trajectory, and at a dt that puts some rows just
    under the 4e6-sample guard and the rest over it: each row byte-identical to the lane form's row with the same dt and init"""
    pb, opt, out = solved(prec)[0]
    res = out[0]
    short = min(scan_length(int(pb.N[i]), int(pb.M[i]), res[i].piece_T_xy, res[i].piece_T_yaw, 1.0) for i in range(pb.B)
                if res[i].ret_code != _lib.UALM_ELIMIT)
    rows = [pb.B - 1, 0, 3, 5, 5, 1, 2]
    for dt in (0.01, 0.0137, 1.0e4, short / (DEV_GUARD - 0.5)):
        lane = opt.mpc_export(pb.N, pb.M, dt=dt, init_v=INIT_V, init_a=INIT_A)
        sub = pb.select(rows)
        N, M = sub.N, sub.M
        _, _, ocx, ocy = pb.offsets()
        cxy = np.concatenate([out[1][ocx[i]:ocx[i + 1]] for i in rows])
        cyaw = np.concatenate([out[2][ocy[i]:ocy[i + 1]] for i in rows])
        held = opt.mpc_export_trajectories(N, M, _piece_T([res[i] for i in rows]), cxy, cyaw, init_v=INIT_V, init_a=INIT_A, dt=dt)
        for j, got in enumerate(_held_rows(pb, rows, held)):
            assert _same(_views(pb, lane, rows[j]), got), (dt, j)
        if dt == 1.0e4:
            assert not held["dev"].any()
        if dt < 1.0e-3:
            over = held["dev"][:, 0] == -1.0
            assert over.any() and not over.all()


@pytest.mark.parametrize("prec", PRECISIONS)
def test_over_the_limits_and_diverged_rows(gpu, solved, prec):
    """a row over the compiled limits is zeros whatever its durations; a record with infinite durations gets its message and
    {-1, 0, -1, 0}"""
    pb, opt, out = solved(prec)[0]
    res, cxy, cyaw = out
    _, _, ocx, ocy = pb.offsets()
    i = 4
    pt = _piece_T(res)
    pt[3] = (0.0, float("nan"))            # the row over the limits (UALM_ELIMIT): its durations are not looked at
    pt[i] = (float("inf"), float("inf"))
    ex = opt.mpc_export_trajectories(pb.N, pb.M, pt, cxy, cyaw, init_v=INIT_V, init_a=INIT_A)
    assert all(not np.asarray(_views(pb, ex, 3)[k]).any() for k in OUTS)
    got = _views(pb, ex, i)
    N = int(pb.N[i])
    assert np.array_equal(got["dev"], [-1.0, 0.0, -1.0, 0.0])
    assert np.array_equal(got["pos_pts"][:N, 0], cxy[ocx[i]:ocx[i] + 6 * N:6]) and np.isinf(got["posT_pts"]).all()
    assert np.array_equal(got["angle_pts"][:-1], cyaw[ocy[i]:ocy[i + 1]:6])
    lane = opt.mpc_export(pb.N, pb.M, init_v=INIT_V, init_a=INIT_A)
    for j in range(pb.B):
        if j not in (3, i):
            assert _same(_views(pb, lane, j), _views(pb, ex, j)), j


@pytest.mark.parametrize("prec", PRECISIONS)
def test_any_output_may_be_null(gpu, solved, prec):
    pb, opt, out = solved(prec)[1]
    N, M = np.ascontiguousarray(pb.N, np.int32), np.ascontiguousarray(pb.M, np.int32)
    pt = _piece_T(out[0])
    v = np.ascontiguousarray(np.tile(INIT_V, (pb.B, 1)))
    a = np.ascontiguousarray(np.tile(INIT_A, (pb.B, 1)))
    full = opt.mpc_export_trajectories(N, M, pt, out[1], out[2], init_v=v, init_a=a)
    P = lambda x, t=dp: x.ctypes.data_as(t)
    for skip in range(len(OUTS)):
        bufs = [np.full(full[k].size, 7.0) for k in OUTS]
        rc = opt.L.ualm_mpc_export_trajectories(opt.h, pb.B, P(N, ip), P(M, ip), P(pt), P(out[1]), P(out[2]), P(v), P(a), 0.01,
                                                *[None if j == skip else P(b) for j, b in enumerate(bufs)])
        assert rc == 0
        for j, k in enumerate(OUTS):
            assert (bufs[j] == 7.0).all() if j == skip else np.array_equal(bufs[j], full[k].ravel()), (skip, k)


# ------------------------------------------------------------------ 6. refusals
@pytest.mark.parametrize("prec", PRECISIONS)
def test_refusals_write_nothing(gpu, solved, prec):
    pb, opt, out = solved(prec)[1]
    L = opt.L
    N, M = np.ascontiguousarray(pb.N, np.int32), np.ascontiguousarray(pb.M, np.int32)
    pt = _piece_T(out[0])
    cxy, cyaw = out[1], out[2]
    v = np.zeros((pb.B, 3)); a = np.zeros((pb.B, 3))
    P = lambda x, t=dp: None if x is None else x.ctypes.data_as(t)
    sN, sM = int(pb.N.sum()), int(pb.M.sum())

    def call(h=opt.h, B=pb.B, N=N, M=M, pt=pt, cxy=cxy, cyaw=cyaw, v=v, a=a, dt=0.01):
        bufs = [np.full(n, 7.0) for n in (2 * (sN + pb.B), sN, sM + pb.B, sM, 12 * sN, 6 * sM, 4 * pb.B)]
        rc = L.ualm_mpc_export_trajectories(h, B, P(N, ip), P(M, ip), P(pt), P(cxy), P(cyaw), P(v), P(a), C.c_double(dt), *[P(b) for b in bufs])
        return rc, all((b == 7.0).all() for b in bufs)

    def with_(arr, idx, val):
        x = arr.copy()
        x[idx] = val
        return x
    nan, inf = float("nan"), float("inf")
    cases = dict(null_ctx=dict(h=None), null_N=dict(N=None), null_M=dict(M=None), null_pt=dict(pt=None), null_cxy=dict(cxy=None),
                 null_cyaw=dict(cyaw=None), negative_B=dict(B=-1), dt_zero=dict(dt=0.0), dt_negative=dict(dt=-0.01), dt_nan=dict(dt=nan),
                 N_zero=dict(N=with_(N, 2, 0)), M_zero=dict(M=with_(M, 1, 0)), v_nan=dict(v=with_(v, (1, 2), nan)),
                 a_inf=dict(a=with_(a, (0, 0), inf)), v_minus_inf=dict(v=with_(v, (pb.B - 1, 1), -inf)),
                 pt_nan=dict(pt=with_(pt, (2, 0), nan)), pt_zero=dict(pt=with_(pt, (1, 1), 0.0)), pt_negative=dict(pt=with_(pt, (0, 0), -1.0)),
                 pt_minus_inf=dict(pt=with_(pt, (3, 1), -inf)), unfilled=dict(pt=with_(pt, 4, 0.0)))
    for name, kw in cases.items():
        rc, untouched = call(**kw)
        assert rc == _lib.UALM_EINVAL, name
        assert untouched, name
    rc, untouched = call(B=0, N=None, M=None, pt=None, cxy=None, cyaw=None)
    assert rc == _lib.UALM_OK and untouched
    rc, untouched = call()
    assert rc == _lib.UALM_OK and not untouched
    with pytest.raises(gpu.UalmError):
        opt.mpc_export_results(pb, (opt.outputs(pb)[0], cxy, cyaw))       # records poll() has not filled: zero durations
    with pytest.raises(ValueError):
        opt.mpc_export_trajectories(pb.N, pb.M, pt, cxy, cyaw, init_v=np.zeros((pb.B, 2)))
    with pytest.raises(ValueError):
        opt.mpc_export_results(pb, out, start="moving")


# ------------------------------------------------------------------ 7. C++
def test_cpp_export_between_submits(gpu, tmp_path):
    """ALMTrajOpt::exportToMpc on waitBatch results, per-row start states, while the next batch is in flight: the printed arrays equal
    mpc_export_trajectories on the Python solve's records (parity path, so the records agree bit for bit)"""
    from uneven_planner_b200 import maps, problems
    exe = build_driver("mpc_held_driver", tmp_path)
    g0 = maps.stand_in_terrain("hill")
    pb = problems.generate(g0, 8, seed=21)
    rng = np.random.default_rng(5)
    v, a = rng.uniform(-1.0, 1.0, (pb.B, 3)), rng.uniform(-1.0, 1.0, (pb.B, 3))
    case = str(tmp_path / "mpc.bin")
    with open(case, "wb") as f:
        f.write(struct.pack("<4i", *g0.shape, pb.B))
        f.write(np.ascontiguousarray(g0.cells, np.float32).tobytes())
        for x in (pb.N, pb.M):
            f.write(np.ascontiguousarray(x, np.int32).tobytes())
        for x in (pb.bnd, pb.total_time, pb.inner_xy, pb.inner_yaw, v, a):
            f.write(np.ascontiguousarray(x, np.float64).tobytes())
    r = subprocess.run([exe, case], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    opt = gpu.BatchALMTrajOpt().init(_lib.default_params()).set_environment(g0)
    out = opt.wait(opt.submit(pb, depth=3))
    t2 = opt.submit(pb, depth=3)
    ex = opt.mpc_export_trajectories(pb.N, pb.M, _piece_T(out[0]), out[1], out[2], init_v=v, init_a=a)
    opt.wait(t2)
    opt.close()
    lines = r.stdout.strip().splitlines()
    assert [ln.split()[0] for ln in lines] == list(OUTS)
    for ln, k in zip(lines, OUTS):
        got = np.array([float(x) for x in ln.split()[1:]])
        assert got.tobytes() == np.ascontiguousarray(ex[k], np.float64).ravel().tobytes(), k
