"""SURVEY 8f-3 on the GPU: the SE2Traj message, the MPC side's MINCO re-solve and the planned-vs-tracked deviation of a solved batch
(ualm_mpc_export_batch, csrc/ualm_kernels.cuh: mpc_export_kernel).

Parity chain: the MPC's own header (mpc_controller/include/utils/minco_traj.hpp:365-444, compiled unmodified) equals orc_minco_generate bit
for bit on such messages (tests/test_ref_pin.py::test_mpc_side_minco_resolve_matches_oracle_bitwise, CPU); here the CUDA kernel equals
orc_minco_generate bit for bit on the messages of solved batches, so the trajectory the MPC tracks behind this back-end is the one it tracks
behind the reference's.  The message itself is compared with the values the reference's publish loop reads off getTraj()
(plan_manager.cpp:159-184): constant coefficients and PolyTrajectory::getValue(total).

Beyond that, every output of every problem is held bit for bit to the host restatements of tests/test_mpc_handover.py (message_ref,
mpc_ref, dev_ref) on the records the solve returned, at precisions 64, 65 and 32: at the piece-count edges and partly filled CTAs,
at nonzero boundary derivatives, at several dt and at the 4e6-sample guard, at tied maxima of both deviations, and after every way a
batch ends (another lane, a budget, a deadline, a cancel, a replan, a problem over the limits)."""
import ctypes as C

import numpy as np
import pytest

from harness import cat, ctx, gpu  # noqa: F401
from uneven_planner_b200 import _lib
from workloads import DEV_GUARD, INIT_A, INIT_V, dev_ref, deviation_samples, message_ref, mpc_ref, scan_length


pytestmark = pytest.mark.gpu
dp = C.POINTER(C.c_double)
P = lambda a: a.ctypes.data_as(dp)
PRECISIONS = [64, 65, 32]
OUTS = ("pos_pts", "posT_pts", "angle_pts", "angleT_pts", "c_mpc_xy", "c_mpc_yaw", "dev")


@pytest.fixture(scope="module")
def orc(built):
    import pyoracle as po
    L = po.lib()
    L.orc_minco_generate.argtypes = [C.c_int, C.c_int, dp, dp, dp, dp, dp]
    return L


def _views(pb, ex, i):
    """problem i's slices of the export's packed outputs"""
    N, M = int(pb.N[i]), int(pb.M[i])
    sN = int(pb.N[:i].astype(np.int64).sum()); sM = int(pb.M[:i].astype(np.int64).sum())
    return dict(pos_pts=ex["pos_pts"][2 * (sN + i):2 * (sN + N + i + 1)].reshape(N + 1, 2), posT_pts=ex["posT_pts"][sN:sN + N],
                angle_pts=ex["angle_pts"][sM + i:sM + M + i + 1], angleT_pts=ex["angleT_pts"][sM:sM + M],
                c_mpc_xy=ex["c_mpc_xy"][12 * sN:12 * (sN + N)], c_mpc_yaw=ex["c_mpc_yaw"][6 * sM:6 * (sM + M)], dev=ex["dev"][i])


def check_export(orc, pb, out, ex, dt, init_v=None, init_a=None):
    """every output of every problem bit for bit against the references on the records out = (results, c_xy, c_yaw); a problem over
    the compiled limits (UALM_ELIMIT) has all-zero rows.  Returns the number of problems compared with the references."""
    from uneven_planner_b200 import _lib
    res, cxy, cyaw = out
    _, _, ocx, ocy = pb.offsets()
    n = 0
    for i in range(pb.B):
        N, M = int(pb.N[i]), int(pb.M[i])
        got = _views(pb, ex, i)
        if res[i].ret_code == _lib.UALM_ELIMIT:
            assert all(not np.asarray(got[k]).any() for k in OUTS), i
            continue
        Tx, Ty = res[i].piece_T_xy, res[i].piece_T_yaw
        c1, c2 = cxy[ocx[i]:ocx[i + 1]], cyaw[ocy[i]:ocy[i + 1]]
        msg = message_ref(c1, c2, N, M, Tx, Ty)
        mx, my = mpc_ref(orc, msg, Tx, Ty, init_v, init_a)
        want = dict(msg, c_mpc_xy=mx, c_mpc_yaw=my, dev=dev_ref(c1, c2, mx, my, N, M, Tx, Ty, dt))
        for k in OUTS:
            assert np.array_equal(got[k], want[k]), (i, k, N, M, got[k], want[k]) if k == "dev" else (i, k, N, M)
        n += 1
    return n


def _export(gpu, opt, pb, out, orc, dt=0.01, init_v=None, init_a=None):
    ex = opt.mpc_export(pb.N, pb.M, dt=dt, init_v=init_v, init_a=init_a)
    assert check_export(orc, pb, out, ex, dt, init_v, init_a) > 0
    return ex


# ------------------------------------------------------------------ the solved batch of the original test
@pytest.mark.parametrize("prec", [64, 32])
def test_message_and_mpc_resolve_of_a_solved_batch(gpu, orc, bumps_map, prec):
    from uneven_planner_b200 import problems
    pb = problems.generate(bumps_map, 24, seed=12)
    opt = ctx(gpu, prec, _lib.default_params(), bumps_map)
    out = opt.optimize(pb)
    ex = opt.mpc_export(pb.N, pb.M, dt=0.01)
    opt.close()
    assert check_export(orc, pb, out, ex, 0.01) == pb.B
    _, _, ocx, _ = pb.offsets()
    for i in range(pb.B):
        # the tracked spline interpolates the same waypoints: the difference comes from the boundary derivatives alone and stays small
        N = int(pb.N[i])
        assert np.allclose(ex["c_mpc_xy"][ocx[i]:ocx[i] + 6 * N:6], out[1][ocx[i]:ocx[i] + 6 * N:6], atol=1e-9)
    assert ex["dev"][:, 0].max() < 0.05     # metres; measured ~ mm: 0.05 m/s of boundary speed (plan_manager.cpp:93-94) against none


def test_export_needs_a_solved_batch_and_skips_oversize_problems(gpu, bumps_map):
    from uneven_planner_b200 import _lib, problems
    from workloads import _with_oversize
    params = _lib.default_params()
    pb = problems.generate(bumps_map, 6, seed=5)
    opt = gpu.BatchALMTrajOpt().init(params).set_environment(bumps_map)
    with pytest.raises(gpu.UalmError):
        opt.mpc_export(pb.N, pb.M)
    pbx = _with_oversize(pb, 2)
    res, cxy, cyaw = opt.optimize(pbx)
    ex = opt.mpc_export(pbx.N, pbx.M)
    opt.close()
    assert res[2].ret_code == _lib.UALM_ELIMIT
    sN = np.concatenate([[0], np.cumsum(pbx.N)])
    assert not ex["pos_pts"][2 * (sN[2] + 2):2 * (sN[3] + 3)].any() and not ex["dev"][2].any()
    assert ex["pos_pts"][2 * (sN[3] + 3)] == cxy[pbx.offsets()[2][3]]


# ------------------------------------------------------------------ shapes, boundary derivatives, dt, the guard
@pytest.fixture(scope="module")
def edge_batches(built, bumps_map):
    """the edge cases of test_gpu_tp_shapes (N1_M1, N1_M128, N64_M128, N40_M3, T < 1 s, yaw seam, off the map, ...) with one generated
    problem after them (B % 4 == 1: a partly filled last CTA), seven generated problems (B % 4 == 3) and one problem alone"""
    from workloads import case_batch
    from uneven_planner_b200 import problems
    gen = problems.generate(bumps_map, 8, seed=12)
    cases = case_batch()
    return [cat([cases, gen.select([0])]), gen.select(range(1, 8)), cases.select([cases.B - 1])]


@pytest.fixture(scope="module")
def solved_edges(gpu, edge_batches, bumps_map):
    """edge_batches solved per precision: one context per (precision, batch) kept open, on its batch's lane 0"""
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


@pytest.mark.parametrize("prec", PRECISIONS)
def test_edge_shapes_against_references(gpu, orc, solved_edges, prec):
    runs = solved_edges(prec)
    assert [pb.B % 4 for pb, _, _ in runs] == [1, 3, 1] and runs[2][0].B == 1
    big = runs[0][0]
    assert {1, 64}.issubset(set(big.N.tolist())) and {1, 128}.issubset(set(big.M.tolist()))
    for pb, opt, out in runs:
        _export(gpu, opt, pb, out, orc)


@pytest.mark.parametrize("prec", PRECISIONS)
def test_boundary_derivatives(gpu, orc, solved_edges, prec):
    """init_v / init_a = {x, y, yaw}, all six values distinct; each alone; NULL is zero bit for bit.  Without the oracle: rows 1 and 2 of
    the band are never eliminated, so the tracked spline's first piece carries init_v and init_a / 2 exactly"""
    pb, opt, out = solved_edges(prec)[0]
    zeros = _export(gpu, opt, pb, out, orc, init_v=np.zeros(3), init_a=np.zeros(3))
    none = opt.mpc_export(pb.N, pb.M)
    assert all(np.array_equal(zeros[k], none[k]) for k in OUTS)
    both = _export(gpu, opt, pb, out, orc, init_v=INIT_V, init_a=INIT_A)
    v_only = _export(gpu, opt, pb, out, orc, init_v=INIT_V)
    a_only = _export(gpu, opt, pb, out, orc, init_a=INIT_A)
    _, _, ocx, ocy = pb.offsets()
    for ex, v, a in ((both, INIT_V, INIT_A), (v_only, INIT_V, (0.0, 0.0, 0.0)), (a_only, (0.0, 0.0, 0.0), INIT_A)):
        for i in range(pb.B):
            N = int(pb.N[i])
            mx, my = ex["c_mpc_xy"][ocx[i]:ocx[i + 1]], ex["c_mpc_yaw"][ocy[i]:ocy[i + 1]]
            assert (mx[1], mx[6 * N + 1], my[1]) == tuple(v), i
            assert (mx[2], mx[6 * N + 2], my[2]) == tuple(x / 2 for x in a), i


@pytest.mark.parametrize("prec", PRECISIONS)
def test_sample_spacing(gpu, orc, solved_edges, prec):
    """a dt that divides no duration; a dt past every trajectory keeps the one sample t = 0, where both splines start at the same point
    and angle (dev = 0); dt = 0, negative or NaN is UALM_EINVAL and writes no output"""
    from uneven_planner_b200 import _lib
    for pb, opt, out in solved_edges(prec)[:2]:
        _export(gpu, opt, pb, out, orc, dt=0.0137, init_v=INIT_V, init_a=INIT_A)
        far = _export(gpu, opt, pb, out, orc, dt=1.0e4)
        assert not far["dev"].any()
    pb, opt, out = solved_edges(prec)[1]
    sN, sM = int(pb.N.sum()), int(pb.M.sum())
    for dt in (0.0, -0.01, float("nan")):
        bufs = [np.full(n, 7.0) for n in (2 * (sN + pb.B), sN, sM + pb.B, sM, 12 * sN, 6 * sM, 4 * pb.B)]
        rc = opt.L.ualm_mpc_export_batch(opt.h, C.c_double(dt), None, None, *[P(b) for b in bufs])
        assert rc == _lib.UALM_EINVAL, dt
        assert all((b == 7.0).all() for b in bufs), dt


@pytest.mark.parametrize("prec", PRECISIONS)
def test_sample_count_guard(gpu, orc, solved_edges, prec):
    """a dt that puts the shortest trajectories of the edge batch (T < 1 s) just under 4e6 samples and every other one over: those are
    scanned in full; the others get {-1, 0, -1, 0} and still their message and re-solve"""
    pb, opt, out = solved_edges(prec)[0]
    res = out[0]
    rows = [(i, int(pb.N[i]), int(pb.M[i]), res[i].piece_T_xy, res[i].piece_T_yaw) for i in range(pb.B)]
    short = min(scan_length(N, M, Tx, Ty, 1.0) for _, N, M, Tx, Ty in rows)
    dt = short / (DEV_GUARD - 0.5)
    n = np.array([scan_length(N, M, Tx, Ty, dt) for _, N, M, Tx, Ty in rows])
    assert (n < DEV_GUARD).any() and (n >= DEV_GUARD).any() and n[n < DEV_GUARD].min() > 0.999999 * DEV_GUARD
    ex = _export(gpu, opt, pb, out, orc, dt=dt)
    assert np.array_equal(ex["dev"][n >= DEV_GUARD], np.tile([-1.0, 0.0, -1.0, 0.0], ((n >= DEV_GUARD).sum(), 1)))
    assert (ex["dev"][n < DEV_GUARD, 1] > 0.0).all()


def tie_kinds(pb, out, orc, dt):
    """which kinds of tied maxima the scans of batch `pb` (records out) reach at dt: ("pos" | "yaw", "lane" | "lanes") where some
    problem's largest deviation, > 0, is reached by two samples of one lane ("lane") or by samples of two lanes ("lanes").  A lane scans
    the samples k, k + 32, .. of its index k.  A deviation that is 0 throughout is no tie: every lane keeps (0, 0) whatever the rule."""
    res, cxy, cyaw = out
    _, _, ocx, ocy = pb.offsets()
    seen = set()
    for i in range(pb.B):
        N, M, Tx, Ty = int(pb.N[i]), int(pb.M[i]), res[i].piece_T_xy, res[i].piece_T_yaw
        c1, c2 = cxy[ocx[i]:ocx[i + 1]], cyaw[ocy[i]:ocy[i + 1]]
        mx, my = mpc_ref(orc, message_ref(c1, c2, N, M, Tx, Ty), Tx, Ty)
        _, ep, ey = deviation_samples(c1, c2, mx, my, N, M, Tx, Ty, dt)
        for name, v in (("pos", ep), ("yaw", ey)):
            if not v.max() > 0.0:
                continue
            k = np.nonzero(v == v.max())[0]
            lanes = set((k % 32).tolist())
            if len(lanes) > 1:
                seen.add((name, "lanes"))
            if len(lanes) < k.size:
                seen.add((name, "lane"))
    return seen


@pytest.mark.parametrize("prec", PRECISIONS)
def test_tied_maxima_keep_the_earliest_sample(gpu, orc, bumps_map, prec):
    """problems planned with zero boundary velocity and acceleration (xy and yaw): the planned splines solve the same MINCO conditions
    as the MPC's re-solve, so both deviations sit at the rounding level and their largest values repeat.  Every dev4 row at dt = 0.01
    and 0.005, times included, is dev_ref's: the largest value at its earliest sample, within a lane and across lanes.  On the parity
    path, whose planned splines are the oracle's MINCO bit for bit, some problem's largest position deviation and some problem's largest
    yaw deviation are each reached twice within one lane and in two lanes, so both tie rules are exercised for both quantities.  The
    throughput path builds its planned splines from its own MINCO tables with FMA contraction: they differ from the re-solve by more
    than a few ulps there, and only some kinds of tie occur (its rows are still compared bit for bit)."""
    from uneven_planner_b200 import problems
    pb = problems.generate(bumps_map, 16, seed=1)
    pb.bnd[:, [2, 3, 4, 5, 8, 9, 10, 11, 13, 14, 16, 17]] = 0.0
    opt = ctx(gpu, prec, _lib.default_params(), bumps_map)
    out = opt.optimize(pb)
    seen = set()
    for dt in (0.01, 0.005):
        _export(gpu, opt, pb, out, orc, dt=dt)
        seen |= tie_kinds(pb, out, orc, dt)
    opt.close()
    if prec == 64:
        assert seen == {(a, b) for a in ("pos", "yaw") for b in ("lane", "lanes")}, seen


# ------------------------------------------------------------------ how the batch ended
@pytest.fixture(scope="module")
def small(built, bumps_map):
    from uneven_planner_b200 import problems
    return problems.generate(bumps_map, 40, seed=77)


@pytest.mark.parametrize("prec", PRECISIONS)
def test_export_reads_the_selected_lane(gpu, orc, bumps_map, small, prec):
    """two tickets on lanes 0 and 1: each lane exports its own batch"""
    a, b = small.select(range(0, 13)), small.select(range(13, 40))
    opt = ctx(gpu, prec, _lib.default_params(), bumps_map)
    ta, tb = opt.submit(a, depth=2), opt.submit(b, depth=2)
    assert (ta, tb) == (0, 1)
    oa, ob = opt.wait(ta), opt.wait(tb)
    opt.select_lane(1)
    _export(gpu, opt, b, ob, orc, init_v=INIT_V, init_a=INIT_A)
    opt.select_lane(0)
    _export(gpu, opt, a, oa, orc, init_v=INIT_V, init_a=INIT_A)
    opt.close()


@pytest.mark.parametrize("prec", PRECISIONS)
def test_export_after_a_budget(gpu, orc, bumps_map, small, prec):
    from uneven_planner_b200 import _lib
    opt = ctx(gpu, prec, _lib.default_params(), bumps_map).set_budget(3)
    out = opt.optimize(small)
    assert sum(r.ret_code == _lib.UALM_RET_STOPPED for r in out[0]) > small.B // 2
    _export(gpu, opt, small, out, orc, init_v=INIT_V, init_a=INIT_A)
    opt.close()


@pytest.mark.parametrize("prec", PRECISIONS)
def test_export_after_a_deadline_and_a_cancel(gpu, orc, bumps_map, small, prec):
    from uneven_planner_b200 import _lib
    opt = ctx(gpu, prec, _lib.default_params(), bumps_map)
    out = opt.wait(opt.submit(small, depth=1), timeout_ms=0)
    assert any(r.ret_code == _lib.UALM_RET_STOPPED for r in out[0])
    _export(gpu, opt, small, out, orc, dt=0.0137)
    t = opt.submit(small, depth=1)
    opt.cancel(t, [1, 4, 6, 39])
    out = opt.wait(t)
    assert any(out[0][i].ret_code == _lib.UALM_RET_STOPPED for i in (1, 4, 6, 39))
    _export(gpu, opt, small, out, orc, init_v=INIT_V, init_a=INIT_A)
    opt.close()


@pytest.mark.parametrize("prec", PRECISIONS)
def test_export_of_a_replan(gpu, orc, bumps_map, small, prec):
    """a replan ticket, exported on its lane with the robot's state at the replan time as the message's boundary derivatives"""
    pb = small.select(range(8))
    opt = ctx(gpu, prec, _lib.default_params(), bumps_map)
    out = opt.optimize(pb)
    t, new = opt.submit_replan(pb, out, [0, 3, 5], 0.5)
    got = opt.wait(t)
    v = (new.bnd[0, 2], new.bnd[0, 3], new.bnd[0, 13])
    a = (new.bnd[0, 4], new.bnd[0, 5], new.bnd[0, 14])
    assert any(v) and any(a)
    opt.select_lane(t)
    _export(gpu, opt, new, got, orc, init_v=v, init_a=a)
    opt.close()


@pytest.mark.parametrize("prec", [65, 32])
def test_throughput_export_skips_a_problem_over_the_limits(gpu, orc, bumps_map, small, prec):
    from workloads import _with_oversize
    from uneven_planner_b200 import _lib
    pbx = _with_oversize(small.select(range(6)), 2)
    opt = ctx(gpu, prec, _lib.default_params(), bumps_map)
    out = opt.optimize(pbx)
    assert out[0][2].ret_code == _lib.UALM_ELIMIT
    ex = opt.mpc_export(pbx.N, pbx.M, init_v=INIT_V, init_a=INIT_A)
    assert check_export(orc, pbx, out, ex, 0.01, INIT_V, INIT_A) == pbx.B - 1
    opt.close()


# ------------------------------------------------------------------ the C call itself
@pytest.mark.parametrize("prec", PRECISIONS)
def test_any_output_may_be_null(gpu, solved_edges, prec):
    """each output pointer NULL in turn: the others are bit for bit those of the call with every pointer"""
    pb, opt, _ = solved_edges(prec)[1]
    full = opt.mpc_export(pb.N, pb.M, init_v=INIT_V, init_a=INIT_A)
    iv, ia = np.array(INIT_V), np.array(INIT_A)
    for skip in range(len(OUTS)):
        bufs = [np.full(full[k].size, 7.0) for k in OUTS]
        rc = opt.L.ualm_mpc_export_batch(opt.h, C.c_double(0.01), P(iv), P(ia), *[None if j == skip else P(b) for j, b in enumerate(bufs)])
        assert rc == 0
        for j, k in enumerate(OUTS):
            assert (bufs[j] == 7.0).all() if j == skip else np.array_equal(bufs[j], full[k].ravel()), (skip, k)


@pytest.mark.parametrize("prec", [65, 32])
def test_throughput_export_needs_a_collected_batch(gpu, bumps_map, small, prec):
    """on the throughput path a batch solved but not yet synchronised is refused (UALM_ESTATE), then exported once collected"""
    from uneven_planner_b200 import _lib
    pb = small.select(range(5))
    opt = ctx(gpu, prec, _lib.default_params(), bumps_map)
    opt.upload(pb)
    opt.solve_resident()
    sN, sM = int(pb.N.sum()), int(pb.M.sum())
    bufs = [np.full(n, 7.0) for n in (2 * (sN + pb.B), sN, sM + pb.B, sM, 12 * sN, 6 * sM, 4 * pb.B)]
    assert opt.L.ualm_mpc_export_batch(opt.h, C.c_double(0.01), None, None, *[P(b) for b in bufs]) == _lib.UALM_ESTATE
    assert all((b == 7.0).all() for b in bufs)
    opt.sync()
    assert opt.mpc_export(pb.N, pb.M)["c_mpc_xy"].any()
    opt.close()
