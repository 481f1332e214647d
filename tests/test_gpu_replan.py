"""Replanning trajectories the caller holds from each robot's current state to its goal, as a submitted ticket (include/ualm.h,
ualm_submit_replan), on both paths and while batches are in flight.  Grids: the seeded stand-ins of hill (G0) and desert (G1), solved
with the hill parameters; the CPU reference of the build is tests/replan_oracle.cpp."""
import collections
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

from harness import bits, box_cells, build_driver, ctx, gpu, pending, pieces, same_pieces, splice  # noqa: F401
from workloads import hill_desert_world


pytestmark = pytest.mark.gpu
PRECISIONS = [64, 32, 65]
BOX = (60, 80, 40, 40)                # a 2 m x 2 m window of the 10 m grid, where the hill problems run
DT = 0.01


@pytest.fixture(scope="module")
def world(gpu, golden):
    w = hill_desert_world(golden)
    opt = gpu.BatchALMTrajOpt().init(w["params"]).set_environment(w["g0"])
    w["held"] = opt.optimize(w["gold_pb"])         # the trajectories the caller holds: the golden problems solved on the parity path
    w["held_b"] = opt.optimize(w["b"])
    opt.close()
    return w


def _total(N, M, Tx, Ty):
    tx = ty = 0.0
    for _ in range(N):
        tx += Tx
    for _ in range(M):
        ty += Ty
    return min(tx, ty)


def _seq(total, dt):
    t, out = 0.0, []
    while t < total:
        out.append(t)
        t += dt
    return out


def _t_from(pb, out, kind, dt=DT):
    """per row: 0, an exact sample time k dt (the sequence's own additions), mid-piece, exactly a piece boundary i T_xy (repeated
    addition, as the lookup subtracts), the last sample before the end; kind rotates them"""
    res = out[0]
    tf = np.zeros(pb.B)
    for i in range(pb.B):
        N, M = int(pb.N[i]), int(pb.M[i])
        Tx, Ty = res[i].piece_T_xy, res[i].piece_T_yaw
        total = _total(N, M, Tx, Ty)
        k = (i + kind) % 5
        if k == 1:
            s = _seq(total, dt)
            tf[i] = s[len(s) // 3]
        elif k == 2:
            tf[i] = 2.5 * Tx if 2.5 * Tx < total else 0.5 * Tx
        elif k == 3:
            t = 0.0
            for _ in range(max(N // 2, 1)):
                t += Tx
            tf[i] = t if t < total else 0.0
        elif k == 4:
            tf[i] = _seq(total, dt)[-1]
    return tf


def _same_pb(a, b):
    return (np.array_equal(a.N, b.N) and np.array_equal(a.M, b.M) and np.array_equal(bits(a.bnd), bits(b.bnd)) and
            np.array_equal(bits(a.total_time), bits(b.total_time)) and np.array_equal(bits(a.inner_xy), bits(b.inner_xy)) and
            np.array_equal(bits(a.inner_yaw), bits(b.inner_yaw)))


def _rp(vals):
    from uneven_planner_b200 import front_end
    return None if vals is None else front_end.resample_params(*vals)


# ---- the built problems against the CPU reference -----------------------------------------------

@pytest.mark.parametrize("precision", PRECISIONS)
def test_built_problems_are_the_reference(gpu, world, precision):
    """every kind of t_from, at two dt and with altered resampler parameters: N', M', bnd', total_time and the inner points bit for bit
    the reference (so the same bits at every precision); the ticket is byte-identical to a submit of the returned arrays"""
    import replan_oracle as ro
    pb, out = world["gold_pb"], world["held"]
    rows = np.arange(pb.B)
    opt = ctx(gpu, precision, world["params"], world["g0"])
    for dt, rp in ((DT, None), (0.023, None), (DT, (0.21, 3.0, 0.7, 1.4))):
        for kind in range(5):
            tf = _t_from(pb, out, kind, dt)
            t, new = opt.submit_replan(pb, out, rows, tf, dt=dt, rparams=_rp(rp))
            got = pieces(new, opt.wait(t))
            ref = ro.problems_of(ro.rows(pb, out, rows, tf, dt, rp or ro.DEFAULT_RP))
            assert _same_pb(new, ref), (dt, rp, kind)
            if kind == 0 and rp is None and dt == DT:
                assert same_pieces(got, pieces(new, opt.wait(opt.submit(new))))
    opt.close()


def test_padded_outputs_of_the_c_call(gpu, world):
    """the fixed-stride inner outputs: the row's points, then zeros"""
    import replan_oracle as ro
    from uneven_planner_b200 import _lib
    pb, (res, cxy, cyaw) = world["gold_pb"], world["held"]
    B = pb.B
    tf = _t_from(pb, world["held"], 2)
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int32)
    P = lambda a, t=dp: a.ctypes.data_as(t)
    N, M = np.ascontiguousarray(pb.N, np.int32), np.ascontiguousarray(pb.M, np.int32)
    pt = np.array([(r.piece_T_xy, r.piece_T_yaw) for r in res], np.float64)
    bnd = np.ascontiguousarray(pb.bnd, np.float64)
    No, Mo, bo, To = np.zeros(B, np.int32), np.zeros(B, np.int32), np.zeros((B, 18)), np.zeros(B)
    ixy, iyaw = np.full((B, 126), 7.0), np.full((B, 127), 7.0)
    opt = ctx(gpu, 64, world["params"], world["g0"])
    t = C.c_int(-1)
    assert _lib.lib().ualm_submit_replan(opt.h, B, P(N, ip), P(M, ip), P(pt), P(cxy), P(cyaw), P(bnd), None, P(tf), DT, None, 2, C.byref(t),
                                          P(No, ip), P(Mo, ip), P(bo), P(To), P(ixy), P(iyaw)) == 0
    ref = ro.rows(pb, world["held"], np.arange(B), tf)
    assert np.array_equal(bits(ixy), bits(ref[:, 21:147])) and np.array_equal(bits(iyaw), bits(ref[:, 147:]))
    assert np.array_equal(No, ref[:, 19]) and np.array_equal(Mo, ref[:, 20]) and np.array_equal(bits(bo), bits(ref[:, :18]))
    opt._tickets = {t.value: (ro.problems_of(ref), None)}
    opt.wait(t.value)
    opt.close()


def test_mixed_environments(gpu, world):
    """a four-environment batch: each row built from its own coefficients and solved in its own environment"""
    import replan_oracle as ro
    from uneven_planner_b200 import configs, maps, problems
    names = ["hill", "desert", "volcano", "forest"]
    grids = [maps.stand_in_terrain(n) for n in names]
    params = [configs.params_for(n) for n in names]
    subs = [problems.generate(g, 32, seed=21 + e, **configs.gen_kwargs(n)) for e, (g, n) in enumerate(zip(grids, names))]
    mixed = problems.concat(subs, range(4)).select(np.array([32 * e + i for i in range(32) for e in range(4)]))
    opt = gpu.BatchALMTrajOpt()
    for e in range(4):
        opt.init(params[e], env=e).set_environment(grids[e], env=e)
    out = opt.optimize(mixed)
    rows = np.arange(1, mixed.B, 3)        # every environment: the batch interleaves them
    tf = _t_from(mixed, out, 1)[rows]
    t, new = opt.submit_replan(mixed, out, rows, tf)
    got = pieces(new, opt.wait(t))
    assert np.array_equal(new.env, mixed.env[rows]) and len(set(new.env.tolist())) == 4
    assert _same_pb(new, ro.problems_of(ro.rows(mixed, out, rows, tf), new.env))
    assert same_pieces(got, pieces(new, opt.wait(opt.submit(new))))
    opt.close()
    for e in range(4):                               # each environment's rows alone on a context of that environment only
        k = np.nonzero(new.env == e)[0]
        one = new.select(k)
        one.env = None
        o = gpu.BatchALMTrajOpt().init(params[e]).set_environment(grids[e])
        assert same_pieces([got[i] for i in k], pieces(one, o.optimize(one)))
        o.close()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_rows_over_the_limits(gpu, world, precision):
    """short pieces push the rows replanned from the start past 64 pieces: UALM_ELIMIT from the first poll with zero coefficients; the
    rows replanned from near the end fit and are unaffected"""
    from uneven_planner_b200 import _lib
    pb, out = world["gold_pb"], world["held"]
    last = np.array([_seq(_total(int(pb.N[i]), int(pb.M[i]), out[0][i].piece_T_xy, out[0][i].piece_T_yaw), DT)[-1] for i in range(pb.B)])
    tf = np.where(np.arange(pb.B) % 2 == 0, 0.0, last)
    rp = (0.05, 2.0, 0.5, 1.2)
    opt = ctx(gpu, precision, world["params"], world["g0"])
    t, new = opt.submit_replan(pb, out, np.arange(pb.B), tf, rparams=_rp(rp))
    over = (new.N > 64) | (new.M > 128)
    assert over.any() and not over.all()
    buf = opt.outputs(new)
    idx, _ = opt.poll(t, buf, 0.0)
    assert set(np.nonzero(over)[0].tolist()) <= set(idx.tolist())
    got = pieces(new, opt.wait(t))
    _, _, ocx, ocy = new.offsets()
    for i in np.nonzero(over)[0]:
        assert buf[0][i].ret_code == _lib.UALM_ELIMIT and not buf[1][ocx[i]:ocx[i + 1]].any() and not buf[2][ocy[i]:ocy[i + 1]].any()
    fit = np.nonzero(~over)[0]
    sub = new.select(fit)
    assert same_pieces([got[i] for i in fit], pieces(sub, opt.wait(opt.submit(sub))))
    opt.close()


# ---- the ticket ---------------------------------------------------------------------------------

@pytest.mark.parametrize("precision", PRECISIONS)
def test_the_ticket_is_any_ticket(gpu, world, precision):
    """polled then waited, the records are byte-identical to a submit of the returned arrays; at 64, 64 rows bit for bit the oracle's
    solve of the reference-built problems; a cancel stops its rows; ualm_wait_batch_for works on the ticket"""
    import pyoracle as po
    import replan_oracle as ro
    from uneven_planner_b200 import _lib
    pb, out = world["b"], world["held_b"]
    rows = np.arange(0, 256, 2)
    tf = _t_from(pb, out, 3)[rows]
    opt = ctx(gpu, precision, world["params"], world["g0"])
    t, new = opt.submit_replan(pb, out, rows, tf)
    buf = opt.outputs(new)
    seen = set()
    while True:
        idx, left = opt.poll(t, buf, 5.0)
        seen |= set(idx.tolist())
        if left == 0:
            break
    waited = pieces(new, opt.wait(t))
    assert seen == set(range(new.B)) and same_pieces(pieces(new, buf), waited)
    lone = pieces(new, opt.wait(opt.submit(new)))
    assert same_pieces(waited, lone)
    t2, new2 = opt.submit_replan(pb, out, rows, tf)
    assert same_pieces(pieces(new2, opt.wait(t2, timeout_ms=600000.0)), lone)
    t3, _ = opt.submit_replan(pb, out, rows, tf)
    stop = np.arange(5, new.B, 3)
    opt.cancel(t3, stop)
    got = pieces(new, opt.wait(t3))
    opt.close()
    codes = [int(np.frombuffer(g[0], np.int32, count=1)[0]) for g in got]
    assert sum(codes[i] == _lib.UALM_RET_STOPPED for i in stop) >= len(stop) // 2
    assert all(codes[i] == _lib.UALM_RET_STOPPED or got[i][0] == lone[i][0] for i in stop)
    keep = np.setdiff1d(np.arange(new.B), stop)
    assert same_pieces([got[i] for i in keep], [lone[i] for i in keep])
    if precision == 64:
        ref = ro.problems_of(ro.rows(pb, out, rows, tf))
        sel = np.arange(64)
        ores = po.solve_batch(po.params_from(world["params"]), po.OracleMap(world["g0"]), ref, threads=min(32, os.cpu_count()), idx=sel)
        for k, i in enumerate(sel):
            r, ocxy, ocyaw, _ = ores[k]
            g = _lib.Result.from_buffer_copy(lone[i][0])
            assert (g.ret_code, g.outer_iters, g.n_evals, g.n_lbfgs_iters, g.total_T, g.inner_cost) == \
                   (r.ret_code, r.outer_iters, r.n_evals, r.n_lbfgs_iters, r.total_T, r.inner_cost), i
            assert np.array_equal(lone[i][1], ocxy) and np.array_equal(lone[i][2], ocyaw), i


# ---- in flight ----------------------------------------------------------------------------------

@pytest.mark.parametrize("precision", PRECISIONS)
def test_replan_while_a_batch_is_in_flight(gpu, world, precision):
    """256 rows replanned while a 1024-problem batch runs: the batch byte-identical to a lone solve (at 64 its golden problems equal the
    goldens), the replanned ticket byte-identical to the same replan idle; on the throughput path the call returns before the batch
    completes"""
    A = world["a64"] if precision == 64 else world["bench"]
    pb, out = world["b"], world["held_b"]
    rows = np.arange(256)
    tf = _t_from(pb, out, 2)
    opt = ctx(gpu, precision, world["params"], world["g0"])
    t0, _ = opt.submit_replan(pb, out, rows, tf, depth=3)
    idle = opt.wait(t0)
    ta = opt.submit(A, depth=3)
    assert pending(opt, ta, A) > 0
    tr, new = opt.submit_replan(pb, out, rows, tf, depth=3)
    if precision != 64:
        assert pending(opt, ta, A) > 0
    got_r = pieces(new, opt.wait(tr))
    got_a = pieces(A, opt.wait(ta))
    opt.close()
    assert same_pieces(got_r, pieces(new, idle))
    o = ctx(gpu, precision, world["params"], world["g0"])
    ref_a = pieces(A, o.optimize(A))
    o.close()
    assert same_pieces(got_a, ref_a)
    if precision == 64:
        g, n = world["gold"], world["gold_pb"].B
        assert [int(np.frombuffer(p[0], dtype=np.int32, count=1)[0]) for p in got_a[:n]] == [int(x) for x in g["ret_code"]]
        assert np.array_equal(np.concatenate([p[1] for p in got_a[:n]]), g["c_xy"])
        assert np.array_equal(np.concatenate([p[2] for p in got_a[:n]]), g["c_yaw"])


@pytest.mark.parametrize("precision", PRECISIONS)
def test_replan_after_a_window_update(gpu, world, precision):
    """after ualm_update_map_window the replanned problems solve byte-identically to a lone solve of the returned arrays on a fresh context
    bound to the grid spliced in numpy"""
    g0, g1 = world["g0"], world["g1"]
    pb, out = world["b"], world["held_b"]
    win = box_cells(g1.cells, BOX)
    spliced = splice(g0, win, BOX)
    opt = ctx(gpu, precision, world["params"], g0)
    t0 = opt.submit(pb, depth=2)
    opt.update_environment_window(BOX[0], BOX[1], win)
    t, new = opt.submit_replan(pb, out, np.arange(pb.B), _t_from(pb, out, 0), depth=2)
    got = pieces(new, opt.wait(t))
    opt.wait(t0)
    opt.close()
    fresh = ctx(gpu, precision, world["params"], spliced)
    ref = pieces(new, fresh.optimize(new))
    fresh.close()
    assert same_pieces(got, ref)


# ---- refusals, memory, C++ ----------------------------------------------------------------------

@pytest.mark.parametrize("precision", PRECISIONS)
def test_refused_replans_write_nothing_and_take_no_lane(gpu, world, precision):
    from uneven_planner_b200 import _lib
    L = _lib.lib()
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int32)
    pb = world["b"].select(np.arange(16))
    opt = ctx(gpu, precision, world["params"], world["g0"])
    out = opt.optimize(pb)
    before = pieces(pb, out)
    res, cxy, cyaw = out
    N, M = np.ascontiguousarray(pb.N, np.int32), np.ascontiguousarray(pb.M, np.int32)
    pt = np.array([(r.piece_T_xy, r.piece_T_yaw) for r in res], np.float64)
    bnd = np.ascontiguousarray(pb.bnd, np.float64)
    tf0 = _t_from(pb, out, 2)
    No, Mo, bo, To = np.full(pb.B, 7, np.int32), np.full(pb.B, 7, np.int32), np.full((pb.B, 18), 7.0), np.full(pb.B, 7.0)
    ixy, iyaw = np.full((pb.B, 126), 7.0), np.full((pb.B, 127), 7.0)
    P = lambda a, t=dp: a.ctypes.data_as(t)
    tk = C.c_int(-5)

    def call(h=opt.h, B=pb.B, n=N, m=M, p=pt, cx=cxy, cy=cyaw, bd=bnd, env=None, tf=tf0, dt=DT, rp=None, depth=2, ticket=True, no=No, mo=Mo,
             b_=bo, to=To):
        return L.ualm_submit_replan(h, B, *[None if a is None else P(a, ip) for a in (n, m)], *[None if a is None else P(a) for a in (p, cx, cy, bd)],
                                    None if env is None else P(env, ip), None if tf is None else P(tf), dt, rp, depth, C.byref(tk) if ticket else None,
                                    None if no is None else P(no, ip), None if mo is None else P(mo, ip), None if b_ is None else P(b_),
                                    None if to is None else P(to), P(ixy), P(iyaw))
    EINVAL, ESTATE = _lib.UALM_EINVAL, _lib.UALM_ESTATE
    bad_n = N.copy(); bad_n[3] = 0
    bad_m = M.copy(); bad_m[5] = -1
    cases = [dict(h=None), dict(B=-1), dict(n=None), dict(m=None), dict(p=None), dict(cx=None), dict(cy=None), dict(bd=None), dict(tf=None),
             dict(ticket=False), dict(no=None), dict(mo=None), dict(b_=None), dict(to=None), dict(dt=0.0), dict(dt=-0.01), dict(dt=float("nan")),
             dict(n=bad_n), dict(m=bad_m), dict(depth=0), dict(depth=1 << 20), dict(p=np.full_like(pt, 1e6), dt=1e-3)]
    end = _total(int(N[7]), int(M[7]), pt[7, 0], pt[7, 1])
    for v in (-1e-9, float("nan"), -np.inf, end, end + 1.0, np.inf):
        tf = tf0.copy()
        tf[7] = v
        cases.append(dict(tf=tf))
    for f in range(4):
        vals = [0.3, 2.0, 0.5, 1.2, 0.05]
        for v in (0.0, -1.0, float("nan")):
            w = list(vals); w[f] = v
            cases.append(dict(rp=C.byref(_lib.ResampleParams(*w))))
    for e in (-1, 4, 1 << 20):
        env = np.zeros(pb.B, np.int32); env[2] = e
        cases.append(dict(env=env))
    for kw in cases:
        assert call(**kw) == EINVAL, kw
    env = np.zeros(pb.B, np.int32); env[9] = 1                     # environment 1 has nothing bound
    assert call(env=env) == ESTATE
    # a lane in flight: depth 1 with the lane's batch still running
    t1 = opt.submit(pb, depth=1)
    assert call(depth=1) == ESTATE
    opt.wait(t1)
    assert np.all(No == 7) and np.all(Mo == 7) and np.all(bo == 7.0) and np.all(To == 7.0) and np.all(ixy == 7.0) and np.all(iyaw == 7.0)
    assert tk.value == -5
    # init_sig_vel is not used: any value is accepted
    ok = call(rp=C.byref(_lib.ResampleParams(0.3, 2.0, 0.5, 1.2, -3.0)), depth=3)
    assert ok == 0
    t_ok = tk.value
    assert np.all(No != 7)
    opt._tickets[t_ok] = (pb, None)
    opt.wait(t_ok)
    # no lane was taken by the refusals: the next submit gets the ticket it would have got
    nxt = opt.submit(pb, depth=3)
    assert nxt == (t_ok + 1) % 3
    assert same_pieces(pieces(pb, opt.wait(nxt)), before)
    # B = 0 is an empty submit
    assert call(B=0, n=None, m=None, p=None, cx=None, cy=None, bd=None, tf=None, no=None, mo=None, b_=None, to=None, depth=3) == 0
    assert tk.value == (nxt + 1) % 3
    opt._tickets[tk.value] = (pb.select([]), None)
    opt.wait(tk.value)
    assert same_pieces(pieces(pb, opt.optimize(pb)), before)
    opt.close()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_replans_do_not_leak(gpu, world, precision):
    import torch
    depth = 3 if precision == 64 else 8
    pb, held = world["b"], world["held_b"]
    opt = ctx(gpu, precision, world["params"], world["g0"])

    def fill():
        return [opt.wait(t) for t in [opt.submit(pb, depth=depth) for _ in range(depth)]][-1]
    fill()
    opt.wait(opt.submit_replan(pb, held, np.arange(pb.B), 0.5, depth=depth)[0])
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    q = collections.deque()
    for i in range(20):
        src = world["g1"] if i % 2 == 0 else world["g0"]
        opt.update_environment_window(BOX[0], BOX[1], box_cells(src.cells, BOX))
        if len(q) >= depth - 1:
            opt.wait(q.popleft())
        if i % 2 == 0:
            q.append(opt.submit_replan(pb, held, np.arange(pb.B), 0.5, depth=depth)[0])
        else:
            q.append(opt.submit(pb, depth=depth))
    while q:
        opt.wait(q.popleft())
    fill()
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    opt.close()
    grid = world["g0"].cells.nbytes
    assert free0 - free1 <= grid, (free0, free1, grid)


def test_cpp_replan_between_submit_and_wait(gpu, world, tmp_path):
    from uneven_planner_b200 import _lib
    exe = build_driver("replan_driver", tmp_path)
    g0 = world["g0"]
    pb = world["bench"].select(np.arange(8))
    tf = np.array([0.0, 0.5, 1.0, 1.5, 2.0, 2.5, 0.25, 0.75])
    case = str(tmp_path / "replan.bin")
    with open(case, "wb") as f:
        f.write(struct.pack("<4i", *g0.shape, pb.B))
        f.write(g0.cells.tobytes())
        for a in (pb.N, pb.M):
            f.write(np.ascontiguousarray(a, np.int32).tobytes())
        for a in (pb.bnd, pb.total_time, pb.inner_xy, pb.inner_yaw, tf):
            f.write(np.ascontiguousarray(a, np.float64).tobytes())
    r = subprocess.run([exe, case], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    opt = gpu.BatchALMTrajOpt().init(_lib.default_params()).set_environment(g0)
    out = opt.wait(opt.submit(pb, depth=3))
    t2 = opt.submit(pb, depth=3)
    t3, new = opt.submit_replan(pb, out, np.arange(pb.B), tf, depth=3)
    opt.wait(t2)
    res, cxy, cyaw = opt.wait(t3)
    opt.close()
    lines = r.stdout.strip().splitlines()
    head = [ln.split() for ln in lines[:pb.B]]
    assert [int(x[0]) for x in head] == list(range(pb.B))
    assert [(int(x[1]), int(x[2])) for x in head] == list(zip(new.N.tolist(), new.M.tolist()))
    got = np.array([[float(v) for v in x[3:22]] for x in head])
    assert np.array_equal(bits(got), bits(np.concatenate([new.total_time[:, None], new.bnd], 1)))
    assert [int(x[22]) for x in head] == [r_.ret_code for r_ in res]
    assert np.array_equal(bits([float(x[23]) for x in head]), bits([r_.total_T for r_ in res]))
    coef = np.array([float(v) for v in lines[pb.B:]])
    assert np.array_equal(bits(coef), bits(np.concatenate([cxy, cyaw])))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_degenerate_inputs_are_refused_or_cut_short(gpu, world, precision):
    """a diverged solve's coefficients and non-finite goals are refused before the build; a goal so far that its length's squares
    overflow is refused after it, before any output; a huge end_yaw or a far goal is cut short and comes back UALM_ELIMIT, the
    reference's bits, while the other rows are unaffected.  Every call returns promptly, and a refusal takes no lane"""
    import time
    import replan_oracle as ro
    from uneven_planner_b200 import _lib
    pb0, out0 = world["b"], world["held_b"]
    sel = np.arange(8)
    pb = pb0.select(sel)
    _, _, ocx, ocy = pb0.offsets()
    res8 = (_lib.Result * 8)(*[out0[0][i] for i in sel])
    out = (res8, out0[1][:ocx[8]].copy(), out0[2][:ocy[8]].copy())
    tf = _t_from(pb, out, 2)
    opt = ctx(gpu, precision, world["params"], world["g0"])
    t_ok, ref_new = opt.submit_replan(pb, out, np.arange(8), tf, depth=3)
    ref_got = pieces(ref_new, opt.wait(t_ok))

    def bad_pb(k, v):
        b = pb.select(np.arange(8))
        b.bnd[3, k] = v
        return b
    cxy_inf = out[1].copy(); cxy_inf[5] = np.inf
    cyaw_nan = out[2].copy(); cyaw_nan[-1] = np.nan
    for p_, o_ in ((pb, (res8, cxy_inf, out[2])), (pb, (res8, out[1], cyaw_nan)), (bad_pb(15, np.nan), out), (bad_pb(6, np.inf), out),
                   (bad_pb(6, 1e300), out)):
        t0 = time.perf_counter()
        with pytest.raises(gpu.UalmError, match="error -2"):
            opt.submit_replan(p_, o_, np.arange(8), tf, depth=3)
        assert time.perf_counter() - t0 < 10.0
    assert opt.submit(pb, depth=3) == (t_ok + 1) % 3           # no lane was taken
    opt.wait((t_ok + 1) % 3)
    for k, v in ((15, 1e300), (6, 1e9)):
        b = bad_pb(k, v)
        t0 = time.perf_counter()
        t, new = opt.submit_replan(b, out, np.arange(8), tf, depth=3)
        assert time.perf_counter() - t0 < 10.0
        assert (new.N[3], new.M[3]) == (4097, 4097)
        buf = opt.outputs(new)
        idx, _ = opt.poll(t, buf, 0.0)
        assert 3 in idx.tolist() and buf[0][3].ret_code == _lib.UALM_ELIMIT
        got = pieces(new, opt.wait(t))
        assert not got[3][1].any() and not got[3][2].any()
        assert _same_pb(new, ro.problems_of(ro.rows(b, out, np.arange(8), tf)))
        keep = [i for i in range(8) if i != 3]
        assert same_pieces([got[i] for i in keep], [ref_got[i] for i in keep])
    opt.close()
