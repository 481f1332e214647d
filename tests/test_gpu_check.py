"""Checking trajectories the caller holds against each environment's current grid (include/ualm.h, ualm_check_trajectories), from any time
on, with the time each limit is first broken, on both paths and while batches are in flight.  Grids: the seeded stand-ins of hill (G0)
and desert (G1), solved with the hill parameters; the CPU reference is tests/check_oracle.cpp."""
import collections
import ctypes as C
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
    return hill_desert_world(golden)


def _piece_T(res):
    return np.array([(r.piece_T_xy, r.piece_T_yaw) for r in res], np.float64)


def _total(N, M, Tx, Ty):
    """the duration the scans use: N piece durations and M yaw piece durations summed in order, the smaller one"""
    tx = ty = 0.0
    for _ in range(N):
        tx += Tx
    for _ in range(M):
        ty += Ty
    return min(tx, ty)


def _t_from(pb, out, kind):
    """per problem: 0, an exact sample time (the sequence's own additions), a mid-piece time, the end or past it; kind rotates them"""
    res = out[0]
    tf = np.zeros(pb.B)
    for i in range(pb.B):
        N, M = int(pb.N[i]), int(pb.M[i])
        Tx, Ty = res[i].piece_T_xy, res[i].piece_T_yaw
        total = _total(N, M, Tx, Ty)
        k = (i + kind) % 5
        if k == 1:
            t = 0.0
            for _ in range(int(total / DT) // 3):
                t += DT
            tf[i] = t
        elif k == 2:
            tf[i] = 2.5 * Tx if 2.5 * Tx < total else 0.5 * Tx
        elif k == 3:
            tf[i] = total
        elif k == 4:
            tf[i] = total + 5.0
    return tf


# ---- t_from = 0: the lane's own scan ------------------------------------------------------------

@pytest.mark.parametrize("precision", PRECISIONS)
def test_full_check_is_the_lane_scan(gpu, world, precision):
    """golden + bench-sized batch: columns 0..9 byte-identical to ualm_feasibility_batch of the lane; a first-violation time exactly
    where the scan's maximum breaks the environment's limit"""
    pb = world["a64"]
    p = world["params"]
    opt = ctx(gpu, precision, world["params"], world["g0"])
    out = opt.optimize(pb)
    feas = opt.feasibility(DT)
    chk = opt.check_results(pb, out)
    opt.close()
    assert chk.shape == (pb.B, 16)
    assert np.array_equal(bits(chk[:, :10]), bits(feas))
    breaks = np.stack([np.abs(chk[:, 0]) > p.max_vel, np.abs(chk[:, 1]) > p.max_acc_lon, np.abs(chk[:, 2]) > p.max_acc_lat,
                       np.abs(chk[:, 3]) > p.max_kap, chk[:, 4] > -p.min_cxi, chk[:, 5] > p.max_sig], 1)
    assert np.array_equal(chk[:, 10:] >= 0.0, breaks & (chk[:, 7:8] > 0))
    assert np.all((chk[:, 10:] == -1.0) | (chk[:, 10:] >= 0.0))


# ---- against the CPU reference ------------------------------------------------------------------

def _oracle_rows(envs, pb, out, tf, lims):
    """check_oracle rows: envs[e] = (OracleMap, gravity, env limits); lims None = each environment's own"""
    from check_oracle import check
    res, cxy, cyaw = out
    _, _, ocx, ocy = pb.offsets()
    env = np.zeros(pb.B, int) if getattr(pb, "env", None) is None else np.asarray(pb.env)
    rows = np.zeros((pb.B, 16))
    for i in range(pb.B):
        om, grav, own = envs[int(env[i])]
        rows[i] = check(om, grav, int(pb.N[i]), int(pb.M[i]), cxy[ocx[i]:ocx[i + 1]], cyaw[ocy[i]:ocy[i + 1]], res[i].piece_T_xy,
                        res[i].piece_T_yaw, DT, tf[i], own if lims is None else lims)
    return rows


def _tight(chk):
    """limits at the median of the batch's maxima: every test fires on about half the problems"""
    m = lambda q: float(np.median(np.abs(chk[:, q])))
    return (m(0), m(1), m(2), m(3), -float(np.median(chk[:, 4])), float(np.median(chk[:, 5])))


def _against_oracle(opt, envs, pb, out):
    full = opt.check_results(pb, out)
    tight = _tight(full)
    fired = np.zeros(6, bool)
    pt = _piece_T(out[0])
    total = np.array([_total(int(pb.N[i]), int(pb.M[i]), *pt[i]) for i in range(pb.B)])
    for kind in range(5):
        tf = _t_from(pb, out, kind)
        for lims in (None, tight):
            got = opt.check_results(pb, out, t_from=tf, limits=lims)
            ref = _oracle_rows(envs, pb, out, tf, lims)
            bad = np.nonzero(np.any(bits(got) != bits(ref), axis=1))[0]
            assert bad.size == 0, (kind, lims, bad[:5], got[bad[:2]], ref[bad[:2]])
            if lims is not None:
                fired |= np.any(got[:, 10:] >= 0.0, axis=0)
            ended = tf >= total
            assert np.all(got[ended, 7] == 0.0) and np.all(got[ended, 10:] == -1.0)
    assert fired.all()


def test_check_matches_the_oracle(gpu, world):
    import pyoracle as po
    from check_oracle import limits_of
    from uneven_planner_b200 import problems
    pb = problems.concat([world["gold_pb"], world["bench"].select(np.arange(250))], [0, 0])
    p = world["params"]
    opt = ctx(gpu, 64, world["params"], world["g0"])
    out = opt.optimize(pb)
    _against_oracle(opt, {0: (po.OracleMap(world["g0"]), p.gravity, limits_of(p))}, pb, out)
    opt.close()


def test_check_matches_the_oracle_mixed_environments(gpu, world):
    import pyoracle as po
    from check_oracle import limits_of
    from uneven_planner_b200 import configs, maps, problems
    names = ["hill", "desert", "volcano", "forest"]
    grids = [maps.stand_in_terrain(n) for n in names]
    params = [configs.params_for(n) for n in names]
    subs = [problems.generate(g, 48, seed=21 + e, **configs.gen_kwargs(n)) for e, (g, n) in enumerate(zip(grids, names))]
    cat = problems.concat(subs, range(4))
    mixed = cat.select(np.array([48 * e + i for i in range(48) for e in range(4)]))
    opt = gpu.BatchALMTrajOpt()
    for e in range(4):
        opt.init(params[e], env=e).set_environment(grids[e], env=e)
    out = opt.optimize(mixed)
    _against_oracle(opt, {e: (po.OracleMap(grids[e]), params[e].gravity, limits_of(params[e])) for e in range(4)}, mixed, out)
    opt.close()


# ---- grid updates after the solve ---------------------------------------------------------------

def _far_from_box(pb, out, geom, box, cells=2):
    """per problem: every sampled position more than `cells` cells from the box"""
    res, cxy, _ = out
    _, _, ocx, _ = pb.offsets()
    r = geom.xy_resolution
    x0, y0 = geom.origin[0] + box[0] * r, geom.origin[1] + box[1] * r
    x1, y1 = x0 + box[2] * r, y0 + box[3] * r
    far = np.zeros(pb.B, bool)
    for i in range(pb.B):
        N, M = int(pb.N[i]), int(pb.M[i])
        Tx, Ty = res[i].piece_T_xy, res[i].piece_T_yaw
        t = np.arange(0.0, _total(N, M, Tx, Ty), DT)
        ip = np.minimum((t / Tx).astype(int), N - 1)
        tl = t - ip * Tx
        c = cxy[ocx[i]:ocx[i + 1]].reshape(2, N, 6)
        px = sum(c[0, ip, k] * tl ** k for k in range(6))
        py = sum(c[1, ip, k] * tl ** k for k in range(6))
        d = np.maximum(np.maximum(x0 - px, px - x1), np.maximum(y0 - py, py - y1))
        far[i] = bool(np.all(d > cells * r))
    return far


@pytest.mark.parametrize("variant", ["window", "whole"])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_check_after_an_update_reads_the_new_grid(gpu, world, precision, variant):
    g0, g1, pb = world["g0"], world["g1"], world["b"]
    win = box_cells(g1.cells, BOX)
    spliced = splice(g0, win, BOX)
    opt = ctx(gpu, precision, world["params"], g0)
    out = opt.optimize(pb)
    tf = _t_from(pb, out, 0)
    before = opt.check_results(pb, out, t_from=tf)
    if variant == "window":
        opt.update_environment_window(BOX[0], BOX[1], win)
    else:
        opt.update_environment(spliced)
    after = opt.check_results(pb, out, t_from=tf)
    opt.close()
    fresh = ctx(gpu, precision, world["params"], spliced)
    ref = fresh.check_results(pb, out, t_from=tf)
    fresh.close()
    assert np.array_equal(bits(after), bits(ref))
    far = _far_from_box(pb, out, g0.geom, BOX)
    assert far.any() and not far.all()
    assert np.array_equal(bits(after[far]), bits(before[far]))
    assert np.any(bits(after) != bits(before))


# ---- in flight ----------------------------------------------------------------------------------

@pytest.mark.parametrize("precision", PRECISIONS)
def test_check_while_a_batch_is_in_flight(gpu, world, precision):
    """an earlier batch's trajectories checked while a 1024-problem batch runs: the same rows as with nothing in flight, and the batch in
    flight byte-identical to a lone solve.  On the throughput path the check returns before that batch completes; on the parity path
    the check waits for SM slots in the batch's tail (DESIGN.md section 3i), so only its result is asserted there"""
    A = world["a64"] if precision == 64 else world["bench"]
    E = world["b"]
    opt = ctx(gpu, precision, world["params"], world["g0"])
    out_e = opt.wait(opt.submit(E, depth=2))
    tf = _t_from(E, out_e, 1)
    idle = opt.check_results(E, out_e, t_from=tf)
    ta = opt.submit(A, depth=2)
    assert pending(opt, ta, A) > 0
    chk = opt.check_results(E, out_e, t_from=tf)
    if precision != 64:
        assert pending(opt, ta, A) > 0
    got_a = pieces(A, opt.wait(ta))
    opt.close()
    assert np.array_equal(bits(chk), bits(idle))
    o = ctx(gpu, precision, world["params"], world["g0"])
    ref_a = pieces(A, o.optimize(A))
    o.close()
    assert same_pieces(got_a, ref_a)
    if precision == 64:
        g, n = world["gold"], world["gold_pb"].B
        assert [int(np.frombuffer(p[0], dtype=np.int32, count=1)[0]) for p in got_a[:n]] == [int(x) for x in g["ret_code"]]
        assert np.array_equal(np.concatenate([p[1] for p in got_a[:n]]), g["c_xy"])
        assert np.array_equal(np.concatenate([p[2] for p in got_a[:n]]), g["c_yaw"])


# ---- refusals, memory, C++ ----------------------------------------------------------------------

@pytest.mark.parametrize("precision", PRECISIONS)
def test_refused_checks_write_nothing(gpu, world, precision):
    from uneven_planner_b200 import _lib
    L = _lib.lib()
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int32)
    pb = world["b"].select(np.arange(16))
    opt = ctx(gpu, precision, world["params"], world["g0"])
    out = opt.optimize(pb)
    before = pieces(pb, out)
    res, cxy, cyaw = out
    N, M = np.ascontiguousarray(pb.N, np.int32), np.ascontiguousarray(pb.M, np.int32)
    pt = np.ascontiguousarray(_piece_T(res))
    o = np.full((pb.B, 16), 7.0)
    P = lambda a, t=dp: a.ctypes.data_as(t)

    def call(h=opt.h, B=pb.B, n=N, m=M, p=pt, cx=cxy, cy=cyaw, env=None, tf=None, dt=DT, o_=o):
        return L.ualm_check_trajectories(h, B, None if n is None else P(n, ip), None if m is None else P(m, ip), None if p is None else P(p),
                                         None if cx is None else P(cx), None if cy is None else P(cy), None if env is None else P(env, ip),
                                         None if tf is None else P(tf), dt, None, None if o_ is None else P(o_))
    EINVAL, ESTATE = _lib.UALM_EINVAL, _lib.UALM_ESTATE
    bad_n = N.copy(); bad_n[3] = 0
    bad_m = M.copy(); bad_m[5] = -1
    cases = [dict(h=None), dict(B=-1), dict(n=None), dict(m=None), dict(p=None), dict(cx=None), dict(cy=None), dict(o_=None), dict(dt=0.0),
             dict(dt=-0.01), dict(dt=float("nan")), dict(n=bad_n), dict(m=bad_m)]
    for v in (-1e-9, float("nan"), -np.inf):
        tf = np.zeros(pb.B); tf[7] = v
        cases.append(dict(tf=tf))
    for e in (-1, 4, 1 << 20):
        env = np.zeros(pb.B, np.int32); env[2] = e
        cases.append(dict(env=env))
    for kw in cases:
        assert call(**kw) == EINVAL, kw
    env = np.zeros(pb.B, np.int32); env[9] = 1                     # environment 1 has nothing bound
    assert call(env=env) == ESTATE
    assert np.all(o == 7.0)
    assert call(B=0) == _lib.UALM_OK and np.all(o == 7.0)
    assert same_pieces(pieces(pb, opt.optimize(pb)), before)
    # over the compiled limits, and too many samples: not scanned
    big = np.array([65], np.int32)
    r = opt.check_trajectories(big, [4], [[0.1, 0.1]], np.zeros(12 * 65), np.zeros(24))
    assert np.array_equal(r[0], [0, 0, 0, 0, 0, 0, 0, -1, 0, 0] + [-1] * 6)
    r = opt.check_trajectories(pb.N[:1], pb.M[:1], [[1e6, 1e6]], cxy[:12 * int(pb.N[0])], cyaw[:6 * int(pb.M[0])])
    assert np.array_equal(r[0], [0, 0, 0, 0, 0, 0, 0, -1, 1e6, 1e6] + [-1] * 6)
    opt.close()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_checks_do_not_leak(gpu, world, precision):
    import torch
    depth = 3 if precision == 64 else 8
    pb = world["b"]
    opt = ctx(gpu, precision, world["params"], world["g0"])

    def fill():
        return [opt.wait(t) for t in [opt.submit(pb, depth=depth) for _ in range(depth)]][-1]
    last = fill()
    opt.check_results(pb, last)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    q = collections.deque()
    for i in range(20):
        src = world["g1"] if i % 2 == 0 else world["g0"]
        opt.update_environment_window(BOX[0], BOX[1], box_cells(src.cells, BOX))
        if len(q) == depth:
            last = opt.wait(q.popleft())
        chk = opt.check_results(pb, last, t_from=0.5)
        assert chk.shape == (pb.B, 16)
        q.append(opt.submit(pb, depth=depth))
    while q:
        opt.wait(q.popleft())
    fill()
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    opt.close()
    grid = world["g0"].cells.nbytes
    assert free0 - free1 <= grid, (free0, free1, grid)


def test_cpp_check_between_submit_and_window(gpu, world, tmp_path):
    from uneven_planner_b200 import _lib
    exe = build_driver("check_driver", tmp_path)
    g0, g1 = world["g0"], world["g1"]
    pb = world["bench"].select(np.arange(8))
    win = np.ascontiguousarray(box_cells(g1.cells, BOX))
    tf = np.array([0.0, 0.5, 1.0, 1.5, 2.0, 2.5, 3.0, 100.0])
    case = str(tmp_path / "check.bin")
    with open(case, "wb") as f:
        f.write(struct.pack("<8i", *g0.shape, pb.B, *BOX))
        f.write(g0.cells.tobytes())
        f.write(win.tobytes())
        for a in (pb.N, pb.M):
            f.write(np.ascontiguousarray(a, np.int32).tobytes())
        for a in (pb.bnd, pb.total_time, pb.inner_xy, pb.inner_yaw, tf):
            f.write(np.ascontiguousarray(a, np.float64).tobytes())
    r = subprocess.run([exe, case], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    opt = gpu.BatchALMTrajOpt().init(_lib.default_params()).set_environment(g0)
    out = opt.wait(opt.submit(pb, depth=3))
    t2 = opt.submit(pb, depth=3)
    c0 = opt.check_results(pb, out, t_from=tf)
    opt.update_environment_window(BOX[0], BOX[1], win, env=0)
    c1 = opt.check_results(pb, out, t_from=tf)
    opt.wait(t2)
    opt.close()
    rows = [ln.split() for ln in r.stdout.strip().splitlines()]
    assert [(int(x[0]), int(x[1])) for x in rows] == [(p, i) for p in range(2) for i in range(pb.B)]
    got = np.array([[float(v) for v in x[2:]] for x in rows])
    assert np.array_equal(bits(got), bits(np.concatenate([c0, c1])))
    assert np.any(bits(c0) != bits(c1))
