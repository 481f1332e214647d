"""Every device-side consumer of the SE(2) map grid on grids that are not the 10 m square (the table GRIDS of
tests/test_map_geometry.py: X != Y both ways, other resolutions, cell counts that are not multiples of the TMA tile, an odd number of
yaw layers, a 20 m x 10 m site), on a grid whose geometry changes while batches are in flight, and on one context whose environments
differ in geometry.

What each comparison is:
  * parity path (precision 64): one evaluation, initScaling, whole solves, the post-solve scan and ualm_check_trajectories against
    the CPU oracle, bit for bit;
  * throughput path (65 / 32): one evaluation against the oracle block by block with the tolerances of tests/test_gpu_tp_shapes.py,
    TMA-staged tiles against the direct gather bit for bit, whole solves as complete records whose scan is the oracle's bit for bit
    and whose converged share is the oracle's within the population bound of tests/test_gpu_tp.py;
  * device map builder and window updates against the host builder / numpy splices, cells as uint32;
  * in flight and mixed environments: byte for byte against the same batch solved alone on a fresh context.
Batches per grid: generated problems over most of the rectangle, plus hand-placed ones from the grid's own bounds (BATCH_CASES).
test_batches_reach_the_rectangle_and_its_edges needs no GPU (the other tests are marked one by one): it fails if the batches stop
reaching the edges, or the window problems stop reading the boxes, that the device tests rely on.
Nothing here is timed, and out-of-range boxes are only ever offered to the library's argument checks."""
import ctypes as C
import functools

import numpy as np
import pytest

import workloads
from harness import alone, bits, cat, ctx, gpu, pieces, same_pieces, splice  # noqa: F401
from workloads import BATCH_CASES, DT, GRIDS, SMALL, THREADS, _arc_problem, _cloud, _parity_evaluation, _scan_and_check, generated, geometry, grid, hand_cases


PRECISIONS = [64, 65, 32]
TP = [65, 32]
WAIT_MS = 300000.0        # no wait here is unbounded: a batch that has not finished by then is stopped and the test fails
N_GEN = 24


@functools.lru_cache(maxsize=None)
def batch(name):
    """N_GEN generated problems on grid `name`, then BATCH_CASES"""
    m = grid(name)
    hc = hand_cases(m.geom)
    return cat([generated(m, N_GEN, GRIDS[name][5])] + [hc[k] for k in BATCH_CASES])


def window_cases(geom):
    """two problems for the window tests: an arc inside the far-corner box of _boxes, and one in the last cell column in x at the y of
    its single-column box"""
    bx, by, oy, r = geom.max_boundary[0], geom.max_boundary[1], geom.origin[1], geom.xy_resolution
    return [_arc_problem(6, 10, radius=0.3, arc=1.5 * np.pi, centre=(bx - 0.5, by - 0.32)),
            _arc_problem(3, 5, radius=0.3, arc=0.6, start=-0.3, centre=(bx - 0.31, oy + 5.5 * r + 0.004))]


def window_source(name):
    """the grid the windows of grid `name` are cut from: another terrain, tilted so that no cell equals the grid's own where both are flat"""
    from uneven_planner_b200 import maps
    m = maps.synthetic_terrain("hills", seed=GRIDS[name][5] + 20, geom=geometry(name))
    m.cells[..., 2] += np.float32(0.05)
    return m


def _boxes(X, Y):
    """nx != ny: the far corner, a full-width strip, a full-height strip, one column"""
    return [(X - 30, Y - 11, 30, 11), (0, Y // 3, X, 3), (X // 4, 0, 2, Y), (X - 1, 5, 1, 1)]


def sides(pb, cxy, geom, K):
    """which clamps and which sides of the map the samples of one problem reach, per axis: lo / hi = a sample inside the map whose
    lower / upper neighbour cell is clamped, off_lo / off_hi = a sample beyond that side (the lookups' formulas in float64)"""
    N = int(pb.N[0])
    Tx = float(pb.total_time[0]) / N
    out = set()
    for i in range(N):
        for j in range(K + 1):
            pw = (j * (Tx / K)) ** np.arange(6)
            pos = (float(cxy[6 * i:6 * i + 6] @ pw), float(cxy[6 * N + 6 * i:6 * N + 6 * i + 6] @ pw))
            off = [a for a in (0, 1) if pos[a] < geom.origin[a] + 1e-4 or pos[a] > geom.max_boundary[a] - 1e-4]
            for a in off:
                out.add(("off_lo_", "off_hi_")[pos[a] > 0] + "xy"[a])
            if off:
                continue
            for a in (0, 1):
                i0 = int(np.floor((pos[a] - 0.5 * geom.xy_resolution - geom.origin[a]) / geom.xy_resolution))
                if i0 < 0:
                    out.add("lo_" + "xy"[a])
                if i0 + 1 > geom.voxel_num[a] - 1:
                    out.add("hi_" + "xy"[a])
    return out


def test_batches_reach_the_rectangle_and_its_edges(built):
    """no GPU: the generated problems span most of both axes of every grid, and each hand case reaches what it is there for"""
    import pyoracle as po
    from uneven_planner_b200 import _lib
    p = _lib.default_params()
    op = po.params_from(p)
    for name in SMALL:
        m = grid(name)
        g = m.geom
        pb = batch(name)
        assert pb.B == N_GEN + len(BATCH_CASES)
        ends = np.vstack([pb.bnd[:N_GEN, 0:2], pb.bnd[:N_GEN, 6:8]])
        assert np.ptp(ends[:, 0]) > 0.7 * (g.max_boundary[0] - g.origin[0]) and np.ptp(ends[:, 1]) > 0.7 * (g.max_boundary[1] - g.origin[1]), name
        om = po.OracleMap(m)
        got = {}
        for k, case in enumerate(BATCH_CASES):
            one = pb.select([N_GEN + k])
            o = po.eval_one(op, om, one, 0, one.x0(0))
            got[case] = sides(one, o["c_xy"], g, p.int_K)
            if case == "yaw_seam":
                assert workloads.reach(one, o["c_xy"], o["c_yaw"], g, p.int_K)["seam"] and not got[case], name
        # fine_yaw's 183 cells in x reach 0.02 m past its 7.3 m, so no sample inside the map has a clamped upper neighbour in x there
        assert got["border_x"] == ({"hi_x"} if name != "fine_yaw" else set()) and got["border_y"] == {"hi_y"}, (name, got)
        assert got["off_x"] >= {"hi_x", "off_hi_x"} - ({"hi_x"} if name == "fine_yaw" else set()) and got["off_y"] >= {"hi_y", "off_hi_y"}, (name, got)
        assert got["off_lo_x"] >= {"lo_x", "off_lo_x"} and got["off_lo_y"] >= {"lo_y", "off_lo_y"}, (name, got)
        assert not (got["off_x"] | got["off_lo_x"]) & {"off_lo_y", "off_hi_y"} and not (got["off_y"] | got["off_lo_y"]) & {"off_lo_x", "off_hi_x"}, (name, got)
    # every box of the window tests is read by some problem of their batch: the oracle's constraint values change with each splice
    for name in ("wide", "tall"):
        base = grid(name)
        pb = cat([batch(name)] + window_cases(base.geom))
        other = window_source(name)
        before = [po.eval_one(op, po.OracleMap(base), pb, i, pb.x0(i))["gx"].tobytes() for i in range(pb.B)]
        for box in _boxes(*base.shape[:2]):
            ix0, iy0, nx, ny = box
            om = po.OracleMap(splice(base, other.cells[ix0:ix0 + nx, iy0:iy0 + ny], box))
            assert [po.eval_one(op, om, pb, i, pb.x0(i))["gx"].tobytes() for i in range(pb.B)] != before, (name, box)


# ------------------------------------------------------------------ fixtures and helpers
def _wait(opt, ticket, pb):
    """wait with a bound; a batch that had to be stopped fails the test"""
    from uneven_planner_b200 import _lib
    out = opt.wait(ticket, timeout_ms=WAIT_MS)
    assert all(r.ret_code != _lib.UALM_RET_STOPPED for r in out[0]), "the batch did not finish within %g ms" % WAIT_MS
    return out


# ------------------------------------------------------------------ a. parity path, one evaluation
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GRIDS))
def test_parity_evaluation_bitwise(gpu, name):
    from uneven_planner_b200 import _lib
    m, params = grid(name), _lib.default_params()
    opt = ctx(gpu, 64, params, m)
    _parity_evaluation(opt, batch(name), params, m)
    opt.close()


@pytest.mark.gpu
@pytest.mark.parametrize("repack", [0, 1])
def test_parity_evaluation_bitwise_double_grid(gpu, repack):
    """`wide` as a double grid through ualm_set_map_f64: read as doubles (repack 0), or rounded to the float grid on the way (1)"""
    from uneven_planner_b200 import _lib, maps
    base, params = grid("wide"), _lib.default_params()
    rng = np.random.default_rng(9)
    c64 = base.cells.astype(np.float64) * (1.0 + 1e-6 * rng.standard_normal(base.cells.shape))      # not float32 values, and other float32 values once rounded
    m64 = maps.UnevenMapData(base.geom, base.cells, "wide-f64", cells64=c64)
    seen = m64 if repack == 0 else maps.UnevenMapData(base.geom, c64.astype(np.float32), "wide-repacked")
    opt = gpu.BatchALMTrajOpt().init(params).set_environment(m64, repack_to_float=bool(repack))
    ev = _parity_evaluation(opt, batch("wide"), params, seen)
    opt.close()
    plain = ctx(gpu, 64, params, base)
    plain.upload(batch("wide"))
    xs, lam, mu, scx, sfx = workloads._inputs(batch("wide"), [params.int_K] * batch("wide").B, seed=0)
    assert not np.array_equal(plain.eval_batch(xs, lam, mu, scx, sfx, rho=workloads.RHO)["grad"], ev["grad"])      # the double grid's own values were read
    plain.close()


# ------------------------------------------------------------------ b, e. parity path, whole solves, their scan and check
@pytest.mark.gpu
@pytest.mark.parametrize("name,pname", [(n, "hill") for n in SMALL] + [("coarse", "forest")])
def test_parity_solves_scan_and_check_match_oracle(gpu, name, pname):
    import pyoracle as po
    from workloads import _assert_solve_parity
    from uneven_planner_b200 import configs
    m, params, pb = grid(name), configs.params_for(pname), batch(name)
    opt = ctx(gpu, 64, params, m)
    out = opt.optimize(pb)
    ores = po.solve_batch(po.params_from(params), po.OracleMap(m), pb, threads=THREADS)
    _assert_solve_parity(pb, out[0], out[1], out[2], ores)
    assert pname != "hill" or sum(1 for r in out[0] if r.ret_code == 0) >= N_GEN // 2
    _scan_and_check(opt, m, params, pb, out)
    opt.close()


# ------------------------------------------------------------------ c. throughput path, one evaluation
def _tiny():
    """7 cells in y: below the 8 x 8 x 8 TMA tile, so no tensor map is kept and UALM_TP_TMA=1 reads through the direct gather.  The
    arcs are centred off y = 0: with an odd cell count that line is a row of cell centres, where the interpolated gradient jumps and
    two implementations may each take either side"""
    from uneven_planner_b200 import _lib, maps
    geom = _lib.map_geometry(10.0, 0.35, 0.05, 0.1)
    assert tuple(geom.voxel_num) == (200, 7, 64)
    m = maps.synthetic_terrain("hills", seed=206, geom=geom)
    pb = cat([_arc_problem(12, 20, radius=40.0, arc=0.1, start=-0.5 * np.pi - 0.05, centre=(0.0, 40.011)),     # along x, |y| < 0.07
                      _arc_problem(3, 5, radius=0.12, arc=1.5 * np.pi, centre=(0.013, 0.011))])
    return m, pb.select(np.repeat(np.arange(pb.B), 2))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GRIDS) + ["tiny"])
@pytest.mark.parametrize("prec", TP)
def test_throughput_evaluation_per_block_and_tile_staging(gpu, capfd, prec, name):
    """against the oracle block by block; TMA-staged tiles (partial last tiles on `coarse` and `fine_yaw`) against the direct
    gather bit for bit"""
    from uneven_planner_b200 import _lib
    m, pb = _tiny() if name == "tiny" else (grid(name), batch(name))
    pb = pb if name == "tiny" else pb.select(np.repeat(np.arange(pb.B), 2))      # each at its guess (even) and perturbed (odd)
    params = _lib.default_params()
    Ks = [params.int_K] * pb.B
    inputs = workloads._inputs(pb, Ks, seed=3)
    want = workloads._oracle(pb, [params] * pb.B, [m] * pb.B, Ks, inputs)
    direct, again = workloads.run_tp(gpu, pb, params, m, prec, inputs)
    capfd.readouterr()
    tma, _ = workloads.run_tp(gpu, pb, params, m, prec, inputs, env={"UALM_TP_TMA": "1", "UALM_DEBUG": "1"})
    log = capfd.readouterr().err
    assert ("tensor map unavailable, TMA staging off" if name == "tiny" else "tensor map encoded, TMA staging on") in log, log
    for i in range(pb.B):
        assert workloads._same(direct[i], again[i]) and workloads._same(direct[i], tma[i]), i
    workloads._check(workloads.block_errors(pb, direct, want, Ks), prec, (prec, name))


# ------------------------------------------------------------------ d, e. throughput path, whole solves, their scan and check
@pytest.mark.gpu
@pytest.mark.parametrize("name", SMALL)
@pytest.mark.parametrize("prec", TP)
def test_throughput_solves_scan_and_check(gpu, prec, name):
    import pyoracle as po
    from uneven_planner_b200 import _lib
    m, params = grid(name), _lib.default_params()
    pb = cat([batch(name), generated(m, 64, GRIDS[name][5] + 50)])
    opt = ctx(gpu, prec, params, m)
    out = opt.optimize(pb)
    res, cxy, cyaw = out
    _, _, ocx, ocy = pb.offsets()
    for i in range(pb.B):
        r = res[i]
        assert r.ret_code in (0, 1, 2) and r.n_evals > 0, (i, r.ret_code, r.n_evals)
        assert np.isfinite(cxy[ocx[i]:ocx[i + 1]]).all() and np.isfinite(cyaw[ocy[i]:ocy[i + 1]]).all() and cxy[ocx[i]:ocx[i + 1]].any(), i
        assert np.isfinite([r.inner_cost, r.jerk_cost, r.total_T, r.piece_T_xy, r.piece_T_yaw]).all() and r.piece_T_xy > 0, i
    _scan_and_check(opt, m, params, pb, out)
    # submitted and polled to the end, the batch is the waited one byte for byte
    t = opt.submit(pb, depth=2)
    polled = opt.outputs(pb)
    left, spins = pb.B, 0
    while left > 0 and spins < 600:
        _, left = opt.poll(t, polled, wait_ms=500.0)
        spins += 1
    assert left == 0, "the submitted batch did not finish"
    assert same_pieces(pieces(pb, polled), pieces(pb, out)) and same_pieces(pieces(pb, _wait(opt, t, pb)), pieces(pb, out))
    opt.close()
    # the converged share of the generated problems against the oracle's on the same problems: test_population_matches_oracle's 0.06
    # on 256 problems is 2.3 standard deviations of a share near 0.8; on these 88 that is 0.10, the bound here.  Worst measured over
    # the four grids and both precisions on an H100 (80 GB HBM3, 700 W): 0.091 (wide, precision 32)
    gen = np.r_[0:N_GEN, N_GEN + len(BATCH_CASES):pb.B]
    ores = po.solve_batch(po.params_from(params), po.OracleMap(m), pb, threads=THREADS, idx=gen)
    rc = np.array([res[i].ret_code for i in gen]); orc = np.array([r[0].ret_code for r in ores])
    assert abs((rc == 0).mean() - (orc == 0).mean()) <= 0.10, ((rc == 0).mean(), (orc == 0).mean())


# ------------------------------------------------------------------ f. the builder on the device
BUILD_GEOMS = {"wide4": (4.0, 2.0, 0.05, 0.1), "tall4": (2.0, 4.0, 0.05, 0.1), "fine_yaw4": (3.1, 2.0, 0.04, 0.05)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BUILD_GEOMS) + ["site"])
def test_device_builder_equals_host_builder(gpu, name):
    """the cloud of tests/test_gpu_map_window.py: its empty patch around (-1, 1) is off the diagonal, at the +y edge of the 4 m x 2 m
    grid and the -x edge of the 2 m x 4 m one"""
    from uneven_planner_b200 import _lib, maps
    if name == "site":
        geom, pts = geometry("site"), _cloud(1200000, 10.3, 4)
    else:
        geom, pts = _lib.map_geometry(*BUILD_GEOMS[name]), _cloud(60000, 2.3, 4)
    host = maps.build_from_cloud(pts, geom)
    o = gpu.BatchALMTrajOpt()
    dev, ms = o.build_map(pts, geom)
    o.close()
    assert ms > 0.0 and dev.shape == tuple(geom.voxel_num)
    assert np.array_equal(bits(dev.cells, np.float32), bits(host.cells, np.float32))
    assert host.cells[..., 1].std() > 0 and host.cells[..., 2].std() > 0


# ------------------------------------------------------------------ g. windows
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["wide", "tall"])
def test_windows_on_a_rectangle(gpu, name):
    """each window, then one evaluation on the parity path against the oracle on the grid spliced in numpy, bit for bit, of a batch
    in which some problem reads every box (so each splice changes the oracle's constraint values); boxes one cell over each edge are refused
    and leave the grid as it is"""
    from uneven_planner_b200 import _lib, maps
    base, params = grid(name), _lib.default_params()
    pb = cat([batch(name)] + window_cases(base.geom))
    X, Y, W = base.shape
    other = window_source(name)
    opt = ctx(gpu, 64, params, base)
    ref = base
    seen = _parity_evaluation(opt, pb, params, ref)["oracle_gx"]
    for box in _boxes(X, Y):
        ix0, iy0, nx, ny = box
        win = other.cells[ix0:ix0 + nx, iy0:iy0 + ny]
        opt.update_environment_window(ix0, iy0, win)
        ref = splice(ref, win, box)
        now = _parity_evaluation(opt, pb, params, ref)["oracle_gx"]
        assert now != seen, box
        seen = now
    L = _lib.lib()
    cp = np.ascontiguousarray(other.cells).ctypes.data_as(C.POINTER(C.c_float))
    for box in [(X - 3, 0, 4, 2), (0, Y - 3, 2, 4), (0, 0, X + 1, 1), (0, 0, 1, Y + 1), (X, 0, 1, 1), (0, Y, 1, 1),
                (Y, 0, 1, 1) if Y > X else (0, X, 1, 1), (-1, 0, 2, 2), (0, -1, 2, 2)]:
        assert L.ualm_update_map_window(opt.h, *box, cp) == _lib.UALM_EINVAL, box
    assert _parity_evaluation(opt, pb, params, ref)["oracle_gx"] == seen
    opt.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["wide4", "tall4"])
@pytest.mark.parametrize("prec", PRECISIONS)
def test_cloud_windows_on_a_rectangle(gpu, prec, name):
    """windows built on the device from a cloud: cells_out is the box of a whole-grid build, and the solves after each window, of a
    batch in which some problem reads every box, change and equal a lone solve on the grid spliced in numpy"""
    from uneven_planner_b200 import _lib, maps
    geom = _lib.map_geometry(*BUILD_GEOMS[name])
    X, Y, W = geom.voxel_num
    pts = _cloud(60000, 2.3, 4)
    base = maps.build_from_cloud(_cloud(60000, 2.3, 5, hole=False), geom, name="base")
    o = gpu.BatchALMTrajOpt()
    full, _ = o.build_map(pts, geom)
    o.close()
    pb = cat([generated(base, 12, 7)] + window_cases(geom))
    opt = ctx(gpu, prec, _lib.default_params(), base)
    ref = base
    seen = pieces(pb, opt.optimize(pb))
    for box in _boxes(X, Y):
        ix0, iy0, nx, ny = box
        cells, ms = opt.update_environment_window_from_cloud(pts, *box)
        assert ms > 0.0 and cells.shape == (nx, ny, W, 4)
        assert np.array_equal(bits(cells, np.float32), bits(full.cells[ix0:ix0 + nx, iy0:iy0 + ny], np.float32)), box
        ref = splice(ref, cells, box)
        now = pieces(pb, opt.optimize(pb))
        assert same_pieces(now, alone(ctx(gpu, prec, _lib.default_params(), ref), pb)[0]) and not same_pieces(now, seen), box
        seen = now
    assert _refuses_windows_outside(opt, X, Y, pts)
    assert same_pieces(pieces(pb, opt.optimize(pb)), seen)
    opt.close()


def _refuses_windows_outside(opt, X, Y, pts):
    from uneven_planner_b200 import _lib
    fp = C.POINTER(C.c_float)
    pp = np.ascontiguousarray(pts, np.float32).ctypes.data_as(fp)
    return all(_lib.lib().ualm_update_map_window_from_cloud(opt.h, pp, len(pts), *box, 0.2, 0.1, 0.1, 2, None, None) == _lib.UALM_EINVAL
               for box in [(X - 3, 0, 4, 2), (0, Y - 3, 2, 4), (0, max(X, Y) - 1, 1, 1) if X > Y else (max(X, Y) - 1, 0, 1, 1)])


# ------------------------------------------------------------------ h. the geometry changes while batches are in flight
@functools.lru_cache(maxsize=None)
def _square():
    """the 10 m square and a batch on it large enough to be in flight while the grid is replaced twice"""
    from uneven_planner_b200 import maps, problems
    m = maps.stand_in_terrain("hill")
    return m, problems.generate(m, 1024, seed=0)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,tma", [(64, 0), (65, 0), (32, 0), (65, 1), (32, 1)])
def test_geometry_change_in_flight(gpu, prec, tma):
    """A on the 10 m square, ualm_update_map to `wide` while A runs, B, a window checked against `wide`'s cell counts, then
    `fine_yaw`, C: each batch is what it is alone on a fresh context of its grid, and the scan of A's lane still reads the square"""
    from uneven_planner_b200 import _lib, maps
    env = {"UALM_TP_TMA": "1"} if tma else {}
    sq, A = _square()
    wide, fine = grid("wide"), grid("fine_yaw")
    B, Cb = batch("wide"), batch("fine_yaw")
    L = _lib.lib()
    opt = ctx(gpu, prec, _lib.default_params(), sq, env=env)
    ta = opt.submit(A, depth=3)
    assert opt.poll(ta, opt.outputs(A), 0.0)[1] > 0
    opt.update_environment(wide)
    tb = opt.submit(B, depth=3)
    # (0, 150): inside the square's 200 x 200, outside wide's 240 x 120 in y; (236, 40): the other way round, where border_x runs
    other = maps.synthetic_terrain("hills", seed=299, geom=wide.geom)
    win = np.ascontiguousarray(other.cells[236:240, 40:80])
    wp = win.ctypes.data_as(C.POINTER(C.c_float))
    assert L.ualm_update_map_window(opt.h, 0, 150, 4, 40, wp) == _lib.UALM_EINVAL
    assert L.ualm_update_map_window(opt.h, 236, 40, 4, 40, wp) == _lib.UALM_OK
    tw = opt.submit(B, depth=4)
    opt.update_environment(fine)
    tc = opt.submit(Cb, depth=4)
    got = {k: pieces(pb, _wait(opt, t, pb)) for k, t, pb in (("a", ta, A), ("b", tb, B), ("w", tw, B), ("c", tc, Cb))}
    opt.select_lane(ta)
    opt.pb = A
    scan_a = opt.feasibility(DT)
    opt.close()
    ref_a, ref_scan = alone(ctx(gpu, prec, _lib.default_params(), sq, env=env), A, feas=True)
    assert same_pieces(got["a"], ref_a) and np.array_equal(bits(scan_a), bits(ref_scan))
    assert same_pieces(got["b"], alone(ctx(gpu, prec, _lib.default_params(), wide, env=env), B)[0])
    assert same_pieces(got["w"], alone(ctx(gpu, prec, _lib.default_params(), splice(wide, win, (236, 40, 4, 40)), env=env), B)[0])
    assert same_pieces(got["c"], alone(ctx(gpu, prec, _lib.default_params(), fine, env=env), Cb)[0])
    assert not same_pieces(got["b"], got["w"])          # border_x runs through the window


# ------------------------------------------------------------------ i. environments of different geometry in one context
@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECISIONS)
def test_environments_of_different_geometry(gpu, prec):
    from uneven_planner_b200 import _lib, problems
    sq = _square()[0]
    grids = [sq, grid("wide"), grid("tall"), grid("coarse")]
    subs = [generated(sq, N_GEN, 77), batch("wide"), batch("tall"), batch("coarse")]
    params = _lib.default_params()
    cat = problems.concat(subs, range(4))
    perm = np.random.default_rng(5).permutation(cat.B)
    mixed = cat.select(perm)
    first = np.concatenate([[0], np.cumsum([s.B for s in subs])])
    opt = gpu.BatchALMTrajOpt(precision=prec)
    for e in range(4):
        opt.init(params, env=e).set_environment(grids[e], env=e)
    solved = opt.optimize(mixed)
    waited = _wait(opt, opt.submit(mixed, depth=2), mixed)
    assert same_pieces(pieces(mixed, solved), pieces(mixed, waited))
    chk = opt.check_results(mixed, solved, t_from=1.0)
    opt.close()
    got = pieces(mixed, solved)
    for e in range(4):
        o = ctx(gpu, prec, params, grids[e])
        out = o.optimize(subs[e])
        alone_chk = o.check_results(subs[e], out, t_from=1.0)
        o.close()
        alone = pieces(subs[e], out)
        rows = [i for i, q in enumerate(perm) if first[e] <= q < first[e + 1]]
        assert len(rows) == subs[e].B
        for i in rows:
            j = int(perm[i] - first[e])
            assert same_pieces([got[i]], [alone[j]]), (e, i, j)
            assert np.array_equal(bits(chk[i]), bits(alone_chk[j])), (e, i, j)
