"""Grids at any origin on the device, and moving an environment's grid by whole cells while batches are in flight (include/ualm.h,
ualm_map_geometry_at, ualm_shift_map / ualm_shift_map_from_cloud), at precision 64, 32 and 65.

Every grid of the shift tests is a slice of one "world" array: the `hills` terrain on a 20 m x 20 m geometry (400 x 400 x 64) with
the hill stand-in (the grid of the golden files) pasted into its middle.  The grid at cell offset (ox, oy) is world[ox:ox + 200,
oy:oy + 200], so the expected grid after a shift is a numpy slice, its geometry maps.shift_geometry of the previous one, and the strip
cells come from the world array.  Off-centre grids are the grids of tests/test_map_geometry.py (and the 10 m square) on the same extent
centred elsewhere (ualm_map_geometry_at), with the problems and hand-placed cases of tests/test_gpu_map_geometry.py moved along.

What each comparison is:
  * off-centre, parity path: one evaluation, initScaling, whole solves (float grid; the double grid with and without repacking), the
    post-solve scan and ualm_check_trajectories against the CPU oracle, bit for bit;
  * off-centre, throughput path: one evaluation against the oracle block by block with the tolerances of tests/test_gpu_tp_shapes.py,
    TMA-staged tiles against the direct gather bit for bit;
  * shifts: byte for byte against the same batch solved alone on a fresh context bound to the expected grid with ualm_set_map; cloud
    strips as uint32 against the box of a whole-grid device build with the moved geometry."""
import collections
import functools
import struct
import subprocess

import numpy as np
import pytest

import workloads
from harness import alone, bits, build_driver, cat, ctx, gpu, pending, pieces, same_pieces  # noqa: F401
from workloads import BATCH_CASES, GRIDS, THREADS, _cloud, _parity_evaluation, _scan_and_check, generated, grid, hand_cases


pytestmark = pytest.mark.gpu
PRECISIONS = [64, 32, 65]
TP = [65, 32]
DT = 0.01
X0 = Y0 = 100                 # the hill stand-in's cell offset in the world


def _moved(pb, cx, cy):
    """batch pb with every position moved by (cx, cy)"""
    import copy
    out = copy.deepcopy(pb)
    out.bnd[:, [0, 6]] += cx
    out.bnd[:, [1, 7]] += cy
    out.inner_xy[0::2] += cx
    out.inner_xy[1::2] += cy
    return out


def _centre(g):
    return (g.origin[0] + g.max_boundary[0]) / 2, (g.origin[1] + g.max_boundary[1]) / 2


def _batch(m, n, seed):
    """n generated problems over grid m, then the hand-placed cases of tests/test_gpu_map_geometry.py moved to m's centre: paths
    leaving through all four sides, arcs in the last cell column in x and in y, an arc over the yaw seam"""
    from uneven_planner_b200 import _lib
    g = m.geom
    ext = (g.max_boundary[0] - g.origin[0], g.max_boundary[1] - g.origin[1])
    centred = _lib.map_geometry(ext[0], ext[1], g.xy_resolution, g.yaw_resolution)
    hc = hand_cases(centred)
    return cat([generated(m, n, seed)] + [_moved(hc[k], *_centre(g)) for k in BATCH_CASES])


# ------------------------------------------------------------------ off-centre grids against the oracle
OFF = {"square": (10.0, 10.0, 0.05, 0.1), "wide": GRIDS["wide"][:4], "fine_yaw": GRIDS["fine_yaw"][:4]}


@functools.lru_cache(maxsize=None)
def off_grid(name, cx, cy):
    from uneven_planner_b200 import _lib, maps
    base = maps.stand_in_terrain("hill") if name == "square" else grid(name)
    return maps.UnevenMapData(_lib.map_geometry_at(*OFF[name], cx, cy), base.cells, "%s@%g,%g" % (name, cx, cy))


@functools.lru_cache(maxsize=None)
def off_batch(name, cx, cy):
    return _batch(off_grid(name, cx, cy), 24, 7)


@pytest.mark.parametrize("centre", [(31.4, -17.25), (-48.6, 23.05)])
@pytest.mark.parametrize("name", ["square", "wide", "fine_yaw"])
def test_off_centre_parity_evaluation_solves_scan_and_check(gpu, name, centre):
    import pyoracle as po
    from workloads import _assert_solve_parity
    from uneven_planner_b200 import _lib
    m, params, pb = off_grid(name, *centre), _lib.default_params(), off_batch(name, *centre)
    opt = gpu.BatchALMTrajOpt(precision=64).init(params).set_environment(m)
    _parity_evaluation(opt, pb, params, m)
    out = opt.optimize(pb)
    ores = po.solve_batch(po.params_from(params), po.OracleMap(m), pb, threads=THREADS)
    _assert_solve_parity(pb, out[0], out[1], out[2], ores)
    assert sum(1 for r in out[0] if r.ret_code == 0) >= 12
    _scan_and_check(opt, m, params, pb, out)
    opt.close()


@pytest.mark.parametrize("repack", [0, 1])
def test_off_centre_parity_evaluation_double_grid(gpu, repack):
    from uneven_planner_b200 import _lib, maps
    base, params = off_grid("wide", 31.4, -17.25), _lib.default_params()
    rng = np.random.default_rng(9)
    c64 = base.cells.astype(np.float64) * (1.0 + 1e-6 * rng.standard_normal(base.cells.shape))
    m64 = maps.UnevenMapData(base.geom, base.cells, "wide-f64", cells64=c64)
    seen = m64 if repack == 0 else maps.UnevenMapData(base.geom, c64.astype(np.float32), "wide-repacked")
    opt = gpu.BatchALMTrajOpt().init(params).set_environment(m64, repack_to_float=bool(repack))
    _parity_evaluation(opt, off_batch("wide", 31.4, -17.25), params, seen)
    opt.close()


# the throughput path's evaluation error against |origin| (printed; DESIGN 6a): its rounding grows with |x|, |y| (float sample positions
# at precision 32; at 65 the velocities are differences of coefficients that carry the positions).  test_gpu_tp_shapes.py's tolerances
# are asserted for every block but the ones that exceed them at that origin, measured on an H100: at 65 the hx cancellation block from
# 30 m on (1.7e-9 at |origin| 34 m, 5.2e-9 at 112 m, 1.5e-8 at 335 m against 1e-9), at 32 grad_xy at 335 m (1.8e-4 against 1e-4).  Those
# blocks are held to twice their measured error there instead, so a regression in them stays visible
TP_ORIGINS = [0.0, 30.0, 100.0, 300.0]
TP_EXCEEDS = {(65, 30.0): {"hx_cancel": 3.5e-9}, (65, 100.0): {"hx_cancel": 1.1e-8}, (65, 300.0): {"hx_cancel": 3.1e-8},
              (32, 300.0): {"grad_xy": 3.7e-4}}


@pytest.mark.parametrize("r", TP_ORIGINS)
@pytest.mark.parametrize("prec", TP)
def test_off_centre_throughput_evaluation_per_block(gpu, capfd, prec, r):
    from uneven_planner_b200 import _lib
    c = (r, -0.5 * r)
    m, pb = off_grid("square", *c), off_batch("square", *c)
    pb = pb.select(np.repeat(np.arange(pb.B), 2))
    params = _lib.default_params()
    Ks = [params.int_K] * pb.B
    inputs = workloads._inputs(pb, Ks, seed=3)
    want = workloads._oracle(pb, [params] * pb.B, [m] * pb.B, Ks, inputs)
    direct, again = workloads.run_tp(gpu, pb, params, m, prec, inputs)
    tma, _ = workloads.run_tp(gpu, pb, params, m, prec, inputs, env={"UALM_TP_TMA": "1"})
    for i in range(pb.B):
        assert workloads._same(direct[i], again[i]) and workloads._same(direct[i], tma[i]), i
    worst = workloads.block_errors(pb, direct, want, Ks)
    with capfd.disabled():
        print("\nTP_ORIGIN_ERR prec=%d |origin|=%g %s" % (prec, float(np.hypot(*c)), " ".join("%s=%.2e" % (k, v[0]) for k, v in sorted(worst.items()))))
    far = TP_EXCEEDS.get((prec, r), {})
    workloads._check({k: v for k, v in worst.items() if k not in far}, prec, (prec, c))
    assert all(worst[k][0] <= bound for k, bound in far.items()), (prec, c, {k: worst[k] for k in far})


# ------------------------------------------------------------------ the world and its slices
@pytest.fixture(scope="module")
def world(built):
    from uneven_planner_b200 import _lib, configs, maps, problems
    g0 = maps.stand_in_terrain("hill")
    w = maps.synthetic_terrain("hills", seed=301, geom=_lib.map_geometry(20.0, 20.0, 0.05, 0.1)).cells
    w[X0:X0 + 200, Y0:Y0 + 200] = g0.cells
    kw = configs.gen_kwargs("hill")
    return dict(cells=w, g0=g0, params=configs.params_for("hill"), kw=kw, bench=problems.generate(g0, 1024, seed=0, **kw))


def _slice(world, ox, oy, geom):
    from uneven_planner_b200 import maps
    return maps.UnevenMapData(geom, np.ascontiguousarray(world["cells"][ox:ox + 200, oy:oy + 200]), "slice%d,%d" % (ox, oy))


def _strips(m_new, geom_old, dx, dy):
    """the cells ualm_shift_map takes for moving geom_old by (dx, dy) to the grid m_new: its boxes A then B, as one list"""
    from uneven_planner_b200 import maps
    return [m_new.cells[ix0:ix0 + nx, iy0:iy0 + ny] for ix0, iy0, nx, ny in maps.shift_boxes(geom_old, dx, dy)]


def _start(d):
    """the start offset on one axis from which a shift by d stays inside the 400-cell world"""
    return 100 if abs(d) <= 100 else (0 if d > 0 else 200)


SHIFTS = [(1, 0), (-1, 0), (0, 1), (0, -1), (9, 0), (0, -13), (4, 6), (-5, 3), (2, -7), (-6, -2), (199, 0), (0, -199), (-199, 150),
          (200, 0), (0, -200), (200, -200)]


@pytest.mark.parametrize("precision", PRECISIONS)
def test_host_cells_shift_equals_the_world_slice(gpu, world, precision):
    from uneven_planner_b200 import maps, problems
    opt = gpu.BatchALMTrajOpt(precision=precision).init(world["params"])
    base = world["g0"].geom
    for dx, dy in SHIFTS:
        ox, oy = _start(dx), _start(dy)
        g_old = maps.shift_geometry(base, ox - X0, oy - Y0)
        old = _slice(world, ox, oy, g_old)
        new = _slice(world, ox + dx, oy + dy, maps.shift_geometry(g_old, dx, dy))
        opt.update_environment(old)
        g = opt.shift_environment(dx, dy, _strips(new, g_old, dx, dy))
        assert bytes(g) == bytes(new.geom)
        pb = _batch(new, 24, 40 + abs(dx) + 3 * abs(dy))
        got = pieces(pb, opt.optimize(pb))
        assert same_pieces(got, alone(ctx(gpu, precision, world["params"], new), pb)[0]), (dx, dy)
        if abs(dx) < 150 and abs(dy) < 150:        # the grid moved under the problems: a lone solve on the old grid differs
            assert not same_pieces(got, alone(ctx(gpu, precision, world["params"], old), pb)[0]), (dx, dy)
    opt.close()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_batch_in_flight_keeps_its_grid_and_geometry(gpu, world, golden, precision):
    from uneven_planner_b200 import maps, problems
    g0 = world["g0"]
    gold = golden("hill", g0)
    gold_pb = problems.generate(g0, int(gold["B"]), seed=int(gold["seed"]), **world["kw"])
    A = problems.concat([gold_pb, world["bench"]], [0, 0]) if precision == 64 else world["bench"]
    dx, dy = 7, -4
    new = _slice(world, X0 + dx, Y0 + dy, maps.shift_geometry(g0.geom, dx, dy))
    B = _batch(new, 96, 5)
    opt = ctx(gpu, precision, world["params"], g0)
    ta = opt.submit(A, depth=2)
    assert pending(opt, ta, A) > 0
    opt.shift_environment(dx, dy, _strips(new, g0.geom, dx, dy))
    assert pending(opt, ta, A) > 0               # the host-cells shift returned while the batch ran, on both paths
    tb = opt.submit(B, depth=2)
    got_a, got_b = pieces(A, opt.wait(ta)), pieces(B, opt.wait(tb))
    opt.close()
    assert same_pieces(got_a, alone(ctx(gpu, precision, world["params"], g0), A)[0])
    assert same_pieces(got_b, alone(ctx(gpu, precision, world["params"], new), B)[0])
    if precision == 64:
        n = gold_pb.B
        rec = [np.frombuffer(p[0], dtype=np.int32, count=3) for p in got_a[:n]]
        assert [int(r[0]) for r in rec] == [int(x) for x in gold["ret_code"]]
        assert [int(r[2]) for r in rec] == [int(x) for x in gold["n_evals"]]
        assert np.array_equal(np.concatenate([p[1] for p in got_a[:n]]), gold["c_xy"])
        assert np.array_equal(np.concatenate([p[2] for p in got_a[:n]]), gold["c_yaw"])


@pytest.mark.parametrize("precision", PRECISIONS)
def test_repeated_shifts_in_flight_follow_a_curve(gpu, world, precision):
    """20 shifts of 1 to 3 cells along a curve with batches in flight end on the expected slice and geometry; free device memory
    stays within one grid of the start"""
    import torch
    from uneven_planner_b200 import maps
    depth = 3 if precision == 64 else 8
    g0 = world["g0"]
    pb = _batch(g0, 64, 3)
    opt = ctx(gpu, precision, world["params"], g0)

    def fill():
        for t in [opt.submit(pb, depth=depth) for _ in range(depth)]:
            opt.wait(t)
    fill()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    ox, oy, geom = X0, Y0, g0.geom
    q = collections.deque()
    for k in range(20):
        a = 0.15 * k
        dx, dy = int(round(3 * np.cos(a))), int(round(-3 * np.sin(a))) or 1
        new = _slice(world, ox + dx, oy + dy, maps.shift_geometry(geom, dx, dy))
        g = opt.shift_environment(dx, dy, _strips(new, geom, dx, dy))
        ox, oy, geom = ox + dx, oy + dy, new.geom
        assert bytes(g) == bytes(geom)
        if len(q) == depth:
            opt.wait(q.popleft())
        q.append(opt.submit(pb, depth=depth))
    while q:
        opt.wait(q.popleft())
    fill()
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    end = _slice(world, ox, oy, geom)
    last = _batch(end, 48, 9)
    got = pieces(last, opt.optimize(last))
    opt.close()
    assert (ox, oy) != (X0, Y0)
    assert free0 - free1 <= g0.cells.nbytes, (free0, free1)
    assert same_pieces(got, alone(ctx(gpu, precision, world["params"], end), last)[0])


@pytest.mark.parametrize("precision", PRECISIONS)
def test_four_environments_only_the_shifted_one_changes(gpu, world, precision):
    from uneven_planner_b200 import configs, maps, problems
    names = ["hill", "desert", "volcano", "forest"]
    offs = [(X0, Y0), (60, 140), (150, 40), (30, 30)]
    grids = [_slice(world, ox, oy, maps.shift_geometry(world["g0"].geom, ox - X0, oy - Y0)) for ox, oy in offs]
    params = [configs.params_for(n) for n in names]
    subs = [_batch(g, 40, 11 + e) for e, g in enumerate(grids)]
    mixed = problems.concat(subs, range(4))
    dx, dy = -6, 5
    new2 = _slice(world, offs[2][0] + dx, offs[2][1] + dy, maps.shift_geometry(grids[2].geom, dx, dy))
    opt = gpu.BatchALMTrajOpt(precision=precision)
    for e in range(4):
        opt.init(params[e], env=e).set_environment(grids[e], env=e)
    t1 = opt.submit(mixed, depth=2)
    opt.shift_environment(dx, dy, _strips(new2, grids[2].geom, dx, dy), env=2)
    t2 = opt.submit(mixed, depth=2)
    first, second = pieces(mixed, opt.wait(t1)), pieces(mixed, opt.wait(t2))
    opt.close()

    def alone(e, grid):
        o = gpu.BatchALMTrajOpt(precision=precision).init(params[e]).set_environment(grid)
        out = pieces(subs[e], o.optimize(subs[e]))
        o.close()
        return out
    ref = [alone(e, grids[e]) for e in range(4)]
    ref2 = alone(2, new2)
    o = 0
    for e in range(4):
        n = subs[e].B
        assert same_pieces(first[o:o + n], ref[e]), e
        assert same_pieces(second[o:o + n], ref2 if e == 2 else ref[e]), e
        o += n
    assert not same_pieces(ref[2], ref2)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_refused_shifts_keep_the_grid(gpu, world, precision):
    import ctypes as C
    from uneven_planner_b200 import _lib, maps
    L = _lib.lib()
    fp = C.POINTER(C.c_float)
    g0 = world["g0"]
    pb = _batch(g0, 32, 2)
    opt = ctx(gpu, precision, world["params"], g0)
    before = pieces(pb, opt.optimize(pb))
    cells = np.ascontiguousarray(g0.cells)
    cp = cells.ctypes.data_as(fp)
    pts = np.zeros((4, 3), np.float32)
    pp = pts.ctypes.data_as(fp)

    def both(dx, dy, h=opt.h):
        return (L.ualm_shift_map(h, dx, dy, cp), L.ualm_shift_map_from_cloud(h, pp, 4, dx, dy, 0.2, 0.1, 0.1, 2, None, None))
    EINVAL, ESTATE = (_lib.UALM_EINVAL,) * 2, (_lib.UALM_ESTATE,) * 2
    assert both(0, 0) == EINVAL
    assert both(1, 0, h=None) == EINVAL
    assert L.ualm_shift_map(opt.h, 1, 0, None) == _lib.UALM_EINVAL
    assert L.ualm_shift_map_from_cloud(opt.h, None, 4, 1, 0, 0.2, 0.1, 0.1, 2, None, None) == _lib.UALM_EINVAL
    assert L.ualm_shift_map_from_cloud(opt.h, pp, -1, 1, 0, 0.2, 0.1, 0.1, 2, None, None) == _lib.UALM_EINVAL
    opt.select_env(1)                                                # no grid bound there
    assert both(1, 0) == ESTATE
    opt.select_env(0)
    assert same_pieces(pieces(pb, opt.optimize(pb)), before)
    opt.close()
    if precision == 64:
        o = ctx(gpu, precision, world["params"], maps.UnevenMapData(g0.geom, g0.cells, "f64", cells64=g0.cells.astype(np.float64)))
        before = pieces(pb, o.optimize(pb))
        assert both(1, 0, h=o.h) == ESTATE
        assert same_pieces(pieces(pb, o.optimize(pb)), before)
        o.close()


# ------------------------------------------------------------------ the cloud form
@pytest.fixture(scope="module")
def cloud(gpu):
    """a seeded surface over [-5, 5]^2 with an empty patch around (-1, 1), and a 4 m grid centred at (2.5, 0.3) built from it: the
    patch is outside the grid, and a shift by -40 cells in x brings it in through strip A"""
    from uneven_planner_b200 import _lib, maps
    pts = _cloud(200000, 5.0, 4)
    geom = _lib.map_geometry_at(4.0, 4.0, 0.05, 0.1, 2.5, 0.3)
    o = gpu.BatchALMTrajOpt()
    dev, _ = o.build_map(pts, geom)
    o.close()
    host = maps.build_from_cloud(pts, geom)
    return dict(pts=pts, geom=geom, dev=dev, host=host)


def _moved_cells(old, dx, dy, strips, boxes):
    """old's cells moved by (dx, dy) cells in numpy, with `strips` in `boxes`"""
    X, Y = old.shape[:2]
    new = np.full_like(old, np.nan)
    xs, ys = slice(max(0, -dx), min(X, X - dx)), slice(max(0, -dy), min(Y, Y - dy))
    if xs.start < xs.stop and ys.start < ys.stop:
        new[xs, ys] = old[xs.start + dx:xs.stop + dx, ys.start + dy:ys.stop + dy]
    for (ix0, iy0, nx, ny), c in zip(boxes, strips):
        new[ix0:ix0 + nx, iy0:iy0 + ny] = c
    assert not np.isnan(new).any()
    return new


CLOUD_SHIFTS = [(-40, 0), (10, -3), (0, 12), (-3, -5)]


@pytest.mark.parametrize("precision", PRECISIONS)
def test_cloud_shift_strips_and_solve(gpu, world, cloud, precision):
    from uneven_planner_b200 import configs, maps, problems
    assert np.array_equal(bits(cloud["dev"].cells, np.float32), bits(cloud["host"].cells, np.float32))      # off-centre: the builders agree bit for bit
    assert np.count_nonzero(cloud["dev"].cells[..., 1]) > 0.9 * cloud["dev"].cells[..., 1].size
    opt = ctx(gpu, precision, world["params"], cloud["dev"])
    cur = cloud["dev"]
    hole = False
    for dx, dy in CLOUD_SHIFTS:
        g2, strips, ms = opt.shift_environment_from_cloud(cloud["pts"], dx, dy)
        assert ms > 0.0 and bytes(g2) == bytes(maps.shift_geometry(cur.geom, dx, dy))
        o = gpu.BatchALMTrajOpt()
        full, _ = o.build_map(cloud["pts"], g2)
        o.close()
        boxes = maps.shift_boxes(cur.geom, dx, dy)
        for (ix0, iy0, nx, ny), c in zip(boxes, strips):
            assert np.array_equal(bits(c, np.float32), bits(full.cells[ix0:ix0 + nx, iy0:iy0 + ny], np.float32)), (dx, dy)
            hole |= bool(np.all(c[..., 1:] == 0.0, axis=(2, 3)).any())       # cells whose ellipsoids hold no point
        cur = maps.UnevenMapData(g2, _moved_cells(cur.cells, dx, dy, strips, boxes), "moved")
        lo = (g2.origin[0] + 0.5, g2.origin[1] + 0.5)
        hi = (g2.max_boundary[0] - 0.5, g2.max_boundary[1] - 0.5)
        pb = problems.generate(cur, 48, seed=3 + abs(dx) + 7 * abs(dy), lo=lo, hi=hi, min_dist=1.0, **configs.gen_kwargs("hill"))
        got = pieces(pb, opt.optimize(pb))
        assert same_pieces(got, alone(ctx(gpu, precision, world["params"], cur), pb)[0]), (dx, dy)
    assert hole                                                         # the first strip covered the empty patch
    opt.close()


FAR = (31.4, -17.25)          # a grid centre whose crop box [c - 10, c + 10]^2 excludes the world origin


@pytest.fixture(scope="module")
def far(gpu):
    """a 4 m grid centred at FAR and a seeded surface around it reaching 3.5 m each way, so that shifts of up to 1.5 m stay on it"""
    from workloads import _cloud_at
    from uneven_planner_b200 import _lib
    return dict(pts=_cloud_at(*FAR, n=120000, half=3.5, seed=2), geom=_lib.map_geometry_at(4.0, 4.0, 0.05, 0.1, *FAR))


def test_device_builders_crop_about_the_grid_centre_far_from_the_origin(gpu, world, far):
    """every device cloud builder on the grid centred at FAR: ualm_map_build_device, ualm_update_map_from_cloud and the window cloud
    form give the host builder's cells bit for bit, and those are built from the cloud (the crop box about the world origin drops it
    all, and every cell then takes the "no points" branch)"""
    from uneven_planner_b200 import maps
    pts, geom = far["pts"], far["geom"]
    host = maps.build_from_cloud(pts, geom)
    assert np.count_nonzero(host.cells[..., 1]) > 0.9 * host.cells[..., 1].size
    o = gpu.BatchALMTrajOpt()
    dev, _ = o.build_map(pts, geom)
    o.close()
    assert np.array_equal(bits(dev.cells, np.float32), bits(host.cells, np.float32))
    opt = ctx(gpu, 32, world["params"], world["g0"])
    upd, _ = opt.update_environment_from_cloud(pts, geom)
    assert np.array_equal(bits(upd.cells, np.float32), bits(host.cells, np.float32))
    box = (10, 25, 30, 20)
    win, _ = opt.update_environment_window_from_cloud(pts, *box)
    opt.close()
    assert np.array_equal(bits(win, np.float32), bits(host.cells[box[0]:box[0] + box[2], box[1]:box[1] + box[3]], np.float32))


@pytest.mark.parametrize("precision", [64, 32])
def test_cloud_shift_far_from_the_origin(gpu, world, far, precision):
    """shifts from a cloud on the grid centred at FAR: the strips are bit for bit the boxes of the host builder's whole grid with the moved
    geometry, and built from the cloud; later solves equal lone solves on the moved grid"""
    from uneven_planner_b200 import configs, maps, problems
    pts = far["pts"]
    cur = maps.build_from_cloud(pts, far["geom"])
    opt = ctx(gpu, precision, world["params"], cur)
    for dx, dy in [(12, -7), (-30, 4)]:
        g2, strips, _ = opt.shift_environment_from_cloud(pts, dx, dy)
        want = maps.build_from_cloud(pts, g2)
        boxes = maps.shift_boxes(cur.geom, dx, dy)
        for (ix0, iy0, nx, ny), c in zip(boxes, strips):
            assert np.array_equal(bits(c, np.float32), bits(want.cells[ix0:ix0 + nx, iy0:iy0 + ny], np.float32)), (dx, dy)
            assert np.count_nonzero(c[..., 1]) > 0.9 * c[..., 1].size, (dx, dy)
        cur = maps.UnevenMapData(g2, _moved_cells(cur.cells, dx, dy, strips, boxes), "moved")
        lo = (g2.origin[0] + 0.5, g2.origin[1] + 0.5)
        hi = (g2.max_boundary[0] - 0.5, g2.max_boundary[1] - 0.5)
        pb = problems.generate(cur, 32, seed=5 + abs(dx), lo=lo, hi=hi, min_dist=1.0, **configs.gen_kwargs("hill"))
        assert same_pieces(pieces(pb, opt.optimize(pb)), alone(ctx(gpu, precision, world["params"], cur), pb)[0]), (dx, dy)
    opt.close()


def test_cloud_shift_returns_while_a_batch_runs(gpu, world):
    """on the throughput path the cloud form's kernel gets SM slots between the batch's rounds"""
    from uneven_planner_b200 import maps
    g0 = world["g0"]
    A = world["bench"]
    pts = _cloud(100000, 7.0, 6)
    opt = ctx(gpu, 32, world["params"], g0)
    ta = opt.submit(A, depth=2)
    assert pending(opt, ta, A) > 0
    g2, strips, _ = opt.shift_environment_from_cloud(pts, 20, 0)
    assert pending(opt, ta, A) > 0
    got_a = pieces(A, opt.wait(ta))
    opt.close()
    assert same_pieces(got_a, alone(ctx(gpu, 32, world["params"], g0), A)[0])
    assert bytes(g2) == bytes(maps.shift_geometry(g0.geom, 20, 0)) and strips[0].shape == (20, 200, 64, 4)


# ------------------------------------------------------------------ check and replan after a shift
def test_check_and_replan_after_a_shift(gpu, world):
    """a batch solved on the hill grid, whose problems include paths that leave it through the -x side; the grid moves 1.5 m towards
    -x.  ualm_check_trajectories of the held trajectories reads the moved grid (bit for bit tests/check_oracle.cpp with it), and the
    replanned rows solve like lone solves on it"""
    import pyoracle as po
    from check_oracle import check, limits_of
    from uneven_planner_b200 import maps
    g0 = world["g0"]
    params = world["params"]
    pb = _batch(g0, 24, 12)
    dx, dy = -30, 0
    new = _slice(world, X0 + dx, Y0 + dy, maps.shift_geometry(g0.geom, dx, dy))
    opt = ctx(gpu, 64, world["params"], g0)
    out = opt.optimize(pb)
    before = opt.check_results(pb, out)
    opt.shift_environment(dx, dy, _strips(new, g0.geom, dx, dy))
    res, cxy, cyaw = out
    _, _, ocx, ocy = pb.offsets()
    om = po.OracleMap(new)
    got = opt.check_results(pb, out)
    for i in range(pb.B):
        ref = check(om, params.gravity, int(pb.N[i]), int(pb.M[i]), cxy[ocx[i]:ocx[i + 1]], cyaw[ocy[i]:ocy[i + 1]], res[i].piece_T_xy,
                    res[i].piece_T_yaw, DT, 0.0, limits_of(params))
        assert np.array_equal(got[i].view(np.uint64), np.asarray(ref, np.float64).view(np.uint64)), i
    assert any(not np.array_equal(got[i], before[i]) for i in range(pb.B))      # the check read the moved grid
    rows = np.arange(pb.B - len(BATCH_CASES))
    rows = rows[[res[i].ret_code == 0 for i in rows]][:12]
    ticket, rp = opt.submit_replan(pb, out, rows, 0.3)
    got_r = pieces(rp, opt.wait(ticket))
    opt.close()
    rp.env = None
    assert same_pieces(got_r, alone(ctx(gpu, 64, world["params"], new), rp)[0])


# ------------------------------------------------------------------ C++
def test_cpp_shifts_between_submits(gpu, world, tmp_path):
    from uneven_planner_b200 import _lib, maps
    exe = build_driver("map_shift_driver", tmp_path)
    g0 = world["g0"]
    pb = world["bench"].select(np.arange(8))
    dx, dy, dx2, dy2 = 5, -3, -2, 4
    new = _slice(world, X0 + dx, Y0 + dy, maps.shift_geometry(g0.geom, dx, dy))
    strips = np.concatenate([c.ravel() for c in _strips(new, g0.geom, dx, dy)])
    n2 = sum(b[2] * b[3] for b in maps.shift_boxes(g0.geom, dx2, dy2)) * 64 * 4
    pts = _cloud(100000, 5.3, 3)
    case = str(tmp_path / "shift.bin")
    with open(case, "wb") as f:
        f.write(struct.pack("<11i", *g0.shape, pb.B, dx, dy, strips.size, dx2, dy2, n2, len(pts)))
        f.write(g0.cells.tobytes())
        f.write(strips.astype(np.float32).tobytes())
        f.write(np.ascontiguousarray(pts).tobytes())
        for a in (pb.N, pb.M):
            f.write(np.ascontiguousarray(a, np.int32).tobytes())
        for a in (pb.bnd, pb.total_time, pb.inner_xy, pb.inner_yaw):
            f.write(np.ascontiguousarray(a, np.float64).tobytes())
    cloud_out = str(tmp_path / "cloud_strips.bin")
    r = subprocess.run([exe, case, cloud_out], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    opt = gpu.BatchALMTrajOpt().init(_lib.default_params()).set_environment(g0)
    t1 = opt.submit(pb, depth=3)
    opt.shift_environment(dx, dy, strips, env=0)
    t2 = opt.submit(pb, depth=3)
    _, cs, _ = opt.shift_environment_from_cloud(pts, dx2, dy2)
    t3 = opt.submit(pb, depth=3)
    outs = [opt.wait(t1), opt.wait(t2), opt.wait(t3)]
    opt.close()
    assert np.array_equal(np.fromfile(cloud_out, np.uint32), np.concatenate([bits(c, np.float32).ravel() for c in cs]))
    _, _, ocx, _ = pb.offsets()
    want = ["%d %d %d %d %r %r" % (p, i, outs[p][0][i].ret_code, outs[p][0][i].n_evals, float(outs[p][0][i].inner_cost), float(outs[p][1][ocx[i] + 1]))
            for p in range(3) for i in range(pb.B)]
    got = [" ".join(ln.split()[:4] + [repr(float(x)) for x in ln.split()[4:]]) for ln in r.stdout.strip().splitlines()]
    assert got == want
