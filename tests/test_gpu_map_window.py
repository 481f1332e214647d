"""Replacing one box of cell columns of an environment's grid while batches are in flight (include/ualm.h, ualm_update_map_window /
ualm_update_map_window_from_cloud), on both paths.  The new grid is a copy of the current one with the box written over it: inside the
box it holds the given cells, or the cells a whole-grid build of the same cloud produces there, bit for bit; outside, the previous
grid's.  Work launched before a window keeps its grid; every later launch reads the new one.  Grids: the seeded stand-ins of hill (G0)
and desert (G1), solved with the hill parameters; for clouds, the seeded analytic cloud of tests/test_gpu_map_build.py on its 4 m grid."""
import collections
import ctypes as C
import struct
import subprocess

import numpy as np
import pytest

from harness import alone, bits, box_cells, build_driver, ctx, gpu, pending, pieces, same_pieces, splice  # noqa: F401
from workloads import _cloud, hill_desert_world


pytestmark = pytest.mark.gpu
PRECISIONS = [64, 32, 65]
BOX = (60, 80, 40, 40)                # a 2 m x 2 m window of the 10 m grid, where the hill problems run


@pytest.fixture(scope="module")
def world(gpu, golden):
    return hill_desert_world(golden)


def _scan(opt, ticket, pb):
    opt.select_lane(ticket)
    opt.pb = pb
    f = opt.feasibility(0.01)
    opt.select_lane(0)
    return f


# ---- host cells ---------------------------------------------------------------------------------

@pytest.mark.parametrize("precision", PRECISIONS)
def test_host_cells_window_equals_the_spliced_grid(gpu, world, precision):
    """Boxes of G1 spliced into G0 one after the other: each later solve is byte-identical to a lone solve on the grid spliced in numpy.
    Covers a box in the middle, boxes at the grid's edges (ix0 = 0, ix0 + nx = X, iy0 + ny = Y) and a one-column box."""
    g0, g1, pb = world["g0"], world["g1"], world["b"]
    X, Y, _ = g0.shape
    boxes = [BOX, (0, 30, 25, 120), (X - 35, Y - 50, 35, 50), (100, 100, 1, 1)]
    opt = ctx(gpu, precision, world["params"], g0)
    before = pieces(pb, opt.optimize(pb))
    ref = g0
    for k, box in enumerate(boxes):
        opt.update_environment_window(box[0], box[1], box_cells(g1.cells, box))
        ref = splice(ref, box_cells(g1.cells, box), box)
        got = pieces(pb, opt.optimize(pb))
        assert same_pieces(got, alone(ctx(gpu, precision, world["params"], ref), pb)[0]), box
        if k == 0:
            assert not same_pieces(got, before)        # the window is where the problems run
    opt.close()


# ---- clouds -------------------------------------------------------------------------------------


# boxes of the 4 m, 80 x 80 x 64 grid: 2 m x 2 m in the middle, one that covers the empty patch (cells 13..27 x 53..67), one at the edges
CLOUD_BOXES = [(20, 30, 40, 40), (8, 48, 26, 26), (0, 60, 20, 20)]


@pytest.fixture(scope="module")
def small(gpu, world):
    from uneven_planner_b200 import _lib, configs, maps, problems
    geom = _lib.map_geometry(4.0, 4.0, 0.05, 0.1)
    pts = _cloud(60000, 2.3, 0)
    host = maps.build_from_cloud(pts, geom)
    o = gpu.BatchALMTrajOpt()
    dev, _ = o.build_map(pts, geom)
    o.close()
    base = maps.build_from_cloud(_cloud(60000, 2.3, 1, hole=False), geom, name="base")     # the grid the windows go into
    pb = problems.generate(base, 128, seed=3, lo=-1.5, hi=1.5, min_dist=1.0, **configs.gen_kwargs("hill"))
    return dict(geom=geom, pts=pts, host=host, dev=dev, base=base, pb=pb)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_cloud_window_cells_and_solve(gpu, world, small, precision):
    """cells_out is bit for bit the box of a whole-grid build of the same cloud (device and host); a solve after the update equals a
    lone solve on the previous grid with that box spliced in"""
    assert np.array_equal(bits(small["dev"].cells, np.float32), bits(small["host"].cells, np.float32))
    pb = small["pb"]
    opt = ctx(gpu, precision, world["params"], small["base"])
    before = pieces(pb, opt.optimize(pb))
    ref = small["base"]
    for box in CLOUD_BOXES:
        cells, ms = opt.update_environment_window_from_cloud(small["pts"], *box)
        assert ms > 0.0
        assert cells.shape == (box[2], box[3], small["geom"].voxel_num[2], 4)
        assert np.array_equal(bits(cells, np.float32), bits(box_cells(small["dev"].cells, box), np.float32)), box
        assert np.array_equal(bits(cells, np.float32), bits(box_cells(small["host"].cells, box), np.float32)), box
        ref = splice(ref, cells, box)
        got = pieces(pb, opt.optimize(pb))
        assert same_pieces(got, alone(ctx(gpu, precision, world["params"], ref), pb)[0]), box
    assert not same_pieces(got, before)
    # the cells at the empty patch's centre, whose ellipsoids (reach 0.32 m) hold no point, took the "no points" branch (sigma 0, zb 0)
    patch = box_cells(ref.cells, (19, 59, 2, 2))
    assert np.all(patch[..., 1:] == 0.0)
    opt.close()


def test_local_scan_window_matches_the_full_cloud(gpu, world, small):
    """A window built from the cloud cut down to the box plus the ellipsoid's reach agrees with the full cloud's build within float
    rounding (its bin grid starts at the local cloud's minimum, so the mean and covariance sums run in another order): at most 0.02 %
    of the cells beyond 3e-7 relative, as the device build against the reference build"""
    g = small["geom"]
    pts = small["pts"]
    margin = 0.2 + 0.12 + 0.2              # box_r + the 0.12 m forward shift, and the empty patch's half width for the nearest point
    opt = ctx(gpu, 64, world["params"], small["base"])
    for box in CLOUD_BOXES:
        ix0, iy0, nx, ny = box
        x0, y0 = g.origin[0] + ix0 * g.xy_resolution, g.origin[1] + iy0 * g.xy_resolution
        x1, y1 = x0 + nx * g.xy_resolution, y0 + ny * g.xy_resolution
        local = pts[(pts[:, 0] >= x0 - margin) & (pts[:, 0] <= x1 + margin) & (pts[:, 1] >= y0 - margin) & (pts[:, 1] <= y1 + margin)]
        assert len(local) < len(pts) // 2
        cells, _ = opt.update_environment_window_from_cloud(local, *box)
        ref = box_cells(small["host"].cells, box).astype(np.float64)
        d = np.abs(cells.astype(np.float64) - ref)
        rel = (d / np.maximum(np.abs(ref), 1e-3)).max(axis=-1)
        assert (rel > 3e-7).mean() <= 2e-4, (box, (rel > 3e-7).mean(), rel.max())
    opt.close()


def test_window_box_helper(built):
    from uneven_planner_b200 import _lib, maps
    g = _lib.map_geometry()               # 10 m, 0.05 m cells, origin -5
    assert maps.window_box(g, -1.0, -1.0, 0.99, 0.99) == (80, 80, 40, 40)
    assert maps.window_box(g, 0.99, 0.99, -1.0, -1.0) == (80, 80, 40, 40)
    assert maps.window_box(g, -9.0, 4.02, -4.88, 9.0) == (0, 180, 3, 20)      # clipped to the grid
    with pytest.raises(ValueError):
        maps.window_box(g, 6.0, 0.0, 7.0, 1.0)


# ---- in flight ----------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def big_cloud():
    return _cloud(400000, 5.3, 3)


@pytest.mark.parametrize("variant", ["cells", "cloud"])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_batch_in_flight_keeps_its_grid_and_its_scan(gpu, world, big_cloud, precision, variant):
    A = world["a64"] if precision == 64 else world["bench"]
    B = world["b"]
    g0 = world["g0"]
    opt = ctx(gpu, precision, world["params"], g0)
    ta = opt.submit(A, depth=2)
    assert pending(opt, ta, A) > 0
    if variant == "cells":
        win = box_cells(world["g1"].cells, BOX)
        opt.update_environment_window(BOX[0], BOX[1], win)
    else:
        win, _ = opt.update_environment_window_from_cloud(big_cloud, *BOX)
    if precision != 64 or variant == "cells":
        # returned while the batch in flight still ran.  (On the parity path a cloud window's kernel waits for a free SM slot,
        # which its solve frees only in the batch's tail: DESIGN section 3h)
        assert pending(opt, ta, A) > 0
    tb = opt.submit(B, depth=2)
    got_a, got_b = pieces(A, opt.wait(ta)), pieces(B, opt.wait(tb))
    scan_a = _scan(opt, ta, A)
    opt.close()
    if variant == "cloud":
        o = gpu.BatchALMTrajOpt()
        full, _ = o.build_map(big_cloud, g0.geom)
        o.close()
        assert np.array_equal(bits(win, np.float32), bits(box_cells(full.cells, BOX), np.float32))
    spliced = splice(g0, win, BOX)
    ref_a, ref_scan = alone(ctx(gpu, precision, world["params"], g0), A, feas=True)
    assert same_pieces(got_a, ref_a)
    assert same_pieces(got_b, alone(ctx(gpu, precision, world["params"], spliced), B)[0])
    assert np.array_equal(scan_a, ref_scan)
    if precision == 64:
        g, n = world["gold"], world["gold_pb"].B      # A's first problems are the golden ones
        rec = [np.frombuffer(p[0], dtype=np.int32, count=3) for p in got_a[:n]]
        assert [int(r[0]) for r in rec] == [int(x) for x in g["ret_code"]]
        assert [int(r[1]) for r in rec] == [int(x) for x in g["outer_iters"]]
        assert [int(r[2]) for r in rec] == [int(x) for x in g["n_evals"]]
        assert np.array_equal(np.array([np.frombuffer(p[0], dtype=np.float64, count=1, offset=32)[0] for p in got_a[:n]]), g["inner_cost"])
        assert np.array_equal(np.concatenate([p[1] for p in got_a[:n]]), g["c_xy"])
        assert np.array_equal(np.concatenate([p[2] for p in got_a[:n]]), g["c_yaw"])


@pytest.mark.parametrize("precision", PRECISIONS)
def test_mixed_environments_only_the_updated_one_changes(gpu, world, precision):
    from uneven_planner_b200 import configs, maps, problems
    names = ["hill", "desert", "volcano", "forest"]
    grids = [maps.stand_in_terrain(n) for n in names]
    params = [configs.params_for(n) for n in names]
    subs = [problems.generate(g, 256, seed=11 + e, **configs.gen_kwargs(n)) for e, (g, n) in enumerate(zip(grids, names))]
    cat = problems.concat(subs, range(4))
    perm = np.array([256 * e + i for i in range(256) for e in range(4)])
    mixed = cat.select(perm)
    box = (50, 50, 100, 100)
    win = box_cells(maps.stand_in_terrain("mountain").cells, box)
    new2 = splice(grids[2], win, box)
    opt = gpu.BatchALMTrajOpt(precision=precision)
    for e in range(4):
        opt.init(params[e], env=e).set_environment(grids[e], env=e)
    t1 = opt.submit(mixed, depth=2)
    opt.update_environment_window(box[0], box[1], win, env=2)
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
    for i, q in enumerate(perm):
        e, j = divmod(int(q), 256)
        assert same_pieces([first[i]], [ref[e][j]]), (i, e)
        assert same_pieces([second[i]], [(ref2 if e == 2 else ref[e])[j]]), (i, e)
    assert any(not same_pieces([ref[2][j]], [ref2[j]]) for j in range(256))      # the window changed environment 2's solves


# ---- refusals, memory, C++ ----------------------------------------------------------------------

@pytest.mark.parametrize("precision", PRECISIONS)
def test_refused_windows_keep_the_grid(gpu, world, precision):
    from uneven_planner_b200 import _lib, maps
    L = _lib.lib()
    fp = C.POINTER(C.c_float)
    pb = world["b"]
    X, Y, W = world["g0"].shape
    opt = ctx(gpu, precision, world["params"], world["g0"])
    before = pieces(pb, opt.optimize(pb))
    cells = np.ascontiguousarray(world["g1"].cells[:X, :Y])          # big enough for every box below
    cp = cells.ctypes.data_as(fp)
    pts = np.zeros((4, 3), np.float32)
    pp = pts.ctypes.data_as(fp)

    def both(ix0, iy0, nx, ny, c=cp, p=pp, h=opt.h, npts=4):
        return (L.ualm_update_map_window(h, ix0, iy0, nx, ny, c),
                L.ualm_update_map_window_from_cloud(h, p, npts, ix0, iy0, nx, ny, 0.2, 0.1, 0.1, 2, None, None))
    EINVAL, ESTATE = (_lib.UALM_EINVAL,) * 2, (_lib.UALM_ESTATE,) * 2
    for box in [(-1, 0, 4, 4), (0, -1, 4, 4), (X - 3, 0, 4, 4), (0, Y - 3, 4, 4), (0, 0, X + 1, 1), (0, 0, 1, Y + 1),
                (0, 0, 0, 4), (0, 0, 4, 0), (0, 0, -1, 4), (0, 0, 4, -2), (X, 0, 1, 1), (2 ** 31 - 1, 0, 1, 1)]:
        assert both(*box) == EINVAL, box
    assert both(0, 0, 4, 4, h=None) == EINVAL
    assert L.ualm_update_map_window(opt.h, 0, 0, 4, 4, None) == _lib.UALM_EINVAL
    assert L.ualm_update_map_window_from_cloud(opt.h, None, 4, 0, 0, 4, 4, 0.2, 0.1, 0.1, 2, None, None) == _lib.UALM_EINVAL
    assert L.ualm_update_map_window_from_cloud(opt.h, pp, -1, 0, 0, 4, 4, 0.2, 0.1, 0.1, 2, None, None) == _lib.UALM_EINVAL
    opt.select_env(1)                                                # no grid bound there
    assert both(0, 0, 4, 4) == ESTATE
    opt.select_env(0)
    assert same_pieces(pieces(pb, opt.optimize(pb)), before)
    opt.close()
    if precision == 64:        # the double grid of ualm_set_map_f64 is not windowed
        g0 = world["g0"]
        o = ctx(gpu, precision, world["params"], maps.UnevenMapData(g0.geom, g0.cells, "f64", cells64=g0.cells.astype(np.float64)))
        before = pieces(pb, o.optimize(pb))
        assert both(0, 0, 4, 4, h=o.h) == ESTATE
        assert same_pieces(pieces(pb, o.optimize(pb)), before)
        o.close()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_windows_do_not_leak(gpu, world, precision):
    import torch
    depth = 3 if precision == 64 else 8
    pb = world["b"]
    opt = ctx(gpu, precision, world["params"], world["g0"])

    def fill():
        for t in [opt.submit(pb, depth=depth) for _ in range(depth)]:
            opt.wait(t)
    fill()                                          # every lane's buffers (and the throughput pool) exist
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    q = collections.deque()
    for i in range(20):
        src = world["g1"] if i % 2 == 0 else world["g0"]
        opt.update_environment_window(BOX[0], BOX[1], box_cells(src.cells, BOX))
        if len(q) == depth:
            opt.wait(q.popleft())
        q.append(opt.submit(pb, depth=depth))
    while q:
        opt.wait(q.popleft())
    fill()                                          # every lane lets go of the grids its earlier launches read
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    opt.close()
    grid = world["g0"].cells.nbytes
    assert free0 - free1 <= grid, (free0, free1, grid)


def test_cpp_window_updates_between_submits(gpu, world, big_cloud, tmp_path):
    from uneven_planner_b200 import _lib
    exe = build_driver("map_window_driver", tmp_path)
    g0, g1 = world["g0"], world["g1"]
    pb = world["bench"].select(np.arange(8))
    win = np.ascontiguousarray(box_cells(g1.cells, BOX))
    pts = big_cloud[:100000]
    case = str(tmp_path / "window.bin")
    with open(case, "wb") as f:
        f.write(struct.pack("<9i", *g0.shape, pb.B, *BOX, len(pts)))
        f.write(g0.cells.tobytes())
        f.write(win.tobytes())
        f.write(np.ascontiguousarray(pts).tobytes())
        for a in (pb.N, pb.M):
            f.write(np.ascontiguousarray(a, np.int32).tobytes())
        for a in (pb.bnd, pb.total_time, pb.inner_xy, pb.inner_yaw):
            f.write(np.ascontiguousarray(a, np.float64).tobytes())
    cloud_out = str(tmp_path / "cloud_window.bin")
    r = subprocess.run([exe, case, cloud_out], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    opt = gpu.BatchALMTrajOpt().init(_lib.default_params()).set_environment(g0)
    t1 = opt.submit(pb, depth=3)
    opt.update_environment_window(BOX[0], BOX[1], win, env=0)
    t2 = opt.submit(pb, depth=3)
    cw, _ = opt.update_environment_window_from_cloud(pts, *BOX)
    t3 = opt.submit(pb, depth=3)
    outs = [opt.wait(t1), opt.wait(t2), opt.wait(t3)]
    opt.close()
    assert np.array_equal(np.fromfile(cloud_out, np.uint32), bits(cw, np.float32).ravel())
    _, _, ocx, _ = pb.offsets()
    want = ["%d %d %d %d %r %r" % (p, i, outs[p][0][i].ret_code, outs[p][0][i].n_evals, float(outs[p][0][i].inner_cost), float(outs[p][1][ocx[i] + 1]))
            for p in range(3) for i in range(pb.B)]
    got = [" ".join(ln.split()[:4] + [repr(float(x)) for x in ln.split()[4:]]) for ln in r.stdout.strip().splitlines()]
    assert got == want
