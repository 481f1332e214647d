"""Replacing an environment's map grid while batches are in flight (include/ualm.h, ualm_update_map / ualm_update_map_from_cloud), on
both paths.  Work launched before an update keeps the grid it was launched with, bit for bit (the batch in flight and the post-solve
scan of its lane); every later launch reads the new grid; superseded grids are freed once no lane holds them.  Grids: the seeded
stand-ins of hill (G0) and desert (G1), same geometry, solved with the hill parameters."""
import collections
import ctypes as C
import struct
import subprocess

import numpy as np
import pytest

from harness import alone, build_driver, ctx, gpu, pending, pieces, same_pieces  # noqa: F401
from workloads import hill_desert_world


pytestmark = pytest.mark.gpu
PRECISIONS = [64, 32, 65]


@pytest.fixture(scope="module")
def world(gpu, golden):
    return hill_desert_world(golden, b_grid="g1")


def _scan(opt, ticket, pb):
    opt.select_lane(ticket)
    opt.pb = pb
    f = opt.feasibility(0.01)
    opt.select_lane(0)
    return f


@pytest.mark.parametrize("precision", PRECISIONS)
def test_batch_in_flight_keeps_its_grid_and_its_scan(gpu, world, precision):
    A = world["a64"] if precision == 64 else world["bench"]
    B = world["b"]
    opt = ctx(gpu, precision, world["params"], world["g0"])
    ta = opt.submit(A, depth=2)
    assert pending(opt, ta, A) > 0
    opt.update_environment(world["g1"])
    tb = opt.submit(B, depth=2)
    got_a, got_b = pieces(A, opt.wait(ta)), pieces(B, opt.wait(tb))
    scan_a = _scan(opt, ta, A)
    opt.close()
    ref_a, ref_scan = alone(ctx(gpu, precision, world["params"], world["g0"]), A, feas=True)
    assert same_pieces(got_a, ref_a)
    assert same_pieces(got_b, alone(ctx(gpu, precision, world["params"], world["g1"]), B)[0])
    assert np.array_equal(scan_a, ref_scan)
    # the scan of A's coefficients against G1 differs: ualm_set_map writes into the grid the lane holds, as it always has
    ref = ctx(gpu, precision, world["params"], world["g0"])
    ref.optimize(A)
    ref.set_environment(world["g1"])
    assert not np.array_equal(ref.feasibility(0.01), ref_scan)
    ref.close()
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
    new2 = maps.stand_in_terrain("mountain")
    opt = gpu.BatchALMTrajOpt(precision=precision)
    for e in range(4):
        opt.init(params[e], env=e).set_environment(grids[e], env=e)
    t1 = opt.submit(mixed, depth=2)
    opt.update_environment(new2, env=2)
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
    assert any(not same_pieces([ref[2][j]], [ref2[j]]) for j in range(256))      # the update changed environment 2's solves


def _cloud(n, half, seed):
    """a seeded analytic surface with noise and an empty patch (as tests/test_gpu_map_build.py)"""
    rng = np.random.default_rng(seed)
    xy = rng.uniform(-half, half, (n, 2))
    z = 0.4 * np.exp(-((xy[:, 0] - 0.5) ** 2 + (xy[:, 1] + 0.3) ** 2) / 0.8) + 0.15 * np.sin(2.0 * xy[:, 0]) * np.cos(1.5 * xy[:, 1]) + 0.3
    z += rng.normal(0.0, 0.004, n)
    pts = np.column_stack([xy, z]).astype(np.float32)
    keep = ~((np.abs(pts[:, 0] + 1.0) < 0.35) & (np.abs(pts[:, 1] - 1.0) < 0.35))
    return pts[keep]


@pytest.fixture(scope="module")
def cloud_world(world):
    from uneven_planner_b200 import _lib, configs, maps, problems
    geom = _lib.map_geometry()
    pts = _cloud(400000, 5.3, 3)
    host = maps.build_from_cloud(pts, geom)
    return dict(pts=pts, geom=geom, host=host, pb=problems.generate(host, 256, seed=4, **configs.gen_kwargs("hill")))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_update_from_cloud(gpu, world, cloud_world, precision):
    cw = cloud_world
    A = world["bench"]
    opt = ctx(gpu, precision, world["params"], world["g0"])
    ta = opt.submit(A, depth=2)
    m, ms = opt.update_environment_from_cloud(cw["pts"], cw["geom"])
    if precision != 64:
        # returned while the batch in flight still had problems running.  (The parity solve's CTAs hold every SM's register file
        # until its work queue runs dry, so there the build kernel only starts in the batch's tail: DESIGN section 3h)
        assert pending(opt, ta, A) > 0
    assert ms > 0.0
    assert np.array_equal(m.cells.view(np.uint32), cw["host"].cells.view(np.uint32))
    tc = opt.submit(cw["pb"], depth=2)
    got = pieces(cw["pb"], opt.wait(tc))
    opt.wait(ta)
    opt.close()
    ref = ctx(gpu, precision, world["params"], world["g0"])
    ref.set_environment(cw["host"])
    want = pieces(cw["pb"], ref.wait(ref.submit(cw["pb"], depth=2)))
    ref.close()
    assert same_pieces(got, want)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_updates_do_not_leak(gpu, world, precision):
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
        opt.update_environment(world["g1"] if i % 2 == 0 else world["g0"])
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


@pytest.mark.parametrize("precision", PRECISIONS)
def test_refused_and_failed_updates_keep_the_grid(gpu, world, precision):
    from uneven_planner_b200 import _lib
    L = _lib.lib()
    fp = C.POINTER(C.c_float)
    pb = world["b"]
    opt = ctx(gpu, precision, world["params"], world["g0"])
    before = pieces(pb, opt.optimize(pb))
    g = world["g1"].geom
    cells = world["g1"].cells.ctypes.data_as(fp)
    pts = np.zeros((4, 3), np.float32)
    ptsp = pts.ctypes.data_as(fp)
    assert L.ualm_update_map(None, C.byref(g), cells) == _lib.UALM_EINVAL
    assert L.ualm_update_map(opt.h, None, cells) == _lib.UALM_EINVAL
    assert L.ualm_update_map(opt.h, C.byref(g), None) == _lib.UALM_EINVAL
    assert L.ualm_update_map_from_cloud(None, ptsp, 4, C.byref(g), 0.2, 0.1, 0.1, 2, None, None) == _lib.UALM_EINVAL
    assert L.ualm_update_map_from_cloud(opt.h, None, 4, C.byref(g), 0.2, 0.1, 0.1, 2, None, None) == _lib.UALM_EINVAL
    assert L.ualm_update_map_from_cloud(opt.h, ptsp, 4, None, 0.2, 0.1, 0.1, 2, None, None) == _lib.UALM_EINVAL
    for k in range(3):
        for v in (0, -1):
            bad = _lib.map_geometry()
            bad.voxel_num[k] = v
            assert L.ualm_update_map(opt.h, C.byref(bad), cells) == _lib.UALM_EINVAL
            assert L.ualm_update_map_from_cloud(opt.h, ptsp, 4, C.byref(bad), 0.2, 0.1, 0.1, 2, None, None) == _lib.UALM_EINVAL
    # a grid no device can hold: the new version's allocation fails before anything is read or built
    huge = _lib.map_geometry()
    huge.voxel_num[0] = huge.voxel_num[1] = 200000
    assert L.ualm_update_map_from_cloud(opt.h, ptsp, 4, C.byref(huge), 0.2, 0.1, 0.1, 2, None, None) == _lib.UALM_ENOCUDA
    assert same_pieces(pieces(pb, opt.optimize(pb)), before)
    opt.close()


def test_cpp_update_environment_between_submits(gpu, world, tmp_path):
    from uneven_planner_b200 import _lib
    exe = build_driver("map_update_driver", tmp_path)
    g0, g1 = world["g0"], world["g1"]
    pb = world["bench"].select(np.arange(8))
    case = str(tmp_path / "update.bin")
    with open(case, "wb") as f:
        f.write(struct.pack("<4i", *g0.shape, pb.B))
        f.write(g0.cells.tobytes())
        f.write(g1.cells.tobytes())
        for a in (pb.N, pb.M):
            f.write(np.ascontiguousarray(a, np.int32).tobytes())
        for a in (pb.bnd, pb.total_time, pb.inner_xy, pb.inner_yaw):
            f.write(np.ascontiguousarray(a, np.float64).tobytes())
    r = subprocess.run([exe, case], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    opt = gpu.BatchALMTrajOpt().init(_lib.default_params()).set_environment(g0)
    t1 = opt.submit(pb, depth=2)
    opt.update_environment(g1, env=0)
    t2 = opt.submit(pb, depth=2)
    outs = [opt.wait(t1), opt.wait(t2)]
    opt.close()
    _, _, ocx, _ = pb.offsets()
    want = ["%d %d %d %d %r %r" % (p, i, outs[p][0][i].ret_code, outs[p][0][i].n_evals, float(outs[p][0][i].inner_cost), float(outs[p][1][ocx[i] + 1]))
            for p in range(2) for i in range(pb.B)]
    got = [" ".join(ln.split()[:4] + [repr(float(x)) for x in ln.split()[4:]]) for ln in r.stdout.strip().splitlines()]
    assert got == want
    assert any(got[i].split()[2:] != got[pb.B + i].split()[2:] for i in range(pb.B))      # the second batch read the new grid
