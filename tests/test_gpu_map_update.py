"""Replacing an environment's map grid while batches are in flight (include/ualm.h, ualm_update_map / ualm_update_map_from_cloud), on
both paths.  Work launched before an update keeps the grid it was launched with, bit for bit (the batch in flight and the post-solve
scan of its lane); every later launch reads the new grid; superseded grids are freed once no lane holds them.  Grids: the seeded
stand-ins of hill (G0) and desert (G1), same geometry, solved with the hill parameters."""
import collections
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRECISIONS = [64, 32, 65]


@pytest.fixture(scope="module")
def gpu(built):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from uneven_planner_b200 import api
    return api


@pytest.fixture(scope="module")
def world(gpu, golden):
    from uneven_planner_b200 import configs, maps, problems
    g0, g1 = maps.stand_in_terrain("hill"), maps.stand_in_terrain("desert")
    kw = configs.gen_kwargs("hill")
    gold = golden("hill", g0)
    gold_pb = problems.generate(g0, int(gold["B"]), seed=int(gold["seed"]), **kw)
    bench = problems.generate(g0, 1024, seed=0, **kw)
    return dict(g0=g0, g1=g1, params=configs.params_for("hill"), gold=gold, gold_pb=gold_pb, bench=bench,
                a64=problems.concat([gold_pb, bench], [0, 0]), b=problems.generate(g1, 256, seed=7, **kw))


def _ctx(gpu, world, precision, grid):
    return gpu.BatchALMTrajOpt(precision=precision).init(world["params"]).set_environment(grid)


def _pieces(pb, out):
    """per problem: (record bytes, c_xy, c_yaw)"""
    res, cxy, cyaw = out
    _, _, ocx, ocy = pb.offsets()
    return [(bytes(res[i]), cxy[ocx[i]:ocx[i + 1]].copy(), cyaw[ocy[i]:ocy[i + 1]].copy()) for i in range(pb.B)]


def _same(a, b):
    return len(a) == len(b) and all(x[0] == y[0] and np.array_equal(x[1], y[1]) and np.array_equal(x[2], y[2]) for x, y in zip(a, b))


def _alone(gpu, world, precision, grid, pb, feas=False):
    """pb solved alone on a fresh context bound to `grid`: (pieces, scan or None)"""
    opt = _ctx(gpu, world, precision, grid)
    out = opt.optimize(pb)
    f = opt.feasibility(0.01) if feas else None
    opt.close()
    return _pieces(pb, out), f


def _pending(opt, t, pb):
    return opt.poll(t, opt.outputs(pb), 0.0)[1]


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
    opt = _ctx(gpu, world, precision, world["g0"])
    ta = opt.submit(A, depth=2)
    assert _pending(opt, ta, A) > 0
    opt.update_environment(world["g1"])
    tb = opt.submit(B, depth=2)
    got_a, got_b = _pieces(A, opt.wait(ta)), _pieces(B, opt.wait(tb))
    scan_a = _scan(opt, ta, A)
    opt.close()
    ref_a, ref_scan = _alone(gpu, world, precision, world["g0"], A, feas=True)
    assert _same(got_a, ref_a)
    assert _same(got_b, _alone(gpu, world, precision, world["g1"], B)[0])
    assert np.array_equal(scan_a, ref_scan)
    # the scan of A's coefficients against G1 differs: ualm_set_map writes into the grid the lane holds, as it always has
    ref = _ctx(gpu, world, precision, world["g0"])
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
    first, second = _pieces(mixed, opt.wait(t1)), _pieces(mixed, opt.wait(t2))
    opt.close()

    def alone(e, grid):
        o = gpu.BatchALMTrajOpt(precision=precision).init(params[e]).set_environment(grid)
        out = _pieces(subs[e], o.optimize(subs[e]))
        o.close()
        return out
    ref = [alone(e, grids[e]) for e in range(4)]
    ref2 = alone(2, new2)
    for i, q in enumerate(perm):
        e, j = divmod(int(q), 256)
        assert _same([first[i]], [ref[e][j]]), (i, e)
        assert _same([second[i]], [(ref2 if e == 2 else ref[e])[j]]), (i, e)
    assert any(not _same([ref[2][j]], [ref2[j]]) for j in range(256))      # the update changed environment 2's solves


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
    opt = _ctx(gpu, world, precision, world["g0"])
    ta = opt.submit(A, depth=2)
    m, ms = opt.update_environment_from_cloud(cw["pts"], cw["geom"])
    if precision != 64:
        # returned while the batch in flight still had problems running.  (The parity solve's CTAs hold every SM's register file
        # until its work queue runs dry, so there the build kernel only starts in the batch's tail: DESIGN section 3h)
        assert _pending(opt, ta, A) > 0
    assert ms > 0.0
    assert np.array_equal(m.cells.view(np.uint32), cw["host"].cells.view(np.uint32))
    tc = opt.submit(cw["pb"], depth=2)
    got = _pieces(cw["pb"], opt.wait(tc))
    opt.wait(ta)
    opt.close()
    ref = _ctx(gpu, world, precision, world["g0"])
    ref.set_environment(cw["host"])
    want = _pieces(cw["pb"], ref.wait(ref.submit(cw["pb"], depth=2)))
    ref.close()
    assert _same(got, want)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_updates_do_not_leak(gpu, world, precision):
    import torch
    depth = 3 if precision == 64 else 8
    pb = world["b"]
    opt = _ctx(gpu, world, precision, world["g0"])

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
    opt = _ctx(gpu, world, precision, world["g0"])
    before = _pieces(pb, opt.optimize(pb))
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
    assert _same(_pieces(pb, opt.optimize(pb)), before)
    opt.close()


def test_cpp_update_environment_between_submits(gpu, world, tmp_path):
    from uneven_planner_b200 import _lib
    exe = str(tmp_path / "map_update_driver")
    lib = os.path.join(ROOT, "uneven_planner_b200")
    subprocess.run(["g++", "-O2", "-std=c++14", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "map_update_driver.cpp"), "-o", exe,
                    "-L", lib, "-lualm", "-Wl,-rpath," + lib], check=True)
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
