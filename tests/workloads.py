"""The workloads, case builders, oracle runs and tolerance tables that more than one test module uses: test modules import
these from here and never from each other."""
import ctypes as C
import functools
import os
import re
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import alm_ref as ar
import stop_oracle as so
import map_build_ref as mref
from harness import bits, cat, ctx
from uneven_planner_b200 import configs, problems


def hill_desert_world(golden, b_grid="g0"):
    """the seeded stand-ins of hill (g0) and desert (g1) with the hill parameters; the golden problems (gold_pb), the bench's 1024
    (bench), both in one batch (a64), and 256 more problems generated on grid `b_grid` (b)"""
    from uneven_planner_b200 import configs, maps, problems
    g0, g1 = maps.stand_in_terrain("hill"), maps.stand_in_terrain("desert")
    kw = configs.gen_kwargs("hill")
    gold = golden("hill", g0)
    gold_pb = problems.generate(g0, int(gold["B"]), seed=int(gold["seed"]), **kw)
    bench = problems.generate(g0, 1024, seed=0, **kw)
    return dict(g0=g0, g1=g1, params=configs.params_for("hill"), gold=gold, gold_pb=gold_pb, bench=bench,
                a64=problems.concat([gold_pb, bench], [0, 0]), b=problems.generate(g1 if b_grid == "g1" else g0, 256, seed=7, **kw))


def _arc_problem(N, M, zero_ends=False, radius=2.5, arc=1.5 * np.pi, speed=0.5, centre=(0.0, 0.0), start=0.0):
    """One problem whose waypoints lie on a circular arc around `centre` (the map centre by default), from polar angle `start`
    counter-clockwise over `arc`: N xy pieces, M yaw pieces.  zero_ends: zero boundary velocity and acceleration, so that those
    right-hand-side rows are exact zeros."""
    from uneven_planner_b200 import problems
    length = radius * arc
    T = 1.2 * length / speed
    a = start + arc * np.linspace(0.0, 1.0, N + 1)
    rel = radius * np.stack([np.cos(a), np.sin(a)], axis=1)
    pts = rel + np.asarray(centre, np.float64)
    yaw = start + arc * np.linspace(0.0, 1.0, M + 1) + 0.5 * np.pi
    tan0, tan1 = np.array([-np.sin(a[0]), np.cos(a[0])]), np.array([-np.sin(a[-1]), np.cos(a[-1])])
    v = 0.0 if zero_ends else speed
    acc0 = np.zeros(2) if zero_ends else -speed ** 2 / radius * rel[0] / radius
    acc1 = np.zeros(2) if zero_ends else -speed ** 2 / radius * rel[-1] / radius
    dyaw = 0.0 if zero_ends else speed / radius
    bnd = np.concatenate([pts[0], v * tan0, acc0, pts[-1], v * tan1, acc1, [yaw[0], dyaw, 0.0, yaw[-1], dyaw, 0.0]])
    return problems.ProblemBatch(np.array([N], np.int32), np.array([M], np.int32), bnd.reshape(1, 18), np.array([T]),
                                 pts[1:-1].ravel().copy(), yaw[1:-1].copy())


TOL = {65: dict(f=1e-9, grad=1e-9, con=1e-9, coef=1e-10, sfx=1e-9, scx=1e-8),
       32: dict(f=1e-4, grad=1e-4, con=1e-4, coef=1e-10, sfx=1e-6, scx=2e-3)}


NAMES = ["hill", "desert", "volcano", "forest"]


def mixed_golden_batch(terrain, golden):
    """(maps, params, goldens, per-terrain batches, mixed batch, perm): the golden problems of the four terrains, terrain k in
    environment k, interleaved (problem i of every terrain, then problem i + 1, ...).  mixed = concat(batches).select(perm)."""
    maps, params, golds, pbs = [], [], [], []
    for name in NAMES:
        m = terrain(name)
        gold = golden(name, m)
        maps.append(m); params.append(configs.params_for(name)); golds.append(gold)
        pbs.append(problems.generate(m, int(gold["B"]), seed=int(gold["seed"]), **configs.gen_kwargs(name)))
    cat = problems.concat(pbs, range(len(NAMES)))
    start = np.concatenate([[0], np.cumsum([p.B for p in pbs])])
    perm = np.array([start[k] + i for i in range(max(p.B for p in pbs)) for k in range(len(pbs)) if i < pbs[k].B])
    return maps, params, golds, pbs, cat.select(perm), perm


def _with_oversize(pb, at):
    """a copy of pb with one problem of N = 70, M = 140 (over the compiled limits 64 / 128) inserted at index `at`"""
    from uneven_planner_b200 import problems
    oxy, oyaw, _, _ = pb.offsets()
    N, M = 70, 140
    t = np.linspace(0.0, 1.0, N + 1)[1:-1]
    ixy = np.column_stack([-4.0 + 8.0 * t, -4.0 + 8.0 * t]).ravel()
    iyaw = np.full(M - 1, np.pi / 4)
    bnd = np.zeros(18); bnd[0:2] = -4.0; bnd[6:8] = 4.0; bnd[12] = bnd[15] = np.pi / 4
    return problems.ProblemBatch(np.insert(pb.N, at, N).astype(np.int32), np.insert(pb.M, at, M).astype(np.int32),
                                 np.insert(pb.bnd, at, bnd, axis=0), np.insert(pb.total_time, at, 30.0),
                                 np.concatenate([pb.inner_xy[:oxy[at]], ixy, pb.inner_xy[oxy[at]:]]),
                                 np.concatenate([pb.inner_yaw[:oyaw[at]], iyaw, pb.inner_yaw[oyaw[at]:]]))


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


REF = os.path.join(ROOT, "oracle", "_ref", "libref.so")


dp = C.POINTER(C.c_double)


def P(a):
    return None if a is None else a.ctypes.data_as(dp)


# ---------------------------------------------------------------------------------------------------------------------
# the whole path: ALMTrajOpt::optimizeSE2Traj of back_end/src/alm_traj_opt.cpp (unmodified) vs the oracle
# ---------------------------------------------------------------------------------------------------------------------
class RefParams(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("rho_T", "rho_ter", "max_vel", "max_acc_lon", "max_acc_lat", "max_kap", "min_cxi", "max_sig")] + \
               [("use_scaling", C.c_int)] + \
               [(n, C.c_double) for n in ("rho", "beta", "gamma", "epsilon_con", "max_iter", "g_epsilon", "min_step", "inner_max_iter", "delta")] + \
               [("mem_size", C.c_int), ("past", C.c_int), ("int_K", C.c_int), ("gravity", C.c_double)]


def _ref_solve(L, params, mapdata, pb, i):
    g = mapdata.geom
    rp = RefParams()
    for n, _ in RefParams._fields_:
        setattr(rp, n, getattr(params, n))
    cells = np.ascontiguousarray(mapdata.cells, dtype=np.float64)
    N, M = int(pb.N[i]), int(pb.M[i])
    S = N * (params.int_K + 1)
    oxy, oyaw, _, _ = pb.offsets()
    ixy = np.ascontiguousarray(pb.inner_xy[oxy[i]:oxy[i + 1]]); iyaw = np.ascontiguousarray(pb.inner_yaw[oyaw[i]:oyaw[i + 1]])
    out = dict(c_xy=np.zeros(12 * N), c_yaw=np.zeros(6 * M), piece_T=np.zeros(2), lam=np.zeros(S), mu=np.zeros(6 * S), hx=np.zeros(S),
               gx=np.zeros(6 * S), sfx=np.zeros(1), scx=np.zeros(7 * S), rho=np.zeros(1), feas=np.zeros(7))
    vn = (C.c_int * 3)(*g.voxel_num); org = (C.c_double * 3)(*g.origin); mxb = (C.c_double * 3)(*g.max_boundary)
    L.ref_alm_solve.restype = C.c_int
    ret = L.ref_alm_solve(C.byref(rp), P(cells), vn, org, mxb, C.c_double(g.xy_resolution), C.c_double(g.yaw_resolution), N, M,
                          P(np.ascontiguousarray(pb.bnd[i])), C.c_double(float(pb.total_time[i])), P(ixy if ixy.size else np.zeros(1)),
                          P(iyaw if iyaw.size else np.zeros(1)), 0, P(out["c_xy"]), P(out["c_yaw"]), P(out["piece_T"]), P(out["lam"]), P(out["mu"]),
                          P(out["hx"]), P(out["gx"]), P(out["sfx"]), P(out["scx"]), P(out["rho"]), P(out["feas"]))
    return ret, out


# ---------------------------------------------------------------- UnevenMap construction (SURVEY 8f-1)
REFMAP = os.path.join(ROOT, "oracle", "_ref", "librefmap.so")


def reference_construct_map(cloud, size, iter_num=2, ellipsoid=(0.2, 0.1, 0.1)):
    """UnevenMap::constructMap + filter of the reference's uneven_map.cpp (compiled unmodified, oracle/ref_map_driver.cpp) on an already
    preprocessed cloud: cells [X, Y, Yaw, 4] in double."""
    from uneven_planner_b200 import _lib
    if not os.path.exists(REFMAP):
        pytest.skip("oracle/_ref/librefmap.so not built (needs the reference sources at build time)")
    R = C.CDLL(REFMAP)
    geom = _lib.map_geometry(size, size, 0.05, 0.1)
    X, Y, W = geom.voxel_num
    cells = np.zeros((X * Y * W, 4))
    vn = (C.c_int * 3)()
    cloud = np.ascontiguousarray(cloud, dtype=np.float32)
    R.ref_map_construct(cloud.ctypes.data_as(C.POINTER(C.c_float)), int(cloud.shape[0]), C.c_double(size), C.c_double(size), C.c_double(0.05), C.c_double(0.1),
                        C.c_double(ellipsoid[0]), C.c_double(ellipsoid[1]), C.c_double(ellipsoid[2]), int(iter_num), cells.ctypes.data_as(C.POINTER(C.c_double)), vn)
    assert tuple(vn) == (X, Y, W)
    return geom, cells.reshape(X, Y, W, 4)


def analytic_cloud(half, n, seed, hole=None):
    """jittered grid on an analytic surface with noise (and an optional empty patch)"""
    rng = np.random.default_rng(seed)
    gx, gy = np.meshgrid(np.linspace(-half, half, n), np.linspace(-half, half, n), indexing="ij")
    px = (gx + rng.uniform(-0.008, 0.008, gx.shape)).ravel(); py = (gy + rng.uniform(-0.008, 0.008, gy.shape)).ravel()
    pz = 0.5 + 0.3 * np.sin(1.3 * px) * np.cos(0.9 * py) + 0.15 * np.exp(-((px - 0.5) ** 2 + (py + 0.3) ** 2) / 0.18) + rng.normal(0, 0.003, px.shape)
    pts = np.column_stack([px, py, pz]).astype(np.float32)
    if hole is not None:
        pts = pts[~((np.abs(pts[:, 0] - hole[0]) < hole[2]) & (np.abs(pts[:, 1] - hole[1]) < hole[2]))]
    return pts


def preprocessed(pts, ellipsoid=(0.2, 0.1, 0.1)):
    """the cloud the builders work on (UnevenMap::init's CropBox + VoxelGrid, through the host tool)"""
    from uneven_planner_b200 import _lib
    L = _lib.lib()
    fp = C.POINTER(C.c_float)
    out = np.zeros((pts.shape[0], 3), np.float32)
    k = L.ualm_map_preprocess_cloud(pts.ctypes.data_as(fp), pts.shape[0], ellipsoid[0], ellipsoid[1], ellipsoid[2], out.ctypes.data_as(fp), pts.shape[0])
    assert k > 0
    return np.ascontiguousarray(out[:k])


# name: (size x, size y [m], xy resolution [m], yaw resolution [rad], cells, terrain seed: one whose bumps reach every edge)
GRIDS = {
    "wide": (12.0, 6.0, 0.05, 0.1, (240, 120, 64), 206),        # X > Y
    "tall": (6.0, 12.0, 0.05, 0.1, (120, 240, 64), 211),        # X < Y, as many cells as `wide`
    "coarse": (9.0, 7.0, 0.1, 0.2, (90, 70, 32), 206),          # other resolutions; only the yaw count is a multiple of 8
    "fine_yaw": (7.3, 5.0, 0.04, 0.05, (183, 125, 127), 206),   # odd counts, ceil rounds up in x, an odd number of yaw layers
    "site": (20.0, 10.0, 0.05, 0.1, (400, 200, 64), 206),       # the largest extent the builder's crop box keeps; 82 MB of float4
}


SMALL = ["wide", "tall", "coarse", "fine_yaw"]


def geometry(name):
    from uneven_planner_b200 import _lib
    sx, sy, rxy, ryaw, _, _ = GRIDS[name]
    return _lib.map_geometry(sx, sy, rxy, ryaw)


@functools.lru_cache(maxsize=None)
def grid(name):
    """the `hills` terrain (the same bits on every host) on grid `name`"""
    from uneven_planner_b200 import maps
    m = maps.synthetic_terrain("hills", seed=GRIDS[name][5], geom=geometry(name))
    m.name = name
    return m


# ------------------------------------------------------------------ 1a. the oracle's map query against a plain reference
def _norm_so2(a):
    while a < -np.pi:
        a += 2 * np.pi
    while a > np.pi:
        a -= 2 * np.pi
    return a


def in_map(geom, pos):
    """UnevenMap::isInMap (uneven_map.h:437-454)"""
    o, b = geom.origin, geom.max_boundary
    return not (any(pos[k] < o[k] + 1e-4 for k in range(3)) or any(pos[k] > b[k] - 1e-4 for k in range(3)))


def ref_query(cells, geom, pos):
    """UnevenMap::getAllWithGrad in float64: cells is the [X, Y, W, 4] array, indexed as an array.  Returns (values[7], grads[7, 3])."""
    X, Y, W = geom.voxel_num
    rxy, ryaw = geom.xy_resolution, geom.yaw_resolution
    ixy, iyaw = 1.0 / rxy, 1.0 / ryaw
    org = np.array(list(geom.origin))
    pos = np.asarray(pos, np.float64)
    rs, rg = np.zeros(3), np.zeros((4, 3))
    if in_map(geom, pos):
        pm = pos - 0.5 * np.array([rxy, rxy, ryaw])
        pm[2] = _norm_so2(pm[2])
        inv = np.array([ixy, ixy, iyaw])
        idx = np.floor((pm - org) * inv).astype(int)
        centre = (idx + 0.5) * np.array([rxy, rxy, ryaw]) + org
        d = (pos - centre) * inv
        d[2] = np.arctan2(np.sin(pos[2] - centre[2]), np.cos(pos[2] - centre[2])) * iyaw
        xs = np.clip([idx[0], idx[0] + 1], 0, X - 1)
        ys = np.clip([idx[1], idx[1] + 1], 0, Y - 1)
        ws = np.mod([idx[2], idx[2] + 1], W)
        v = cells[np.ix_(xs, ys, ws)][..., 1:].astype(np.float64)          # [x, y, w, (sigma, zbx, zby)]
        vx = v[0] * (1 - d[0]) + v[1] * d[0]                                # [y, w, 3]
        vy = vx[0] * (1 - d[1]) + vx[1] * d[1]                              # [w, 3]
        rs = vy[0] * (1 - d[2]) + vy[1] * d[2]
        rg[:3, 2] = (vy[1] - vy[0]) * iyaw
        dy = vx[1] - vx[0]                                                  # [w, 3]
        rg[:3, 1] = (dy[0] * (1 - d[2]) + dy[1] * d[2]) * ixy
        dx = v[1] - v[0]                                                    # [y, w, 3]
        rg[:3, 0] = ((1 - d[2]) * (1 - d[1]) * dx[0, 0] + (1 - d[2]) * d[1] * dx[1, 0] + d[2] * (1 - d[1]) * dx[0, 1] + d[2] * d[1] * dx[1, 1]) * ixy
        c = np.sqrt(1.0 - rs[1] ** 2 - rs[2] ** 2)
        rg[3] = -(rg[1] * rs[1] + rg[2] * rs[2]) / c
    c = np.sqrt(1.0 - rs[1] ** 2 - rs[2] ** 2)
    inv_c = 1.0 / c
    cy, sy = np.cos(pos[2]), np.sin(pos[2])
    t = cy * rs[1] + sy * rs[2]
    s = -(-sy * rs[1] + cy * rs[2])
    q = np.sqrt(1.0 - t * t)
    iq = 1.0 / q
    iq3 = iq ** 3
    dt = rg[1] * cy + rg[2] * sy
    ds = -(rg[1] * -sy + rg[2] * cy)
    dt[2] -= s
    ds[2] += t
    values = np.array([iq, -c * t * iq, q * inv_c, s * iq, c, inv_c, rs[0]])
    grads = np.stack([t * iq3 * dt, -(t * iq * rg[3] + iq3 * c * dt), -inv_c * (t * iq * dt + q * inv_c * rg[3]), iq * ds + t * iq3 * s * dt,
                      rg[3], -inv_c * inv_c * rg[3], rg[0]])
    return values, grads


OUTSIDE = np.array([1.0, 0.0, 1.0, 0.0, 1.0, 1.0, 0.0])      # zero terrain: flat ground, no roughness, zero gradients


def query_poses(geom, n=2000, seed=0):
    """seeded poses over the rectangle enlarged by 0.2 m, then the edges: the first and last cell of each axis, the four corners just
    inside and just outside the 1e-4 margin, yaw at +-pi -+ 1e-6, at origin[2], and around the last yaw layer's centre, from where
    the upper neighbour is layer 0"""
    rng = np.random.default_rng(seed)
    o, b = np.array(list(geom.origin)), np.array(list(geom.max_boundary))
    W = geom.voxel_num[2]
    rxy, ryaw = geom.xy_resolution, geom.yaw_resolution
    pts = [np.column_stack([rng.uniform(o[0] - 0.2, b[0] + 0.2, n), rng.uniform(o[1] - 0.2, b[1] + 0.2, n), rng.uniform(-np.pi, np.pi, n)])]
    mid = 0.5 * (o + b) + np.array([0.013, -0.017, 0.3])
    edge = []
    for k in range(2):
        for f in (0.2, 0.7, 1.3):                       # below the first cell's centre (clamped), inside it, in the second
            for at in (o[k] + f * rxy, b[k] - f * rxy):
                p = mid.copy()
                p[k] = at
                edge.append(p)
    for sx in (0, 1):
        for sy in (0, 1):
            for eps in (2e-4, 0.5e-4):                   # inside / outside the margin
                x = o[0] + eps if sx == 0 else b[0] - eps
                y = o[1] + eps if sy == 0 else b[1] - eps
                edge.append(np.array([x, y, 0.4]))
    last = _norm_so2(o[2] + (W - 0.5) * ryaw)
    for yaw in (np.pi - 1e-6, -np.pi + 1e-6, o[2], o[2] + 2e-4, last, last - 0.3 * ryaw, last + 0.3 * ryaw, -np.pi + 0.3 * ryaw, np.pi - 0.3 * ryaw):
        edge.append(np.array([mid[0], mid[1], yaw]))
    for f in (0.3, 0.6):                                 # every layer pair once, the seam pair included
        for w in range(W):
            edge.append(np.array([mid[0], mid[1], _norm_so2(o[2] + (w + 0.5 + f) * ryaw)]))
    pts.append(np.array(edge))
    return np.vstack(pts)


def _cloud(n, half, seed, hole=True):
    """a seeded analytic surface with noise and an empty patch (as tests/test_gpu_map_build.py)"""
    rng = np.random.default_rng(seed)
    xy = rng.uniform(-half, half, (n, 2))
    z = 0.4 * np.exp(-((xy[:, 0] - 0.5) ** 2 + (xy[:, 1] + 0.3) ** 2) / 0.8) + 0.15 * np.sin(2.0 * xy[:, 0]) * np.cos(1.5 * xy[:, 1]) + 0.3
    z += rng.normal(0.0, 0.004, n)
    pts = np.column_stack([xy, z]).astype(np.float32)
    if hole:   # an empty patch around (-1, 1): cells there take the "no points in the ellipsoid" branch
        keep = ~((np.abs(pts[:, 0] + 1.0) < 0.35) & (np.abs(pts[:, 1] - 1.0) < 0.35))
        pts = pts[keep]
    return pts


REL_TOL = 0.0          # bitwise; the north-star bound is 1e-5


def _rel(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    if a.size == 0:
        return 0.0
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def _assert_solve_parity(pb, res, cxy, cyaw, ores):
    _, _, ocx, ocy = pb.offsets()
    for i in range(pb.B):
        r, ocxy, ocyaw, _ = ores[i]
        g = res[i]
        assert (g.ret_code, g.outer_iters, g.n_evals, g.n_lbfgs_iters, g.last_lbfgs_ret) == \
               (r.ret_code, r.outer_iters, r.n_evals, r.n_lbfgs_iters, r.last_lbfgs_ret), i
        assert abs(g.inner_cost - r.inner_cost) <= REL_TOL * abs(r.inner_cost), i
        assert _rel(cxy[ocx[i]:ocx[i + 1]], ocxy) <= REL_TOL and _rel(cyaw[ocy[i]:ocy[i + 1]], ocyaw) <= REL_TOL, i
        assert g.res_h == r.res_h and g.res_g == r.res_g and g.total_T == r.total_T and g.jerk_cost == r.jerk_cost


def _cloud_at(cx, cy, n=40000, half=2.2, seed=0):
    rng = np.random.default_rng(seed)
    xy = rng.uniform(-half, half, (n, 2))
    z = 0.3 + 0.2 * np.sin(1.7 * xy[:, 0]) * np.cos(1.3 * xy[:, 1]) + rng.normal(0.0, 0.003, n)
    return np.column_stack([xy[:, 0] + cx, xy[:, 1] + cy, z]).astype(np.float32)


DEV_GUARD = 4.0e6          # mpc_export_kernel scans only when total / dt < DEV_GUARD


INIT_V = (0.7, -0.3, 0.25)   # every component distinct, and distinct from INIT_A's: a swapped index changes the result


INIT_A = (-1.1, 0.4, -0.6)


def _P(a):
    return a.ctypes.data_as(dp)


@pytest.fixture(scope="module")
def orc(built):
    import pyoracle as po
    L = po.lib()
    L.orc_minco_generate.argtypes = [C.c_int, C.c_int, dp, dp, dp, dp, dp]
    return L


# ------------------------------------------------------------------ the references
def summed(dur, P):
    """the duration of P pieces of `dur` as the kernel and PolyTrajectory::getTotalDuration form it: added one piece at a time"""
    total = 0.0
    for _ in range(P):
        total += dur
    return total


def locate(P, dur, t):
    """PolyTrajectory::locatePieceIdx (se2traj.hpp:343-361) for uniform durations, over an array of times: (piece index, local time)"""
    t = np.array(t, dtype=np.float64, copy=True).reshape(-1)
    idx = np.zeros(t.size, np.int64)
    act = np.nonzero(t > dur)[0]
    while act.size:
        t[act] -= dur
        idx[act] += 1
        act = act[(idx[act] < P) & (t[act] > dur)]
    last = idx == P
    idx[last] -= 1
    t[last] += dur
    return idx, t


def evaluate(c, P, dur, t):
    """Piece::getValue (se2traj.hpp:106-118) of the P-piece spline with coefficients c (6 per piece, low -> high) at times t"""
    idx, tl = locate(P, dur, t)
    c6 = np.asarray(c, np.float64)[:6 * P].reshape(P, 6)[idx]
    v = np.zeros(tl.size)
    tn = np.ones(tl.size)
    for k in range(6):
        v = v + tn * c6[:, k]
        tn = tn * tl
    return v


def message_ref(c_xy, c_yaw, N, M, Tx, Ty):
    """the SE2Traj message of one planned trajectory: pos_pts (N + 1, 2), posT_pts (N), angle_pts (M + 1), angleT_pts (M)"""
    c_xy, c_yaw = np.asarray(c_xy, np.float64), np.asarray(c_yaw, np.float64)
    pos = np.empty((N + 1, 2))
    pos[:N, 0], pos[:N, 1] = c_xy[0:6 * N:6], c_xy[6 * N::6]
    end = summed(Tx, N)
    pos[N, 0], pos[N, 1] = evaluate(c_xy[:6 * N], N, Tx, end)[0], evaluate(c_xy[6 * N:], N, Tx, end)[0]
    ang = np.empty(M + 1)
    ang[:M] = c_yaw[0::6]
    ang[M] = evaluate(c_yaw, M, Ty, summed(Ty, M))[0]
    return dict(pos_pts=pos, posT_pts=np.full(N, Tx), angle_pts=ang, angleT_pts=np.full(M, Ty))


def minco(orc, pts, dur, v0, a0):
    """orc_minco_generate over the points pts (P + 1, Dim) with uniform durations, head (pts[0], v0, a0), tail (pts[P], 0, 0):
    the 6P x Dim coefficients, column-major"""
    pts = np.asarray(pts, np.float64)
    Pn, Dim = pts.shape[0] - 1, pts.shape[1]
    head = np.ascontiguousarray(np.stack([pts[0], np.asarray(v0, np.float64), np.asarray(a0, np.float64)]))   # Dim x 3 column-major
    tail = np.zeros((3, Dim))
    tail[0] = pts[Pn]
    inPs = np.ascontiguousarray(pts[1:Pn]).ravel()        # Dim x (P - 1) column-major == (P - 1) x Dim row-major
    c = np.zeros(6 * Pn * Dim)
    orc.orc_minco_generate(Dim, Pn, _P(inPs if inPs.size else np.zeros(1)), _P(np.full(Pn, float(dur))), _P(head.ravel()),
                           _P(np.ascontiguousarray(tail).ravel()), _P(c))
    return c


def mpc_ref(orc, message, Tx, Ty, init_v=None, init_a=None):
    """the MPC side's re-solve of a message (TrajAnalyzer::setTraj, traj_anal.hpp:125-181): (c_mpc_xy, c_mpc_yaw); init_v / init_a
    = {x, y, yaw}, None = zero"""
    v = np.zeros(3) if init_v is None else np.asarray(init_v, np.float64)
    a = np.zeros(3) if init_a is None else np.asarray(init_a, np.float64)
    cx = minco(orc, message["pos_pts"], Tx, v[:2], a[:2])
    cy = minco(orc, np.asarray(message["angle_pts"]).reshape(-1, 1), Ty, v[2:], a[2:])
    return cx, cy


def scan_times(total, dt):
    """the samples 0, dt, 2dt, .. by repeated addition (cumsum adds in order), kept while t < total"""
    n = int(total / dt) + 64
    while True:
        t = np.cumsum(np.concatenate([[0.0], np.full(n - 1, dt)]))
        if t[-1] >= total:
            return t[:int(np.searchsorted(t, total, side="left"))]
        n *= 2


def first_max(vals, t):
    """(largest value, its earliest sample time); (0, 0) when no value exceeds 0 (the kernel starts from 0 and keeps strict
    increases, so a NaN is never kept)"""
    hit = vals > 0.0
    if not hit.any():
        return 0.0, 0.0
    m = vals[hit].max()
    return float(m), float(t[int(np.argmax(vals == m))])


def deviation_samples(c_xy, c_yaw, m_xy, m_yaw, N, M, Tx, Ty, dt):
    """(sample times, position deviation, yaw deviation) of the scan, or None when the kernel does not scan"""
    total_xy, total_yaw = summed(Tx, N), summed(Ty, M)
    total = total_xy if total_xy < total_yaw else total_yaw
    if not (total / dt < DEV_GUARD):
        return None
    t = scan_times(total, dt)
    nx = 6 * N
    dx = evaluate(c_xy[:nx], N, Tx, t) - evaluate(m_xy[:nx], N, Tx, t)
    dy = evaluate(c_xy[nx:], N, Tx, t) - evaluate(m_xy[nx:], N, Tx, t)
    ep = np.sqrt(dx * dx + dy * dy)
    ey = np.abs(evaluate(c_yaw, M, Ty, t) - evaluate(m_yaw, M, Ty, t))
    return t, ep, ey


def dev_ref(c_xy, c_yaw, m_xy, m_yaw, N, M, Tx, Ty, dt):
    """dev4 of one problem: {max position deviation, its time, max yaw deviation, its time}"""
    s = deviation_samples(c_xy, c_yaw, m_xy, m_yaw, N, M, Tx, Ty, dt)
    if s is None:
        return np.array([-1.0, 0.0, -1.0, 0.0])
    t, ep, ey = s
    return np.array(first_max(ep, t) + first_max(ey, t))


def scan_length(N, M, Tx, Ty, dt):
    """total / dt as the kernel's guard forms it"""
    a, b = summed(Tx, N), summed(Ty, M)
    return (a if a < b else b) / dt


# ------------------------------------------------------------------------------------------------------ clouds
def _one_per_voxel(p):
    """float32 points, the first of each 1 cm voxel kept (the builder's VoxelGrid then returns them unchanged)"""
    p = np.asarray(p, np.float64).astype(np.float32)
    keys = np.floor(p * (np.float32(1.0) / np.float32(0.01))).astype(np.int64)
    _, first = np.unique(keys, axis=0, return_index=True)
    return np.ascontiguousarray(p[np.sort(first)])


def _lattice(cx, cy, half, step, rng, jitter=0.35):
    g = np.arange(-half, half + 1e-9, step)
    gx, gy = np.meshgrid(g, g, indexing="ij")
    x = gx.ravel() + rng.uniform(-jitter, jitter, gx.size) * step
    y = gy.ravel() + rng.uniform(-jitter, jitter, gy.size) * step
    return x, y


def terrain(kind, cx=0.0, cy=0.0, half=0.75, seed=0):
    """one scenario's cloud about (cx, cy), coordinates relative to the centre in the formulas"""
    rng = np.random.default_rng(seed)
    x, y = _lattice(0.0, 0.0, half, 0.025, rng)
    if kind == "smooth":
        z = 0.5 + 0.3 * np.sin(1.3 * x) * np.cos(0.9 * y) + rng.normal(0, 0.003, x.size)
    elif kind == "slope68":                 # 68 degrees: z rises 2.475 m per metre in x
        x, y = _lattice(0.0, 0.0, half, 0.012, rng)
        z = 2.5 + np.tan(np.radians(68.0)) * x + rng.normal(0, 0.002, x.size)
    elif kind == "step":                    # a 0.4 m step along x = 0.05
        z = np.where(x < 0.05, 0.3, 0.7) + rng.normal(0, 0.002, x.size)
    elif kind in ("sparse", "very_sparse"):  # 3 % of a 1.2 cm / 2.5 cm lattice: footprints of a few points, of one or two
        if kind == "sparse":
            x, y = _lattice(0.0, 0.0, half, 0.012, rng)
        keep = rng.uniform(size=x.size) < 0.03
        x, y = x[keep], y[keep]
        z = 0.4 + 0.2 * np.sin(2.0 * x) + rng.normal(0, 0.003, x.size)
    elif kind == "corner":                  # only the corner x, y < -0.2 of the grid
        keep = (x < -0.2) & (y < -0.2)
        x, y = x[keep], y[keep]
        z = 0.6 + 0.1 * x - 0.05 * y + rng.normal(0, 0.002, x.size)
    elif kind == "plane":                   # one exact float height
        z = np.full(x.size, 0.5)
    elif kind == "hole":
        keep = x ** 2 + (y - 0.1) ** 2 > 0.25 ** 2
        x, y = x[keep], y[keep]
        z = 0.5 + 0.3 * np.sin(1.3 * x) * np.cos(0.9 * y) + rng.normal(0, 0.003, x.size)
    elif kind == "wall":                    # a vertical wall up to 1.2 m on flat ground, along (3, 4) / 5 through the centre
        z = 0.02 + rng.uniform(0, 0.004, x.size)
        gs, gz = np.meshgrid(np.arange(-0.9, 0.9, 0.02), np.arange(0.04, 1.2, 0.02), indexing="ij")
        k = np.round((gs.ravel() + rng.uniform(-0.006, 0.006, gs.size)) * 256)   # at (0.75 k, k) / 256: on the plane 4x = 3y exactly
        x = np.concatenate([x, 0.75 * k / 256])
        y = np.concatenate([y, k / 256])
        z = np.concatenate([z, gz.ravel() + rng.uniform(-0.006, 0.006, gz.size)])
    else:
        raise ValueError(kind)
    return _one_per_voxel(np.column_stack([np.asarray(x, np.float64) + cx, np.asarray(y, np.float64) + cy, z]))


def build_ref_grid(name, cx=0.0, cy=0.0):
    from uneven_planner_b200 import _lib
    size = {"square": (1.0, 1.0, 0.05, 0.1), "fine_yaw": (0.73, 0.5, 0.04, 0.05), "coarse": (1.4, 1.2, 0.1, 0.2)}[name]
    return _lib.map_geometry_at(*size, cx, cy)


# name: (terrain, grid, centre, iter_num, ellipsoid, largest ambiguous share, largest plausibility-only share, least counts the
# scenario must reach).  The shares bound what was measured: ambiguous / plausibility-only cells of all cells, 0 / 0 on every
# scenario but wall 654 / 0 of 25600, wall_it3 93 / 0 of 5376, wall_far 1019 / 0 of 31369, sparse 21 / 18, very_sparse_it3 1310 / 1235 of
# 5376, corner 93 / 70, hole 95 / 62, corner_far 130 / 113.  Plausibility-only cells are those whose footprint was degenerate before
# the last iteration, so that every later iteration depends on an arbitrary normal.
SCENARIOS = {
    "smooth": ("smooth", "square", (0.0, 0.0), 2, (0.2, 0.1, 0.1), 0.0, 0.0, {}),
    "smooth_it1": ("smooth", "square", (0.0, 0.0), 1, (0.2, 0.1, 0.1), 0.0, 0.0, {}),
    "smooth_it3_flat_ellipsoid": ("smooth", "square", (0.0, 0.0), 3, (0.3, 0.15, 0.05), 0.0, 0.0, {}),
    "smooth_fine_yaw": ("smooth", "fine_yaw", (0.0, 0.0), 2, (0.2, 0.1, 0.1), 0.0, 0.0, {}),
    "smooth_coarse_tall_ellipsoid": ("smooth", "coarse", (0.0, 0.0), 2, (0.1, 0.1, 0.25), 0.0, 0.0, {"clamped_queries": 1}),
    "slope68": ("slope68", "square", (0.0, 0.0), 2, (0.2, 0.1, 0.1), 0.0, 0.0, {}),
    "slope68_it3": ("slope68", "square", (0.0, 0.0), 3, (0.2, 0.1, 0.1), 0.0, 0.0, {}),
    "wall": ("wall", "square", (0.0, 0.0), 2, (0.2, 0.1, 0.1), 0.03, 0.0, {"nanc_it0": 1, "ties": 1, "empty_it1": 1}),
    "wall_it3_tall_ellipsoid": ("wall", "coarse", (0.0, 0.0), 3, (0.1, 0.1, 0.25), 0.03, 0.0, {"nanc_it0": 1}),
    "step": ("step", "square", (0.0, 0.0), 2, (0.2, 0.1, 0.1), 0.0, 0.0, {}),
    "sparse": ("sparse", "square", (0.0, 0.0), 2, (0.2, 0.1, 0.1), 0.001, 0.001, {"degenerate_it0": 1}),
    "very_sparse_it3": ("very_sparse", "coarse", (0.0, 0.0), 3, (0.3, 0.15, 0.05), 0.25, 0.24, {"n1": 1, "degenerate_it2": 1, "empty_it0": 1}),
    "corner": ("corner", "square", (0.0, 0.0), 2, (0.2, 0.1, 0.1), 0.004, 0.003, {"clamped_queries": 1000, "far_nearest": 1000, "empty_it0": 1000, "n1": 1}),
    "plane": ("plane", "square", (0.0, 0.0), 2, (0.2, 0.1, 0.1), 0.0, 0.0, {}),
    "hole": ("hole", "square", (0.0, 0.0), 2, (0.2, 0.1, 0.1), 0.004, 0.003, {"empty_it0": 1}),
    "smooth_off_centre": ("smooth", "square", (31.4, -17.25), 2, (0.2, 0.1, 0.1), 0.0, 0.0, {}),
    "wall_far": ("wall", "fine_yaw", (300.0, 150.0), 2, (0.2, 0.1, 0.1), 0.035, 0.0, {"nanc_it0": 1}),
    "corner_far": ("corner", "square", (300.0, 150.0), 3, (0.1, 0.1, 0.25), 0.006, 0.005, {"clamped_queries": 1000, "far_nearest": 1000}),
}


def scenario(name):
    kind, gname, (cx, cy), iter_num, ell, share, plausible, reach = SCENARIOS[name]
    pts = terrain(kind, cx, cy)
    return dict(pts=pts, geom=build_ref_grid(gname, cx, cy), iter_num=iter_num, ellipsoid=ell, share=share, plausible=plausible, reach=reach)


_REF = {}


def reference(name):
    """(scenario, reference rows); the reference runs once per scenario and process"""
    if name not in _REF:
        s = scenario(name)
        cen, cnt, _ = mref.preprocess(s["pts"], *_centre(s["geom"]))
        assert cnt.max() == 1 and cen.shape[0] == s["pts"].shape[0]          # the cloud is its own preprocessing
        _REF[name] = (s, mref.Reference(s["pts"], s["ellipsoid"], s["iter_num"]).build(s["geom"]))
    return _REF[name]


def _centre(g):
    return (0.5 * (g.origin[0] + g.max_boundary[0]), 0.5 * (g.origin[1] + g.max_boundary[1]))


def assert_matches_reference(cells, s, rows, label=""):
    """the assertion every builder's grid is held to (the host builder here, the device builders in test_gpu_map_build_ref.py);
    returns the cells that matched only a NaN-c variant"""
    bad, nanc_only, dev = mref.compare(rows, cells)
    f = rows["features"]
    assert bad.size == 0, (label, bad.size, f, [(int(c), np.asarray(cells).reshape(-1, 4)[c]) for c in bad[:5]])
    assert dev["z_ulp"] <= 1 and dev["zbx_ulp"] <= 1 and dev["zby_ulp"] <= 1 and dev["sigma_ulp"] <= 1, (label, dev)
    assert max(dev["z_abs_small"], dev["zbx_abs_small"], dev["zby_abs_small"]) <= mref.VALUE_ABS, (label, dev)
    assert dev["sigma_abs_small"] <= mref.SIGMA_ABS, (label, dev)
    assert f["ambiguous"] <= s["share"] * f["cells"], (label, f)
    assert f["plausible_only"] <= s["plausible"] * f["cells"], (label, f)
    for k, least in s["reach"].items():
        assert f[k] >= least, (label, k, f)
    return nanc_only


def _host(s, nthreads=0):
    from uneven_planner_b200 import maps
    return maps.build_from_cloud(s["pts"], s["geom"], ellipsoid=s["ellipsoid"], iter_num=s["iter_num"], nthreads=nthreads).cells


CSRC = os.path.join(ROOT, "uneven_planner_b200", "csrc")


RHO = 8.0


# which tolerance of TOL applies to which block
KIND = dict(f="f", grad_tau="grad", grad_xy="grad", grad_yaw="grad", hx="con", hx_cancel="hx_cancel", c_xy="coef", c_yaw="coef",
            scale_fx="sfx",
            **{"gx%d" % t: "con" for t in range(6)}, **{"scale_cx%d" % t: "scx" for t in range(7)})


# hx where it is a cancellation: at an initial guess (the even problems of every batch here) the yaw waypoints follow the path
# tangent, and at int_K = 1 every sample is a waypoint, where the 1e-3 perturbation leaves the yaw within a few mrad of the tangent.
# There hx = (vx sin(yaw) - vy cos(yaw)) scale has a norm of ~1e-3 of |v| scale (N64_M128 and border_cells at their guesses,
# N2_M100 perturbed at int_K = 1), and the float kinematics carry ~1e-7 of |v| scale into it.  Worst measured at precision 32 on an
# H100: 1.4e-4 at the guesses (N64_M128, int_K 31 .. 127), 1.7e-4 perturbed at int_K = 1 (N2_M100); the perturbed points at
# int_K >= 16 measure <= 2.0e-5 and keep TOL[32], as does every other block.
TOLS = {65: dict(TOL[65], hx_cancel=TOL[65]["con"]), 32: dict(TOL[32], hx_cancel=1e-3)}


THREADS = min(32, os.cpu_count() or 1)


# ------------------------------------------------------------------ the cases
def _short_path():
    """a resampled path shorter than one piece: N = 1, M = 1, T = 0.24 s"""
    from uneven_planner_b200 import problems
    return problems.from_paths([problems.dubins([0.0, 0.0, 0.0], [0.1, 0.0, 0.0])])


def _off_map():
    """leaves the +x edge of the +-5 m maps (the parity path's edge case)"""
    from uneven_planner_b200 import problems
    return problems.from_paths([problems.dubins([4.2, 0.0, 0.0], [5.6, 0.3, 0.2])])


TP_CASES = {
    "N1_M1": lambda: _arc_problem(1, 1, arc=0.5 * np.pi),
    "N1_M128": lambda: _arc_problem(1, 128, arc=0.5 * np.pi),
    "N2_M1": lambda: _arc_problem(2, 1),
    "N2_M100": lambda: _arc_problem(2, 100),
    "N3_M40": lambda: _arc_problem(3, 40),
    "N5_M128": lambda: _arc_problem(5, 128),
    "N40_M3": lambda: _arc_problem(40, 3),
    "N13_M26": lambda: _arc_problem(13, 26),
    "N64_M128": lambda: _arc_problem(64, 128),
    "zero_boundary_rows": lambda: _arc_problem(12, 20, zero_ends=True),
    "border_cells": lambda: _arc_problem(12, 20, radius=4.99, arc=0.3, start=-0.15),      # x in [4.975, 5): the clamped last cell
    "off_map": _off_map,
    "yaw_seam": lambda: _arc_problem(10, 24, radius=2.0, arc=0.4 * np.pi, start=0.3 * np.pi),  # yaw 0.8 pi .. 1.2 pi
    "short_path": _short_path,
}


def case_batch():
    """every case twice: at its initial guess (even index) and at a perturbed point (odd index)"""
    one = cat([TP_CASES[k]() for k in TP_CASES])
    return one.select(np.repeat(np.arange(one.B), 2))


def _inputs(pb, Ks, seed=0):
    """decision vectors (odd problems perturbed), random duals (both branches of every inequality), scales, scale_fx"""
    rng = np.random.default_rng(seed)
    S = int((pb.N.astype(np.int64) * (np.asarray(Ks, np.int64) + 1)).sum())
    lam = rng.standard_normal(S) * 0.1
    mu = np.abs(rng.standard_normal(6 * S)) * 0.1 * (rng.random(6 * S) < 0.5)
    scx = rng.uniform(0.01, 1.0, 7 * S)
    sfx = rng.uniform(1e-6, 1e-3, pb.B)
    xs = np.concatenate([pb.x0(i) * (1 + (i % 2) * 1e-3 * rng.standard_normal(pb.nvar()[i])) for i in range(pb.B)])
    return xs, lam, mu, scx, sfx


def _offsets(pb, Ks):
    offx = np.concatenate([[0], np.cumsum(pb.nvar())])
    offs = np.concatenate([[0], np.cumsum(pb.N.astype(np.int64) * (np.asarray(Ks, np.int64) + 1))])
    _, _, ocx, ocy = pb.offsets()
    return offx, offs, ocx, ocy


def _per_problem(pb, Ks, ev, sfx, scx):
    """the packed outputs of a batch, split per problem"""
    offx, offs, ocx, ocy = _offsets(pb, Ks)
    return [dict(f=ev["f"][i], grad=ev["grad"][offx[i]:offx[i + 1]], hx=ev["hx"][offs[i]:offs[i + 1]], gx=ev["gx"][6 * offs[i]:6 * offs[i + 1]],
                 c_xy=ev["c_xy"][ocx[i]:ocx[i + 1]], c_yaw=ev["c_yaw"][ocy[i]:ocy[i + 1]], sfx=sfx[i], scx=scx[7 * offs[i]:7 * offs[i + 1]])
            for i in range(pb.B)]


def _oracle(pb, params, maps, Ks, inputs):
    """pyoracle eval_one and init_scaling of every problem, with problem i's parameters params[i] on maps[i]"""
    import pyoracle as po
    xs, lam, mu, scx, sfx = inputs
    offx, offs, _, _ = _offsets(pb, Ks)
    ops = {id(p): po.params_from(p) for p in params}
    oms = {id(m): po.OracleMap(m) for m in maps}

    def one(i):
        op, om = ops[id(params[i])], oms[id(maps[i])]
        o = po.eval_one(op, om, pb, i, xs[offx[i]:offx[i + 1]], lam[offs[i]:offs[i + 1]], mu[6 * offs[i]:6 * offs[i + 1]],
                        scx[7 * offs[i]:7 * offs[i + 1]], sfx[i], RHO)
        o["sfx"], o["scx"] = po.init_scaling(op, om, pb, i)
        return o
    with ThreadPoolExecutor(THREADS) as ex:
        return list(ex.map(one, range(pb.B)))


def _blocks(N, M, g, o, cancel):
    """(name, got, want, whole vector of want) for every block of one problem's outputs; cancel: hx is a cancellation (see TOLS)"""
    nxy = 2 * (N - 1)
    out = [("f", [g["f"]], [o["f"]], [o["f"]]),
           ("grad_tau", g["grad"][:1], o["grad"][:1], o["grad"]),
           ("grad_xy", g["grad"][1:1 + nxy], o["grad"][1:1 + nxy], o["grad"]),
           ("grad_yaw", g["grad"][1 + nxy:], o["grad"][1 + nxy:], o["grad"]),
           ("hx_cancel" if cancel else "hx", g["hx"], o["hx"], np.concatenate([o["hx"], o["gx"]])),
           ("c_xy", g["c_xy"], o["c_xy"], o["c_xy"]),
           ("c_yaw", g["c_yaw"], o["c_yaw"], o["c_yaw"]),
           ("scale_fx", [g["sfx"]], [o["sfx"]], [o["sfx"]])]
    out += [("gx%d" % t, g["gx"][t::6], o["gx"][t::6], np.concatenate([o["hx"], o["gx"]])) for t in range(6)]
    out += [("scale_cx%d" % t, g["scx"][t::7], o["scx"][t::7], o["scx"]) for t in range(7)]
    return out


def block_errors(pb, got, want, Ks):
    """{block: (worst relative error over the batch, problem)}; an empty block is skipped, a block that is zero up to fp64 rounding
    is measured against its whole vector"""
    worst = {}
    for i in range(pb.B):
        for name, a, b, whole in _blocks(int(pb.N[i]), int(pb.M[i]), got[i], want[i], i % 2 == 0 or Ks[i] == 1):
            a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
            if b.size == 0:
                continue
            d = float(np.linalg.norm(a - b))
            nb, nw = float(np.linalg.norm(b)), float(np.linalg.norm(np.asarray(whole, np.float64)))
            if nb <= 1e-9 * nw:
                nb = nw
            err = d / nb if nb > 0 else (0.0 if d == 0 else np.inf)
            if not np.isfinite(a).all():
                err = np.inf
            if err > worst.get(name, (-1.0, None))[0]:
                worst[name] = (err, i)
    return worst


def _check(worst, prec, what):
    tol = TOLS[prec]
    bad = {k: v for k, v in worst.items() if not v[0] <= tol[KIND[k]]}
    assert not bad, (what, bad)


def run_tp(gpu, pb, params, mapdata, precision, inputs, env=None):
    """one evaluation and initScaling of `pb` on a fresh throughput-path context, split per problem"""
    opt = ctx(gpu, precision, params, mapdata, env=env)
    opt.upload(pb)
    xs, lam, mu, scx, sfx = inputs
    ev = opt.eval_batch(xs, lam, mu, scx, sfx, rho=RHO)
    ev2 = opt.eval_batch(xs, lam, mu, scx, sfx, rho=RHO)
    s_fx, s_cx = opt.init_scaling_batch()
    opt.close()
    Ks = [params.int_K] * pb.B
    return _per_problem(pb, Ks, ev, s_fx, s_cx), _per_problem(pb, Ks, ev2, s_fx, s_cx)


def _same(a, b):
    return all(np.array_equal(np.asarray(a[k]), np.asarray(b[k])) for k in a)


# ------------------------------------------------------------------ coverage guard (no GPU)
def _define(name):
    for f in ("ualm_tp_kernels.cuh", "ualm_tp_samples.cuh"):
        with open(os.path.join(CSRC, f)) as fh:
            mt = re.search(r"^#define\s+%s\s+(\d+)" % name, fh.read(), re.M)
        if mt:
            return int(mt.group(1))
    raise AssertionError("no #define %s" % name)


def reach(pb, cxy, cyaw, geom, K):
    """what the kernels' chunk loop (kb_kernel / ks_kernel) and map lookups see for one problem at the decision vector whose
    MINCO coefficients are cxy / cyaw, with the kernels' own formulas in float64"""
    MAXPPC, YCAP, THREADS_KB = _define("TP_MAXPPC"), _define("TP_YCAP"), _define("TP_KB_THREADS")
    N, M, T = int(pb.N[0]), int(pb.M[0]), float(pb.total_time[0])
    Tx, Ty = T / N, T / M
    K1 = K + 1
    ppc = max(1, min(MAXPPC, THREADS_KB // K1))
    out = dict(ppc=ppc, partial=False, full=False, overflow=False, off_map=False, border=False, seam=False)
    vn, org, mx = geom.voxel_num, geom.origin, geom.max_boundary
    prev = None
    for p0 in range(0, N, ppc):
        np_ = min(ppc, N - p0)
        out["partial"] |= np_ < ppc
        out["full"] |= np_ * K1 == THREADS_KB
        ybase = max(0, min(int(p0 * Tx / Ty), M - 1) - 1)
        for pl in range(np_):
            i = p0 + pl
            for j in range(K1):
                s1 = j * (Tx / K)
                pw = s1 ** np.arange(6)
                x, y = float(cxy[6 * i:6 * i + 6] @ pw), float(cxy[6 * N + 6 * i:6 * N + 6 * i + 6] @ pw)
                yi = min(int((s1 + i * Tx) / Ty), M - 1)
                y1 = (s1 + i * Tx) - yi * Ty
                yaw = float(cyaw[6 * yi:6 * yi + 6] @ (y1 ** np.arange(6)))
                out["overflow"] |= yi - ybase >= YCAP
                yawn = yaw - 2 * np.pi * np.rint(yaw / (2 * np.pi))
                if prev is not None and abs(yawn - prev) > np.pi:
                    out["seam"] = True
                prev = yawn
                inside = not (x < org[0] + 1e-4 or y < org[1] + 1e-4 or yawn < org[2] + 1e-4 or x > mx[0] - 1e-4 or y > mx[1] - 1e-4 or
                              yawn > mx[2] - 1e-4)
                out["off_map"] |= not inside
                if inside:
                    i0 = int(np.floor((x - 0.5 * geom.xy_resolution - org[0]) / geom.xy_resolution))
                    i1 = int(np.floor((y - 0.5 * geom.xy_resolution - org[1]) / geom.xy_resolution))
                    out["border"] |= i0 < 0 or i1 < 0 or i0 + 1 > vn[0] - 1 or i1 + 1 > vn[1] - 1
    return out


# lbfgs return codes (oracle/oracle.cpp)
LBFGS_CONVERGENCE, LBFGS_STOP, LBFGS_CANCELED = 0, 1, 2


LBFGSERR_MINIMUMSTEP, LBFGSERR_MAXIMUMITERATION = -1011, -1008


DISCRETE = ("ret_code", "outer_iters", "n_evals", "n_lbfgs_iters", "last_lbfgs_ret", "max_bound")


CONTINUOUS = ("inner_cost", "jerk_cost", "total_T", "res_h", "res_g", "scale_fx")


# the per-trajectory rule of the throughput path against the oracle (test_gpu_solver_control.py says what was measured):
# relative perturbation of the inputs that decides a trajectory, and the bound on its continuous fields and coefficients
EPS = {65: 1e-11, 32: 1e-5}


TOLC = {65: 1e-7, 32: 1e-3}


BUDGETS = {65: [1, 2, 3, 5, 8, 13, 21, 34], 32: [1, 2, 3]}


def _p(**kw):
    from uneven_planner_b200 import _lib
    p = _lib.default_params()
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _any(pred):
    return lambda rs: any(pred(r) for r in rs)


def _all(pred):
    return lambda rs: all(pred(r) for r in rs)


# name -> (overrides of default_params(), what the oracle's records must show over the case problems)
SOLVER_CASES = {
    # the history ring wraps: a full ring (max_bound == mem_size) in inner solves of more than 2 mem_size iterations each
    "ring_m2": (dict(mem_size=2, past=0, g_epsilon=1e-12, inner_max_iter=40),
                _any(lambda r: r.max_bound == 2 and r.n_lbfgs_iters >= 40 * (r.outer_iters + 1) - 1)),
    "ring_m3": (dict(mem_size=3, past=0, g_epsilon=1e-12, inner_max_iter=60),
                _any(lambda r: r.max_bound == 3 and r.n_lbfgs_iters >= 60 * (r.outer_iters + 1) - 1)),
    "ring_m17": (dict(mem_size=17, past=0, g_epsilon=1e-12, inner_max_iter=80),
                 _any(lambda r: r.max_bound == 17 and r.n_lbfgs_iters >= 80 * (r.outer_iters + 1) - 1)),
    # the accepted maxima: more history than the yaml's 256 slots, and the 16-slot pf ring past its first wrap ending in LBFGS_STOP
    "max_mem_past": (dict(mem_size=1024, past=16),
                     lambda rs: any(r.max_bound > 256 for r in rs) and any(r.last_lbfgs_ret == LBFGS_STOP for r in rs)),
    # past 0: neither delta test (never LBFGS_STOP)
    "past0": (dict(past=0, inner_max_iter=300),
              lambda rs: all(r.last_lbfgs_ret != LBFGS_STOP for r in rs) and any(r.last_lbfgs_ret == LBFGS_CONVERGENCE for r in rs)),
    # past 1: the line search's early exit at delta / 1 and the one-slot pf ring
    "past1": (dict(past=1), _any(lambda r: r.last_lbfgs_ret == LBFGS_STOP)),
    # LBFGSERR_MAXIMUMITERATION, then the ALM loop goes on
    "inner1": (dict(inner_max_iter=1), _any(lambda r: r.last_lbfgs_ret == LBFGSERR_MAXIMUMITERATION and r.outer_iters >= 1)),
    "inner2": (dict(inner_max_iter=2), _any(lambda r: r.last_lbfgs_ret == LBFGSERR_MAXIMUMITERATION and r.outer_iters >= 1 and r.max_bound == 1)),
    # ret_code 2 after the first / second inner solve
    "max_iter0": (dict(max_iter=0), lambda rs: all(r.outer_iters <= 1 for r in rs) and any(r.ret_code == 2 and r.outer_iters == 1 for r in rs)),
    "max_iter1": (dict(max_iter=1), lambda rs: all(r.outer_iters <= 2 for r in rs) and any(r.ret_code == 2 and r.outer_iters == 2 for r in rs)),
    "max_iter0_inner1": (dict(max_iter=0, inner_max_iter=1),
                         _all(lambda r: r.outer_iters <= 1 and r.n_lbfgs_iters <= 1 and r.ret_code in (0, 2))),
    # every inner solve converges at its first evaluation (no line search at all)
    "g_eps_large": (dict(g_epsilon=1e3), _any(lambda r: r.n_lbfgs_iters == 0 and r.n_evals == r.outer_iters and r.ret_code == 2)),
    # converged at the first dual update (after a two-iteration inner solve, so that the outcome does not hinge on the trajectory)
    "eps_con_large": (dict(epsilon_con=1e6, inner_max_iter=2),_all(lambda r: r.ret_code == 0 and r.outer_iters == 0)),
    # rho reaches the cap beta
    "beta_cap": (dict(beta=3.0), _any(lambda r: r.rho_final == 3.0 and r.outer_iters >= 2)),
    # a hard line-search error: ret_code 1 before any dual update
    "min_step_large": (dict(min_step=1e3),
                       _all(lambda r: r.ret_code == 1 and r.last_lbfgs_ret == LBFGSERR_MINIMUMSTEP and r.outer_iters == 0 and r.rho_final == 1.0)),
    # LBFGS_STOP within a few iterations of every inner solve
    "delta_large": (dict(delta=0.5), _any(lambda r: r.last_lbfgs_ret == LBFGS_STOP and r.n_lbfgs_iters <= 5 * (r.outer_iters + 1))),
}


# the cases whose outcome is fixed by their structure rather than by the trajectory: the only ones precision 32 is compared at
STRUCTURAL = ("max_iter0_inner1", "g_eps_large", "eps_con_large")


# evaluation budget of the cases where the throughput path is compared with the oracle at precision 65: long enough for the case to
# reach its branch (ring_m17 fills its ring, max_mem_past wraps its pf ring), short enough that most trajectories stay decided
CASE_BUDGET = dict({c: 40 for c in SOLVER_CASES}, ring_m2=20, ring_m3=20)


def case_budget(name, prec):
    return CASE_BUDGET[name] if prec == 65 else 0


def case_params(name):
    return _p(**SOLVER_CASES[name][0])


def case_problems(bumps, hill):
    """[(label, map, batch)]: generated problems on the bumps map and on the hill terrain, and the edge shapes on the bumps map"""
    from uneven_planner_b200 import configs, problems
    shapes = problems.concat([TP_CASES[k]() for k in ("N1_M1", "N64_M128", "off_map")], [0, 0, 0])
    shapes.env = None
    gb = problems.generate(bumps, 6, seed=7)
    gh = problems.generate(hill, 6, seed=11, **configs.gen_kwargs("hill"))
    both = problems.concat([gb, shapes], [0, 0])
    both.env = None
    return [("bumps", bumps, both), ("hill", hill, gh)]


def bench_problems(hill, B):
    """the first B problems of the bench's workload (BASELINE config 2, hill parameters, seed 0)"""
    from uneven_planner_b200 import configs, problems
    return problems.generate(hill, B, seed=0, **configs.gen_kwargs("hill"))


def perturb(pb, eps, seed):
    """pb with its inner waypoints and total time moved by a relative eps in a seeded random direction"""
    import copy
    rng = np.random.default_rng(seed)
    out = copy.copy(pb)
    for f in ("inner_xy", "inner_yaw", "total_time"):
        a = np.asarray(getattr(pb, f), np.float64)
        setattr(out, f, a + eps * np.maximum(np.abs(a), 1.0) * rng.choice([-1.0, 1.0], a.shape))
    return out


def oracle(params, mapdata, pb, max_evals=0):
    """stop_oracle's budget (max_evals 0: the oracle's own solve) of every problem: [(record, c_xy, c_yaw)]"""
    import pyoracle as po
    out = so.budget_batch(po.params_from(params), po.OracleMap(mapdata), pb, max_evals, threads=THREADS)
    return [(r, cxy, cyaw) for r, cxy, cyaw, _ in out]


def _rel_floor(a, b, floor):
    return abs(float(a) - float(b)) / max(abs(float(b)), floor)


def trajectory_error(got, want):
    """(discrete fields and rho_final all equal, worst relative error of the continuous fields and coefficients) of one trajectory.
    A residual is measured against max(|oracle|, 1e-6) (near zero it is a cancellation), everything else against its own size."""
    g, gx, gy = got
    w, wx, wy = want
    same = all(getattr(g, f) == getattr(w, f) for f in DISCRETE) and g.rho_final == w.rho_final
    err = max(_rel_floor(getattr(g, f), getattr(w, f), 1e-6 if f in ("res_h", "res_g") else 1e-300) for f in CONTINUOUS)
    for a, b in ((gx, wx), (gy, wy)):
        err = max(err, float(np.linalg.norm(np.asarray(a) - b) / max(np.linalg.norm(b), 1e-300)))
    if not np.isfinite(err):
        err = np.inf
    return same, err


def agrees(got, want, prec):
    same, err = trajectory_error(got, want)
    return same and err <= TOLC[prec]


def decided(params, mapdata, pb, prec, max_evals=0):
    """(oracle solves, boolean mask of the decided trajectories): three runs from seeded perturbations of the inputs by EPS[prec]
    all agree with the unperturbed run under the same rule the GPU is held to"""
    ref = oracle(params, mapdata, pb, max_evals)
    mask = np.ones(pb.B, bool)
    for s in range(3):
        alt = oracle(params, mapdata, perturb(pb, EPS[prec], 1000 + s), max_evals)
        mask &= np.array([agrees(alt[i], ref[i], prec) for i in range(pb.B)])
    return ref, mask


ALM_INT_K = [1, 16, 64, 127]


TERRAINS = ["hill", "desert", "volcano", "forest"]


# the bounds, about 10x the worst relative error measured over the whole table (restatement against the oracle, x86-64):
#   f 8.9e-14 (N1_M128 at its guess); gradient 3.6e-12 (tau part, forest), 7.3e-13 (yaw waypoints), 6.6e-13 (xy waypoints, forest);
#   hx 6.5e-12, a cancellation: at an initial guess the yaw follows the path tangent and hx ~ 1e-3 |v| (border_cells);
#   gx 1.0e-13 (curvature, volcano); c_xy 3.8e-14, c_yaw 5.3e-13 (N1_M128); scale_fx 8.2e-14 (forest);
#   scale_cx 9.5e-12 entry by entry (lateral acceleration, volcano)
ALM_TOL = dict(f=1e-12, grad=4e-11, hx=1e-10, hx_cancel=1e-10, con=1e-12, coef=5e-12, sfx=1e-12, scx=1e-10)


LOOSE = 1e-3            # f and gradient of a problem that holds a near-face sample


ALM_KIND = dict(f="f", grad_tau="grad", grad_xy="grad", grad_yaw="grad", hx="hx", hx_cancel="hx_cancel", c_xy="coef", c_yaw="coef", scale_fx="sfx",
            **{"gx%d" % t: "con" for t in range(6)}, **{"scale_cx%d" % t: "scx" for t in range(7)})


# ------------------------------------------------------------------ the table
def alm_pairs(pb):
    """every problem twice: at its initial guess (even index) and at a perturbed point (odd index)"""
    return pb.select(np.repeat(np.arange(pb.B), 2))


def alm_cases():
    """test_gpu_tp_shapes' case batch and a fast tight turn (4 m/s on a 0.8 m radius: 20 m/s^2 lateral), where the lateral
    acceleration limit is active, each at its guess and perturbed"""
    fast = alm_pairs(_arc_problem(8, 16, radius=0.8, arc=np.pi, speed=4.0))
    return cat([case_batch(), fast])


def ridge():
    """a corrugated grid: the normal tilts by up to 37 degrees in x with a 1 m period, so that cos_xi has a large gradient and, on the
    one-piece problems (x = tau alone), initScaling's attitude scales are set by their tau component"""
    from uneven_planner_b200 import _lib, maps
    g = _lib.map_geometry()
    X, Y, W = g.voxel_num
    xs = (np.arange(X) + 0.5) * g.xy_resolution + g.origin[0]
    cells = np.zeros((X, Y, W, 4), np.float32)
    cells[..., 1] = (0.02 * (1.0 + np.cos(2 * np.pi * xs)))[:, None, None]
    cells[..., 2] = (0.6 * np.sin(2 * np.pi * xs))[:, None, None]
    return maps.UnevenMapData(g, cells, "ridge")


def table_entry(key, terrain, bumps_map):
    """(batch, params, grid) of one entry of the case table"""
    from uneven_planner_b200 import _lib, configs, maps, problems
    if key.startswith("K"):
        p = _lib.default_params()
        p.int_K = int(key[1:])
        return alm_cases(), p, bumps_map
    if key in TERRAINS:
        return alm_cases(), configs.params_for(key), terrain(key)
    if key == "tilt":
        return alm_cases(), _lib.default_params(), maps.synthetic_terrain("tilt")
    if key == "ridge":
        return alm_cases(), _lib.default_params(), ridge()
    assert key == "generated"
    gen = [problems.generate(bumps_map, 6, seed=23), problems.generate(terrain("hill"), 6, seed=29, **configs.gen_kwargs("hill"))]
    return alm_pairs(cat(gen)), _lib.default_params(), None


KEYS = ["K%d" % k for k in ALM_INT_K] + TERRAINS + ["tilt", "ridge", "generated"]


def restated(pb, params, mapdata, Ks, inputs):
    """the restatement's evaluation at `inputs` and initScaling at the initial guess of every problem (problem i with params[i] on
    mapdata[i]), in the layout of _per_problem, plus the per-sample flags"""
    xs, lam, mu, scx, sfx = inputs
    offx, offs, _, _ = _offsets(pb, Ks)
    grids = {id(m): ar.Grid(m) for m in mapdata}
    out = []
    for i in range(pb.B):
        prob, p, g = ar.Problem(pb, i), params[i], grids[id(mapdata[i])]
        r = ar.evaluate(prob, p, g, xs[offx[i]:offx[i + 1]], lam[offs[i]:offs[i + 1]], mu[6 * offs[i]:6 * offs[i + 1]],
                        scx[7 * offs[i]:7 * offs[i + 1]], sfx[i], RHO)
        if i % 2 == 1 and np.array_equal(pb.bnd[i], pb.bnd[i - 1]) and np.array_equal(pb.x0(i), pb.x0(i - 1)):
            r["sfx"], r["scx"], r["near_face_scaling"] = out[i - 1]["sfx"], out[i - 1]["scx"], out[i - 1]["near_face_scaling"]
        else:                                   # the perturbed twin of a problem shares its initial guess and so its initScaling
            r["sfx"], r["scx"], r["near_face_scaling"] = ar.init_scaling(prob, p, g)
        out.append(r)
    return out


# ------------------------------------------------------------------ the comparison
def _alm_blocks(N, g, o, cancel=False):
    """(name, got, want, whole vector of want, per-entry) for every block of one problem's outputs; cancel: hx is a cancellation
    (TOLS) and is reported as hx_cancel"""
    nxy = 2 * (N - 1)
    con = np.concatenate([o["hx"], o["gx"]])
    out = [("f", [g["f"]], [o["f"]], [o["f"]], False),
           ("grad_tau", g["grad"][:1], o["grad"][:1], o["grad"], False),
           ("grad_xy", g["grad"][1:1 + nxy], o["grad"][1:1 + nxy], o["grad"], False),
           ("grad_yaw", g["grad"][1 + nxy:], o["grad"][1 + nxy:], o["grad"], False),
           ("hx_cancel" if cancel else "hx", g["hx"], o["hx"], con, False),
           ("c_xy", g["c_xy"], o["c_xy"], o["c_xy"], False),
           ("c_yaw", g["c_yaw"], o["c_yaw"], o["c_yaw"], False),
           ("scale_fx", [g["sfx"]], [o["sfx"]], [o["sfx"]], False)]
    out += [("gx%d" % t, g["gx"][t::6], o["gx"][t::6], con, False) for t in range(6)]
    out += [("scale_cx%d" % t, g["scx"][t::7], o["scx"][t::7], o["scx"], True) for t in range(7)]
    return out


def alm_block_errors(pb, got, want, near=None, cancel=None, entrywise_scales=True):
    """{block: (worst relative error over the batch, problem)}.  A block is measured by the norm of its difference over its own
    norm; a block that is zero up to fp64 rounding (below 1e-9 of its whole vector) against its whole vector; scale_cx entry by
    entry.  near[i]: problem i's near-face samples (a bool per sample), left out of the per-sample blocks; the error of f and the
    gradient of such a problem is reported under "<block>_near".  entrywise_scales=False: scale_cx by norm too, the measure
    TOLS bound for the float kernels """
    worst = {}
    for i in range(pb.B):
        N = int(pb.N[i])
        nf = None if near is None else np.asarray(near[i], bool)
        for name, a, b, whole, entrywise in _alm_blocks(N, got[i], want[i], cancel is not None and cancel[i]):
            a = np.asarray(a, np.float64)
            b = np.asarray(b, np.float64)
            whole = np.asarray(whole, np.float64)
            if nf is not None and nf.any():
                if name.startswith(("hx", "gx", "scale_cx")):
                    keep = ~nf
                    a, b = a[keep], b[keep]
                elif name.startswith(("f", "grad")):
                    name += "_near"
            if b.size == 0:
                continue
            if entrywise and entrywise_scales:
                err = float(np.max(np.abs(a - b) / np.abs(b)))
            else:
                d = float(np.linalg.norm(a - b))
                nb, nw = float(np.linalg.norm(b)), float(np.linalg.norm(whole))
                if nb <= 1e-9 * nw:
                    nb = nw
                err = d / nb if nb > 0 else (0.0 if d == 0 else np.inf)
            if not np.isfinite(a).all():
                err = np.inf
            if err > worst.get(name, (-1.0, None))[0]:
                worst[name] = (err, i)
    return worst


def alm_check(worst, tol, loose, what):
    bad = {k: v for k, v in worst.items()
           if not v[0] <= (loose if k.endswith("_near") else tol[ALM_KIND[k]])}
    assert not bad, (what, bad)


def near_face(ref):
    """per problem: the samples near a cell face in the evaluation or in initScaling"""
    return [r["near_face"] | r["near_face_scaling"] for r in ref]


SHAPES = {"N64_M128": (64, 128), "N63_M127": (63, 127), "N48_M128": (48, 128), "N64_M64": (64, 64), "N64_M1": (64, 1),
          "N1_M128": (1, 128), "N2_M1": (2, 1), "N1_M1": (1, 1)}


def _shape(N, M):
    return _arc_problem(N, M, arc=0.5 * np.pi if N == 1 else 1.5 * np.pi)


DT = 0.01


BATCH_CASES = ("border_x", "border_y", "off_x", "off_y", "off_lo_x", "off_lo_y", "yaw_seam")


# ------------------------------------------------------------------ batches
def hand_cases(geom):
    """problems placed from the grid's own bounds: an arc inside the last cell column in x / in y (clamped upper neighbours), paths
    that leave through the +x, +y, -x and -y sides (the last two pass the clamped first cells on their way), and an arc whose yaw
    runs over +-pi"""
    from uneven_planner_b200 import problems
    bx, by = geom.max_boundary[0], geom.max_boundary[1]
    ox, oy = geom.origin[0], geom.origin[1]
    return {
        "border_x": _arc_problem(12, 20, radius=4.99, arc=0.3, start=-0.15, centre=(bx - 5.0, 0.1)),
        "border_y": _arc_problem(12, 20, radius=4.99, arc=0.3, start=0.5 * np.pi - 0.15, centre=(-0.1, by - 5.0)),
        "off_x": problems.from_paths([problems.dubins([bx - 0.8, 0.0, 0.0], [bx + 0.6, 0.3, 0.2])]),
        "off_y": problems.from_paths([problems.dubins([0.2, by - 0.8, 0.5 * np.pi], [-0.1, by + 0.6, 0.5 * np.pi + 0.2])]),
        "off_lo_x": problems.from_paths([problems.dubins([ox + 0.8, 0.3, np.pi], [ox - 0.6, 0.1, np.pi - 0.2])]),
        "off_lo_y": problems.from_paths([problems.dubins([-0.3, oy + 0.8, -0.5 * np.pi], [0.1, oy - 0.6, -0.5 * np.pi + 0.2])]),
        "yaw_seam": _arc_problem(10, 24, radius=2.0, arc=0.4 * np.pi, start=0.3 * np.pi),      # yaw 0.8 pi .. 1.2 pi
    }


def generated(m, n, seed):
    from uneven_planner_b200 import problems
    g = m.geom
    return problems.generate(m, n, seed=seed, lo=(g.origin[0] + 0.5, g.origin[1] + 0.5), hi=(g.max_boundary[0] - 0.5, g.max_boundary[1] - 0.5))


def _parity_evaluation(opt, pb, params, oracle_map, seed=0):
    """one evaluation at random duals and a perturbed point, and initScaling, of the parity context `opt` against the oracle on
    `oracle_map`: bit for bit.  Returns the evaluation, with the oracle's constraint values of every problem as `oracle_gx`"""
    import pyoracle as po
    K = params.int_K
    inputs = _inputs(pb, [K] * pb.B, seed=seed)
    xs, lam, mu, scx, sfx = inputs
    offx, offs, ocx, ocy = _offsets(pb, [K] * pb.B)
    opt.upload(pb)
    ev = opt.eval_batch(xs, lam, mu, scx, sfx, rho=RHO)
    s_fx, s_cx = opt.init_scaling_batch()
    op, om = po.params_from(params), po.OracleMap(oracle_map)
    ev["oracle_gx"] = []
    for i in range(pb.B):
        o = po.eval_one(op, om, pb, i, xs[offx[i]:offx[i + 1]], lam[offs[i]:offs[i + 1]], mu[6 * offs[i]:6 * offs[i + 1]],
                        scx[7 * offs[i]:7 * offs[i + 1]], sfx[i], RHO)
        ev["oracle_gx"].append(o["gx"].tobytes())
        assert ev["f"][i] == o["f"], i
        assert np.array_equal(ev["grad"][offx[i]:offx[i + 1]], o["grad"]), i
        assert np.array_equal(ev["hx"][offs[i]:offs[i + 1]], o["hx"]) and np.array_equal(ev["gx"][6 * offs[i]:6 * offs[i + 1]], o["gx"]), i
        assert np.array_equal(ev["c_xy"][ocx[i]:ocx[i + 1]], o["c_xy"]) and np.array_equal(ev["c_yaw"][ocy[i]:ocy[i + 1]], o["c_yaw"]), i
        osfx, oscx = po.init_scaling(op, om, pb, i)
        assert s_fx[i] == osfx and np.array_equal(s_cx[7 * offs[i]:7 * offs[i + 1]], oscx), i
    return ev


def _scan_and_check(opt, m, params, pb, out):
    """the lane's scan against orc_feasibility, and ualm_check_trajectories from t = 0 and from mid-trajectory against
    tests/check_oracle.cpp, on the coefficients and piece durations of `out`: bit for bit"""
    import pyoracle as po
    from check_oracle import check, limits_of
    res, cxy, cyaw = out
    feas = opt.feasibility(DT)
    om = po.OracleMap(m)
    _, _, ocx, ocy = pb.offsets()
    total = np.zeros(pb.B)
    for i in range(pb.B):
        r, N, M = res[i], int(pb.N[i]), int(pb.M[i])
        assert r.piece_T_xy == feas[i, 8] and r.piece_T_yaw == feas[i, 9], i
        ref = po.feasibility(om, params.gravity, N, M, cxy[ocx[i]:ocx[i + 1]], cyaw[ocy[i]:ocy[i + 1]], r.piece_T_xy, r.piece_T_yaw, DT)
        assert np.array_equal(feas[i, :8], ref), (i, feas[i, :8], ref)
        total[i] = min(N * r.piece_T_xy, M * r.piece_T_yaw)
    for tf in (np.zeros(pb.B), 0.4 * total):
        got = opt.check_results(pb, out, t_from=tf)
        for i in range(pb.B):
            ref = check(om, params.gravity, int(pb.N[i]), int(pb.M[i]), cxy[ocx[i]:ocx[i + 1]], cyaw[ocy[i]:ocy[i + 1]], res[i].piece_T_xy,
                        res[i].piece_T_yaw, DT, tf[i], limits_of(params))
            assert np.array_equal(bits(got[i]), bits(ref)), (i, tf[i], got[i], ref)
        if not tf.any():
            assert np.array_equal(bits(got[:, :10]), bits(feas))
        else:
            assert np.all(got[:, 7] < feas[:, 7]) and np.all(got[:, 7] > 0)
