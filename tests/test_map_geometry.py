"""Every host-side consumer of the SE(2) map grid on grids that are not the 10 m square: X != Y, other resolutions, odd cell counts
and an odd number of yaw layers (GRIDS below; tests/test_gpu_map_geometry.py runs the device side on the same table).

What each comparison is:
  * the oracle's map query (orc_map_query) against ref_query, a float64 numpy restatement of UnevenMap::getAllWithGrad
    (uneven_map.h:258-377) that indexes cells[x, y, w] as an array instead of computing addresses: 1e-12 relative (the oracle's
    sin / cos / atan2 are include/ualm_detmath.h's, numpy's are libm's), the in / out decision exact; ref_query's 21 gradients are
    themselves held up by central differences;
  * ualm_map_occupancy against three lines of numpy, the .umap file against itself, window_box against the grid's bounds: exact;
  * ualm_map_build on a 4 m x 2 m grid against the rows it shares with the 4 m x 4 m grid of the same cloud: 2 float ulps, but
    for a measured share of cells (see test_host_builder_rectangle_shares_its_rows_with_the_square);
  * the front end on `wide` and `tall`: properties of the returned paths only -- there is no second implementation to compare with
    where the reference's sources are absent."""
import ctypes as C
import os

import numpy as np
import pytest

from workloads import GRIDS, OUTSIDE, SMALL, _norm_so2, geometry, grid, in_map, query_poses, ref_query


def test_grid_table(built):
    """the cell counts the table states, and a terrain that a swapped x / y index cannot map onto itself"""
    for name, (sx, sy, rxy, ryaw, cells, _) in GRIDS.items():
        g = geometry(name)
        assert tuple(g.voxel_num) == cells, name
        assert (g.origin[0], g.origin[1], g.max_boundary[0], g.max_boundary[1]) == (-sx / 2, -sy / 2, sx / 2, sy / 2), name
        m = grid(name)
        n = min(cells[0], cells[1])
        sq = m.cells[:n, :n]
        assert m.shape == cells and np.isfinite(m.cells).all()
        # not symmetric under x <-> y: more than half of the square sub-block's cells differ from their transpose
        assert (sq != sq.transpose(1, 0, 2, 3)).any(axis=(2, 3)).mean() > 0.5, name
        # every row and every column carries slope in both directions (the seeds are chosen so): no border cell is flat ground,
        # where a wrong index would read the same zeros
        for k in (2, 3):
            assert m.cells[..., k].std(axis=(1, 2)).min() > 1e-3 and m.cells[..., k].std(axis=(0, 2)).min() > 1e-3, (name, k)


def test_default_terrain_and_generator_keep_their_bits(built):
    """geom=None is the 10 m square as before, a square geometry given explicitly gives the same cells, and scalar lo / hi draw the
    same problems as the pair (the committed golden files pin the absolute bits)"""
    from uneven_planner_b200 import _lib, maps, problems
    a, b = maps.synthetic_terrain("hills", seed=101), maps.synthetic_terrain("hills", seed=101, geom=_lib.map_geometry())
    assert a.shape == (200, 200, 64) and np.array_equal(a.cells.view(np.uint32), b.cells.view(np.uint32))
    p, q = problems.generate(a, 6, seed=5, lo=-4.0, hi=4.0), problems.generate(a, 6, seed=5, lo=(-4.0, -4.0), hi=(4.0, 4.0))
    assert np.array_equal(p.bnd, q.bnd) and np.array_equal(p.inner_xy, q.inner_xy) and np.array_equal(p.inner_yaw, q.inner_yaw)


@pytest.mark.parametrize("name", list(GRIDS))
def test_oracle_map_query_matches_the_plain_reference(built, name):
    import pyoracle as po
    m = grid(name)
    om = po.OracleMap(m)
    poses = query_poses(m.geom, seed=GRIDS[name][5])
    inside = seam = terrain = 0
    W = m.geom.voxel_num[2]
    for p in poses:
        v, g = om.query(p)
        rv, rgr = ref_query(m.cells, m.geom, p)
        if not in_map(m.geom, p):
            assert np.array_equal(v, OUTSIDE) and not g.any(), p
            assert np.array_equal(rv, OUTSIDE) and not rgr.any(), p
            continue
        inside += 1
        seam += int(np.floor((_norm_so2(p[2] - 0.5 * m.geom.yaw_resolution) - m.geom.origin[2]) / m.geom.yaw_resolution)) == W - 1
        terrain += not np.array_equal(v, OUTSIDE)
        assert np.abs(v - rv).max() <= 1e-12 * np.linalg.norm(rv), (p, v, rv)
        for r in range(7):
            assert np.abs(g[r] - rgr[r]).max() <= 1e-12 * max(np.linalg.norm(rgr[r]), 1e-3 * np.linalg.norm(rgr)), (p, r, g[r], rgr[r])
    # poses on both sides of the in / out decision (which the oracle and ref_query took alike at every pose: outside is exact), on
    # sloping ground, and with the seam's layer pair
    assert inside > 1500 and len(poses) - inside > 50 and terrain > 0.75 * inside and seam >= 2


@pytest.mark.parametrize("name", SMALL)
def test_reference_gradients_are_the_derivatives_of_its_values(built, name):
    """central differences of ref_query's values at poses away from the cell faces (the field is trilinear between cell centres)"""
    m = grid(name)
    g = m.geom
    rng = np.random.default_rng(GRIDS[name][5])
    o, b = np.array(list(g.origin)), np.array(list(g.max_boundary))
    res = np.array([g.xy_resolution, g.xy_resolution, g.yaw_resolution])
    done = 0
    while done < 60:
        p = np.array([rng.uniform(o[0] + 0.1, b[0] - 0.1), rng.uniform(o[1] + 0.1, b[1] - 0.1), rng.uniform(-3.0, 3.0)])
        frac = ((p - o) / res - 0.5) % 1.0
        if np.any(frac < 0.05) or np.any(frac > 0.95):
            continue
        done += 1
        _, gr = ref_query(m.cells, g, p)
        for k in range(3):
            h = np.zeros(3)
            h[k] = 1e-6
            fd = (ref_query(m.cells, g, p + h)[0] - ref_query(m.cells, g, p - h)[0]) / 2e-6
            assert np.all(np.abs(fd - gr[:, k]) <= 1e-5 * np.abs(gr[:, k]) + 1e-8), (p, k, fd, gr[:, k])


# ------------------------------------------------------------------ 1b. occupancy
@pytest.mark.parametrize("name", list(GRIDS))
def test_occupancy_matches_numpy(built, name):
    from uneven_planner_b200 import maps
    base = grid(name)
    cells = base.cells.copy()
    X, Y, W = base.shape
    sig = np.sort(cells[..., 1].ravel())
    max_rho = float(sig[int(0.9 * sig.size)])                         # a tenth of the cells too rough
    # a cell whose zb is just over unit length: c is NaN, `c < min_cnormal` is false, and the cell stays free by the first term
    nan_cell = (X - 2, 1, W - 1)
    cells[nan_cell] = (0.0, 0.0, 1.0, 1e-3)
    steep = (1, Y - 2, 0)
    cells[steep] = (0.0, 0.0, 0.7, 0.0)                               # c = 0.714 < 0.8
    m = maps.UnevenMapData(base.geom, cells, name)
    occ3, occ2 = m.occupancy(0.8, max_rho)
    c64 = cells.astype(np.float64)
    with np.errstate(invalid="ignore"):
        c = np.sqrt(1.0 - c64[..., 2] ** 2 - c64[..., 3] ** 2)
        want3 = (c < 0.8) | (c64[..., 1] > max_rho)
    assert np.isnan(c[nan_cell]) and not want3[nan_cell] and want3[steep]
    assert np.array_equal(occ3.astype(bool), want3) and np.array_equal(occ2.astype(bool), want3.any(axis=2))
    assert 0.05 < want3.mean() < 0.5 and not occ2.all()


# ------------------------------------------------------------------ 1c. the .umap file and window_box
@pytest.mark.parametrize("name", list(GRIDS))
def test_umap_round_trip(built, tmp_path, name):
    from uneven_planner_b200 import maps
    m = grid(name)
    path = str(tmp_path / (name + ".umap"))
    m.save(path)
    assert os.path.getsize(path) == 64 + m.cells.nbytes
    back = maps.UnevenMapData.load(path)
    assert bytes(back.geom) == bytes(m.geom)
    assert np.array_equal(back.cells.view(np.uint32), m.cells.view(np.uint32))


@pytest.mark.parametrize("name", list(GRIDS))
def test_window_box_on_a_rectangle(built, name):
    from uneven_planner_b200 import maps
    g = geometry(name)
    X, Y, _ = g.voxel_num
    o, b, r = g.origin, g.max_boundary, g.xy_resolution
    # rectangles 1.0 m x 0.4 m (x by y) reaching over each edge and the far corner, and one inside
    cases = {"x0": (o[0] - 1.0, 0.1, o[0] + 1.0, 0.5), "x1": (b[0] - 1.0, 0.1, b[0] + 1.0, 0.5), "y0": (0.1, o[1] - 0.2, 1.1, o[1] + 0.4),
             "y1": (0.1, b[1] - 0.4, 1.1, b[1] + 0.2), "far": (b[0] - 0.97, b[1] - 0.38, b[0] + 3.0, b[1] + 3.0), "in": (0.1, 0.1, 1.1, 0.5)}
    for what, rect in cases.items():
        ix0, iy0, nx, ny = maps.window_box(g, *rect)
        assert 0 <= ix0 and ix0 + nx <= X and 0 <= iy0 and iy0 + ny <= Y and nx > 0 and ny > 0 and nx != ny, (what, ix0, iy0, nx, ny)
        # the box holds the rectangle's corners (clipped to the grid) and no cell column beyond them
        x0, x1, y0, y1 = max(rect[0], o[0]), min(rect[2], b[0] - 1e-9), max(rect[1], o[1]), min(rect[3], b[1] - 1e-9)
        assert o[0] + ix0 * r <= x0 + 1e-9 and x1 <= o[0] + (ix0 + nx) * r + 1e-9 and x0 >= o[0] + ix0 * r - 1e-9 and x1 >= o[0] + (ix0 + nx - 1) * r - 1e-9, what
        assert o[1] + iy0 * r <= y0 + 1e-9 and y1 <= o[1] + (iy0 + ny) * r + 1e-9 and y0 >= o[1] + iy0 * r - 1e-9 and y1 >= o[1] + (iy0 + ny - 1) * r - 1e-9, what
    fx, fy = int((b[0] - 0.97 - o[0]) / r), int((b[1] - 0.38 - o[1]) / r)
    assert maps.window_box(g, *cases["far"]) == (fx, fy, X - fx, Y - fy)
    assert maps.window_box(g, *cases["x0"])[0] == 0 and maps.window_box(g, *cases["y0"])[1] == 0
    with pytest.raises(ValueError):
        maps.window_box(g, 0.0, b[1] + 0.5, 1.0, b[1] + 1.0)          # beyond y only
    with pytest.raises(ValueError):
        maps.window_box(g, b[0] + 0.5, 0.0, b[0] + 1.0, 1.0)          # beyond x only


# ------------------------------------------------------------------ 1d. the host builder
def ulp_distance(a, b):
    """distance in float32 steps between two float32 arrays (signed zeros coincide)"""
    def key(x):
        i = np.ascontiguousarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(key(a) - key(b))


@pytest.mark.parametrize("axis", [0, 1])
def test_host_builder_rectangle_shares_its_rows_with_the_square(built, axis):
    """ualm_map_build of one cloud on a 4 m x 2 m (axis 1) or 2 m x 4 m (axis 0) grid and on the 4 m x 4 m grid: the cells both grids
    hold are the same cells.  Their origins differ on the short axis (-1 against -2), so a cell centre can differ in its last bit and
    a cloud point on an ellipsoid's surface can change sides, which moves that cell's mean and covariance: up to 0.02 % of the cells
    may differ by more than 2 float ulps (the share tests/test_ref_pin.py allows at the rim of a hole).  Measured on an x86-64 host
    (the builder runs on host threads), both ways round: no cell of the 204 800 differs in any bit."""
    from workloads import _cloud
    from uneven_planner_b200 import _lib, maps
    pts = _cloud(60000, 2.3, 0)
    size = [4.0, 4.0]
    size[axis] = 2.0
    rect = maps.build_from_cloud(pts, _lib.map_geometry(size[0], size[1], 0.05, 0.1))
    square = maps.build_from_cloud(pts, _lib.map_geometry(4.0, 4.0, 0.05, 0.1))
    assert rect.shape == ((40, 80, 64) if axis == 0 else (80, 40, 64)) and square.shape == (80, 80, 64)
    shared = square.cells[20:60] if axis == 0 else square.cells[:, 20:60]
    d = ulp_distance(rect.cells, shared).max(axis=-1)
    share = (d > 2).mean()
    assert share <= 2e-4, share
    # and a wrong row offset or stride is not within that share: the neighbouring rows are nowhere near
    off = square.cells[21:61] if axis == 0 else square.cells[:, 21:61]
    assert (ulp_distance(rect.cells, off).max(axis=-1) > 2).mean() > 0.5


# ------------------------------------------------------------------ 1e. the front end (a property test: no reference to compare with)
def _front_end_view(name):
    from uneven_planner_b200 import front_end
    m = grid(name)
    sig = np.sort(m.cells[..., 1].ravel())
    return front_end.MapView(m, 0.8, float(sig[int(0.97 * sig.size)]))


def _pairs(name, n, seed):
    g = geometry(name)
    rng = np.random.default_rng(seed)
    lo = np.array([g.origin[0] + 0.5, g.origin[1] + 0.5, -np.pi])
    hi = np.array([g.max_boundary[0] - 0.5, g.max_boundary[1] - 0.5, np.pi])
    return rng.uniform(lo, hi, (n, 3)), rng.uniform(lo, hi, (n, 3))


@pytest.mark.parametrize("name", ["wide", "tall"])
def test_front_end_paths_on_a_rectangle(built, name):
    """KinoAstar on a grid with X != Y: every returned path starts at the requested pose and ends at the goal, stays inside the
    rectangle but for the closing one-shot, keeps off the occupied columns, some pairs span most of the long axis, and the batch
    does not depend on the thread count"""
    from uneven_planner_b200 import front_end
    view = _front_end_view(name)
    g = view.geom
    X, Y, _ = g.voxel_num
    assert 0.02 < view.occ2.mean() < 0.6
    starts, goals = _pairs(name, 40, GRIDS[name][5])
    pb1, packed1, nexp1 = front_end.plan_batch(view, starts, goals, nthreads=1)
    pb3, packed3, nexp3 = front_end.plan_batch(view, starts, goals, nthreads=3)
    assert np.array_equal(packed1, packed3) and np.array_equal(nexp1, nexp3)
    for f in ("N", "M", "bnd", "total_time", "inner_xy", "inner_yaw"):
        assert np.array_equal(getattr(pb1, f), getattr(pb3, f)), f
    assert pb1.B >= 10
    long_axis = 0 if name == "wide" else 1
    spans, points, touched = [], 0, 0
    for b in np.flatnonzero(packed1 >= 0):
        path, _ = front_end.plan(view, starts[b], goals[b])
        assert len(path) >= 2
        # the one-shot that closes a path is sampled every collision_interval (0.06 m): its last sample is within that of the goal
        assert np.array_equal(path[0], starts[b]) and np.hypot(*(path[-1, :2] - goals[b, :2])) < 0.06 + 1e-9, b
        assert abs(_norm_so2(path[-1, 2] - goals[b, 2])) < 0.06 / 0.26, b
        ix = np.floor((path[:, 0] - g.origin[0]) / g.xy_resolution).astype(int)
        iy = np.floor((path[:, 1] - g.origin[1]) / g.xy_resolution).astype(int)
        # the search's nodes are inside the map; the one-shot's arcs are only tested for occupied cells, as in the reference, and
        # may swing outside near the goal.  Measured on these pairs: at most 0.36 m beyond the edge, and no point outside is further
        # than 1.43 m from its goal (the one-shot starts within oneshot_range = 1 m of it)
        inside = (ix >= 0) & (ix < X) & (iy >= 0) & (iy < Y)
        beyond = np.maximum.reduce([g.origin[0] - path[:, 0], path[:, 0] - g.max_boundary[0], g.origin[1] - path[:, 1], path[:, 1] - g.max_boundary[1]])
        assert beyond.max() < 0.4 and np.all(np.hypot(*(path[~inside, :2] - goals[b, :2]).T) < 1.5), b
        points += int(inside.sum())
        touched += int(view.occ2[ix[inside], iy[inside]].sum())
        # the optimizer's inputs of the batch form are this path's: its boundary positions
        k = packed1[b]
        assert np.array_equal(pb1.bnd[k, 0:2], path[0, :2]) and np.array_equal(pb1.bnd[k, 6:8], path[-1, :2]), b
        spans.append(np.ptp(path[:, long_axis]))
    # the collision test samples every 0.06 m over 0.05 m cells and skips an expansion's end state at half speed (as the reference's),
    # and a start is tested in its own yaw layer only, so a path can clip an occupied column: measured 2 points of about 3 000 per
    # grid, with 5 - 9 % of the columns occupied
    assert touched <= 0.005 * points, (touched, points)
    assert max(spans) > 8.0            # longer than the short side and the one-shot's reach: not a path of the transposed grid


def test_front_end_goal_inside_one_rectangle_and_outside_the_other(built):
    """a goal at x = 5.5 is inside `wide` (x to 6) and outside `tall` (x to 3); one at y = 5.5 the other way round"""
    from uneven_planner_b200 import front_end
    for name, goal, planned in (("wide", [5.5, 0.3, 0.0], True), ("tall", [5.5, 0.3, 0.0], False),
                                ("wide", [0.3, 5.5, 1.5], False), ("tall", [0.3, 5.5, 1.5], True)):
        m = grid(name)
        view = front_end.MapView(m, 0.0, 1e9)                      # nothing occupied: only the bounds decide
        assert not view.occ2.any()
        path, _ = front_end.plan(view, [0.2, 0.1, 0.5 * np.pi * (goal[1] > 1)], goal)
        assert (len(path) > 0) == planned, (name, goal, len(path))
        if planned:
            assert np.hypot(*(path[-1, :2] - goal[:2])) < 0.06 + 1e-9


# ------------------------------------------------------------------ 1f. the reference's own map query, where its build exists
@pytest.mark.parametrize("name", ["wide", "fine_yaw"])
def test_reference_map_query_matches_oracle_bitwise_on_a_rectangle(built, name):
    """UnevenMap::getAllWithGrad of the reference build against orc_map_query, as tests/test_ref_pin.py does on the 10 m square"""
    from workloads import REF
    import pyoracle as po
    if not os.path.exists(REF):
        pytest.skip("oracle/_ref/libref.so not present (built where the reference's sources exist)")
    ref = C.CDLL(REF)
    dp = C.POINTER(C.c_double)
    P = lambda a: a.ctypes.data_as(dp)
    m = grid(name)
    g = m.geom
    om = po.OracleMap(m)
    cells = np.ascontiguousarray(m.cells, dtype=np.float64)
    vn = (C.c_int * 3)(*g.voxel_num); org = (C.c_double * 3)(*g.origin); mxb = (C.c_double * 3)(*g.max_boundary)
    ref.ref_map_create.restype = C.c_void_p
    ref.ref_map_destroy.argtypes = [C.c_void_p]
    ref.ref_map_query.argtypes = [C.c_void_p, dp, dp, dp]
    h = C.c_void_p(ref.ref_map_create(P(cells), vn, org, mxb, C.c_double(g.xy_resolution), C.c_double(g.yaw_resolution), C.c_double(9.81)))
    try:
        for p in query_poses(g, n=400, seed=17):
            p = np.ascontiguousarray(p)
            vr = np.zeros(7); gr = np.zeros(21)
            ref.ref_map_query(h, P(p), P(vr), P(gr))
            vo, go = om.query(p)
            assert np.array_equal(vr, vo) and np.array_equal(gr, go.ravel()), p
    finally:
        ref.ref_map_destroy(h)
