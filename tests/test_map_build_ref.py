"""The host map builder (ualm_map_build, csrc/map_cell.h) and its preprocessing (ualm_map_preprocess_cloud) against the float64
restatement of tests/map_build_ref.py, which shares no code or algorithm with them, on terrains where such builders go wrong: walls,
steps, a 68 degree slope, sparse clouds, a cloud over one corner of the grid, an exact plane and a hole, at iter_num 1 to 3, three
ellipsoids (one whose largest semi-axis, the bin size, is z) and grids off the world origin.

What is asserted, and the bounds measured on these scenarios:
* unambiguous cells: z, zb.x and zb.y within 1 float ulp of float32(reference) (or 1e-12 where the value is 0), sigma within
  1 ulp or 1e-9 absolute;
* ambiguous cells (map_build_ref's docstring): one of the reference's variants, or the properties a degenerate footprint leaves;
* per scenario, bounds on the ambiguous share and on the share checked for plausibility only (SCENARIOS), and counts showing the
  scenario reaches the case it exists for;
* on the wall, the cells written flat because c came out NaN (DESIGN section 6): their count, and where the reference build exists,
  the same cells with the same values in it.

Every cloud here holds at most one point per 1 cm voxel and lies inside the crop box, so that the builder's VoxelGrid keeps it as it is
and both sides work on the same points; the preprocessing itself is tested on its own."""
import ctypes as C

import numpy as np
import pytest

import map_build_ref as mref

from workloads import SCENARIOS, _host, assert_matches_reference, reference, scenario, terrain


# cells of the wall scenario whose normal came out horizontal with zb.x^2 + zb.y^2 rounded above 1 after the first iteration, so
# that c is NaN: the second iteration's frame is NaN, no point passes the ellipsoid test, and the cell is written as flat ground at
# its first-iteration height (DESIGN section 6)
WALL_NAN_C_CELLS = 110


def assert_same_nan_c_cells(rows, other, cells):
    """`other` (the reference build's grid) writes the NaN-c cells `cells` (a builder's grid) writes, no more and no fewer, and the
    same values there within 2 float ulps"""
    _, mine, _ = mref.compare(rows, cells)
    _, theirs, _ = mref.compare(rows, other)
    assert np.array_equal(mine, theirs), (mine.size, theirs.size, np.setxor1d(mine, theirs)[:10])
    a = np.asarray(cells, np.float32).reshape(-1, 4)[mine].astype(np.float64)
    b = np.asarray(other, np.float64).reshape(-1, 4)[mine].astype(np.float32).astype(np.float64)
    assert np.all(np.abs(a - b) <= 2 * mref.ulp32(b) + mref.VALUE_ABS)


def _finite_c_instead(rows, cells, nanc):
    """the grid `cells` with each cell of `nanc` written as its variant with a finite c (the wall's normal) instead"""
    alt = np.array(cells, np.float32).reshape(-1, 4)
    for c in nanc:
        r = np.nonzero((rows["cell"] == c) & ~rows["nanc"] & (rows["kind"] == mref.EXACT))[0][0]
        alt[c] = rows["z"][r], rows["sigma"][r], rows["zbx"][r], rows["zby"][r]
    return alt.reshape(np.shape(cells))


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_host_builder_matches_the_float64_reference(built, name):
    s, rows = reference(name)
    cells = _host(s)
    nanc_only = assert_matches_reference(cells, s, rows, name)
    if name == "wall":
        assert nanc_only.size == WALL_NAN_C_CELLS
        b = cells.reshape(-1, 4)[nanc_only]
        assert np.all(b[:, 1:] == 0.0) and np.all(b[:, 0] > 0.1)        # flat, at a height on the wall, not the ground's 0.02 m
        # the check the reference build is held to tells a grid with the wall's normal on those cells apart
        assert_same_nan_c_cells(rows, cells, cells)
        with pytest.raises(AssertionError):
            assert_same_nan_c_cells(rows, _finite_c_instead(rows, cells, nanc_only), cells)


# ------------------------------------------------------------------------------------------------------ preprocessing
def _preprocess_host(pts):
    from uneven_planner_b200 import _lib
    fp = C.POINTER(C.c_float)
    pts = np.ascontiguousarray(pts, np.float32)
    out = np.zeros((max(pts.shape[0], 1), 3), np.float32)
    k = _lib.lib().ualm_map_preprocess_cloud(pts.ctypes.data_as(fp), pts.shape[0], 0.2, 0.1, 0.1, out.ctypes.data_as(fp), out.shape[0])
    assert k >= 0
    return out[:k]


def _assert_same_voxels(host, pts):
    cen, cnt, _ = mref.preprocess(pts)
    assert host.shape[0] == cen.shape[0]
    if cen.shape[0] == 0:
        return
    from scipy.spatial import cKDTree
    d, i = cKDTree(cen).query(host.astype(np.float64))
    assert np.unique(i).size == i.size                                  # one host point per voxel of the reference
    # a float sum of n points, then a division: n + 1 roundings of the largest coordinate
    tol = (cnt[i] + 1) * np.abs(cen[i]).max(axis=1) * 2.0 ** -24
    assert np.all(d <= tol * np.sqrt(3.0)), float((d / tol).max())


def test_preprocess_matches_the_numpy_crop_and_voxel_grid(built):
    rng = np.random.default_rng(5)
    n = 60000
    p = np.column_stack([rng.uniform(-10.5, 10.5, n), rng.uniform(-10.5, 10.5, n), rng.uniform(-0.3, 5.3, n)])
    dense = rng.uniform(-0.02, 0.02, (20000, 3)) + [1.234, -2.5, 0.7]     # many points per voxel
    pts = np.concatenate([p, dense]).astype(np.float32)
    host = _preprocess_host(pts)
    _assert_same_voxels(host, pts)
    assert host.shape[0] < pts.shape[0] - 10000
    # preprocessing a preprocessed cloud keeps it: same voxels, each centroid its own voxel's only point
    again = _preprocess_host(host)
    assert again.shape == host.shape
    key = lambda a: a[np.lexsort(a.T[::-1])]
    assert np.array_equal(key(again), key(host))


def test_preprocess_bounds_and_non_finite_points(built):
    f = np.float32
    on = [(-10.0, 0.5, 1.0), (10.0, 0.5, 1.0), (0.5, -10.0, 1.0), (0.5, 10.0, 1.0), (0.3, 0.3, f(-0.01)), (0.6, 0.6, f(5.0))]
    off = [(np.nextafter(f(10.0), f(11.0)), 0.7, 1.0), (np.nextafter(f(-10.0), f(-11.0)), 0.7, 1.0), (0.8, 0.8, np.nextafter(f(-0.01), f(-1.0))),
           (0.9, 0.9, np.nextafter(f(5.0), f(6.0))), (np.nan, 0, 0), (0, np.inf, 0), (0, 0, -np.inf), (np.inf, np.nan, 1.0)]
    pts = np.array(on + off, np.float32)
    host = _preprocess_host(pts)
    _assert_same_voxels(host, pts)
    key = lambda a: a[np.lexsort(a.T[::-1])]
    assert np.array_equal(key(host), key(np.array(on, np.float32)))        # each bound itself is inside, the next float outside
    assert _preprocess_host(np.array(off, np.float32)).shape[0] == 0


# ------------------------------------------------------------------------------------------------------ the reference itself
class _Geom:
    def __init__(self, nx, ny, nw, res=0.05, yaw_res=0.1, origin=(-0.1, -0.1, -3.2)):
        self.voxel_num, self.xy_resolution, self.yaw_resolution, self.origin = (nx, ny, nw), res, yaw_res, origin


def _brute_force(P, geom, ell, iter_num):
    """constructMap as a plain loop over cells with brute-force neighbour searches"""
    X, Y, W = geom.voxel_num
    out = np.zeros((X, Y, W, 4))
    e = np.asarray(ell)
    for x in range(X):
        for y in range(Y):
            for w in range(W):
                px, py = (x + 0.5) * geom.xy_resolution + geom.origin[0], (y + 0.5) * geom.xy_resolution + geom.origin[1]
                yaw = (w + 0.5) * geom.yaw_resolution + geom.origin[2]
                z, sg, zb = 0.0, 0.0, np.array([0.0, 0.0, 1.0])
                for it in range(iter_num):
                    yb = np.cross(zb, [np.cos(yaw), np.sin(yaw), 0.0])
                    if np.linalg.norm(yb) > 0:
                        yb = yb / np.linalg.norm(yb)
                    xb = np.cross(yb, zb)
                    wp = np.array([px + 0.12 * xb[0], py + 0.12 * xb[1], z])
                    if it == 0:
                        q = wp[:2].astype(np.float32).astype(np.float64)
                        wp[2] = P[np.argmin(((P[:, :2] - q) ** 2).sum(axis=1)), 2]
                    d = P - wp
                    r2 = ((d @ xb) / e[0]) ** 2 + ((d @ yb) / e[1]) ** 2 + ((d @ zb) / e[2]) ** 2
                    F = P[r2 < 1.0]
                    if F.shape[0] == 0:
                        z, sg, zb = wp[2], 0.0, np.array([0.0, 0.0, 1.0])
                        continue
                    m = F.mean(axis=0)
                    lam, V = np.linalg.eigh((F - m).T @ (F - m) / F.shape[0])
                    nrm = V[:, 0] / np.linalg.norm(V[:, 0])
                    nrm = -nrm if nrm[2] < 0 else nrm
                    sg = 3.0 * lam[0] / lam.sum() if lam.sum() != 0 else np.nan
                    if np.isnan(sg):
                        sg, nrm = 1.0, np.array([1.0, 0.0, 0.0])
                    z = m[2]
                    zb = np.array([nrm[0], nrm[1], np.sqrt(1.0 - nrm[0] ** 2 - nrm[1] ** 2)])
                out[x, y, w] = z, sg, zb[0], zb[1]
    return out


def test_reference_equals_a_brute_force_loop(built):
    P = terrain("smooth", half=0.4, seed=3)[::4].astype(np.float64)
    geom = _Geom(4, 5, 6)
    for ell, it in (((0.2, 0.1, 0.1), 2), ((0.1, 0.1, 0.25), 3)):
        rows = mref.Reference(P, ell, it).build(geom)
        bf = _brute_force(P, geom, ell, it).reshape(-1, 4)
        una = ~rows["ambiguous"][rows["cell"]]
        assert una.sum() == bf.shape[0]
        c = rows["cell"][una]
        got = np.stack([rows[k][una] for k in ("z", "sigma", "zbx", "zby")], axis=1)
        assert np.allclose(got, bf[c], rtol=0, atol=1e-12)


def test_reference_on_an_exact_plane_and_hand_built_footprints(built):
    # an exact horizontal plane: sigma exactly 0, normal exactly (0, 0, 1)
    rows = mref.Reference(terrain("plane", half=0.3), (0.2, 0.1, 0.1), 2).build(_Geom(4, 4, 8))
    assert rows["features"]["ambiguous"] == 0
    assert np.all(rows["sigma"] == 0.0) and np.all(rows["zbx"] == 0.0) and np.all(rows["zby"] == 0.0) and np.all(rows["z"] == np.float32(0.5))
    g = _Geom(1, 1, 1, origin=(-0.025, -0.025, -0.05))            # one cell at (0, 0), yaw 0: wp = (0.12, 0, z)
    # one point: filter's NaN rule, sigma 1 and zb (1, 0)
    one = mref.Reference(np.array([[0.12, 0.0, 0.3]]), (0.2, 0.1, 0.1), 1).build(g)
    assert one["features"]["ambiguous"] == 0 and (one["z"][0], one["sigma"][0], one["zbx"][0], one["zby"][0]) == (0.3, 1.0, 1.0, 0.0)
    # two points: degenerate, z their mean, sigma 0, normal any unit vector across their line
    two = mref.Reference(np.array([[0.12, 0.0, 0.3], [0.14, 0.03, 0.31]]), (0.2, 0.1, 0.1), 1).build(g)
    assert two["kind"][0] == mref.DEGENERATE and abs(two["z"][0] - 0.305) < 1e-12 and abs(two["sigma"][0]) < 1e-12
    line = np.array([0.02, 0.03, 0.01])
    good = np.zeros((1, 1, 1, 4), np.float32)
    n = np.cross(line, [0.0, 1.0, 0.0]); n /= np.linalg.norm(n); n = n if n[2] >= 0 else -n
    good[0, 0, 0] = np.float32(0.305), 0.0, n[0], n[1]
    assert mref.row_matches(two, good).all()
    good[0, 0, 0, 2:] = 0.0                                         # (0, 0, 1) is not across the line
    assert not mref.row_matches(two, good).any()
    # a point exactly on the ellipsoid's surface (r^2 = 1 on the x axis: 0.12 + 0.2): one variant with it, one without
    P = np.array([[0.12, 0.0, 0.3], [0.12, 0.02, 0.3], [0.10, -0.02, 0.301], [0.32, 0.0, 0.3]])
    s = mref.Reference(P, (0.2, 0.1, 0.1), 1).build(g)
    assert s["ambiguous"][0] and sorted(np.round(s["z"], 12)) == sorted(np.round([P[:3, 2].mean(), P[:, 2].mean()], 12))


# ------------------------------------------------------------------------------------------------------ the reference build
@pytest.mark.parametrize("name", ["wall", "slope68", "sparse"])
def test_float64_reference_against_the_reference_build(built, name):
    """where oracle/_ref/librefmap.so exists (the reference's own constructMap + filter), its cells are one of this reference's
    variants, and it writes the NaN-c cells the host builder writes, the same cells with the same values: if it wrote the wall's
    normal there instead, map_cell.h would be wrong on them.  Elsewhere it skips like the other pins of test_ref_pin.py."""
    from workloads import reference_construct_map
    s = scenario(name)
    geom, ref64 = reference_construct_map(s["pts"], 1.0, iter_num=s["iter_num"], ellipsoid=s["ellipsoid"])
    assert bytes(geom) == bytes(s["geom"])
    _, rows = reference(name)
    bad, _, _ = mref.compare(rows, ref64.astype(np.float32))
    assert bad.size == 0, bad[:10]
    assert_same_nan_c_cells(rows, ref64, _host(s))
