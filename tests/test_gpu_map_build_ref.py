"""The device map builders against the host builder and the float64 restatement of tests/map_build_ref.py, on the scenario table of
tests/test_map_build_ref.py (walls, steps, a 68 degree slope, sparse and partial clouds, an exact plane, a hole, iter_num 1 to 3,
three ellipsoids, grids off the world origin).

* ualm_map_build_device (opt.build_map): bit for bit the host builder on every scenario, and the reference's cells through the same
  assertion the host builder is held to;
* the cloud forms on the wall scenario off the world origin: ualm_update_map_from_cloud (with its cells), the window cloud form on a box
  at the cloud's edge and the shift cloud form give the reference's cells in the boxes they build."""
import numpy as np
import pytest

import map_build_ref as mref
from harness import bits
from workloads import SCENARIOS, _host, assert_matches_reference, reference, terrain

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def opt(built):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from uneven_planner_b200 import api
    o = api.BatchALMTrajOpt()
    yield o
    o.close()


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_device_builder_matches_host_and_reference(opt, name):
    s, rows = reference(name)
    dev, _ = opt.build_map(s["pts"], s["geom"], ellipsoid=s["ellipsoid"], iter_num=s["iter_num"])
    assert np.array_equal(bits(dev.cells, np.float32), bits(_host(s), np.float32))
    assert_matches_reference(dev.cells, s, rows, name)


def _box_rows(rows, geom, ix0, iy0, nx, ny):
    """the reference's rows of the cells of a box, renumbered as cells of the box's own (nx, ny, W) grid"""
    X, Y, W = geom.voxel_num
    c = rows["cell"]
    x, y, w = c // (Y * W), (c // W) % Y, c % W
    sel = (x >= ix0) & (x < ix0 + nx) & (y >= iy0) & (y < iy0 + ny)
    out = {k: rows[k][sel] for k in ("z", "sigma", "zbx", "zby", "c", "kind", "nanc", "cov", "w")}
    out["cell"] = ((x[sel] - ix0) * ny + (y[sel] - iy0)) * W + w[sel]
    bx, by, bw = np.meshgrid(np.arange(nx) + ix0, np.arange(ny) + iy0, np.arange(W), indexing="ij")
    out["ambiguous"] = rows["ambiguous"][((bx * Y + by) * W + bw).ravel()]          # per cell of the box, in the box's numbering
    out["zrange"], out["features"] = rows["zrange"], rows["features"]
    return out


def _assert_box(cells, rows, geom, box, label):
    ix0, iy0, nx, ny = box
    br = _box_rows(rows, geom, ix0, iy0, nx, ny)
    bad, _, _ = mref.compare(br, cells)
    assert cells.shape[:2] == (nx, ny) and bad.size == 0, (label, box, bad[:5])


def test_cloud_forms_match_the_reference_on_the_wall_off_centre(opt):
    from uneven_planner_b200 import _lib, maps
    cx, cy = 31.4, -17.25
    pts = terrain("wall", cx, cy)
    geom = _lib.map_geometry_at(1.0, 1.0, 0.05, 0.1, cx, cy)
    rows = mref.Reference(pts, (0.2, 0.1, 0.1), 2).build(geom)
    assert rows["features"]["nanc_it0"] > 0
    X, Y, W = geom.voxel_num
    # the whole grid, with the cells handed back
    m, _ = opt.update_environment_from_cloud(pts, geom)
    _assert_box(m.cells, rows, geom, (0, 0, X, Y), "update")
    assert np.array_equal(bits(m.cells, np.float32), bits(maps.build_from_cloud(pts, geom).cells, np.float32))
    # a window at the cloud's edge (the last columns of the grid, the cloud ending 0.25 m past them)
    box = (X - 6, 3, 6, 9)
    win, _ = opt.update_environment_window_from_cloud(pts, *box)
    _assert_box(win, rows, geom, box, "window")
    # a shift: the uncovered strips are the reference's cells of the moved grid
    dx, dy = 3, -2
    g2, strips, _ = opt.shift_environment_from_cloud(pts, dx, dy)
    rows2 = mref.Reference(pts, (0.2, 0.1, 0.1), 2).build(g2)
    for b, cells in zip(maps.shift_boxes(geom, dx, dy), strips):
        _assert_box(cells, rows2, g2, tuple(b), "shift")
