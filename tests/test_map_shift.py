"""Grids at any origin and the host side of ualm_shift_map (no GPU): maps.shift_boxes / maps.shift_geometry, ualm_map_geometry_at,
the .umap file of a grid that is not centred at the world origin, the host builder's crop box moved with the grid, and the oracle's
map query on off-centre grids against the float64 numpy restatement of tests/test_map_geometry.py (1e-12 relative, in / out exact)."""
import struct

import numpy as np
import pytest

from workloads import OUTSIDE, _cloud_at, grid, in_map, query_poses, ref_query


CENTRES = [(31.4, -17.25), (-100.0, 250.0), (300.0, 300.0)]


def _geoms():
    from uneven_planner_b200 import _lib
    return {"square": _lib.map_geometry(), "wide": _lib.map_geometry(12.0, 6.0, 0.05, 0.1), "odd": _lib.map_geometry(7.3, 5.0, 0.04, 0.05)}


def _shifts(X, Y):
    """+-1, one axis only, both signs, |d| = X - 1 / Y - 1, |d| >= X / Y, and mixed"""
    out = []
    for d in (1, -1, 3, -7, X - 1, -(X - 1), X, -X - 5):
        out += [(d, 0), (0, d if abs(d) < X else (Y if d > 0 else -Y - 5))]
    out += [(0, Y - 1), (0, -(Y - 1)), (1, 1), (-1, -1), (2, -3), (-5, 4), (X - 1, Y - 1), (-(X - 1), 1), (X + 2, 3), (4, -Y), (X, Y)]
    return out


def _covered(boxes, X, Y):
    hit = np.zeros((X, Y), np.int32)
    for ix0, iy0, nx, ny in boxes:
        assert nx > 0 and ny > 0 and 0 <= ix0 and ix0 + nx <= X and 0 <= iy0 and iy0 + ny <= Y, (ix0, iy0, nx, ny)
        hit[ix0:ix0 + nx, iy0:iy0 + ny] += 1
    return hit


@pytest.mark.parametrize("name", ["square", "wide", "odd"])
def test_shift_boxes_are_exactly_the_cells_without_a_source(built, name):
    from uneven_planner_b200 import maps
    g = _geoms()[name]
    X, Y, _ = g.voxel_num
    xs, ys = np.meshgrid(np.arange(X), np.arange(Y), indexing="ij")
    for dx, dy in _shifts(X, Y):
        boxes = maps.shift_boxes(g, dx, dy)
        hit = _covered(boxes, X, Y)
        assert hit.max() <= 1, (dx, dy)                                          # disjoint
        nosrc = ~((xs + dx >= 0) & (xs + dx < X) & (ys + dy >= 0) & (ys + dy < Y))
        assert np.array_equal(hit.astype(bool), nosrc), (dx, dy)
        assert len(boxes) <= 2
        if dx:                                                                   # A first, and A is the x strip over all of Y
            assert boxes[0][1] == 0 and boxes[0][3] == Y and boxes[0][2] == min(abs(dx), X), (dx, dy, boxes)
        if dx == 0 and dy:
            assert boxes == [(0, Y - min(dy, Y) if dy > 0 else 0, X, min(abs(dy), Y))]
    assert maps.shift_boxes(g, 0, 0) == []


def test_shift_geometry_is_the_stated_expression(built):
    from uneven_planner_b200 import _lib, maps
    for g in list(_geoms().values()) + [_lib.map_geometry_at(10.0, 10.0, 0.05, 0.1, *c) for c in CENTRES]:
        for dx, dy in [(1, 0), (0, -1), (37, -5), (-400, 1000), (3, 3)]:
            s = maps.shift_geometry(g, dx, dy)
            r = g.xy_resolution
            assert (s.origin[0], s.max_boundary[0]) == (g.origin[0] + dx * r, g.max_boundary[0] + dx * r)
            assert (s.origin[1], s.max_boundary[1]) == (g.origin[1] + dy * r, g.max_boundary[1] + dy * r)
            assert tuple(s.voxel_num) == tuple(g.voxel_num) and (s.origin[2], s.max_boundary[2]) == (g.origin[2], g.max_boundary[2])
            assert (s.xy_resolution, s.yaw_resolution) == (g.xy_resolution, g.yaw_resolution)
        assert bytes(maps.shift_geometry(g, 0, 0)) == bytes(g)


def test_geometry_at_the_world_origin_is_map_geometry(built):
    from uneven_planner_b200 import _lib
    for args in [(10.0, 10.0, 0.05, 0.1), (12.0, 6.0, 0.05, 0.1), (7.3, 5.0, 0.04, 0.05), (20.0, 10.0, 0.05, 0.1), (9.0, 7.0, 0.1, 0.2)]:
        assert bytes(_lib.map_geometry_at(*args, 0.0, 0.0)) == bytes(_lib.map_geometry(*args))
        g, a = _lib.map_geometry(*args), _lib.map_geometry_at(*args, 31.4, -17.25)
        assert tuple(a.voxel_num) == tuple(g.voxel_num) and (a.origin[2], a.max_boundary[2]) == (g.origin[2], g.max_boundary[2])
        assert (a.origin[0], a.max_boundary[0]) == (31.4 - args[0] / 2, 31.4 + args[0] / 2)
        assert (a.origin[1], a.max_boundary[1]) == (-17.25 - args[1] / 2, -17.25 + args[1] / 2)


def _parent_umap_bytes(m):
    """the .umap file as the format's first version writes it: 64-byte header {magic, voxel_num, 2|origin|, resolutions}, then cells"""
    g = m.geom
    hdr = b"UMAP0001" + struct.pack("<3i", *g.voxel_num) + struct.pack("<4d", abs(g.origin[0]) * 2, abs(g.origin[1]) * 2, g.xy_resolution,
                                                                      g.yaw_resolution)
    return hdr.ljust(64, b"\0") + m.cells.tobytes()


def test_umap_centred_stays_v1_and_off_centre_is_v2(built, tmp_path):
    from uneven_planner_b200 import _lib, maps
    m = grid("fine_yaw")
    p = str(tmp_path / "c.umap")
    m.save(p)
    assert open(p, "rb").read() == _parent_umap_bytes(m)
    for c in CENTRES:
        for moved in (_lib.map_geometry_at(7.3, 5.0, 0.04, 0.05, *c), maps.shift_geometry(m.geom, 17, -3)):
            off = maps.UnevenMapData(moved, m.cells, "off")
            q = str(tmp_path / "off.umap")
            off.save(q)
            raw = open(q, "rb").read()
            assert raw[:8] == b"UMAP0002" and len(raw) == 128 + m.cells.nbytes
            back = maps.UnevenMapData.load(q)
            assert bytes(back.geom) == bytes(moved)
            assert np.array_equal(back.cells.view(np.uint32), m.cells.view(np.uint32))


def test_umap_symmetric_grid_that_map_geometry_does_not_give_is_v2(built, tmp_path):
    """a grid symmetric about the world origin whose bounds map_geometry does not reproduce (shifted away and back, 1 ulp wider on
    both sides; or 2 |origin| whose cell count rounds up) round-trips exactly, as UMAP0002"""
    from uneven_planner_b200 import _lib, maps
    m = grid("fine_yaw")
    wider = _lib.MapGeom.from_buffer_copy(m.geom)
    for k in (0, 1):
        wider.origin[k] = np.nextafter(m.geom.origin[k], -np.inf)
        wider.max_boundary[k] = -wider.origin[k]
    g10 = _lib.map_geometry()
    odd = _lib.MapGeom.from_buffer_copy(g10)
    odd.origin[0], odd.max_boundary[0] = -5.000000000000001, 5.000000000000001      # ceil(10.000000000000002 / 0.05) = 201 != 200
    for g, cells in ((wider, m.cells), (odd, _zero_cells(g10))):
        assert all(g.origin[k] == -g.max_boundary[k] for k in (0, 1))
        q = str(tmp_path / "sym.umap")
        maps.UnevenMapData(g, cells, "sym").save(q)
        assert open(q, "rb").read(8) == b"UMAP0002"
        back = maps.UnevenMapData.load(q)
        assert bytes(back.geom) == bytes(g) and np.array_equal(back.cells.view(np.uint32), cells.view(np.uint32))


def _zero_cells(g):
    return np.zeros(tuple(g.voxel_num) + (4,), np.float32)


def test_host_builder_crops_about_the_grid_centre(built):
    """a cloud around (31.4, -17.25) on the 4 m grid centred there: non-empty cells (the crop box about the world origin dropped it
    all), equal within float rounding to the same cloud built about the world origin; a cloud about the world origin keeps its cells"""
    from uneven_planner_b200 import _lib, maps
    cx, cy = 31.4, -17.25
    g = _lib.map_geometry_at(4.0, 4.0, 0.05, 0.1, cx, cy)
    off = maps.build_from_cloud(_cloud_at(cx, cy), g)
    assert np.count_nonzero(off.cells[..., 1]) > 0.9 * off.cells[..., 1].size
    at0 = maps.build_from_cloud(_cloud_at(0.0, 0.0), _lib.map_geometry(4.0, 4.0, 0.05, 0.1))
    assert np.abs(off.cells[..., 0] - at0.cells[..., 0]).max() < 1e-3          # the same surface, its points rounded at another place
    # points outside [c - 10, c + 10]^2 are dropped: adding far points changes nothing
    far = np.array([[cx + 10.5, cy, 0.3], [cx, cy - 10.5, 0.3], [0.0, 0.0, 0.3]], np.float32)
    again = maps.build_from_cloud(np.vstack([_cloud_at(cx, cy), far]), g)
    assert np.array_equal(again.cells.view(np.uint32), off.cells.view(np.uint32))


@pytest.mark.parametrize("centre", CENTRES + [(0.0, 0.0)])
@pytest.mark.parametrize("name", ["wide", "fine_yaw"])
def test_oracle_map_query_off_centre(built, name, centre):
    """the grid `name`'s cells on the same extent centred at `centre`: the oracle's query against ref_query, as at the world origin"""
    import pyoracle as po
    from uneven_planner_b200 import _lib, maps
    base = grid(name)
    g0 = base.geom
    geom = _lib.map_geometry_at(g0.max_boundary[0] * 2, g0.max_boundary[1] * 2, g0.xy_resolution, g0.yaw_resolution, *centre)
    m = maps.UnevenMapData(geom, base.cells, name + "-off")
    om = po.OracleMap(m)
    inside = 0
    for p in query_poses(geom, n=800, seed=5):
        v, gr = om.query(p)
        rv, rgr = ref_query(m.cells, geom, p)
        if not in_map(geom, p):
            assert np.array_equal(v, OUTSIDE) and not gr.any(), p
            continue
        inside += 1
        assert np.abs(v - rv).max() <= 1e-12 * np.linalg.norm(rv), (p, v, rv)
        for r in range(7):
            assert np.abs(gr[r] - rgr[r]).max() <= 1e-12 * max(np.linalg.norm(rgr[r]), 1e-3 * np.linalg.norm(rgr)), (p, r)
    assert inside > 500
