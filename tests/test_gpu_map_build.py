"""UnevenMap construction on the GPU (SURVEY 8f-1, ualm_map_build_device) against the host builder (ualm_map_build).

Both run csrc/map_cell.h (one restatement of UnevenMap::constructMap + filter, uneven_map.cpp:317-398, 5-43), compiled once for
the host and once for sm_90a with contraction off, so the grids must agree bit for bit (float32 cells compared as integers).
The reference's .pcd clouds do not travel to the GPU box; the clouds here are seeded analytic surfaces with noise and holes."""
import numpy as np
import pytest

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


def _cloud(n, half, seed, hole=True):
    rng = np.random.default_rng(seed)
    xy = rng.uniform(-half, half, (n, 2))
    z = 0.4 * np.exp(-((xy[:, 0] - 0.5) ** 2 + (xy[:, 1] + 0.3) ** 2) / 0.8) + 0.15 * np.sin(2.0 * xy[:, 0]) * np.cos(1.5 * xy[:, 1]) + 0.3
    z += rng.normal(0.0, 0.004, n)
    pts = np.column_stack([xy, z]).astype(np.float32)
    if hole:   # an empty patch: cells there take the "no points in the ellipsoid" branch (uneven_map.cpp:379-386)
        keep = ~((np.abs(pts[:, 0] + 1.0) < 0.35) & (np.abs(pts[:, 1] - 1.0) < 0.35))
        pts = pts[keep]
    return pts


@pytest.mark.parametrize("seed,n", [(0, 60000), (1, 4000)])
def test_device_map_is_bit_identical_to_host_map(opt, seed, n):
    from uneven_planner_b200 import _lib, maps
    geom = _lib.map_geometry(4.0, 4.0, 0.05, 0.1)            # 80 x 80 x 64 cells
    pts = _cloud(n, 2.3, seed)
    host = maps.build_from_cloud(pts, geom)
    dev, ms = opt.build_map(pts, geom)
    assert ms > 0.0
    assert np.array_equal(host.cells.view(np.uint32), dev.cells.view(np.uint32))
    # sanity of the content: unit normals, sigma in [0, 1], the surface height where there are points
    zb2 = dev.cells[..., 2] ** 2 + dev.cells[..., 3] ** 2
    assert np.all(zb2 <= 1.0 + 1e-6) and np.all(dev.cells[..., 1] >= -1e-6) and np.all(dev.cells[..., 1] <= 1.0 + 1e-6)   # Jacobi rounding can leave the smallest eigenvalue at -1e-20


def test_device_map_edge_cases(opt):
    from uneven_planner_b200 import _lib, maps
    geom = _lib.map_geometry(1.0, 1.0, 0.05, 0.1)
    for pts in (np.zeros((0, 3), np.float32),                                   # empty cloud: every cell keeps RXS2() defaults
                np.array([[0.1, 0.1, 0.2]], np.float32),                        # one point: covariance 0 -> sigma NaN branch (uneven_map.cpp:30-36)
                np.array([[np.nan, 0, 0], [50.0, 0, 0], [0.0, 0.0, 7.0], [0.2, -0.2, 0.1], [0.21, -0.2, 0.1]], np.float32)):   # crop box + nan
        host = maps.build_from_cloud(pts, geom)
        dev, _ = opt.build_map(pts, geom)
        assert np.array_equal(host.cells.view(np.uint32), dev.cells.view(np.uint32))


def test_device_map_matches_the_reference_build(opt):
    """ualm_map_build_device against the reference's OWN constructMap + filter (oracle/_ref/librefmap.so = uneven_map.cpp compiled
    unmodified, tests/test_ref_pin.py) on the same preprocessed cloud: float32 cells = the reference's doubles rounded, up to 2 ulps,
    except the <= 0.02 % of cells at the rim of the empty patch (degenerate footprints)."""
    from workloads import analytic_cloud, preprocessed, reference_construct_map
    pts = analytic_cloud(1.1, 100, seed=1, hole=(0.35, -0.3, 0.14))
    geom, ref = reference_construct_map(preprocessed(pts), 1.6)
    dev, _ = opt.build_map(pts, geom)
    d = np.abs(dev.cells.astype(np.float64) - ref)
    rel = (d / np.maximum(np.abs(ref), 1e-3)).max(axis=-1)
    assert (rel > 3e-7).mean() <= 2e-4
