"""Environments (include/ualm.h, ualm_select_env: up to UALM_MAX_ENVS parameter sets + map grids per context, one per problem) on
the CPU: the new C ABI entry points, mixed batches in problems.py, and the fixture the GPU tests (tests/test_gpu_envs.py) build on --
one batch interleaving the golden problems of the four terrains, which the oracle, run per environment, solves to the goldens."""
import ctypes as C

import numpy as np
import pytest

from uneven_planner_b200 import problems

from workloads import NAMES, mixed_golden_batch


def test_env_entry_points_exported_and_reject_null_context(built):
    from uneven_planner_b200 import _lib
    L = _lib.lib()
    for name in ("ualm_select_env", "ualm_upload_env", "ualm_solve_batch_env", "ualm_submit_batch_env", "ualm_solve_batch_multi_env"):
        assert hasattr(L, name), name
    assert _lib.UALM_MAX_ENVS == 4
    t = C.c_int()
    assert L.ualm_select_env(None, 0) == _lib.UALM_EINVAL
    assert L.ualm_upload_env(None, 0, None, None, None, None, None, None, None) == _lib.UALM_EINVAL
    assert L.ualm_solve_batch_env(None, 0, None, None, None, None, None, None, None, None, None, None) == _lib.UALM_EINVAL
    assert L.ualm_submit_batch_env(None, 0, None, None, None, None, None, None, None, 1, C.byref(t)) == _lib.UALM_EINVAL
    assert L.ualm_solve_batch_multi_env(None, 1, 0, None, None, None, None, None, None, None, None, None, None) == _lib.UALM_EINVAL


def test_concat_and_select_round_trip(built, bumps_map):
    a = problems.generate(bumps_map, 5, seed=1)
    b = problems.generate(bumps_map, 3, seed=2)
    assert a.env is None
    cat = problems.concat([a, b], [2, 0])
    assert cat.B == 8 and cat.env.dtype == np.int32 and list(cat.env) == [2] * 5 + [0] * 3
    oxy, oyaw, ocx, ocy = cat.offsets()
    for part, lo in ((a, 0), (b, 5)):
        px, py, pcx, pcy = part.offsets()
        assert np.array_equal(cat.N[lo:lo + part.B], part.N) and np.array_equal(cat.M[lo:lo + part.B], part.M)
        assert np.array_equal(cat.bnd[lo:lo + part.B], part.bnd) and np.array_equal(cat.total_time[lo:lo + part.B], part.total_time)
        assert np.array_equal(cat.inner_xy[oxy[lo]:oxy[lo + part.B]], part.inner_xy)
        assert np.array_equal(cat.inner_yaw[oyaw[lo]:oyaw[lo + part.B]], part.inner_yaw)
        assert np.array_equal(ocx[lo:lo + part.B + 1] - ocx[lo], pcx) and np.array_equal(ocy[lo:lo + part.B + 1] - ocy[lo], pcy)
    perm = np.array([5, 0, 6, 1, 7, 2, 3, 4])
    mixed = cat.select(perm)
    assert list(mixed.env) == [0, 2, 0, 2, 0, 2, 2, 2]
    back = mixed.select(np.argsort(perm))
    for f in ("N", "M", "bnd", "total_time", "inner_xy", "inner_yaw", "env", "starts", "goals"):
        assert np.array_equal(getattr(back, f), getattr(cat, f)), f
    assert np.array_equal(mixed.select(np.nonzero(mixed.env == 0)[0]).inner_xy, b.inner_xy)
    assert problems.concat([], []).B == 0
    with pytest.raises(ValueError):
        problems.concat([a, b], [0])


def test_oracle_per_environment_on_mixed_golden_batch(built, terrain, golden):
    import pyoracle as po
    maps, params, golds, _, mixed, _ = mixed_golden_batch(terrain, golden)
    assert mixed.B == sum(int(g["B"]) for g in golds) and len(set(mixed.env[:4])) == 4
    for e, name in enumerate(NAMES):
        sub = mixed.select(np.nonzero(mixed.env == e)[0])
        out = po.solve_batch(po.params_from(params[e]), po.OracleMap(maps[e]), sub, threads=4)
        g = golds[e]
        assert np.array_equal(np.array([r[0].ret_code for r in out]), g["ret_code"]), name
        assert np.array_equal(np.array([r[0].n_evals for r in out]), g["n_evals"]), name
        assert np.array_equal(np.array([r[0].outer_iters for r in out]), g["outer_iters"]), name
        assert np.array_equal(np.array([r[0].inner_cost for r in out]), g["inner_cost"]), name
        assert np.array_equal(np.concatenate([r[1] for r in out]), g["c_xy"]), name
        assert np.array_equal(np.concatenate([r[2] for r in out]), g["c_yaw"]), name
