"""Per-problem parameters without a GPU: the *_pp entry points exist and refuse a null context, ualm_problem_params_t is the first
eight members of ualm_params_t, ProblemBatch carries its rows through select and concat, and the oracle given a row equal to the
yaml values reproduces the goldens."""
import ctypes as C

import numpy as np
import pytest

EINVAL = -2
NAMES = ("ualm_upload_pp", "ualm_solve_batch_pp", "ualm_submit_batch_pp", "ualm_solve_batch_multi_pp", "ualm_check_trajectories_pp",
         "ualm_submit_replan_pp")


def test_symbols_and_null_ctx(built):
    from uneven_planner_b200 import _lib
    L = _lib.lib()
    i32, d, t = np.ones(1, np.int32), np.ones(18), C.c_int()
    ip, dp = i32.ctypes.data_as(C.POINTER(C.c_int32)), d.ctypes.data_as(C.POINTER(C.c_double))
    res = (_lib.Result * 1)()
    assert L.ualm_upload_pp(None, 1, ip, ip, dp, dp, dp, dp, None, None) == EINVAL
    assert L.ualm_solve_batch_pp(None, 1, ip, ip, dp, dp, dp, dp, None, None, res, dp, dp) == EINVAL
    assert L.ualm_submit_batch_pp(None, 1, ip, ip, dp, dp, dp, dp, None, None, 1, C.byref(t)) == EINVAL
    assert L.ualm_solve_batch_multi_pp(None, 1, 1, ip, ip, dp, dp, dp, dp, None, None, res, dp, dp) == EINVAL
    assert L.ualm_check_trajectories_pp(None, 1, ip, ip, dp, dp, dp, None, None, None, 0.01, None, dp) == EINVAL
    assert L.ualm_submit_replan_pp(None, 1, ip, ip, dp, dp, dp, dp, None, None, dp, 0.01, None, 1, C.byref(t), ip, ip, dp, dp, dp, dp) == EINVAL
    assert all(hasattr(L, n) for n in NAMES)


def test_layout_is_the_head_of_ualm_params_t(built):
    from uneven_planner_b200 import _lib
    assert C.sizeof(_lib.ProblemParams) == 64
    for name, _ in _lib.ProblemParams._fields_:
        assert getattr(_lib.ProblemParams, name).offset == getattr(_lib.Params, name).offset, name
    p = _lib.default_params()
    assert np.array_equal(_lib.problem_params(p), np.frombuffer(bytes(p)[:64], np.float64))


def test_select_and_concat_carry_rows(built, bumps_map):
    from uneven_planner_b200 import problems
    a = problems.generate(bumps_map, 5, seed=1)
    b = problems.generate(bumps_map, 3, seed=2)
    a.params = np.arange(40, dtype=np.float64).reshape(5, 8)
    b.params = -np.arange(24, dtype=np.float64).reshape(3, 8)
    cat = problems.concat([a, b], [1, 0])
    assert np.array_equal(cat.params, np.concatenate([a.params, b.params]))
    sel = cat.select([6, 0, 3])
    assert np.array_equal(sel.params, cat.params[[6, 0, 3]]) and list(sel.env) == [0, 1, 1]
    assert problems.concat([a.select([]), b.select([])], [0, 0]).params.shape == (0, 8)
    b.params = None
    with pytest.raises(ValueError):
        problems.concat([a, b], [0, 0])
    assert problems.concat([b], [0]).params is None


def test_oracle_with_the_yaml_row_reproduces_the_goldens(built, golden):
    import pyoracle as po
    from uneven_planner_b200 import _lib, configs, maps, problems
    m = maps.stand_in_terrain("hill")
    gold = golden("hill", m)
    params = configs.params_for("hill")
    pb = problems.generate(m, int(gold["B"]), seed=int(gold["seed"]), **configs.gen_kwargs("hill"))
    row = _lib.problem_params(params)
    op = po.params_from(params)
    for f, v in zip([n for n, _ in _lib.ProblemParams._fields_], row):
        setattr(op, f, float(v))
    _, _, ocx, _ = pb.offsets()
    for i in range(4):
        r, cxy, _, _ = po.solve_one(op, po.OracleMap(m), pb, i)
        assert (r.ret_code, r.n_evals, r.inner_cost) == (gold["ret_code"][i], gold["n_evals"][i], gold["inner_cost"][i]), i
        assert np.array_equal(cxy, gold["c_xy"][ocx[i]:ocx[i + 1]]), i
