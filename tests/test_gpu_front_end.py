"""SURVEY 8f-2 end to end on the GPU: (start, goal) pairs -> KinoAstar::plan + PlanManager's resampler on host threads
(ualm_front_end_batch, pinned against the reference in tests/test_ref_pin.py) -> the batched optimizer, against the oracle solving the
same resampled problems: bit-identical on the parity path."""
import numpy as np
import pytest

from harness import gpu  # noqa: F401


pytestmark = pytest.mark.gpu


def test_start_goal_batch_through_the_front_end_matches_oracle(gpu, hill_map):
    import pyoracle as po
    from uneven_planner_b200 import _lib, front_end
    params = _lib.default_params()
    view = front_end.MapView(hill_map, 0.8, 0.05)
    rng = np.random.default_rng(21)
    B = 64
    starts = np.column_stack([rng.uniform(-4.3, 4.3, B), rng.uniform(-4.3, 4.3, B), rng.uniform(-np.pi, np.pi, B)])
    goals = np.column_stack([rng.uniform(-4.3, 4.3, B), rng.uniform(-4.3, 4.3, B), rng.uniform(-np.pi, np.pi, B)])
    pb, packed, nexp = front_end.plan_batch(view, starts, goals)
    assert pb.B >= B // 4 and (packed >= 0).sum() == pb.B          # random poses: about half of the starts or goals lie in occupied cells
    opt = gpu.BatchALMTrajOpt().init(params).set_environment(hill_map)
    res, cxy, cyaw = opt.optimize(pb)
    opt.close()
    ores = po.solve_batch(po.params_from(params), po.OracleMap(hill_map), pb, threads=8)
    _, _, ocx, ocy = pb.offsets()
    for i in range(pb.B):
        o, oxy, oyaw, _ = ores[i]
        assert (res[i].ret_code, res[i].n_evals, res[i].inner_cost, res[i].total_T) == (o.ret_code, o.n_evals, o.inner_cost, o.total_T), i
        assert np.array_equal(cxy[ocx[i]:ocx[i + 1]], oxy) and np.array_equal(cyaw[ocy[i]:ocy[i + 1]], oyaw), i
    conv = np.mean([r.ret_code == 0 for r in res])
    assert conv > 0.5
