"""Both paths' eval_batch and init_scaling_batch against the float64 restatement of innerCallback and initScaling
(tests/alm_ref.py), not through the oracle: the parity path (precision 64) with the bounds of test_alm_ref.TOL, the throughput path
(precisions 65 and 32) with test_gpu_tp_shapes.TOLS.

The table is test_alm_ref's (the edge cases at int_K 1, 16, 64 and 127, the four terrains' parameter sets, generated problems on
two grids, the constant tilt), plus the shapes of test_gpu_parity_limits at int_K 128 and one batch that mixes the four
terrains' parameter sets and grids in one context.  The comparison is test_alm_ref.block_errors: every block against its own
norm, scale_cx entry by entry at precision 64, near-face samples left out of the per-sample blocks."""

import numpy as np
import pytest

import workloads
from harness import cat, gpu  # noqa: F401
from workloads import SHAPES, TOLS, _inputs, _per_problem, _shape


KEYS = workloads.KEYS + ["limits", "mixed"]
# the throughput path takes int_K up to 127, so the int_K 128 shapes run on the parity path only
RUNS = [(64, k) for k in KEYS] + [(p, k) for p in (65, 32) for k in KEYS if k != "limits"]


def _tol(prec):
    """(bounds by block kind, bound of a near-face problem's f and gradient) at a precision"""
    if prec == 64:
        return workloads.ALM_TOL, workloads.LOOSE
    t = TOLS[prec]
    return dict(t, hx=t["con"]), max(workloads.LOOSE, t["grad"])


def _entry(key, terrain, bumps_map):
    """(batch, params per problem, grid per problem) of one table entry"""
    from uneven_planner_b200 import _lib, configs
    if key == "limits":
        p = _lib.default_params()
        p.int_K = 128
        pb = workloads.alm_pairs(cat([_shape(N, M) for N, M in SHAPES.values()]))
        return pb, [p] * pb.B, [bumps_map] * pb.B
    if key == "mixed":
        one = workloads.alm_cases()
        parts, ps, ms = [], [], []
        for e, name in enumerate(workloads.TERRAINS):
            idx = [k for k in range(one.B) if (k // 2) % len(workloads.TERRAINS) == e]
            sel = one.select(idx)
            parts.append(sel)
            ps += [configs.params_for(name)] * sel.B
            ms += [terrain(name)] * sel.B
        return cat(parts), ps, ms
    pb, p, m = workloads.table_entry(key, terrain, bumps_map)
    ms = [m] * pb.B if m is not None else [bumps_map] * (pb.B // 2) + [terrain("hill")] * (pb.B - pb.B // 2)
    return pb, [p] * pb.B, ms


@pytest.fixture(scope="module")
def table(built, terrain, bumps_map):
    """table(key) -> (batch with one environment per (params, grid) pair, params, grids, int_K per problem, inputs, restatement)"""
    cache = {}

    def get(key):
        if key not in cache:
            pb, ps, ms = _entry(key, terrain, bumps_map)
            pairs = []
            for p, m in zip(ps, ms):
                if (id(p), id(m)) not in pairs:
                    pairs.append((id(p), id(m)))
            pb.env = np.array([pairs.index((id(p), id(m))) for p, m in zip(ps, ms)], np.int32)
            Ks = [p.int_K for p in ps]
            inputs = _inputs(pb, Ks, seed=KEYS.index(key))
            cache[key] = (pb, ps, ms, Ks, inputs, workloads.restated(pb, ps, ms, Ks, inputs))
        return cache[key]
    return get


def _run(gpu, pb, ps, ms, prec, inputs, Ks):
    """eval_batch at `inputs` and init_scaling_batch of pb in one context, environment e holding its problems' params and grid"""
    opt = gpu.BatchALMTrajOpt(precision=prec)
    try:
        for e in range(int(pb.env.max()) + 1):
            i = int(np.nonzero(pb.env == e)[0][0])
            opt.init(ps[i], env=e).set_environment(ms[i], env=e)
        opt.upload(pb)
        xs, lam, mu, scx, sfx = inputs
        ev = opt.eval_batch(xs, lam, mu, scx, sfx, rho=workloads.RHO)
        s_fx, s_cx = opt.init_scaling_batch()
    finally:
        opt.close()
    return _per_problem(pb, Ks, ev, s_fx, s_cx)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,key", RUNS)
def test_kernels_match_restatement_per_block(gpu, table, prec, key):
    pb, ps, ms, Ks, inputs, ref = table(key)
    got = _run(gpu, pb, ps, ms, prec, inputs, Ks)
    # hx is a cancellation at the initial guesses and at int_K = 1 (test_gpu_tp_shapes.TOLS): there it takes hx_cancel
    cancel = [i % 2 == 0 or Ks[i] == 1 for i in range(pb.B)]
    # scale_cx entry by entry on the parity path; by norm on the throughput path, as TOLS are stated (at precision 32 one scale
    # entry at int_K 127 measures 7.7e-3 on an H100, its block 3.1e-4 against the bound 2e-3)
    worst = workloads.alm_block_errors(pb, got, ref, workloads.near_face(ref), cancel if prec != 64 else None, entrywise_scales=prec == 64)
    print("precision %d, %s: worst %s" % (prec, key, {k: "%.1e" % v[0] for k, v in sorted(worst.items())}))
    tol, loose = _tol(prec)
    workloads.alm_check(worst, tol, loose, (prec, key))
