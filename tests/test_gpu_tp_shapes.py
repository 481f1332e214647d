"""The throughput path (precision 65 / 32: ka_kernel, kb_kernel, ks_kernel, MINCO through the per-piece-count tables) against the
CPU oracle at the shapes, sample chunkings, parameter sets and map positions the generated workload never reaches:

  * sample-chunk geometry: ppc = max(1, min(TP_MAXPPC, TP_KB_THREADS / (int_K + 1))) pieces per chunk for every int_K of INT_K
    (ppc 7, 6, 4, 2, 1), a partial last chunk, and int_K = 127 whose chunk fills all TP_KB_THREADS threads;
  * chunks that span TP_YCAP or more yaw pieces past their first one, whose yaw contributions bypass the fixed-order table
    (chunk_scatter's overflow branch), in kb_kernel and in ks_kernel;
  * the MINCO tables at their ends: one piece, and the compiled limits (64 xy pieces, 128 yaw pieces);
  * one piece with T < 1 s (a resampled 0.1 m path), the T <= 1 branch of the tau <-> T map;
  * map edges: samples in the clamped border cells, off the map, and across the yaw seam;
  * the four terrains' parameter sets (volcano: int_K = 64; forest: use_scaling = 0), alone and mixed in one context.

Every block of every output is compared against its own norm, so an error in one block is not diluted by the others:
f; the gradient's tau, xy-waypoint and yaw-waypoint parts; hx; each of the six gx fields; c_xy; c_yaw; scale_fx; and scale_cx
per constraint type.  A block whose oracle value is exactly zero must come back within the tolerance times the norm of its whole
vector (the constraint vector [hx, gx] for hx and the gx fields).  So must a block whose oracle norm is zero up to fp64 rounding,
below 1e-9 of its whole vector: hx at an initial guess with int_K = 1 is sampled only at the waypoints, where the yaw is the path
tangent, and comes out ~1e-17.  Tolerances: TOL of test_gpu_tp.py, except hx where it is a cancellation at precision 32 (TOLS).

Also bit for bit on the path itself: TMA-staged tiles against the direct gather, a repeated evaluation, and the edge cases alone
against the same cases inside a generated batch; whole solves at the edge shapes give complete, finite records whose post-solve
scan is the oracle's bit for bit.  On both paths, eval_batch at a caller's point leaves the uploaded initial guesses that
init_scaling_batch and a later solve start from.  test_case_table_reaches_the_edges (no GPU) fails if the case table stops reaching
any of it."""

import numpy as np
import pytest

from harness import cat, gpu  # noqa: F401
from workloads import RHO, _check, _define, _inputs, _offsets, _oracle, _per_problem, _same, block_errors, case_batch, reach, run_tp


INT_K = [1, 16, 18, 31, 42, 64, 127]
PRECISIONS = [65, 32]


# ------------------------------------------------------------------ fixtures
@pytest.fixture(scope="module")
def cases(built):
    return case_batch()


@pytest.fixture(scope="module")
def oracle_at(cases, bumps_map):
    """oracle outputs of the case batch at default parameters with int_K = K on the bumps map (shared by both precisions)"""
    from uneven_planner_b200 import _lib
    cache = {}

    def get(K):
        if K not in cache:
            p = _lib.default_params()
            p.int_K = K
            Ks = [K] * cases.B
            inputs = _inputs(cases, Ks)
            cache[K] = (p, inputs, _oracle(cases, [p] * cases.B, [bumps_map] * cases.B, Ks, inputs))
        return cache[K]
    return get


# ------------------------------------------------------------------ the sweeps against the oracle
@pytest.mark.gpu
@pytest.mark.parametrize("K", INT_K)
@pytest.mark.parametrize("prec", PRECISIONS)
def test_cases_against_oracle_per_block(gpu, cases, oracle_at, bumps_map, prec, K):
    """every case at int_K = K (ppc 7, 7, 6, 4, 2, 1, 1), default parameters otherwise; the evaluation repeats bit for bit"""
    params, inputs, want = oracle_at(K)
    got, again = run_tp(gpu, cases, params, bumps_map, prec, inputs)
    for i in range(cases.B):
        assert _same(got[i], again[i]), i
    _check(block_errors(cases, got, want, [K] * cases.B), prec, (prec, K))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["hill", "desert", "volcano", "forest"])
@pytest.mark.parametrize("prec", PRECISIONS)
def test_cases_against_oracle_per_terrain_parameters(gpu, cases, terrain, prec, name):
    """the cases with configs.params_for(name) (volcano int_K = 64, forest use_scaling = 0) on that terrain's grid"""
    from uneven_planner_b200 import configs
    m, params = terrain(name), configs.params_for(name)
    Ks = [params.int_K] * cases.B
    inputs = _inputs(cases, Ks, seed=1)
    want = _oracle(cases, [params] * cases.B, [m] * cases.B, Ks, inputs)
    got, _ = run_tp(gpu, cases, params, m, prec, inputs)
    _check(block_errors(cases, got, want, Ks), prec, (prec, name))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECISIONS)
def test_mixed_environments_against_oracle_per_block(gpu, terrain, golden, prec):
    """the mixed golden batch (four terrains, int_K 16 and 64, use_scaling 1 and 0) in one context: every problem against the
    oracle with its own environment's parameters and grid"""
    from workloads import NAMES, mixed_golden_batch
    maps, params, _, pbs, mixed, perm = mixed_golden_batch(terrain, golden)
    env = [int(e) for e in mixed.env]
    Ks = [params[e].int_K for e in env]
    inputs = _inputs(mixed, Ks, seed=2)
    opt = gpu.BatchALMTrajOpt(precision=prec)
    for e in range(len(NAMES)):
        opt.init(params[e], env=e).set_environment(maps[e], env=e)
    opt.upload(mixed)
    xs, lam, mu, scx, sfx = inputs
    ev = opt.eval_batch(xs, lam, mu, scx, sfx, rho=RHO)
    s_fx, s_cx = opt.init_scaling_batch()
    opt.close()
    got = _per_problem(mixed, Ks, ev, s_fx, s_cx)
    want = _oracle(mixed, [params[e] for e in env], [maps[e] for e in env], Ks, inputs)
    _check(block_errors(mixed, got, want, Ks), prec, (prec, "mixed"))


# ------------------------------------------------------------------ bitwise self-consistency at the edge cases
@pytest.mark.gpu
@pytest.mark.parametrize("K", [16, 127])
@pytest.mark.parametrize("prec", PRECISIONS)
def test_cases_tile_staging_and_batch_composition_bitwise(gpu, cases, bumps_map, prec, K):
    """TMA-staged map tiles against the direct gather, and the cases alone against the same cases inside a generated batch"""
    from uneven_planner_b200 import _lib, problems
    params = _lib.default_params()
    params.int_K = K
    inputs = _inputs(cases, [K] * cases.B)
    direct, _ = run_tp(gpu, cases, params, bumps_map, prec, inputs)
    tma, _ = run_tp(gpu, cases, params, bumps_map, prec, inputs, env={"UALM_TP_TMA": "1"})
    for i in range(cases.B):
        assert _same(direct[i], tma[i]), i
    # embedded: generated problems before, between and after the cases; the cases' inputs are the same
    gen = problems.generate(bumps_map, 12, seed=41)
    big = cat([gen.select(range(0, 5)), cases.select(range(0, 9)), gen.select(range(5, 12)), cases.select(range(9, cases.B))])
    where = list(range(5, 14)) + list(range(21, 21 + cases.B - 9))
    gin = _inputs(gen, [K] * gen.B, seed=5)
    xs, lam, mu, scx, sfx = inputs
    offx, offs, _, _ = _offsets(cases, [K] * cases.B)
    gx, gs, _, _ = _offsets(gen, [K] * gen.B)
    parts = {k: [] for k in range(5)}
    for (src, lo, hi) in (("g", 0, 5), ("c", 0, 9), ("g", 5, 12), ("c", 9, cases.B)):
        ox, os_, inp = (gx, gs, gin) if src == "g" else (offx, offs, inputs)
        parts[0].append(inp[0][ox[lo]:ox[hi]]); parts[1].append(inp[1][os_[lo]:os_[hi]]); parts[2].append(inp[2][6 * os_[lo]:6 * os_[hi]])
        parts[3].append(inp[3][7 * os_[lo]:7 * os_[hi]]); parts[4].append(inp[4][lo:hi])
    binp = tuple(np.concatenate(parts[k]) for k in range(5))
    embedded, _ = run_tp(gpu, big, params, bumps_map, prec, binp)
    for k, i in enumerate(where):
        assert _same(direct[k], embedded[i]), k


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [64, 65, 32])
def test_eval_batch_leaves_the_uploaded_initial_guesses(gpu, cases, bumps_map, prec):
    """ualm_eval_batch at a caller's x does not replace the uploaded initial guesses (include/ualm.h): initScaling afterwards, and a
    solve of the resident batch, start from the uploaded guesses exactly as without the evaluation"""
    from uneven_planner_b200 import _lib
    params = _lib.default_params()
    pb = cases.select(np.arange(1, cases.B, 2))         # the cases once each; the point evaluated is away from the guesses
    rng = np.random.default_rng(3)
    xs = np.concatenate([pb.x0(i) * (1 + 1e-3 * rng.standard_normal(pb.nvar()[i])) for i in range(pb.B)])

    def run(evaluate):
        opt = gpu.BatchALMTrajOpt(precision=prec).init(params).set_environment(bumps_map)
        opt.upload(pb)
        if evaluate:
            opt.eval_batch(xs, rho=RHO)
        s_fx, s_cx = opt.init_scaling_batch()
        if evaluate:
            opt.eval_batch(xs, rho=RHO)
        opt.solve_resident()
        opt.sync()
        res, cxy, cyaw = opt.download()
        opt.close()
        return s_fx, s_cx, [bytes(r) for r in res], cxy, cyaw
    plain, after_eval = run(False), run(True)
    for a, b in zip(plain, after_eval):
        if isinstance(a, list):
            assert a == b
        else:
            assert np.array_equal(a, b)


# ------------------------------------------------------------------ whole solves at the edge shapes
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["hill", "forest"])
@pytest.mark.parametrize("prec", PRECISIONS)
def test_solves_at_edge_shapes(gpu, cases, terrain, prec, name):
    """complete records, finite coefficients, total_T = N piece_T_xy summed, and the post-solve scan (ualm_feasibility_batch) equal to
    the oracle's bit for bit on the path's own coefficients and piece durations"""
    import pyoracle as po
    from uneven_planner_b200 import configs
    m, params = terrain(name), configs.params_for(name)
    pb = cases.select(np.arange(0, cases.B, 2))
    opt = gpu.BatchALMTrajOpt(precision=prec).init(params).set_environment(m)
    res, cxy, cyaw = opt.optimize(pb)
    feas = opt.feasibility(0.01)
    opt.close()
    _, _, ocx, ocy = pb.offsets()
    om = po.OracleMap(m)
    for i in range(pb.B):
        r, N, M = res[i], int(pb.N[i]), int(pb.M[i])
        assert r.ret_code in (0, 1, 2) and r.n_evals > 0, (i, r.ret_code, r.n_evals)
        c1, c2 = cxy[ocx[i]:ocx[i + 1]], cyaw[ocy[i]:ocy[i + 1]]
        assert np.isfinite(c1).all() and np.isfinite(c2).all() and c1.any(), i
        assert np.isfinite([r.inner_cost, r.jerk_cost, r.total_T, r.piece_T_xy, r.piece_T_yaw]).all() and r.piece_T_xy > 0, i
        tt = 0.0
        for _ in range(N):
            tt += r.piece_T_xy
        assert tt == r.total_T, i
        assert r.piece_T_xy == feas[i, 8] and r.piece_T_yaw == feas[i, 9], i
        ref = po.feasibility(om, params.gravity, N, M, c1, c2, r.piece_T_xy, r.piece_T_yaw, 0.01)
        assert np.array_equal(feas[i, :8], ref), (i, feas[i, :8], ref)


def test_case_table_reaches_the_edges(built, bumps_map):
    """the case table and INT_K reach every chunking (ppc 1, 2, 4, 6, 7), a partial last chunk, a chunk of all TP_KB_THREADS
    samples, a chunk past TP_YCAP yaw pieces, one piece and the compiled limits of both MINCO systems (xy: TP_NMAX = 64,
    yaw: TP_MMAX = 128), and a sample off the map, one in the clamped border cells and one across the yaw seam"""
    import pyoracle as po
    from uneven_planner_b200 import _lib
    pb = case_batch()
    pb = pb.select(np.arange(0, pb.B, 2))
    assert set(pb.N) >= {1, _define("TP_NMAX")} and set(pb.M) >= {1, _define("TP_MMAX")}
    assert max(pb.N) <= _define("TP_NMAX") and max(pb.M) <= _define("TP_MMAX")
    got = {k: set() for k in ("ppc", "partial", "full", "overflow", "off_map", "border", "seam")}
    short = [i for i in range(pb.B) if pb.N[i] == 1 and pb.M[i] == 1 and pb.total_time[i] < 1.0]
    assert short, "no one-piece case with T < 1 s"
    for K in INT_K:
        p = _lib.default_params()
        p.int_K = K
        op, om = po.params_from(p), po.OracleMap(bumps_map)
        for i in range(pb.B):
            one = pb.select([i])
            o = po.eval_one(op, om, one, 0, one.x0(0))
            r = reach(one, o["c_xy"], o["c_yaw"], bumps_map.geom, K)
            got["ppc"].add(r["ppc"])
            for k in got:
                if k != "ppc" and r[k]:
                    got[k].add(K)
    assert got["ppc"] >= {1, 2, 4, 6, 7}, got["ppc"]
    for k in ("partial", "full", "overflow", "off_map", "border", "seam"):
        assert got[k], k
    assert 16 in got["overflow"] and 127 in got["overflow"], got["overflow"]
