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
import os
import re
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_minco_fused import _arc_problem  # noqa: E402
from test_gpu_tp import TOL  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "uneven_planner_b200", "csrc")
INT_K = [1, 16, 18, 31, 42, 64, 127]
PRECISIONS = [65, 32]
RHO = 8.0
# which tolerance of TOL applies to which block
KIND = dict(f="f", grad_tau="grad", grad_xy="grad", grad_yaw="grad", hx="con", hx_cancel="hx_cancel", c_xy="coef", c_yaw="coef",
            scale_fx="sfx",
            **{"gx%d" % t: "con" for t in range(6)}, **{"scale_cx%d" % t: "scx" for t in range(7)})
# hx where it is a cancellation: at an initial guess (the even problems of every batch here) the yaw waypoints follow the path
# tangent, and at int_K = 1 every sample is a waypoint, where the 1e-3 perturbation leaves the yaw within a few mrad of the tangent.
# There hx = (vx sin(yaw) - vy cos(yaw)) scale has a norm of ~1e-3 of |v| scale (N64_M128 and border_cells at their guesses,
# N2_M100 perturbed at int_K = 1), and the float kinematics carry ~1e-7 of |v| scale into it.  Worst measured at precision 32 on an
# H100: 1.4e-4 at the guesses (N64_M128, int_K 31 .. 127), 1.7e-4 perturbed at int_K = 1 (N2_M100); the perturbed points at
# int_K >= 16 measure <= 2.0e-5 and keep TOL[32], as does every other block.
TOLS = {65: dict(TOL[65], hx_cancel=TOL[65]["con"]), 32: dict(TOL[32], hx_cancel=1e-3)}
THREADS = min(32, os.cpu_count() or 1)


# ------------------------------------------------------------------ the cases
def _short_path():
    """a resampled path shorter than one piece: N = 1, M = 1, T = 0.24 s"""
    from uneven_planner_b200 import problems
    return problems.from_paths([problems.dubins([0.0, 0.0, 0.0], [0.1, 0.0, 0.0])])


def _off_map():
    """leaves the +x edge of the +-5 m maps (the parity path's edge case)"""
    from uneven_planner_b200 import problems
    return problems.from_paths([problems.dubins([4.2, 0.0, 0.0], [5.6, 0.3, 0.2])])


CASES = {
    "N1_M1": lambda: _arc_problem(1, 1, arc=0.5 * np.pi),
    "N1_M128": lambda: _arc_problem(1, 128, arc=0.5 * np.pi),
    "N2_M1": lambda: _arc_problem(2, 1),
    "N2_M100": lambda: _arc_problem(2, 100),
    "N3_M40": lambda: _arc_problem(3, 40),
    "N5_M128": lambda: _arc_problem(5, 128),
    "N40_M3": lambda: _arc_problem(40, 3),
    "N13_M26": lambda: _arc_problem(13, 26),
    "N64_M128": lambda: _arc_problem(64, 128),
    "zero_boundary_rows": lambda: _arc_problem(12, 20, zero_ends=True),
    "border_cells": lambda: _arc_problem(12, 20, radius=4.99, arc=0.3, start=-0.15),      # x in [4.975, 5): the clamped last cell
    "off_map": _off_map,
    "yaw_seam": lambda: _arc_problem(10, 24, radius=2.0, arc=0.4 * np.pi, start=0.3 * np.pi),  # yaw 0.8 pi .. 1.2 pi
    "short_path": _short_path,
}


def _cat(pbs):
    from uneven_planner_b200 import problems
    out = problems.concat(pbs, [0] * len(pbs))
    out.env = None
    return out


def case_batch():
    """every case twice: at its initial guess (even index) and at a perturbed point (odd index)"""
    one = _cat([CASES[k]() for k in CASES])
    return one.select(np.repeat(np.arange(one.B), 2))


def _inputs(pb, Ks, seed=0):
    """decision vectors (odd problems perturbed), random duals (both branches of every inequality), scales, scale_fx"""
    rng = np.random.default_rng(seed)
    S = int((pb.N.astype(np.int64) * (np.asarray(Ks, np.int64) + 1)).sum())
    lam = rng.standard_normal(S) * 0.1
    mu = np.abs(rng.standard_normal(6 * S)) * 0.1 * (rng.random(6 * S) < 0.5)
    scx = rng.uniform(0.01, 1.0, 7 * S)
    sfx = rng.uniform(1e-6, 1e-3, pb.B)
    xs = np.concatenate([pb.x0(i) * (1 + (i % 2) * 1e-3 * rng.standard_normal(pb.nvar()[i])) for i in range(pb.B)])
    return xs, lam, mu, scx, sfx


def _offsets(pb, Ks):
    offx = np.concatenate([[0], np.cumsum(pb.nvar())])
    offs = np.concatenate([[0], np.cumsum(pb.N.astype(np.int64) * (np.asarray(Ks, np.int64) + 1))])
    _, _, ocx, ocy = pb.offsets()
    return offx, offs, ocx, ocy


def _per_problem(pb, Ks, ev, sfx, scx):
    """the packed outputs of a batch, split per problem"""
    offx, offs, ocx, ocy = _offsets(pb, Ks)
    return [dict(f=ev["f"][i], grad=ev["grad"][offx[i]:offx[i + 1]], hx=ev["hx"][offs[i]:offs[i + 1]], gx=ev["gx"][6 * offs[i]:6 * offs[i + 1]],
                 c_xy=ev["c_xy"][ocx[i]:ocx[i + 1]], c_yaw=ev["c_yaw"][ocy[i]:ocy[i + 1]], sfx=sfx[i], scx=scx[7 * offs[i]:7 * offs[i + 1]])
            for i in range(pb.B)]


def _oracle(pb, params, maps, Ks, inputs):
    """pyoracle eval_one and init_scaling of every problem, with problem i's parameters params[i] on maps[i]"""
    import pyoracle as po
    xs, lam, mu, scx, sfx = inputs
    offx, offs, _, _ = _offsets(pb, Ks)
    ops = {id(p): po.params_from(p) for p in params}
    oms = {id(m): po.OracleMap(m) for m in maps}

    def one(i):
        op, om = ops[id(params[i])], oms[id(maps[i])]
        o = po.eval_one(op, om, pb, i, xs[offx[i]:offx[i + 1]], lam[offs[i]:offs[i + 1]], mu[6 * offs[i]:6 * offs[i + 1]],
                        scx[7 * offs[i]:7 * offs[i + 1]], sfx[i], RHO)
        o["sfx"], o["scx"] = po.init_scaling(op, om, pb, i)
        return o
    with ThreadPoolExecutor(THREADS) as ex:
        return list(ex.map(one, range(pb.B)))


def _blocks(N, M, g, o, cancel):
    """(name, got, want, whole vector of want) for every block of one problem's outputs; cancel: hx is a cancellation (see TOLS)"""
    nxy = 2 * (N - 1)
    out = [("f", [g["f"]], [o["f"]], [o["f"]]),
           ("grad_tau", g["grad"][:1], o["grad"][:1], o["grad"]),
           ("grad_xy", g["grad"][1:1 + nxy], o["grad"][1:1 + nxy], o["grad"]),
           ("grad_yaw", g["grad"][1 + nxy:], o["grad"][1 + nxy:], o["grad"]),
           ("hx_cancel" if cancel else "hx", g["hx"], o["hx"], np.concatenate([o["hx"], o["gx"]])),
           ("c_xy", g["c_xy"], o["c_xy"], o["c_xy"]),
           ("c_yaw", g["c_yaw"], o["c_yaw"], o["c_yaw"]),
           ("scale_fx", [g["sfx"]], [o["sfx"]], [o["sfx"]])]
    out += [("gx%d" % t, g["gx"][t::6], o["gx"][t::6], np.concatenate([o["hx"], o["gx"]])) for t in range(6)]
    out += [("scale_cx%d" % t, g["scx"][t::7], o["scx"][t::7], o["scx"]) for t in range(7)]
    return out


def block_errors(pb, got, want, Ks):
    """{block: (worst relative error over the batch, problem)}; an empty block is skipped, a block that is zero up to fp64 rounding
    is measured against its whole vector"""
    worst = {}
    for i in range(pb.B):
        for name, a, b, whole in _blocks(int(pb.N[i]), int(pb.M[i]), got[i], want[i], i % 2 == 0 or Ks[i] == 1):
            a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
            if b.size == 0:
                continue
            d = float(np.linalg.norm(a - b))
            nb, nw = float(np.linalg.norm(b)), float(np.linalg.norm(np.asarray(whole, np.float64)))
            if nb <= 1e-9 * nw:
                nb = nw
            err = d / nb if nb > 0 else (0.0 if d == 0 else np.inf)
            if not np.isfinite(a).all():
                err = np.inf
            if err > worst.get(name, (-1.0, None))[0]:
                worst[name] = (err, i)
    return worst


def _check(worst, prec, what):
    tol = TOLS[prec]
    bad = {k: v for k, v in worst.items() if not v[0] <= tol[KIND[k]]}
    assert not bad, (what, bad)


# ------------------------------------------------------------------ fixtures
@pytest.fixture(scope="module")
def gpu(built):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from uneven_planner_b200 import api
    return api


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


def run_tp(gpu, pb, params, mapdata, precision, inputs, env=None):
    """one evaluation and initScaling of `pb` on a fresh throughput-path context, split per problem"""
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        opt = gpu.BatchALMTrajOpt(precision=precision).init(params).set_environment(mapdata)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k)
            else:
                os.environ[k] = v
    opt.upload(pb)
    xs, lam, mu, scx, sfx = inputs
    ev = opt.eval_batch(xs, lam, mu, scx, sfx, rho=RHO)
    ev2 = opt.eval_batch(xs, lam, mu, scx, sfx, rho=RHO)
    s_fx, s_cx = opt.init_scaling_batch()
    opt.close()
    Ks = [params.int_K] * pb.B
    return _per_problem(pb, Ks, ev, s_fx, s_cx), _per_problem(pb, Ks, ev2, s_fx, s_cx)


def _same(a, b):
    return all(np.array_equal(np.asarray(a[k]), np.asarray(b[k])) for k in a)


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
    from test_envs import NAMES, mixed_golden_batch
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
    big = _cat([gen.select(range(0, 5)), cases.select(range(0, 9)), gen.select(range(5, 12)), cases.select(range(9, cases.B))])
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
    """complete records, finite coefficients, total_T = N piece_T_xy summed, and the post-solve scan (feasibility_kernel) equal to
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


# ------------------------------------------------------------------ coverage guard (no GPU)
def _define(name):
    for f in ("ualm_tp_kernels.cuh", "ualm_tp_samples.cuh"):
        with open(os.path.join(CSRC, f)) as fh:
            mt = re.search(r"^#define\s+%s\s+(\d+)" % name, fh.read(), re.M)
        if mt:
            return int(mt.group(1))
    raise AssertionError("no #define %s" % name)


def reach(pb, cxy, cyaw, geom, K):
    """what the kernels' chunk loop (kb_kernel / ks_kernel) and map lookups see for one problem at the decision vector whose
    MINCO coefficients are cxy / cyaw, with the kernels' own formulas in float64"""
    MAXPPC, YCAP, THREADS_KB = _define("TP_MAXPPC"), _define("TP_YCAP"), _define("TP_KB_THREADS")
    N, M, T = int(pb.N[0]), int(pb.M[0]), float(pb.total_time[0])
    Tx, Ty = T / N, T / M
    K1 = K + 1
    ppc = max(1, min(MAXPPC, THREADS_KB // K1))
    out = dict(ppc=ppc, partial=False, full=False, overflow=False, off_map=False, border=False, seam=False)
    vn, org, mx = geom.voxel_num, geom.origin, geom.max_boundary
    prev = None
    for p0 in range(0, N, ppc):
        np_ = min(ppc, N - p0)
        out["partial"] |= np_ < ppc
        out["full"] |= np_ * K1 == THREADS_KB
        ybase = max(0, min(int(p0 * Tx / Ty), M - 1) - 1)
        for pl in range(np_):
            i = p0 + pl
            for j in range(K1):
                s1 = j * (Tx / K)
                pw = s1 ** np.arange(6)
                x, y = float(cxy[6 * i:6 * i + 6] @ pw), float(cxy[6 * N + 6 * i:6 * N + 6 * i + 6] @ pw)
                yi = min(int((s1 + i * Tx) / Ty), M - 1)
                y1 = (s1 + i * Tx) - yi * Ty
                yaw = float(cyaw[6 * yi:6 * yi + 6] @ (y1 ** np.arange(6)))
                out["overflow"] |= yi - ybase >= YCAP
                yawn = yaw - 2 * np.pi * np.rint(yaw / (2 * np.pi))
                if prev is not None and abs(yawn - prev) > np.pi:
                    out["seam"] = True
                prev = yawn
                inside = not (x < org[0] + 1e-4 or y < org[1] + 1e-4 or yawn < org[2] + 1e-4 or x > mx[0] - 1e-4 or y > mx[1] - 1e-4 or
                              yawn > mx[2] - 1e-4)
                out["off_map"] |= not inside
                if inside:
                    i0 = int(np.floor((x - 0.5 * geom.xy_resolution - org[0]) / geom.xy_resolution))
                    i1 = int(np.floor((y - 0.5 * geom.xy_resolution - org[1]) / geom.xy_resolution))
                    out["border"] |= i0 < 0 or i1 < 0 or i0 + 1 > vn[0] - 1 or i1 + 1 > vn[1] - 1
    return out


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
