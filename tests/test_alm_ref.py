"""The CPU oracle's innerCallback and initScaling (oracle/oracle.cpp: ALM::evaluate, calConstrainCostGrad, initScaling) against
an independent float64 restatement of the same mathematics (tests/alm_ref.py: dense MINCO solve, torch autograd, Gauss-Legendre
jerk, the geometric terrain frame, a full forward-mode Jacobian for initScaling).  The parity path is held to the oracle bit for
bit and the throughput path to it within TOL, so this is what checks the mathematics all three compute.

The case table: the edge cases of test_gpu_tp_shapes (one piece and the compiled limits, N > M with the yaw index clamped at M - 1,
zero boundary rows, the clamped border cells, off the map, the yaw seam, tau < 0) at int_K 1, 16, 64 and 127 on the bumps grid;
the same cases with the four terrains' parameter sets (volcano int_K 64, forest use_scaling 0) on their grids; generated problems
on the bumps grid and the hill grid; and the cases on the constant tilt, where the gravity terms are nonzero everywhere.  Every
problem at its initial guess and at a perturbed point, with random duals and scales, so both branches of every inequality are
taken.

Every block is compared against its own norm (block_errors): f; the gradient's tau, xy-waypoint and yaw-waypoint parts; hx and
each gx field; c_xy and c_yaw; scale_fx; and scale_cx per constraint type entry by entry.  Every coordinate and every scale is
compared, nothing is sampled.  Samples the restatement flags as near a cell face (alm_ref.FACE) must be rare; they are left out
of the per-sample blocks, and a problem that holds one has its f and gradient held to LOOSE instead of TOL."""
import os
import sys

import numpy as np
import pytest


sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import alm_ref as ar  # noqa: E402
from workloads import ALM_TOL, KEYS, LOOSE, _inputs, alm_block_errors, alm_check, near_face, restated, table_entry  # noqa: E402

MAX_NEAR_FACE = 1e-3    # share of the table's samples that may be near a face


def alm_oracle(pb, params, mapdata, Ks, inputs):
    from workloads import _oracle
    return _oracle(pb, params, mapdata, Ks, inputs)


# ------------------------------------------------------------------ fixtures
@pytest.fixture(scope="module")
def table(built, terrain, bumps_map):
    """table(key) -> (batch, params per problem, grid per problem, int_K per problem, inputs, restatement, oracle), cached"""
    cache = {}

    def get(key):
        if key not in cache:
            pb, p, m = table_entry(key, terrain, bumps_map)
            if m is None:                                   # generated: the first half on the bumps grid, the second on hill's
                half = pb.B // 2
                ms = [bumps_map] * half + [terrain("hill")] * (pb.B - half)
            else:
                ms = [m] * pb.B
            ps = [p] * pb.B
            Ks = [p.int_K] * pb.B
            inputs = _inputs(pb, Ks, seed=KEYS.index(key))
            cache[key] = (pb, ps, ms, Ks, inputs, restated(pb, ps, ms, Ks, inputs), alm_oracle(pb, ps, ms, Ks, inputs))
        return cache[key]
    return get


# ------------------------------------------------------------------ the oracle against the restatement
@pytest.mark.parametrize("key", KEYS)
def test_oracle_matches_restatement_per_block(table, key):
    pb, ps, ms, Ks, inputs, ref, want = table(key)
    near = near_face(ref)
    n = sum(int(v.sum()) for v in near)
    S = sum(len(v) for v in near)
    worst = alm_block_errors(pb, want, ref, near)
    print("%s: %d of %d samples near a face; worst %s" % (key, n, S, {k: "%.1e" % v[0] for k, v in sorted(worst.items())}))
    assert n <= MAX_NEAR_FACE * S, (key, n, S)
    alm_check(worst, ALM_TOL, LOOSE, key)


# ------------------------------------------------------------------ what the table reaches (fails if it stops reaching an edge)
def test_case_table_reaches_the_edges(table):
    """each inequality both active and inactive; samples off the map, in the clamped border cells, interpolating across the yaw
    seam, and with the yaw index clamped at M - 1; N > M, tau < 0, int_K = 1, use_scaling 0 and 1"""
    got = dict(active=np.zeros(6, np.int64), inactive=np.zeros(6, np.int64), off_map=0, border=0, seam=0, yaw_clamped=0,
               n_gt_m=0, tau_neg=0, int_K_1=0, use_scaling=set())
    for key in KEYS:
        pb, ps, _, Ks, inputs, ref, _ = table(key)
        offx = np.concatenate([[0], np.cumsum(pb.nvar())])
        for i, r in enumerate(ref):
            got["active"] += r["active"].sum(0)
            got["inactive"] += (~r["active"]).sum(0)
            for k in ("off_map", "border", "seam", "yaw_clamped"):
                got[k] += int(r[k].sum())
            got["n_gt_m"] += int(pb.N[i] > pb.M[i])
            got["tau_neg"] += int(inputs[0][offx[i]] < 0)
            got["int_K_1"] += int(Ks[i] == 1)
            got["use_scaling"].add(int(ps[i].use_scaling))
    print("reach:", got)
    assert (got["active"] > 0).all() and (got["inactive"] > 0).all(), got
    for k in ("off_map", "border", "seam", "yaw_clamped", "n_gt_m", "tau_neg", "int_K_1"):
        assert got[k] > 0, k
    assert got["use_scaling"] == {0, 1}


# ------------------------------------------------------------------ the restatement on its own
def _query(m, pos):
    """the restatement's terrain frame and sigma at positions pos (n, 3), and its Jacobian in x and y"""
    import torch
    g = ar.Grid(m)
    pos = torch.tensor(np.asarray(pos, np.float64), requires_grad=True)
    mp = ar._cells(g, pos[:, :2].detach().numpy(), pos[:, 2].detach().numpy())
    sigma, zbx, zby, yn = ar.terrain(g, mp, pos[:, :2], pos[:, 2])
    v = torch.stack(list(ar.frame(zbx, zby, yn)) + [sigma], 1)
    jac = torch.stack([torch.autograd.grad(v[:, k].sum(), pos, retain_graph=True)[0] for k in range(7)], 1)
    return v.detach().numpy(), jac.numpy()


def test_restated_frame_flat_and_tilt_closed_forms(built):
    """flat: inv_cos = 1, sin = 0, cos_xi = 1, no gradient; constant tilt: the closed forms of test_map_constant_tilt_closed_form and
    no x / y dependence; off the map: the flat frame"""
    from uneven_planner_b200 import maps
    flat = maps.synthetic_terrain("flat")
    v, jac = _query(flat, [[0.33, -1.2, 0.7], [-3.0, 2.0, -2.5], [7.0, 0.0, 0.0]])
    assert np.array_equal(v, np.tile([1, 0, 1, 0, 1, 1, 0], (3, 1))) and np.all(jac == 0)
    m = maps.synthetic_terrain("tilt")
    a, b = float(m.cells[0, 0, 0, 2]), float(m.cells[0, 0, 0, 3])
    c = np.sqrt(1 - a * a - b * b)
    yaws = np.array([-2.0, 0.0, 0.9, 3.0])
    v, jac = _query(m, np.stack([np.full(4, 0.7), np.full(4, -0.4), yaws], 1))
    t = np.cos(yaws) * a + np.sin(yaws) * b
    s = np.sin(yaws) * a - np.cos(yaws) * b
    r = 1 / np.sqrt(1 - t * t)
    want = np.stack([r, -c * t * r, 1 / (r * c), s * r, np.full(4, c), np.full(4, 1 / c), np.zeros(4)], 1)
    assert np.allclose(v, want, rtol=1e-12, atol=1e-15)
    assert np.abs(jac[:, :, :2]).max() < 1e-9
    v, _ = _query(m, [[5.2, 0.0, 0.3]])
    assert np.array_equal(v[0], [1, 0, 1, 0, 1, 1, 0])


def test_restated_gradient_matches_its_own_central_differences(bumps_map):
    """the restatement's autograd gradient (without Q3) against central differences of its own f, at every coordinate of two
    problems at points whose samples stay inside their cells over the stencil"""
    from uneven_planner_b200 import _lib, problems
    p = _lib.default_params()
    grid = ar.Grid(bumps_map)
    pb = problems.generate(bumps_map, 2, seed=11)
    rng = np.random.default_rng(0)
    h = 1e-6
    for i in range(pb.B):
        prob = ar.Problem(pb, i)
        S = prob.N * (p.int_K + 1)
        lam, mu = rng.standard_normal(S) * 0.05, np.abs(rng.standard_normal(6 * S)) * 0.05
        scx = rng.uniform(0.2, 1.0, 7 * S)
        x = prob.x0 * (1 + 1e-3 * rng.standard_normal(prob.nvar))
        ev = lambda y, **kw: ar.evaluate(prob, p, grid, y, lam, mu, scx, 1e-3, 4.0, **kw)
        base = ev(x, q3=False)
        cells = ar._Setup(prob, p, grid, x).mp["corners"]
        for k in range(prob.nvar):
            xp, xm = x.copy(), x.copy()
            xp[k] += h
            xm[k] -= h
            if not (np.array_equal(ar._Setup(prob, p, grid, xp).mp["corners"], cells) and
                    np.array_equal(ar._Setup(prob, p, grid, xm).mp["corners"], cells)):
                continue
            fd = (ev(xp)["f"] - ev(xm)["f"]) / (2 * h)
            # truncation ~ h^2, cancellation ~ eps |f| / h
            assert abs(fd - base["grad"][k]) < 1e-6 * max(1.0, abs(fd)) + 100 * np.finfo(float).eps * abs(base["f"]) / h, \
                (i, k, fd, base["grad"][k])
