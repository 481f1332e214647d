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
from test_gpu_tp_shapes import _cat, _inputs, _offsets, case_batch  # noqa: E402

INT_K = [1, 16, 64, 127]
TERRAINS = ["hill", "desert", "volcano", "forest"]
RHO = 8.0
# the bounds, about 10x the worst relative error measured over the whole table (restatement against the oracle, x86-64):
#   f 8.9e-14 (N1_M128 at its guess); gradient 3.6e-12 (tau part, forest), 7.3e-13 (yaw waypoints), 6.6e-13 (xy waypoints, forest);
#   hx 6.5e-12, a cancellation: at an initial guess the yaw follows the path tangent and hx ~ 1e-3 |v| (border_cells);
#   gx 1.0e-13 (curvature, volcano); c_xy 3.8e-14, c_yaw 5.3e-13 (N1_M128); scale_fx 8.2e-14 (forest);
#   scale_cx 9.5e-12 entry by entry (lateral acceleration, volcano)
TOL = dict(f=1e-12, grad=4e-11, hx=1e-10, hx_cancel=1e-10, con=1e-12, coef=5e-12, sfx=1e-12, scx=1e-10)
LOOSE = 1e-3            # f and gradient of a problem that holds a near-face sample
MAX_NEAR_FACE = 1e-3    # share of the table's samples that may be near a face
KIND = dict(f="f", grad_tau="grad", grad_xy="grad", grad_yaw="grad", hx="hx", hx_cancel="hx_cancel", c_xy="coef", c_yaw="coef", scale_fx="sfx",
            **{"gx%d" % t: "con" for t in range(6)}, **{"scale_cx%d" % t: "scx" for t in range(7)})


# ------------------------------------------------------------------ the table
def _pairs(pb):
    """every problem twice: at its initial guess (even index) and at a perturbed point (odd index)"""
    return pb.select(np.repeat(np.arange(pb.B), 2))


def cases():
    """test_gpu_tp_shapes' case batch and a fast tight turn (4 m/s on a 0.8 m radius: 20 m/s^2 lateral), where the lateral
    acceleration limit is active, each at its guess and perturbed"""
    from test_gpu_minco_fused import _arc_problem
    fast = _pairs(_arc_problem(8, 16, radius=0.8, arc=np.pi, speed=4.0))
    return _cat([case_batch(), fast])


def ridge():
    """a corrugated grid: the normal tilts by up to 37 degrees in x with a 1 m period, so that cos_xi has a large gradient and, on the
    one-piece problems (x = tau alone), initScaling's attitude scales are set by their tau component"""
    from uneven_planner_b200 import _lib, maps
    g = _lib.map_geometry()
    X, Y, W = g.voxel_num
    xs = (np.arange(X) + 0.5) * g.xy_resolution + g.origin[0]
    cells = np.zeros((X, Y, W, 4), np.float32)
    cells[..., 1] = (0.02 * (1.0 + np.cos(2 * np.pi * xs)))[:, None, None]
    cells[..., 2] = (0.6 * np.sin(2 * np.pi * xs))[:, None, None]
    return maps.UnevenMapData(g, cells, "ridge")


def table_entry(key, terrain, bumps_map):
    """(batch, params, grid) of one entry of the case table"""
    from uneven_planner_b200 import _lib, configs, maps, problems
    if key.startswith("K"):
        p = _lib.default_params()
        p.int_K = int(key[1:])
        return cases(), p, bumps_map
    if key in TERRAINS:
        return cases(), configs.params_for(key), terrain(key)
    if key == "tilt":
        return cases(), _lib.default_params(), maps.synthetic_terrain("tilt")
    if key == "ridge":
        return cases(), _lib.default_params(), ridge()
    assert key == "generated"
    gen = [problems.generate(bumps_map, 6, seed=23), problems.generate(terrain("hill"), 6, seed=29, **configs.gen_kwargs("hill"))]
    return _pairs(_cat(gen)), _lib.default_params(), None


KEYS = ["K%d" % k for k in INT_K] + TERRAINS + ["tilt", "ridge", "generated"]


def restated(pb, params, mapdata, Ks, inputs):
    """the restatement's evaluation at `inputs` and initScaling at the initial guess of every problem (problem i with params[i] on
    mapdata[i]), in the layout of test_gpu_tp_shapes._per_problem, plus the per-sample flags"""
    xs, lam, mu, scx, sfx = inputs
    offx, offs, _, _ = _offsets(pb, Ks)
    grids = {id(m): ar.Grid(m) for m in mapdata}
    out = []
    for i in range(pb.B):
        prob, p, g = ar.Problem(pb, i), params[i], grids[id(mapdata[i])]
        r = ar.evaluate(prob, p, g, xs[offx[i]:offx[i + 1]], lam[offs[i]:offs[i + 1]], mu[6 * offs[i]:6 * offs[i + 1]],
                        scx[7 * offs[i]:7 * offs[i + 1]], sfx[i], RHO)
        if i % 2 == 1 and np.array_equal(pb.bnd[i], pb.bnd[i - 1]) and np.array_equal(pb.x0(i), pb.x0(i - 1)):
            r["sfx"], r["scx"], r["near_face_scaling"] = out[i - 1]["sfx"], out[i - 1]["scx"], out[i - 1]["near_face_scaling"]
        else:                                   # the perturbed twin of a problem shares its initial guess and so its initScaling
            r["sfx"], r["scx"], r["near_face_scaling"] = ar.init_scaling(prob, p, g)
        out.append(r)
    return out


def oracle(pb, params, mapdata, Ks, inputs):
    from test_gpu_tp_shapes import _oracle
    return _oracle(pb, params, mapdata, Ks, inputs)


# ------------------------------------------------------------------ the comparison
def _blocks(N, g, o, cancel=False):
    """(name, got, want, whole vector of want, per-entry) for every block of one problem's outputs; cancel: hx is a cancellation
    (test_gpu_tp_shapes.TOLS) and is reported as hx_cancel"""
    nxy = 2 * (N - 1)
    con = np.concatenate([o["hx"], o["gx"]])
    out = [("f", [g["f"]], [o["f"]], [o["f"]], False),
           ("grad_tau", g["grad"][:1], o["grad"][:1], o["grad"], False),
           ("grad_xy", g["grad"][1:1 + nxy], o["grad"][1:1 + nxy], o["grad"], False),
           ("grad_yaw", g["grad"][1 + nxy:], o["grad"][1 + nxy:], o["grad"], False),
           ("hx_cancel" if cancel else "hx", g["hx"], o["hx"], con, False),
           ("c_xy", g["c_xy"], o["c_xy"], o["c_xy"], False),
           ("c_yaw", g["c_yaw"], o["c_yaw"], o["c_yaw"], False),
           ("scale_fx", [g["sfx"]], [o["sfx"]], [o["sfx"]], False)]
    out += [("gx%d" % t, g["gx"][t::6], o["gx"][t::6], con, False) for t in range(6)]
    out += [("scale_cx%d" % t, g["scx"][t::7], o["scx"][t::7], o["scx"], True) for t in range(7)]
    return out


def block_errors(pb, got, want, near=None, cancel=None, entrywise_scales=True):
    """{block: (worst relative error over the batch, problem)}.  A block is measured by the norm of its difference over its own
    norm; a block that is zero up to fp64 rounding (below 1e-9 of its whole vector) against its whole vector; scale_cx entry by
    entry.  near[i]: problem i's near-face samples (a bool per sample), left out of the per-sample blocks; the error of f and the
    gradient of such a problem is reported under "<block>_near".  entrywise_scales=False: scale_cx by norm too, the measure
    test_gpu_tp_shapes.TOLS bound for the float kernels """
    worst = {}
    for i in range(pb.B):
        N = int(pb.N[i])
        nf = None if near is None else np.asarray(near[i], bool)
        for name, a, b, whole, entrywise in _blocks(N, got[i], want[i], cancel is not None and cancel[i]):
            a = np.asarray(a, np.float64)
            b = np.asarray(b, np.float64)
            whole = np.asarray(whole, np.float64)
            if nf is not None and nf.any():
                if name.startswith(("hx", "gx", "scale_cx")):
                    keep = ~nf
                    a, b = a[keep], b[keep]
                elif name.startswith(("f", "grad")):
                    name += "_near"
            if b.size == 0:
                continue
            if entrywise and entrywise_scales:
                err = float(np.max(np.abs(a - b) / np.abs(b)))
            else:
                d = float(np.linalg.norm(a - b))
                nb, nw = float(np.linalg.norm(b)), float(np.linalg.norm(whole))
                if nb <= 1e-9 * nw:
                    nb = nw
                err = d / nb if nb > 0 else (0.0 if d == 0 else np.inf)
            if not np.isfinite(a).all():
                err = np.inf
            if err > worst.get(name, (-1.0, None))[0]:
                worst[name] = (err, i)
    return worst


def check(worst, tol, loose, what):
    bad = {k: v for k, v in worst.items()
           if not v[0] <= (loose if k.endswith("_near") else tol[KIND[k]])}
    assert not bad, (what, bad)


def near_face(ref):
    """per problem: the samples near a cell face in the evaluation or in initScaling"""
    return [r["near_face"] | r["near_face_scaling"] for r in ref]


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
            cache[key] = (pb, ps, ms, Ks, inputs, restated(pb, ps, ms, Ks, inputs), oracle(pb, ps, ms, Ks, inputs))
        return cache[key]
    return get


# ------------------------------------------------------------------ the oracle against the restatement
@pytest.mark.parametrize("key", KEYS)
def test_oracle_matches_restatement_per_block(table, key):
    pb, ps, ms, Ks, inputs, ref, want = table(key)
    near = near_face(ref)
    n = sum(int(v.sum()) for v in near)
    S = sum(len(v) for v in near)
    worst = block_errors(pb, want, ref, near)
    print("%s: %d of %d samples near a face; worst %s" % (key, n, S, {k: "%.1e" % v[0] for k, v in sorted(worst.items())}))
    assert n <= MAX_NEAR_FACE * S, (key, n, S)
    check(worst, TOL, LOOSE, key)


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
