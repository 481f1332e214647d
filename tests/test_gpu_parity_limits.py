"""The parity path (precision 64: solve_kernel, eval_kernel, scaling_kernel) against the CPU oracle, bit for bit, at int_K up to 128
and at its largest shared-memory layouts:

  * int_K in INT_K: K + 1 = 32, 33, 64, 66, 83, 84, 101, 128 and 129 samples per piece, on both sides of the 32 / 64 / 128 lanes of
    a one-, two- or four-warp group, and on both sides of the largest int_K whose N = 64, M = 128 layout fits four slots to a CTA;
  * the piece-count edges (64 xy / 128 yaw pieces, one piece, and pairs of them), the map-edge cases of test_gpu_tp_shapes, and long
    generated problems (N > 32), with sample counts S = N (int_K + 1) that are not multiples of 4 (the packed yaw-index table) or
    of 32 (the cost chain's last 32-sample block);
  * eval_batch at the guesses and at perturbed points with random duals on both branches of every inequality, init_scaling_batch,
    solves under budgets of 1, 5 and 30 evaluations against stop_oracle's budget, and unbudgeted solves against the oracle's own;
  * the same solves as four-warp groups, as two-warp groups (UALM_F4=0 UALM_F2=1) and as single warps (UALM_GROUPS=0, which
    refuses a batch holding a problem whose layout does not fit four to a CTA), byte for byte the same;
  * the shared-memory boundary: one N = 64, M = 128 problem at the largest int_K that fits four to a CTA and the next one up (past
    0 and 16), a pair that is over only as maxima, one such problem among 31 ordinary ones (which come back byte for byte as
    without it), and two environments in one batch;
  * the post-solve scan (feasibility) and ualm_check_trajectories of those solves against the oracle's, bit for bit;
  * the throughput path (precision 65) at int_K = 127 on the same cases, trajectory by trajectory (test_solver_control.decided).

test_case_table_reaches_the_edges (no GPU) restates make_layout and fails if the case table stops reaching any of it, and pins the
largest int_K whose N = 64, M = 128 layout fits four slots to a CTA."""
import functools
import os
import re

import numpy as np
import pytest

import workloads
from harness import cat, environ, gpu, same_values, solve_diff, split  # noqa: F401
from workloads import RHO, SHAPES, TP_CASES, _arc_problem, _inputs, _oracle, _per_problem, _shape


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "uneven_planner_b200", "csrc")
INT_K = [31, 32, 63, 65, 81, 82, 83, 100, 127, 128]
BUDGETS = (1, 5, 30)
PASTS = (0, 16)
SMEM_OPTIN = 227 * 1024        # shared memory one CTA may use on an H100 (cudaDevAttrMaxSharedMemoryPerBlockOptin)
RESERVED_SMEM = 1024           # shared memory the device reserves per CTA on sm_80 and later
PARITY_KERNELS = ("solve_kernel", "eval_kernel", "scaling_kernel", "penalty_only_kernel")
MAP_EDGES = ("border_cells", "off_map", "yaw_seam", "short_path")


# ------------------------------------------------------------------ the shared-memory layout, restated
def _define(name):
    with open(os.path.join(CSRC, "ualm_kernels.cuh")) as fh:
        mt = re.search(r"^#define\s+%s\s+(\d+)" % name, fh.read(), re.M)
    assert mt, "no #define %s" % name
    return int(mt.group(1))


def layout_doubles(N, M, n, past, K, S):
    """make_layout(N, M, n, m, past, K, S).total_doubles (ualm_kernels.cuh): one trajectory slot, in doubles"""
    FW, RINGB = _define("UALM_FW"), _define("UALM_RINGB")
    o = 12 * N + 6 * M + 12 * N + 6 * M + N + M + 5 * n + max(past, 1) + (K + 1) + N + 48
    o = (o + 1) & ~1
    o += max(2 * 16 * FW + 2 * 12 * FW, 2 * RINGB * 6 * FW)
    o += 13 * 16 * 2
    o += (S + 3) // 4
    return (o + 1) & ~1


@functools.lru_cache(maxsize=None)
def static_smem():
    """the largest static shared memory of the parity kernels in the built library: a CTA's dynamic shared memory is at most
    SMEM_OPTIN less this.  cuobjdump -res-usage counts in SHARED the 1 KB the device reserves per CTA
    (cudaDevAttrReservedSharedMemoryPerBlock), which SMEM_OPTIN already leaves out"""
    import subprocess
    from uneven_planner_b200 import build
    tool = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    out = subprocess.run([tool, "-res-usage", build.OUT], capture_output=True, text=True, check=True).stdout
    got = {}
    for fn, body in re.findall(r"Function (\S+):\s*\n?(.*)", out):
        for k in PARITY_KERNELS:
            if "ualm%d%s" % (len(k), k) in fn:
                got[k] = int(re.search(r"SHARED:(\d+)", body).group(1))
    assert set(got) == set(PARITY_KERNELS), got
    return max(got.values()) - RESERVED_SMEM


def nvar(N, M):
    return 1 + 2 * (N - 1) + (M - 1)


def four_slots(shapes, K, past):
    """bytes of four slots of the layout sized by the maxima of `shapes` [(N, M)]"""
    N, M = max(s[0] for s in shapes), max(s[1] for s in shapes)
    n, S = max(nvar(*s) for s in shapes), max(s[0] * (K + 1) for s in shapes)
    return 4 * 8 * layout_doubles(N, M, n, past, K, S)


def fits_four(shapes, K, past, cap=None):
    return four_slots(shapes, K, past) <= (SMEM_OPTIN - static_smem() if cap is None else cap)


def largest_fitting_K(N, M, past):
    cap = SMEM_OPTIN - static_smem()
    return max(K for K in range(1, 129) if fits_four([(N, M)], K, past, cap))


# ------------------------------------------------------------------ the cases
def _long(mapdata, B, seed):
    """generated problems whose paths are long enough for N > 32 pieces"""
    from uneven_planner_b200 import problems
    return problems.generate(mapdata, B, seed=seed, min_dist=9.0, n_max=64)


def case_batch(mapdata):
    """the shapes, the map-edge cases and three long generated problems, once each (at their initial guesses)"""
    return cat([_arc_problem(N, M, arc=0.5 * np.pi if N == 1 else 1.5 * np.pi) for N, M in SHAPES.values()] +
                [TP_CASES[k]() for k in MAP_EDGES] + [_long(mapdata, 3, seed=17)])


def _params(K=None, past=None):
    from uneven_planner_b200 import _lib
    p = _lib.default_params()
    if K is not None:
        p.int_K = K
    if past is not None:
        p.past = past
    return p


# ------------------------------------------------------------------ running the path
# the group sizes: UALM_GROUPS is read at ualm_create, UALM_F4 / UALM_F2 at upload, so each covers both
MODES = {"four_warps": {}, "two_warps": {"UALM_F4": "0", "UALM_F2": "1"}, "one_warp": {"UALM_GROUPS": "0"}}


def _solve(gpu, params, mapdata, pb, budget=0, mode="four_warps", prec=64, feas=False):
    """[(record, c_xy, c_yaw)] of pb solved in one context (params / mapdata: one, or one per environment of pb); with feas=True
    also the post-solve scan and ualm_check_trajectories of the solved batch"""
    ps = params if isinstance(params, list) else [params]
    ms = mapdata if isinstance(mapdata, list) else [mapdata]
    with environ(MODES[mode]):
        opt = gpu.BatchALMTrajOpt(precision=prec)
        try:
            for e in range(len(ps)):
                opt.init(ps[e], env=e).set_environment(ms[e], env=e)
            opt.set_budget(budget)
            out = opt.optimize(pb)
            extra = (opt.feasibility(0.01), opt.check_results(pb, out)) if feas else None
        finally:
            opt.close()
    return (split(pb, out), extra) if feas else split(pb, out)


def _same_bits(a, b):
    """equal entry by entry, as the rest of the suite compares the parity path with the oracle (0.0 == -0.0; NaN == NaN)"""
    a, b = np.atleast_1d(np.asarray(a, np.float64)), np.atleast_1d(np.asarray(b, np.float64))
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def _fit_mask(pb, K, past):
    return np.array([fits_four([(int(pb.N[i]), int(pb.M[i]))], K, past) for i in range(pb.B)])


def _every_group_size(gpu, params, mapdata, pb, budget, what):
    """pb solved as four-warp groups, as two-warp groups and as single warps, byte for byte the same; returns the four-warp run.
    Single warps refuse a batch that holds a problem whose layout does not fit four to a CTA: then they solve the others."""
    base = _solve(gpu, params, mapdata, pb, budget)
    two = _solve(gpu, params, mapdata, pb, budget, "two_warps")
    for i in range(pb.B):
        assert same_values(two[i], base[i], equal_nan=True), (what, "two_warps", i)
    fit = _fit_mask(pb, params.int_K, params.past)
    if not fit.all():
        with pytest.raises(gpu.UalmError, match="error -4: UALM_GROUPS=0"):
            _solve(gpu, params, mapdata, pb, budget, "one_warp")
    idx = np.nonzero(fit)[0]
    if idx.size:
        one = _solve(gpu, params, mapdata, pb.select(idx), budget, "one_warp")
        for j, i in enumerate(idx):
            assert same_values(one[j], base[i], equal_nan=True), (what, "one_warp", int(i))
    return base


def _feasibility_against_oracle(pb, params, mapdata, out, feas, chk, what):
    import pyoracle as po
    from check_oracle import check, limits_of
    om = po.OracleMap(mapdata)
    for i, (r, c1, c2) in enumerate(out):
        ref = po.feasibility(om, params.gravity, int(pb.N[i]), int(pb.M[i]), c1, c2, r.piece_T_xy, r.piece_T_yaw, 0.01)
        assert _same_bits(feas[i, :8], ref), (what, "feasibility", i, feas[i, :8], ref)
        rows = check(om, params.gravity, int(pb.N[i]), int(pb.M[i]), c1, c2, r.piece_T_xy, r.piece_T_yaw, 0.01, 0.0, limits_of(params))
        assert _same_bits(chk[i], rows), (what, "check", i, chk[i], rows)


# ------------------------------------------------------------------ fixtures
@pytest.fixture(scope="module")
def cases(bumps_map):
    return case_batch(bumps_map)


# ------------------------------------------------------------------ evaluations against the oracle
@pytest.mark.gpu
@pytest.mark.parametrize("K", INT_K)
def test_eval_and_scaling_bitwise(gpu, cases, bumps_map, K):
    """every case at its guess and at a perturbed point: f, gradient, hx, gx, c_xy, c_yaw, and initScaling's scale_fx and scale_cx"""
    p = _params(K)
    pb = cases.select(np.repeat(np.arange(cases.B), 2))
    Ks = [K] * pb.B
    inputs = _inputs(pb, Ks, seed=K)
    want = _oracle(pb, [p] * pb.B, [bumps_map] * pb.B, Ks, inputs)
    opt = gpu.BatchALMTrajOpt(precision=64).init(p).set_environment(bumps_map)
    try:
        opt.upload(pb)
        xs, lam, mu, scx, sfx = inputs
        ev = opt.eval_batch(xs, lam, mu, scx, sfx, rho=RHO)
        s_fx, s_cx = opt.init_scaling_batch()
    finally:
        opt.close()
    got = _per_problem(pb, Ks, ev, s_fx, s_cx)
    for i in range(pb.B):
        for key in ("f", "grad", "hx", "gx", "c_xy", "c_yaw", "sfx", "scx"):
            assert _same_bits(got[i][key], want[i][key]), (K, i, key)


# ------------------------------------------------------------------ solves against the oracle, in every group size
@pytest.mark.gpu
@pytest.mark.parametrize("K", INT_K)
def test_budgeted_solves_bitwise_in_every_group_size(gpu, cases, bumps_map, K):
    """budgets 1, 5, 30: whole record and coefficients against stop_oracle's budget; the post-solve scan and ualm_check_trajectories of
    the 30-evaluation solves against the oracle's"""
    p = _params(K)
    for k in BUDGETS:
        want = workloads.oracle(p, bumps_map, cases, k)
        got = _every_group_size(gpu, p, bumps_map, cases, k, (K, k))
        for i in range(cases.B):
            assert not solve_diff(got[i], want[i], equal_nan=True), ((K, k, i), solve_diff(got[i], want[i], equal_nan=True))
    out, (feas, chk) = _solve(gpu, p, bumps_map, cases, 30, feas=True)
    _feasibility_against_oracle(cases, p, bumps_map, out, feas, chk, K)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [83, 128])
def test_unbudgeted_solves_bitwise(gpu, cases, bumps_map, K):
    """the oracle's own solve of every case, past the four-slot boundary and at the largest int_K"""
    p = _params(K)
    want = workloads.oracle(p, bumps_map, cases)
    out, (feas, chk) = _solve(gpu, p, bumps_map, cases, feas=True)
    for i in range(cases.B):
        assert not solve_diff(out[i], want[i], equal_nan=True), ((K, i), solve_diff(out[i], want[i], equal_nan=True))
    _feasibility_against_oracle(cases, p, bumps_map, out, feas, chk, K)


# ------------------------------------------------------------------ the shared-memory boundary
@pytest.mark.gpu
@pytest.mark.parametrize("past", PASTS)
def test_largest_problem_on_both_sides_of_four_slots(gpu, bumps_map, past):
    """one N = 64, M = 128 problem at the largest int_K that fits four slots to a CTA, the next one up and 128: evaluation and
    budgeted solves bit for bit the oracle's in every group size that can hold it"""
    k0 = largest_fitting_K(64, 128, past)
    pb = _shape(64, 128)
    for K in (k0, k0 + 1, 128):
        p = _params(K, past)
        want = workloads.oracle(p, bumps_map, pb, 30)
        got = _every_group_size(gpu, p, bumps_map, pb, 30, (past, K))
        assert not solve_diff(got[0], want[0], equal_nan=True), ((past, K), solve_diff(got[0], want[0], equal_nan=True))
        inputs = _inputs(pb, [K], seed=past + K)
        w = _oracle(pb, [p], [bumps_map], [K], inputs)[0]
        opt = gpu.BatchALMTrajOpt(precision=64).init(p).set_environment(bumps_map)
        try:
            opt.upload(pb)
            ev = opt.eval_batch(*inputs, rho=RHO)
        finally:
            opt.close()
        g = _per_problem(pb, [K], ev, inputs[4], inputs[3])[0]
        for key in ("f", "grad", "hx", "gx", "c_xy", "c_yaw"):
            assert _same_bits(g[key], w[key]), (past, K, key)


@pytest.mark.gpu
@pytest.mark.parametrize("past", PASTS)
def test_pair_over_only_as_maxima(gpu, bumps_map, past):
    """N = 64, M = 1 and N = 1, M = 128 at int_K = 128: each fits four slots to a CTA, their maxima do not; as single warps they
    are two launches"""
    p = _params(128, past)
    pb = cat([_shape(64, 1), _shape(1, 128)])
    assert _fit_mask(pb, 128, past).all() and not fits_four([(64, 1), (1, 128)], 128, past)
    want = workloads.oracle(p, bumps_map, pb, 30)
    got = _every_group_size(gpu, p, bumps_map, pb, 30, past)
    for i in range(pb.B):
        assert not solve_diff(got[i], want[i], equal_nan=True), ((past, i), solve_diff(got[i], want[i], equal_nan=True))


@pytest.mark.gpu
@pytest.mark.parametrize("past", PASTS)
def test_one_large_problem_among_ordinary_ones(gpu, hill_map, past):
    """one N = 64, M = 128 problem past the four-slot boundary among 31 bench problems: every problem is solved, the large one bit
    for bit the oracle's, the 31 byte for byte as without it, in every group size"""
    K = largest_fitting_K(64, 128, past) + 1
    p = _params(K, past)
    ordinary = workloads.bench_problems(hill_map, 31)
    pb = cat([ordinary.select(range(0, 13)), _shape(64, 128), ordinary.select(range(13, 31))])
    at = 13
    rest = [i for i in range(pb.B) if i != at]
    alone = _solve(gpu, p, hill_map, ordinary, 30)
    got = _every_group_size(gpu, p, hill_map, pb, 30, past)
    assert all(r.ret_code in (0, 1, 2, 3) and r.n_evals > 0 for r, _, _ in got), [r.ret_code for r, _, _ in got]
    for j, i in enumerate(rest):
        assert same_values(got[i], alone[j], equal_nan=True), (past, i)
    want = workloads.oracle(p, hill_map, pb.select([at]), 30)[0]
    assert not solve_diff(got[at], want, equal_nan=True), ((past, "large"), solve_diff(got[at], want, equal_nan=True))
    # unbudgeted: the large problem still does not hold the others back
    full = _solve(gpu, p, hill_map, pb)
    full_alone = _solve(gpu, p, hill_map, ordinary)
    for j, i in enumerate(rest):
        assert same_values(full[i], full_alone[j], equal_nan=True), (past, "unbudgeted", i)


@pytest.mark.gpu
def test_two_environments_in_one_batch(gpu, bumps_map, hill_map):
    """environment 0 at int_K = 128 with N = 64, M = 128 problems, environment 1 at the default parameters with large problems, in
    one interleaved batch: each problem bit for bit the oracle's with its own environment, and byte for byte each environment alone"""
    ps = [_params(128), _params()]
    ms = [bumps_map, hill_map]
    pbs = [cat([_shape(64, 128), _shape(63, 127), _long(bumps_map, 2, seed=5)]),
           cat([_shape(64, 128), _long(hill_map, 3, seed=9)])]
    mixed = cat(pbs, [0, 1])
    order = np.array([0, 4, 1, 5, 2, 6, 3, 7])
    mixed = mixed.select(order)
    for mode in ("four_warps", "two_warps"):
        got = _solve(gpu, ps, ms, mixed, 30, mode)
        for e in range(2):
            alone = _solve(gpu, ps[e], ms[e], pbs[e], 30, mode)
            want = workloads.oracle(ps[e], ms[e], pbs[e], 30)
            for j in range(pbs[e].B):
                i = int(np.nonzero(order == 4 * e + j)[0][0])
                assert same_values(got[i], alone[j], equal_nan=True), (mode, e, j)
                assert not solve_diff(alone[j], want[j], equal_nan=True), ((mode, e, j), solve_diff(alone[j], want[j], equal_nan=True))


# ------------------------------------------------------------------ the throughput path at int_K = 127
@pytest.mark.gpu
def test_throughput_solves_at_int_K_127(gpu, cases, bumps_map):
    """precision 65, budget 30: every decided trajectory within test_solver_control's rule"""
    p = _params(127)
    ref, mask = workloads.decided(p, bumps_map, cases, 65, 30)
    got = _solve(gpu, p, bumps_map, cases, 30, prec=65)
    n = 0
    for i in np.nonzero(mask)[0]:
        same, err = workloads.trajectory_error(got[i], ref[i])
        assert same and err <= workloads.TOLC[65], (int(i), err)
        n += 1
    print("precision 65, int_K 127, budget 30: %d of %d trajectories decided" % (n, cases.B))
    assert n >= cases.B // 2, n


# ------------------------------------------------------------------ coverage guard (no GPU)
def test_case_table_reaches_the_edges(built, bumps_map):
    """samples per piece on both sides of 32, 64 and 128; S mod 4 != 0 and S mod 32 != 0; a layout over four slots per CTA alone,
    one over only as maxima, and the largest fitting int_K and the next one; long generated problems with N > 32.  Pins the largest
    int_K whose N = 64, M = 128 layout fits four slots to a CTA: a layout change that moves it must say so here"""
    pb = case_batch(bumps_map)
    shapes = [(int(pb.N[i]), int(pb.M[i])) for i in range(pb.B)]
    assert {(64, 128), (63, 127), (48, 128), (64, 64), (64, 1), (1, 128), (2, 1), (1, 1)} <= set(shapes)
    assert (pb.N[-3:] > 32).all(), shapes
    spp = {K + 1 for K in INT_K}
    for lanes in (32, 64, 128):
        assert lanes in spp and any(lanes < s <= lanes + 2 for s in spp), (lanes, spp)
    S = [N * (K + 1) for K in INT_K for N, _ in shapes]
    assert any(s % 4 for s in S) and any(s % 32 and s % 4 == 0 for s in S) and any(s % 32 == 0 for s in S)
    # four slots of the N = 64, M = 128 layout, and the cap they must stay within
    assert four_slots([(64, 128)], 81, 0) == 231744 and four_slots([(64, 128)], 82, 0) == 232256
    assert four_slots([(64, 128)], 128, 0) == 257280
    assert static_smem() == 560
    assert largest_fitting_K(64, 128, 0) == 81 and largest_fitting_K(64, 128, 16) == 80
    for past in PASTS:
        k0 = largest_fitting_K(64, 128, past)
        assert fits_four([(64, 128)], k0, past) and not fits_four([(64, 128)], k0 + 1, past)
        assert not fits_four([(64, 128)], 128, past) and k0 + 1 < 128
        # over only as maxima, and the shapes near the limits that fit at int_K = 128
        assert fits_four([(64, 1)], 128, past) and fits_four([(1, 128)], 128, past) and not fits_four([(64, 1), (1, 128)], 128, past)
        assert fits_four([(48, 128)], 128, past) and fits_four([(64, 64)], 128, past)
    # INT_K reaches both sides of the boundary at past 0, and a case over it in the evaluation and solve sweeps
    k0 = largest_fitting_K(64, 128, 0)
    assert k0 in INT_K and k0 + 1 in INT_K
    assert any(not fits_four([s], K, 0) for K in INT_K for s in shapes)
