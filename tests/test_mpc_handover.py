"""The hand-over to the MPC (ualm_mpc_export_batch, csrc/ualm_kernels.cuh: mpc_export_kernel) restated on the host, and checked here
without a GPU.

The three outputs of the hand-over are restated operation for operation, so that tests/test_gpu_mpc_export.py holds the kernel to
them bit for bit (libualm's C ABI translation unit is compiled with -fmad=false, as the oracle is without contraction):
  message_ref  the SE2Traj message: piece start points and PolyTrajectory::getValue(total), total = the piece duration added once per
               piece;
  mpc_ref      the MPC side's MINCO re-solve of that message (orc_minco_generate == mpc_controller's MinJerkOpt::generate, pinned by
               tests/test_ref_pin.py) with the message's init_v / init_a = {x, y, yaw} and zero tail derivatives;
  dev_ref      the planned-vs-tracked scan: samples 0, dt, 2dt, .. formed by repeated addition and kept while t < the shorter of the
               two summed durations, locatePieceIdx's subtract loop, Piece::getValue's Horner-free power order, sqrt(dx*dx + dy*dy),
               the largest value with the earliest sample among equal ones; a scan of 4e6 samples or more is not made: {-1, 0, -1, 0}.

The oracle's re-solve is itself checked against the same MINCO conditions solved in 50-digit arithmetic (mpmath) at nonzero head
derivatives, and its spline against those conditions at the first and last knot."""
import ctypes as C

import numpy as np
import pytest

from workloads import DEV_GUARD, INIT_A, INIT_V, dev_ref, evaluate, first_max, message_ref, minco, mpc_ref, orc, summed


# ------------------------------------------------------------------ the references against plain loops
def _loop_eval(c, P, dur, t):
    idx = 0
    while idx < P and t > dur:
        t -= dur
        idx += 1
    if idx == P:
        idx -= 1
        t += dur
    v, tn = 0.0, 1.0
    for k in range(6):
        v += tn * c[6 * idx + k]
        tn *= t
    return v


def _loop_dev(cxy, cyaw, mxy, myaw, N, M, Tx, Ty, dt):
    """the scan as one sequential loop, the order of the reference's own scans"""
    total = min(summed(Tx, N), summed(Ty, M))
    if not (total / dt < DEV_GUARD):
        return [-1.0, 0.0, -1.0, 0.0]
    t, bp, bpt, by, byt = 0.0, 0.0, 0.0, 0.0, 0.0
    nx = 6 * N
    while t < total:
        dx = _loop_eval(cxy[:nx], N, Tx, t) - _loop_eval(mxy[:nx], N, Tx, t)
        dy = _loop_eval(cxy[nx:], N, Tx, t) - _loop_eval(mxy[nx:], N, Tx, t)
        ep = float(np.sqrt(dx * dx + dy * dy))
        ey = abs(_loop_eval(cyaw, M, Ty, t) - _loop_eval(myaw, M, Ty, t))
        if bp < ep:
            bp, bpt = ep, t
        if by < ey:
            by, byt = ey, t
        t += dt
    return [bp, bpt, by, byt]


@pytest.fixture(scope="module")
def solved(built, bumps_map):
    """three oracle solves on the bumps map (N, M of a few pieces each) with their piece durations"""
    import pyoracle as po
    from uneven_planner_b200 import _lib, problems
    params = _lib.default_params()
    pb = problems.generate(bumps_map, 3, seed=8)
    out = []
    for i, (r, cxy, cyaw, _) in enumerate(po.solve_batch(po.params_from(params), po.OracleMap(bumps_map), pb)):
        N, M = int(pb.N[i]), int(pb.M[i])
        out.append((N, M, cxy, cyaw, r.total_T / N, r.total_T / M))
    return out


def test_locate_and_evaluate_match_the_sequential_restatement(solved):
    """the vectorised locatePieceIdx / getValue equal the scalar loop at every knot, next to it and past the end"""
    for N, M, cxy, cyaw, Tx, Ty in solved:
        for c, P, dur in ((cxy[:6 * N], N, Tx), (cxy[6 * N:], N, Tx), (cyaw, M, Ty)):
            knots = np.cumsum(np.full(P, dur))
            t = np.concatenate([[0.0], knots, np.nextafter(knots, 0.0), np.nextafter(knots, np.inf), [summed(dur, P) * 1.5]])
            got = evaluate(c, P, dur, t)
            assert np.array_equal(got, [_loop_eval(c, P, dur, x) for x in t])


def test_message_ref_is_the_publish_loop(solved):
    """start points are the constant coefficients; the end point is getValue at the summed duration"""
    for N, M, cxy, cyaw, Tx, Ty in solved:
        m = message_ref(cxy, cyaw, N, M, Tx, Ty)
        assert np.array_equal(m["pos_pts"][:N, 0], cxy[0:6 * N:6]) and np.array_equal(m["angle_pts"][:M], cyaw[0::6])
        assert m["pos_pts"][N, 1] == _loop_eval(cxy[6 * N:], N, Tx, summed(Tx, N))
        assert m["angle_pts"][M] == _loop_eval(cyaw, M, Ty, summed(Ty, M))


@pytest.mark.parametrize("dt", [0.01, 0.0137, 0.37, 1e3])
def test_dev_ref_matches_the_sequential_scan(orc, solved, dt):
    """dev_ref (vectorised) equals the scan written as one loop in time order, bit for bit, at zero and nonzero heads; a dt past
    every duration keeps the one sample t = 0, where both splines start at the same point and angle"""
    for N, M, cxy, cyaw, Tx, Ty in solved:
        for v, a in ((None, None), (INIT_V, INIT_A)):
            mx, my = mpc_ref(orc, message_ref(cxy, cyaw, N, M, Tx, Ty), Tx, Ty, v, a)
            got = dev_ref(cxy, cyaw, mx, my, N, M, Tx, Ty, dt)
            assert np.array_equal(got, _loop_dev(cxy, cyaw, mx, my, N, M, Tx, Ty, dt)), (N, M, dt)
            if dt == 1e3:
                assert np.array_equal(got, np.zeros(4))


def test_dev_ref_guard_and_ties(orc, solved):
    """at the guard: total / dt just under 4e6 is scanned, at or over it gives {-1, 0, -1, 0}.  Ties: equal maxima keep the earliest
    sample; a deviation that is zero everywhere keeps (0, 0)"""
    N, M, cxy, cyaw, Tx, Ty = solved[0]
    mx, my = mpc_ref(orc, message_ref(cxy, cyaw, N, M, Tx, Ty), Tx, Ty)
    total = min(summed(Tx, N), summed(Ty, M))
    over = total / DEV_GUARD
    assert not (total / over < DEV_GUARD)
    assert np.array_equal(dev_ref(cxy, cyaw, mx, my, N, M, Tx, Ty, over), [-1.0, 0.0, -1.0, 0.0])
    under = np.nextafter(over, np.inf)
    assert total / under < DEV_GUARD
    assert dev_ref(cxy, cyaw, mx, my, N, M, Tx, Ty, under)[0] > 0.0
    vals = np.array([0.0, 2.0, 1.0, 2.0, np.nan, 2.0])
    t = np.arange(6) * 0.5
    assert first_max(vals, t) == (2.0, 0.5)
    assert first_max(np.zeros(6), t) == (0.0, 0.0)
    # the same spline as planned and tracked: zero everywhere
    assert np.array_equal(dev_ref(cxy, cyaw, cxy, cyaw, N, M, Tx, Ty, 0.01), np.zeros(4))


# ------------------------------------------------------------------ the oracle's re-solve against a 50-digit solve
def _mp_minco(pts, T, v0, a0, dps=50):
    """the MINCO conditions of a P-piece quintic spline with uniform durations T, solved in `dps`-digit arithmetic:
    interpolation of pts (P + 1, Dim), head position / velocity / acceleration (pts[0], v0, a0), tail (pts[P], 0, 0), and continuity of
    derivatives 1 to 4 at every interior knot.  Gaussian elimination with partial pivoting on sparse rows.  Returns 6P x Dim
    coefficients (column-major, as orc_minco_generate) as mpf."""
    import mpmath as mp
    mp.mp.dps = dps
    P, Dim = pts.shape[0] - 1, pts.shape[1]
    T = mp.mpf(float(T))
    n = 6 * P

    def drow(piece, d, t):          # d-th derivative of piece `piece` at local time t, as {column: coefficient}
        r = {}
        for k in range(d, 6):
            f = mp.mpf(1)
            for j in range(d):
                f *= k - j
            r[6 * piece + k] = f * (t ** (k - d) if k > d else mp.mpf(1))
        return r

    rows, rhs = [], []
    zero = [mp.mpf(0)] * Dim
    for d, val in ((0, pts[0]), (1, v0), (2, a0)):
        rows.append(drow(0, d, mp.mpf(0)))
        rhs.append([mp.mpf(float(x)) for x in val])
    for i in range(1, P):
        rows.append(drow(i - 1, 0, T)); rhs.append([mp.mpf(float(x)) for x in pts[i]])
        rows.append(drow(i, 0, mp.mpf(0))); rhs.append([mp.mpf(float(x)) for x in pts[i]])
        for d in range(1, 5):
            r = drow(i - 1, d, T)
            for k, x in drow(i, d, mp.mpf(0)).items():
                r[k] = r.get(k, 0) - x
            rows.append(r); rhs.append(list(zero))
    for d, val in ((0, pts[P]), (1, zero), (2, zero)):
        rows.append(drow(P - 1, d, T))
        rhs.append([mp.mpf(float(x)) for x in val])
    assert len(rows) == n
    for k in range(n):
        cand = [i for i in range(k, n) if rows[i].get(k, 0) != 0]
        p = max(cand, key=lambda i: abs(rows[i][k]))
        rows[k], rows[p] = rows[p], rows[k]
        rhs[k], rhs[p] = rhs[p], rhs[k]
        piv = rows[k][k]
        for i in range(k + 1, n):
            if rows[i].get(k, 0) == 0:
                continue
            f = rows[i][k] / piv
            for j, x in rows[k].items():
                rows[i][j] = rows[i].get(j, 0) - f * x
            rows[i].pop(k)
            rhs[i] = [a - f * b for a, b in zip(rhs[i], rhs[k])]
    x = [[mp.mpf(0)] * Dim for _ in range(n)]
    for k in range(n - 1, -1, -1):
        s = list(rhs[k])
        for j, a in rows[k].items():
            if j > k:
                s = [u - a * w for u, w in zip(s, x[j])]
        x[k] = [u / rows[k][k] for u in s]
    return [[x[k][d] for k in range(n)] for d in range(Dim)]


def _waypoints(P, Dim, seed):
    """P + 1 seeded points of a smooth path: xy a few metres long, yaw within a few radians"""
    rng = np.random.default_rng(seed)
    steps = rng.uniform(0.2, 0.5, (P, Dim)) * rng.choice([-1.0, 1.0], (P, Dim))
    return np.vstack([rng.uniform(-2.0, 2.0, (1, Dim)), rng.uniform(-2.0, 2.0, (1, Dim)) + np.cumsum(steps, axis=0)])


# Relative error of orc_minco_generate against the 50-digit solve, per dimension: ||c - c_mp|| / ||c_mp||, over N in {1, 2, 5, 64},
# T in {0.24, 1.0, 2.7} s, xy and yaw right-hand sides, head (INIT_V, INIT_A).  Measured worst case (x86-64, g++ without FMA
# contraction): 3.3e-15 (N = 64, T = 0.24 s, yaw).  The tolerance keeps a margin of 30x over it.  KNOT_TOL: the tail conditions
# at the last knot, |p(T) - point|, |p'(T)| T and |p''(T)| T^2 over the largest |c_k T^k| of the last piece; measured worst 2.9e-15
# (N = 64, T = 2.7 s, yaw), margin 34x.
MINCO_TOL = 1e-13
KNOT_TOL = 1e-13


@pytest.mark.parametrize("T", [0.24, 1.0, 2.7])
@pytest.mark.parametrize("N", [1, 2, 5, 64])
def test_oracle_minco_at_nonzero_heads_against_50_digits(orc, N, T):
    """orc_minco_generate at a nonzero head velocity / acceleration solves the MINCO conditions: within MINCO_TOL of the 50-digit
    solution, its first knot meets the head exactly (c0 = point, c1 = v0, c2 = a0 / 2: rows 0-2 of the band are never eliminated)
    and its last knot meets the tail within rounding"""
    import mpmath as mp
    for Dim, v0, a0, seed in ((2, INIT_V[:2], INIT_A[:2], 10 * N + 1), (1, INIT_V[2:], INIT_A[2:], 10 * N + 2)):
        pts = _waypoints(N, Dim, seed)
        c = minco(orc, pts, T, v0, a0)
        want = _mp_minco(pts, T, v0, a0)
        for d in range(Dim):
            cd = c[6 * N * d:6 * N * (d + 1)]
            wd = want[d]
            err = mp.sqrt(mp.fsum((mp.mpf(float(a)) - b) ** 2 for a, b in zip(cd, wd))) / mp.sqrt(mp.fsum(b ** 2 for b in wd))
            assert float(err) <= MINCO_TOL, (N, T, Dim, d, float(err))
            assert cd[0] == pts[0, d] and cd[1] == v0[d] and cd[2] == a0[d] / 2, (N, T, Dim, d)
            last = cd[6 * (N - 1):]
            tp = T ** np.arange(6)
            p = float(last @ tp)
            v = float(last[1:] @ (np.arange(1, 6) * tp[:5]))
            a = float(last[2:] @ (np.arange(2, 6) * np.arange(1, 5) * tp[:4]))
            scale = float(np.abs(last * tp).max())
            assert max(abs(p - pts[N, d]), abs(v) * T, abs(a) * T * T) <= KNOT_TOL * scale, (N, T, Dim, d)
