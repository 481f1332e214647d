"""Float64 restatement of ALMTrajOpt's cost evaluation, for tests: innerCallback (alm_traj_opt.cpp:280-347) with
calConstrainCostGrad (:663-991), and initScaling (:349-661), one problem at a time, vectorised over its samples.

It shares no code and no formulation with oracle/oracle.cpp or the kernels:

* MINCO is the dense 6N x 6N system in the row layout of test_oracle_pins.dense_A_b, solved by torch.linalg.solve (partial
  pivoting) instead of the banded LU, and the gradient is torch autograd through it instead of the hand-written adjoint;
* the jerk cost is the integral of the squared third derivative by 4-point Gauss-Legendre (exact at degree 4) instead of the
  closed-form Gram sums;
* the terrain frame is built geometrically from the interpolated unit normal z_b = (zbx, zby, c) and the heading
  h = (cos yaw, sin yaw, 0): x_b = normalise(h - (h.z_b) z_b), y_b = z_b x x_b, instead of the closed forms of getAllWithGrad;
* initScaling's |grad_x c|_inf of every constraint comes from its full Jacobian (forward mode, every direction of x, tau
  included) instead of one adjoint solve per constraint.

What the reference does on purpose is restated explicitly: the repeated-addition sample times and the yaw piece index
int(now / T_yaw) clamped to M - 1 (Q4), zero terrain outside isInMap's 1e-4 margin (Q5), the fixed curvature / sigma scales
without use_scaling (Q6), the x1000 jerk weight in the cost but not in initScaling's scale_fx (Q7), and Q3: the reference
differentiates the sigma^2 running cost in T_i as user_cost / int_K instead of user_cost / T_i (alm_traj_opt.cpp:827), which is
added here to the tau component as sum user_cost (1 / int_K - 1 / T_i) (1 / N) dT/dtau, in the gradient and in scale_fx.

Cell indices carry no gradient: they are fixed in a first pass on the values.  A sample whose position lies within FACE of a
cell face (or of isInMap's margin, or of normSO2's wrap) may pick a different cell in an implementation whose MINCO
coefficients differ at the 1e-15 level, so the map part of the gradient there is legitimately ambiguous: such samples are
flagged in `near_face`.
"""
import math

import numpy as np
import torch

DELTA_SIGL = 0.01       # alm_traj_opt.h:16-19
CUR_SCALE = 10.0
SIG_SCALE = 1000.0
JERK_TRICK = 1000.0
FACE = 1e-9             # in cells: closer than this to a face (or to a margin, in units of the resolution) is ambiguous
F64 = torch.float64
GL_X, GL_W = np.polynomial.legendre.leggauss(4)


class Grid:
    """The double grid the cost reads (the map's own double cells where it has them) and its geometry."""

    def __init__(self, mapdata):
        c64 = getattr(mapdata, "cells64", None)
        cells = np.asarray(mapdata.cells if c64 is None else c64, np.float64)
        g = mapdata.geom
        self.vn = [int(v) for v in g.voxel_num]
        self.origin = [float(v) for v in g.origin]
        self.maxb = [float(v) for v in g.max_boundary]
        self.res, self.yres = float(g.xy_resolution), float(g.yaw_resolution)
        self.cells = torch.from_numpy(np.ascontiguousarray(cells.reshape(-1, 4)[:, 1:]))     # sigma, zbx, zby


class Problem:
    """Problem i of a ProblemBatch: piece counts, boundary states and initial guess."""

    def __init__(self, pb, i):
        self.N, self.M = int(pb.N[i]), int(pb.M[i])
        b = np.asarray(pb.bnd[i], np.float64)
        self.head_xy, self.tail_xy = b[0:6].reshape(3, 2).T, b[6:12].reshape(3, 2).T       # (2, 3): p, v, a columns
        self.head_yaw, self.tail_yaw = b[12:15].reshape(1, 3), b[15:18].reshape(1, 3)
        self.x0 = pb.x0(i)

    @property
    def nvar(self):
        return 1 + 2 * (self.N - 1) + (self.M - 1)


# ------------------------------------------------------------------------------------------------ tau -> T, MINCO
def expC2(tau):
    """alm_traj_opt.h:232-235"""
    return torch.where(tau > 0, (0.5 * tau + 1.0) * tau + 1.0, 1.0 / ((0.5 * tau - 1.0) * tau + 1.0))


def _beta(t, d):
    """d-th derivative of (1, t, ..., t^5)"""
    return torch.stack([(t * 0 if k < d else math.perm(k, d) * t ** (k - d)) for k in range(6)])


def minco(N, Tp, inner, head, tail):
    """coefficients c (6N, D), low power first per piece, of the minimum-jerk spline with N pieces of duration Tp through the
    inner waypoints inner (N - 1, D) with boundary states head / tail (D, 3): the dense system of test_oracle_pins.dense_A_b"""
    n, D = 6 * N, head.shape[0]
    at0 = lambda d: np.array([math.factorial(d) if k == d else 0.0 for k in range(6)])    # _beta(0, d)
    A0 = np.zeros((n, n))
    b0 = np.zeros((n, D))
    b0[0:3] = head.T
    b0[n - 3:] = tail.T
    for d in range(3):
        A0[d, :6] = at0(d)
    for i in range(N - 1):
        r = 6 * i
        for row, d in ((3, 3), (4, 4), (6, 0), (7, 1), (8, 2)):
            A0[r + row, r + 6:r + 12] = -at0(d)
    # the duration-dependent blocks: rows 6i+3 .. 6i+8 (jerk and snap continuity, waypoint, position, velocity and acceleration
    # continuity) and the three tail rows
    blk = torch.stack([_beta(Tp, 3), _beta(Tp, 4), _beta(Tp, 0), _beta(Tp, 0), _beta(Tp, 1), _beta(Tp, 2)])
    tail_blk = torch.stack([_beta(Tp, 0), _beta(Tp, 1), _beta(Tp, 2)])
    rows, cols = [], []
    for i in range(N - 1):
        rr, cc = np.meshgrid(np.arange(6 * i + 3, 6 * i + 9), np.arange(6 * i, 6 * i + 6), indexing="ij")
        rows.append(rr.ravel()); cols.append(cc.ravel())
    rr, cc = np.meshgrid(np.arange(n - 3, n), np.arange(n - 6, n), indexing="ij")
    rows.append(rr.ravel()); cols.append(cc.ravel())
    flat = torch.from_numpy(np.concatenate(rows) * n + np.concatenate(cols))
    vals = torch.cat([blk.reshape(-1).repeat(N - 1), tail_blk.reshape(-1)])
    A = torch.from_numpy(A0) + torch.zeros(n * n, dtype=F64).scatter(0, flat, vals).reshape(n, n)
    wp_rows = torch.from_numpy(np.arange(N - 1) * 6 + 5)
    b = torch.from_numpy(b0) + torch.zeros(n, D, dtype=F64).index_add(0, wp_rows, inner.reshape(N - 1, D))
    return torch.linalg.solve(A, b)


def jerk_cost(c, N, Tp):
    """sum over pieces and dimensions of the integral of the squared third derivative, 4-point Gauss-Legendre"""
    t = 0.5 * Tp * (torch.from_numpy(GL_X) + 1.0)                             # (4,)
    b3 = torch.stack([_beta(tk, 3) for tk in t])                               # (4, 6)
    j = torch.einsum("gk,pkd->pgd", b3, c.reshape(N, 6, -1))
    return 0.5 * Tp * torch.einsum("g,pgd->", torch.from_numpy(GL_W), j * j)


# ------------------------------------------------------------------------------------------------ sample times
def _times(prob, K, Tx, Ty):
    """per sample (piece i, index j): s1 by repeated addition of T_i / int_K, now = s1 + base_time, yaw piece and local time,
    the trapezoid weight; all from the float durations, as the reference computes them"""
    N, M = prob.N, prob.M
    i_s, j_s, s1, now = [], [], [], []
    base = 0.0
    for i in range(N):
        step, s = Tx / K, 0.0
        for j in range(K + 1):
            i_s.append(i); j_s.append(j); s1.append(s); now.append(s + base)
            s += step
        base += Tx
    now = np.array(now)
    yi = np.minimum((now / Ty).astype(np.int64), M - 1)                       # Q4
    j_s = np.array(j_s)
    w = np.where((j_s == 0) | (j_s == K), 0.5, 1.0)
    return dict(i=np.array(i_s), j=j_s, alpha=j_s / K, s1=np.array(s1), now=now, yi=yi, w=w, yaw_clamped=(now / Ty).astype(np.int64) >= M)


def _kinematics(c_xy, c_yaw, Tx, Ty, tm, N, M):
    """position, velocity, acceleration of the xy spline and yaw, its rate and acceleration at every sample.  The sample times
    keep the reference's float values and carry the exact derivative in the piece durations: s1 = alpha T_i, now = (i + alpha) T_i
    (uniform durations)."""
    i_s = torch.from_numpy(tm["i"]); yi = torch.from_numpy(tm["yi"])
    alpha = torch.from_numpy(tm["alpha"])
    dTx = Tx - Tx.detach()
    s1 = torch.from_numpy(tm["s1"]) + alpha * dTx
    now = torch.from_numpy(tm["now"]) + (i_s + alpha) * dTx
    sy = now - yi * Ty
    cx = c_xy.reshape(N, 6, 2)[i_s]                                            # (S, 6, 2)
    cy = c_yaw.reshape(M, 6)[yi]                                               # (S, 6)
    B = [_beta(s1, d).T for d in range(3)]                                     # (S, 6)
    Y = [_beta(sy, d).T for d in range(3)]
    p, v, a = (torch.einsum("sk,skd->sd", Bd, cx) for Bd in B)
    yaw, dyaw, d2yaw = ((Yd * cy).sum(1) for Yd in Y)
    return p, v, a, yaw, dyaw, d2yaw


# ------------------------------------------------------------------------------------------------ the map query
def _norm_so2(y):
    """uneven_map.cpp:64-71 on float values"""
    y = y.copy()
    while True:
        lo, hi = y < -np.pi, y > np.pi
        if not (lo.any() or hi.any()):
            return y
        y = np.where(lo, y + 2 * np.pi, np.where(hi, y - 2 * np.pi, y))


def _cells(grid, p, yaw):
    """the cell choice of uneven_map.h:258-315 at the float positions: isInMap (1e-4 margin), the pos - res/2 base index,
    boundIndex (clamp in x and y, wrap in yaw) of the eight corners, and the flags"""
    x, y = p[:, 0], p[:, 1]
    yn = _norm_so2(yaw)
    o, mx, res, yres, vn = grid.origin, grid.maxb, grid.res, grid.yres, grid.vn
    pos = [x, y, yn]
    inside = np.ones(len(x), bool)
    margin = np.zeros(len(x), bool)
    for k in range(3):
        r = res if k < 2 else yres
        inside &= ~((pos[k] < o[k] + 1e-4) | (pos[k] > mx[k] - 1e-4))
        margin |= (np.abs(pos[k] - (o[k] + 1e-4)) < FACE * r) | (np.abs(pos[k] - (mx[k] - 1e-4)) < FACE * r)
    pm = [x - 0.5 * res, y - 0.5 * res, yn - 0.5 * yres]
    wrap = np.abs(np.abs(pm[2]) - np.pi) < FACE * yres
    pm[2] = _norm_so2(pm[2])
    u = [(pm[0] - o[0]) / res, (pm[1] - o[1]) / res, (pm[2] - o[2]) / yres]
    idx = [np.floor(uk).astype(np.int64) for uk in u]
    face = np.zeros(len(x), bool)
    for uk in u:
        face |= np.abs(uk - np.rint(uk)) < FACE
    corners = []
    for dx in (0, 1):
        for dy in (0, 1):
            for dw in (0, 1):
                cx = np.clip(idx[0] + dx, 0, vn[0] - 1)
                cy = np.clip(idx[1] + dy, 0, vn[1] - 1)
                cw = np.mod(idx[2] + dw, vn[2])
                corners.append((cx * vn[1] + cy) * vn[2] + cw)
    return dict(yn_shift=yn - yaw, inside=inside, idx=np.stack(idx, 1), corners=np.stack(corners, 1),
                near_face=inside & (face | wrap) | margin,
                border=inside & ((idx[0] < 0) | (idx[1] < 0) | (idx[0] + 1 > vn[0] - 1) | (idx[1] + 1 > vn[1] - 1)),
                seam=inside & ((idx[2] < 0) | (idx[2] + 1 > vn[2] - 1)))


def terrain(grid, mp, p, yaw):
    """(sigma, zbx, zby) by trilinear interpolation, zero outside the map (Q5); the weights are differentiable, the cells fixed"""
    o, res, yres = grid.origin, grid.res, grid.yres
    idx = torch.from_numpy(mp["idx"]).to(F64)
    yn = yaw + torch.from_numpy(mp["yn_shift"])
    d0 = (p[:, 0] - ((idx[:, 0] + 0.5) * res + o[0])) / res
    d1 = (p[:, 1] - ((idx[:, 1] + 0.5) * res + o[1])) / res
    e = yn - ((idx[:, 2] + 0.5) * yres + o[2])
    d2 = torch.atan2(torch.sin(e), torch.cos(e)) / yres
    v = grid.cells[torch.from_numpy(mp["corners"])].reshape(-1, 2, 2, 2, 3)    # [x][y][yaw]
    wx = torch.stack([1 - d0, d0], 1)
    wy = torch.stack([1 - d1, d1], 1)
    ww = torch.stack([1 - d2, d2], 1)
    val = torch.einsum("sa,sb,sc,sabck->sk", wx, wy, ww, v)
    val = torch.where(torch.from_numpy(mp["inside"])[:, None], val, torch.zeros_like(val))
    return val[:, 0], val[:, 1], val[:, 2], yn


def frame(zbx, zby, yaw):
    """the terrain frame from the unit normal z_b and the heading h: (inv_cos_vphix, sin_phix, inv_cos_vphiy, sin_phiy, cos_xi,
    inv_cos_xi)"""
    c = torch.sqrt(1.0 - zbx * zbx - zby * zby)
    zb = torch.stack([zbx, zby, c], 1)
    h = torch.stack([torch.cos(yaw), torch.sin(yaw), torch.zeros_like(yaw)], 1)
    p = h - (h * zb).sum(1, keepdim=True) * zb
    np_ = torch.sqrt((p * p).sum(1))
    xb = p / np_[:, None]
    yb = torch.linalg.cross(zb, xb, dim=1)
    return 1.0 / np_, xb[:, 2], 1.0 / torch.sqrt(1.0 - yb[:, 2] ** 2), yb[:, 2], zb[:, 2], 1.0 / zb[:, 2]


# ------------------------------------------------------------------------------------------------ the cost
class _Setup:
    """everything that carries no gradient: durations' float values, sample times, cell choices and flags"""

    def __init__(self, prob, prm, grid, x):
        self.prob, self.prm, self.grid = prob, prm, grid
        self.K = int(prm.int_K)
        N, M = prob.N, prob.M
        with torch.no_grad():
            xt = torch.as_tensor(np.asarray(x, np.float64))
            T = expC2(xt[0])
            self.Tx, self.Ty = float(T / N), float(T / M)
            self.tm = _times(prob, self.K, self.Tx, self.Ty)
            c_xy, c_yaw = self.splines(xt)
            p, _, _, yaw, _, _ = _kinematics(c_xy, c_yaw, T / N, T / M, self.tm, N, M)
            self.mp = _cells(grid, p.numpy(), yaw.numpy())

    def splines(self, x):
        prob, N, M = self.prob, self.prob.N, self.prob.M
        T = expC2(x[0])
        c_xy = minco(N, T / N, x[1:1 + 2 * (N - 1)], prob.head_xy, prob.tail_xy)
        c_yaw = minco(M, T / M, x[1 + 2 * (N - 1):], prob.head_yaw, prob.tail_yaw)
        return c_xy, c_yaw

    def samples(self, x):
        """T, the splines, and per sample: sigma, the unscaled constraints (S, 7) and the trapezoid weights"""
        prm, N, M = self.prm, self.prob.N, self.prob.M
        T = expC2(x[0])
        Tx, Ty = T / N, T / M
        c_xy, c_yaw = self.splines(x)
        p, v, a, yaw, dyaw, _ = _kinematics(c_xy, c_yaw, Tx, Ty, self.tm, N, M)
        sigma, zbx, zby, yn = terrain(self.grid, self.mp, p, yaw)
        icvx, spx, icvy, spy, cxi, icxi = frame(zbx, zby, yn)
        cy, sy = torch.cos(yaw), torch.sin(yaw)
        lon = a[:, 0] * cy + a[:, 1] * sy
        lat = -a[:, 0] * sy + a[:, 1] * cy
        vx2 = (v * v).sum(1) * icvx * icvx
        wz = dyaw * icxi
        ax = lon * icvx + prm.gravity * spx
        ay = lat * icvy + prm.gravity * spy
        curv = wz * wz / (vx2 + DELTA_SIGL)
        con = torch.stack([v[:, 0] * sy - v[:, 1] * cy,
                           vx2 - prm.max_vel ** 2,
                           ax * ax - prm.max_acc_lon ** 2,
                           ay * ay - prm.max_acc_lat ** 2,
                           curv - prm.max_kap ** 2,
                           prm.min_cxi - cxi,
                           sigma - prm.max_sig], 1)
        return T, Tx, c_xy, c_yaw, sigma, con

    def f_part(self, T, Tx, c_xy, c_yaw, sigma, scale_fx):
        """jerk (unweighted), rho_T T and the sigma^2 running cost, the last two times scale_fx; and the running cost per sample"""
        N, M, prm = self.prob.N, self.prob.M, self.prm
        jerk = jerk_cost(c_xy, N, Tx) + jerk_cost(c_yaw, M, T / M)
        user = prm.rho_ter * (Tx / self.K) * torch.from_numpy(self.tm["w"]) * scale_fx * sigma * sigma
        return jerk, prm.rho_T * T * scale_fx, user

    def q3(self, x, user):
        """Q3: the reference's tau gradient of the running cost minus the exact one, sum user (1 / int_K - 1 / T_i) (1 / N) dT/dtau"""
        tau = torch.tensor(float(x[0]), dtype=F64, requires_grad=True)
        dT = float(torch.autograd.grad(expC2(tau), tau)[0])
        return float(user.detach().sum()) * (1.0 / self.K - 1.0 / self.Tx) / self.prob.N * dT


def evaluate(prob, prm, grid, x, lam=None, mu=None, scale_cx=None, scale_fx=1.0, rho=None, q3=True):
    """innerCallback at x with duals lam (S) / mu (6S), scales scale_cx (7S, 7 per sample: hx, then the six gx) and scale_fx, and
    penalty weight rho: f, grad, hx, gx, c_xy (6N x 2 column-major), c_yaw, and per sample near_face, active (S, 6) and the reach
    flags off_map / border / seam / yaw_clamped.  q3=False: the exact gradient, without the reference's Q3"""
    st = _Setup(prob, prm, grid, x)
    S = prob.N * (st.K + 1)
    lam = torch.zeros(S, dtype=F64) if lam is None else torch.as_tensor(np.asarray(lam, np.float64))
    mu = torch.zeros(S, 6, dtype=F64) if mu is None else torch.as_tensor(np.asarray(mu, np.float64)).reshape(S, 6)
    scx = torch.ones(S, 7, dtype=F64) if scale_cx is None else torch.as_tensor(np.asarray(scale_cx, np.float64)).reshape(S, 7)
    rho = float(prm.rho if rho is None else rho)
    xt = torch.tensor(np.asarray(x, np.float64), requires_grad=True)
    T, Tx, c_xy, c_yaw, sigma, con = st.samples(xt)
    fixed = torch.ones(S, 7, dtype=F64)
    if not prm.use_scaling:                                                     # Q6
        fixed[:, 4], fixed[:, 6] = CUR_SCALE, SIG_SCALE
    scale = torch.where(fixed != 1.0, fixed, scx)
    c = con * scale
    hx, gx = c[:, 0], c[:, 1:]
    aug = hx * (lam + 0.5 * rho * hx)
    active = rho * gx + mu > 0
    ineq = torch.where(active, gx * (mu + 0.5 * rho * gx), -0.5 * mu * mu / rho)
    jerk, tcost, user = st.f_part(T, Tx, c_xy, c_yaw, sigma, scale_fx)
    jerk = jerk * scale_fx * (JERK_TRICK if prm.use_scaling else 1.0)
    f = jerk + tcost + user.sum() + aug.sum() + ineq.sum()
    grad = torch.autograd.grad(f, xt)[0].numpy().copy()
    if q3:
        grad[0] += st.q3(x, user)
    mp = st.mp
    return dict(f=float(f.detach()), grad=grad, hx=hx.detach().numpy(), gx=gx.detach().numpy().ravel(),
                c_xy=c_xy.detach().numpy().T.ravel(), c_yaw=c_yaw.detach().numpy().ravel(),
                near_face=mp["near_face"], active=active.numpy(), off_map=~mp["inside"], border=mp["border"], seam=mp["seam"],
                yaw_clamped=st.tm["yaw_clamped"])


def init_scaling(prob, prm, grid, x0=None, chunk=32):
    """initScaling at x0 (default: the problem's initial guess): scale_fx, scale_cx (7 per sample) and near_face per sample"""
    x0 = prob.x0 if x0 is None else np.asarray(x0, np.float64)
    st = _Setup(prob, prm, grid, x0)
    xt = torch.tensor(x0)

    def cons(x):
        return st.samples(x)[5].reshape(-1)

    def column(e):
        return torch.func.jvp(cons, (xt,), (e,))[1]
    J = torch.func.vmap(column, chunk_size=chunk)(torch.eye(len(x0), dtype=F64))  # (nvar, 7S)
    scale_cx = 1.0 / torch.clamp(J.abs().amax(0), min=1.0)
    xg = torch.tensor(x0, requires_grad=True)
    T, Tx, c_xy, c_yaw, sigma, _ = st.samples(xg)
    jerk, tcost, user = st.f_part(T, Tx, c_xy, c_yaw, sigma, 1.0)              # Q7: no x1000 here
    g = torch.autograd.grad(jerk + tcost + user.sum(), xg)[0].numpy().copy()
    g[0] += st.q3(x0, user)
    return 1.0 / max(1.0, float(np.abs(g).max())), scale_cx.numpy(), st.mp["near_face"]
