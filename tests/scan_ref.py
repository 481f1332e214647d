"""Float64 restatement of the stages around the solve, for tests: the post-solve scan (ALMTrajOpt::getMaxVxAxAyCurAttSig with
getNonHolError, alm_traj_opt.h:170-229), the check of trajectories a caller holds (ualm_check_trajectories: the same scan from t_from
on, with the first time each of six limits is broken) and the replan build (ualm_submit_replan: the state at t_from, the polyline of
the trajectory's samples and PlanManager's resampler, plan_manager.cpp:62-122), one trajectory at a time, vectorised over its samples.

It shares no code and no formulation with oracle/oracle.cpp, tests/check_oracle.cpp, tests/replan_oracle.cpp or the kernels:

* a piece is chosen by comparing the time with the piece boundaries i T (not by repeated subtraction), and evaluated by Horner's
  rule with np.polynomial (polyval, polyder) instead of the power loop.  The splines are C4 at the joins, so where the two choices
  differ (a time within rounding of a boundary) both give the same values to rounding;
* the terrain values and frame are alm_ref's (trilinear interpolation of the cells alm_ref._cells picks, zero outside isInMap's 1e-4
  margin; the frame built geometrically from the unit normal and the heading), and each scanned quantity is written from the
  constraint definitions of alm_ref._Setup.samples, so the scan reports what the cost constrains: vx = |v| inv_cos_vphix (vx2 = vx^2),
  ax = lon inv_cos_vphix + g sin_phix, ay = lat inv_cos_vphiy + g sin_phiy, cur = dyaw inv_cos_xi / sqrt(vx^2 + 0.01) (curv = cur^2),
  att = -cos_xi, sig = sigma, and the non-holonomic term |v_x sin yaw - v_y cos yaw| (constraint 0);
* the reductions are numpy's: the signed abs-max keeps the earliest sample of the largest magnitude, the non-holonomic error is
  math.fsum, the first violation is the first index of a boolean mask;
* the yaw smoothing is written in closed form with floor, and the arc-length resampling places waypoint k at the arc length
  k piece_len by a search in the cumulative length, instead of the reference's running remainders.

Only what the reference defines by its float additions is reused, not restated: the durations N T_xy and M T_yaw summed one piece at a
time and their minimum (workloads.summed), and the sample sequence t = 0, dt, 2dt.. by repeated addition (workloads.scan_times).

What the reference does on purpose, restated explicitly:
  S1  the map is queried at the yaw normalised to [-pi, pi] (getNormSE2Pos), while lon / lat and the non-holonomic term take sin / cos
      of the yaw as the trajectory carries it;
  S2  the maxima start at 0 (vx, ax, ay, cur, sig) and -1 (att) and keep strict increases, so an empty window reports those;
  S3  a row is not scanned when total / dt >= 4e6 (a diverged solve), or, on the device, when N > 64 or M > 128;
  S4  the replan polyline keeps the samples t_from < t < duration (strictly after t_from: the point at t_from is its first point);
  S5  the yaw smoothing is pm.cpp:62-77's two loops, subtract whole turns while dyaw >= pi/2, then add them while dyaw <= -pi/2.  A
      difference of exactly pi/2 (mod 2 pi) therefore ends at +pi/2, not inside (-pi/2, pi/2);
  S6  the product's bound on the replan build: a polyline that needs more than 4095 waypoints of either kind, a yaw of magnitude 2^40
      or more or more than 65536 whole turns of smoothing is cut short, N' = M' = 4097, total_time still its whole length's.

Ambiguity, flagged as alm_ref flags it: trilinear interpolation is continuous across interior cell faces, the clamped border and the
yaw seam, so only a sample within FACE (in resolutions) of isInMap's margin is ambiguous (`margin`).  In the resampler, a waypoint
whose arc length lies within a relative COUNT_TIE of the total is a count tie: there the counts may differ by one, and only the
waypoints before it are compared (`tie_xy`, `tie_yaw`; one at an interior segment end is the same point whichever segment takes it).
Likewise a smoothing difference within SMOOTH_TIE of +-pi/2 (`tie_smooth`: the smoothed yaws may differ by a turn from there on).
"""
import math

import numpy as np
import torch

import alm_ref as ar
from workloads import scan_times, summed

DELTA_SIGL = 0.01            # alm_traj_opt.h:16-19
GUARD = 4.0e6                # S3
NMAX, MMAX = 64, 128         # the compiled limits
MAX_WAYPOINTS = 4095         # S6
MAX_YAW, MAX_TURNS = 2.0 ** 40, 65536.0
COUNT_TIE = 1e-12
SMOOTH_TIE = 1e-9
CHUNK = 1 << 18              # samples per chunk of the map query
QUANTITIES = ("vx", "ax", "ay", "cur", "att", "sig")


# ------------------------------------------------------------------------------------------------ splines
def duration(N, M, Tx, Ty):
    """the duration the scan uses: the smaller of the two sums (workloads.summed)"""
    a, b = summed(Tx, N), summed(Ty, M)
    return a if a < b else b


def pieces(P, dur, t):
    """(piece index, local time) of times t: the number of boundaries i dur (i = 1 .. P - 1) strictly below t, at most P - 1"""
    t = np.asarray(t, np.float64)
    idx = np.clip(np.ceil(t / dur) - 1.0, 0, P - 1).astype(np.int64)
    return idx, t - idx * dur


def spline(c, P, dur, t, order=2):
    """value and derivatives up to `order` of the P-piece spline c (6 per piece, low power first) at times t: a list of arrays"""
    idx, tl = pieces(P, dur, t)
    cp = np.asarray(c, np.float64)[:6 * P].reshape(P, 6)[idx].T          # (6, S)
    out = []
    for d in range(order + 1):
        out.append(np.polynomial.polynomial.polyval(tl, cp, tensor=False))
        cp = np.polynomial.polynomial.polyder(cp, axis=0)
    return out


def state(N, M, c_xy, c_yaw, Tx, Ty, t):
    """[px, py, vx, vy, ax, ay, yaw, dyaw, ddyaw] at times t, each an array"""
    c_xy = np.asarray(c_xy, np.float64)
    x = spline(c_xy[:6 * N], N, Tx, t)
    y = spline(c_xy[6 * N:], N, Tx, t)
    w = spline(c_yaw, M, Ty, t)
    return [x[0], y[0], x[1], y[1], x[2], y[2], w[0], w[1], w[2]]


# ------------------------------------------------------------------------------------------------ the scan
def _margin(grid, p, yn):
    """samples within FACE (in resolutions) of isInMap's 1e-4 margin: the terrain there is zero or not by rounding"""
    o, mx = grid.origin, grid.maxb
    out = np.zeros(len(yn), bool)
    for k, v in enumerate((p[:, 0], p[:, 1], yn)):
        r = grid.res if k < 2 else grid.yres
        out |= (np.abs(v - (o[k] + 1e-4)) < ar.FACE * r) | (np.abs(v - (mx[k] - 1e-4)) < ar.FACE * r)
    return out


def samples(grid, gravity, N, M, c_xy, c_yaw, Tx, Ty, t):
    """the scanned quantities at times t: dict of arrays vx, ax, ay, cur, att, sig, term, and the flags margin, off_map, border, seam;
    also vx2 and curv, the squares the cost constrains"""
    out = {k: [] for k in QUANTITIES + ("term", "vx2", "curv", "margin", "off_map", "border", "seam")}
    for s in range(0, max(len(t), 1), CHUNK):
        tc = np.asarray(t[s:s + CHUNK], np.float64)
        if tc.size == 0:
            break
        px, py, vxw, vyw, axw, ayw, yaw, dyaw, _ = state(N, M, c_xy, c_yaw, Tx, Ty, tc)
        p = np.stack([px, py], 1)
        mp = ar._cells(grid, p, yaw)
        with torch.no_grad():
            sigma, zbx, zby, yn = ar.terrain(grid, mp, torch.from_numpy(p), torch.from_numpy(yaw))
            icvx, spx, icvy, spy, cxi, icxi = (v.numpy() for v in ar.frame(zbx, zby, yn))       # S1: the frame at the normalised yaw
        sigma = sigma.numpy()
        cy, sy = np.cos(yaw), np.sin(yaw)                                                       # S1: lon / lat at the raw yaw
        lon = axw * cy + ayw * sy
        lat = -axw * sy + ayw * cy
        vx2 = (vxw * vxw + vyw * vyw) * icvx * icvx
        vx = np.sqrt(vxw * vxw + vyw * vyw) * icvx
        cur = dyaw * icxi / np.sqrt(vx2 + DELTA_SIGL)
        vals = dict(vx=vx, ax=lon * icvx + gravity * spx, ay=lat * icvy + gravity * spy, cur=cur, att=-cxi, sig=sigma,
                    term=np.abs(vxw * sy - vyw * cy), vx2=vx2, curv=(dyaw * icxi) ** 2 / (vx2 + DELTA_SIGL),
                    margin=_margin(grid, p, yn.numpy()), off_map=~mp["inside"], border=mp["border"], seam=mp["seam"])
        for k in out:
            out[k].append(vals[k])
    return {k: np.concatenate(v) if v else np.zeros(0) for k, v in out.items()}


def _abs_max(v):
    """S2: the signed value of the largest magnitude, the earliest on a tie; 0 when no value is nonzero"""
    if v.size == 0:
        return 0.0
    i = int(np.argmax(np.abs(v)))
    return float(v[i]) if abs(v[i]) > 0.0 else 0.0


def scan(grid, gravity, N, M, c_xy, c_yaw, Tx, Ty, dt=0.01, t_from=0.0, limits=None, device=False):
    """the check row of one trajectory, restated: dict with
      out16 - the 16 numbers of ualm_check_trajectories (with t_from = 0 and no limits: orc_feasibility's 8, T_xy, T_yaw, six -1);
      t, kept, s - the full sample sequence, its kept mask and the samples (see `samples`; None when not scanned);
      ambiguous - a kept sample lies on isInMap's margin.
    device: also S3's compiled limits on N and M"""
    out = np.zeros(16)
    out[10:] = -1.0
    out[4] = -1.0
    out[8], out[9] = Tx, Ty
    if device and (N > NMAX or M > MMAX):
        out[:] = 0.0
        out[7] = -1.0
        out[10:] = -1.0
        return dict(out16=out, t=None, kept=None, s=None, ambiguous=False)
    total = duration(N, M, Tx, Ty)
    if not (total / dt < GUARD):
        out[4] = 0.0
        out[7] = -1.0
        return dict(out16=out, t=None, kept=None, s=None, ambiguous=False)
    t = scan_times(total, dt)
    return window(dict(out16=out, t=t, s=samples(grid, gravity, N, M, c_xy, c_yaw, Tx, Ty, t)), t_from, limits)


def window(full, t_from=0.0, limits=None):
    """a scanned result (scan's, any window) reduced again over the samples t >= t_from, with `limits`: the samples are not recomputed"""
    out, t, s = full["out16"].copy(), full["t"], full["s"]
    if t is None:
        return full
    out[10:] = -1.0
    kept = t >= t_from
    q = {k: s[k][kept] for k in QUANTITIES}
    out[0], out[1], out[2], out[3] = (_abs_max(q[k]) for k in ("vx", "ax", "ay", "cur"))
    out[4] = max(-1.0, float(q["att"].max())) if kept.any() else -1.0
    out[5] = max(0.0, float(q["sig"].max())) if kept.any() else 0.0
    out[6] = math.fsum(s["term"][kept])
    out[7] = float(kept.sum())
    if limits is not None:
        for j, (v, lim) in enumerate(zip(tested(q), test_limits(limits))):
            hit = np.nonzero(v > lim)[0]
            out[10 + j] = float(t[kept][hit[0]]) if hit.size else -1.0
    return dict(out16=out, t=t, kept=kept, s=s, ambiguous=bool(s["margin"][kept].any()))


def tested(q):
    """the six tested values of samples q, each compared with `> limit`: |vx|, |ax|, |ay|, |cur|, att, sig"""
    return [np.abs(q["vx"]), np.abs(q["ax"]), np.abs(q["ay"]), np.abs(q["cur"]), q["att"], q["sig"]]


def test_limits(limits):
    """the thresholds of the six tests: max_vel, max_acc_lon, max_acc_lat, max_kap, -min_cxi (att > -min_cxi), max_sig"""
    lim = [float(v) for v in limits]
    return [lim[0], lim[1], lim[2], lim[3], -lim[4], lim[5]]


# ------------------------------------------------------------------------------------------------ the resampler
def smooth(yaw):
    """S5 in closed form over a polyline's yaws: (smoothed yaws, turns each point needed in the product's bound (S6), tie index or
    None).  Point k + 1 is moved by n1 turns down when d = yaw[k + 1] - smoothed[k] >= pi/2, n1 = floor((d - pi/2) / 2pi) + 1, then
    by n2 turns up when the result is <= -pi/2, n2 = floor((-pi/2 - d') / 2pi) + 1."""
    y = np.array(yaw, np.float64, copy=True)
    need = np.zeros(len(y))
    tie = None
    two = 2.0 * math.pi
    for k in range(1, len(y)):
        d = y[k] - y[k - 1]
        need[k] = math.floor(abs(d) / two) + 1.0
        n1 = math.floor((d - 0.5 * math.pi) / two) + 1.0 if d >= 0.5 * math.pi else 0.0
        d1 = d - n1 * two
        n2 = math.floor((-0.5 * math.pi - d1) / two) + 1.0 if d1 <= -0.5 * math.pi else 0.0
        r = (d - 0.5 * math.pi) / two
        if tie is None and abs(r - round(r)) * two < SMOOTH_TIE * max(1.0, abs(y[k]), abs(y[k - 1])):
            tie = k
        y[k] = y[k] + (n2 - n1) * two
    return y, need, tie


def _waypoints(cum, pts, col, step, count):
    """`count` waypoints at the arc lengths k step (k = 1 ..): linear interpolation of pts[:, col] inside the segment that holds each"""
    s = step * np.arange(1, count + 1)
    j = np.clip(np.searchsorted(cum, s, side="right") - 1, 0, len(cum) - 2)
    seg = cum[j + 1] - cum[j]
    w = (s - cum[j]) / np.where(seg > 0, seg, 1.0)
    return [pts[j, c] + w * (pts[j + 1, c] - pts[j, c]) for c in col]


def _count(L, step):
    """the number of arc lengths k step (k = 1, 2, ..) strictly below L"""
    n = int(math.ceil(L / step)) - 1 if L > 0 else 0
    while (n + 1) * step < L:
        n += 1
    while n > 0 and n * step >= L:
        n -= 1
    return n


def resample(path, rp=(0.3, 2.0, 0.5, 1.2), bounded=False):
    """PlanManager's resampler over an (n, 3) polyline, restated: dict N, M, total_time, inner_xy (nx, 2), inner_yaw (ny,), smoothed
    (n, 3), cut, and tie_xy / tie_yaw (index of the first waypoint at a count tie, None: none).  bounded: S6's bound"""
    piece_len, yaw_times, mean_vel, init_times = (float(v) for v in rp)
    p = np.array(path, np.float64, copy=True).reshape(-1, 3)
    seg = np.hypot(np.diff(p[:, 0]), np.diff(p[:, 1])) if len(p) > 1 else np.zeros(0)
    cum = np.concatenate([[0.0], np.cumsum(seg)])
    L = float(cum[-1])
    cut = False
    last = len(p)
    if bounded and len(p) > 1:
        big = ~(np.abs(p[:, 2]) < MAX_YAW)
        if big.any():
            last = max(int(np.argmax(big)), 1)
            cut = True
    sm, need, tie_s = smooth(p[:last, 2])
    if bounded and len(need) > 1:
        over = np.nonzero(np.cumsum(need[1:]) > MAX_TURNS)[0]
        if over.size:
            cut = True
            last = min(last, int(over[0]) + 1)
    sm = np.concatenate([sm[:last], p[last:, 2]])
    p[:, 2] = sm
    step_yaw = piece_len / yaw_times
    Lc = float(cum[last - 1]) if cut else L                 # waypoints only before the cut
    nxy, nyaw = _count(Lc, piece_len), _count(Lc, step_yaw)
    if bounded and (nxy > MAX_WAYPOINTS or nyaw > MAX_WAYPOINTS):
        cut = True
    out = dict(total_time=L / mean_vel * init_times, smoothed=p, cut=cut, tie_smooth=tie_s)
    if cut:
        out.update(N=MAX_WAYPOINTS + 2, M=MAX_WAYPOINTS + 2, inner_xy=np.zeros((0, 2)), inner_yaw=np.zeros(0), tie_xy=None, tie_yaw=None)
        return out
    xs, ys = _waypoints(cum, p, (0, 1), piece_len, nxy)
    (hs,) = _waypoints(cum, p, (2,), step_yaw, nyaw)
    out.update(N=nxy + 1, M=nyaw + 1, inner_xy=np.stack([xs, ys], 1), inner_yaw=hs,
               tie_xy=_tie(cum, piece_len, nxy), tie_yaw=_tie(cum, step_yaw, nyaw))
    return out


def _tie(cum, step, n):
    """index of the waypoint at a count tie: n when the last counted (index n - 1) or the next one (index n) lies within a relative
    COUNT_TIE of the total, None otherwise.  A waypoint at an interior segment end is no tie: the reference places it at the end of
    one segment or at the start of the next, the same point, and counts it once either way."""
    L = float(cum[-1])
    near = [k for k in (n, n + 1) if k > 0 and abs(k * step - L) <= COUNT_TIE * max(L, step)]
    return min(near) - 1 if near else None


def replan(N, M, c_xy, c_yaw, Tx, Ty, bnd, t_from, dt=0.01, rp=(0.3, 2.0, 0.5, 1.2)):
    """one replan row, restated: dict head (9: px, py, vx, vy, ax, ay, yaw, dyaw, ddyaw at t_from), polyline (n, 3), bnd' (18), and
    `resample`'s result of the polyline with S6's bound"""
    head = np.array([v[0] for v in state(N, M, c_xy, c_yaw, Tx, Ty, np.array([float(t_from)]))])
    total = duration(N, M, Tx, Ty)
    t = scan_times(total, dt)
    t = t[t > t_from]                                                                        # S4
    mid = np.stack(state(N, M, c_xy, c_yaw, Tx, Ty, t), 1)[:, [0, 1, 6]] if t.size else np.zeros((0, 3))
    bnd = np.asarray(bnd, np.float64)
    poly = np.vstack([head[[0, 1, 6]], mid, [bnd[6], bnd[7], bnd[15]]])
    b2 = np.concatenate([head[:6], bnd[6:12], head[6:9], bnd[15:18]])
    return dict(head=head, polyline=poly, times=t, bnd=b2, **resample(poly, rp, bounded=True))


# ------------------------------------------------------------------------------------------------ comparisons
def compare(got, ref, limits=None, tol=1e-11):
    """a check row `got` (16 numbers; the first 8 or 10 of a scan) against the restated `ref` (scan's result): (worst relative error per
    block, list of what breaks).  Exact: the not-scanned rows, the sample count, T_xy / T_yaw.  Maxima: within tol of the quantity's
    scale (its largest kept magnitude, at least 1e-3), equal signs unless at that level.  Non-holonomic sum: within tol of the summed
    speeds.  First violations (limits given): a time is a kept sample, where the restated value is >= limit - band while every earlier
    kept sample is <= limit + band; -1 needs every kept sample <= limit + band (band = tol max(|limit|, scale))."""
    got = np.asarray(got, np.float64)
    r = ref["out16"]
    n = min(len(got), 16)
    worst, bad = {}, []
    if r[7] < 0 or ref["t"] is None:
        if not np.array_equal(got[:n], r[:n]):
            bad.append(("not scanned", got[:n], r[:n]))
        return worst, bad
    for k, want in ((7, r[7]), (8, r[8]), (9, r[9])):
        if k < n and got[k] != want:
            bad.append(("exact", k, got[k], want))
    kept = ref["kept"]
    q = {k: ref["s"][k][kept] for k in QUANTITIES}
    scale = [max(float(np.abs(q[k]).max()) if q[k].size else 0.0, 1e-3) for k in QUANTITIES]
    for j, k in enumerate(QUANTITIES):
        e = abs(got[j] - r[j]) / scale[j]
        worst[k] = e
        if e > tol or (np.sign(got[j]) != np.sign(r[j]) and max(abs(got[j]), abs(r[j])) > tol * scale[j]):
            bad.append((k, got[j], r[j]))
    speed = math.fsum(np.abs(q["vx"])) + 1e-3
    worst["nonhol"] = abs(got[6] - r[6]) / speed
    if worst["nonhol"] > tol:
        bad.append(("nonhol", got[6], r[6]))
    if limits is None or n < 16:
        return worst, bad
    tk = ref["t"][kept]
    for j, (v, lim) in enumerate(zip(tested(q), test_limits(limits))):
        band = tol * max(abs(lim), scale[j])
        t = got[10 + j]
        if t == -1.0:
            if v.size and v.max() > lim + band:
                bad.append(("no violation", j, lim, float(v.max())))
            continue
        at = np.nonzero(tk == t)[0]
        if at.size != 1:
            bad.append(("not a kept sample", j, t))
            continue
        i = int(at[0])
        if v[i] < lim - band or (i and v[:i].max() > lim + band):
            bad.append(("first violation", j, t, lim, float(v[i]), float(v[:i].max()) if i else None))
    return worst, bad


def worst_of(acc, worst):
    """acc[k] = max(acc[k], worst[k]) over the blocks of `worst`"""
    for k, v in worst.items():
        acc[k] = max(acc.get(k, 0.0), v)
    return acc


def compare_replan(N, M, bnd, total_time, inner_xy, inner_yaw, ref, tol=1e-11, caps=(NMAX, MMAX)):
    """one built replan row (counts, bnd' 18, total_time, inner points as flat arrays; a row over the compiled limits carries none)
    against the restated `ref` (replan's result): (worst error per block, list of what breaks).  Exact: the counts away from a count
    tie, the goal fields of bnd' (copied).  Within tol: the head state relative to its magnitude, total_time relative, the waypoints
    relative to the polyline's extent (before a count or smoothing tie only).  caps: the counts N, M past which a row carries no inner
    points (None: every row carries them)"""
    worst, bad = {}, []
    ixy, iyaw = np.asarray(inner_xy, np.float64).reshape(-1, 2), np.asarray(inner_yaw, np.float64).ravel()
    for k, g, w, tie in (("N", N, ref["N"], ref["tie_xy"]), ("M", M, ref["M"], ref["tie_yaw"])):
        if g != w and not (tie is not None and abs(g - w) == 1):
            bad.append((k, g, w))
    goal = [6, 7, 8, 9, 10, 11, 15, 16, 17]
    if not np.array_equal(np.asarray(bnd)[goal], ref["bnd"][goal]):
        bad.append(("goal fields", np.asarray(bnd)[goal], ref["bnd"][goal]))
    head = [0, 1, 2, 3, 4, 5, 12, 13, 14]
    worst["head"] = float(np.max(np.abs(np.asarray(bnd)[head] - ref["bnd"][head]) / np.maximum(np.abs(ref["bnd"][head]), 1.0)))
    worst["total_time"] = abs(total_time - ref["total_time"]) / max(abs(ref["total_time"]), 1e-300)
    ext = max(1.0, float(np.abs(ref["polyline"][:, :2]).max()))
    yext = max(1.0, float(np.abs(ref["smoothed"][:, 2]).max()))
    fits = caps is None or (N <= caps[0] and M <= caps[1])
    if fits:
        nx, ny = len(ixy), len(iyaw)
        if ref["tie_smooth"] is not None:
            ny = 0                                   # the smoothed yaws may differ by a turn: compare the counts only
        cx = min(nx, len(ref["inner_xy"]), ref["tie_xy"] if ref["tie_xy"] is not None else nx)
        cy = min(ny, len(ref["inner_yaw"]), ref["tie_yaw"] if ref["tie_yaw"] is not None else ny)
        worst["inner_xy"] = float(np.abs(ixy[:cx] - ref["inner_xy"][:cx]).max() / ext) if cx else 0.0
        worst["inner_yaw"] = float(np.abs(iyaw[:cy] - ref["inner_yaw"][:cy]).max() / yext) if cy else 0.0
    elif ixy.any() or iyaw.any():
        bad.append(("over the limits with inner points", N, M))
    for k in ("head", "total_time", "inner_xy", "inner_yaw"):
        if worst.get(k, 0.0) > tol:
            bad.append((k, worst[k]))
    return worst, bad


# ------------------------------------------------------------------------------------------------ the case table
def _minco(pts, T, v0, v1):
    """the minimum-jerk spline through the rows of pts (P + 1, D), P pieces of duration T, boundary velocities v0 / v1 and zero
    accelerations (alm_ref.minco, C4 at the joins): 6 P D coefficients, column-major as the solves return them"""
    import torch
    pts = np.asarray(pts, np.float64)
    P, D = pts.shape[0] - 1, pts.shape[1]
    head = np.stack([pts[0], np.asarray(v0, np.float64).reshape(D), np.zeros(D)], 1)
    tail = np.stack([pts[-1], np.asarray(v1, np.float64).reshape(D), np.zeros(D)], 1)
    c = ar.minco(P, torch.tensor(float(T), dtype=torch.float64), torch.from_numpy(np.ascontiguousarray(pts[1:-1])), head, tail)
    return np.ascontiguousarray(c.numpy().T).ravel()


def _steepest(m):
    """the (x, y, yaw) centre of the cell whose normal is furthest from vertical (smallest cos xi), one cell in from the border"""
    c = np.asarray(m.cells, np.float64)
    cz = np.sqrt(np.clip(1.0 - c[..., 2] ** 2 - c[..., 3] ** 2, 0.0, 1.0))
    cz[:2], cz[-2:], cz[:, :2], cz[:, -2:] = 2.0, 2.0, 2.0, 2.0
    ix, iy, iw = np.unravel_index(int(np.argmin(cz)), cz.shape)
    g = m.geom
    return (g.origin[0] + (ix + 0.5) * g.xy_resolution, g.origin[1] + (iy + 0.5) * g.xy_resolution, g.origin[2] + (iw + 0.5) * g.yaw_resolution)


def _path(kind, m, N, M):
    """waypoints (N + 1, 2), yaws (M + 1), boundary velocity (2) and yaw rate of a trajectory of `kind` placed from grid m's bounds"""
    g = m.geom
    o, b = np.array(list(g.origin[:2])), np.array(list(g.max_boundary[:2]))
    mid = 0.5 * (o + b) + np.array([0.031, -0.047])
    s, u = np.linspace(0.0, 1.0, N + 1), np.linspace(0.0, 1.0, M + 1)
    line = lambda a, z: a[None, :] + s[:, None] * (np.asarray(z) - a)[None, :]
    if kind == "arc":                      # a 1.5 pi arc of radius 1.2, the heading along it
        a = 1.5 * np.pi * s
        return mid + 1.2 * np.stack([np.cos(a), np.sin(a)], 1), 0.5 * np.pi + 1.5 * np.pi * u, np.array([0.0, 0.4]), 0.3
    if kind == "standstill":               # v = 0 everywhere while the yaw turns: vx 0, cur at its sqrt(0.01) floor, no side slip
        return np.repeat(mid[None, :], N + 1, 0), 0.4 + 3.0 * u, np.zeros(2), 0.0
    if kind == "reverse":                  # out along x and back over the same line, heading fixed: the velocity reverses
        return mid + np.stack([0.9 * np.sin(2.0 * np.pi * s), 0.05 * s], 1), np.full(M + 1, 0.2), np.array([0.3, 0.0]), 0.0
    if kind == "spin":                     # raw yaws from -3 pi - 0.4 on, 2.5 rad per yaw piece: high yaw rates, many seam crossings
        return line(mid - 0.6, mid + 0.6), -3.0 * np.pi - 0.4 + 2.5 * M * u, np.array([0.2, 0.2]), 1.0
    if kind == "far_yaw":                  # yaws around 5 pi: the map query wraps them, sin / cos take them raw
        return line(mid - [0.7, 0.2], mid + [0.5, 0.6]), 5.0 * np.pi - 0.3 + 0.8 * u, np.array([0.3, 0.1]), 0.0
    if kind == "off_hi":                   # out through the +x side past the clamped last cells, yaw over the seam
        return line(np.array([b[0] - 0.4, mid[1]]), [b[0] + 0.5, mid[1] + 0.3]), 0.8 * np.pi + 0.5 * np.pi * u, np.array([0.3, 0.0]), 0.0
    if kind == "off_lo":                   # out through the -y side
        return line(np.array([mid[0], o[1] + 0.4]), [mid[0] - 0.2, o[1] - 0.5]), -0.5 * np.pi + 0.2 * u, np.array([0.0, -0.3]), 0.0
    if kind == "steep":                    # through the steepest cell, heading at its yaw layer
        x, y, w = _steepest(m)
        c = np.array([x, y])
        return line(c - [0.4, 0.3], c + [0.4, 0.3]), w + 0.3 * (u - 0.5), np.array([0.2, 0.15]), 0.0
    raise KeyError(kind)


def _nudge(a, b, N, M, sign):
    """(a', b') within 40 ulps of (a, b) whose sums summed(b', M) and summed(a', N) are adjacent doubles, b's above for sign = +1"""
    step = lambda x, k: x + k * np.spacing(x)
    for ka in range(-40, 41):
        ta = summed(step(a, ka), N)
        want = np.nextafter(ta, np.inf if sign > 0 else -np.inf)
        for kb in range(-40, 41):
            if summed(step(b, kb), M) == want:
                return step(a, ka), step(b, kb)
    raise RuntimeError("no durations whose sums are one ulp apart")


# name: (kind, N, M, duration, durations, dts).  durations: None (T / N, T / M), "xy_min" / "yaw_min" (the sums one ulp apart, the
# smaller on that side), "yaw_first" / "xy_first" (that spline ends at 0.8 of the other's duration, as a caller's trajectory may),
# "on_sample" (T_xy is sample 25 of t = 0, 0.01, ..: a piece boundary on a sample), "exact" (binary durations,
# dt 0.125: every boundary i T on a sample).  dts: the sequences scanned ("long": one longer than the trajectory, one sample)
SCAN_CASES = {
    "N1_M1": ("arc", 1, 1, 2.0, None, (0.01, "long")),
    "N64_M128": ("arc", 64, 128, 16.0, None, (0.01, 0.0137)),
    "N64_M1": ("far_yaw", 64, 1, 6.0, None, (0.0137,)),
    "N1_M128": ("spin", 1, 128, 9.0, None, (0.01,)),
    "xy_min": ("arc", 7, 13, 3.3, "xy_min", (0.01,)),
    "yaw_min": ("reverse", 13, 7, 3.3, "yaw_min", (0.01,)),
    "yaw_first": ("arc", 10, 24, 3.0, "yaw_first", (0.01,)),
    "xy_first": ("spin", 12, 20, 3.0, "xy_first", (0.0137,)),
    "short_pieces": ("reverse", 40, 80, 0.16, None, (0.01, 0.0137)),
    "on_sample": ("arc", 8, 16, None, "on_sample", (0.01,)),
    "exact": ("spin", 8, 16, 4.0, "exact", (0.125, 0.01)),
    "standstill": ("standstill", 5, 9, 3.0, None, (0.01,)),
    "spin": ("spin", 10, 30, 3.0, None, (0.01, 0.0137)),
    "off_hi": ("off_hi", 10, 20, 4.0, None, (0.01,)),
    "off_lo": ("off_lo", 9, 17, 4.0, None, (0.0137,)),
    "steep": ("steep", 10, 20, 3.0, None, (0.01,)),
}


def scan_case(name, m):
    """trajectory `name` of SCAN_CASES placed on grid m: dict N, M, c_xy, c_yaw, Tx, Ty, bnd (its goal: the end point and end yaw), dts"""
    kind, N, M, T, durs, dts = SCAN_CASES[name]
    if durs == "on_sample":
        Tx = scan_times(1.0, 0.01)[25]
        Ty, T = 0.5 * Tx, N * Tx
    else:
        Tx, Ty = T / N, T / M
    if durs == "yaw_first":
        Ty = 0.8 * T / M
    elif durs == "xy_first":
        Tx = 0.8 * T / N
    if durs in ("xy_min", "yaw_min"):
        Tx, Ty = _nudge(Tx, Ty, N, M, +1 if durs == "xy_min" else -1)
    elif durs == "exact":
        Tx, Ty = 0.5, 0.25
    pts, yaw, v, w = _path(kind, m, N, M)
    c_xy = _minco(pts, Tx, v, v)
    c_yaw = _minco(yaw.reshape(-1, 1), Ty, [w], [w])
    bnd = np.zeros(18)
    bnd[6:8], bnd[8:10], bnd[15], bnd[16] = pts[-1], v, yaw[-1], w
    total = min(summed(Tx, N), summed(Ty, M))
    return dict(N=N, M=M, c_xy=c_xy, c_yaw=c_yaw, Tx=float(Tx), Ty=float(Ty), bnd=bnd, dts=[2.0 * total if d == "long" else d for d in dts])


def scan_t_froms(total, dt):
    """the window starts of a check: 0, an exact sample time, one ulp below it (0 when that time is 0), mid-piece, a few samples before the end, the end and past
    it (those two keep no sample)"""
    t = scan_times(total, dt)
    k = t[len(t) // 3]
    return [0.0, float(k), float(np.nextafter(k, -np.inf)) if k > 0.0 else 0.0, 0.37 * total + 0.0031, float(t[max(len(t) - 3, 0)]), total, total + 1.0]


def scan_limits(ref, kind):
    """six limits from the restated kept samples of one check (scan_ref.scan): "none" above every value, "median" the median of each
    tested value (fires in the middle), "first" just below the first kept value (fires there), "last" just below the last kept value
    when that is the largest (fires at the last kept sample), else the median"""
    q = {k: ref["s"][k][ref["kept"]] for k in QUANTITIES}
    out = []
    for j, v in enumerate(tested(q)):
        if v.size == 0 or kind == "none":
            lim = float(np.max(v)) + 1.0 if v.size else 1e9
        elif kind == "first":
            lim = float(v[0]) - 1e-6 * max(abs(float(v[0])), 1e-3)
        elif kind == "last" and v[-1] >= v.max():
            lim = float(v[-1]) - 1e-6 * max(abs(float(v[-1])), 1e-3)
        else:
            lim = float(np.median(v))
        out.append(-lim if j == 4 else lim)              # att > -min_cxi
    return tuple(out)
