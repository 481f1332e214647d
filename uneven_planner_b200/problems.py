"""Seeded batches of optimizeSE2Traj problems (BASELINE.json configs 1-5; SURVEY 8d).

(start, goal) pairs are drawn with a counter-based SplitMix64 stream so C++/Python agree; the initial
polyline is a forward Dubins curve (libualm ualm_dubins_path, standing in for KinoAstar::plan) and the
optimizer inputs are produced by the reference's own input contract, PlanManager's resampler
(plan_manager/src/plan_manager.cpp:62-122 -> ualm_resample_path).
Rejection rules follow KinoAstar::plan's entry checks (front_end/src/kino_astar.cpp:86-95) and its
XY-occupancy collision test (kino_astar.cpp:175-185).
"""
import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _lib

MASK = (1 << 64) - 1
N_MAX, M_MAX = 64, 128   # compiled limits of the CUDA path


def splitmix64(state):
    state = (state + 0x9E3779B97F4A7C15) & MASK
    z = state
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK
    return state, z ^ (z >> 31)


class Rng:
    def __init__(self, seed):
        self.s = seed & MASK

    def uniform(self, lo, hi):
        self.s, z = splitmix64(self.s)
        return lo + (hi - lo) * ((z >> 11) * (1.0 / (1 << 53)))


@dataclass
class ProblemBatch:
    N: np.ndarray            # int32 [B]
    M: np.ndarray            # int32 [B]
    bnd: np.ndarray          # float64 [B,18]
    total_time: np.ndarray   # float64 [B]
    inner_xy: np.ndarray     # float64 packed sum 2(N-1)
    inner_yaw: np.ndarray    # float64 packed sum (M-1)
    starts: np.ndarray = None
    goals: np.ndarray = None
    env: np.ndarray = None   # int32 [B]: environment of every problem (include/ualm.h, ualm_select_env); None = all environment 0
    # float64 [B, 8]: every problem's vehicle limits and cost weights (ualm_problem_params_t, rows of _lib.problem_params); None = each
    # problem uses its environment's
    params: np.ndarray = None

    @property
    def B(self):
        return len(self.N)

    def offsets(self):
        oxy = np.concatenate([[0], np.cumsum(2 * (self.N.astype(np.int64) - 1))])
        oyaw = np.concatenate([[0], np.cumsum(self.M.astype(np.int64) - 1)])
        ocx = np.concatenate([[0], np.cumsum(12 * self.N.astype(np.int64))])
        ocy = np.concatenate([[0], np.cumsum(6 * self.M.astype(np.int64))])
        return oxy, oyaw, ocx, ocy

    def nvar(self):
        return 1 + 2 * (self.N.astype(np.int64) - 1) + (self.M.astype(np.int64) - 1)

    def nsamples(self, int_K):
        return self.N.astype(np.int64) * (int_K + 1)

    def select(self, idx):
        idx = np.asarray(idx, dtype=np.int64)
        oxy, oyaw, _, _ = self.offsets()
        return ProblemBatch(self.N[idx].copy(), self.M[idx].copy(), self.bnd[idx].copy(), self.total_time[idx].copy(),
                            np.concatenate([self.inner_xy[oxy[i]:oxy[i + 1]] for i in idx]) if len(idx) else np.zeros(0),
                            np.concatenate([self.inner_yaw[oyaw[i]:oyaw[i + 1]] for i in idx]) if len(idx) else np.zeros(0),
                            None if self.starts is None else self.starts[idx].copy(),
                            None if self.goals is None else self.goals[idx].copy(),
                            None if self.env is None else self.env[idx].copy(),
                            None if self.params is None else self.params[idx].copy())

    def x0(self, i):
        """Initial decision vector [tau | Pxy | Pyaw] of problem i (alm_traj_opt.cpp:205-216)."""
        oxy, oyaw, _, _ = self.offsets()
        T = self.total_time[i]
        tau = (np.sqrt(2.0 * T - 1.0) - 1.0) if T > 1.0 else (1.0 - np.sqrt(2.0 / T - 1.0))
        return np.concatenate([[tau], self.inner_xy[oxy[i]:oxy[i + 1]], self.inner_yaw[oyaw[i]:oyaw[i + 1]]])


def concat(batches, envs):
    """One batch of the problems of `batches` back to back, batch k's in environment envs[k] (a mixed batch; select() reorders it).
    Parameter rows are carried when every batch has them."""
    if len(batches) != len(envs):
        raise ValueError("one environment per batch")
    if len({b.params is None for b in batches}) > 1:
        raise ValueError("concat: either every batch or none carries parameter rows")
    cat = lambda f, empty: np.concatenate([getattr(b, f) for b in batches]) if batches else empty
    have = lambda f: all(getattr(b, f) is not None for b in batches)
    return ProblemBatch(cat("N", np.zeros(0, np.int32)).astype(np.int32), cat("M", np.zeros(0, np.int32)).astype(np.int32),
                        cat("bnd", np.zeros((0, 18))), cat("total_time", np.zeros(0)), cat("inner_xy", np.zeros(0)), cat("inner_yaw", np.zeros(0)),
                        cat("starts", None) if batches and have("starts") else None, cat("goals", None) if batches and have("goals") else None,
                        np.concatenate([np.full(b.B, int(e), np.int32) for b, e in zip(batches, envs)]) if batches else np.zeros(0, np.int32),
                        np.concatenate([np.asarray(b.params, np.float64).reshape(-1, 8) for b in batches]) if batches and have("params") else None)


def dubins(start, goal, radius=0.6, ds=0.06, max_pts=4096):
    buf = np.zeros((max_pts, 3))
    s = np.ascontiguousarray(start, dtype=np.float64)
    g = np.ascontiguousarray(goal, dtype=np.float64)
    dp = C.POINTER(C.c_double)
    n = _lib.lib().ualm_dubins_path(s.ctypes.data_as(dp), g.ctypes.data_as(dp), radius, ds, buf.ctypes.data_as(dp), max_pts)
    if n < 0:
        raise RuntimeError(f"ualm_dubins_path: {n}")
    return buf[:n].copy()


def resample(path, piece_len=0.3, yaw_piece_times=2.0, mean_vel=0.5, init_time_times=1.2, init_sig_vel=0.05):
    """manager/* defaults from run_hill.yaml:57-62."""
    path = np.ascontiguousarray(path, dtype=np.float64)
    bnd = np.zeros(18)
    ixy = np.zeros(2 * 512)
    iyaw = np.zeros(1024)
    N, M, T = C.c_int32(), C.c_int32(), C.c_double()
    dp = C.POINTER(C.c_double)
    rc = _lib.lib().ualm_resample_path(path.ctypes.data_as(dp), path.shape[0], piece_len, yaw_piece_times, mean_vel,
                                       init_time_times, init_sig_vel, bnd.ctypes.data_as(dp), ixy.ctypes.data_as(dp), 512,
                                       iyaw.ctypes.data_as(dp), 1024, C.byref(N), C.byref(M), C.byref(T))
    if rc != 0:
        raise RuntimeError(f"ualm_resample_path: {rc}")
    return N.value, M.value, bnd, T.value, ixy[:2 * (N.value - 1)].copy(), iyaw[:M.value - 1].copy()


def from_paths(paths, **kw):
    Ns, Ms, bnds, Ts, xys, yaws = [], [], [], [], [], []
    for p in paths:
        N, M, bnd, T, ixy, iyaw = resample(p, **kw)
        Ns.append(N); Ms.append(M); bnds.append(bnd); Ts.append(T); xys.append(ixy); yaws.append(iyaw)
    return ProblemBatch(np.array(Ns, np.int32), np.array(Ms, np.int32), np.array(bnds).reshape(-1, 18), np.array(Ts),
                        np.concatenate(xys) if xys else np.zeros(0), np.concatenate(yaws) if yaws else np.zeros(0))


def _per_axis(v):
    """(x, y) of a range bound given as one number or as a pair"""
    x, y = np.broadcast_to(np.asarray(v, np.float64), (2,))
    return float(x), float(y)


def generate(mapdata, B, seed=0, max_rho=0.05, min_cnormal=0.8, lo=-4.5, hi=4.5, min_dist=1.5, radius=0.6, ds=0.06,
             n_max=56, max_tries=200000):
    """B random SE(2) start/goal problems on `mapdata` (config 2/3 recipe, SURVEY 8d).  lo / hi: the range the positions are drawn
    from, one number for both axes or an (x, y) pair for a map that is not square."""
    g = mapdata.geom
    (lox, loy), (hix, hiy) = _per_axis(lo), _per_axis(hi)
    occ3, occ2 = mapdata.occupancy(min_cnormal, max_rho)
    X, Y, W = mapdata.shape
    rng = Rng(seed)

    def idx3(p):
        return (int(np.floor((p[0] - g.origin[0]) / g.xy_resolution)), int(np.floor((p[1] - g.origin[1]) / g.xy_resolution)),
                int(np.floor((p[2] - g.origin[2]) / g.yaw_resolution)))

    paths, starts, goals = [], [], []
    tries = 0
    while len(paths) < B:
        tries += 1
        if tries > max_tries:
            raise RuntimeError("problem generator: too many rejections")
        s = np.array([rng.uniform(lox, hix), rng.uniform(loy, hiy), rng.uniform(-np.pi, np.pi)])
        e = np.array([rng.uniform(lox, hix), rng.uniform(loy, hiy), rng.uniform(-np.pi, np.pi)])
        if np.hypot(*(s[:2] - e[:2])) < min_dist:
            continue
        i = idx3(s)
        if not (0 <= i[0] < X and 0 <= i[1] < Y and 0 <= i[2] < W) or occ3[i]:
            continue
        j = idx3(e)
        if occ2[j[0], j[1]]:
            continue
        path = dubins(s, e, radius, ds)
        ix = np.floor((path[:, 0] - g.origin[0]) / g.xy_resolution).astype(int)
        iy = np.floor((path[:, 1] - g.origin[1]) / g.xy_resolution).astype(int)
        if ix.min() < 2 or iy.min() < 2 or ix.max() > X - 3 or iy.max() > Y - 3:
            continue
        if occ2[ix, iy].any():
            continue
        seg = np.hypot(np.diff(path[:, 0]), np.diff(path[:, 1])).sum()
        if int(seg / 0.3) + 1 > n_max:
            continue
        paths.append(path); starts.append(s); goals.append(e)
    pb = from_paths(paths)
    pb.starts = np.array(starts); pb.goals = np.array(goals)
    return pb


def generate_astar(mapdata, B, seed=0, max_rho=0.05, min_cnormal=0.8, lo=-4.5, hi=4.5, min_dist=1.5, nthreads=0):
    """B random SE(2) start/goal problems whose initial paths come from the reference's own front-end (KinoAstar::plan restated in
    libualm, ualm_front_end_batch) instead of one Dubins curve: same random stream and entry checks as generate(); pairs without a path or
    over the optimizer's limits are skipped.  Deterministic in (map, B, seed), independent of the thread count."""
    from . import front_end
    g = mapdata.geom
    (lox, loy), (hix, hiy) = _per_axis(lo), _per_axis(hi)
    view = front_end.MapView(mapdata, min_cnormal, max_rho)
    rng = Rng(seed)
    parts, starts, goals = [], [], []
    have = 0
    while have < B:
        cs, cg = [], []
        while len(cs) < max(2 * (B - have), 64):
            s = np.array([rng.uniform(lox, hix), rng.uniform(loy, hiy), rng.uniform(-np.pi, np.pi)])
            e = np.array([rng.uniform(lox, hix), rng.uniform(loy, hiy), rng.uniform(-np.pi, np.pi)])
            if np.hypot(*(s[:2] - e[:2])) < min_dist:
                continue
            cs.append(s); cg.append(e)
        pb, packed, _ = front_end.plan_batch(view, np.array(cs), np.array(cg), nthreads=nthreads)
        take = min(pb.B, B - have)
        if take > 0:
            oxy, oyaw, _, _ = pb.offsets()
            parts.append(ProblemBatch(pb.N[:take].copy(), pb.M[:take].copy(), pb.bnd[:take].copy(), pb.total_time[:take].copy(), pb.inner_xy[:oxy[take]].copy(),
                                      pb.inner_yaw[:oyaw[take]].copy()))
            starts.append(pb.starts[:take]); goals.append(pb.goals[:take])
            have += take
    out = ProblemBatch(np.concatenate([p.N for p in parts]), np.concatenate([p.M for p in parts]), np.concatenate([p.bnd for p in parts]),
                       np.concatenate([p.total_time for p in parts]), np.concatenate([p.inner_xy for p in parts]), np.concatenate([p.inner_yaw for p in parts]))
    out.starts = np.concatenate(starts); out.goals = np.concatenate(goals)
    return out
