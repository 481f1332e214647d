"""ctypes wrapper of tests/replan_oracle.cpp: the CPU reference of ualm_submit_replan's build (include/ualm.h) -- the state at t_from and
the polyline of the trajectory by the oracle's own evaluation, then PlanManager's resampler restated on its own.

TEST INFRASTRUCTURE.  The library is compiled on first use, with the oracle's own flags (oracle/Makefile), into the system temporary
directory: the tree is not written.
"""
import ctypes as C

import numpy as np

from harness import load_oracle_ext

CAP_XY, CAP_YAW = 63, 127                 # the compiled limits N 64, M 128: inner points per row
STRIDE = 21 + 2 * CAP_XY + CAP_YAW        # bnd' 18 | total_time | N' | M' | inner xy | inner yaw
DEFAULT_RP = (0.3, 2.0, 0.5, 1.2)         # run_*.yaml manager/*: piece_len, yaw_piece_times, mean_vel, init_time_times

dp = C.POINTER(C.c_double)
_lib = None


def _P(a):
    return None if a is None else a.ctypes.data_as(dp)


def lib():
    global _lib
    if _lib is None:
        L = load_oracle_ext("replan_oracle.cpp", "replan_oracle")
        ll = C.POINTER(C.c_longlong)
        L.orc_resample.argtypes = [dp, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, dp, C.c_longlong, dp, C.c_longlong, ll, ll, dp, dp,
                                   C.c_int, C.POINTER(C.c_int)]
        L.orc_resample.restype = None
        L.orc_replan_polyline.argtypes = [C.c_int, C.c_int, dp, dp, C.c_double, C.c_double, dp, C.c_double, C.c_double, dp, dp, C.c_longlong, dp]
        L.orc_replan_polyline.restype = C.c_longlong
        L.orc_replan.argtypes = [C.c_int, C.c_int, dp, dp, C.c_double, C.c_double, dp, C.c_double, C.c_double, dp, C.c_int, C.c_int, dp]
        L.orc_replan.restype = None
        _lib = L
    return _lib


def resample(path, rp=DEFAULT_RP, cap_xy=4096, cap_yaw=8192, bounded=False):
    """the restated resampler over an (n, 3) polyline: (N, M, total_time, inner_xy, inner_yaw, smoothed polyline); bounded: with the
    replan build's bound (a cut polyline reports N = M = 4097)"""
    path = np.ascontiguousarray(path, np.float64).reshape(-1, 3)
    ixy, iyaw, sm = np.zeros(2 * cap_xy), np.zeros(cap_yaw), np.zeros(path.shape)
    N, M, T = C.c_longlong(), C.c_longlong(), C.c_double()
    lib().orc_resample(_P(path), path.shape[0], *[float(v) for v in rp], _P(ixy), cap_xy, _P(iyaw), cap_yaw, C.byref(N), C.byref(M), C.byref(T), _P(sm),
                       1 if bounded else 0, None)
    nx, ny = min(N.value - 1, cap_xy), min(M.value - 1, cap_yaw)
    return N.value, M.value, T.value, ixy[:2 * nx].copy(), iyaw[:ny].copy(), sm


def polyline(N, M, c_xy, c_yaw, T_xy, T_yaw, bnd, t_from, dt=0.01):
    """(points [n, 3], times [n] with -1 for the goal, head state [9]) of the build's polyline"""
    c_xy, c_yaw, bnd = (np.ascontiguousarray(a, np.float64) for a in (c_xy, c_yaw, bnd))
    args = (int(N), int(M), _P(c_xy), _P(c_yaw), float(T_xy), float(T_yaw), _P(bnd), float(t_from), float(dt))
    n = lib().orc_replan_polyline(*args, None, None, 0, None)
    pts, ts, head = np.zeros((n, 3)), np.zeros(n), np.zeros(9)
    lib().orc_replan_polyline(*args, _P(pts), _P(ts), n, _P(head))
    return pts, ts, head


def replan(N, M, c_xy, c_yaw, T_xy, T_yaw, bnd, t_from, dt=0.01, rp=DEFAULT_RP):
    """one built row in the kernel's layout (STRIDE doubles)"""
    c_xy, c_yaw, bnd = (np.ascontiguousarray(a, np.float64) for a in (c_xy, c_yaw, bnd))
    rp4 = np.ascontiguousarray([float(v) for v in rp[:4]], np.float64)
    out = np.zeros(STRIDE)
    lib().orc_replan(int(N), int(M), _P(c_xy), _P(c_yaw), float(T_xy), float(T_yaw), _P(bnd), float(t_from), float(dt), _P(rp4), CAP_XY, CAP_YAW,
                     _P(out))
    return out


def rows(pb, out, idx, t_from, dt=0.01, rp=DEFAULT_RP):
    """the built rows of problems idx of batch pb as wait() returned it: [len(idx), STRIDE]"""
    res, cxy, cyaw = out
    _, _, ocx, ocy = pb.offsets()
    tf = np.broadcast_to(np.asarray(t_from, np.float64), (len(idx),))
    return np.array([replan(pb.N[i], pb.M[i], cxy[ocx[i]:ocx[i + 1]], cyaw[ocy[i]:ocy[i + 1]], res[i].piece_T_xy, res[i].piece_T_yaw, pb.bnd[i],
                            tf[k], dt, rp) for k, i in enumerate(idx)]).reshape(len(idx), STRIDE)


def problems_of(built, env=None):
    """ProblemBatch of built rows, packed as api.submit_replan packs them"""
    from uneven_planner_b200 import problems
    N = built[:, 19].astype(np.int32)
    M = built[:, 20].astype(np.int32)
    fits = [(n - 1) <= CAP_XY and (m - 1) <= CAP_YAW for n, m in zip(N, M)]
    xy = [built[b, 21:21 + 2 * (N[b] - 1)] if fits[b] else np.zeros(2 * (int(N[b]) - 1)) for b in range(len(N))]
    yw = [built[b, 21 + 2 * CAP_XY:21 + 2 * CAP_XY + M[b] - 1] if fits[b] else np.zeros(int(M[b]) - 1) for b in range(len(N))]
    return problems.ProblemBatch(N, M, built[:, :18].copy(), built[:, 18].copy(), np.concatenate(xy) if len(N) else np.zeros(0),
                                 np.concatenate(yw) if len(N) else np.zeros(0), env=None if env is None else np.asarray(env, np.int32).copy())
