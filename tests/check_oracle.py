"""ctypes wrapper of tests/check_oracle.cpp: the oracle's post-solve scan (orc_feasibility) from a time t_from on, with the first time each
of six limits is broken (include/ualm.h, ualm_check_trajectories).

TEST INFRASTRUCTURE.  The library is compiled on first use, with the oracle's own flags (oracle/Makefile), into the system temporary
directory: the tree is not written.
"""
import ctypes as C

import numpy as np

import pyoracle as po
from harness import load_oracle_ext

LIMIT_NAMES = ("max_vel", "max_acc_lon", "max_acc_lat", "max_kap", "min_cxi", "max_sig")
NO_LIMITS = (np.inf, np.inf, np.inf, np.inf, -np.inf, np.inf)      # no test fires

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = load_oracle_ext("check_oracle.cpp", "check_oracle")
        L.orc_check.argtypes = [C.POINTER(po.OMap), C.c_double, C.c_int, C.c_int, po.dp, po.dp, C.c_double, C.c_double, C.c_double, C.c_double,
                                po.dp, po.dp, po.dp]
        L.orc_check.restype = None
        _lib = L
    return _lib


def limits_of(params):
    """the six limits of a parameter set (Params or OParams)"""
    return tuple(float(getattr(params, n)) for n in LIMIT_NAMES)


def check(omap, gravity, N, M, c_xy, c_yaw, T_xy, T_yaw, dt=0.01, t_from=0.0, limits=NO_LIMITS, trace=False):
    """out16 of one trajectory (see check_oracle.cpp); with trace=True also the [samples, 9] trace of the full sequence"""
    c_xy = np.ascontiguousarray(c_xy, np.float64); c_yaw = np.ascontiguousarray(c_yaw, np.float64)
    lim = np.ascontiguousarray(limits, np.float64)
    out = np.zeros(16)
    args = (C.byref(omap.c), float(gravity), int(N), int(M), po.P(c_xy), po.P(c_yaw), float(T_xy), float(T_yaw), float(dt))
    if not trace:
        lib().orc_check(*args, float(t_from), po.P(lim), po.P(out), None)
        return out
    full = np.zeros(16)
    lib().orc_check(*args, 0.0, po.P(lim), po.P(full), None)
    tr = np.zeros((max(int(full[7]), 0), 9))
    lib().orc_check(*args, float(t_from), po.P(lim), po.P(out), po.P(tr))
    return out, tr
