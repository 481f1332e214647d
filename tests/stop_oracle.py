"""ctypes wrapper of tests/stop_oracle.cpp: the oracle's solve stopped by the evaluation budget of include/ualm.h (UALM_RET_STOPPED,
orc_solve_budget), the solve of a problem cancelled so that its s-th stop test is the first to see the cancel (orc_solve_cancel), and
the log of the stop tests of the solve without a stop (orc_stop_tests).

TEST INFRASTRUCTURE.  The library is compiled on first use, with the oracle's own flags (oracle/Makefile), into the system temporary
directory: the tree is not written.  Load it (lib()) before solving from several threads.
"""
import ctypes as C
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np

import pyoracle as po
from harness import RECORD, load_oracle_ext

STOPPED = 3

_lib = None
_lock = threading.Lock()


def lib():
    global _lib
    with _lock:
        if _lib is None:
            _lib = _load()
    return _lib


def _load():
    L = load_oracle_ext("stop_oracle.cpp", "stop_oracle")
    solve_args = [C.POINTER(po.OParams), C.POINTER(po.OMap), C.POINTER(po.OProblem), C.c_int, C.POINTER(po.OResult), po.dp, po.dp, po.dp]
    L.orc_solve_budget.argtypes = solve_args
    L.orc_solve_cancel.argtypes = solve_args
    L.orc_stop_tests.argtypes = [C.POINTER(po.OParams), C.POINTER(po.OMap), C.POINTER(po.OProblem), C.c_int, C.POINTER(C.c_int),
                                 C.POINTER(C.c_int)]
    L.orc_stop_tests.restype = C.c_int
    return L


def _solve(fn, params, omap, pb, i, arg):
    keep = []
    pr = po._problem(pb, i, keep)
    N, M = int(pb.N[i]), int(pb.M[i])
    res = po.OResult()
    cxy = np.zeros(12 * N); cyaw = np.zeros(6 * M); x = np.zeros(1 + 2 * (N - 1) + (M - 1))
    fn(C.byref(params), C.byref(omap.c), C.byref(pr), int(arg), C.byref(res), po.P(cxy), po.P(cyaw), po.P(x))
    return res, cxy, cyaw, x


def budget_one(params, omap, pb, i, max_evals):
    """(OResult, c_xy, c_yaw, x) of problem i under the budget (0 = none: the oracle's orc_solve)"""
    return _solve(lib().orc_solve_budget, params, omap, pb, i, max_evals)


def budget_batch(params, omap, pb, max_evals, threads=1):
    lib()
    idx = range(pb.B)
    if threads <= 1:
        return [budget_one(params, omap, pb, i, max_evals) for i in idx]
    with ThreadPoolExecutor(threads) as ex:
        return list(ex.map(lambda i: budget_one(params, omap, pb, i, max_evals), idx))


def cancel_one(params, omap, pb, i, s):
    """(OResult, c_xy, c_yaw, x) of problem i with a stop predicate that holds from its s-th stop test on (1-based)"""
    return _solve(lib().orc_solve_cancel, params, omap, pb, i, s)


def stop_tests(params, omap, pb, i):
    """(n_evals, site) arrays of the stop tests of problem i's solve without a stop, in execution order (site 0: the earlyExit
    point, 1: after judgeConvergence)"""
    keep = []
    pr = po._problem(pb, i, keep)
    cap = 4096
    while True:
        ne = np.zeros(cap, np.int32); site = np.zeros(cap, np.int32)
        ip = C.POINTER(C.c_int)
        n = lib().orc_stop_tests(C.byref(params), C.byref(omap.c), C.byref(pr), cap, ne.ctypes.data_as(ip), site.ctypes.data_as(ip))
        if n <= cap:
            return ne[:n].copy(), site[:n].copy()
        cap = n


def same_record(g, o):
    """a GPU record (ualm Result) equal to an oracle record (OResult) in every field the two share"""
    return all(getattr(g, f) == getattr(o, f) for f in RECORD)


def match_stopped(params, omap, pb, i, rec, cxy, cyaw):
    """the s for which the stop-from-test-s solve of problem i equals the GPU record `rec` and its coefficients bit for bit, or None.
    Candidates are the stop tests whose n_evals is the record's (at most two: the last test of an inner solve and the test after
    judgeConvergence can share a count)"""
    ne, _ = stop_tests(params, omap, pb, i)
    for s in np.flatnonzero(ne == rec.n_evals) + 1:
        o = cancel_one(params, omap, pb, i, int(s))
        if same_record(rec, o[0]) and np.array_equal(cxy, o[1]) and np.array_equal(cyaw, o[2]):
            return int(s)
    return None
