"""ctypes wrapper of tests/budget_oracle.cpp: the oracle's solve with the evaluation budget of include/ualm.h (UALM_RET_STOPPED).

TEST INFRASTRUCTURE.  The library is compiled on first use, with the oracle's own flags (oracle/Makefile), into the system temporary
directory: the tree is not written.
"""
import ctypes as C
from concurrent.futures import ThreadPoolExecutor

import numpy as np

import pyoracle as po
from harness import load_oracle_ext

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = load_oracle_ext("budget_oracle.cpp", "budget_oracle")
        L.orc_solve_budget.argtypes = [C.POINTER(po.OParams), C.POINTER(po.OMap), C.POINTER(po.OProblem), C.c_int, C.POINTER(po.OResult),
                                       po.dp, po.dp, po.dp]
        _lib = L
    return _lib


def solve_one(params, omap, pb, i, max_evals):
    """(OResult, c_xy, c_yaw, x) of problem i under the budget (0 = none: the oracle's orc_solve)"""
    keep = []
    pr = po._problem(pb, i, keep)
    N, M = int(pb.N[i]), int(pb.M[i])
    res = po.OResult()
    cxy = np.zeros(12 * N); cyaw = np.zeros(6 * M); x = np.zeros(1 + 2 * (N - 1) + (M - 1))
    lib().orc_solve_budget(C.byref(params), C.byref(omap.c), C.byref(pr), int(max_evals), C.byref(res), po.P(cxy), po.P(cyaw), po.P(x))
    return res, cxy, cyaw, x


def solve_batch(params, omap, pb, max_evals, threads=1):
    lib()
    idx = range(pb.B)
    if threads <= 1:
        return [solve_one(params, omap, pb, i, max_evals) for i in idx]
    with ThreadPoolExecutor(threads) as ex:
        return list(ex.map(lambda i: solve_one(params, omap, pb, i, max_evals), idx))
