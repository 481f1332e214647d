"""ualm_poll_batch without a device: the symbol is exported, a null context is refused, and the Python wrapper checks its arguments
before it calls the library."""
import ctypes as C

import numpy as np
import pytest


def test_poll_symbol_is_exported_and_refuses_a_null_context(built):
    from uneven_planner_b200 import _lib
    L = _lib.lib()
    assert hasattr(L, "ualm_poll_batch")
    idx = np.zeros(4, np.int32)
    n_new, n_pending = C.c_int(-7), C.c_int(-7)
    rc = L.ualm_poll_batch(None, 0, 0.0, idx.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(n_new), C.byref(n_pending), None, None, None)
    assert rc == _lib.UALM_EINVAL
    assert (n_new.value, n_pending.value) == (-7, -7)
    assert b"ticket" in L.ualm_last_error()


def test_python_poll_checks_its_arguments(built, bumps_map):
    from uneven_planner_b200 import _lib, api, problems
    pb = problems.generate(bumps_map, 3, seed=2)
    # a context object without a device: the checks below come before any library call (the handle is null)
    opt = api.BatchALMTrajOpt.__new__(api.BatchALMTrajOpt)
    opt.L, opt.h = _lib.lib(), C.c_void_p()
    opt._tickets = {0: (pb, None)}
    out = opt.outputs(pb)
    assert len(out[0]) == 3 and out[1].size == 12 * int(pb.N.sum()) and out[2].size == 6 * int(pb.M.sum())
    with pytest.raises(ValueError, match="not a ticket"):
        opt.poll(1, out)
    with pytest.raises(ValueError, match="wait_ms"):
        opt.poll(0, out, wait_ms=-1.0)
    with pytest.raises(ValueError, match="wait_ms"):
        opt.poll(0, out, wait_ms=float("nan"))
    with pytest.raises(ValueError, match="Result records"):
        opt.poll(0, ((_lib.Result * 2)(), out[1], out[2]))
    with pytest.raises(ValueError, match="c_xy"):
        opt.poll(0, (out[0], np.zeros(5), out[2]))
    with pytest.raises(ValueError, match="c_yaw"):
        opt.poll(0, (out[0], out[1], out[2].astype(np.float32)))
    # well-formed arguments reach the library, which refuses the null context
    with pytest.raises(api.UalmError, match="error %d" % _lib.UALM_EINVAL):
        opt.poll(0, out)
    with pytest.raises(api.UalmError, match="error %d" % _lib.UALM_EINVAL):
        opt.poll(0, (out[0], None, None), wait_ms=2.0)
