"""Python face of the C ABI (include/ualm.h) used by tests and bench.py.

`BatchALMTrajOpt` mirrors the reference's ALMTrajOpt wiring for a batch of problems:
    init(params)            <- ALMTrajOpt::init(nh)                 (alm_traj_opt.cpp:5-45)
    set_environment(map)    <- ALMTrajOpt::setEnvironment(map)      (alm_traj_opt.h:127-130)
    optimize(problems)      <- B x ALMTrajOpt::optimizeSE2Traj(...) (alm_traj_opt.h:92-98), then getTraj()
A context holds up to UALM_MAX_ENVS environments (parameter set + map grid): init(params, env=k) / set_environment(map, env=k)
bind environment k, and a batch whose `env` array is set solves every problem in its own environment (ProblemBatch.env).
A batch whose `params` rows are set solves every problem with its own vehicle limits and cost weights (ProblemBatch.params,
_lib.problem_params); everything else comes from its environment.
All compute happens inside libualm.so on the GPU; this file only marshals numpy arrays.
"""
import contextlib
import ctypes as C

import numpy as np

from . import _lib
from ._lib import Params, Result

dp = C.POINTER(C.c_double)
ip = C.POINTER(C.c_int32)


def _p(a, t=dp):
    return None if a is None else a.ctypes.data_as(t)


def _env(pb):
    """int32 environment index per problem, or None (= all environment 0)"""
    return None if getattr(pb, "env", None) is None else np.ascontiguousarray(pb.env, np.int32)


def _pp(pb):
    """float64 [B, 8] parameter rows (ualm_problem_params_t), or None (= every problem uses its environment's)"""
    pp = getattr(pb, "params", None)
    if pp is None:
        return None
    pp = np.ascontiguousarray(pp, np.float64)
    if pp.shape != (pb.B, 8):
        raise ValueError("params must be float64 [B, 8] = [%d, 8], got %r" % (pb.B, pp.shape))
    return pp


ppp = C.POINTER(_lib.ProblemParams)


class UalmError(RuntimeError):
    pass


def _check(rc):
    if rc != 0:
        msg = _lib.lib().ualm_last_error()
        raise UalmError(f"libualm error {rc}: {msg.decode() if msg else ''}")


class BatchALMTrajOpt:
    def __init__(self, device=0, precision=64):
        L = _lib.lib()
        if not hasattr(L, "ualm_create"):
            raise ImportError("libualm.so was built without the CUDA translation unit")
        self.L = L
        self.h = C.c_void_p()
        _check(L.ualm_create(C.byref(self.h), device, precision))
        self.params = None
        self.env_params = {}
        self.env = 0            # the selected environment (ualm_select_env)
        self.geoms = {}         # the geometry of each environment's grid, as last bound
        self.pb = None

    def close(self):
        if self.h:
            self.L.ualm_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def select_env(self, env):
        """ualm_select_env: init / set_environment without an `env` argument bind environment `env` from now on."""
        _check(self.L.ualm_select_env(self.h, int(env)))
        self.env = int(env)
        return self

    def init(self, params=None, env=None):
        """ualm_set_params for environment `env` (None: the selected one, environment 0 unless select_env chose another; a given
        `env` stays selected).  self.params keeps environment 0's."""
        params = params or _lib.default_params()
        if env is not None:
            self.select_env(env)
        _check(self.L.ualm_set_params(self.h, C.byref(params)))
        self.env_params[self.env] = params
        if self.env == 0:
            self.params = params
        return self

    def set_budget(self, max_evals):
        """ualm_set_budget: evaluation budget per problem of the solves launched afterwards (0 = none).  A problem it stops ends
        with ret_code UALM_RET_STOPPED (3) after max_evals..max_evals + 64 evaluations."""
        _check(self.L.ualm_set_budget(self.h, int(max_evals)))
        return self

    def set_stream(self, cuda_stream_ptr):
        _check(self.L.ualm_set_stream(self.h, C.c_void_p(cuda_stream_ptr)))
        return self

    def set_environment(self, mapdata, repack_to_float=False, env=None):
        """Binds the map grid of environment `env` (None: the selected one, as for init).  A map that carries the reference's own double
        grid (`cells64`, RXS2 = 4 doubles per cell) goes through ualm_set_map_f64; repack_to_float rounds it to the float4 grid on the way."""
        if env is not None:
            self.select_env(env)
        if self.env == 0:
            self.map = mapdata
        self.geoms[self.env] = mapdata.geom
        c64 = getattr(mapdata, "cells64", None)
        if c64 is not None:
            _check(self.L.ualm_set_map_f64(self.h, C.byref(mapdata.geom), c64.ctypes.data_as(dp), 1 if repack_to_float else 0))
        else:
            _check(self.L.ualm_set_map(self.h, C.byref(mapdata.geom), mapdata.cells.ctypes.data_as(C.POINTER(C.c_float))))
        return self

    def update_environment(self, mapdata, env=None):
        """ualm_update_map: replaces the float grid of environment `env` (None: the selected one, as for set_environment) while batches
        may be in flight.  Work launched before keeps its grid (batches in flight, feasibility of a lane solved before); every later
        launch reads the new one.  Returns once the new grid is on the device, without waiting for running batches."""
        if env is not None:
            self.select_env(env)
        if self.env == 0:
            self.map = mapdata
        cells = np.ascontiguousarray(mapdata.cells, np.float32)
        _check(self.L.ualm_update_map(self.h, C.byref(mapdata.geom), cells.ctypes.data_as(C.POINTER(C.c_float))))
        self.geoms[self.env] = mapdata.geom
        return self

    def update_environment_from_cloud(self, pts, geom=None, ellipsoid=(0.2, 0.1, 0.1), iter_num=2, env=None, name="map"):
        """ualm_update_map_from_cloud: update_environment with the grid built on the device from a point cloud (as build_map) straight
        into the new grid.  Returns (UnevenMapData of the new grid, as the host front end needs it; kernel ms)."""
        from . import maps
        geom = geom or _lib.map_geometry()
        if env is not None:
            self.select_env(env)
        X, Y, W = geom.voxel_num
        cells = np.zeros((X, Y, W, 4), np.float32)
        pts = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 3)
        ms = C.c_float()
        fp = C.POINTER(C.c_float)
        _check(self.L.ualm_update_map_from_cloud(self.h, pts.ctypes.data_as(fp), pts.shape[0], C.byref(geom), ellipsoid[0], ellipsoid[1], ellipsoid[2],
                                                 iter_num, cells.ctypes.data_as(fp), C.byref(ms)))
        m = maps.UnevenMapData(geom, cells, name)
        if self.env == 0:
            self.map = m
        self.geoms[self.env] = geom
        return m, ms.value

    def update_environment_window(self, ix0, iy0, cells, env=None):
        """ualm_update_map_window: replaces the cell columns [ix0, ix0+nx) x [iy0, iy0+ny), all yaw layers, of environment `env`'s grid
        (None: the selected one) with `cells` = (nx, ny, Yaw, 4) float32, with update_environment's guarantees.  The geometry stays
        the current grid's (maps.window_box turns a metric rectangle into a box).  self.map is not spliced: the host grid is not
        copied for a window."""
        if env is not None:
            self.select_env(env)
        cells = np.ascontiguousarray(cells, np.float32)
        geom = self.geoms.get(self.env)
        if cells.ndim != 4 or cells.shape[3] != 4 or (geom is not None and cells.shape[2] != geom.voxel_num[2]):
            raise ValueError("cells must be (nx, ny, Yaw, 4) with the grid's Yaw, got %r" % (cells.shape,))
        _check(self.L.ualm_update_map_window(self.h, int(ix0), int(iy0), cells.shape[0], cells.shape[1], cells.ctypes.data_as(C.POINTER(C.c_float))))
        return self

    def update_environment_window_from_cloud(self, pts, ix0, iy0, nx, ny, ellipsoid=(0.2, 0.1, 0.1), iter_num=2, env=None):
        """ualm_update_map_window_from_cloud: the same box built on the device from a point cloud (e.g. a local scan) with the
        current grid's geometry.  Returns (the box's cells, (nx, ny, Yaw, 4) float32; kernel ms)."""
        if env is not None:
            self.select_env(env)
        pts = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 3)
        fp = C.POINTER(C.c_float)
        geom = self.geoms.get(self.env)           # None: no grid bound, which the call refuses
        cells = np.zeros((max(int(nx), 0), max(int(ny), 0), geom.voxel_num[2] if geom else 0, 4), np.float32)
        ms = C.c_float()
        _check(self.L.ualm_update_map_window_from_cloud(self.h, pts.ctypes.data_as(fp), pts.shape[0], int(ix0), int(iy0), int(nx), int(ny), ellipsoid[0],
                                                        ellipsoid[1], ellipsoid[2], iter_num, cells.ctypes.data_as(fp) if cells.size else None, C.byref(ms)))
        return cells, ms.value

    def _shift_geom(self):
        """the selected environment's geometry as this object last bound it; a shift needs it to lay out the strips and to return the
        moved geometry, so a grid bound without this object (or none at all) is refused before the library is called"""
        geom = self.geoms.get(self.env)
        if geom is None:
            raise UalmError("environment %d has no grid bound through set_environment / update_environment*: its geometry is unknown" % self.env)
        return geom

    def shift_environment(self, dx, dy, cells, env=None):
        """ualm_shift_map: moves environment `env`'s grid (None: the selected one) by (dx, dy) whole cells, with
        update_environment_window's guarantees.  `cells` holds the cells of the boxes maps.shift_boxes gives, one after the other: a
        sequence of (nx, ny, Yaw, 4) float32 arrays, or one flat float32 array of them all.  Returns the moved geometry
        (maps.shift_geometry).  self.map is not moved: the host grid is not copied for a shift."""
        from . import maps
        if env is not None:
            self.select_env(env)
        flat = np.ascontiguousarray(np.concatenate([np.asarray(c, np.float32).ravel() for c in cells])
                                    if isinstance(cells, (list, tuple)) else np.asarray(cells, np.float32).ravel())
        geom = self._shift_geom()
        want = sum(b[2] * b[3] for b in maps.shift_boxes(geom, dx, dy)) * geom.voxel_num[2] * 4
        if flat.size != want:
            raise ValueError("cells must hold %d floats for the shift (%d, %d), got %d" % (want, dx, dy, flat.size))
        _check(self.L.ualm_shift_map(self.h, int(dx), int(dy), flat.ctypes.data_as(C.POINTER(C.c_float))))
        self.geoms[self.env] = g = maps.shift_geometry(geom, dx, dy)
        return g

    def shift_environment_from_cloud(self, pts, dx, dy, ellipsoid=(0.2, 0.1, 0.1), iter_num=2, env=None):
        """ualm_shift_map_from_cloud: the same shift with the uncovered boxes built on the device from a point cloud (e.g. a local scan)
        with the moved geometry.  Returns (the moved geometry; the boxes' cells, a list of (nx, ny, Yaw, 4) float32 arrays in
        maps.shift_boxes's order; kernel ms)."""
        from . import maps
        if env is not None:
            self.select_env(env)
        pts = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 3)
        fp = C.POINTER(C.c_float)
        geom = self._shift_geom()
        boxes = maps.shift_boxes(geom, dx, dy)
        W = geom.voxel_num[2]
        flat = np.zeros(sum(b[2] * b[3] for b in boxes) * W * 4, np.float32)
        ms = C.c_float()
        _check(self.L.ualm_shift_map_from_cloud(self.h, pts.ctypes.data_as(fp), pts.shape[0], int(dx), int(dy), ellipsoid[0], ellipsoid[1],
                                                ellipsoid[2], iter_num, flat.ctypes.data_as(fp) if flat.size else None, C.byref(ms)))
        out, o = [], 0
        for b in boxes:
            n = b[2] * b[3] * W * 4
            out.append(flat[o:o + n].reshape(b[2], b[3], W, 4))
            o += n
        self.geoms[self.env] = g = maps.shift_geometry(geom, dx, dy)
        return g, out, ms.value

    def reset_stream(self):
        _check(self.L.ualm_reset_stream(self.h))
        return self

    # ---- lanes: several resident batches in flight on this context ----------------------
    def select_lane(self, lane):
        _check(self.L.ualm_select_lane(self.h, int(lane)))
        self.pb = self._lane_pb.get(int(lane), self.pb) if hasattr(self, "_lane_pb") else self.pb
        self._lane = int(lane)
        return self

    def mark_begin(self):
        _check(self.L.ualm_mark_begin(self.h))

    def mark_end(self):
        ms = C.c_float()
        _check(self.L.ualm_mark_end(self.h, C.byref(ms)))
        return ms.value

    @contextlib.contextmanager
    def _urgency(self, urgent):
        """ualm_set_urgent(urgent) around one call, and the context's flag back to 0 after it"""
        if not urgent:
            yield
            return
        _check(self.L.ualm_set_urgent(self.h, 1))
        try:
            yield
        finally:
            _check(self.L.ualm_set_urgent(self.h, 0))

    def submit(self, pb, depth=2, host=None, urgent=False):
        """ualm_submit_batch: returns a ticket; `host` = optional pre-made (N, M, bnd, T, ixy, iyaw) host arrays (e.g. pinned).
        urgent: the ticket goes ahead of the batches in flight (ualm_set_urgent), with the same results."""
        if host is None:
            host = [np.ascontiguousarray(a) for a in (pb.N.astype(np.int32), pb.M.astype(np.int32), pb.bnd.astype(np.float64),
                                                        pb.total_time.astype(np.float64), pb.inner_xy.astype(np.float64),
                                                        pb.inner_yaw.astype(np.float64))]
        N, M, bnd, T, ixy, iyaw = host
        t = C.c_int(-1)
        env, pp = _env(pb), _pp(pb)
        with self._urgency(urgent):
            _check(self.L.ualm_submit_batch_pp(self.h, pb.B, _p(N, ip), _p(M, ip), _p(bnd), _p(T), _p(ixy), _p(iyaw), _p(env, ip), _p(pp, ppp),
                                               int(depth), C.byref(t)))
        if not hasattr(self, "_tickets"):
            self._tickets = {}
        self._tickets[t.value] = (pb, (host, env, pp))
        return t.value

    def wait(self, ticket, out=None, timeout_ms=None):
        """ualm_wait_batch: (results, c_xy, c_yaw) of the ticket's batch; `out` = optional preallocated (res, cxy, cyaw).
        timeout_ms (ualm_wait_batch_for): if the batch is not complete by then, its running problems are stopped (ret_code
        UALM_RET_STOPPED) and the complete records of the drained batch come back."""
        pb, _ = self._tickets.pop(ticket)
        if out is None:
            out = self.outputs(pb)
        res, cxy, cyaw = out
        if timeout_ms is None:
            _check(self.L.ualm_wait_batch(self.h, int(ticket), res, _p(cxy), _p(cyaw)))
        else:
            _check(self.L.ualm_wait_batch_for(self.h, int(ticket), float(timeout_ms), res, _p(cxy), _p(cyaw)))
        return res, cxy, cyaw

    @staticmethod
    def outputs(pb):
        """Empty (results, c_xy, c_yaw) for batch `pb`, the buffers wait(out=) and poll(out) fill."""
        return (Result * pb.B)(), np.zeros(int(12 * pb.N.astype(np.int64).sum())), np.zeros(int(6 * pb.M.astype(np.int64).sum()))

    def poll(self, ticket, out, wait_ms=0.0):
        """ualm_poll_batch: the problems of the ticket's batch that finished since the last poll, without waiting for the rest.
        Their records and coefficients go to their problem-order places in `out` = (results, c_xy, c_yaw), as wait(out=) fills them
        (c_xy / c_yaw may be None); nothing else in `out` is touched.  wait_ms > 0 blocks until at least one problem is new or
        wait_ms has passed.  Returns (new problem indices as an int32 array, number of problems not yet returned).  wait(ticket)
        afterwards returns the whole batch as before."""
        if ticket not in getattr(self, "_tickets", {}):
            raise ValueError("poll: %r is not a ticket in flight on this context" % (ticket,))
        wait_ms = float(wait_ms)
        if not wait_ms >= 0.0:
            raise ValueError("poll: wait_ms must be >= 0")
        pb = self._tickets[ticket][0]
        res, cxy, cyaw = out
        if not isinstance(res, C.Array) or res._type_ is not Result or len(res) != pb.B:
            raise ValueError("poll: out[0] must be a ctypes array of %d Result records" % pb.B)
        for a, n, name in ((cxy, 12 * int(pb.N.astype(np.int64).sum()), "c_xy"), (cyaw, 6 * int(pb.M.astype(np.int64).sum()), "c_yaw")):
            if a is not None and (not isinstance(a, np.ndarray) or a.dtype != np.float64 or not a.flags.c_contiguous or a.size != n):
                raise ValueError("poll: out %s must be None or a contiguous float64 array of %d entries" % (name, n))
        idx = np.zeros(max(pb.B, 1), np.int32)
        n_new, n_pending = C.c_int(), C.c_int()
        _check(self.L.ualm_poll_batch(self.h, int(ticket), wait_ms, _p(idx, ip), C.byref(n_new), C.byref(n_pending), res, _p(cxy), _p(cyaw)))
        return idx[:n_new.value].copy(), n_pending.value

    def cancel(self, ticket, idx):
        """ualm_cancel_problems: stop the problems `idx` (integer indices into the ticket's batch) at their next stop test.  Each comes
        back through poll / wait, with ret_code UALM_RET_STOPPED or, if it was final first, its own result; every other problem and
        ticket is unaffected.  Duplicates and repeated calls are harmless.  Nothing is cancelled when an argument is refused."""
        if ticket not in getattr(self, "_tickets", {}):
            raise ValueError("cancel: %r is not a ticket in flight on this context" % (ticket,))
        a = np.asarray(idx)
        if a.ndim > 1 or (a.size and not np.issubdtype(a.dtype, np.integer)):
            raise ValueError("cancel: idx must be a 1-D sequence of problem indices")
        a = np.ascontiguousarray(a.reshape(-1), np.int64)
        B = self._tickets[ticket][0].B
        if a.size and (a.min() < 0 or a.max() >= B):
            raise ValueError("cancel: problem index out of range [0, %d)" % B)
        a = a.astype(np.int32)
        _check(self.L.ualm_cancel_problems(self.h, int(ticket), int(a.size), _p(a, ip)))

    # ---- three-step path -------------------------------------------------------------
    def upload(self, pb):
        self.pb = pb
        if not hasattr(self, "_lane_pb"):
            self._lane_pb = {}
        self._lane_pb[getattr(self, "_lane", 0)] = pb
        self._keep = [np.ascontiguousarray(a) for a in (pb.N.astype(np.int32), pb.M.astype(np.int32), pb.bnd.astype(np.float64),
                                                        pb.total_time.astype(np.float64), pb.inner_xy.astype(np.float64),
                                                        pb.inner_yaw.astype(np.float64))]
        self._keep += [_env(pb), _pp(pb)]
        N, M, bnd, T, ixy, iyaw, env, pp = self._keep
        _check(self.L.ualm_upload_pp(self.h, pb.B, _p(N, ip), _p(M, ip), _p(bnd), _p(T), _p(ixy), _p(iyaw), _p(env, ip), _p(pp, ppp)))

    def solve_resident(self):
        _check(self.L.ualm_solve_resident(self.h))

    def sync(self):
        _check(self.L.ualm_sync(self.h))

    def last_solve_ms(self):
        ms, n = C.c_float(), C.c_int()
        _check(self.L.ualm_last_solve_ms(self.h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def download(self):
        pb = self.pb
        res = (Result * pb.B)()
        cxy = np.zeros(int(12 * pb.N.astype(np.int64).sum()))
        cyaw = np.zeros(int(6 * pb.M.astype(np.int64).sum()))
        _check(self.L.ualm_download(self.h, res, _p(cxy), _p(cyaw)))
        return res, cxy, cyaw

    # ---- one call, host buffers in / host buffers out (the drop-in call) ---------------
    def optimize(self, pb):
        self.pb = pb
        N = np.ascontiguousarray(pb.N, np.int32); M = np.ascontiguousarray(pb.M, np.int32)
        bnd = np.ascontiguousarray(pb.bnd, np.float64); T = np.ascontiguousarray(pb.total_time, np.float64)
        ixy = np.ascontiguousarray(pb.inner_xy, np.float64); iyaw = np.ascontiguousarray(pb.inner_yaw, np.float64)
        res = (Result * pb.B)()
        cxy = np.zeros(int(12 * N.astype(np.int64).sum()))
        cyaw = np.zeros(int(6 * M.astype(np.int64).sum()))
        env, pp = _env(pb), _pp(pb)
        _check(self.L.ualm_solve_batch_pp(self.h, pb.B, _p(N, ip), _p(M, ip), _p(bnd), _p(T), _p(ixy), _p(iyaw), _p(env, ip), _p(pp, ppp), res,
                                          _p(cxy), _p(cyaw)))
        return res, cxy, cyaw

    def pack_records(self, dev_ptr, stride, wait=True):
        f = self.L.ualm_pack_records_device if wait else self.L.ualm_pack_records_device_async
        _check(f(self.h, C.c_void_p(dev_ptr), stride))

    # ---- phase entry points ----------------------------------------------------------
    def _samples(self, pb):
        """samples per problem: N (int_K + 1) with the int_K of the problem's environment"""
        K = np.array([self.env_params[e].int_K if e in self.env_params else 0 for e in range(_lib.UALM_MAX_ENVS)], np.int64)
        env = np.zeros(pb.B, np.int64) if getattr(pb, "env", None) is None else np.asarray(pb.env, np.int64)
        return pb.N.astype(np.int64) * (K[env] + 1)

    def eval_batch(self, x=None, lam=None, mu=None, scale_cx=None, scale_fx=None, rho=None):
        """ualm_eval_batch at one penalty weight `rho` for every problem.  rho=None: the `rho` parameter of the batch's environments,
        which must then agree (pass rho explicitly for a batch whose environments differ in it)."""
        pb = self.pb
        if rho is None:
            envs = [0] if getattr(pb, "env", None) is None else sorted({int(e) for e in pb.env})
            rhos = {self.env_params[e].rho for e in envs if e in self.env_params}
            if len(rhos) != 1:
                raise ValueError("eval_batch: the batch's environments differ in rho (or have no parameters bound): pass rho")
            rho = rhos.pop()
        nx = int(pb.nvar().sum()); S = int(self._samples(pb).sum())
        f = np.zeros(pb.B); grad = np.zeros(nx); hx = np.zeros(S); gx = np.zeros(6 * S)
        cxy = np.zeros(int(12 * pb.N.astype(np.int64).sum())); cyaw = np.zeros(int(6 * pb.M.astype(np.int64).sum()))
        arrs = [None if a is None else np.ascontiguousarray(a, np.float64) for a in (x, lam, mu, scale_cx, scale_fx)]
        _check(self.L.ualm_eval_batch(self.h, _p(arrs[0]), _p(arrs[1]), _p(arrs[2]), _p(arrs[3]), _p(arrs[4]),
                                      float(rho), _p(f), _p(grad), _p(hx), _p(gx), _p(cxy), _p(cyaw)))
        return dict(f=f, grad=grad, hx=hx, gx=gx, c_xy=cxy, c_yaw=cyaw)

    def init_scaling_batch(self):
        pb = self.pb
        S = int(self._samples(pb).sum())
        sfx = np.zeros(pb.B); scx = np.zeros(7 * S)
        _check(self.L.ualm_init_scaling_batch(self.h, _p(sfx), _p(scx)))
        return sfx, scx

    def time_penalty_kernel(self, reps=10):
        ms, by = C.c_float(), C.c_double()
        _check(self.L.ualm_time_penalty_kernel(self.h, reps, C.byref(ms), C.byref(by)))
        return ms.value, by.value

    def mpc_export(self, N, M, dt=0.01, init_v=None, init_a=None):
        """SE2Traj message arrays, the MPC side's re-solved coefficients and the planned-vs-tracked deviation of the resident solved
        batch (see ualm_mpc_export_batch).  N, M: the piece counts of the batch."""
        out = self._mpc_outputs(N, M)
        dp = C.POINTER(C.c_double)
        P = lambda a: a.ctypes.data_as(dp)
        iv = None if init_v is None else np.ascontiguousarray(init_v, dtype=np.float64)
        ia = None if init_a is None else np.ascontiguousarray(init_a, dtype=np.float64)
        _check(self.L.ualm_mpc_export_batch(self.h, float(dt), None if iv is None else P(iv), None if ia is None else P(ia), P(out["pos_pts"]), P(out["posT_pts"]),
                                            P(out["angle_pts"]), P(out["angleT_pts"]), P(out["c_mpc_xy"]), P(out["c_mpc_yaw"]), P(out["dev"])))
        return out

    @staticmethod
    def _mpc_outputs(N, M):
        """zeroed output arrays of a hand-over of trajectories with piece counts N, M (mpc_export's dict)"""
        N = np.asarray(N, dtype=np.int64); M = np.asarray(M, dtype=np.int64)
        B, sN, sM = len(N), int(N.sum()), int(M.sum())
        return dict(pos_pts=np.zeros(2 * (sN + B)), posT_pts=np.zeros(sN), angle_pts=np.zeros(sM + B), angleT_pts=np.zeros(sM),
                    c_mpc_xy=np.zeros(12 * sN), c_mpc_yaw=np.zeros(6 * sM), dev=np.zeros((B, 4)))

    def mpc_export_trajectories(self, N, M, piece_T, c_xy, c_yaw, init_v=None, init_a=None, dt=0.01, urgent=False):
        """ualm_mpc_export_trajectories: mpc_export's hand-over for trajectories the caller holds, in check_trajectories' layouts (N, M:
        [B]; piece_T: [B, 2]; c_xy / c_yaw packed as wait() returns them), each row from its own start state: init_v / init_a = {x, y,
        yaw} as None (zero, what the reference publishes), one triple for every row, or [B, 3].  Reads no grid, lane or record; may be
        called while batches are in flight.  urgent: the export goes ahead of the batches in flight (ualm_set_urgent).  Returns the
        dict mpc_export returns, rows packed in call order."""
        N = np.ascontiguousarray(N, np.int32).reshape(-1)
        M = np.ascontiguousarray(M, np.int32).reshape(-1)
        B = N.size
        pt = np.ascontiguousarray(piece_T, np.float64).reshape(-1)
        cxy = np.ascontiguousarray(c_xy, np.float64).reshape(-1)
        cyaw = np.ascontiguousarray(c_yaw, np.float64).reshape(-1)
        for a, n, name in ((M, B, "M"), (pt, 2 * B, "piece_T"), (cxy, 12 * int(N.astype(np.int64).sum()), "c_xy"),
                           (cyaw, 6 * int(M.astype(np.int64).sum()), "c_yaw")):
            if a.size != n:
                raise ValueError("mpc_export_trajectories: %s has %d entries, the piece counts need %d" % (name, a.size, n))
        init = []
        for v, name in ((init_v, "init_v"), (init_a, "init_a")):
            if v is None:
                init.append(None)
                continue
            v = np.asarray(v, np.float64)
            if v.shape not in ((3,), (B, 3)):
                raise ValueError("mpc_export_trajectories: %s must be None, 3 numbers or [B, 3] = [%d, 3], got %r" % (name, B, v.shape))
            init.append(np.ascontiguousarray(np.broadcast_to(v, (B, 3))))
        out = self._mpc_outputs(N, M)
        with self._urgency(urgent):
            _check(self.L.ualm_mpc_export_trajectories(self.h, B, _p(N, ip), _p(M, ip), _p(pt), _p(cxy), _p(cyaw), _p(init[0]), _p(init[1]), float(dt),
                                                       *[_p(out[k]) for k in ("pos_pts", "posT_pts", "angle_pts", "angleT_pts", "c_mpc_xy",
                                                                              "c_mpc_yaw", "dev")]))
        return out

    def mpc_export_results(self, pb, out, rows=None, start="rest", dt=0.01, urgent=False):
        """mpc_export_trajectories of rows `rows` (None: all) of batch `pb` as wait() / poll() returned it: out = (results, c_xy,
        c_yaw); a record poll() has not filled yet is refused.  start: "rest" = zero boundary derivatives, as the reference publishes;
        "bnd" = each row's own start state from pb.bnd, v = (bnd[2], bnd[3], bnd[13]) and a = (bnd[4], bnd[5], bnd[14]), which is
        what a replanned batch (submit_replan) carries.  Returns mpc_export's dict, rows packed in the order of `rows`."""
        rows = np.arange(pb.B) if rows is None else np.asarray(rows)
        if rows.ndim != 1 or (rows.size and not np.issubdtype(rows.dtype, np.integer)):
            raise ValueError("mpc_export_results: rows must be a 1-D sequence of problem indices")
        rows = rows.astype(np.int64)
        if rows.size and (rows.min() < 0 or rows.max() >= pb.B):
            raise ValueError("mpc_export_results: row index out of range [0, %d)" % pb.B)
        if start not in ("rest", "bnd"):
            raise ValueError("mpc_export_results: start must be 'rest' or 'bnd', got %r" % (start,))
        res, cxy, cyaw = out
        if len(res) != pb.B:
            raise ValueError("mpc_export_results: out holds %d records, the batch has %d" % (len(res), pb.B))
        _, _, ocx, ocy = pb.offsets()
        B = rows.size
        pt = np.array([(res[i].piece_T_xy, res[i].piece_T_yaw) for i in rows], np.float64).reshape(B, 2)
        c_xy = np.concatenate([cxy[ocx[i]:ocx[i + 1]] for i in rows]) if B else np.zeros(0)
        c_yaw = np.concatenate([cyaw[ocy[i]:ocy[i + 1]] for i in rows]) if B else np.zeros(0)
        v = a = None
        if start == "bnd":
            bnd = np.asarray(pb.bnd, np.float64).reshape(pb.B, 18)[rows]
            v, a = bnd[:, [2, 3, 13]], bnd[:, [4, 5, 14]]
        return self.mpc_export_trajectories(pb.N[rows], pb.M[rows], pt, c_xy, c_yaw, init_v=v, init_a=a, dt=dt, urgent=urgent)

    def feasibility(self, dt=0.01):
        """Post-solve scan of the resident batch: array [B, 10] (see ualm_feasibility_batch)."""
        out = np.zeros((self.pb.B, 10))
        _check(self.L.ualm_feasibility_batch(self.h, float(dt), out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    def check_trajectories(self, N, M, piece_T, c_xy, c_yaw, env=None, t_from=None, dt=0.01, limits=None, params=None):
        """ualm_check_trajectories: the post-solve scan of trajectories the caller holds, against each environment's grid as it is now,
        over the samples t >= t_from of the full scan, with the time each limit is first broken.  N, M: [B]; piece_T: [B, 2]
        (piece_T_xy, piece_T_yaw of the records); c_xy / c_yaw packed as wait() returns them; env: [B] or None (all 0); t_from: [B],
        one number or None (0); limits: None (each environment's own), six numbers (max_vel, max_acc_lon, max_acc_lat, max_kap,
        min_cxi, max_sig) or an object with those attributes, e.g. Params; params: None or [B, 8] parameter rows, whose limits each
        row takes where `limits` is None (ualm_check_trajectories_pp).  May be called while batches are in flight.
        Returns [B, 16]: ualm_feasibility_batch's ten columns over the kept samples, then the six first-violation times (-1: none)."""
        N = np.ascontiguousarray(N, np.int32).reshape(-1)
        M = np.ascontiguousarray(M, np.int32).reshape(-1)
        B = N.size
        pt = np.ascontiguousarray(piece_T, np.float64).reshape(-1)
        cxy = np.ascontiguousarray(c_xy, np.float64).reshape(-1)
        cyaw = np.ascontiguousarray(c_yaw, np.float64).reshape(-1)
        for a, n, name in ((M, B, "M"), (pt, 2 * B, "piece_T"), (cxy, 12 * int(N.astype(np.int64).sum()), "c_xy"),
                           (cyaw, 6 * int(M.astype(np.int64).sum()), "c_yaw")):
            if a.size != n:
                raise ValueError("check_trajectories: %s has %d entries, the piece counts need %d" % (name, a.size, n))
        e = None if env is None else np.ascontiguousarray(env, np.int32).reshape(-1)
        tf = None if t_from is None else np.ascontiguousarray(np.broadcast_to(np.asarray(t_from, np.float64), (B,)))
        if e is not None and e.size != B:
            raise ValueError("check_trajectories: env must have B = %d entries" % B)
        lim = None
        if limits is not None:
            names = [n for n, _ in _lib.Limits._fields_]
            vals = [getattr(limits, n) for n in names] if hasattr(limits, "max_vel") else list(limits)
            if len(vals) != 6:
                raise ValueError("check_trajectories: limits must be six numbers %s" % (names,))
            lim = _lib.Limits(*[float(v) for v in vals])
        pp = None if params is None else np.ascontiguousarray(params, np.float64)
        if pp is not None and pp.shape != (B, 8):
            raise ValueError("check_trajectories: params must be [B, 8] = [%d, 8], got %r" % (B, pp.shape))
        out = np.zeros((B, 16))
        _check(self.L.ualm_check_trajectories_pp(self.h, B, _p(N, ip), _p(M, ip), _p(pt), _p(cxy), _p(cyaw), _p(e, ip), _p(pp, ppp), _p(tf),
                                                 float(dt), None if lim is None else C.byref(lim), _p(out)))
        return out

    def check_results(self, pb, out, t_from=None, dt=0.01, limits=None, urgent=False):
        """check_trajectories of batch `pb` as wait() / poll() returned it: out = (results, c_xy, c_yaw).  A record poll() has not
        filled yet has zero durations and keeps no sample.  The limits are `limits` when given, else the batch's parameter rows', else each
        environment's.  urgent: the check goes ahead of the batches in flight (ualm_set_urgent)."""
        res, cxy, cyaw = out
        pt = np.array([(r.piece_T_xy, r.piece_T_yaw) for r in res], np.float64).reshape(pb.B, 2)
        with self._urgency(urgent):
            return self.check_trajectories(pb.N, pb.M, pt, cxy, cyaw, env=_env(pb), t_from=t_from, dt=dt, limits=limits, params=_pp(pb))

    def submit_replan(self, pb, out, rows, t_from, dt=0.01, rparams=None, depth=2, urgent=False):
        """ualm_submit_replan: replans rows `rows` of batch `pb` as wait() / poll() returned it (out = (results, c_xy, c_yaw)) from each
        robot's state at time t_from (one number or one per row) on its trajectory to the row's original goal, with PlanManager's
        resampler over the trajectory's samples t_from < t of the sequence t = 0, dt, 2dt.. (rparams: front_end.resample_params(), None
        = its defaults), and submits the built problems as one ticket on the next lane of `depth`.  Returns (ticket, ProblemBatch of the
        built problems, in the order of `rows`, with their environments and parameter rows, which the ticket solves with); poll / wait /
        cancel / check_results work on it as on any.
        urgent: the build and the ticket go ahead of the batches in flight (ualm_set_urgent)."""
        from . import problems
        rows = np.asarray(rows)
        if rows.ndim != 1 or (rows.size and not np.issubdtype(rows.dtype, np.integer)):
            raise ValueError("submit_replan: rows must be a 1-D sequence of problem indices")
        rows = rows.astype(np.int64)
        if rows.size and (rows.min() < 0 or rows.max() >= pb.B):
            raise ValueError("submit_replan: row index out of range [0, %d)" % pb.B)
        res, cxy, cyaw = out
        if len(res) != pb.B:
            raise ValueError("submit_replan: out holds %d records, the batch has %d" % (len(res), pb.B))
        B = rows.size
        tf = np.ascontiguousarray(np.broadcast_to(np.asarray(t_from, np.float64), (B,)))
        sub = pb.select(rows)
        _, _, ocx, ocy = pb.offsets()
        N, M = np.ascontiguousarray(sub.N, np.int32), np.ascontiguousarray(sub.M, np.int32)
        pt = np.array([(res[i].piece_T_xy, res[i].piece_T_yaw) for i in rows], np.float64).reshape(B, 2)
        c_xy = np.concatenate([cxy[ocx[i]:ocx[i + 1]] for i in rows]) if B else np.zeros(0)
        c_yaw = np.concatenate([cyaw[ocy[i]:ocy[i + 1]] for i in rows]) if B else np.zeros(0)
        bnd = np.ascontiguousarray(sub.bnd, np.float64).reshape(B, 18)
        env, pp = _env(sub), _pp(sub)
        rp = None if rparams is None else C.byref(rparams)
        No, Mo = np.zeros(B, np.int32), np.zeros(B, np.int32)
        bo, To = np.zeros((B, 18)), np.zeros(B)
        ixy, iyaw = np.zeros((B, _lib.UALM_REPLAN_INNER_XY)), np.zeros((B, _lib.UALM_REPLAN_INNER_YAW))
        t = C.c_int(-1)
        with self._urgency(urgent):
            _check(self.L.ualm_submit_replan_pp(self.h, B, _p(N, ip), _p(M, ip), _p(pt), _p(c_xy), _p(c_yaw), _p(bnd), _p(env, ip), _p(pp, ppp), _p(tf),
                                                float(dt), rp, int(depth), C.byref(t), _p(No, ip), _p(Mo, ip), _p(bo), _p(To), _p(ixy), _p(iyaw)))
        # a row over the compiled limits (N 64, M 128): zeros, as the C call packs it
        fits = lambda b: 2 * (No[b] - 1) <= _lib.UALM_REPLAN_INNER_XY and Mo[b] - 1 <= _lib.UALM_REPLAN_INNER_YAW
        pxy = [ixy[b, :2 * (No[b] - 1)] if fits(b) else np.zeros(2 * (int(No[b]) - 1)) for b in range(B)]
        pyaw = [iyaw[b, :Mo[b] - 1] if fits(b) else np.zeros(int(Mo[b]) - 1) for b in range(B)]
        new = problems.ProblemBatch(No, Mo, bo, To, np.concatenate(pxy) if B else np.zeros(0), np.concatenate(pyaw) if B else np.zeros(0),
                                    env=None if env is None else env.copy(), params=None if pp is None else pp.copy())
        if not hasattr(self, "_tickets"):
            self._tickets = {}
        self._tickets[t.value] = (new, (None, env, pp))
        return t.value, new

    def build_map(self, pts, geom=None, ellipsoid=(0.2, 0.1, 0.1), iter_num=2, name="map"):
        """UnevenMap grid from a point cloud on the GPU (ualm_map_build_device): (UnevenMapData, kernel ms)."""
        from . import maps
        geom = geom or _lib.map_geometry()
        X, Y, W = geom.voxel_num
        cells = np.zeros((X, Y, W, 4), np.float32)
        pts = np.ascontiguousarray(pts, dtype=np.float32)
        ms = C.c_float()
        fp = C.POINTER(C.c_float)
        _check(self.L.ualm_map_build_device(self.h, pts.ctypes.data_as(fp), pts.shape[0], C.byref(geom), ellipsoid[0], ellipsoid[1], ellipsoid[2],
                                            iter_num, cells.ctypes.data_as(fp), C.byref(ms)))
        return maps.UnevenMapData(geom, cells, name), ms.value

    PHASES = ("fill", "lu", "solve", "jerk", "tables", "samples", "accumulate", "combine", "adjoint", "tail", "twoloop", "linesearch",
              "scaling", "dual", "other", "total")

    def profile(self, enable=True, read=False):
        out = (C.c_longlong * 16)()
        _check(self.L.ualm_profile(self.h, 1 if enable else 0, out if read else None))
        return dict(zip(self.PHASES, list(out))) if read else None


def solve_batch_multi(opts, pb):
    """ualm_solve_batch_multi_pp: one host process, one BatchALMTrajOpt per device (same params and maps bound on each)."""
    L = opts[0].L
    hs = (C.c_void_p * len(opts))(*[o.h for o in opts])
    N = np.ascontiguousarray(pb.N, np.int32); M = np.ascontiguousarray(pb.M, np.int32)
    bnd = np.ascontiguousarray(pb.bnd, np.float64); T = np.ascontiguousarray(pb.total_time, np.float64)
    ixy = np.ascontiguousarray(pb.inner_xy, np.float64); iyaw = np.ascontiguousarray(pb.inner_yaw, np.float64)
    res = (Result * pb.B)()
    cxy = np.zeros(int(12 * N.astype(np.int64).sum())); cyaw = np.zeros(int(6 * M.astype(np.int64).sum()))
    env, pp = _env(pb), _pp(pb)
    _check(L.ualm_solve_batch_multi_pp(hs, len(opts), pb.B, _p(N, ip), _p(M, ip), _p(bnd), _p(T), _p(ixy), _p(iyaw), _p(env, ip), _p(pp, ppp), res,
                                       _p(cxy), _p(cyaw)))
    return res, cxy, cyaw
