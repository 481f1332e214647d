"""The mechanics the test modules share: the `gpu` fixture, contexts, per-problem slices of a solve, the result comparisons, the
C++ drivers of tests/cpp and the compile-on-first-use oracle extensions.

The comparisons return a value and assert nothing: pytest rewrites `assert` only in test modules, so the test asserts on what they
return and keeps its own message.  What each one checks:

  * same_bytes(a, b): records and coefficients equal as bytes (+0.0 != -0.0, a NaN equals the same NaN bits);
  * same_values(a, b): records equal as bytes, coefficients equal as values (np.array_equal: +0.0 == -0.0, NaN != NaN), or with
    equal_nan=True NaN == NaN;
  * same_pieces(a, b): two lists of pieces (see pieces), each pair as same_values;
  * same_problem(pb, a, b, i): problem i of two solves as same_bytes, or with values=True as same_values;
  * solve_diff(a, b): what differs between two solves of one problem, GPU or oracle: the RECORD fields (NaN != NaN), and the
    arrays as values; with equal_nan=True NaN == NaN in both.
"""
import contextlib
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def gpu(built):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from uneven_planner_b200 import api
    return api


# ------------------------------------------------------------------ contexts
@contextlib.contextmanager
def environ(env):
    """environment variables `env` set inside the block, restored after it"""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k)
            else:
                os.environ[k] = v


def ctx(api, precision, params, grid, env=None):
    """a context of `precision` bound to one parameter set and one grid, or (lists) to params[e] and grid[e] in environment e;
    env: environment variables set while the context is created"""
    with environ(env or {}):
        opt = api.BatchALMTrajOpt(precision=precision)
        if not isinstance(params, list):
            return opt.init(params).set_environment(grid)
        for e in range(len(params)):
            opt.init(params[e], env=e).set_environment(grid[e], env=e)
        return opt


def alone(opt, pb, feas=False, dt=0.01):
    """pb solved on the fresh context `opt`, which is closed: (pieces, the post-solve scan or None)"""
    out = opt.optimize(pb)
    f = opt.feasibility(dt) if feas else None
    opt.close()
    return pieces(pb, out), f


def pending(opt, ticket, pb):
    """problems of `ticket` not yet returned"""
    return opt.poll(ticket, opt.outputs(pb), 0.0)[1]


# ------------------------------------------------------------------ per problem
def part(pb, out, i):
    """problem i of a solve (results, c_xy, c_yaw): (record, c_xy, c_yaw)"""
    _, _, ocx, ocy = pb.offsets()
    return out[0][i], out[1][ocx[i]:ocx[i + 1]], out[2][ocy[i]:ocy[i + 1]]


def split(pb, out):
    """[(record, c_xy, c_yaw)] of every problem; the coefficients are views of the solve's arrays"""
    res, cxy, cyaw = out
    _, _, ocx, ocy = pb.offsets()
    return [(res[i], cxy[ocx[i]:ocx[i + 1]], cyaw[ocy[i]:ocy[i + 1]]) for i in range(pb.B)]


def pieces(pb, out):
    """[(record bytes, c_xy, c_yaw)] of every problem, copied"""
    return [(bytes(r), x.copy(), y.copy()) for r, x, y in split(pb, out)]


def cat(pbs, envs=None):
    """one batch of `pbs`; without envs it carries no environment indices"""
    from uneven_planner_b200 import problems
    out = problems.concat(pbs, envs or [0] * len(pbs))
    if envs is None:
        out.env = None
    return out


# ------------------------------------------------------------------ grids
def box_cells(cells, b):
    ix0, iy0, nx, ny = b
    return cells[ix0:ix0 + nx, iy0:iy0 + ny]


def splice(base, cells, b, name="spliced"):
    """base's grid with `cells` in the box b, done in numpy"""
    from uneven_planner_b200 import maps
    out = base.cells.copy()
    ix0, iy0, nx, ny = b
    out[ix0:ix0 + nx, iy0:iy0 + ny] = cells
    return maps.UnevenMapData(base.geom, out, name)


# ------------------------------------------------------------------ comparisons
def bits(a, dtype=np.float64):
    """the bit patterns of a float64 (uint64) or float32 (uint32) array"""
    return np.ascontiguousarray(a, dtype).view(np.uint64 if np.dtype(dtype) == np.float64 else np.uint32)


def same_bytes(a, b):
    """(records, c_xy, c_yaw) of a whole solve or of one problem: all three equal as bytes"""
    return bytes(a[0]) == bytes(b[0]) and a[1].tobytes() == b[1].tobytes() and a[2].tobytes() == b[2].tobytes()


def same_values(a, b, equal_nan=False):
    """(record, c_xy, c_yaw) of one problem: records equal as bytes, coefficients as values (np.array_equal)"""
    return bytes(a[0]) == bytes(b[0]) and np.array_equal(a[1], b[1], equal_nan=equal_nan) and \
        np.array_equal(a[2], b[2], equal_nan=equal_nan)


def same_problem(pb, a, b, i, values=False):
    """problem i of two solves of pb: same_bytes, or with values=True same_values"""
    return (same_values if values else same_bytes)(part(pb, a, i), part(pb, b, i))


def same_pieces(a, b):
    """two lists of pieces, pair by pair as same_values"""
    return len(a) == len(b) and all(same_values(x, y) for x, y in zip(a, b))


# the fields a GPU record (ualm Result) shares with the oracle's (OResult)
RECORD = ("ret_code", "outer_iters", "n_evals", "n_lbfgs_iters", "last_lbfgs_ret", "max_bound", "inner_cost", "jerk_cost", "total_T",
          "res_h", "res_g", "scale_fx", "rho_final")


def solve_diff(a, b, equal_nan=False):
    """(record, c_xy, c_yaw, ...) of one problem in two solves, GPU or oracle: [(field, a's, b's)] of the RECORD fields that differ,
    then ("array", k) for each later array k that differs as values (np.array_equal); equal_nan: NaN equals NaN in both"""
    def same(x, y):
        return x == y or (equal_nan and x != x and y != y)
    d = [(f, getattr(a[0], f), getattr(b[0], f)) for f in RECORD if not same(getattr(a[0], f), getattr(b[0], f))]
    return d + [("array", k) for k, (x, y) in enumerate(zip(a[1:], b[1:]), 1) if not np.array_equal(x, y, equal_nan=equal_nan)]


# ------------------------------------------------------------------ native code of the tests
def build_driver(name, dir):
    """tests/cpp/<name>.cpp compiled against include/ and libualm into `dir`: the executable's path"""
    exe = os.path.join(str(dir), name)
    lib = os.path.join(ROOT, "uneven_planner_b200")
    subprocess.run(["g++", "-O2", "-std=c++14", "-I", os.path.join(ROOT, "include"), os.path.join(HERE, "cpp", name + ".cpp"), "-o", exe,
                    "-L", lib, "-lualm", "-Wl,-rpath," + lib], check=True)
    return exe


ORACLE_FLAGS = ["-O3", "-std=c++14", "-fPIC", "-ffp-contract=off", "-w", "-shared"]   # oracle/Makefile's CXXFLAGS


def load_oracle_ext(src, stem):
    """the shared library of tests/<src>, which includes oracle/oracle.cpp, compiled with the oracle's own flags on first use into
    the system temporary directory as ualm_<stem>_<uid>_<hash>.so (the tree is not written); the hash covers the compiler, the
    flags and every source, so an edit compiles it again"""
    src = os.path.join(HERE, src)
    deps = [src, os.path.join(ROOT, "oracle", "oracle.cpp"), os.path.join(ROOT, "oracle", "oracle.h"), os.path.join(ROOT, "include", "ualm_detmath.h")]
    cxx = os.environ.get("CXX", "g++")
    h = hashlib.sha256((cxx + " ".join(ORACLE_FLAGS)).encode())
    for p in deps:
        with open(p, "rb") as f:
            h.update(f.read())
    out = os.path.join(tempfile.gettempdir(), "ualm_%s_%d_%s.so" % (stem, os.getuid(), h.hexdigest()[:16]))
    if not os.path.exists(out):
        tmp = "%s.%d.tmp" % (out, os.getpid())
        subprocess.run([cxx] + ORACLE_FLAGS + ["-o", tmp, src], check=True)
        os.replace(tmp, out)
    return C.CDLL(out)
