"""Float64 restatement of the map builders' input pipeline, for tests: UnevenMap::init's CropBox + 1 cm VoxelGrid
(uneven_map.cpp:127-143) and UnevenMap::constructMap + filter (uneven_map.cpp:317-398, 5-43), from the rules DESIGN section 6 gives.

It shares no code and no algorithm with csrc/map_cell.h: scipy KD-trees instead of the bin grid and its ring search, numpy's eigh
(LAPACK) instead of the cyclic Jacobi, all cells of a grid at once instead of one cell per thread.

Where the float32 grid a builder writes is not a function of the exact arithmetic, a cell is ambiguous and the reference carries one
row per variant instead of one answer (each cell is independent of every other, so a variant is the same cell re-run with one choice
fixed):

* nearest-point near-ties (iteration 0): the second-nearest point in XY is within a relative 1e-6 of the nearest in squared
  distance; the builder compares float distances.  One row per candidate's z.
* points on the ellipsoid's surface: |r^2 - 1| < 1e-9.  One row with them, one without.
* degenerate eigenproblems: two points, or a relative gap lambda_mid - lambda_min <= 1e-9 lambda_max.  The normal is not unique: in
  the last iteration the row is checked by properties (z, sigma, the normal in the smallest eigenspace); before it, every later
  iteration depends on the choice and the row is checked for plausibility only.
* horizontal normals, |n_z| < 1e-6: the sign of (n_x, n_y) follows rounding noise where n_z is 0 up to rounding, and
  c = sqrt(1 - zbx^2 - zby^2) may come out NaN.  With c NaN, the next iteration's frame is NaN and no point passes the ellipsoid
  test, so the cell takes the empty-footprint branch with its previous z.  Rows: both signs, each with c and with c NaN.
"""
import itertools

import numpy as np
from scipy.spatial import cKDTree

TIE_REL = 1e-6          # nearest-point near-ties, relative in squared distance
SURFACE = 1e-9          # |r^2 - 1| below this: on the ellipsoid's surface
GAP_REL = 1e-9          # lambda_mid - lambda_min <= GAP_REL * lambda_max: degenerate
HORIZONTAL = 1e-6       # |n_z| below this: sign and NaN-c variants
MAX_ROWS = 512          # variants per cell before the cell is checked for plausibility only

EXACT, DEGENERATE, PLAUSIBLE = 0, 1, 2


# ------------------------------------------------------------------------------------------------------ preprocessing
def preprocess(pts, cx=0.0, cy=0.0):
    """CropBox [cx-10, cx+10]^2 x [-0.01, 5] (x and y compared in double, z against the float bounds), non-finite points dropped,
    then the 1 cm VoxelGrid: voxel = floor(p * (1 / 0.01f)) in float, one centroid per voxel.  Returns (centroids float64 (n, 3),
    points per voxel (n,), voxel keys (n, 3))."""
    p = np.asarray(pts, np.float32).reshape(-1, 3)
    p = p[np.isfinite(p).all(axis=1)]
    x, y = p[:, 0].astype(np.float64), p[:, 1].astype(np.float64)
    keep = ((x >= cx - 10.0) & (x <= cx + 10.0) & (y >= cy - 10.0) & (y <= cy + 10.0)
            & (p[:, 2] >= np.float32(-0.01)) & (p[:, 2] <= np.float32(5.0)))
    p = p[keep]
    if p.shape[0] == 0:
        return np.zeros((0, 3)), np.zeros(0, np.int64), np.zeros((0, 3), np.int64)
    inv_leaf = np.float32(1.0) / np.float32(0.01)
    keys = np.floor(p * inv_leaf).astype(np.int64)            # float32 product, as the builder's VoxelGrid
    uk, inv, cnt = np.unique(keys, axis=0, return_inverse=True, return_counts=True)
    inv = inv.ravel()
    cen = np.zeros((uk.shape[0], 3))
    np.add.at(cen, inv, p.astype(np.float64))
    return cen / cnt[:, None], cnt, uk


# ------------------------------------------------------------------------------------------------------ constructMap
def _cross(a, b):
    return np.stack([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])


def _flatten(lists):
    lens = np.fromiter(map(len, lists), np.int64, count=len(lists))
    idx = np.fromiter(itertools.chain.from_iterable(lists), np.int64, count=int(lens.sum()))
    return np.repeat(np.arange(len(lists)), lens), idx


class Reference:
    """constructMap + filter over one cloud, which must already be what the builder works on (preprocess(...) of it, or a cloud the
    preprocessing keeps as it is).  build(geom) runs every cell of a grid."""

    def __init__(self, cloud, ellipsoid=(0.2, 0.1, 0.1), iter_num=2):
        self.P = np.asarray(cloud, np.float64).reshape(-1, 3)
        self.e = np.asarray(ellipsoid, np.float64)
        self.box_r = float(self.e.max())             # the radius of the reference's radiusSearch (uneven_map.cpp:319)
        self.iter_num = int(iter_num)
        if self.P.shape[0]:
            self.t2 = cKDTree(self.P[:, :2])
            self.t3 = cKDTree(self.P)

    # one iteration for every row; a row is (cell, state, choices)
    def _step(self, px, py, cy, sy, z, zbx, zby, c, it, snap, surf_in):
        R = px.shape[0]
        xyaw = np.stack([cy, sy, np.zeros(R)])
        zb = np.stack([zbx, zby, c])
        yb = _cross(zb, xyaw)
        nyb = np.sqrt((yb * yb).sum(axis=0))
        yb = np.where(nyb > 0, yb / np.where(nyb > 0, nyb, 1.0), yb)          # Eigen's normalized(): the zero vector stays
        xb = _cross(yb, zb)
        wp = np.stack([px + xb[0] * 0.12, py + xb[1] * 0.12, z.copy()])
        out = dict(tie=np.zeros(R, bool), d0=np.full(R, np.inf), q=None)
        if it == 0 and self.P.shape[0]:
            q = wp[:2].astype(np.float32).astype(np.float64).T                 # the query is a float point (pcl::PointXY)
            k = 2 if self.P.shape[0] > 1 else 1
            d, i = self.t2.query(q, k=k)
            d, i = d.reshape(R, k), i.reshape(R, k)
            d2 = d * d
            wp[2] = np.where(np.isnan(snap), self.P[i[:, 0], 2], snap)
            if k == 2:
                out["tie"] = (d2[:, 1] - d2[:, 0] <= TIE_REL * d2[:, 0]) & np.isnan(snap)
            out["d0"], out["q"] = d[:, 0], q
        # the ellipsoid about wp in the frame (xb, yb, zb); a NaN frame admits no point (NaN < 1 is false)
        ok = np.isfinite(wp).all(axis=0) & np.isfinite(xb).all(axis=0) & np.isfinite(yb).all(axis=0) & np.isfinite(zb).all(axis=0)
        rows = np.nonzero(ok)[0]
        if self.P.shape[0] and rows.size:
            lists = self.t3.query_ball_point(wp[:, rows].T, self.box_r * (1 + 1e-7), return_sorted=False)
            if rows.size == 1:
                lists = [lists] if not isinstance(lists, np.ndarray) else list(lists)
            cell, idx = _flatten(lists)
            cell = rows[cell]
        else:
            cell, idx = np.zeros(0, np.int64), np.zeros(0, np.int64)
        d = self.P[idx].T - wp[:, cell]
        r2 = (((xb[:, cell] * d).sum(axis=0) / self.e[0]) ** 2 + ((yb[:, cell] * d).sum(axis=0) / self.e[1]) ** 2
              + ((zb[:, cell] * d).sum(axis=0) / self.e[2]) ** 2)
        on = np.abs(r2 - 1.0) < SURFACE
        inside = (r2 < 1.0) & ~on | on & surf_in[cell]
        out["surface"] = np.bincount(cell[on], minlength=R) > 0
        cell, idx = cell[inside], idx[inside]
        n = np.bincount(cell, minlength=R).astype(np.float64)
        m = np.stack([np.bincount(cell, self.P[idx, a], minlength=R) for a in range(3)]) / np.maximum(n, 1.0)
        v = self.P[idx].T - m[:, cell]
        cov = np.zeros((R, 3, 3))
        for a in range(3):
            for b in range(a, 3):
                cov[:, a, b] = cov[:, b, a] = np.bincount(cell, v[a] * v[b], minlength=R) / np.maximum(n, 1.0)
        w, V = np.linalg.eigh(cov)
        nn = V[:, :, 0]
        nn = nn / np.sqrt((nn * nn).sum(axis=1))[:, None]
        nn = np.where(nn[:, 2:3] < 0, -nn, nn)
        with np.errstate(invalid="ignore", divide="ignore"):
            sg = 3.0 * w[:, 0] / w.sum(axis=1)
        bad = np.isnan(sg)                                                      # filter's NaN rule (uneven_map.cpp:30-36)
        sg = np.where(bad, 1.0, sg)
        nn = np.where(bad[:, None], np.array([1.0, 0.0, 0.0]), nn)
        empty = n == 0
        out.update(z=np.where(empty, wp[2], m[2]), sigma=np.where(empty, 0.0, sg), zbx=np.where(empty, 0.0, nn[:, 0]),
                   zby=np.where(empty, 0.0, nn[:, 1]), nz=np.where(empty, 1.0, nn[:, 2]), n=n, cov=cov, w=w)
        with np.errstate(invalid="ignore"):
            out["c"] = np.where(empty, 1.0, np.sqrt(1.0 - out["zbx"] ** 2 - out["zby"] ** 2))
        out["degenerate"] = ~empty & ((n == 2) | (n >= 3) & (w[:, 1] - w[:, 0] <= GAP_REL * w[:, 2]))
        out["horizontal"] = ~empty & ~bad & (np.abs(out["nz"]) < HORIZONTAL)
        return out

    def build(self, geom):
        """every cell of `geom` (origin, xy_resolution, yaw_resolution, voxel_num): a dict of rows, each one variant of one cell:
        'cell' (flat index x*Y*W + y*W + w), 'z', 'sigma', 'zbx', 'zby' (float64), 'kind' (EXACT / DEGENERATE / PLAUSIBLE), 'cov',
        'w' (the last eigenproblem, for DEGENERATE rows), 'nanc' (the row took a NaN c after some iteration), and per cell
        'features': counts of what the grid exercised."""
        X, Y, W = (int(v) for v in geom.voxel_num)
        N = X * Y * W
        cell = np.arange(N)
        xi, yi, wi = cell // (Y * W), (cell // W) % Y, cell % W
        px = (xi + 0.5) * geom.xy_resolution + geom.origin[0]
        py = (yi + 0.5) * geom.xy_resolution + geom.origin[1]
        yaw = (wi + 0.5) * geom.yaw_resolution + geom.origin[2]
        cyaw, syaw = np.cos(yaw), np.sin(yaw)
        st = dict(cell=cell, z=np.zeros(N), zbx=np.zeros(N), zby=np.zeros(N), c=np.ones(N), sigma=np.zeros(N),
                  kind=np.zeros(N, np.int8), nanc=np.zeros(N, bool), cov=np.zeros((N, 3, 3)), w=np.zeros((N, 3)))
        feat = dict(cells=N)
        for it in range(self.iter_num):
            last = it == self.iter_num - 1
            act = st["kind"] == EXACT
            R = st["cell"]
            snap = np.full(R.size, np.nan)
            surf_in = np.zeros(R.size, bool)
            o = self._step(px[R], py[R], cyaw[R], syaw[R], st["z"], st["zbx"], st["zby"], st["c"], it, snap, surf_in)
            add = []
            if it == 0 and o["q"] is not None:
                feat["clamped_queries"] = int(((o["q"][:, 0] < self.P[:, 0].min()) | (o["q"][:, 0] > self.P[:, 0].max())
                                               | (o["q"][:, 1] < self.P[:, 1].min()) | (o["q"][:, 1] > self.P[:, 1].max())).sum())
                feat["far_nearest"] = int((o["d0"] > 3 * self.box_r).sum())
                feat["ties"] = int(o["tie"].sum())
                for r in np.nonzero(o["tie"] & act)[0]:            # one row per candidate z
                    cand = self.t2.query_ball_point(o["q"][r], o["d0"][r] * np.sqrt(1 + TIE_REL) * (1 + 1e-12))
                    for zc in np.unique(self.P[cand, 2]):
                        add.append((r, zc, False))
            for r in np.nonzero(o["surface"] & act)[0]:              # one row with the surface points inside
                add.append((r, np.nan, True))
            if add:                                                 # the variants re-run this iteration from the same state
                rr = np.array([a[0] for a in add])
                c2 = st["cell"][rr]
                o2 = self._step(px[c2], py[c2], cyaw[c2], syaw[c2], st["z"][rr], st["zbx"][rr], st["zby"][rr], st["c"][rr], it,
                                np.array([a[1] for a in add]), np.array([a[2] for a in add]))
                st = {k: np.concatenate([v, v[rr]]) for k, v in st.items()}
                o = {k: (np.concatenate([v, o2[k]]) if isinstance(v, np.ndarray) and v.shape[:1] == (R.size,) else v) for k, v in o.items()}
            act = st["kind"] == EXACT
            new = dict(st)
            for k in ("z", "sigma", "zbx", "zby", "c", "cov", "w"):
                new[k] = np.where(act.reshape((-1,) + (1,) * (o[k].ndim - 1)), o[k], st[k])
            kind = st["kind"].copy()
            kind[act & o["degenerate"]] = DEGENERATE if last else PLAUSIBLE
            new["kind"] = kind
            cells_with = lambda m: int(np.unique(st["cell"][m]).size)          # features count cells, not variants
            if it == 0:
                feat["n1"] = cells_with(act & (o["n"] == 1))
            feat["empty_it%d" % it] = cells_with(act & (o["n"] == 0))
            feat["degenerate_it%d" % it] = cells_with(act & o["degenerate"])
            feat["nanc_it%d" % it] = cells_with(act & np.isnan(o["c"]))
            # horizontal normals: both signs where n_z is 0 up to rounding; before the last iteration also c NaN
            hz = act & o["horizontal"] & ~o["degenerate"]
            flip = hz & (np.abs(o["nz"]) < 1e-12)
            nanc = hz & (np.abs(o["nz"]) < 1e-7) & (not last)
            new["c"] = np.where(hz, np.sqrt(np.maximum(0.0, 1.0 - new["zbx"] ** 2 - new["zby"] ** 2)), new["c"])
            parts = []
            for sgn, cnan, sel in ((-1.0, False, flip), (1.0, True, nanc), (-1.0, True, flip & nanc)):
                h = np.nonzero(sel)[0]
                if h.size:
                    part = {k: v[h].copy() for k, v in new.items()}
                    part["zbx"] *= sgn
                    part["zby"] *= sgn
                    if cnan:
                        part["c"][:] = np.nan
                        part["nanc"][:] = True
                    parts.append(part)
            new = {k: np.concatenate([new[k]] + [p[k] for p in parts]) for k in new}
            st = new
            # a cell with too many variants is checked for plausibility only
            cnt = np.bincount(st["cell"], minlength=N)
            many = cnt[st["cell"]] > MAX_ROWS
            if many.any():
                st["kind"][many] = PLAUSIBLE
                first = np.ones(st["cell"].size, bool)
                first[many] = False
                _, fi = np.unique(st["cell"][many], return_index=True)
                first[np.nonzero(many)[0][fi]] = True
                st = {k: v[first] for k, v in st.items()}
        # one row per distinct variant
        key = np.stack([st["cell"], st["kind"], st["z"], st["sigma"], st["zbx"], st["zby"]]).T
        _, keep = np.unique(key, axis=0, return_index=True)
        st = {k: v[np.sort(keep)] for k, v in st.items()}
        cnt = np.bincount(st["cell"], minlength=N)
        amb = (cnt > 1) | (np.bincount(st["cell"], st["kind"] != EXACT, minlength=N) > 0)
        feat["ambiguous"] = int(amb.sum())
        feat["plausible_only"] = int((np.bincount(st["cell"], st["kind"] == PLAUSIBLE, minlength=N) > 0).sum())
        st["features"] = feat
        st["ambiguous"] = amb
        st["zrange"] = (self.P[:, 2].min(), self.P[:, 2].max()) if self.P.shape[0] else (0.0, 0.0)
        return st


# ------------------------------------------------------------------------------------------------------ comparison
def ulp32(x):
    """spacing of float32 at float32(x)"""
    return np.spacing(np.abs(np.asarray(x, np.float64).astype(np.float32))).astype(np.float64)


# absolute floors below which values are equal: sigma where lambda_min is rounding noise; z and zb where the exact value is 0
SIGMA_ABS = 1e-9
VALUE_ABS = 1e-12


def row_matches(rows, cells):
    """per row: does the builder's float32 cell (cells[X, Y, W, 4] flattened) match this variant?"""
    b = np.asarray(cells, np.float32).reshape(-1, 4)[rows["cell"]].astype(np.float64)
    kind = rows["kind"]
    close = np.ones(kind.size, bool)
    for j, k in ((0, "z"), (2, "zbx"), (3, "zby")):
        close &= np.abs(b[:, j] - rows[k].astype(np.float32)) <= ulp32(rows[k]) + VALUE_ABS
    sig_ok = np.abs(b[:, 1] - rows["sigma"].astype(np.float32)) <= np.maximum(ulp32(rows["sigma"]), SIGMA_ABS)
    exact = close & sig_ok
    # degenerate: z and sigma as computed, the normal any unit vector of the smallest eigenspace
    nb = np.stack([b[:, 2], b[:, 3], np.sqrt(np.maximum(0.0, 1.0 - b[:, 2] ** 2 - b[:, 3] ** 2))], axis=1)
    rq = np.einsum("ri,rij,rj->r", nb, rows["cov"], nb)
    w = rows["w"]
    in_space = rq <= w[:, 1] + 1e-6 * np.abs(w[:, 2]) + 1e-15
    unit = b[:, 2] ** 2 + b[:, 3] ** 2 <= 1.0 + 1e-6
    zok = np.abs(b[:, 0] - rows["z"].astype(np.float32)) <= ulp32(rows["z"]) + VALUE_ABS
    degen = zok & sig_ok & in_space & unit
    lo, hi = rows["zrange"]
    plaus = np.isfinite(b).all(axis=1) & (b[:, 0] >= np.float32(lo)) & (b[:, 0] <= np.float32(hi)) & (b[:, 1] >= -1e-6) & (b[:, 1] <= 1 + 1e-6) & unit
    return np.where(kind == EXACT, exact, np.where(kind == DEGENERATE, degen, plaus))


def compare(rows, cells):
    """(cells matched by none of their variants (flat indices), cells matched only by a variant that took a NaN c, the builder's
    largest deviation on unambiguous cells in float ulps for z, zbx, zby and sigma, absolute where the value is below 1e-6)"""
    N = int(np.prod(np.asarray(cells).shape[:3]))
    m = row_matches(rows, cells)
    ok = np.bincount(rows["cell"], m, minlength=N) > 0
    nanc_only = np.nonzero(ok & ~(np.bincount(rows["cell"], m & ~rows["nanc"], minlength=N) > 0))[0]
    b = np.asarray(cells, np.float32).reshape(-1, 4).astype(np.float64)
    una = ~rows["ambiguous"][rows["cell"]] & (rows["kind"] == EXACT)
    c = rows["cell"][una]
    dev = {}
    for j, k in ((0, "z"), (1, "sigma"), (2, "zbx"), (3, "zby")):
        r = rows[k][una]
        d = np.abs(b[c, j] - r.astype(np.float32))
        big = np.abs(r) > 1e-6
        dev[k + "_ulp"] = float((d[big] / ulp32(r[big])).max()) if big.any() else 0.0
        dev[k + "_abs_small"] = float(d[~big].max()) if (~big).any() else 0.0
    return np.nonzero(~ok)[0], nanc_only, dev
