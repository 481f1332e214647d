// host_tools.cpp -- host-side input pipeline of the batched optimizer (no GPU code here).
//
//  * ualm_map_geometry / ualm_map_build / ualm_map_occupancy : the UnevenMap the optimizer queries, built from
//    a point cloud the way UnevenMap::init + constructMap + filter do it
//    (uneven_map/src/uneven_map.cpp:96-114, 127-163, 169-179, 317-398, 5-43), with a bin-grid neighbour search
//    on host threads instead of PCL kd-trees and a Jacobi 3x3 eigen-solver instead of Eigen::EigenSolver; the per-cell
//    arithmetic lives in map_cell.h and is shared with the CUDA builder (ualm_map_build_device).
//  * ualm_dubins_path : initial (x,y,yaw) polyline standing in for KinoAstar::plan (front_end/src/kino_astar.cpp:67-236);
//    the reference's own one-shot expansion is this Dubins family (front_end/include/front_end/kino_astar.h:242-258).
//  * ualm_resample_path : the PlanManager input contract (plan_manager/src/plan_manager.cpp:62-122).
//
// Written from the behaviour of those files; shares no code with them.
#include "ualm.h"
#include "map_prep.h"
#include "resample_stream.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

extern "C" void ualm_default_params(ualm_params_t *p)
{
    // plan_manager/params/run_hill.yaml:30-55, uneven_map gravity :13
    p->rho_T = 100000.0; p->rho_ter = 10.0; p->max_vel = 0.5; p->max_acc_lon = 5.0; p->max_acc_lat = 10.0;
    p->max_kap = 2.1; p->min_cxi = 0.8; p->max_sig = 0.05; p->use_scaling = 1; p->rho = 1.0; p->beta = 1000.0;
    p->gamma = 1.0; p->epsilon_con = 0.001; p->max_iter = 10; p->g_epsilon = 1.0e-3; p->min_step = 1.0e-32;
    p->inner_max_iter = 10000; p->delta = 1.0e-4; p->mem_size = 256; p->past = 3; p->int_K = 16; p->gravity = 9.81;
}

extern "C" void ualm_map_geometry(double sx, double sy, double xy_res, double yaw_res, ualm_map_geom_t *g)
{
    // uneven_map.cpp:96-114
    double size[3] = {sx, sy, 2.0 * M_PI + 5e-2};
    for (int k = 0; k < 3; k++) {
        g->origin[k] = -size[k] / 2.0;
        g->max_boundary[k] = size[k] / 2.0;
    }
    g->xy_resolution = xy_res;
    g->yaw_resolution = yaw_res;
    g->voxel_num[0] = (int)std::ceil(size[0] / xy_res);
    g->voxel_num[1] = (int)std::ceil(size[1] / xy_res);
    g->voxel_num[2] = (int)std::ceil(size[2] / yaw_res);
}

extern "C" void ualm_map_geometry_at(double sx, double sy, double xy_res, double yaw_res, double cx, double cy, ualm_map_geom_t *g)
{
    ualm_map_geometry(sx, sy, xy_res, yaw_res, g);
    const double c[2] = {cx, cy}, size[2] = {sx, sy};
    for (int k = 0; k < 2; k++) {
        g->origin[k] = c[k] - size[k] / 2.0;        // c = 0: -size / 2, ualm_map_geometry's value
        g->max_boundary[k] = c[k] + size[k] / 2.0;
    }
}

namespace {
struct P3 { float x, y, z; };
} // namespace

void ualm_map_preprocess(const float *pin, int64_t npts, double ex, double ey, double ez, double cx, double cy, UalmMapHostPrep &out)
{
    // ---- CropBox [cx-10,cx+10]x[cy-10,cy+10]x[-0.01,5]  (uneven_map.cpp:133-137, whose box is about the world origin: c = 0 there,
    // where the double bounds are the reference's float bounds exactly)
    const double xlo = cx - 10.0, xhi = cx + 10.0, ylo = cy - 10.0, yhi = cy + 10.0;
    std::vector<P3> crop;
    crop.reserve((size_t)npts);
    for (int64_t i = 0; i < npts; i++) {
        P3 p{pin[3 * i], pin[3 * i + 1], pin[3 * i + 2]};
        if (!(std::isfinite(p.x) && std::isfinite(p.y) && std::isfinite(p.z))) continue;
        if (p.x < xlo || p.x > xhi || p.y < ylo || p.y > yhi || p.z < -0.01f || p.z > 5.0f) continue;
        crop.push_back(p);
    }
    // ---- VoxelGrid, leaf 1 cm: centroid of the points of each voxel (uneven_map.cpp:140-143)
    std::vector<P3> cloud;
    {
        const float inv_leaf = 1.0f / 0.01f;
        float mn[3] = {1e30f, 1e30f, 1e30f}, mx[3] = {-1e30f, -1e30f, -1e30f};
        for (auto &p : crop) { mn[0] = std::min(mn[0], p.x); mn[1] = std::min(mn[1], p.y); mn[2] = std::min(mn[2], p.z); mx[0] = std::max(mx[0], p.x); mx[1] = std::max(mx[1], p.y); mx[2] = std::max(mx[2], p.z); }
        int64_t minb[3], divb[3];
        for (int k = 0; k < 3; k++) { minb[k] = (int64_t)std::floor(mn[k] * inv_leaf); divb[k] = (int64_t)std::floor(mx[k] * inv_leaf) - minb[k] + 1; }
        std::vector<std::pair<int64_t, int>> keyed(crop.size());
        for (size_t i = 0; i < crop.size(); i++) {
            int64_t a = (int64_t)std::floor(crop[i].x * inv_leaf) - minb[0];
            int64_t b = (int64_t)std::floor(crop[i].y * inv_leaf) - minb[1];
            int64_t c = (int64_t)std::floor(crop[i].z * inv_leaf) - minb[2];
            keyed[i] = {a + b * divb[0] + c * divb[0] * divb[1], (int)i};
        }
        std::sort(keyed.begin(), keyed.end());
        for (size_t i = 0; i < keyed.size();) {
            size_t j = i;
            float sx = 0, sy = 0, sz = 0;
            while (j < keyed.size() && keyed[j].first == keyed[i].first) { const P3 &p = crop[keyed[j].second]; sx += p.x; sy += p.y; sz += p.z; j++; }
            float n = (float)(j - i);
            cloud.push_back(P3{sx / n, sy / n, sz / n});
            i = j;
        }
    }
    // ---- uniform XY bin grid, bin = the search radius of constructMap (uneven_map.cpp:319)
    const double bin = std::max(std::max(ex, ey), ez);
    double xmin = 1e30, ymin = 1e30, xmax = -1e30, ymax = -1e30;
    for (auto &p : cloud) { xmin = std::min<double>(xmin, p.x); xmax = std::max<double>(xmax, p.x); ymin = std::min<double>(ymin, p.y); ymax = std::max<double>(ymax, p.y); }
    if (cloud.empty()) { xmin = ymin = 0; xmax = ymax = 1; }
    out.box_r = bin; out.x0 = xmin; out.y0 = ymin; out.inv = 1.0 / bin;
    out.nx = (int)((xmax - xmin) * out.inv) + 1; out.ny = (int)((ymax - ymin) * out.inv) + 1;
    out.start.assign((size_t)out.nx * out.ny + 1, 0);
    auto key = [&](const P3 &p) {
        int bx = std::min(out.nx - 1, std::max(0, (int)((p.x - out.x0) * out.inv)));
        int by = std::min(out.ny - 1, std::max(0, (int)((p.y - out.y0) * out.inv)));
        return bx * out.ny + by;
    };
    for (auto &p : cloud) out.start[key(p) + 1]++;
    for (size_t i = 1; i < out.start.size(); i++) out.start[i] += out.start[i - 1];
    out.pts.resize(3 * cloud.size());
    std::vector<int> fill(out.start.begin(), out.start.end() - 1);
    for (auto &p : cloud) { const int q = fill[key(p)]++; out.pts[3 * q] = p.x; out.pts[3 * q + 1] = p.y; out.pts[3 * q + 2] = p.z; }
}

extern "C" int64_t ualm_map_preprocess_cloud(const float *pin, int64_t npts, double ex, double ey, double ez, float *pts_out, int64_t max_pts)
{
    if (!pin || npts < 0) return UALM_EINVAL;
    UalmMapHostPrep prep;
    ualm_map_preprocess(pin, npts, ex, ey, ez, 0.0, 0.0, prep);      // the crop of a grid centred at the world origin
    const int64_t n = (int64_t)(prep.pts.size() / 3);
    if (pts_out) {
        if (n > max_pts) return UALM_ELIMIT;
        std::copy(prep.pts.begin(), prep.pts.end(), pts_out);
    }
    return n;
}

extern "C" int ualm_map_build(const float *pin, int64_t npts, const ualm_map_geom_t *g, double ex, double ey,
                              double ez, int iter_num, int nthreads, float *cells)
{
    if (!pin || !g || !cells || npts < 0) return UALM_EINVAL;
    UalmMapHostPrep prep;
    ualm_map_preprocess(pin, npts, ex, ey, ez, ualm_map_centre(*g, 0), ualm_map_centre(*g, 1), prep);
    const UalmMapPrep view = prep.view(ex, ey, ez, iter_num);
    const int X = g->voxel_num[0], Y = g->voxel_num[1], W = g->voxel_num[2];
    if (nthreads <= 0) nthreads = (int)std::max(1u, std::thread::hardware_concurrency());
    std::atomic<int> next_x(0);
    auto worker = [&]() {
        while (true) {
            const int x = next_x.fetch_add(1);
            if (x >= X) break;
            for (int y = 0; y < Y; y++)
                for (int w = 0; w < W; w++) ualm_map_cell(view, *g, x, y, w, cells + 4 * ((size_t)x * Y * W + (size_t)y * W + w));   // map_cell.h
        }
    };
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; t++) th.emplace_back(worker);
    for (auto &t : th) t.join();
    return UALM_OK;
}

extern "C" int ualm_map_occupancy(const float *cells, const ualm_map_geom_t *g, double min_cnormal, double max_rho,
                                  uint8_t *occ3, uint8_t *occ2)
{
    if (!cells || !g) return UALM_EINVAL;
    const int X = g->voxel_num[0], Y = g->voxel_num[1], W = g->voxel_num[2];
    if (occ2) std::memset(occ2, 0, (size_t)X * Y);
    for (int x = 0; x < X; x++)
        for (int y = 0; y < Y; y++)
            for (int w = 0; w < W; w++) {
                size_t a = (size_t)x * Y * W + (size_t)y * W + w;
                const double zbx = cells[4 * a + 2], zby = cells[4 * a + 3];
                const double c = std::sqrt(1.0 - zbx * zbx - zby * zby);
                // the reference's rule as written (uneven_map.cpp:174): a NaN c (zb rounded to just over unit length) compares false
                // and is NOT flagged by the first term
                const bool occ = c < min_cnormal || cells[4 * a + 1] > max_rho;
                if (occ3) occ3[a] = occ;
                if (occ && occ2) occ2[(size_t)x * Y + y] = 1;
            }
    return UALM_OK;
}

// ------------------------------------------------------------------------------------------------
// Dubins shortest path (forward only)
// ------------------------------------------------------------------------------------------------
namespace {
static inline double mod2pi(double a)
{
    a = std::fmod(a, 2.0 * M_PI);
    if (a < 0) a += 2.0 * M_PI;
    return a;
}
// segment types: 0 = L, 1 = S, 2 = R
struct DubinsSol { double t, p, q; int ty[3]; double len; bool ok; };
} // namespace

extern "C" int ualm_dubins_path(const double start[3], const double goal[3], double radius, double ds, double *out,
                                int max_pts)
{
    if (!start || !goal || !out || radius <= 0 || ds <= 0 || max_pts < 2) return UALM_EINVAL;
    const double dx = goal[0] - start[0], dy = goal[1] - start[1];
    const double D = std::sqrt(dx * dx + dy * dy), d = D / radius;
    const double phi = std::atan2(dy, dx);
    const double a = mod2pi(start[2] - phi), b = mod2pi(goal[2] - phi);
    const double sa = std::sin(a), sb = std::sin(b), ca = std::cos(a), cb = std::cos(b), cab = std::cos(a - b);
    DubinsSol best{0, 0, 0, {0, 0, 0}, 1e300, false};
    auto consider = [&](double t, double p, double q, int t0, int t1, int t2) {
        double L = t + p + q;
        if (L < best.len) best = DubinsSol{t, p, q, {t0, t1, t2}, L, true};
    };
    { // LSL
        double tmp = 2 + d * d - 2 * cab + 2 * d * (sa - sb);
        if (tmp >= 0) { double th = std::atan2(cb - ca, d + sa - sb); consider(mod2pi(-a + th), std::sqrt(tmp), mod2pi(b - th), 0, 1, 0); }
    }
    { // RSR
        double tmp = 2 + d * d - 2 * cab + 2 * d * (sb - sa);
        if (tmp >= 0) { double th = std::atan2(ca - cb, d - sa + sb); consider(mod2pi(a - th), std::sqrt(tmp), mod2pi(-b + th), 2, 1, 2); }
    }
    { // LSR
        double tmp = -2 + d * d + 2 * cab + 2 * d * (sa + sb);
        if (tmp >= 0) { double p = std::sqrt(tmp); double th = std::atan2(-ca - cb, d + sa + sb) - std::atan2(-2.0, p); consider(mod2pi(-a + th), p, mod2pi(-mod2pi(b) + th), 0, 1, 2); }
    }
    { // RSL
        double tmp = d * d - 2 + 2 * cab - 2 * d * (sa + sb);
        if (tmp >= 0) { double p = std::sqrt(tmp); double th = std::atan2(ca + cb, d - sa - sb) - std::atan2(2.0, p); consider(mod2pi(a - th), p, mod2pi(b - th), 2, 1, 0); }
    }
    { // RLR
        double tmp = (6 - d * d + 2 * cab + 2 * d * (sa - sb)) / 8;
        if (std::fabs(tmp) <= 1) { double p = mod2pi(2 * M_PI - std::acos(tmp)); double t = mod2pi(a - std::atan2(ca - cb, d - sa + sb) + p / 2); consider(t, p, mod2pi(a - b - t + p), 2, 0, 2); }
    }
    { // LRL
        double tmp = (6 - d * d + 2 * cab + 2 * d * (sb - sa)) / 8;
        if (std::fabs(tmp) <= 1) { double p = mod2pi(2 * M_PI - std::acos(tmp)); double t = mod2pi(-a - std::atan2(ca - cb, d + sa - sb) + p / 2); consider(t, p, mod2pi(mod2pi(b) - a - t + p), 0, 2, 0); }
    }
    if (!best.ok) return UALM_EINVAL;
    const double seg[3] = {best.t, best.p, best.q};
    const double total = best.len * radius;
    // sample l = 0, ds, 2ds, ... <= total (kino_astar.h:252-257 samples the one-shot the same way)
    int n = 0;
    for (double l = 0.0; l <= total; l += ds) {
        if (n >= max_pts) return UALM_ELIMIT;
        double rem = l / radius; // normalized arc length
        double x = 0, y = 0, th = start[2];
        for (int k = 0; k < 3 && rem > 0; k++) {
            double u = std::min(rem, seg[k]);
            if (best.ty[k] == 1) { x += u * std::cos(th); y += u * std::sin(th); }
            else if (best.ty[k] == 0) { x += std::sin(th + u) - std::sin(th); y += -std::cos(th + u) + std::cos(th); th += u; }
            else { x += -std::sin(th - u) + std::sin(th); y += std::cos(th - u) - std::cos(th); th -= u; }
            rem -= u;
        }
        out[3 * n] = start[0] + x * radius; out[3 * n + 1] = start[1] + y * radius;
        double yaw = th;
        while (yaw > M_PI) yaw -= 2 * M_PI; // KinoAstar states carry normalised yaw (kino_astar.h:197-205)
        while (yaw < -M_PI) yaw += 2 * M_PI;
        out[3 * n + 2] = yaw;
        n++;
    }
    // the goal itself terminates the polyline (retrievePath appends the shot path ending at the goal state)
    if (n < max_pts) {
        double lx = out[3 * (n - 1)] - goal[0], ly = out[3 * (n - 1) + 1] - goal[1];
        if (lx * lx + ly * ly > 1e-12) {
            out[3 * n] = goal[0]; out[3 * n + 1] = goal[1];
            double yaw = goal[2];
            while (yaw > M_PI) yaw -= 2 * M_PI;
            while (yaw < -M_PI) yaw += 2 * M_PI;
            out[3 * n + 2] = yaw;
            n++;
        }
    }
    return n;
}

// ------------------------------------------------------------------------------------------------
// PlanManager::rcvWpsCallBack input contract (plan_manager/src/plan_manager.cpp:62-122)
// ------------------------------------------------------------------------------------------------
extern "C" int ualm_resample_path(const double *path_in, int npts, double piece_len, double yaw_piece_times,
                                  double mean_vel, double init_time_times, double init_sig_vel, double *bnd,
                                  double *inner_xy, int max_inner_xy, double *inner_yaw, int max_inner_yaw, int32_t *N,
                                  int32_t *M, double *total_time)
{
    if (!path_in || npts < 2 || !bnd || !inner_xy || !inner_yaw || !N || !M || !total_time) return UALM_EINVAL;
    std::vector<double> p(path_in, path_in + 3 * (size_t)npts);
    // smooth yaw (pm.cpp:62-77); the steps of resample_stream.h, which replan_kernel takes one point at a time
    for (int i = 0; i < npts - 1; i++) ualm_rs_smooth(p[3 * i + 2], p[3 * (i + 1) + 2]);
    // boundary states (pm.cpp:80-94): 2x3 column-major [p | v | a], yaw [psi,0,0]
    const double *f = &p[0], *l = &p[3 * (size_t)(npts - 1)];
    // sin / cos from ualm_detmath.h like every other trig call of the path (so the reference build of tests/test_ref_pin.py, whose
    // trig is redirected to the same functions, produces bit-identical boundary states)
    bnd[0] = f[0]; bnd[1] = f[1]; bnd[2] = init_sig_vel * ualm_cos(f[2]); bnd[3] = init_sig_vel * ualm_sin(f[2]); bnd[4] = 0; bnd[5] = 0;
    bnd[6] = l[0]; bnd[7] = l[1]; bnd[8] = init_sig_vel * ualm_cos(l[2]); bnd[9] = init_sig_vel * ualm_sin(l[2]); bnd[10] = 0; bnd[11] = 0;
    bnd[12] = f[2]; bnd[13] = 0; bnd[14] = 0;
    bnd[15] = l[2]; bnd[16] = 0; bnd[17] = 0;
    // arc-length resampling (pm.cpp:96-121)
    UalmResampleStream s;
    ualm_rs_init(s, piece_len, yaw_piece_times);
    for (int k = 0; k < npts - 1; k++)
        if (!ualm_rs_segment(s, &p[3 * k], &p[3 * (k + 1)], inner_xy, max_inner_xy, inner_yaw, max_inner_yaw, true, 0)) return UALM_ELIMIT;
    *total_time = ualm_rs_total_time(s, mean_vel, init_time_times); // pm.cpp:122
    *N = (int32_t)(s.nxy + 1);
    *M = (int32_t)(s.nyaw + 1);
    return UALM_OK;
}
