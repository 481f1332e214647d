// replan_oracle.cpp -- the CPU reference of ualm_submit_replan's build (include/ualm.h): the state at t_from and the (x, y, yaw) points of
// the trajectory by the oracle's own durations and evaluation (traj_duration, se2_eval: oracle/oracle.cpp, included unmodified), and
// PlanManager's resampler (plan_manager.cpp:62-122) restated here on its own.  TEST INFRASTRUCTURE ONLY, built by tests/replan_oracle.py.
#include "../oracle/oracle.cpp"

#include <vector>

// the replan build's bound (include/ualm.h, ualm_submit_replan): a polyline that needs more than 4095 waypoints of either kind, a yaw of
// magnitude 2^40 or more, or more than 65536 whole turns of smoothing in all is cut short: N' = M' = 4097, total_time from its whole length
static const long long MAX_WAYPOINTS = 4095;
static const double MAX_YAW = 1099511627776.0, MAX_TURNS = 65536.0;

// pm.cpp:62-77 then 96-122 over a whole polyline; waypoints past cap_xy / cap_yaw are counted, not written.  bounded: the replan
// build's bound above (*cut set when it applies); otherwise none, as ualm_resample_path
extern "C" void orc_resample(const double *path_in, int npts, double piece_len, double yaw_piece_times, double mean_vel, double init_time_times,
                             double *inner_xy, long long cap_xy, double *inner_yaw, long long cap_yaw, long long *N, long long *M, double *total_time,
                             double *smoothed, int bounded, int *cut_out)
{
    std::vector<double> p(path_in, path_in + 3 * (size_t)npts);
    bool cut = false;
    double turns = 0.0;
    for (int i = 0; i + 1 < npts; i++) {
        if (bounded) {
            const double a = p[3 * i + 2], b = p[3 * (i + 1) + 2];
            if (!(std::fabs(a) < MAX_YAW && std::fabs(b) < MAX_YAW)) { cut = true; break; }
            const double need = std::floor(std::fabs(b - a) / (M_PI * 2)) + 1.0;
            if (turns + need > MAX_TURNS) { cut = true; break; }
            turns += need;
        }
        double dyaw = p[3 * (i + 1) + 2] - p[3 * i + 2];
        while (dyaw >= M_PI / 2) { p[3 * (i + 1) + 2] -= M_PI * 2; dyaw = p[3 * (i + 1) + 2] - p[3 * i + 2]; }
        while (dyaw <= -M_PI / 2) { p[3 * (i + 1) + 2] += M_PI * 2; dyaw = p[3 * (i + 1) + 2] - p[3 * i + 2]; }
    }
    if (smoothed) for (size_t q = 0; q < p.size(); q++) smoothed[q] = p[q];
    double temp_len_yaw = 0.0, temp_len_pos = 0.0, total_len = 0.0;
    const double piece_len_yaw = piece_len / yaw_piece_times;
    long long nxy = 0, nyaw = 0;
    for (int k = 0; k + 1 < npts; k++) {
        const double *a = &p[3 * k], *b = &p[3 * (k + 1)];
        const double temp_seg = std::sqrt((b[0] - a[0]) * (b[0] - a[0]) + (b[1] - a[1]) * (b[1] - a[1]));
        temp_len_yaw += temp_seg; temp_len_pos += temp_seg; total_len += temp_seg;
        if (cut) continue;                               // lengths only
        while (temp_len_yaw > piece_len_yaw) {
            if (bounded && nyaw >= MAX_WAYPOINTS) { cut = true; break; }
            if (nyaw < cap_yaw) inner_yaw[nyaw] = a[2] + (1.0 - (temp_len_yaw - piece_len_yaw) / temp_seg) * (b[2] - a[2]);
            nyaw++;
            temp_len_yaw -= piece_len_yaw;
        }
        while (!cut && temp_len_pos > piece_len) {
            if (bounded && nxy >= MAX_WAYPOINTS) { cut = true; break; }
            const double w = (1.0 - (temp_len_pos - piece_len) / temp_seg);
            if (nxy < cap_xy) { inner_xy[2 * nxy] = a[0] + w * (b[0] - a[0]); inner_xy[2 * nxy + 1] = a[1] + w * (b[1] - a[1]); }
            nxy++;
            temp_len_pos -= piece_len;
        }
    }
    *total_time = total_len / mean_vel * init_time_times;
    *N = cut ? MAX_WAYPOINTS + 2 : nxy + 1;
    *M = cut ? MAX_WAYPOINTS + 2 : nyaw + 1;
    if (cut_out) *cut_out = cut ? 1 : 0;
}

// The polyline of the build: the point at t_from, the points at t_from < t < duration of t = 0, dt, 2dt.. (repeated addition), the goal
// (bnd's end position and end angle).  Returns its number of points; writes them as (x, y, yaw) and their times (the goal: -1) when
// path / times are not null and hold `cap` points.  head9 (optional) = [px, py, vx, vy, ax, ay, yaw, dyaw, ddyaw] at t_from
extern "C" long long orc_replan_polyline(int N, int M, const double *c_xy, const double *c_yaw, double T_xy, double T_yaw, const double *bnd,
                                         double t_from, double dt, double *path, double *times, long long cap, double *head9)
{
    const double total = traj_duration(N, M, T_xy, T_yaw);
    long long n = 0;
    auto put = [&](double x, double y, double yaw, double t) {
        if (path && n < cap) { path[3 * n] = x; path[3 * n + 1] = y; path[3 * n + 2] = yaw; }
        if (times && n < cap) times[n] = t;
        n++;
    };
    const SE2State h = se2_eval(N, M, c_xy, c_yaw, T_xy, T_yaw, t_from);
    if (head9) {
        const double v[9] = {h.x, h.y, h.vx, h.vy, h.ax, h.ay, h.yaw, h.dyaw, h.ddyaw};
        for (int q = 0; q < 9; q++) head9[q] = v[q];
    }
    put(h.x, h.y, h.yaw, t_from);
    for (double t = 0.0; t < total; t += dt) {
        if (!(t > t_from)) continue;
        const SE2State e = se2_eval(N, M, c_xy, c_yaw, T_xy, T_yaw, t);
        put(e.x, e.y, e.yaw, t);
    }
    put(bnd[6], bnd[7], bnd[15], -1.0);
    return n;
}

// One row of the build: out = bnd' (18) | total_time | N' | M' | inner xy (cap_xy points, zeros past them) | inner yaw (cap_yaw);
// a row over the caps keeps its counts and zero inner points.  rp4 = piece_len, yaw_piece_times, mean_vel, init_time_times
extern "C" void orc_replan(int N, int M, const double *c_xy, const double *c_yaw, double T_xy, double T_yaw, const double *bnd, double t_from,
                           double dt, const double *rp4, int cap_xy, int cap_yaw, double *out)
{
    const long long n = orc_replan_polyline(N, M, c_xy, c_yaw, T_xy, T_yaw, bnd, t_from, dt, nullptr, nullptr, 0, nullptr);
    std::vector<double> path(3 * (size_t)n);
    double head[9];
    orc_replan_polyline(N, M, c_xy, c_yaw, T_xy, T_yaw, bnd, t_from, dt, path.data(), nullptr, n, head);
    double *ixy = out + 21, *iyaw = ixy + 2 * (size_t)cap_xy;
    for (int q = 0; q < 2 * cap_xy + cap_yaw; q++) ixy[q] = 0.0;
    long long Nn, Mn;
    orc_resample(path.data(), (int)n, rp4[0], rp4[1], rp4[2], rp4[3], ixy, cap_xy, iyaw, cap_yaw, &Nn, &Mn, &out[18], nullptr, 1, nullptr);
    if (Nn - 1 > cap_xy || Mn - 1 > cap_yaw) for (int q = 0; q < 2 * cap_xy + cap_yaw; q++) ixy[q] = 0.0;
    const double b2[18] = {head[0], head[1], head[2], head[3], head[4], head[5], bnd[6], bnd[7], bnd[8], bnd[9], bnd[10], bnd[11],
                           head[6], head[7], head[8], bnd[15], bnd[16], bnd[17]};
    for (int q = 0; q < 18; q++) out[q] = b2[q];
    out[19] = (double)Nn; out[20] = (double)Mn;
}
