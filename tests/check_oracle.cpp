// check_oracle.cpp -- the CPU reference of ualm_check_trajectories (include/ualm.h): orc_feasibility's loop (oracle/oracle.cpp, included
// unmodified so the sample values are its code) restricted to the samples t >= t_from of the full sequence t = 0, dt, 2dt.., with the
// time of the first kept sample that breaks each of six limits.  TEST INFRASTRUCTURE ONLY, built by tests/check_oracle.py.
//
//   out16 = {max_vx, max_ax, max_ay, max_cur, max_att, max_sig, nonhol_error, kept samples, T_xy, T_yaw, first |vx| > max_vel,
//            |ax| > max_acc_lon, |ay| > max_acc_lat, |cur| > max_kap, att > -min_cxi, sig > max_sig (-1: none)}
//   trace (optional): 9 doubles per sample of the full sequence {t, vx, ax, ay, cur, att, sig, nonhol term, kept}
#include "../oracle/oracle.cpp"

extern "C" void orc_check(const orc_map_t *map, double gravity, int N, int M, const double *c_xy, const double *c_yaw, double T_xy, double T_yaw,
                          double dt, double t_from, const double lim[6], double *out16, double *trace)
{
    MapQ<double> mq(*map);
    const int nx = 6 * N;
    double tot_xy = 0.0, tot_yaw = 0.0;
    for (int i = 0; i < N; i++) tot_xy += T_xy;
    for (int i = 0; i < M; i++) tot_yaw += T_yaw;
    const double total = std::min(tot_xy, tot_yaw);
    for (int q = 0; q < 16; q++) out16[q] = q >= 10 ? -1.0 : 0.0;
    out16[8] = T_xy; out16[9] = T_yaw;
    if (!(total / dt < 4.0e6)) { out16[7] = -1.0; return; }     // not scanned, as the kernels
    double max_ax = 0.0, max_ay = 0.0, max_vx = 0.0, max_cur = 0.0, max_att = -1.0, max_sig = 0.0, err = 0.0;
    long count = 0, k = 0;
    for (double t = 0.0; t < total; t += dt, k++) {
        double tl = t;
        const int ip = locate_piece(N, T_xy, tl);
        const double *cx = c_xy + 6 * ip, *cy = c_xy + nx + 6 * ip;
        const double px = piece_value(cx, tl), py = piece_value(cy, tl);
        const double vxw = piece_dot(cx, tl), vyw = piece_dot(cy, tl);
        const double axw = piece_ddot(cx, tl), ayw = piece_ddot(cy, tl);
        double ty = t;
        const int iy = locate_piece(M, T_yaw, ty);
        const double *cw = c_yaw + 6 * iy;
        const double yaw = piece_value(cw, ty), dyaw = piece_dot(cw, ty);
        double se2[3] = {px, py, yaw};
        while (se2[2] < -M_PI) se2[2] += 2 * M_PI;
        while (se2[2] > M_PI) se2[2] -= 2 * M_PI;
        double tv[7], tg[7][3];
        mq.getAllWithGrad(se2, tv, tg);
        const double cy_ = Mth<double>::cos(yaw), sy_ = Mth<double>::sin(yaw);
        const double vnorm = std::sqrt(vxw * vxw + vyw * vyw);
        const double lon = axw * cy_ + ayw * sy_;
        const double lat = -axw * sy_ + ayw * cy_;
        const double vx = vnorm * tv[0];
        const double ax = lon * tv[0] + gravity * tv[1];
        const double ay = lat * tv[2] + gravity * tv[3];
        const double wz = dyaw * tv[5];
        const double cur = wz / std::sqrt(vx * vx + delta_sigl);
        const double att = -1.0 / tv[5];
        const double term = std::fabs(vxw * sy_ + vyw * (-cy_));
        const bool kept = t >= t_from;
        if (trace) {
            const double row[9] = {t, vx, ax, ay, cur, att, tv[6], term, kept ? 1.0 : 0.0};
            for (int q = 0; q < 9; q++) trace[9 * k + q] = row[q];
        }
        if (!kept) continue;
        if (std::fabs(max_ax) < std::fabs(ax)) max_ax = ax;
        if (std::fabs(max_ay) < std::fabs(ay)) max_ay = ay;
        if (std::fabs(max_vx) < std::fabs(vx)) max_vx = vx;
        if (std::fabs(max_cur) < std::fabs(cur)) max_cur = cur;
        if (max_att < att) max_att = att;
        if (max_sig < tv[6]) max_sig = tv[6];
        err += term;
        count++;
        const bool viol[6] = {std::fabs(vx) > lim[0], std::fabs(ax) > lim[1], std::fabs(ay) > lim[2], std::fabs(cur) > lim[3], att > -lim[4], tv[6] > lim[5]};
        for (int q = 0; q < 6; q++) if (viol[q] && out16[10 + q] < 0.0) out16[10 + q] = t;
    }
    out16[0] = max_vx; out16[1] = max_ax; out16[2] = max_ay; out16[3] = max_cur; out16[4] = max_att; out16[5] = max_sig; out16[6] = err;
    out16[7] = (double)count;
}
