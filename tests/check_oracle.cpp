// check_oracle.cpp -- the CPU reference of ualm_check_trajectories (include/ualm.h): orc_feasibility's loop over the oracle's scanned
// sample (scan_sample in oracle/oracle.cpp, included unmodified) restricted to the samples t >= t_from of the full sequence t = 0, dt,
// 2dt.., with the time of the first kept sample that breaks each of six limits.  TEST INFRASTRUCTURE ONLY, built by tests/check_oracle.py.
//
//   out16 = {max_vx, max_ax, max_ay, max_cur, max_att, max_sig, nonhol_error, kept samples, T_xy, T_yaw, first |vx| > max_vel,
//            |ax| > max_acc_lon, |ay| > max_acc_lat, |cur| > max_kap, att > -min_cxi, sig > max_sig (-1: none)}
//   trace (optional): 9 doubles per sample of the full sequence {t, vx, ax, ay, cur, att, sig, nonhol term, kept}
#include "../oracle/oracle.cpp"

extern "C" void orc_check(const orc_map_t *map, double gravity, int N, int M, const double *c_xy, const double *c_yaw, double T_xy, double T_yaw,
                          double dt, double t_from, const double lim[6], double *out16, double *trace)
{
    MapQ<double> mq(*map);
    const double total = traj_duration(N, M, T_xy, T_yaw);
    for (int q = 0; q < 16; q++) out16[q] = q >= 10 ? -1.0 : 0.0;
    out16[8] = T_xy; out16[9] = T_yaw;
    if (!(total / dt < 4.0e6)) { out16[7] = -1.0; return; }     // not scanned, as the kernels
    double max_ax = 0.0, max_ay = 0.0, max_vx = 0.0, max_cur = 0.0, max_att = -1.0, max_sig = 0.0, err = 0.0;
    long count = 0, k = 0;
    for (double t = 0.0; t < total; t += dt, k++) {
        const ScanSample s = scan_sample(mq, gravity, N, M, c_xy, c_yaw, T_xy, T_yaw, t);
        const bool kept = t >= t_from;
        if (trace) {
            const double row[9] = {t, s.vx, s.ax, s.ay, s.cur, s.att, s.sig, s.term, kept ? 1.0 : 0.0};
            for (int q = 0; q < 9; q++) trace[9 * k + q] = row[q];
        }
        if (!kept) continue;
        if (std::fabs(max_ax) < std::fabs(s.ax)) max_ax = s.ax;
        if (std::fabs(max_ay) < std::fabs(s.ay)) max_ay = s.ay;
        if (std::fabs(max_vx) < std::fabs(s.vx)) max_vx = s.vx;
        if (std::fabs(max_cur) < std::fabs(s.cur)) max_cur = s.cur;
        if (max_att < s.att) max_att = s.att;
        if (max_sig < s.sig) max_sig = s.sig;
        err += s.term;
        count++;
        const bool viol[6] = {std::fabs(s.vx) > lim[0], std::fabs(s.ax) > lim[1], std::fabs(s.ay) > lim[2], std::fabs(s.cur) > lim[3], s.att > -lim[4],
                              s.sig > lim[5]};
        for (int q = 0; q < 6; q++) if (viol[q] && out16[10 + q] < 0.0) out16[10 + q] = t;
    }
    out16[0] = max_vx; out16[1] = max_ax; out16[2] = max_ay; out16[3] = max_cur; out16[4] = max_att; out16[5] = max_sig; out16[6] = err;
    out16[7] = (double)count;
}
