// resample_stream.h -- PlanManager::rcvWpsCallBack's yaw smoothing and arc-length resampling (plan_manager/src/plan_manager.cpp:62-77,
// 96-122) as a stream that takes the (x, y, yaw) polyline one point at a time.  Shared by the host resampler (host_tools.cpp,
// ualm_resample_path) and the replan builder (ualm_kernels.cuh, replan_kernel), so both run the SAME arithmetic (IEEE double, no
// contraction: nvcc -fmad=false, gcc -ffp-contract=off).  Smoothing point k + 1 needs only the smoothed point k, so taking the points
// one at a time performs the reference's operations in its order.  Shares no code with the reference.
//
// The host resampler stops at its caps.  The replan builder counts past them, so its stream is bounded instead (ualm_rs_push): a polyline
// that would need more than UALM_RS_MAX_WAYPOINTS waypoints of either kind, a yaw of magnitude 2^40 or more, or more than
// UALM_RS_MAX_TURNS whole turns of smoothing is cut short (`cut`): from there on only the segment lengths are summed.  Without the bound
// a huge or non-finite length or yaw would keep one warp looping (practically) forever.
#pragma once

#include <math.h>

#include "ualm_detmath.h"

struct UalmResampleStream {
    double prev[3];                     // the last point taken, its yaw smoothed
    double piece_len, piece_len_yaw;
    double temp_len_yaw, temp_len_pos, total_len;
    long long npts, nxy, nyaw;          // points taken; inner xy / yaw waypoints counted, past the caps too
    double turns;                       // whole turns of smoothing so far (ualm_rs_push)
    bool cut;                           // cut short: no more waypoints or smoothing, lengths only
};

#define UALM_RS_MAX_WAYPOINTS 4095      // ualm_rs_push: waypoints of one kind before a polyline is cut short
#define UALM_RS_MAX_YAW 0x1p40          //   |yaw| bound (its ulp stays far below a turn, so smoothing always moves it)
#define UALM_RS_MAX_TURNS 65536.0       //   whole turns of smoothing, summed over the polyline

UALM_HD void ualm_rs_init(UalmResampleStream &s, double piece_len, double yaw_piece_times)
{
    s.prev[0] = s.prev[1] = s.prev[2] = 0.0;
    s.piece_len = piece_len;
    s.piece_len_yaw = piece_len / yaw_piece_times;
    s.temp_len_yaw = 0.0; s.temp_len_pos = 0.0; s.total_len = 0.0;
    s.npts = 0; s.nxy = 0; s.nyaw = 0;
    s.turns = 0.0; s.cut = false;
}

// pm.cpp:62-77 for one point: yaw moved by whole turns until it is within (-pi/2, pi/2) of the previous point's smoothed yaw
UALM_HD void ualm_rs_smooth(double prev_yaw, double &yaw)
{
    double dyaw = yaw - prev_yaw;
    while (dyaw >= M_PI / 2) { yaw -= M_PI * 2; dyaw = yaw - prev_yaw; }
    while (dyaw <= -M_PI / 2) { yaw += M_PI * 2; dyaw = yaw - prev_yaw; }
}

// pm.cpp:96-121 for the segment a -> b of the smoothed polyline.  Waypoint k goes to inner_xy[2k, 2k+1] / inner_yaw[k] while
// k < max_xy / max_yaw and the array is not null; one past a cap is counted but not written.  stop: return false at the first waypoint
// past a cap, as the reference's caller gives up there (the counts are then not final); otherwise always true.  max_count > 0: the
// waypoint that would be number max_count + 1 of its kind cuts the stream short instead (0: no bound).  A cut stream sums lengths only.
UALM_HD bool ualm_rs_segment(UalmResampleStream &s, const double *a, const double *b, double *inner_xy, long long max_xy, double *inner_yaw,
                             long long max_yaw, bool stop, long long max_count)
{
    const double temp_seg = sqrt((b[0] - a[0]) * (b[0] - a[0]) + (b[1] - a[1]) * (b[1] - a[1]));
    s.temp_len_yaw += temp_seg; s.temp_len_pos += temp_seg; s.total_len += temp_seg;
    if (s.cut) return true;
    while (s.temp_len_yaw > s.piece_len_yaw) {
        if (max_count > 0 && s.nyaw >= max_count) { s.cut = true; return true; }
        if (s.nyaw >= max_yaw) { if (stop) return false; }
        else if (inner_yaw) inner_yaw[s.nyaw] = a[2] + (1.0 - (s.temp_len_yaw - s.piece_len_yaw) / temp_seg) * (b[2] - a[2]);
        s.nyaw++;
        s.temp_len_yaw -= s.piece_len_yaw;
    }
    while (s.temp_len_pos > s.piece_len) {
        if (max_count > 0 && s.nxy >= max_count) { s.cut = true; return true; }
        if (s.nxy >= max_xy) { if (stop) return false; }
        else if (inner_xy) {
            const double w = (1.0 - (s.temp_len_pos - s.piece_len) / temp_seg);
            inner_xy[2 * s.nxy] = a[0] + w * (b[0] - a[0]);
            inner_xy[2 * s.nxy + 1] = a[1] + w * (b[1] - a[1]);
        }
        s.nxy++;
        s.temp_len_pos -= s.piece_len;
    }
    return true;
}

// the next point of the polyline: its yaw smoothed against the previous point's, then the segment from that point (none for the first).
// Bounded: both yaws below UALM_RS_MAX_YAW in magnitude and the turns it needs within UALM_RS_MAX_TURNS overall, else the stream is cut
// short; at most UALM_RS_MAX_WAYPOINTS waypoints of each kind, else cut short (every loop then runs a bounded number of times)
UALM_HD void ualm_rs_push(UalmResampleStream &s, double x, double y, double yaw, double *inner_xy, long long max_xy, double *inner_yaw, long long max_yaw)
{
    double p[3] = {x, y, yaw};
    if (s.npts > 0) {
        if (!s.cut) {
            if (!(fabs(s.prev[2]) < UALM_RS_MAX_YAW && fabs(p[2]) < UALM_RS_MAX_YAW)) {
                s.cut = true;
            } else {
                const double turns = floor(fabs(p[2] - s.prev[2]) / (M_PI * 2)) + 1.0;
                if (s.turns + turns > UALM_RS_MAX_TURNS) s.cut = true;
                else { s.turns += turns; ualm_rs_smooth(s.prev[2], p[2]); }
            }
        }
        ualm_rs_segment(s, s.prev, p, inner_xy, max_xy, inner_yaw, max_yaw, false, UALM_RS_MAX_WAYPOINTS);
    }
    s.prev[0] = p[0]; s.prev[1] = p[1]; s.prev[2] = p[2];
    s.npts++;
}

// pm.cpp:122
UALM_HD double ualm_rs_total_time(const UalmResampleStream &s, double mean_vel, double init_time_times)
{
    return s.total_len / mean_vel * init_time_times;
}
