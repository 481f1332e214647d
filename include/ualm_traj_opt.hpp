// ualm_traj_opt.hpp -- C++ host-side mirror of the reference's back-end interface, over the C ABI of ualm.h.
//
// The reference class is uneven_planner::ALMTrajOpt (back_end/include/back_end/alm_traj_opt.h:21-120):
//     init(nh), setEnvironment(map), optimizeSE2Traj(initXY, endXY, innerXY, initYaw, endYaw, innerYaw, totalTime) -> int,
//     getTraj() -> SE2Trajectory
// This header keeps those names, argument meaning (column-major Eigen layouts) and return codes (0 ok / 1 L-BFGS error /
// 2 ALM max-iter, alm_traj_opt.cpp:176,252,267) so PlanManager::rcvWpsCallBack (plan_manager.cpp:134-138) compiles against
// it unchanged when Eigen is present (define UALM_WITH_EIGEN), and adds the batch entry point the GPU is built for.
// No ROS, no Eigen required: the plain-pointer overloads are always available.  Header-only; link libualm.so.
#pragma once

#include <stdexcept>
#include <string>
#include <vector>

#include "ualm.h"

#ifdef UALM_WITH_EIGEN
#include <Eigen/Eigen>
#endif

namespace uneven_planner_b200 {

// Result container with the reference's Piece / PolyTrajectory / SE2Trajectory conventions (se2traj.hpp:31-150, 255-414):
// per piece a duration and a Dim x 6 coefficient matrix, HIGHEST power first (MinJerkOpt::getTraj reverses the solver's
// low->high order, se2traj.hpp:682-695).
template <int Dim>
struct Piece {
    double duration = 0.0;
    double coeff[Dim][6];                       // coeff[d][0] * t^5 + ... + coeff[d][5]
    void getValue(double t, double *out) const  // Piece::getValue, se2traj.hpp:106-118
    {
        for (int d = 0; d < Dim; d++) {
            double v = 0.0, tn = 1.0;
            for (int i = 5; i >= 0; i--) { v += tn * coeff[d][i]; tn *= t; }
            out[d] = v;
        }
    }
    double getDuration() const { return duration; }
};

struct SE2Trajectory {
    std::vector<Piece<2>> pos_traj;
    std::vector<Piece<1>> yaw_traj;
    double getTotalDuration() const
    {
        double a = 0, b = 0;
        for (auto &p : pos_traj) a += p.duration;
        for (auto &p : yaw_traj) b += p.duration;
        return a < b ? a : b;                   // SE2Trajectory::getTotalDuration, se2traj.hpp:416-419
    }
};

// PolyTrajectory::locatePieceIdx + getValue (se2traj.hpp:343-367): piece containing time t (t is reduced to the piece-local time)
template <int Dim>
inline int locatePieceIdx(const std::vector<Piece<Dim>> &pieces, double &t)
{
    const int N = (int)pieces.size();
    int idx;
    double dur;
    for (idx = 0; idx < N && t > (dur = pieces[idx].getDuration()); idx++) t -= dur;
    if (idx == N) {
        idx--;
        t += pieces[idx].getDuration();
    }
    return idx;
}
template <int Dim>
inline void getValue(const std::vector<Piece<Dim>> &pieces, double t, double *out)
{
    const int idx = locatePieceIdx(pieces, t);
    pieces[idx].getValue(t, out);
}
template <int Dim>
inline double getTotalDuration(const std::vector<Piece<Dim>> &pieces)   // PolyTrajectory::getTotalDuration, se2traj.hpp:291-300
{
    double total = 0.0;
    for (const auto &p : pieces) total += p.getDuration();
    return total;
}

// What PlanManager publishes to the MPC (mpc_controller/msg/SE2Traj.msg; plan_manager.cpp:151-185): the piece start points,
// the end point and the piece durations of both splines; the boundary velocity / acceleration fields are zero in the reference.
// A replanned robot's message carries its own state at the replan time instead ({x, y, yaw}: bnd' entries 2, 3, 13 and 4, 5, 14 of
// submitReplan), one message per robot (exportToMpc).
struct SE2TrajMsg {
    std::vector<double> pos_pts;      // (N + 1) x 2, row-major: pos_traj[i].getValue(0), then pos_traj.getValue(total)
    std::vector<double> posT_pts;     // N
    std::vector<double> angle_pts;    // M + 1
    std::vector<double> angleT_pts;   // M
    double init_v[3] = {0, 0, 0}, init_a[3] = {0, 0, 0};
};
inline SE2TrajMsg toSE2TrajMsg(const SE2Trajectory &tr)
{
    SE2TrajMsg m;
    double p[2], a[1];
    for (const auto &pc : tr.pos_traj) {
        pc.getValue(0.0, p);
        m.pos_pts.push_back(p[0]); m.pos_pts.push_back(p[1]);
        m.posT_pts.push_back(pc.getDuration());
    }
    getValue(tr.pos_traj, getTotalDuration(tr.pos_traj), p);
    m.pos_pts.push_back(p[0]); m.pos_pts.push_back(p[1]);
    for (const auto &pc : tr.yaw_traj) {
        pc.getValue(0.0, a);
        m.angle_pts.push_back(a[0]);
        m.angleT_pts.push_back(pc.getDuration());
    }
    getValue(tr.yaw_traj, getTotalDuration(tr.yaw_traj), a);
    m.angle_pts.push_back(a[0]);
    return m;
}

// c_xy: 6N x 2 column-major, c_yaw: 6M (solver order, low -> high power); T_xy / T_yaw: the uniform piece durations T1(i) the
// reference's getTraj() carries (MinJerkOpt::getTraj, se2traj.hpp:682-695; calTfromTau, alm_traj_opt.h:257-261) --
// ualm_result_t::piece_T_xy / piece_T_yaw, NOT total_T / N (the N-fold sum divided back differs by a few ulps)
inline SE2Trajectory make_traj(int N, int M, const double *c_xy, const double *c_yaw, double T_xy, double T_yaw)
{
    SE2Trajectory tr;
    tr.pos_traj.resize(N);
    tr.yaw_traj.resize(M);
    for (int i = 0; i < N; i++) {
        tr.pos_traj[i].duration = T_xy;
        for (int d = 0; d < 2; d++)
            for (int k = 0; k < 6; k++) tr.pos_traj[i].coeff[d][5 - k] = c_xy[6 * i + k + d * 6 * N];
    }
    for (int i = 0; i < M; i++) {
        tr.yaw_traj[i].duration = T_yaw;
        for (int k = 0; k < 6; k++) tr.yaw_traj[i].coeff[0][5 - k] = c_yaw[6 * i + k];
    }
    return tr;
}
inline SE2Trajectory make_traj(int N, int M, const double *c_xy, const double *c_yaw, const ualm_result_t &r)
{
    return make_traj(N, M, c_xy, c_yaw, r.piece_T_xy, r.piece_T_yaw);
}

class ALMTrajOpt {
public:
    // the reference's public parameter members (alm_traj_opt.h:29-53) live in `params`
    ualm_params_t params;

    explicit ALMTrajOpt(int device = 0, int precision = 64)
    {
        ualm_default_params(&params);
        if (ualm_create(&ctx_, device, precision) != UALM_OK) throw std::runtime_error(std::string("ualm_create: ") + ualm_last_error());
    }
    ~ALMTrajOpt() { ualm_destroy(ctx_); }
    ALMTrajOpt(const ALMTrajOpt &) = delete;
    ALMTrajOpt &operator=(const ALMTrajOpt &) = delete;

    // ALMTrajOpt::init(nh): the caller fills `params` from its rosparam server, then calls init()
    void init() { check(ualm_set_params(ctx_, &params), "ualm_set_params"); }
    // evaluation budget per problem of the following solves (0 = none); a stopped problem returns UALM_RET_STOPPED (ualm.h)
    void setBudget(int max_evals) { check(ualm_set_budget(ctx_, max_evals), "ualm_set_budget"); }
    // ualm_set_urgent: the submitBatch / submitReplan / checkTrajectories / exportToMpc calls after it go ahead of the batches in flight, with the same
    // results, until setUrgent(false)
    void setUrgent(bool urgent) { check(ualm_set_urgent(ctx_, urgent ? 1 : 0), "ualm_set_urgent"); }

    // ALMTrajOpt::setEnvironment(UnevenMap::Ptr): the map grid (UnevenMap::map_buffer is private in the reference,
    // uneven_map.h:91, so the maintainer-side binding passes geometry + a float4 view of the cells; INTEGRATION.md)
    void setEnvironment(const ualm_map_geom_t &geom, const float *cells_xyzw) { check(ualm_set_map(ctx_, &geom, cells_xyzw), "ualm_set_map"); }
    // the same from the reference's own double grid (UnevenMap::map_buffer, RXS2 = 4 doubles per cell, uneven_map.h:36-64)
    void setEnvironment(const ualm_map_geom_t &geom, const double *rxs2_cells, bool repack_to_float = false)
    {
        check(ualm_set_map_f64(ctx_, &geom, rxs2_cells, repack_to_float ? 1 : 0), "ualm_set_map_f64");
    }

    // Environment `env` (0 <= env < UALM_MAX_ENVS): a parameter set and a map grid of its own, for batches that mix terrains or
    // vehicle classes (optimizeBatch / submitBatch with env[]).  init() and setEnvironment() above bind environment 0.
    void setEnvironment(int env, const ualm_params_t &p, const ualm_map_geom_t &geom, const float *cells_xyzw)
    {
        bindEnv(env, p, [&] { return ualm_set_map(ctx_, &geom, cells_xyzw); }, "ualm_set_map");
    }
    void setEnvironment(int env, const ualm_params_t &p, const ualm_map_geom_t &geom, const double *rxs2_cells, bool repack_to_float = false)
    {
        bindEnv(env, p, [&] { return ualm_set_map_f64(ctx_, &geom, rxs2_cells, repack_to_float ? 1 : 0); }, "ualm_set_map_f64");
    }

    // Replace the grid of environment `env` while batches are in flight (ualm_update_map): work launched before keeps its grid, every
    // later launch reads the new one; the call does not wait for running batches.  The parameters of `env` stay as bound
    void updateEnvironment(int env, const ualm_map_geom_t &geom, const float *cells_xyzw)
    {
        onEnv(env, [&] { return ualm_update_map(ctx_, &geom, cells_xyzw); }, "ualm_update_map");
    }
    // the same with the grid built on the device from a point cloud (npts x 3 floats); cells_out (optional) receives the grid
    void updateEnvironmentFromCloud(int env, const float *pts, int64_t npts, const ualm_map_geom_t &geom, double ellipsoid_x = 0.2, double ellipsoid_y = 0.1,
                                    double ellipsoid_z = 0.1, int iter_num = 2, float *cells_out = nullptr, float *kernel_ms = nullptr)
    {
        onEnv(env, [&] { return ualm_update_map_from_cloud(ctx_, pts, npts, &geom, ellipsoid_x, ellipsoid_y, ellipsoid_z, iter_num, cells_out, kernel_ms); },
              "ualm_update_map_from_cloud");
    }
    // Replace the cell columns [ix0, ix0+nx) x [iy0, iy0+ny), all yaw layers, of environment `env`'s grid while batches are in flight
    // (ualm_update_map_window), same guarantees as updateEnvironment; cells: nx*ny*Yaw float4 in the grid's [x][y][yaw] order
    void updateEnvironmentWindow(int env, int ix0, int iy0, int nx, int ny, const float *cells_xyzw)
    {
        onEnv(env, [&] { return ualm_update_map_window(ctx_, ix0, iy0, nx, ny, cells_xyzw); }, "ualm_update_map_window");
    }
    // the same box built on the device from a point cloud, e.g. a local scan (npts x 3 floats); cells_out (optional) receives the box
    void updateEnvironmentWindowFromCloud(int env, const float *pts, int64_t npts, int ix0, int iy0, int nx, int ny, double ellipsoid_x = 0.2,
                                          double ellipsoid_y = 0.1, double ellipsoid_z = 0.1, int iter_num = 2, float *cells_out = nullptr,
                                          float *kernel_ms = nullptr)
    {
        onEnv(env, [&] { return ualm_update_map_window_from_cloud(ctx_, pts, npts, ix0, iy0, nx, ny, ellipsoid_x, ellipsoid_y, ellipsoid_z, iter_num, cells_out, kernel_ms); },
              "ualm_update_map_window_from_cloud");
    }
    // Move environment `env`'s grid by (dx, dy) whole cells while batches are in flight (ualm_shift_map), same guarantees as
    // updateEnvironmentWindow; cells: the uncovered boxes A then B, each in the window layout
    void shiftEnvironment(int env, int dx, int dy, const float *cells_xyzw)
    {
        onEnv(env, [&] { return ualm_shift_map(ctx_, dx, dy, cells_xyzw); }, "ualm_shift_map");
    }
    // the same shift with A and B built on the device from a point cloud, e.g. a local scan; cells_out (optional) receives A then B
    void shiftEnvironmentFromCloud(int env, const float *pts, int64_t npts, int dx, int dy, double ellipsoid_x = 0.2, double ellipsoid_y = 0.1,
                                   double ellipsoid_z = 0.1, int iter_num = 2, float *cells_out = nullptr, float *kernel_ms = nullptr)
    {
        onEnv(env, [&] { return ualm_shift_map_from_cloud(ctx_, pts, npts, dx, dy, ellipsoid_x, ellipsoid_y, ellipsoid_z, iter_num, cells_out, kernel_ms); },
              "ualm_shift_map_from_cloud");
    }

    // ---- single problem, the reference's call (alm_traj_opt.h:92-98), plain pointers ----
    // initStateXY/endStateXY: 2x3 column-major; innerPtsXY: 2 x (N-1) column-major; initYaw/endYaw: 3; innerPtsYaw: M-1
    int optimizeSE2Traj(const double *initStateXY, const double *endStateXY, const double *innerPtsXY, int n_inner_xy,
                        const double *initYaw, const double *endYaw, const double *innerPtsYaw, int n_inner_yaw, double totalTime)
    {
        const int32_t N = n_inner_xy + 1, M = n_inner_yaw + 1;
        double bnd[18];
        for (int k = 0; k < 6; k++) { bnd[k] = initStateXY[k]; bnd[6 + k] = endStateXY[k]; }
        for (int k = 0; k < 3; k++) { bnd[12 + k] = initYaw[k]; bnd[15 + k] = endYaw[k]; }
        last_N_ = N; last_M_ = M;
        c_xy_.assign(12 * (size_t)N, 0.0);
        c_yaw_.assign(6 * (size_t)M, 0.0);
        check(ualm_solve_batch(ctx_, 1, &N, &M, bnd, &totalTime, innerPtsXY, innerPtsYaw, &last_, c_xy_.data(), c_yaw_.data()), "ualm_solve_batch");
        return last_.ret_code;
    }
    SE2Trajectory getTraj() const { return make_traj(last_N_, last_M_, c_xy_.data(), c_yaw_.data(), last_); }
    const ualm_result_t &lastResult() const { return last_; }

#ifdef UALM_WITH_EIGEN
    // the reference's exact signature (alm_traj_opt.h:92-98)
    int optimizeSE2Traj(const Eigen::MatrixXd &initStateXY, const Eigen::MatrixXd &endStateXY, const Eigen::MatrixXd &innerPtsXY,
                        const Eigen::VectorXd &initYaw, const Eigen::VectorXd &endYaw, const Eigen::VectorXd &innerPtsYaw,
                        const double &totalTime)
    {
        return optimizeSE2Traj(initStateXY.data(), endStateXY.data(), innerPtsXY.data(), (int)innerPtsXY.cols(), initYaw.data(),
                               endYaw.data(), innerPtsYaw.data(), (int)innerPtsYaw.size(), totalTime);
    }
#endif

    // ---- batch: B independent optimizeSE2Traj problems, packed as in ualm.h ----
    void optimizeBatch(int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time, const double *inner_xy,
                       const double *inner_yaw, ualm_result_t *results, double *c_xy, double *c_yaw)
    {
        check(ualm_solve_batch(ctx_, B, N, M, bnd, total_time, inner_xy, inner_yaw, results, c_xy, c_yaw), "ualm_solve_batch");
    }
    // the same with the environment of every problem (env[B], nullptr = all 0)
    void optimizeBatch(int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time, const double *inner_xy,
                       const double *inner_yaw, const int32_t *env, ualm_result_t *results, double *c_xy, double *c_yaw)
    {
        check(ualm_solve_batch_env(ctx_, B, N, M, bnd, total_time, inner_xy, inner_yaw, env, results, c_xy, c_yaw), "ualm_solve_batch_env");
    }
    // ... and each problem's own vehicle limits and cost weights (pp[B], nullptr = its environment's; ualm_problem_params_t)
    void optimizeBatch(int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time, const double *inner_xy,
                       const double *inner_yaw, const int32_t *env, const ualm_problem_params_t *pp, ualm_result_t *results, double *c_xy, double *c_yaw)
    {
        check(ualm_solve_batch_pp(ctx_, B, N, M, bnd, total_time, inner_xy, inner_yaw, env, pp, results, c_xy, c_yaw), "ualm_solve_batch_pp");
    }

    // pipelined form: submit returns once the batch is uploaded and queued (up to `depth` batches in flight), wait collects it
    int submitBatch(int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time, const double *inner_xy,
                    const double *inner_yaw, int depth = 2)
    {
        int ticket = -1;
        check(ualm_submit_batch(ctx_, B, N, M, bnd, total_time, inner_xy, inner_yaw, depth, &ticket), "ualm_submit_batch");
        return ticket;
    }
    int submitBatch(int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time, const double *inner_xy,
                    const double *inner_yaw, const int32_t *env, int depth)
    {
        int ticket = -1;
        check(ualm_submit_batch_env(ctx_, B, N, M, bnd, total_time, inner_xy, inner_yaw, env, depth, &ticket), "ualm_submit_batch_env");
        return ticket;
    }
    int submitBatch(int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time, const double *inner_xy,
                    const double *inner_yaw, const int32_t *env, const ualm_problem_params_t *pp, int depth)
    {
        int ticket = -1;
        check(ualm_submit_batch_pp(ctx_, B, N, M, bnd, total_time, inner_xy, inner_yaw, env, pp, depth, &ticket), "ualm_submit_batch_pp");
        return ticket;
    }
    void waitBatch(int ticket, ualm_result_t *results, double *c_xy, double *c_yaw) { check(ualm_wait_batch(ctx_, ticket, results, c_xy, c_yaw), "ualm_wait_batch"); }
    // the same with a deadline: after timeout_ms the problems still running are stopped (UALM_RET_STOPPED) and the batch drains
    void waitBatchFor(int ticket, double timeout_ms, ualm_result_t *results, double *c_xy, double *c_yaw)
    {
        check(ualm_wait_batch_for(ctx_, ticket, timeout_ms, results, c_xy, c_yaw), "ualm_wait_batch_for");
    }
    // the problems of a submitted batch that finished since the last poll (ualm_poll_batch): their indices into idx (capacity B),
    // their records and coefficients at their problem-order places of results / c_xy / c_yaw (the buffers waitBatch takes; c_xy /
    // c_yaw may be null).  Returns how many; *pending = problems not returned yet.  wait_ms > 0 blocks until one is new or wait_ms
    // has passed.  waitBatch afterwards returns the whole batch as before.  The batch runs on the device whether or not anyone polls
    // (both paths), so the caller may sleep or do other work between polls
    int pollBatch(int ticket, double wait_ms, int32_t *idx, int *pending, ualm_result_t *results, double *c_xy, double *c_yaw)
    {
        int n_new = 0;
        check(ualm_poll_batch(ctx_, ticket, wait_ms, idx, &n_new, pending, results, c_xy, c_yaw), "ualm_poll_batch");
        return n_new;
    }
    // stop the problems idx[0, n) of a submitted batch at their next stop test (ualm_cancel_problems): they come back through
    // pollBatch / waitBatch with UALM_RET_STOPPED, or with their own result if they were final first; the rest is unaffected.
    // The cancel reaches running problems on both paths without a further call
    void cancelProblems(int ticket, int n, const int32_t *idx) { check(ualm_cancel_problems(ctx_, ticket, n, idx), "ualm_cancel_problems"); }

    // What the MPC receives and tracks, for the batch solved last on the selected lane (ualm_mpc_export_batch): the SE2Traj message
    // arrays of PlanManager (plan_manager.cpp:151-185), the MPC side's own MINCO over them (traj_anal.hpp:125-181) and the largest
    // planned-vs-tracked deviation.  Any pointer may be null.
    void exportToMpcBatch(double dt, double *pos_pts, double *posT_pts, double *angle_pts, double *angleT_pts, double *c_mpc_xy, double *c_mpc_yaw,
                          double *dev4, const double *init_v = nullptr, const double *init_a = nullptr)
    {
        check(ualm_mpc_export_batch(ctx_, dt, init_v, init_a, pos_pts, posT_pts, angle_pts, angleT_pts, c_mpc_xy, c_mpc_yaw, dev4), "ualm_mpc_export_batch");
    }

    // The same hand-over for B trajectories the caller holds (e.g. from waitBatch / pollBatch, in checkTrajectories' layouts), each row
    // from its own start state: init_v / init_a = 3 doubles {x, y, yaw} per row, null = zero (ualm_mpc_export_trajectories).  Outputs
    // packed row after row; any output may be null.  Reads no grid or lane and may be called while batches are in flight
    void exportToMpc(int B, const int32_t *N, const int32_t *M, const double *piece_T, const double *c_xy, const double *c_yaw, const double *init_v,
                     const double *init_a, double dt, double *pos_pts, double *posT_pts, double *angle_pts, double *angleT_pts, double *c_mpc_xy,
                     double *c_mpc_yaw, double *dev4)
    {
        check(ualm_mpc_export_trajectories(ctx_, B, N, M, piece_T, c_xy, c_yaw, init_v, init_a, dt, pos_pts, posT_pts, angle_pts, angleT_pts, c_mpc_xy,
                                           c_mpc_yaw, dev4), "ualm_mpc_export_trajectories");
    }

    // The post-solve scan of B trajectories the caller holds (e.g. from waitBatch: piece_T = {piece_T_xy, piece_T_yaw} per record)
    // against each environment's grid as it is now, over the samples t >= t_from[b] of the full scan, with the time of the first
    // violation of each limit (ualm_check_trajectories).  env / t_from / limits may be null (all 0 / all 0 / each environment's own).
    // out16: 16 doubles per trajectory.  May be called while batches are in flight
    void checkTrajectories(int B, const int32_t *N, const int32_t *M, const double *piece_T, const double *c_xy, const double *c_yaw, const int32_t *env,
                           const double *t_from, double dt, const ualm_limits_t *limits, double *out16)
    {
        check(ualm_check_trajectories(ctx_, B, N, M, piece_T, c_xy, c_yaw, env, t_from, dt, limits, out16), "ualm_check_trajectories");
    }
    // the same with each trajectory's own limits from its row pp[b] where `limits` is null (ualm_check_trajectories_pp)
    void checkTrajectories(int B, const int32_t *N, const int32_t *M, const double *piece_T, const double *c_xy, const double *c_yaw, const int32_t *env,
                           const ualm_problem_params_t *pp, const double *t_from, double dt, const ualm_limits_t *limits, double *out16)
    {
        check(ualm_check_trajectories_pp(ctx_, B, N, M, piece_T, c_xy, c_yaw, env, pp, t_from, dt, limits, out16), "ualm_check_trajectories_pp");
    }

    // Replans B trajectories the caller holds (as for checkTrajectories, plus each one's original problem row bnd, 18 doubles) from the
    // state at t_from[b] to the original goal, and submits the built problems as one ticket (ualm_submit_replan; wait on it with
    // waitBatch).  rp may be null (run_*.yaml's resampler).  Outputs: the built N, M, bnd (18 per row), total_time and, optional,
    // inner points at UALM_REPLAN_INNER_XY / UALM_REPLAN_INNER_YAW doubles per row.  Returns the ticket
    int submitReplan(int B, const int32_t *N, const int32_t *M, const double *piece_T, const double *c_xy, const double *c_yaw, const double *bnd,
                     const int32_t *env, const double *t_from, double dt, const ualm_resample_params_t *rp, int depth, int32_t *N_out, int32_t *M_out,
                     double *bnd_out, double *total_time_out, double *inner_xy_out = nullptr, double *inner_yaw_out = nullptr)
    {
        int ticket = -1;
        check(ualm_submit_replan(ctx_, B, N, M, piece_T, c_xy, c_yaw, bnd, env, t_from, dt, rp, depth, &ticket, N_out, M_out, bnd_out, total_time_out,
                                 inner_xy_out, inner_yaw_out), "ualm_submit_replan");
        return ticket;
    }
    // the same with row b of the ticket solved with pp[b] (ualm_submit_replan_pp)
    int submitReplan(int B, const int32_t *N, const int32_t *M, const double *piece_T, const double *c_xy, const double *c_yaw, const double *bnd,
                     const int32_t *env, const ualm_problem_params_t *pp, const double *t_from, double dt, const ualm_resample_params_t *rp, int depth,
                     int32_t *N_out, int32_t *M_out, double *bnd_out, double *total_time_out, double *inner_xy_out = nullptr, double *inner_yaw_out = nullptr)
    {
        int ticket = -1;
        check(ualm_submit_replan_pp(ctx_, B, N, M, piece_T, c_xy, c_yaw, bnd, env, pp, t_from, dt, rp, depth, &ticket, N_out, M_out, bnd_out,
                                    total_time_out, inner_xy_out, inner_yaw_out), "ualm_submit_replan_pp");
        return ticket;
    }

    // The reference's whole chain for B (start, goal) pairs: KinoAstar::plan + PlanManager's resampler on host threads
    // (ualm_front_end_batch), then the batched optimizer.  packed[b] = index of pair b in the outputs or -1 (no path / over the
    // optimizer's limits); results / c_xy / c_yaw hold the packed problems back to back like optimizeBatch.  Returns their number.
    int planAndOptimizeBatch(const ualm_astar_map_t &map, const ualm_astar_params_t &ap, const ualm_resample_params_t &rp, int B, const double *starts,
                             const double *goals, std::vector<int32_t> &packed, std::vector<int32_t> &N, std::vector<int32_t> &M, std::vector<ualm_result_t> &results,
                             std::vector<double> &c_xy, std::vector<double> &c_yaw, int nthreads = 0)
    {
        packed.assign(B, -1); N.assign(B, 0); M.assign(B, 0);
        std::vector<double> bnd(18 * (size_t)B), T(B), ixy(2 * 63 * (size_t)B + 2), iyaw(127 * (size_t)B + 1);
        const int k = ualm_front_end_batch(&map, &ap, &rp, B, starts, goals, nthreads, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), (long long)ixy.size(),
                                           iyaw.data(), (long long)iyaw.size(), packed.data(), nullptr);
        if (k < 0) throw std::runtime_error("ualm_front_end_batch failed");
        N.resize(k); M.resize(k);
        size_t ncx = 0, ncy = 0;
        for (int i = 0; i < k; i++) { ncx += 12 * (size_t)N[i]; ncy += 6 * (size_t)M[i]; }
        results.assign(k, ualm_result_t{}); c_xy.assign(ncx, 0.0); c_yaw.assign(ncy, 0.0);
        if (k > 0) optimizeBatch(k, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), results.data(), c_xy.data(), c_yaw.data());
        return k;
    }

    ualm_ctx_t *handle() { return ctx_; }

private:
    static void check(int rc, const char *what)
    {
        if (rc != UALM_OK) throw std::runtime_error(std::string(what) + ": " + ualm_last_error());
    }
    // select `env`, bind its parameters and grid, select environment 0 again (also when a call throws)
    template <class F>
    void bindEnv(int env, const ualm_params_t &p, F set_map, const char *what)
    {
        check(ualm_select_env(ctx_, env), "ualm_select_env");
        int rc = ualm_set_params(ctx_, &p);
        const std::string msg = rc != UALM_OK ? std::string("ualm_set_params: ") + ualm_last_error() : std::string();
        if (rc == UALM_OK) rc = set_map();
        const std::string msg2 = msg.empty() && rc != UALM_OK ? std::string(what) + ": " + ualm_last_error() : msg;
        ualm_select_env(ctx_, 0);
        if (rc != UALM_OK) throw std::runtime_error(msg2);
    }
    // select `env`, run `call`, select environment 0 again (also when the call fails)
    template <class F>
    void onEnv(int env, F call, const char *what)
    {
        check(ualm_select_env(ctx_, env), "ualm_select_env");
        const int rc = call();
        const std::string msg = rc != UALM_OK ? std::string(what) + ": " + ualm_last_error() : std::string();
        ualm_select_env(ctx_, 0);
        if (rc != UALM_OK) throw std::runtime_error(msg);
    }
    ualm_ctx_t *ctx_ = nullptr;
    ualm_result_t last_{};
    int last_N_ = 0, last_M_ = 0;
    std::vector<double> c_xy_, c_yaw_;
};

} // namespace uneven_planner_b200
