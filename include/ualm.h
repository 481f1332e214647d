/*
 * ualm.h -- C ABI of the H100-native batched MINCO / augmented-Lagrangian trajectory optimizer.
 *
 * Drop-in boundary for ONE hot path of ZJU-FAST-Lab/uneven_planner: the back-end
 *   uneven_planner::ALMTrajOpt::optimizeSE2Traj(...)            back_end/include/back_end/alm_traj_opt.h:92-98
 *   uneven_planner::ALMTrajOpt::getTraj()                        alm_traj_opt.h:165-168
 * with its environment binding
 *   ALMTrajOpt::setEnvironment(UnevenMap::Ptr)                   alm_traj_opt.h:127-130
 *   ALMTrajOpt::init(nh)  (the alm_traj_opt/ * rosparams)        back_end/src/alm_traj_opt.cpp:5-45
 * (paths relative to /root/reference/src/uneven_planner/).  Plain pointers and sizes only; no
 * torch / Eigen / ROS types.  Every entry point returns 0 on success or a negative UALM_E* code
 * and never falls back to a CPU implementation: without a CUDA device the compute calls fail.
 *
 * All matrices use the reference's (Eigen column-major) layouts:
 *   init_xy / end_xy : 2x3  [px,py, vx,vy, ax,ay]       (alm_traj_opt.cpp:183-186, pm.cpp:80-94)
 *   inner_xy         : 2x(N-1) [x1,y1, x2,y2, ...]      (alm_traj_opt.cpp:211,215)
 *   c_xy             : 6N x 2  (x column then y column; per piece 6 coefficients low->high power,
 *                      se2traj.hpp:585, 712-715);  c_yaw : 6M
 */
#ifndef UALM_H
#define UALM_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UALM_OK 0
#define UALM_ENOCUDA (-1)   /* no usable CUDA device / CUDA runtime error (message via ualm_last_error) */
#define UALM_EINVAL (-2)    /* bad argument */
#define UALM_ESTATE (-3)    /* call order (no map / no params / nothing uploaded) */
#define UALM_ELIMIT (-4)    /* problem exceeds compiled limits (N, M; int_K, mem_size, past in ualm_set_params) */

/* ret_code of a problem whose solve was stopped early (no such exit exists in the reference; it is modelled on its earlyExit).
 * Three causes stop a problem: its evaluation budget (ualm_set_budget), a deadline (ualm_wait_batch_for, which cancels every
 * problem of its batch) and a cancel of the problem itself (ualm_cancel_problems).
 * stop = (max_evals > 0 && n_evals >= max_evals) || the problem's stop word is raised, tested after every accepted line search (where
 * earlyExit tests k > 1000): L-BFGS then returns CANCELED, the ALM loop updates the duals and judges convergence as after any
 * cancel, and ends with UALM_RET_STOPPED even when that test passes (res_h / res_g tell whether epsilon_con was met).  The ALM
 * loop tests `stop` once more after judgeConvergence, so no inner solve starts after it holds.  A running line search is not
 * interrupted: a problem stopped by the budget has max_evals <= n_evals <= max_evals + 64.  The outputs are those of the last
 * evaluation, as for every exit.  A record with another ret_code never had a stop act on it: it is the unbudgeted result. */
#define UALM_RET_STOPPED 3

/* ---- parameters: the 21 alm_traj_opt/ * values (alm_traj_opt.cpp:7-27) + uneven_map/gravity ---- */
typedef struct {
    double rho_T, rho_ter, max_vel, max_acc_lon, max_acc_lat, max_kap, min_cxi, max_sig;
    int    use_scaling;
    double rho, beta, gamma, epsilon_con, max_iter;
    double g_epsilon, min_step, inner_max_iter, delta;
    int    mem_size, past, int_K;
    double gravity;          /* UnevenMap::getGravity(), uneven_map.cpp:85 */
} ualm_params_t;

/* run_hill.yaml defaults (plan_manager/params/run_hill.yaml:30-55) */
void ualm_default_params(ualm_params_t *p);

/* ---- per-problem parameters: what describes one vehicle and one request ----
 * The first eight members of ualm_params_t, in its order: the two cost weights (rho_T, time against smoothness; rho_ter, the sigma^2
 * terrain cost) and the six limits.  None of them shapes a buffer or a shared-memory layout, so every problem of a batch may carry its
 * own row.  int_K, mem_size, past, use_scaling, gravity and the ALM / L-BFGS settings stay per environment.
 * The *_pp entry points take their *_env counterpart's arguments plus pp[B] (NULL = every problem uses its environment's values; each
 * *_env entry point is its *_pp form with pp = NULL).  Contract:
 *   bits:      problem b with row pp[b] gives, bit for bit, the record and coefficients the same problem gets in a batch of an
 *              environment whose ualm_params_t is env[b]'s with these eight fields replaced, at every precision; at precision 64 that is
 *              the CPU oracle's solve with those parameters;
 *   phases:    ualm_eval_batch, ualm_init_scaling_batch and ualm_time_penalty_kernel on a batch uploaded with rows use each problem's
 *              row; ualm_feasibility_batch and ualm_mpc_export_batch read no limit and do not change;
 *   tickets:   polls, cancels, the budget, deadlines, urgency, map updates and the lane ring act as on any ticket;
 *   refusals:  a non-finite field in any row is UALM_EINVAL, decided before anything is touched: nothing is written and no lane is
 *              taken.  Every other refusal is the *_env form's. */
typedef struct {
    double rho_T, rho_ter, max_vel, max_acc_lon, max_acc_lat, max_kap, min_cxi, max_sig;
} ualm_problem_params_t;

/* ---- environment: what ALMTrajOpt reads of UnevenMap (uneven_map.h:258-377, 398-454) ---- */
typedef struct {
    int    voxel_num[3];     /* X, Y, Yaw cells (uneven_map.cpp:108-110) */
    double origin[3];        /* map_origin = min_boundary (uneven_map.cpp:99-101) */
    double max_boundary[3];
    double xy_resolution, yaw_resolution;
} ualm_map_geom_t;

/* geometry for map_size_x/y and resolutions exactly as UnevenMap::init computes it (uneven_map.cpp:96-114) */
void ualm_map_geometry(double map_size_x, double map_size_y, double xy_resolution, double yaw_resolution,
                       ualm_map_geom_t *g);
/* the same grid centred at (centre_x, centre_y) instead of the world origin: ualm_map_geometry's voxel counts, resolutions and yaw axis,
 * with origin = centre - size / 2 and max_boundary = centre + size / 2 in x and y.  centre (0, 0) gives ualm_map_geometry's struct bit
 * for bit.  Every cloud builder crops the cloud to [c - 10, c + 10]^2 about the grid's centre c = (origin + max_boundary) / 2 (the
 * reference's fixed CropBox about the world origin, uneven_map.cpp:133-137, moved with the grid) */
void ualm_map_geometry_at(double map_size_x, double map_size_y, double xy_resolution, double yaw_resolution, double centre_x,
                          double centre_y, ualm_map_geom_t *g);

/* ---- per-problem result record (what the reference prints / returns: alm_traj_opt.cpp:176,252,267,272-273;
 *      alm_traj_opt.h:142) ---- */
typedef struct {
    int32_t ret_code;        /* 0 converged / 1 L-BFGS hard error / 2 ALM max_iter (the reference's codes); UALM_RET_STOPPED (3):
                                the evaluation budget (ualm_set_budget), a deadline (ualm_wait_batch_for) or a cancel
                                (ualm_cancel_problems) stopped it, see above;
                                UALM_ELIMIT (-4): this problem exceeds the compiled limits (N <= 64, M <= 128) and was not solved --
                                the rest of its batch is unaffected.  Every problem within them is solved at any int_K that
                                ualm_set_params accepts, in any batch, bit for bit what it gives alone: on the parity path one
                                whose shared-memory layout does not fit four one-warp slots to a CTA is given a group of two or
                                four warps (with UALM_GROUPS=0, a developer switch, ualm_upload refuses such a batch instead) */
    int32_t outer_iters;
    int32_t n_evals;         /* cost+gradient evaluations */
    int32_t n_lbfgs_iters;   /* accepted line searches */
    int32_t last_lbfgs_ret;
    int32_t max_bound;
    int32_t sum_bound;       /* sum over L-BFGS iterations of the history depth used (bytes accounting) */
    int32_t reserved;
    double  inner_cost, jerk_cost, total_T, res_h, res_g, scale_fx, rho_final;
    double  piece_T_xy, piece_T_yaw;   /* the uniform piece durations getTraj() carries: T1(i) of the LAST evaluation
                                          (alm_traj_opt.h:257-261, se2traj.hpp:682-695); total_T is their N-fold sum */
} ualm_result_t;

typedef struct ualm_ctx ualm_ctx_t;

/* precision: 64 = parity path (IEEE double, bit-identical to the CPU oracle / the reference sources); 65 = "fast64", the
 * throughput path in double (re-associated reductions, FMA, prefactored MINCO system: not bit-reproducible); 32 = the
 * throughput path in float.  device = CUDA ordinal. */
int ualm_create(ualm_ctx_t **ctx, int device, int precision);
int ualm_destroy(ualm_ctx_t *ctx);
const char *ualm_last_error(void);
/* Run the work of the selected lane on a caller-owned CUDA stream.  The handle is taken literally: NULL is the legacy
 * default stream (torch.cuda.current_stream().cuda_stream == 0 when torch runs on its default stream).  ualm_reset_stream
 * goes back to the lane's own non-blocking stream.  ualm_solve_resident is asynchronous on that stream: follow it with
 * ualm_sync (or a stream-ordered consumer on the SAME stream) before touching its outputs. */
int ualm_set_stream(ualm_ctx_t *ctx, void *cuda_stream);
int ualm_reset_stream(ualm_ctx_t *ctx);
/* ---- environments ----
 * An environment is one parameter set (ualm_set_params) plus one map grid (ualm_set_map / ualm_set_map_f64).  A context holds up
 * to UALM_MAX_ENVS of them, and every problem of a batch names its own (the *_env entry points below; the entry points without
 * the suffix put every problem in environment 0).  A problem's result is exactly what it is in a batch of its environment alone.
 *   ualm_select_env(ctx, e): ualm_set_params / ualm_set_map / ualm_set_map_f64 bind environment e from now on (0 <= e <
 *                            UALM_MAX_ENVS; environment 0 is selected at creation).  Each environment owns its grid. */
#define UALM_MAX_ENVS 4
int ualm_select_env(ualm_ctx_t *ctx, int env);
/* ALMTrajOpt::init, for the selected environment.  int_K, mem_size and past are baked into uploaded batches: a parameter change
 * (of any environment) invalidates every resident batch (upload again before the next solve / eval); it is refused while a
 * submitted batch is in flight. */
int ualm_set_params(ualm_ctx_t *ctx, const ualm_params_t *p);
/* cells: host, [X][Y][Yaw][4] float {z, sigma, zbx, zby}, address x*Y*Yaw + y*Yaw + yaw (uneven_map.h:427-435), for the selected
 * environment.  One-time upload (replaces setEnvironment; the reference's map_buffer is private, uneven_map.h:91).  Refused while
 * a submitted batch is in flight. */
int ualm_set_map(ualm_ctx_t *ctx, const ualm_map_geom_t *g, const float *cells);
/* The reference's own grid: UnevenMap::map_buffer is RXS2 {double z, sigma; Vector2d zb} (uneven_map.h:36-64), i.e. 4 doubles
 * per cell in the same address order.  repack_to_float = 0 keeps the doubles on the device (82 MB for 200x200x64: bit parity
 * for maps built in-process by the reference); != 0 rounds them to the float4 grid of ualm_set_map (41 MB, what a map read
 * back from this repo's .umap file or from the reference's 6-digit CSV cache holds anyway). */
int ualm_set_map_f64(ualm_ctx_t *ctx, const ualm_map_geom_t *g, const double *cells, int repack_to_float);
/* Replace (or bind) the grid of the selected environment for every launch from now on; allowed while batches are in flight.
 * Work launched before the call keeps the grid it was launched with, bit for bit: batches in flight, and ualm_feasibility_batch
 * of a lane solved before the call.  Every later launch reads the new grid: ualm_submit_batch*, ualm_solve_resident,
 * ualm_solve_batch*, the phase entry points.  On return the new grid is complete on the device; the call never waits for
 * running batches.  On any error the previous grid stays current.  The geometry may differ from the previous grid's.  A null
 * ctx / g / cells or a voxel_num <= 0 is UALM_EINVAL.
 * Memory: the grid an environment had before an update stays allocated while a lane still holds it (a lane holds the grids its
 * last launch read until its next launch or ualm_destroy), so an environment holds at most one grid per such lane plus the
 * current one.  The grid is float4 (41 MB for 200x200x64); ualm_set_map_f64 keeps serving the double grid when nothing is in
 * flight.  ualm_set_map / ualm_set_map_f64 keep writing into the current grid in place. */
int ualm_update_map(ualm_ctx_t *ctx, const ualm_map_geom_t *g, const float *cells);
/* The same, with the grid built on the device from a point cloud (ualm_map_build_device's preprocessing and kernel) straight into
 * the new grid: no host round trip.  cells_out (optional, host) receives the grid, which the host front end needs
 * (ualm_astar_map_t reads sigma from it).  kernel_ms optional.  A null pts or npts < 0 is UALM_EINVAL as well.  The call queues
 * nothing behind a batch, but its kernel needs free SMs: on the parity path the solve holds them until its work queue runs dry, so
 * there the call can last into the tail of the batches in flight (DESIGN.md section 3h). */
int ualm_update_map_from_cloud(ualm_ctx_t *ctx, const float *pts, int64_t npts, const ualm_map_geom_t *g, double ellipsoid_x,
                               double ellipsoid_y, double ellipsoid_z, int iter_num, float *cells_out, float *kernel_ms);
/* Replace the cell columns [ix0, ix0+nx) x [iy0, iy0+ny), all yaw layers, of the selected environment's current grid, with the
 * guarantees of ualm_update_map: work launched before keeps its grid bit for bit, every later launch reads the new one, which is
 * complete on the device on return, and the call never waits for running batches.  Every cell outside the box is bit for bit the
 * previous grid's; a window never changes the geometry.  The new grid is a copy of the current one (staged through 8 MB of pinned
 * host memory, so only the copy engines serve it) with the box written over it: the call moves the grid twice over PCIe plus the
 * box, and never needs a free SM.
 * cells: nx*ny*W float4 {z, sigma, zb.x, zb.y}, in the grid's own [x][y][yaw] order restricted to the box.
 * No grid bound in the selected environment, or a double grid of ualm_set_map_f64: UALM_ESTATE.  A null argument, nx or ny <= 0,
 * or a box outside voxel_num: UALM_EINVAL.  On any error the previous grid stays current. */
int ualm_update_map_window(ualm_ctx_t *ctx, int ix0, int iy0, int nx, int ny, const float *cells);
/* The same box, built on the device from a point cloud, e.g. a local scan.  The preprocessing of ualm_map_build_device runs on this
 * cloud only, and the geometry is that of the current grid; inside the box the cells are bit for bit those a full
 * ualm_map_build_device of the same cloud with that geometry produces.  A cloud cut down to the box plus the ellipsoid's reach gives
 * the full cloud's cells up to float rounding (its bin grid starts elsewhere, so sums run in another order: DESIGN.md section 3h).
 * cells_out (optional, host) receives the box's cells in the layout above; kernel_ms (optional) is the CUDA-event time of the cell
 * kernel.  A null pts or npts < 0 is UALM_EINVAL as well.  Like ualm_update_map_from_cloud, the kernel needs a free SM slot, which on
 * the parity path can mean the tail of the batches in flight. */
int ualm_update_map_window_from_cloud(ualm_ctx_t *ctx, const float *pts, int64_t npts, int ix0, int iy0, int nx, int ny,
                                      double ellipsoid_x, double ellipsoid_y, double ellipsoid_z, int iter_num, float *cells_out,
                                      float *kernel_ms);
/* Move the selected environment's current grid by (dx, dy) whole cells, e.g. to keep a robot-centred grid around a robot that drives,
 * with the guarantees of ualm_update_map_window: a new version, complete on the device on return, made current; work launched before
 * keeps its grid and geometry bit for bit; every later launch, ualm_check_trajectories and ualm_submit_replan read the moved one; the
 * call never waits for running batches.  On any error the previous grid stays current and nothing is written.
 *   geometry: origin[0] + dx * xy_resolution and max_boundary[0] + dx * xy_resolution (one double expression each), likewise in y with
 *             dy; voxel_num, the resolutions and the yaw axis stay.
 *   cells:    new cell (x, y, w) is old cell (x + dx, y + dy, w) wherever that exists, bit for bit.  The cells without a source form at
 *             most two boxes of the new grid, all yaw layers:
 *               A, the x strip: [X - min(dx, X), X) x [0, Y) for dx > 0, [0, min(-dx, X)) x [0, Y) for dx < 0, none for dx = 0;
 *               B, the y strip over the x columns not in A: [Y - min(dy, Y), Y) for dy > 0, [0, min(-dy, Y)) for dy < 0.
 *             |dx| >= X or |dy| >= Y leaves no source: the whole grid is A and B.
 *   `cells` (host) holds A's cells, then B's, each in the window layout ([x][y][yaw] float4 restricted to the box).
 * The kept cells move from version to version through the 8 MB pinned staging buffer of the windows (each x row of the overlap is
 * contiguous in both), so the host-cells form only needs the copy engines, on both paths.
 * No grid bound in the selected environment, or a double grid of ualm_set_map_f64: UALM_ESTATE.  dx == dy == 0, a null ctx or cells:
 * UALM_EINVAL. */
int ualm_shift_map(ualm_ctx_t *ctx, int dx, int dy, const float *cells);
/* The same shift with A and B built on the device from a point cloud, e.g. a local scan: the cloud is preprocessed once with the
 * moved grid's crop, then map_build_kernel runs over both boxes.  Inside the boxes the cells are bit for bit those of a whole-grid
 * ualm_map_build_device of the same cloud with the moved geometry.  cells_out (optional, host) receives them in `cells`'s layout;
 * kernel_ms (optional) is the CUDA-event time of both launches.  A null pts or npts < 0 is UALM_EINVAL as well.  Like
 * ualm_update_map_window_from_cloud, the kernel needs a free SM slot, which on the parity path can mean the tail of the batches in
 * flight. */
int ualm_shift_map_from_cloud(ualm_ctx_t *ctx, const float *pts, int64_t npts, int dx, int dy, double ellipsoid_x, double ellipsoid_y,
                              double ellipsoid_z, int iter_num, float *cells_out, float *kernel_ms);

/* ---- batch solve = B independent optimizeSE2Traj calls ----
 * Ragged inputs are packed back to back in problem order: inner_xy has sum 2(N_b-1) doubles,
 * inner_yaw sum (M_b-1); outputs c_xy sum 12 N_b, c_yaw sum 6 M_b.  bnd is B x 18:
 * [init_xy(6) | end_xy(6) | init_yaw(3) | end_yaw(3)].  Host pointers. */
int ualm_solve_batch(ualm_ctx_t *ctx, int B, const int32_t *N, const int32_t *M, const double *bnd,
                     const double *total_time, const double *inner_xy, const double *inner_yaw,
                     ualm_result_t *results, double *c_xy, double *c_yaw);

/* The same in three steps, so a caller can keep inputs resident in HBM (bench `value`):
 *   upload (H2D) -> solve_resident (kernels only, asynchronous on the context stream) -> download (D2H). */
int ualm_upload(ualm_ctx_t *ctx, int B, const int32_t *N, const int32_t *M, const double *bnd,
                const double *total_time, const double *inner_xy, const double *inner_yaw);
/* The *_env forms take the arguments of their counterparts plus env[B], the environment of every problem (NULL = all 0; the
 * counterparts are these with env = NULL).  An index outside [0, UALM_MAX_ENVS) is UALM_EINVAL, an environment without both
 * parameters and a grid bound is UALM_ESTATE; nothing is touched on either error.  The budget (ualm_set_budget) and the deadline
 * (ualm_wait_batch_for) act on every problem of a batch alike.  ualm_eval_batch, ualm_init_scaling_batch,
 * ualm_feasibility_batch and ualm_mpc_export_batch use each problem's environment; ualm_time_penalty_kernel refuses a batch
 * that mixes environments (UALM_EINVAL). */
int ualm_upload_env(ualm_ctx_t *ctx, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                    const double *inner_xy, const double *inner_yaw, const int32_t *env);
int ualm_solve_batch_env(ualm_ctx_t *ctx, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                         const double *inner_xy, const double *inner_yaw, const int32_t *env, ualm_result_t *results, double *c_xy,
                         double *c_yaw);
/* ... with a parameter row per problem (ualm_problem_params_t above) */
int ualm_upload_pp(ualm_ctx_t *ctx, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                   const double *inner_xy, const double *inner_yaw, const int32_t *env, const ualm_problem_params_t *pp);
int ualm_solve_batch_pp(ualm_ctx_t *ctx, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                        const double *inner_xy, const double *inner_yaw, const int32_t *env, const ualm_problem_params_t *pp,
                        ualm_result_t *results, double *c_xy, double *c_yaw);
int ualm_solve_resident(ualm_ctx_t *ctx);
int ualm_sync(ualm_ctx_t *ctx);
int ualm_download(ualm_ctx_t *ctx, ualm_result_t *results, double *c_xy, double *c_yaw);
/* elapsed GPU time of the last solve_resident in ms (CUDA events on the context stream) and the
 * number of kernel launches it made */
int ualm_last_solve_ms(ualm_ctx_t *ctx, float *ms, int *launches);

/* ---- several batches in flight on one context ("lanes") ----
 * A lane is one resident batch with its own buffers, launch plan and streams; kernels of different lanes run concurrently, so
 * the slow tail of batch k (a few long-running trajectories) overlaps the bulk of batch k+1.
 *   ualm_select_lane(ctx, i): upload / solve_resident / sync / download / pack_records / last_solve_ms / eval / feasibility act
 *                             on lane i (0 <= i < ualm_max_lanes(); lane 0 is selected at creation).
 *   ualm_submit_batch:  upload + launch on the next lane of a `depth`-deep ring, returns a ticket without waiting for the solve
 *                       (host inputs are consumed before it returns); the batch then runs to completion on the device on both
 *                       paths.  UALM_ESTATE when that lane is still in flight.
 *   ualm_wait_batch:    blocks until the ticket's batch is complete, D2H of its results (same outputs as ualm_solve_batch).
 *   ualm_mark_begin / ualm_mark_end: CUDA-event time (ms) from the selected lane's stream at mark_begin to the completion of the
 *                       last solve of every lane at mark_end. */
int ualm_max_lanes(void);
int ualm_select_lane(ualm_ctx_t *ctx, int lane);
int ualm_submit_batch(ualm_ctx_t *ctx, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                      const double *inner_xy, const double *inner_yaw, int depth, int *ticket);
int ualm_submit_batch_env(ualm_ctx_t *ctx, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                          const double *inner_xy, const double *inner_yaw, const int32_t *env, int depth, int *ticket);
int ualm_submit_batch_pp(ualm_ctx_t *ctx, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                         const double *inner_xy, const double *inner_yaw, const int32_t *env, const ualm_problem_params_t *pp, int depth,
                         int *ticket);
int ualm_wait_batch(ualm_ctx_t *ctx, int ticket, ualm_result_t *results, double *c_xy, double *c_yaw);
/* ualm_wait_batch with a deadline: if the batch is not complete timeout_ms after the call, every problem of the batch is cancelled
 * as by ualm_cancel_problems (the problems still running stop at their next stop test with UALM_RET_STOPPED), the batch drains
 * and complete records come back.  The request ends with the batch: the next batch on the lane starts without one. */
int ualm_wait_batch_for(ualm_ctx_t *ctx, int ticket, double timeout_ms, ualm_result_t *results, double *c_xy, double *c_yaw);
/* Problems of a submitted batch that have finished since the last poll of this ticket, without waiting for the rest.
 * wait_ms = 0: return at once; > 0: block until at least one new problem is final or wait_ms has passed; < 0: UALM_EINVAL.
 * idx[0 .. *n_new) = their problem indices (capacity B of the ticket); each problem is returned exactly once per ticket.
 * Their records and coefficients are written at their problem-order positions of results / c_xy / c_yaw, the buffers and
 * layout ualm_wait_batch takes (c_xy / c_yaw may be NULL); other entries are not touched.  *n_pending = problems not yet
 * returned.  Every record and coefficient returned is bit for bit what ualm_wait_batch returns for that problem.
 * ualm_wait_batch / ualm_wait_batch_for after any number of polls behave exactly as today and return all B records.
 * A problem over the compiled limits (UALM_ELIMIT) is returned by the first poll; one the budget or a deadline stops is returned
 * when it stops (UALM_RET_STOPPED).  A null ctx, a bad ticket, wait_ms < 0 or a null idx / n_new / n_pending is UALM_EINVAL; a
 * ticket not in flight (also one already waited) is UALM_ESTATE.  Only tickets of ualm_submit_batch* can be polled.  On both
 * paths a submitted batch runs to completion on the device with no further host call, and each problem is published into the
 * ticket's mailbox from the device as it finishes; a poll only reads that mailbox, so the caller may sleep or do other work between
 * polls without holding any batch back. */
int ualm_poll_batch(ualm_ctx_t *ctx, int ticket, double wait_ms, int32_t *idx, int *n_new, int *n_pending,
                    ualm_result_t *results, double *c_xy, double *c_yaw);
/* Stop the listed problems of a submitted batch.  Each one stops at its next stop test, exactly as a deadline stops it
 * (UALM_RET_STOPPED, the trajectory of its last evaluation).  Problems that are already final keep their records bit for bit.
 * A problem not yet started runs to its first stop test.  Every other problem of the batch, and every other ticket, is
 * unaffected bit for bit.  Cancelled problems come back through ualm_poll_batch / ualm_wait_batch like any other.
 * A null ctx, a bad ticket, n < 0, a null idx with n > 0 or an index outside [0, B) is UALM_EINVAL; a ticket not in flight (also
 * one already waited) is UALM_ESTATE; a refused call raises nothing.  n = 0 does nothing; duplicate indices and repeated calls are
 * harmless.  Only tickets of ualm_submit_batch* can be cancelled, from the thread that polls.  On both paths the stop words are
 * raised by a copy on a stream of their own that lands while the batch runs, so the cancel reaches problems that are running
 * without any further host call. */
int ualm_cancel_problems(ualm_ctx_t *ctx, int ticket, int n, const int32_t *idx);
/* Evaluation budget per problem for the solves launched afterwards by every solving entry point (ualm_solve_batch,
 * ualm_solve_resident, ualm_submit_batch, ualm_solve_batch_multi through each context): max_evals = 0 (the default) is none,
 * negative values are UALM_EINVAL.  Refused (UALM_ESTATE) while a submitted batch is in flight. */
int ualm_set_budget(ualm_ctx_t *ctx, int32_t max_evals);
/* Urgent work: urgent = 1 makes the calls after it urgent until urgent = 0: ualm_submit_batch / ualm_submit_batch_env,
 * ualm_submit_replan (its build and the ticket it submits), ualm_check_trajectories and ualm_mpc_export_trajectories.  No other call changes.  Any other value or
 * a null ctx is UALM_EINVAL.  Allowed at any time, also while batches are in flight; like ualm_set_budget it acts on the calls made
 * after it.
 * Every record, coefficient, built replan row and check row is bit for bit what the same call gives without urgency, and so is
 * every other ticket's, on both paths: urgency only changes when work runs.
 * Parity path (precision 64): from the point an urgent piece of work is reached on its stream, every non-urgent solve launch of the
 * context (every ticket, and the batches of ualm_solve_resident / ualm_solve_batch) stops taking new problems from its work queue.
 * A problem already running is never interrupted; a launch's CTAs exit once their slots are between problems (a slot that stops may
 * join its CTA mate's problem, as at the end of the queue).  The held launches resume on the device, without a host call, when the
 * urgent work no longer needs slots: for an urgent ticket once every one of its problems has been taken (started, not finished),
 * so a ticket larger than the resident slots holds others back only until its last wave has started; for an urgent check or replan
 * build or held MPC export once its kernels have completed.  The urgent ticket's launches run on streams of the greatest priority.
 * Throughput path (precision 32 / 65): an urgent ticket's admission and round loops run on streams of the greatest priority.  The
 * check, the replan build and the held MPC export run on the greatest-priority check stream on both paths anyway, so urgency changes nothing else there.
 * Bound: the launches of a held solve wait at most 2 s in all (by the device's global timer, summed over every hold it meets); after
 * that the solve resumes and takes no further hold for the rest of its run, so a hold that is never released can only slow work
 * down, never hang the device.  The hold of an urgent ticket is raised after the submit's host-side allocations: a submit whose lane
 * must grow first waits for the device, as without urgency, and nothing is held meanwhile.  Cost: on the parity path every hold
 * leaves the SMs it empties idle until the urgent work is placed, so frequent urgent calls lower the throughput of everything else
 * (DESIGN.md section 3k).
 * Polls, cancels, deadlines (ualm_wait_batch_for) and the budget behave as documented on urgent and on held tickets; a held ticket's
 * deadline drain can be delayed by the hold, at most by the bound. */
int ualm_set_urgent(ualm_ctx_t *ctx, int urgent);
int ualm_mark_begin(ualm_ctx_t *ctx);
int ualm_mark_end(ualm_ctx_t *ctx, float *ms);

/* ---- several GPUs from one host process (SURVEY 8b item 4) ----
 * ctxs[r] lives on its own device with the same parameters and map bound (in every environment the batch uses).  The batch is dealt over the contexts (cost-sorted
 * snake), every device solves its shard concurrently, and the results come back in problem order.  There is no collective: the
 * problems never interact and one host gathers by D2H copies.  (One process per GPU: ualm_pack_records_device + an NCCL
 * all-gather of the records on the caller's communicator, uneven_planner_b200/distributed.py.) */
int ualm_solve_batch_multi(ualm_ctx_t **ctxs, int nctx, int B, const int32_t *N, const int32_t *M, const double *bnd,
                           const double *total_time, const double *inner_xy, const double *inner_yaw, ualm_result_t *results,
                           double *c_xy, double *c_yaw);
int ualm_solve_batch_multi_env(ualm_ctx_t **ctxs, int nctx, int B, const int32_t *N, const int32_t *M, const double *bnd,
                               const double *total_time, const double *inner_xy, const double *inner_yaw, const int32_t *env,
                               ualm_result_t *results, double *c_xy, double *c_yaw);
/* pp rows are dealt with their problems */
int ualm_solve_batch_multi_pp(ualm_ctx_t **ctxs, int nctx, int B, const int32_t *N, const int32_t *M, const double *bnd,
                              const double *total_time, const double *inner_xy, const double *inner_yaw, const int32_t *env,
                              const ualm_problem_params_t *pp, ualm_result_t *results, double *c_xy, double *c_yaw);

/* Fixed-stride result records for the multi-GPU all-gather: writes B records of `stride` doubles into
 * a DEVICE buffer (e.g. a torch tensor): [ret, outer, evals, iters, cost, jerk, T, res_h, res_g, N, M, pad,
 * c_xy(12N) , c_yaw(6M), zero pad].  stride >= 12 + 12 Nmax + 6 Mmax.  The _async form does not wait for the kernel. */
int ualm_pack_records_device(ualm_ctx_t *ctx, double *d_records, int stride);
int ualm_pack_records_device_async(ualm_ctx_t *ctx, double *d_records, int stride);

/* ---- phase entry points (kernel-level parity; SURVEY 8b item 3) ----
 * One innerCallback evaluation (alm_traj_opt.cpp:280-347) per problem of the uploaded batch at the given
 * decision vectors x (packed, n_b = 1+2(N_b-1)+(M_b-1)) with duals lambda[S_b], mu[6 S_b], scale_cx[7 S_b]
 * in the reference's index layout (alm_traj_opt.cpp:705-707, 832-946), S_b = N_b (int_K+1) with the int_K of problem b's
 * environment.
 * Outputs (host): f[B], grad (packed n_b), hx (packed S_b), gx (packed 6 S_b). Any input dual may be
 * NULL (zeros / ones).  scale_fx[B], rho scalar.  x NULL evaluates at the uploaded initial guesses; a given x does not
 * replace them. */
int ualm_eval_batch(ualm_ctx_t *ctx, const double *x, const double *lambda, const double *mu,
                    const double *scale_cx, const double *scale_fx, double rho,
                    double *f, double *grad, double *hx, double *gx, double *c_xy, double *c_yaw);
/* initScaling (alm_traj_opt.cpp:349-661) at the uploaded initial guesses: scale_fx[B], scale_cx packed 7 S_b */
int ualm_init_scaling_batch(ualm_ctx_t *ctx, double *scale_fx, double *scale_cx);
/* time `reps` back-to-back launches of the penalty-sampling kernel alone over the uploaded batch
 * (roofline of calConstrainCostGrad, alm_traj_opt.cpp:663-991): average ms per launch */
int ualm_time_penalty_kernel(ualm_ctx_t *ctx, int reps, float *ms_per_launch, double *algorithmic_bytes);

/* developer aid: per-phase SM-cycle counters of the last solve (thread 0 of every CTA) summed over the batch into out16[16]
 * (order: fill, LU, solve, jerk, tables, samples, accumulate, combine, adjoint, tail, two-loop, line-search, initScaling,
 * dual-update, other, total).  enable != 0 switches collection on for the following solves. */
int ualm_profile(ualm_ctx_t *ctx, int enable, long long *out16);

/* Post-solve quality scan of the solved resident batch (SURVEY 8f-4): ALMTrajOpt::getMaxVxAxAyCurAttSig
 * (alm_traj_opt.h:170-229) and SE2Trajectory::getNonHolError (se2traj.hpp:551-561), sampled every dt (0.01 in the
 * reference).  out10[10 * b + ...] = {max_vx, max_ax, max_ay, max_cur, max_att (= -min cos xi), max_sig, nonhol_error,
 * number of samples, T_xy piece duration, T_yaw piece duration}.  A trajectory whose duration would need more than 4e6 samples (a
 * diverged solve) is not scanned: zeros and a sample count of -1. */
int ualm_feasibility_batch(ualm_ctx_t *ctx, double dt, double *out10);

/* Limits of ualm_check_trajectories' six tests, as in ualm_params_t. */
typedef struct { double max_vel, max_acc_lon, max_acc_lat, max_kap, min_cxi, max_sig; } ualm_limits_t;
/* The scan of ualm_feasibility_batch over B trajectories the caller holds, e.g. those ualm_wait_batch / ualm_poll_batch returned,
 * against each problem's environment's grid as it is at the call (float or double; the version after every ualm_update_map* that
 * returned before).  Read-only: no solve, record or lane is touched, and it may be called while batches are in flight.
 * Inputs (host) in the layouts ualm_wait_batch returns: N[B], M[B], piece_T[2B] = {piece_T_xy, piece_T_yaw} of each record, packed
 * c_xy (12 N_b each) and c_yaw (6 M_b each); env[B] (NULL = all 0); t_from[B] (NULL = all 0).
 * Samples: the reference's t = 0, dt, 2dt.. formed by repeated addition, as ualm_feasibility_batch forms them; problem b keeps those
 * with t >= t_from[b] and t < its duration (the sequence is not restarted at t_from, so every kept sample is bit for bit the full
 * scan's).  out16[16 * b + ...]:
 *   0..9   ualm_feasibility_batch's ten values over the kept samples (signed abs-max of vx, ax, ay, cur, max att, max sig, the
 *          non-holonomic error summed in sample order, the number of kept samples, T_xy, T_yaw);
 *   10..15 the time of the first kept sample with |vx| > max_vel, |ax| > max_acc_lon, |ay| > max_acc_lat, |cur| > max_kap,
 *          att > -min_cxi (cos xi < min_cxi), sig > max_sig; -1 where none does.
 * The limits and gravity are each problem's environment's (ualm_set_params) unless `limits` (non-NULL) sets the six limits for the
 * whole call: a solve meets its constraints only at its int_K + 1 samples per piece, within epsilon_con, so a dense scan finds small
 * excursions and a caller sets its own margin here.  With t_from = 0, columns 0..9 equal ualm_feasibility_batch's on the same grid.
 * Not scanned (a sample count of -1, every time -1): a problem over the compiled limits (N > UALM_NMAX or M > UALM_MMAX; the rest of
 * the row 0) and one that would need more than 4e6 samples (0..6 zero, T_xy and T_yaw kept).  A t_from at or past the end keeps no
 * sample: the initial maxima (0, att -1, sig 0), a count of 0 and no violation.
 * A null ctx or pointer, B < 0, dt <= 0 (or NaN), N or M < 1, a negative or NaN t_from or an env outside [0, UALM_MAX_ENVS) is
 * UALM_EINVAL; an environment used without both parameters and a grid bound is UALM_ESTATE; out16 is not written on either.
 * The kernels run on a stream of the context that no solve occupies, created at the greatest priority; the call synchronises that
 * stream only.  On the throughput path a check gets SM slots between a batch's rounds; on the parity path the solve holds every SM
 * until its work queue runs dry, so there a check made in flight runs in the tail of the batches (DESIGN.md section 3i). */
int ualm_check_trajectories(ualm_ctx_t *ctx, int B, const int32_t *N, const int32_t *M, const double *piece_T, const double *c_xy,
                            const double *c_yaw, const int32_t *env, const double *t_from, double dt, const ualm_limits_t *limits,
                            double *out16);
/* The same with a parameter row per trajectory: row b's six limits are `limits` when that is non-NULL (call-wide, as above), otherwise
 * pp[b]'s, otherwise its environment's.  Gravity stays the environment's.  A non-finite field of pp is UALM_EINVAL (with out16 not
 * written), also when `limits` is given. */
int ualm_check_trajectories_pp(ualm_ctx_t *ctx, int B, const int32_t *N, const int32_t *M, const double *piece_T, const double *c_xy,
                               const double *c_yaw, const int32_t *env, const ualm_problem_params_t *pp, const double *t_from, double dt,
                               const ualm_limits_t *limits, double *out16);

/* Hand-over to the MPC for the solved batch of the selected lane, on the device (SURVEY 8f-3):
 *   (1) the mpc_controller/SE2Traj message PlanManager publishes (plan_manager.cpp:151-185, msg/SE2Traj.msg:1-9): pos_pts = the
 *       start point of every xy piece and the end point, (N + 1) x {x, y} per problem, posT_pts = the N piece durations,
 *       angle_pts (M + 1) / angleT_pts (M) likewise for yaw; problems packed back to back;
 *   (2) the trajectory the MPC tracks: TrajAnalyzer::setTraj (traj_anal.hpp:125-181) re-solves MINCO over those points with the
 *       message's init_v / init_a = {x, y, yaw} (NULL = zero, what the reference publishes) and zero tail derivatives, using
 *       MinJerkOpt::generate (minco_traj.hpp:365-444): c_mpc_xy / c_mpc_yaw in the layout of ualm_solve_batch's c_xy / c_yaw,
 *       bit-identical to that header compiled unmodified (tests/test_ref_pin.py + tests/test_gpu_mpc_export.py);
 *   (3) dev4[4 * b + ..] = {max |planned - tracked| position (m), its time, max |planned - tracked| yaw (rad), its time}, sampled
 *       every dt: the planned spline carries the boundary speed of plan_manager.cpp:93-94, the message does not.  The samples are
 *       t = 0, dt, 2dt, .. formed by repeated addition, kept while t < the shorter of the two durations (each the piece duration
 *       added once per piece); each time is that of the earliest sample among equal maxima (0 when the deviation is 0 throughout).
 *       A problem that would need 4e6 samples or more (duration / dt >= 4e6) is not scanned: {-1, 0, -1, 0}, while its message and
 *       re-solve are still written.
 * Any output pointer may be NULL.  Unsolved problems (ret_code UALM_ELIMIT) produce zeros.  The inputs are each problem's records as
 * the solve returned them, so a problem stopped by a budget, a deadline or a cancel is handed over with the trajectory it carries.
 * A null ctx, or dt <= 0 or NaN, is UALM_EINVAL; a lane without a solved batch (on the throughput path: not yet collected by
 * ualm_sync / ualm_download / a wait) is UALM_ESTATE; no output is written on either. */
int ualm_mpc_export_batch(ualm_ctx_t *ctx, double dt, const double *init_v, const double *init_a, double *pos_pts, double *posT_pts,
                          double *angle_pts, double *angleT_pts, double *c_mpc_xy, double *c_mpc_yaw, double *dev4);

/* The same hand-over for B trajectories the caller holds, each from its own start state, e.g. rows of batches ualm_poll_batch /
 * ualm_wait_batch returned, or of several lanes.  Inputs (host) in the layouts ualm_check_trajectories takes: N[B], M[B], piece_T[2B]
 * = {piece_T_xy, piece_T_yaw} of each record, packed c_xy (12 N_b each) and c_yaw (6 M_b each); init_v[3B] / init_a[3B] = {x, y, yaw}
 * per row, the message's boundary velocity / acceleration (NULL = zero, what the reference publishes; a replanned robot's message
 * carries its state at the replan time, ualm_submit_replan's bnd' entries 2, 3, 13 and 4, 5, 14).  Outputs as ualm_mpc_export_batch's,
 * packed row after row in call order; any output pointer may be NULL.  Row b is bit for bit what ualm_mpc_export_batch gives for the
 * same record with init_v + 3b / init_a + 3b, at every precision (the parity translation unit's double arithmetic).  A row over the
 * compiled limits (N > UALM_NMAX or M > UALM_MMAX) is zeros; a diverged record (infinite durations, or duration / dt >= 4e6) gets its
 * message and re-solve and dev4 = {-1, 0, -1, 0}.
 * Read-only: no grid, parameter, lane or record is read or touched (no environment needs to be bound), and it may be called while
 * batches are in flight.  It runs on the stream of ualm_check_trajectories and synchronises that stream only; under ualm_set_urgent
 * it goes ahead of the parity path's batches in flight as the check does, without it it waits there for SM slots in their tail.
 * A null ctx, or a null N, M, piece_T, c_xy or c_yaw with B > 0, B < 0, dt <= 0 or NaN, N or M < 1, a non-finite init_v / init_a
 * entry, or a row within the limits whose piece_T is NaN or <= 0 (a record ualm_poll_batch has not filled yet; +inf is a diverged
 * solve and is accepted) is UALM_EINVAL, and no output is written.  B = 0 is UALM_OK and writes nothing. */
int ualm_mpc_export_trajectories(ualm_ctx_t *ctx, int B, const int32_t *N, const int32_t *M, const double *piece_T, const double *c_xy,
                                 const double *c_yaw, const double *init_v, const double *init_a, double dt, double *pos_pts,
                                 double *posT_pts, double *angle_pts, double *angleT_pts, double *c_mpc_xy, double *c_mpc_yaw, double *dev4);

/* UnevenMap construction on the GPU (SURVEY 8f-1: UnevenMap::init preprocessing on the host, then constructMap + filter,
 * uneven_map.cpp:317-398, 5-43, one thread per (x, y, yaw) cell).  Same arguments and the same arithmetic as ualm_map_build
 * below (csrc/map_cell.h is compiled for both sides): the cells are bit-identical to the host builder's.  cells: host
 * buffer [X][Y][Yaw][4] float; kernel_ms (optional): CUDA-event time of the cell kernel. */
int ualm_map_build_device(ualm_ctx_t *ctx, const float *pts, int64_t npts, const ualm_map_geom_t *g, double ellipsoid_x,
                          double ellipsoid_y, double ellipsoid_z, int iter_num, float *cells, float *kernel_ms);

/* =====================  host-side input pipeline (no GPU needed)  ===================== */

/* UnevenMap::init cloud preprocessing + constructMap (uneven_map.cpp:127-163, 317-398, 5-43) on host
 * threads.  pts: npts x 3 float (x,y,z) as read from the .pcd.  cells out: [X][Y][Yaw][4] float.
 * ellipsoid = {0.2,0.1,0.1}, iter_num = 2 in every reference yaml. */
int ualm_map_build(const float *pts, int64_t npts, const ualm_map_geom_t *g, double ellipsoid_x,
                   double ellipsoid_y, double ellipsoid_z, int iter_num, int nthreads, float *cells);
/* the cloud ualm_map_build / ualm_map_build_device work on for a grid centred at the world origin: UnevenMap::init's CropBox
 * [-10, 10]^2 + 1 cm VoxelGrid (uneven_map.cpp:133-143), as xyz floats (a grid centred at c crops [c - 10, c + 10]^2 instead).  Returns the number of points (pts_out may be NULL to query it; UALM_ELIMIT when max_pts is too small). */
int64_t ualm_map_preprocess_cloud(const float *pts, int64_t npts, double ellipsoid_x, double ellipsoid_y, double ellipsoid_z, float *pts_out,
                                  int64_t max_pts);
/* occupancy (uneven_map.cpp:169-179): occ3[X*Y*Yaw], occ2[X*Y] (1 = occupied) */
int ualm_map_occupancy(const float *cells, const ualm_map_geom_t *g, double min_cnormal, double max_rho,
                       uint8_t *occ3, uint8_t *occ2);

/* Initial-guess path (stands in for KinoAstar::plan, front_end/src/kino_astar.cpp:67-236, whose one-shot is
 * the same Dubins curve family, kino_astar.h:242-258): shortest forward Dubins path start->goal with
 * turning radius `radius`, sampled every `ds` metres as (x,y,yaw).  Returns the number of points written
 * (<= max_pts) or a negative error. */
int ualm_dubins_path(const double start[3], const double goal[3], double radius, double ds, double *path_xyyaw,
                     int max_pts);

/* PlanManager::rcvWpsCallBack input contract (plan_manager/src/plan_manager.cpp:62-122): yaw unwrap, boundary
 * states, arc-length resampling into inner xy / yaw waypoints, total_time.  Outputs: bnd[18], inner_xy
 * (2 x (N-1)), inner_yaw (M-1); returns 0 and sets *N, *M, *total_time. */
int ualm_resample_path(const double *path_xyyaw, int npts, double piece_len, double yaw_piece_times,
                       double mean_vel, double init_time_times, double init_sig_vel, double *bnd,
                       double *inner_xy, int max_inner_xy, double *inner_yaw, int max_inner_yaw, int32_t *N,
                       int32_t *M, double *total_time);

/* ---- front-end: KinoAstar (SURVEY 8f-2) ---- */
/* kino_astar/* parameters (front_end/src/kino_astar.cpp:7-20) */
typedef struct {
    double yaw_resolution, lambda_heu, weight_r2, weight_so2, weight_v_change, weight_delta_change, weight_sigma;
    double time_interval, collision_interval, oneshot_range, wheel_base, max_steer, max_vel;
} ualm_astar_params_t;
/* plan_manager/params/run_*.yaml:16-30 (the same values in every terrain file) */
void ualm_astar_default_params(ualm_astar_params_t *p);
/* what KinoAstar reads of UnevenMap (isOccupancy, isOccupancyXY, isInMap, getTerrainSig; uneven_map.h:389-500): the cell grid
 * ([X][Y][Yaw][4] = z, sigma, zb.x, zb.y; float as ualm_set_map takes it, or double as ualm_set_map_f64 does -- one of the two) and
 * the occupancy grids of ualm_map_occupancy (occ3: [X][Y][Yaw], occ2: [X][Y]) */
typedef struct {
    const ualm_map_geom_t *geom;
    const float *cells;
    const double *cells64;
    const uint8_t *occ3, *occ2;
} ualm_astar_map_t;
/* plan_manager/* parameters of the resampler (plan_manager.cpp:24-30; run_hill.yaml:57-62) */
typedef struct { double piece_len, yaw_piece_times, mean_vel, init_time_times, init_sig_vel; } ualm_resample_params_t;

/* Replanned problems of B trajectories the caller holds, from each robot's state at time t_from[b] on its trajectory to the goal of
 * its original problem, submitted as one ticket.  Inputs (host) in the layouts ualm_wait_batch returns, as for ualm_check_trajectories:
 * N[B], M[B], piece_T[2B] = {piece_T_xy, piece_T_yaw} of each record, packed c_xy (12 N_b each) and c_yaw (6 M_b each); bnd[18B], the
 * original problems' boundary states; env[B] (NULL = all 0); t_from[B].  rp: the resampler's parameters (NULL = run_*.yaml's piece_len
 * 0.3, yaw_piece_times 2, mean_vel 0.5, init_time_times 1.2; init_sig_vel is not used).  Row b is built as follows:
 *   duration = min(N T_xy, M T_yaw), each summed by repeated addition as ualm_check_trajectories sums it;
 *   the state at tau = t_from[b]: init_xy = [px, py, vx, vy, ax, ay], init_yaw = [yaw, dyaw, ddyaw] (yaw as the trajectory carries
 *   it, not normalised), from the reference's piece lookup for uniform durations (se2traj.hpp:343-361);
 *   the polyline: the point (x, y, yaw) at tau, the points at every t of the check's sequence t = 0, dt, 2dt.. (the same additions)
 *   with tau < t < duration, then the goal (the position of bnd's end_xy, the angle of its end_yaw);
 *   PlanManager's resampler on it, its steps in its order (yaw smoothing, pm.cpp:62-77; arc-length resampling and total_time,
 *   pm.cpp:96-122, bit for bit ualm_resample_path's arithmetic): N', M', inner_xy, inner_yaw, total_time;
 *   bnd' = [init_xy | bnd's end_xy | init_yaw | bnd's end_yaw] (a moving start state, within optimizeSE2Traj's 2 x 3 head state).
 * The B problems are then submitted exactly as ualm_submit_batch_env submits the returned arrays with env, on the next lane of the
 * `depth` ring: *ticket and row b of it = row b of the inputs, for ualm_poll_batch / ualm_cancel_problems / ualm_wait_batch(_for) and
 * the budget as for any ticket.  Outputs: N_out[B], M_out[B], bnd_out[18B], total_time_out[B] and, optional, inner_xy_out /
 * inner_yaw_out at a fixed stride of UALM_REPLAN_INNER_XY / UALM_REPLAN_INNER_YAW doubles per row, zeros past the row's points.
 * A row over the compiled limits (N' > 64 or M' > 128) keeps its counts, zero inner points, and is submitted as ualm_submit_batch_env
 * submits such a problem (a UALM_ELIMIT record from the first poll, zero coefficients).  The build's work per row is bounded: a
 * polyline that would need more than 4095 waypoints of either kind, a yaw of magnitude 2^40 or more, or more than 65536 whole turns of
 * yaw smoothing in all is cut short and reported as N' = M' = 4097, an over-limit row; its total_time is still its whole length's.
 * The build is the same bits at every precision.
 * A null ctx or pointer, B < 0, dt <= 0 (or NaN), depth outside [1, UALM_MAX_LANES], N or M < 1, a t_from that is negative, NaN or not
 * before the row's duration, a duration / dt >= 4e6, a non-finite piece_T, c_xy or c_yaw entry (a diverged solve) or goal entry of bnd
 * (6..11, 15..17), an rp field (but init_sig_vel) <= 0 or NaN, or an env out of range is UALM_EINVAL; an environment without
 * parameters and a grid, or the next lane still in flight, is UALM_ESTATE.  These are decided before anything is built.  One refusal
 * comes after the build: a row whose polyline has zero or non-finite length (a robot already at its goal; coordinates whose squares
 * overflow) has no usable total_time and is UALM_EINVAL for the call.  On every refusal no output is written and no lane is taken.
 * B = 0 is ualm_submit_batch_env with B = 0.  The build reads no grid; it runs on the stream of ualm_check_trajectories and synchronises that stream only, so in
 * flight on the parity path it waits for SM slots in the batches' tail (DESIGN.md section 3j). */
#define UALM_REPLAN_INNER_XY 126       /* 2 (64 - 1) */
#define UALM_REPLAN_INNER_YAW 127      /* 128 - 1 */
int ualm_submit_replan(ualm_ctx_t *ctx, int B, const int32_t *N, const int32_t *M, const double *piece_T, const double *c_xy,
                       const double *c_yaw, const double *bnd, const int32_t *env, const double *t_from, double dt,
                       const ualm_resample_params_t *rp, int depth, int *ticket, int32_t *N_out, int32_t *M_out, double *bnd_out,
                       double *total_time_out, double *inner_xy_out, double *inner_yaw_out);
/* The same with a parameter row per trajectory: row b of the ticket solves with pp[b] (ualm_submit_batch_pp of the returned arrays).
 * The build reads no parameter and gives the same bits.  A non-finite field of pp is refused with the refusals decided before the
 * build. */
int ualm_submit_replan_pp(ualm_ctx_t *ctx, int B, const int32_t *N, const int32_t *M, const double *piece_T, const double *c_xy,
                          const double *c_yaw, const double *bnd, const int32_t *env, const ualm_problem_params_t *pp, const double *t_from,
                          double dt, const ualm_resample_params_t *rp, int depth, int *ticket, int32_t *N_out, int32_t *M_out,
                          double *bnd_out, double *total_time_out, double *inner_xy_out, double *inner_yaw_out);

/* KinoAstar::plan(start_state, end_state) (front_end/src/kino_astar.cpp:67-236): hybrid A* over (x, y, yaw) with 3 x 5 motion
 * primitives and a Dubins one-shot near the goal.  Writes the (x, y, yaw) polyline start .. goal and returns its number of points;
 * 0 = no path (start or goal occupied, open set exhausted, node pool exhausted), like the reference's empty vector.
 * n_expanded (optional): nodes closed.  The Dubins curve is OMPL's in the reference (absent here): csrc/dubins.h restates it. */
int ualm_kino_astar_plan(const ualm_astar_map_t *map, const ualm_astar_params_t *p, const double start[3], const double goal[3],
                         double *path_xyyaw, int max_pts, int *n_expanded);

/* The one-shot curve of KinoAstar::asignShotTraj alone (kino_astar.h:246-258, without its occupancy test): the shortest Dubins curve of
 * turning radius `radius` sampled every `interval` metres from its start; *length (optional) receives its length. */
int ualm_dubins_shot(const double start[3], const double goal[3], double radius, double interval, double *path_xyyaw, int max_pts, double *length);

/* The reference's whole front half for B (start, goal) pairs, one search per host thread (nthreads <= 0: all cores):
 * KinoAstar::plan -> PlanManager's resampler (ualm_resample_path).  Outputs are the ragged arrays ualm_solve_batch /
 * ualm_submit_batch take, packed back to back for the problems that have a path and fit the optimizer's limits; packed[b] = index of
 * pair b in them or -1; n_expanded[b] (optional) = nodes closed.  Returns the number of packed problems (or a negative error;
 * UALM_ELIMIT when cap_xy / cap_yaw doubles are not enough). */
int ualm_front_end_batch(const ualm_astar_map_t *map, const ualm_astar_params_t *ap, const ualm_resample_params_t *rp, int B,
                         const double *starts, const double *goals, int nthreads, int32_t *N, int32_t *M, double *bnd, double *total_time,
                         double *inner_xy, long long cap_xy, double *inner_yaw, long long cap_yaw, int32_t *packed, int32_t *n_expanded);

#ifdef __cplusplus
}
#endif
#endif
