// ualm_tp_host.h -- internal C++ interface between the C ABI (ualm_api.cu) and the throughput engine (ualm_tp.cu).
// The engine is its own translation unit because it is compiled with FMA contraction on (the parity path needs -fmad=false).
#pragma once

#include <cstdint>
#include <string>
#include <vector>

#include "ualm.h"

// The host-side layout of one uploaded batch, built and validated once by the C ABI (ualm_api.cu: batch_layout) for both paths.
// skip[b]: problem b is over the compiled limits (UALM_NMAX / UALM_MMAX); it is not solved, its record says UALM_ELIMIT, and n[b] =
// S[b] = 0.  off_x / off_s advance over the solved problems only, off_cxy / off_cyaw over all.  x0: the solved problems' initial
// decision vectors [logC2(total_time) | inner_xy | inner_yaw], packed at off_x.  Nmax / Mmax: maxima over the solved problems (>= 1)
struct BatchLayout {
    int B = 0, Nmax = 1, Mmax = 1, n_active = 0;
    std::vector<int32_t> N, M, env, n, S;
    std::vector<unsigned char> skip;
    std::vector<long long> off_x, off_s, off_cxy, off_cyaw;
    std::vector<double> x0;
    // pp[8 b ..]: problem b's ualm_problem_params_t (the batch's row, or its environment's first eight ualm_params_t fields)
    std::vector<double> pp;
    long long tot_x = 0, tot_s = 0, tot_cxy = 0, tot_cyaw = 0;
    // every problem grouped by environment (ascending within one, skipped ones included): environment e at eidx[eoff[e], eoff[e + 1])
    std::vector<int> eidx;
    int eoff[UALM_MAX_ENVS + 1] = {};
    unsigned env_mask = 0;               // bit e set: the batch has a problem in environment e
    bool mixed() const { return (env_mask & (env_mask - 1)) != 0; }
};

namespace ualm_tp {

struct TpEngine;

// every function returns UALM_OK or a negative UALM_E* code; *err receives the message
int tp_create(TpEngine **e, int device, int precision, std::string *err);
void tp_destroy(TpEngine *e);
// parameters / grid of environment `env` (0 <= env < UALM_MAX_ENVS)
int tp_set_params(TpEngine *e, int env, const ualm_params_t *p, std::string *err);
// the grid the batches admitted from now on read: a device buffer of the context ([X][Y][Yaw] float4), which stays allocated and
// unchanged while a batch admitted with it is in flight (ualm_api.cu keeps every such version).  Also encodes its TMA descriptor
void tp_bind_map(TpEngine *e, int env, const ualm_map_geom_t *g, const float4 *cells);
// lanes = tickets: a lane holds one uploaded batch; admit puts it into the pool of running trajectories and launches the round loop
// of each of its groups on the device, collect waits for those loops to end and gathers the batch's results on the device.  The
// caller has validated the batch (L), checked that the lane is not in flight, and keeps L unchanged until the lane's next upload;
// bnd[18 B] and total_time[B] are the arrays L was built from
int tp_upload(TpEngine *e, int lane, const BatchLayout &L, const double *bnd, const double *total_time, std::string *err);
// asynchronous: the batch runs to completion without further calls.  publish: the group loops copy the batch's problems into the
// lane's result mailbox as they finish (ualm_submit_batch, for tp_poll)
int tp_admit(TpEngine *e, int lane, std::string *err, bool publish = false, bool urgent = false);   // urgent: admission and group loops on greatest-priority streams
// ualm_poll_batch on a lane admitted with publish: reads the mailbox only (wait_ms > 0: yield-polls its flags until a problem is
// new or wait_ms has passed); it neither synchronises nor queues anything
int tp_poll(TpEngine *e, int lane, double wait_ms, int32_t *idx, int *n_new, int *n_pending, ualm_result_t *results, double *c_xy, double *c_yaw,
            std::string *err);
// ualm_cancel_problems on a lane admitted with publish: raises the stop words idx[0, n) (the caller checked n and idx) by a copy on
// the cancel stream, which reaches the rounds that are running.  UALM_ESTATE when the lane is not in flight, UALM_EINVAL for an index
// outside [0, B); nothing is raised on either
int tp_cancel(TpEngine *e, int lane, int n, const int32_t *idx, std::string *err);
// blocks until the lane's group loops have ended.  timeout_ms >= 0: once that much time has passed since the call, every stop word
// of the lane's batch is raised (its trajectories stop at their next stop test) and the loops drain
int tp_collect(TpEngine *e, int lane, std::string *err, double timeout_ms = -1.0);
void tp_set_budget(TpEngine *e, int max_evals);              // evaluation budget of the solves admitted afterwards (no batch in flight)
int tp_download(TpEngine *e, int lane, ualm_result_t *results, double *c_xy, double *c_yaw, std::string *err);
int tp_pack_records(TpEngine *e, int lane, double *d_records, int stride, std::string *err);
bool tp_lane_in_flight(TpEngine *e, int lane);
bool tp_lane_collected(TpEngine *e, int lane);
int tp_last_solve(TpEngine *e, int lane, float *ms, int *launches);
int tp_mark_begin(TpEngine *e, std::string *err);
int tp_mark_end(TpEngine *e, float *ms, std::string *err);
// kernel-level entry points over the lane's uploaded batch (mode 1: one innerCallback at the given x / duals; mode 2: initScaling)
int tp_eval(TpEngine *e, int lane, const double *x, const double *lambda, const double *mu, const double *scale_cx, const double *scale_fx, double rho,
            double *f, double *grad, double *hx, double *gx, double *c_xy, double *c_yaw, std::string *err);
int tp_init_scaling(TpEngine *e, int lane, double *scale_fx, double *scale_cx, std::string *err);
// time `reps` launches of kb_kernel alone over the lane's batch (the trajectories sit at their initial guess); UALM_EINVAL when the
// batch mixes environments
int tp_time_penalty(TpEngine *e, int lane, int reps, int use_tma, float *ms_per_launch, double *algorithmic_bytes, std::string *err);
// device pointers of the lane's gathered outputs (for the post-solve scan)
int tp_lane_outputs(TpEngine *e, int lane, const ualm_result_t **d_res, const double **d_cxy, const double **d_cyaw);

} // namespace ualm_tp
