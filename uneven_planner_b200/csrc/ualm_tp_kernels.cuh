// ualm_tp_kernels.cuh -- the THROUGHPUT path of the batched MINCO / PHR-ALM / L-BFGS optimizer (precision 32 and 65 of include/ualm.h).
//
// Same algorithm as the parity path (ualm_kernels.cuh; reference: back_end/src/alm_traj_opt.cpp:168-347, 349-661, 663-991,
// utils/lbfgs.hpp:276-722, utils/se2traj.hpp:595-816, uneven_map.h:258-377), laid out for throughput instead of for bit parity:
//
//   * LOCKSTEP EVALUATION ROUNDS with continuous batching.  A pool of trajectory slots holds every problem in flight (several
//     batches).  One round = one cost/gradient evaluation of every active trajectory, as three bulk kernels:
//       ka_kernel  one WARP per trajectory: finishes the previous evaluation (gradient assembly through the tables), runs the
//                  per-trajectory control flow up to the next evaluation request (Lewis-Overton line search, L-BFGS two-loop on the
//                  coalesced [slot][n] history, ALM dual update / convergence) and the MINCO coefficients of the new point;
//       ks_kernel  (rounds after an admission only) initScaling, one CTA per new trajectory, one thread per constraint sample;
//       kb_kernel  the per-constraint-sample penalty cost + gradient (calConstrainCostGrad): one CTA per trajectory, one thread per
//                  sample, the UnevenMap tiles of the pieces staged into shared memory by TMA (cp.async.bulk.tensor + mbarrier),
//                  duals / scales / constraint values streamed as coalesced SoA arrays, gradients reduced onto the control
//                  points in shared memory.
//     Finished trajectories leave the active list, new ones join between rounds: no trajectory waits for a batch mate.
//   * The MINCO system is NONDIMENSIONALISED AND SOLVED ONCE: piece durations are uniform (alm_traj_opt.h:257-261), so
//     A(T) = R(T) A(1) C(T) with diagonal R = diag(T^-ord), C = diag(T^k), and A(1) depends only on the piece count P.  A MINCO
//     right-hand side is non-zero in P + 5 rows only (head / tail position, velocity, acceleration and the P - 1 waypoints), so
//     the P + 5 columns of A(1)^-1 those rows excite are tabulated per piece count at engine creation and an evaluation needs NO
//     banded solve at all:  c = C^-1 W b^ (rows over lanes),  dcost/dq = W^T C^-1 dcost/dc (waypoints over lanes),  and because the
//     T-dependence of c is explicit (c^ = c^0 + T c^1 + T^2 c^2) so is dc/dT -- the adjoint solve and the B1/B2 contraction of
//     calGradCTtoQT (se2traj.hpp:751-816) collapse into one dot product with z = dc/dT.  initScaling uses the same tables.
//   * Mixed precision: ka_kernel (short serial chains, latency bound) always computes in double; the penalty kernel computes
//     in R = float (precision 32) or double (precision 65); duals, constraint values, exchanged gradients and the L-BFGS history are
//     stored in R.
// FMA contraction is on, libm sincos/atan2 are CUDA's, reductions are re-associated: results are NOT bit-comparable with the oracle;
// tests/test_gpu_tp.py bounds the difference per evaluation and reports the end-to-end distribution (BASELINE config 5's sweep).
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ualm.h"

namespace ualm_tp {

#define TP_NMAX 64
#define TP_MMAX 128
#define TP_NVAR 256                     // >= 1 + 2 (NMAX - 1) + (MMAX - 1)
#define TP_CSTRIDE (12 * TP_NMAX + 6 * TP_MMAX)   // per-slot coefficient block: c_xy (6N x 2 column-major) at 0, c_yaw at 12 * TP_NMAX
#define TP_CYAW (12 * TP_NMAX)
#define TP_TSTRIDE (TP_NMAX + TP_MMAX)  // per-slot time-gradient block: gdT_xy at 0, gdT_yaw at TP_NMAX
#define TP_NDUAL 21                     // dual block fields (each S long): 0 lambda | 1..6 mu | 7..13 scale_cx | 14 hx | 15..20 gx
#define TP_FW 14                        // doubles per LU factor row: 13 band entries + 1 / diagonal
#define TP_FPAD 6                       // zero rows before and after each factor table
#define TP_KA_WARPS 4
#define TP_HRING 8                      // two-loop history ring slots in shared memory (cp.async, TP_HRING - 1 steps ahead)
#define TP_KB_THREADS 128
#define TP_TILE 8                       // map tile = 8 x 8 cells x 8 yaw layers of float4 = 8 KB
#define TP_TILE_BYTES (TP_TILE * TP_TILE * TP_TILE * 16)
#define TP_MAXPPC 7                     // pieces per sample chunk (<= TP_KB_THREADS / (K + 1))
#define TP_MAX_TICKETS 64
#define TP_SUBGROUPS 4                  // every batch in flight is split into up to this many independently advancing groups
#define TP_MAXLANES 16                  // batches in flight (= UALM_MAX_LANES of ualm_api.cu)
#define TP_NGROUPS (TP_MAXLANES * TP_SUBGROUPS)   // lanes x subgroups: each group has its own stream, active list and round sequence

#define TP_DELTA_SIGL 0.01
#define TP_CUR_SCALE 10.0
#define TP_SIG_SCALE 1000.0
#define TP_SCALE_TRICK_JERK 1000.0

enum { PH_FREE = 0, PH_NEW, PH_REQ_FIRST, PH_REQ_LS, PH_REQ_EVALONLY, PH_DONE };

// lbfgs return codes (lbfgs.hpp:135-184)
enum {
    LB_CONVERGENCE = 0, LB_STOP, LB_CANCELED,
    LBERR_UNKNOWNERROR = -1024, LBERR_INVALID_N, LBERR_INVALID_MEMSIZE, LBERR_INVALID_GEPSILON, LBERR_INVALID_TESTPERIOD, LBERR_INVALID_DELTA,
    LBERR_INVALID_MINSTEP, LBERR_INVALID_MAXSTEP, LBERR_INVALID_FDECCOEFF, LBERR_INVALID_SCURVCOEFF, LBERR_INVALID_MACHINEPREC,
    LBERR_INVALID_MAXLINESEARCH, LBERR_INVALID_FUNCVAL, LBERR_MINIMUMSTEP, LBERR_MAXIMUMSTEP, LBERR_MAXIMUMLINESEARCH, LBERR_MAXIMUMITERATION,
    LBERR_WIDTHTOOSMALL, LBERR_INVALIDPARAMETERS, LBERR_INCREASEGRADIENT,
};

// what is per environment; the eight per-problem values (ualm_problem_params_t) are the slot's TpState::pp
struct TpParams {
    int use_scaling;
    double rho, beta, gamma, epsilon_con, max_iter, g_epsilon, min_step, delta;
    int inner_max_iter, mem_size, past, int_K;
    double gravity;
    int max_evals;          // evaluation budget per problem (ualm_set_budget), 0 = none
};

struct TpMap {
    const float4 *cells;   // {z, sigma, zbx, zby}
    int vn[3];
    double origin[3], maxb[3], xy_res, yaw_res, xy_inv, yaw_inv;
};

struct TpState {
    int phase, N, M, n, S, ticket, index, need_scale;
    int mode, group, padm1, padm2;   // 0 = solve, 1 = one evaluation at the given duals (kernel-level parity), 2 = initScaling only
    int n_evals, iters_total, outer_iter, last_ret, ret_code, max_bound, sum_bound, pad0;
    int k, end, bound, ls_count, brackt, touched, pad1, pad2;
    double fx, step, stp, ls_mu, ls_nu, dginit, finit, dgtest, dstest;
    double pf[16];
    double rho, scale_fx, inner_cost, res_h, res_g;
    double tau, T, Tx, Ty, jerk_raw;          // of the last forward solve (the state getTraj() / the dual update see, SURVEY Q1)
    double f_last;
    double bnd[18];
    double pp[8];           // the problem's ualm_problem_params_t (its row, or its environment's values), written by admit_kernel
};

struct TpPool {
    int capacity, m, K, Smax, use_tma, ka_col_bytes, ka_hist_stride, ka_hist_bytes;
    TpState *st;
    int *active;            // [TP_NGROUPS][capacity] active slot list per group
    int *n_active;          // [TP_NGROUPS]
    int *remaining;         // per ticket: trajectories not yet done
    // per lane: its stop words, one per problem of its batch (ualm_cancel_problems, ualm_wait_batch_for); the host may raise them
    // while a round runs
    const int *stop[TP_MAXLANES];
    double *vec;            // [cap][5][TP_NVAR]  x | g | xp | gp | d
    double *cd;             // [cap][TP_CSTRIDE]  coefficients of the last forward solve (double)
    double *gw;             // [cap][TP_CSTRIDE]  z = dc/dT(piece) of the last forward solve (same layout as cd)
    void *cr;               // [cap][TP_CSTRIDE]  R copy of the coefficients for the sample kernels (== cd when R is double)
    void *gdc;              // [cap][TP_CSTRIDE]  R  constraint part of dcost/dc from kb_kernel
    void *gdt;              // [cap][TP_TSTRIDE]  R  constraint part of dcost/dT
    double *kb_cost;        // [cap]              constraint cost
    void *dual;             // [cap][TP_NDUAL * Smax]  R  (field f of slot s at s * 21 * Smax + f * S_slot)
    void *hs, *hy;          // [cap][m][TP_NVAR]  R  L-BFGS history, vector j of slot s at (s * m + j) * TP_NVAR
    double *lm_ys, *lm_alpha;   // [cap][m]
    const double *wf;       // W[P][j][r]  = A(1)^-1 (r, J(j)), j < P + 5 (rhs_row): (P + 5) x 6P at wf_off[P]
    const long long *wf_off;
    const double *wt;       // WT[P][r][w] = A(1)^-1 (r, 6w + 5): 6P x (P - 1) at wway_off[P] (the waypoint columns, transposed)
    const void *wway;       // R  the waypoint columns again, [w][r]: (P - 1) x 6P at wway_off[P]  (ks_kernel)
    const long long *wway_off;
    long long *prof;        // developer profile: [16] SM-cycle sums per ka phase (lane 0 of every warp), or null
};
enum { KP_FIN_PRE = 0, KP_FIN_SWEEP, KP_FIN_POST, KP_ADV_LS, KP_ADV_POST, KP_TWOLOOP, KP_ALM, KP_FWD_PRE, KP_FWD_SWEEP, KP_FWD_POST, KP_SCALEZ, KP_WARPS, KP_N };
struct KProf {
    long long *p; long long last;
    __device__ __forceinline__ void start(long long *pp, int lane) { p = lane == 0 ? pp : nullptr; if (p) last = clock64(); }
    __device__ __forceinline__ void mark(int ph) { if (p) { const long long c = clock64(); atomicAdd((unsigned long long *)&p[ph], (unsigned long long)(c - last)); last = c; } }
};

// ---------------------------------------------------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double expC2(double tau) { return tau > 0.0 ? ((0.5 * tau + 1.0) * tau + 1.0) : 1.0 / ((0.5 * tau - 1.0) * tau + 1.0); } // alm_traj_opt.h:232-235
__device__ __forceinline__ double dTdtau(double tau)   // getTtoTauGrad, alm_traj_opt.h:244-253
{
    if (tau > 0) return tau + 1.0;
    const double den = (0.5 * tau - 1.0) * tau + 1.0;
    return (1.0 - tau) / (den * den);
}
__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_max(double v)
{
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
template <class T>
__device__ __forceinline__ double vdot(const double *a, const T *b, int n, int lane)
{
    double s = 0.0;
    for (int i = lane; i < n; i += 32) s += a[i] * (double)b[i];
    return warp_sum(s);
}
__device__ __forceinline__ double vabsmax(const double *a, int n, int lane)
{
    double m = 0.0;
    for (int i = lane; i < n; i += 32) m = fmax(m, fabs(a[i]));
    return warp_max(m);
}

// derivative order of row r of the MINCO system of P pieces (se2traj.hpp:609-674): the row scale of A(T) = R(T) A(1) C(T) is T^-ord
__device__ __host__ __forceinline__ int row_ord(int r, int n6)
{
    if (r < 3) return r;
    if (r >= n6 - 3) return r - (n6 - 3);
    const int tt = (r - 3) % 6;
    return tt == 0 ? 3 : tt == 1 ? 4 : tt == 4 ? 1 : tt == 5 ? 2 : 0;
}

// entry A(r, c) of the P-piece system at T = 1 (se2traj.hpp:609-674)
__device__ __host__ inline double a1_entry(int P, int r, int c)
{
    const int n6 = 6 * P;
    if (c < 0 || c >= n6 || r < 0 || r >= n6) return 0.0;
    if (r < 3) return c == r ? (r == 2 ? 2.0 : 1.0) : 0.0;
    if (r >= n6 - 3) {
        const int e = c - (n6 - 6), tr = r - (n6 - 3);
        if (e < 0) return 0.0;
        const double pos[6] = {1, 1, 1, 1, 1, 1}, vel[6] = {0, 1, 2, 3, 4, 5}, acc[6] = {0, 0, 2, 6, 12, 20};
        return tr == 0 ? pos[e] : tr == 1 ? vel[e] : acc[e];
    }
    const int i = (r - 3) / 6, tt = (r - 3) - 6 * i, e = c - 6 * i;
    if (e < 0 || e > 11) return 0.0;
    switch (tt) {
    case 0: return e == 3 ? 6.0 : e == 4 ? 24.0 : e == 5 ? 60.0 : e == 9 ? -6.0 : 0.0;          // jerk continuity
    case 1: return e == 4 ? 24.0 : e == 5 ? 120.0 : e == 10 ? -24.0 : 0.0;                     // snap continuity
    case 2: return e <= 5 ? 1.0 : 0.0;                                                          // waypoint
    case 3: return e <= 5 ? 1.0 : e == 6 ? -1.0 : 0.0;                                          // position continuity
    case 4: return (e >= 1 && e <= 5) ? (double)e : e == 7 ? -1.0 : 0.0;                        // velocity continuity
    default: return e == 2 ? 2.0 : e == 3 ? 6.0 : e == 4 ? 12.0 : e == 5 ? 20.0 : e == 8 ? -2.0 : 0.0;   // acceleration continuity
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// engine set-up: LU of A(1) for every piece count (banded_system.hpp:66-91, no pivoting), and the waypoint rows of A(1)^-T
// ---------------------------------------------------------------------------------------------------------------------
__global__ void lu_tables_kernel(double *lu, const int *lu_off, int Pmax)
{
    const int P = blockIdx.x * blockDim.x + threadIdx.x + 1;
    if (P > Pmax) return;
    const int n6 = 6 * P;
    double *F = lu + lu_off[P];
    for (int r = -TP_FPAD; r < n6 + TP_FPAD; r++)
        for (int q = 0; q < TP_FW; q++) F[r * TP_FW + q] = (r >= 0 && r < n6 && q < 13) ? a1_entry(P, r, r - 6 + q) : 0.0;
    for (int k = 0; k < n6; k++) {
        const double piv = F[k * TP_FW + 6];
        const int last = min(k + 6, n6 - 1);
        for (int i = k + 1; i <= last; i++) {
            double &l = F[i * TP_FW + 6 - (i - k)];
            if (l == 0.0) continue;
            l = l / piv;
            for (int j = k + 1; j <= last; j++) {
                const double u = F[k * TP_FW + 6 + (j - k)];
                if (u != 0.0) F[i * TP_FW + 6 + (j - i)] -= l * u;
            }
        }
    }
    for (int r = 0; r < n6; r++) F[r * TP_FW + 13] = 1.0 / F[r * TP_FW + 6];
}

// A(1) x = b in place (one thread, plain loops; set-up only)
__device__ inline void solve_a1_serial(const double *F, int n6, double *b)
{
    for (int r = 0; r < n6; r++) {
        double v = b[r];
        for (int d = 1; d <= 6 && r - d >= 0; d++) v -= F[r * TP_FW + 6 - d] * b[r - d];
        b[r] = v;
    }
    for (int r = n6 - 1; r >= 0; r--) {
        double v = b[r];
        for (int d = 1; d <= 6 && r + d < n6; d++) v -= F[r * TP_FW + 6 + d] * b[r + d];
        b[r] = v * F[r * TP_FW + 13];
    }
}
// Row of the MINCO right-hand side that column j < P + 5 of the tables belongs to (se2traj.hpp:609-674): 0..2 head position /
// velocity / acceleration, then the P - 1 waypoint rows 6w + 5, then the three tail rows
__device__ __host__ __forceinline__ int rhs_row(int P, int j) { return j < 3 ? j : (j < P + 2 ? 6 * (j - 3) + 5 : 6 * P - 3 + (j - (P + 2))); }

// One thread per (piece count, column): solve A(1) x = e_row in place in the W table, then scatter the waypoint columns into
// the transposed table and the R copy ks_kernel reads
template <class R>
__global__ void w_tables_kernel(const double *lu, const int *lu_off, double *wf, const long long *wf_off, double *wt, R *wway, const long long *wway_off, int Pmax)
{
    const int P = blockIdx.y + 1;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (P > Pmax || j >= P + 5) return;
    const int n6 = 6 * P;
    double *b = wf + wf_off[P] + (size_t)j * n6;
    for (int r = 0; r < n6; r++) b[r] = 0.0;
    b[rhs_row(P, j)] = 1.0;
    solve_a1_serial(lu + lu_off[P], n6, b);
    if (j >= 3 && j < P + 2) {
        const int w = j - 3;
        double *t = wt + wway_off[P];
        R *o = wway + wway_off[P] + (size_t)w * n6;
        for (int r = 0; r < n6; r++) { t[(size_t)r * (P - 1) + w] = b[r]; o[r] = (R)b[r]; }
    }
}

__device__ __forceinline__ void cp_async16(unsigned dst, const void *src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int NP>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(NP) : "memory"); }

// jerk energy of one piece and its T-derivative (se2traj.hpp:702-707, 739-744); a = first column block, b = second (or null)
__device__ __forceinline__ void jerk_piece(const double *a, const double *b, double T1, double T2, double T3, double T4, double T5, double &e, double &gt)
{
    double d33 = a[3] * a[3], d43 = a[4] * a[3], d44 = a[4] * a[4], d53 = a[5] * a[3], d54 = a[5] * a[4], d55 = a[5] * a[5];
    if (b) { d33 += b[3] * b[3]; d43 += b[4] * b[3]; d44 += b[4] * b[4]; d53 += b[5] * b[3]; d54 += b[5] * b[4]; d55 += b[5] * b[5]; }
    e = 36.0 * d33 * T1 + 144.0 * d43 * T2 + 192.0 * d44 * T3 + 240.0 * d53 * T3 + 720.0 * d54 * T4 + 720.0 * d55 * T5;
    gt = 36.0 * d33 + 288.0 * d43 * T1 + 576.0 * d44 * T2 + 720.0 * d53 * T2 + 2880.0 * d54 * T3 + 3600.0 * d55 * T4;
}
__device__ __forceinline__ double jerk_gc(const double *c6, int k, double T1, double T2, double T3, double T4, double T5)   // se2traj.hpp:719-737
{
    const double c3 = c6[3], c4 = c6[4], c5 = c6[5];
    if (k == 5) return 240.0 * c3 * T3 + 720.0 * c4 * T4 + 1440.0 * c5 * T5;
    if (k == 4) return 144.0 * c3 * T2 + 384.0 * c4 * T3 + 720.0 * c5 * T4;
    if (k == 3) return 72.0 * c3 * T1 + 144.0 * c4 * T2 + 240.0 * c5 * T3;
    return 0.0;
}
struct SlotView {
    TpState *st;
    double *x, *g, *xp, *gp, *d;
    double *cd, *gw;
    double *sm;                // this warp's buffer in shared memory (12N + 6M doubles; aliased by the two-loop's history ring)
    int N, M, n, S, slot;
};

__device__ __forceinline__ SlotView slot_view(const TpPool &E, int slot, double *sm)
{
    SlotView v;
    v.slot = slot;
    v.sm = sm;
    v.st = E.st + slot;
    v.N = v.st->N; v.M = v.st->M; v.n = v.st->n; v.S = v.st->S;
    double *vb = E.vec + (size_t)slot * 5 * TP_NVAR;
    v.x = vb; v.g = vb + TP_NVAR; v.xp = vb + 2 * TP_NVAR; v.gp = vb + 3 * TP_NVAR; v.d = vb + 4 * TP_NVAR;
    v.cd = E.cd + (size_t)slot * TP_CSTRIDE;
    v.gw = E.gw + (size_t)slot * TP_CSTRIDE;
    return v;
}

__device__ __forceinline__ void load6(const double *p, double (&w)[6])
{
    const double2 a = __ldg((const double2 *)p), b = __ldg((const double2 *)p + 1), c = __ldg((const double2 *)p + 2);
    w[0] = a.x; w[1] = a.y; w[2] = b.x; w[3] = b.y; w[4] = c.x; w[5] = c.y;
}

// one 6-coefficient block out of the table pass: c_k = c^_k T^-k, z_k = dc_k/dT = T^-k dc^_k/dT - k c_k / T; stores c (double and
// the sample kernels' R copy) and z, returns the block's jerk energy
// (se2traj.hpp:697-710, 852-855: per piece 36 c3^2 T + 144 c3 c4 T^2 + 192 c4^2 T^3 + 240 c3 c5 T^3 + 720 c4 c5 T^4 + 720 c5^2 T^5)
template <class R>
__device__ __forceinline__ double emit_block(const double (&ch)[6], const double (&eh)[6], double T1, double *c, R *cr, double *z)
{
    const double rT = 1.0 / T1;
    double inv[6];
    inv[0] = 1.0;
#pragma unroll
    for (int k = 1; k < 6; k++) inv[k] = inv[k - 1] * rT;
    double c6[6];
#pragma unroll
    for (int k = 0; k < 6; k++) {
        c6[k] = ch[k] * inv[k];
        c[k] = c6[k];
        if (sizeof(R) != sizeof(double)) cr[k] = (R)c6[k];
        z[k] = eh[k] * inv[k] - (double)k * c6[k] * rT;
    }
    const double T2 = T1 * T1, T3 = T2 * T1, T4 = T2 * T2, T5 = T4 * T1;
    return 36.0 * c6[3] * c6[3] * T1 + 144.0 * c6[4] * c6[3] * T2 + 192.0 * c6[4] * c6[4] * T3 + 240.0 * c6[5] * c6[3] * T3 + 720.0 * c6[5] * c6[4] * T4 +
           720.0 * c6[5] * c6[5] * T5;
}

// MINCO forward for the decision vector in v.x (alm_traj_opt.cpp:293-299 + se2traj.hpp:595-680) through the tabulated columns of
// A(1)^-1: one lane per piece (both columns of an xy piece share the table loads), a loop over the P + 5 excitable right-hand-side
// rows, no dependence between lanes.  Leaves the coefficients in v.cd (and their R copy), z = dc/dT(piece) in v.gw, and
// T / Tx / Ty / jerk_raw in the state
template <class R>
__device__ void minco_forward(const TpPool &E, const SlotView &v, int lane, KProf &kp)
{
    TpState *st = v.st;
    const int N = v.N, M = v.M, nx = 6 * N;
    const double tau = v.x[0];
    const double T = expC2(tau), Tx = T / (double)N, Ty = T / (double)M;
    // nondimensional right-hand sides (se2traj.hpp:615-617, 672-674 scaled by T^ord): [head p, v T, a T^2 | waypoints | tail p, v T, a T^2]
    double *bx = v.sm, *by = bx + (N + 5), *bw = by + (N + 5);
    const double *bnd = st->bnd;
    const double *Pxy = v.x + 1, *Pyaw = v.x + 1 + 2 * (N - 1);
    if (lane < 2) {
        const int d = lane;
        double *b = d ? by : bx;
        b[0] = bnd[d]; b[1] = bnd[d + 2] * Tx; b[2] = bnd[d + 4] * Tx * Tx;
        b[N + 2] = bnd[6 + d]; b[N + 3] = bnd[6 + d + 2] * Tx; b[N + 4] = bnd[6 + d + 4] * Tx * Tx;
    }
    if (lane == 2) {
        bw[0] = bnd[12]; bw[1] = bnd[13] * Ty; bw[2] = bnd[14] * Ty * Ty;
        bw[M + 2] = bnd[15]; bw[M + 3] = bnd[16] * Ty; bw[M + 4] = bnd[17] * Ty * Ty;
    }
    for (int i = lane; i < N - 1; i += 32) { bx[3 + i] = Pxy[2 * i]; by[3 + i] = Pxy[2 * i + 1]; }
    for (int i = lane; i < M - 1; i += 32) bw[3 + i] = Pyaw[i];
    __syncwarp();
    kp.mark(KP_FWD_PRE);
    const double *Wn = E.wf + E.wf_off[N], *Wm = E.wf + E.wf_off[M];
    double *c = v.cd, *z = v.gw;
    R *cr = (R *)E.cr + (size_t)v.slot * TP_CSTRIDE;
    double e = 0.0;
    // One code path for xy and yaw pieces (a yaw lane carries an unused second column): lanes only differ in trip count, so the
    // warp never executes the two kinds one after the other.  Four table rows in flight per step: the loop is bound by the latency
    // of its loads, not by their number; rows past the end are clamped and weighted zero.
    for (int q = lane; q < N + M; q += 32) {
        const bool isy = q >= N;
        const int P = isy ? M : N, i = isy ? q - N : q, n6 = 6 * P, nj = P + 5;
        const double *Wp = (isy ? Wm : Wn) + 6 * i;
        const double *b0 = isy ? bw : bx, *b1 = isy ? bw : by;
        const double T1 = isy ? Ty : Tx;
        double a0[6] = {0, 0, 0, 0, 0, 0}, a1[6] = {0, 0, 0, 0, 0, 0};
        for (int j0 = 0; j0 < nj; j0 += 4) {
            double wa[6], wb[6], wc[6], wd[6];
            const int j1 = min(j0 + 1, nj - 1), j2 = min(j0 + 2, nj - 1), j3 = min(j0 + 3, nj - 1);
            load6(Wp + (size_t)j0 * n6, wa); load6(Wp + (size_t)j1 * n6, wb); load6(Wp + (size_t)j2 * n6, wc); load6(Wp + (size_t)j3 * n6, wd);
            const double xa = b0[j0], ya = b1[j0];
            const double xb = j0 + 1 < nj ? b0[j1] : 0.0, yb = j0 + 1 < nj ? b1[j1] : 0.0;
            const double xc = j0 + 2 < nj ? b0[j2] : 0.0, yc = j0 + 2 < nj ? b1[j2] : 0.0;
            const double xd = j0 + 3 < nj ? b0[j3] : 0.0, yd = j0 + 3 < nj ? b1[j3] : 0.0;
#pragma unroll
            for (int k = 0; k < 6; k++) {
                a0[k] += wa[k] * xa; a1[k] += wa[k] * ya; a0[k] += wb[k] * xb; a1[k] += wb[k] * yb;
                a0[k] += wc[k] * xc; a1[k] += wc[k] * yc; a0[k] += wd[k] * xd; a1[k] += wd[k] * yd;
            }
        }
        // dc^/dT: the velocity (T) and acceleration (T^2) columns only
        double e0[6], e1[6];
        {
            double wa[6], wb[6], wc[6], wd[6];
            load6(Wp + (size_t)1 * n6, wa); load6(Wp + (size_t)(P + 3) * n6, wb); load6(Wp + (size_t)2 * n6, wc); load6(Wp + (size_t)(P + 4) * n6, wd);
            const double t2 = 2.0 * T1;
            const double vh0 = isy ? bnd[13] : bnd[2], vt0 = isy ? bnd[16] : bnd[8], ah0 = t2 * (isy ? bnd[14] : bnd[4]), at0 = t2 * (isy ? bnd[17] : bnd[10]);
            const double vh1 = bnd[3], vt1 = bnd[9], ah1 = t2 * bnd[5], at1 = t2 * bnd[11];
#pragma unroll
            for (int k = 0; k < 6; k++) {
                e0[k] = vh0 * wa[k] + vt0 * wb[k] + (ah0 * wc[k] + at0 * wd[k]);
                e1[k] = vh1 * wa[k] + vt1 * wb[k] + (ah1 * wc[k] + at1 * wd[k]);
            }
        }
        const int off0 = isy ? TP_CYAW + 6 * i : 6 * i;
        e += emit_block<R>(a0, e0, T1, c + off0, cr + off0, z + off0);
        if (!isy) e += emit_block<R>(a1, e1, T1, c + nx + 6 * i, cr + nx + 6 * i, z + nx + 6 * i);
    }
    kp.mark(KP_FWD_SWEEP);
    e = warp_sum(e);
    if (lane == 0) { st->tau = tau; st->T = T; st->Tx = Tx; st->Ty = Ty; st->jerk_raw = e; }
    __syncwarp();
    kp.mark(KP_FWD_POST);
}

// ---------------------------------------------------------------------------------------------------------------------
// ka_kernel pieces
// ---------------------------------------------------------------------------------------------------------------------
// finish the evaluation whose sample part kb_kernel left in gdc / gdt / kb_cost: f -> st->f_last, gradient -> v.g
// (alm_traj_opt.cpp:318-346; se2traj.hpp:751-816 through the tables: dq = W^T C^-1 dcost/dc, dT = z . dcost/dc + explicit terms)
template <class R>
__device__ void finish_eval(const TpPool &E, const TpParams &p, const SlotView &v, int lane, KProf &kp)
{
    TpState *st = v.st;
    const int N = v.N, M = v.M, nx = 6 * N;
    const double Tx = st->Tx, Ty = st->Ty, scale_fx = st->scale_fx;
    const double js = (p.use_scaling ? TP_SCALE_TRICK_JERK : 1.0) * scale_fx;
    const double X1 = Tx, X2 = Tx * Tx, X3 = X2 * Tx, X4 = X2 * X2, X5 = X4 * Tx;
    const double Y1 = Ty, Y2 = Ty * Ty, Y3 = Y2 * Ty, Y4 = Y2 * Y2, Y5 = Y4 * Ty;
    const double *c = v.cd, *z = v.gw;
    double *sm = v.sm;             // g^ = C^-1 dcost/dc: x at [0, 6N), y at [6N, 12N), yaw at [12N, 12N + 6M)
    const R *gdc = (const R *)E.gdc + (size_t)v.slot * TP_CSTRIDE;
    const R *gdt = (const R *)E.gdt + (size_t)v.slot * TP_TSTRIDE;
    double ix[6], iy[6];
    ix[0] = iy[0] = 1.0;
#pragma unroll
    for (int k = 1; k < 6; k++) { ix[k] = ix[k - 1] / Tx; iy[k] = iy[k - 1] / Ty; }
    // dcost/dc = jerk part + constraint part (alm_traj_opt.cpp:322-332); one lane per 6-coefficient block: the jerk gradient
    // needs c3..c5 of the block only (se2traj.hpp:719-737).  Its dot product with z is the implicit part of the time gradient
    double sx = 0.0, sy = 0.0;
    for (int blk = lane; blk < 2 * N + M; blk += 32) {
        const bool isy = blk >= 2 * N;
        const int off = isy ? TP_CYAW + 6 * (blk - 2 * N) : 6 * blk;
        const double T1 = isy ? Y1 : X1, T2 = isy ? Y2 : X2, T3 = isy ? Y3 : X3, T4 = isy ? Y4 : X4, T5 = isy ? Y5 : X5;
        const double c3 = c[off + 3], c4 = c[off + 4], c5 = c[off + 5];
        double g6[6];
#pragma unroll
        for (int k = 0; k < 6; k++) g6[k] = (double)gdc[off + k];
        g6[3] += (72.0 * c3 * T1 + 144.0 * c4 * T2 + 240.0 * c5 * T3) * js;
        g6[4] += (144.0 * c3 * T2 + 384.0 * c4 * T3 + 720.0 * c5 * T4) * js;
        g6[5] += (240.0 * c3 * T3 + 720.0 * c4 * T4 + 1440.0 * c5 * T5) * js;
        double td = 0.0;
#pragma unroll
        for (int k = 0; k < 6; k++) td += g6[k] * z[off + k];
        if (isy) {
            sy += td;
            double *o = sm + 12 * N + 6 * (blk - 2 * N);
#pragma unroll
            for (int k = 0; k < 6; k++) o[k] = g6[k] * iy[k];
        } else {
            sx += td;
            double *o = sm + 6 * blk;
#pragma unroll
            for (int k = 0; k < 6; k++) o[k] = g6[k] * ix[k];
        }
    }
    // explicit time dependence of the jerk energy and of the constraint samples, per piece (se2traj.hpp:739-744; gdt from kb_kernel)
    for (int q = lane; q < N + M; q += 32) {
        const bool isy = q >= N;
        const int i = isy ? q - N : q;
        const double T1 = isy ? Ty : Tx, T2 = T1 * T1, T3 = T2 * T1, T4 = T2 * T2, T5 = T4 * T1;
        double e, gj;
        jerk_piece(c + (isy ? TP_CYAW : 0) + 6 * i, isy ? nullptr : c + nx + 6 * i, T1, T2, T3, T4, T5, e, gj);
        const double gt = gj * js + (double)gdt[isy ? TP_NMAX + i : i];
        if (isy) sy += gt; else sx += gt;
    }
    sx = warp_sum(sx); sy = warp_sum(sy);
    __syncwarp();
    kp.mark(KP_FIN_PRE);
    // waypoint gradients: one lane per waypoint (x and y of an xy waypoint share the table loads), a loop over the rows.  One code
    // path for both kinds (a yaw lane reads its vector twice); twelve table rows in flight per step, the second six weighted zero
    // past the end (branch-free, so that all loads are issued before the first use)
    const double *WTn = E.wt + E.wway_off[N], *WTm = E.wt + E.wway_off[M];
    for (int q = lane; q < (N - 1) + (M - 1); q += 32) {
        const bool isy = q >= N - 1;
        const int w = isy ? q - (N - 1) : q, sd = isy ? M - 1 : N - 1, nr = isy ? 6 * M : nx;
        const double *t = (isy ? WTm : WTn) + w;
        const double *ga = isy ? sm + 2 * nx : sm, *gb = isy ? ga : sm + nx;
        double a0 = 0.0, a1 = 0.0, a2 = 0.0, b0 = 0.0, b1 = 0.0, b2 = 0.0;
        for (int r = 0; r < nr; r += 12) {
            const bool h2 = r + 6 < nr;
            const int r2 = h2 ? r + 6 : r;
            const double hw = h2 ? 1.0 : 0.0;
            const double w0 = __ldg(t + (size_t)r * sd), w1 = __ldg(t + (size_t)(r + 1) * sd), w2 = __ldg(t + (size_t)(r + 2) * sd);
            const double w3 = __ldg(t + (size_t)(r + 3) * sd), w4 = __ldg(t + (size_t)(r + 4) * sd), w5 = __ldg(t + (size_t)(r + 5) * sd);
            const double u0 = __ldg(t + (size_t)r2 * sd), u1 = __ldg(t + (size_t)(r2 + 1) * sd), u2 = __ldg(t + (size_t)(r2 + 2) * sd);
            const double u3 = __ldg(t + (size_t)(r2 + 3) * sd), u4 = __ldg(t + (size_t)(r2 + 4) * sd), u5 = __ldg(t + (size_t)(r2 + 5) * sd);
            a0 += w0 * ga[r]; b0 += w0 * gb[r]; a1 += w1 * ga[r + 1]; b1 += w1 * gb[r + 1]; a2 += w2 * ga[r + 2]; b2 += w2 * gb[r + 2];
            a0 += w3 * ga[r + 3]; b0 += w3 * gb[r + 3]; a1 += w4 * ga[r + 4]; b1 += w4 * gb[r + 4]; a2 += w5 * ga[r + 5]; b2 += w5 * gb[r + 5];
            const double v0 = u0 * hw, v1 = u1 * hw, v2 = u2 * hw, v3 = u3 * hw, v4 = u4 * hw, v5 = u5 * hw;
            a0 += v0 * ga[r2]; b0 += v0 * gb[r2]; a1 += v1 * ga[r2 + 1]; b1 += v1 * gb[r2 + 1]; a2 += v2 * ga[r2 + 2]; b2 += v2 * gb[r2 + 2];
            a0 += v3 * ga[r2 + 3]; b0 += v3 * gb[r2 + 3]; a1 += v4 * ga[r2 + 4]; b1 += v4 * gb[r2 + 4]; a2 += v5 * ga[r2 + 5]; b2 += v5 * gb[r2 + 5];
        }
        if (isy) v.g[1 + 2 * (N - 1) + w] = (a0 + a1) + a2;
        else { v.g[1 + 2 * w] = (a0 + a1) + a2; v.g[2 + 2 * w] = (b0 + b1) + b2; }
    }
    kp.mark(KP_FIN_SWEEP);
    if (lane == 0) {
        const double tau = st->tau;
        const double rho_T = st->pp[0];
        v.g[0] = (rho_T * scale_fx + sx / (double)N + sy / (double)M) * dTdtau(tau);
        st->f_last = st->jerk_raw * js + E.kb_cost[v.slot] + rho_T * st->T * scale_fx;
    }
    __syncwarp();
    kp.mark(KP_FIN_POST);
}

template <class H>
__device__ __forceinline__ H *hist(void *base, const TpPool &E, int slot, int j) { return (H *)base + ((size_t)slot * E.m + j) * TP_NVAR; }

// start of a line search from (x, fx, g, d, step): lbfgs.hpp:276-316.  Returns 0 and leaves the first trial point in v.x, or the
// (negative) error code
__device__ int ls_begin(const SlotView &v, int lane)
{
    TpState *st = v.st;
    const int n = v.n;
    for (int q = lane; q < n; q += 32) { v.xp[q] = v.x[q]; v.gp[q] = v.g[q]; }
    __syncwarp();
    const double dginit = vdot(v.gp, v.d, n, lane);
    const double stp = st->step;
    if (!(stp > 0.0)) return LBERR_INVALIDPARAMETERS;
    if (0.0 < dginit) return LBERR_INCREASEGRADIENT;
    if (lane == 0) {
        st->ls_count = 0; st->brackt = 0; st->touched = 0; st->stp = stp; st->ls_mu = 0.0; st->ls_nu = 1.0e20;
        st->dginit = dginit; st->finit = st->fx; st->dgtest = 1.0e-4 * dginit; st->dstest = 0.9 * dginit;
    }
    for (int q = lane; q < n; q += 32) v.x[q] = v.xp[q] + stp * v.d[q];
    __syncwarp();
    return 0;
}

// the stop predicate of include/ualm.h (UALM_RET_STOPPED), tested where earlyExit is and by the ALM loop after judgeConvergence.
// Lane 0 alone reads the trajectory's stop word and broadcasts it: a raise that lands in the middle of a round cannot split the
// warp's decision
__device__ __forceinline__ bool stop_requested(const TpPool &E, const TpParams &p, const TpState *st, int lane)
{
    int c = 0;
    if (lane == 0) c = ((const volatile int *)E.stop[st->ticket])[st->index];
    c = __shfl_sync(0xffffffffu, c, 0);
    return (p.max_evals > 0 && st->n_evals >= p.max_evals) || c != 0;
}

// the stop test at the earlyExit point; a stop that fires is marked in ret_code for the ALM loop (alm_ends)
__device__ __forceinline__ bool stop_fires(const TpPool &E, const TpParams &p, TpState *st, int lane)
{
    const bool s = stop_requested(E, p, st, lane);
    if (s && lane == 0) st->ret_code = UALM_RET_STOPPED;
    return s;
}

// the ALM loop's exits after judgeConvergence failed (alm_traj_opt.cpp:262-267): the stop fired inside the inner solve that just
// ended or holds now (UALM_RET_STOPPED), else ++iter > max_iter (2).  Not inlined: inside ka_kernel (128 registers) the stop test
// costs a spill
__device__ __noinline__ bool alm_ends(const TpPool &E, const TpParams &p, TpState *st, int lane)
{
    if (st->ret_code == UALM_RET_STOPPED || stop_requested(E, p, st, lane)) { if (lane == 0) st->ret_code = UALM_RET_STOPPED; return true; }
    const int iter = st->outer_iter + 1;
    if (lane == 0) st->outer_iter = iter;
    if ((double)iter > p.max_iter) { if (lane == 0) st->ret_code = 2; return true; }
    return false;
}

// one ka step for a trajectory whose evaluation at v.x has just been finished: runs the optimizer's control flow up to the next
// evaluation request (returns the new phase) or to the end of the solve (PH_DONE).  alm_traj_opt.cpp:234-271, lbfgs.hpp:439-722
template <class R>
__device__ int advance(const TpPool &E, const TpParams &p, const SlotView &v, int lane, KProf &kp)
{
    TpState *st = v.st;
    const int n = v.n, m = p.mem_size;
    int ph = st->phase;
    const double fnew = st->f_last;
    int lret = 0;                  // lbfgs_optimize return code once it ends
    bool ended = false;
    if (ph == PH_REQ_FIRST) {      // lbfgs.hpp:523-550
        if (lane == 0) { st->fx = fnew; st->pf[0] = fnew; }
        for (int q = lane; q < n; q += 32) v.d[q] = -v.g[q];
        __syncwarp();
        const double gn = vabsmax(v.g, n, lane), xn = vabsmax(v.x, n, lane);
        if (gn / fmax(1.0, xn) < p.g_epsilon) { lret = LB_CONVERGENCE; ended = true; }
        else {
            const double dd = vdot(v.d, v.d, n, lane);
            if (lane == 0) { st->step = 1.0 / sqrt(dd); st->k = 1; st->end = 0; st->bound = 0; }
            __syncwarp();
            const int r = ls_begin(v, lane);
            if (r < 0) { lret = r; ended = true; for (int q = lane; q < n; q += 32) { v.x[q] = v.xp[q]; v.g[q] = v.gp[q]; } }
            else return PH_REQ_LS;
        }
    } else {                       // PH_REQ_LS: line_search_lewisoverton after the evaluation of a trial point (lbfgs.hpp:318-388)
        const double fx = fnew, finit = st->finit;
        int count = st->ls_count + 1;
        double stp = st->stp, mu = st->ls_mu, nu = st->ls_nu;
        int brackt = st->brackt, touched = st->touched;
        int ls = 0;
        bool done = false;
        if (isinf(fx) || isnan(fx)) { ls = LBERR_INVALID_FUNCVAL; done = true; }
        else if (p.past > 0 && fabs(finit - fx) / (fabs(finit) + 1.0) < p.delta / (double)p.past) { ls = count; done = true; }   // lbfgs.hpp:327-330
        else {
            if (fx > finit + stp * st->dgtest) { nu = stp; brackt = 1; }
            else {
                const double dg = vdot(v.g, v.d, n, lane);
                if (dg < st->dstest) mu = stp;
                else { ls = count; done = true; }
            }
            if (!done) {
                if (64 <= count) { ls = LBERR_MAXIMUMLINESEARCH; done = true; }
                else if (brackt && (nu - mu) < 1.0e-16 * nu) { ls = LBERR_WIDTHTOOSMALL; done = true; }
                else {
                    stp = brackt ? 0.5 * (mu + nu) : stp * 2.0;
                    if (stp < p.min_step) { ls = LBERR_MINIMUMSTEP; done = true; }
                    else if (stp > 1.0e20) {
                        if (touched) { ls = LBERR_MAXIMUMSTEP; done = true; }
                        else { touched = 1; stp = 1.0e20; }
                    }
                }
            }
        }
        if (!done) {               // next trial point
            if (lane == 0) { st->ls_count = count; st->stp = stp; st->ls_mu = mu; st->ls_nu = nu; st->brackt = brackt; st->touched = touched; }
            for (int q = lane; q < n; q += 32) v.x[q] = v.xp[q] + stp * v.d[q];
            __syncwarp();
            return PH_REQ_LS;
        }
        if (lane == 0) { st->fx = fx; st->step = stp; }
        __syncwarp();
        if (ls < 0) {              // revert to the previous point (lbfgs.hpp:575-582)
            for (int q = lane; q < n; q += 32) { v.x[q] = v.xp[q]; v.g[q] = v.gp[q]; }
            __syncwarp();
            lret = ls; ended = true;
        } else {
            int k = st->k;
            if (lane == 0) st->iters_total++;
            if (stop_fires(E, p, st, lane) || k > 1000) { lret = LB_CANCELED; ended = true; }        // earlyExit, alm_traj_opt.cpp:1016
            if (!ended) {
                const double gn = vabsmax(v.g, n, lane), xn = vabsmax(v.x, n, lane);
                if (gn / fmax(1.0, xn) < p.g_epsilon) { lret = LB_CONVERGENCE; ended = true; }
            }
            if (!ended && p.past > 0) {
                if (p.past <= k) {
                    const double rate = fabs(st->pf[k % p.past] - fx) / fmax(1.0, fabs(fx));
                    if (rate < p.delta) { lret = LB_STOP; ended = true; }
                }
                if (!ended) { __syncwarp(); if (lane == 0) st->pf[k % p.past] = fx; __syncwarp(); }
            }
            if (!ended && p.inner_max_iter != 0 && p.inner_max_iter <= k) { lret = LBERR_MAXIMUMITERATION; ended = true; }
            if (!ended) {          // history update, cautious test, two-loop recursion (lbfgs.hpp:640-711)
                ++k;
                int end = st->end, bound = st->bound;
                R *sE = hist<R>(E.hs, E, v.slot, end), *yE = hist<R>(E.hy, E, v.slot, end);
                double ys = 0.0, yy = 0.0, ss = 0.0, gpn = 0.0;
                for (int q = lane; q < n; q += 32) {
                    const double s_ = v.x[q] - v.xp[q], y_ = v.g[q] - v.gp[q];
                    sE[q] = (R)s_; yE[q] = (R)y_;
                    v.d[q] = -v.g[q];
                    ys += y_ * s_; yy += y_ * y_; ss += s_ * s_; gpn += v.gp[q] * v.gp[q];
                }
                ys = warp_sum(ys); yy = warp_sum(yy); ss = warp_sum(ss); gpn = warp_sum(gpn);
                double *lys = E.lm_ys + (size_t)v.slot * E.m, *lal = E.lm_alpha + (size_t)v.slot * E.m;
                if (lane == 0) lys[end] = 1.0 / ys;        // only ever used as a divisor: keep the reciprocal
                __syncwarp();
                kp.mark(KP_ADV_POST);
                if (ys > ss * sqrt(gpn) * 1.0e-6) {
                    ++bound;
                    bound = m < bound ? m : bound;
                    end = (end + 1) % m;
                    // Each lane owns elements lane, lane + 32, ... of d in registers.  The 2 * bound history steps (newest -> oldest,
                    // then oldest -> newest) stream through a four-slot shared-memory ring by cp.async, three steps ahead of the
                    // dependent chain (dot product -> warp reduction -> axpy), so no global-memory latency sits on it.
                    constexpr int NR = TP_NVAR / 32;
                    constexpr int HR = TP_HRING;                          // ring slots: HR - 1 steps in flight ahead of the chain (the history streams from DRAM)
                    const int hstride = E.ka_hist_stride;                 // elements per vector slot (n rounded up to 16 bytes)
                    R *hring = (R *)v.sm;                                 // [HR][2][hstride], aliases the column buffer (idle here)
                    const unsigned hring0 = (unsigned)__cvta_generic_to_shared(hring);
                    const int nchunk = (n * (int)sizeof(R) + 15) / 16;
                    const int nsteps = 2 * bound, ne = (n + 31) >> 5;
                    // 1 / (y_j . s_j) of the steps and the alphas of the first loop sit in shared memory behind the ring (no global
                    // load on the chain)
                    double *rys_s = (double *)((char *)v.sm + E.ka_hist_bytes), *al_s = rys_s + m;
                    // ring index of the history pair step t works on: newest -> oldest, then oldest -> newest (t < 2 bound <= 2 m: no division needed)
                    auto jof = [&](int t) {
                        int j = t < bound ? end - 1 - t : end - bound + (t - bound);
                        j += j < 0 ? m : 0; j += j < 0 ? m : 0;
                        return j >= m ? j - m : j;
                    };
                    auto hissue = [&](int t) {
                        if (t < nsteps) {
                            const int j = jof(t);
                            const R *sj = hist<R>(E.hs, E, v.slot, j), *yj = hist<R>(E.hy, E, v.slot, j);
                            const unsigned dst = hring0 + (unsigned)((t % HR) * 2 * hstride * (int)sizeof(R));
                            for (int q = lane; q < nchunk; q += 32) {
                                cp_async16(dst + 16u * q, (const char *)sj + 16 * q);
                                cp_async16(dst + (unsigned)(hstride * (int)sizeof(R)) + 16u * q, (const char *)yj + 16 * q);
                            }
                        }
                        cp_async_commit();
                    };
                    double dreg[NR];
#pragma unroll
                    for (int e = 0; e < NR; e++) { const int q = lane + 32 * e; dreg[e] = q < n ? v.d[q] : 0.0; }
                    for (int t = lane; t < bound; t += 32) rys_s[t] = lys[(end + m - 1 - t % m + m) % m];
                    __syncwarp();
#pragma unroll
                    for (int t0 = 0; t0 < HR - 1; t0++) hissue(t0);
                    const double scl = ys / yy;
                    for (int t = 0; t < nsteps; t++) {
                        hissue(t + HR - 1);
                        cp_async_wait<HR - 1>();
                        __syncwarp();
                        const int j = jof(t);
                        const R *sv = hring + (size_t)(t % HR) * 2 * hstride, *yv = sv + hstride;
                        const bool first = t < bound;
                        const int tf = first ? t : nsteps - 1 - t;       // the first-loop step that handled this history vector
                        const double rysj = rys_s[tf];
                        const double alj = first ? 0.0 : al_s[tf];
                        double pacc = 0.0;
                        double ax[NR];
#pragma unroll
                        for (int e = 0; e < NR; e++) {
                            ax[e] = 0.0;
                            if (e < ne) {                 // warp-uniform: only the 32-element groups the vector really has
                                const int q = lane + 32 * e;
                                const double sq = q < n ? (double)sv[q] : 0.0, yq = q < n ? (double)yv[q] : 0.0;
                                pacc += (first ? sq : yq) * dreg[e];
                                ax[e] = first ? yq : sq;
                            }
                        }
                        pacc = warp_sum(pacc);
                        double cf;
                        if (first) { cf = -(pacc * rysj); if (lane == 0) al_s[tf] = -cf; }
                        else cf = alj - pacc * rysj;
#pragma unroll
                        for (int e = 0; e < NR; e++) if (e < ne) dreg[e] += cf * ax[e];
                        if (t == bound - 1) {
#pragma unroll
                            for (int e = 0; e < NR; e++) dreg[e] *= scl;
                        }
                        __syncwarp();
                    }
                    cp_async_wait<0>();
                    __syncwarp();
#pragma unroll
                    for (int e = 0; e < NR; e++) { const int q = lane + 32 * e; if (q < n) v.d[q] = dreg[e]; }
                    if (lane == 0) { if (bound > st->max_bound) st->max_bound = bound; st->sum_bound += bound; }
                }
                if (lane == 0) { st->k = k; st->end = end; st->bound = bound; st->step = 1.0; }
                __syncwarp();
                kp.mark(KP_TWOLOOP);
                const int r = ls_begin(v, lane);
                if (r < 0) { lret = r; ended = true; for (int q = lane; q < n; q += 32) { v.x[q] = v.xp[q]; v.g[q] = v.gp[q]; } }
                else return PH_REQ_LS;
            }
        }
    }
    // ---- lbfgs_optimize ended with lret: the ALM loop (alm_traj_opt.cpp:236-270) ----
    __syncwarp();
    kp.mark(KP_ADV_LS);
    if (lane == 0) { st->inner_cost = st->fx; st->last_ret = lret; }
    if (!(lret == LB_CONVERGENCE || lret == LB_CANCELED || lret == LB_STOP || lret == LBERR_MAXIMUMITERATION || lret == LBERR_MAXIMUMLINESEARCH)) {
        if (lane == 0) st->ret_code = 1;
        return PH_DONE;
    }
    // updateDualVars with hx / gx of the LAST evaluation (Q1), judgeConvergence with the updated rho (alm_traj_opt.h:132-151)
    {
        const int S = v.S;
        R *du = (R *)E.dual + (size_t)v.slot * TP_NDUAL * E.Smax;
        const double rho = st->rho, rho_new = fmin((1.0 + p.gamma) * rho, p.beta);
        double mh = 0.0, mg = 0.0;
        for (int q = lane; q < S; q += 32) {
            const double h = (double)du[14 * S + q];
            du[q] = (R)((double)du[q] + rho * h);
            mh = fmax(mh, fabs(h));
        }
        for (int q = lane; q < 6 * S; q += 32) {
            const double gq = (double)du[15 * S + q];
            const double mq = fmax((double)du[S + q] + rho * gq, 0.0);
            du[S + q] = (R)mq;
            mg = fmax(mg, fabs(fmax(gq, -mq / rho_new)));
        }
        mh = warp_max(mh); mg = warp_max(mg);
        if (lane == 0) { st->rho = rho_new; st->res_h = mh; st->res_g = mg; }
        if (fmax(mh, mg) < p.epsilon_con) return PH_DONE;         // a stop that fired in this inner solve keeps its mark in ret_code
        if (alm_ends(E, p, st, lane)) return PH_DONE;
    }
    __syncwarp();
    return PH_REQ_FIRST;           // next lbfgs_optimize starts with an evaluation at the current x
}

// 128 registers = 4 CTAs of four warps per SM.  Measured: allowing 6 / 8 CTAs (80 / 64 registers, 0.5 - 1 KB of spills) makes every warp-round
// 1.5 - 2x longer (the table and history loads contend) and lowers the throughput by 8 / 17 %
template <class R>
__global__ void __launch_bounds__(32 * TP_KA_WARPS, 4) ka_kernel(const __grid_constant__ TpPool E, const __grid_constant__ TpParams p, int group)
{
    const int lane = threadIdx.x & 31, widx = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);      // 1, 2 or 4 warps per CTA (TpEngine::ka_warps)
    if (widx >= E.n_active[group]) return;
    extern __shared__ __align__(16) unsigned char ka_smem[];     // per warp: ka_col_bytes
    unsigned char *wbase = ka_smem + (size_t)(threadIdx.x >> 5) * E.ka_col_bytes;
    const int slot = E.active[(size_t)group * E.capacity + widx];
    SlotView v = slot_view(E, slot, (double *)wbase);
    TpState *st = v.st;
    const int ph = st->phase;
    if (ph == PH_DONE || ph == PH_FREE) return;
    KProf kp;
    kp.start(E.prof, lane);
    if (kp.p) atomicAdd((unsigned long long *)&kp.p[KP_WARPS], 1ull);
    int next;
    if (ph == PH_NEW) {
        const int mode = st->mode;
        if (lane == 0) {
            if (mode != 1) { st->rho = p.rho; st->scale_fx = 1.0; }
            st->outer_iter = 0; st->n_evals = 0; st->iters_total = 0; st->ret_code = 0; st->last_ret = 0;
            st->max_bound = 0; st->sum_bound = 0; st->inner_cost = 0.0; st->res_h = 0.0; st->res_g = 0.0;
        }
        next = mode == 0 ? PH_REQ_FIRST : PH_REQ_EVALONLY;
    } else {
        finish_eval<R>(E, p, v, lane, kp);
        if (lane == 0) st->n_evals++;
        __syncwarp();
        next = (ph == PH_REQ_EVALONLY) ? PH_DONE : advance<R>(E, p, v, lane, kp);
        kp.mark(next == PH_REQ_LS ? KP_ADV_LS : KP_ALM);
    }
    __syncwarp();
    if (next == PH_DONE) {
        if (lane == 0) { st->phase = PH_DONE; atomicSub(E.remaining + st->ticket, 1); }
        return;
    }
    minco_forward<R>(E, v, lane, kp);
    if (lane == 0) st->phase = next;
}

// rebuild the active list of one group from the slot phases (one CTA); slots in PH_NEW join here
__global__ void compact_kernel(const __grid_constant__ TpPool E, int hi, int group)
{
    __shared__ int s_count;
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    int *list = E.active + (size_t)group * E.capacity;
    for (int s0 = 0; s0 < hi; s0 += blockDim.x) {
        const int s = s0 + threadIdx.x;
        bool live = false;
        if (s < hi) { const int ph = E.st[s].phase; live = ph != PH_FREE && ph != PH_DONE && E.st[s].group == group; }
        const unsigned bal = __ballot_sync(0xffffffffu, live);
        int base = 0;
        if ((threadIdx.x & 31) == 0 && bal) base = atomicAdd(&s_count, __popc(bal));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (live) list[base + __popc(bal & ((1u << (threadIdx.x & 31)) - 1u))] = s;
        __syncthreads();
    }
    if (threadIdx.x == 0) E.n_active[group] = s_count;
}

// the device-side round loop of one group (ualm_tp.cu: start_loops): what it has run, and whether it hit the round cap
struct GroupLoop { long long rounds; int launches, err; };
#define TP_ROUND_CAP 400000             // rounds of one group's loop; a trajectory still running after them did not terminate

// last node of a group's loop body, after the body's compaction: counts the body's rounds and kernel launches, and runs the body
// again while the group still has a trajectory that is not PH_DONE (n_active > 0) and the round cap is not reached (err = 1 there)
__global__ void loop_ctrl_kernel(cudaGraphConditionalHandle h, const int *n_active, GroupLoop *gl, int group, int rounds, int launches)
{
    GroupLoop &s = gl[group];
    s.rounds += rounds;
    s.launches += launches;
    const bool capped = s.rounds >= TP_ROUND_CAP;
    if (capped && n_active[group] > 0) s.err = 1;
    cudaGraphSetConditional(h, (n_active[group] > 0 && !capped) ? 1u : 0u);
}

// ---------------------------------------------------------------------------------------------------------------------
// admission: problem b of a submitted batch -> slot.  One launch covers problems of one environment (use_scaling, K are its own);
// off_s[b]: sample offset of ad[b] in the caller's dual arrays, sfx is indexed by the problem's index in its batch
// ---------------------------------------------------------------------------------------------------------------------
struct AdmitDesc { int slot, N, M, ticket, index, mode, group, pad1; long long off_x; double total_time; double bnd[18]; double pp[8]; };

template <class R>
__global__ void admit_kernel(const __grid_constant__ TpPool E, const AdmitDesc *ad, const double *x0, int B, int use_scaling, int K,
                             const double *lam, const double *mu, const double *scx, const double *sfx, double rho_eval, const long long *off_s)
{
    const int b = blockIdx.x;
    if (b >= B) return;
    const AdmitDesc a = ad[b];
    TpState *st = E.st + a.slot;
    const int n = 1 + 2 * (a.N - 1) + (a.M - 1), S = a.N * (K + 1);
    double *x = E.vec + (size_t)a.slot * 5 * TP_NVAR;
    for (int q = threadIdx.x; q < n; q += blockDim.x) x[q] = x0[a.off_x + q];
    R *du = (R *)E.dual + (size_t)a.slot * TP_NDUAL * E.Smax;
    if (a.mode != 1) {             // solve: duals 0, scales 1 (alm_traj_opt.cpp:193-203)
        for (int q = threadIdx.x; q < TP_NDUAL * S; q += blockDim.x) du[q] = (q >= 7 * S && q < 14 * S) ? (R)1.0 : (R)0.0;
    } else {                       // single evaluation at caller-provided duals (reference index layout: mu[6 s + t], scale_cx[7 s + t])
        const long long os = off_s[b];
        for (int q = threadIdx.x; q < S; q += blockDim.x) {
            du[q] = (R)(lam ? lam[os + q] : 0.0);
            for (int t = 0; t < 6; t++) du[(1 + t) * S + q] = (R)(mu ? mu[6 * (os + q) + t] : 0.0);
            for (int t = 0; t < 7; t++) du[(7 + t) * S + q] = (R)(scx ? scx[7 * (os + q) + t] : 1.0);
            for (int t = 0; t < 7; t++) du[(14 + t) * S + q] = (R)0.0;
        }
    }
    if (threadIdx.x == 0) {
        st->N = a.N; st->M = a.M; st->n = n; st->S = S; st->ticket = a.ticket; st->index = a.index;
        for (int k = 0; k < 18; k++) st->bnd[k] = a.bnd[k];
        for (int k = 0; k < 8; k++) st->pp[k] = a.pp[k];
        st->mode = a.mode; st->group = a.group;
        st->need_scale = ((a.mode == 0 && use_scaling) || a.mode == 2) ? 1 : 0;
        st->phase = PH_NEW;
        if (a.mode == 1) { st->rho = rho_eval; st->scale_fx = sfx ? sfx[a.index] : 1.0; }
    }
}

} // namespace ualm_tp
