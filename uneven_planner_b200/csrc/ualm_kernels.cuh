// ualm_kernels.cuh -- sm_90a device code of the batched MINCO / PHR-ALM / L-BFGS trajectory optimizer.
//
// A WARP GROUP (1, 2 or 4 warps of a 4-warp CTA) owns one optimizeSE2Traj problem from the first evaluation to the last dual
// update (no host round trips): its first warp runs the whole algorithm, the others serve its parallel phases; a batch of
// ~10^3 problems is resident on the 132 SMs of an H100 (8 warps per SM).
// The arithmetic is IEEE double with contraction OFF (-fmad=false) and is ordered so that every floating-point result is
// bit-identical to the CPU oracle (oracle/oracle.cpp):
//   * work that is independent per element (band-matrix entries inside one pivot step, constraint samples,
//     coefficient-gradient entries, history vectors) is spread over the 32 lanes;
//   * every reduction whose order is visible in the reference source is evaluated in that order (cost accumulation
//     alm_traj_opt.cpp:825-943, gdC/gdT accumulation :969-985, triangular sweeps banded_system.hpp:96-145);
//   * dot products / norms of the L-BFGS driver (order left to Eigen in the reference) use the canonical 32-lane order:
//     lane-strided partial sums + xor-butterfly 16,8,4,2,1 (warp shuffles).
// Memory plan per trajectory: coefficients, gradients and the decision vectors live in shared memory (20-36 KB); the band
// LU runs on a 12-row window in shared memory and streams its factors to global memory (L2), row-major with the reciprocal
// of the diagonal in column 13; the four triangular sweeps read them back through cp.async rings with the last six solution
// values in registers; L-BFGS history, duals, constraint values and the per-sample scratch are coalesced global arrays.
// Reference citations are relative to /root/reference/src/uneven_planner/.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "ualm.h"
#include "ualm_detmath.h"
#include "ualm_mailbox.h"
#include "resample_stream.h"

#define UALM_THREADS 32         // threads per warp slot
#define UALM_WPB 4              // warp slots per CTA (4 / 2 / 1 trajectories with 1 / 2 / 4 warps each)
#define UALM_NFIELD 26          // per-sample scratch fields (see SF_* below)
#define UALM_NPROF 16
#define UALM_FW 14              // doubles per factor row (13 band entries + 1 pad -> 112 B = 7 x 16 B)
#define UALM_FPAD 8             // zero pad rows before and after each factor array (chunked prefetch may overrun)
#define UALM_SYNC() __syncwarp()
#define UALM_RINGB 4            // factor-ring depth in 6-row blocks per system (prefetch distance UALM_RINGB - 2)
#define UALM_NMAX 64            // compiled limits on the piece counts of one problem (a problem over them is skipped with
#define UALM_MMAX 128           //   ret_code = UALM_ELIMIT; the rest of its batch is solved)
#define UALM_NREG 8             // L-BFGS two-loop register tile: each lane owns elements lane, lane + 32, ... (n <= 32 * UALM_NREG)
static_assert(1 + 2 * (UALM_NMAX - 1) + (UALM_MMAX - 1) <= 32 * UALM_NREG, "decision vector must fit the two-loop register tile");

namespace ualm {

typedef double R;

// ---- compile-time constants of the reference (alm_traj_opt.h:16-19) ----
#define UALM_DELTA_SIGL 0.01
#define UALM_CUR_SCALE 10.0
#define UALM_SIG_SCALE 1000.0
#define UALM_SCALE_TRICK_JERK 1000.0

// lbfgs return codes (lbfgs.hpp:135-184)
enum {
    LBFGS_CONVERGENCE = 0, LBFGS_STOP, LBFGS_CANCELED,
    LBFGSERR_UNKNOWNERROR = -1024, LBFGSERR_INVALID_N, LBFGSERR_INVALID_MEMSIZE, LBFGSERR_INVALID_GEPSILON,
    LBFGSERR_INVALID_TESTPERIOD, LBFGSERR_INVALID_DELTA, LBFGSERR_INVALID_MINSTEP, LBFGSERR_INVALID_MAXSTEP,
    LBFGSERR_INVALID_FDECCOEFF, LBFGSERR_INVALID_SCURVCOEFF, LBFGSERR_INVALID_MACHINEPREC,
    LBFGSERR_INVALID_MAXLINESEARCH, LBFGSERR_INVALID_FUNCVAL, LBFGSERR_MINIMUMSTEP, LBFGSERR_MAXIMUMSTEP,
    LBFGSERR_MAXIMUMLINESEARCH, LBFGSERR_MAXIMUMITERATION, LBFGSERR_WIDTHTOOSMALL, LBFGSERR_INVALIDPARAMETERS,
    LBFGSERR_INCREASEGRADIENT,
};

// what is per environment; the eight per-problem values (ualm_problem_params_t) travel in ProbDesc::pp and are read from SC_PP
struct DevParams {
    int use_scaling;
    R rho, beta, gamma, epsilon_con, max_iter;
    R g_epsilon, min_step, delta;
    int inner_max_iter;
    int mem_size, past, int_K;
    R gravity;
    // stop predicate of the solve (ualm_set_budget / ualm_cancel_problems / ualm_wait_batch_for): evaluation budget (0 = none)
    // and the lane's stop words in device memory, one per problem of its batch (null = none), set per launch
    int max_evals;
    const volatile int *cancel;
};

struct DevMap {
    const float4 *cells;   // {z, sigma, zbx, zby} as float32, or null when
    const double *cells64; //   the reference's own RXS2 grid (4 doubles per cell, uneven_map.h:36-64) is bound instead
    int vn[3];
    R origin[3], maxb[3], xy_res, yaw_res, xy_inv, yaw_inv;
};

// one problem; offsets index the packed batch arrays
struct ProbDesc {
    int N, M, n, S;
    long long off_x;      // n-sized vectors (x0, x_out, grad)
    long long off_s;      // S-sized (lambda, hx); 6*off_s for mu/gx; 7*off_s for scale_cx
    long long off_cxy;    // 12 N
    long long off_cyaw;   // 6 M
    long long off_hist;   // mem_size * n  (lm_s, lm_y)
    long long off_scr;    // UALM_NFIELD * S per-sample scratch
    long long off_fac;    // factor arrays: Fxy ((6N + 2 pad) rows), Fyaw ((6M + 2 pad) rows), UALM_FW doubles per row
    long long off_ws;     // initScaling adjoint workspace (12 N + 6 M) * 32
    long long off_aux;    // 3 * mem_size of the problem's environment (lm_aux)
    R bnd[18];
    R total_time;
    R pp[8];              // the problem's ualm_problem_params_t (its row, or its environment's values): copied to SC_PP by traj_setup
};

struct BatchPtrs {
    int B;
    int n_active;            // problems within the compiled limits = entries of `order`
    int *queue;              // solve_kernel: the launch's work counter (zero at launch); slots take order[atomicAdd(queue, 1)]
    int n_leader_slots;      // solve_kernel: full per-trajectory slots per CTA (4 / G); helper rings follow them
    int adopt;               // solve_kernel: warps of a finished trajectory join the other trajectory of a two-slot CTA
    const ProbDesc *desc;
    const int *order;        // launch order (largest first) -> problem index
    const R *x0;             // packed initial decision vectors
    R *x;                    // packed final decision vectors
    R *lambda, *mu, *scale_cx, *hx, *gx;
    R *lm_s, *lm_y;
    R *lm_aux;               // per problem 3 * mem_size at off_aux: lm_alpha | lm_ys | RN(1 / lm_ys)
    R *scratch;
    R *fac;                  // LU factors
    R *ws_scaling;           // initScaling adjoint workspace
    R *c_xy, *c_yaw;
    ualm_result_t *results;
    R *piece_T;              // per problem {T_xy piece, T_yaw piece} of the LAST evaluation (the durations getTraj() carries, Q1)
    // eval entry
    R *f_out, *grad_out, *scale_fx_io;
    long long *prof;         // optional [grid][UALM_NPROF] phase cycle counters (lane 0 of each warp)
    ualm_mbox::Ptrs mbox;    // solve_kernel: the lane's result mailbox (ualm_poll_batch), flag null = publish nothing
    // solve_kernel, urgent work (ualm_set_urgent): the context's UALM_HOLD_BYTES hold bytes (null = no holds), any of them raised =
    // urgent work needs SM slots; the lane's words {problems its urgent launches have taken, 1 = this solve takes no further hold,
// microseconds its gates have waited};
    // urgent_slot >= 0: the launch is urgent, ignores holds, and the take of the lane's n_urgent-th problem lowers hold byte urgent_slot
    unsigned char *hold;
    int *hctl;
    int urgent_slot, n_urgent;
};

// hold bytes: one per lane (its urgent ticket) and one for the check stream (an urgent check or replan build).  The host raises and
// lowers them by copies, which need no SM; a slot of a non-urgent launch reads them before each take
#define UALM_HOLD_BYTES 32
static_assert(UALM_HOLD_BYTES % 8 == 0, "read as 8-byte words");
// the longest a held launch waits (hold_gate_kernel): after it, its solve takes no further hold, so a hold never released only slows
// work down
#define UALM_HOLD_BOUND_NS 2000000000ull

__device__ __forceinline__ bool hold_raised(const unsigned char *hold)
{
    const volatile unsigned long long *h = (const volatile unsigned long long *)hold;
    unsigned long long v = 0;
#pragma unroll
    for (int k = 0; k < UALM_HOLD_BYTES / 8; k++) v |= h[k];
    return v != 0;
}

// per-sample scratch fields (SoA: scratch[field * S + s])
enum {
    SF_COST0 = 0,              // 8 cost terms in accumulation order: user, nonhol, vx, ax, ay, curv, att, sig
    SF_GP = 8, SF_GV = 10, SF_GA = 12, SF_GYAW = 14, SF_GDYAW = 15,
    SF_VEL = 16, SF_ACC = 18, SF_JER = 20, SF_DYAW = 22, SF_D2YAW = 23, SF_S1YAW = 24, SF_USER = 25
};

// ---------------------------------------------------------------------------------------------
// shared-memory layout (doubles), sized on the host from the batch maxima
// ---------------------------------------------------------------------------------------------
struct SmemLayout {
    int cxy, cyaw, gCxy, gCyaw, gTxy, gTyaw, x, g, xp, gp, d, pf, s1tab, base, sc, win, tmpl, ring, lutab /* 13 x 16 uint4 */, yawidx /* shorts */, total_doubles;
};

__host__ __device__ inline SmemLayout make_layout(int Nmax, int Mmax, int nmax, int m, int past, int K, int Smax)
{
    SmemLayout L;
    int o = 0;
    L.cxy = o; o += 12 * Nmax;
    L.cyaw = o; o += 6 * Mmax;
    L.gCxy = o; o += 12 * Nmax;
    L.gCyaw = o; o += 6 * Mmax;
    L.gTxy = o; o += Nmax;
    L.gTyaw = o; o += Mmax;
    L.x = o; o += nmax;
    L.g = o; o += nmax;
    L.xp = o; o += nmax;
    L.gp = o; o += nmax;
    L.d = o; o += nmax;
    L.pf = o; o += (past > 1 ? past : 1);
    L.s1tab = o; o += K + 1;
    L.base = o; o += Nmax;
    L.sc = o; o += 48;                   // scalars
    o = (o + 1) & ~1;                    // 16-byte alignment for the cp.async destinations
    // LU scratch (sliding windows + template rows) and the factor ring of the sweeps are never live at the same time: they alias
    L.win = o;
    L.tmpl = o + 2 * 16 * UALM_FW;
    L.ring = o;
    {
        const int lu = 2 * 16 * UALM_FW + 2 * 12 * UALM_FW, rg = 2 * UALM_RINGB * 6 * UALM_FW;
        o += lu > rg ? lu : rg;
    }
    L.lutab = o; o += 13 * 16 * 2;        // LU step constants: 13 pivot types x 16 half-warp lanes x 16 bytes
    L.yawidx = o; o += (Smax + 3) / 4;   // shorts packed
    L.total_doubles = (o + 1) & ~1;
    (void)m;
    return L;
}

// scalar slots in sm[L.sc + ...]
enum {
    SC_TX1 = 0, SC_TX2, SC_TX3, SC_TX4, SC_TX5, SC_TY1, SC_TY2, SC_TY3, SC_TY4, SC_TY5,
    SC_SCALE_FX, SC_RHO, SC_F, SC_JERK, SC_CONSTR, SC_TAUCOST, SC_JERKRAW, SC_RTY, SC_CMD,
    SC_STOPPED,  // != 0: the stop predicate fired inside the inner solve that just ended
    SC_PROB,     // the problem a CMD_NEXT hands to the helpers
    // the problem's ualm_problem_params_t, written by the leader's traj_setup: every warp of the group (helpers, a mate that joins)
    // reads them here, and the launch's DevParams holds only what is per environment
    SC_PP = 24, SC_RHO_T = SC_PP, SC_RHO_TER, SC_MAX_VEL, SC_MAX_ACC_LON, SC_MAX_ACC_LAT, SC_MAX_KAP, SC_MIN_CXI, SC_MAX_SIG
};
static_assert(SC_MAX_SIG < 48, "the scalar slots of SmemLayout::sc");

// Handles to shared memory: a 32-bit address in the shared state space.  Accesses through them are explicit ld.shared /
// st.shared with 32-bit address arithmetic.  (Plain `double*` members become generic loads, and C++ references into the
// `extern __shared__` array make the compiler rebuild the generic shared-window base -- S2UR SR_CgaCtaId + ULEA -- at every
// use inside the __noinline__ functions: measured at ~20 % of the LU pivot loop in profiles/solve_kernel_r01_summary.md.)
extern __shared__ __align__(16) double ualm_smem[];
__device__ __forceinline__ double lds64(unsigned a)
{
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts64(unsigned a, double v) { asm volatile("st.shared.f64 [%0], %1;" ::"r"(a), "d"(v) : "memory"); }
// 16-byte accesses (a must be 16-byte aligned)
__device__ __forceinline__ double2 lds2f64(unsigned a)
{
    double2 v;
    asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts2f64(unsigned a, double x, double y)
{
    asm volatile("st.shared.v2.f64 [%0], {%1, %2};" ::"r"(a), "d"(x), "d"(y) : "memory");
}
// a store under a predicate: keeps the compiler from turning a guarded store into a divergent branch
__device__ __forceinline__ void sts64_if(bool p, unsigned a, double v)
{
    asm volatile("{\n .reg .pred q;\n setp.ne.u32 q, %0, 0;\n @q st.shared.f64 [%1], %2;\n}" ::"r"((unsigned)p), "r"(a), "d"(v) : "memory");
}
struct SRef {   // proxy "reference" to one shared double
    unsigned a;
    __device__ __forceinline__ operator double() const { return lds64(a); }
    __device__ __forceinline__ const SRef &operator=(double v) const { sts64(a, v); return *this; }
    __device__ __forceinline__ const SRef &operator=(const SRef &o) const { sts64(a, lds64(o.a)); return *this; }
    __device__ __forceinline__ const SRef &operator+=(double v) const { sts64(a, lds64(a) + v); return *this; }
    __device__ __forceinline__ const SRef &operator-=(double v) const { sts64(a, lds64(a) - v); return *this; }
    __device__ __forceinline__ const SRef &operator*=(double v) const { sts64(a, lds64(a) * v); return *this; }
};
struct SPtr {
    unsigned a;   // byte address in the shared window
    __device__ __forceinline__ SRef operator[](int i) const { return SRef{a + 8u * (unsigned)i}; }
    __device__ __forceinline__ SRef operator*() const { return SRef{a}; }
    __device__ __forceinline__ SPtr operator+(int d) const { return SPtr{a + 8u * (unsigned)d}; }
};
struct SRefU16 {
    unsigned a;
    __device__ __forceinline__ operator int() const
    {
        unsigned short v;
        asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(a) : "memory");
        return (int)v;
    }
    __device__ __forceinline__ const SRefU16 &operator=(unsigned short v) const
    {
        asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "h"(v) : "memory");
        return *this;
    }
};
struct SPtrU16 {
    unsigned a;
    __device__ __forceinline__ SRefU16 operator[](int i) const { return SRefU16{a + 2u * (unsigned)i}; }
};
// element access that works for both handle kinds
__device__ __forceinline__ SRef at(SPtr p, int i) { return p[i]; }
__device__ __forceinline__ double &at(double *p, int i) { return p[i]; }
__device__ __forceinline__ const double &at(const double *p, int i) { return p[i]; }

struct Traj {
    // problem
    int N, M, n, S, K;
    const ProbDesc *pd;
    // smem
    SPtr cxy, cyaw, gCxy, gCyaw, gTxy, gTyaw;
    SPtr x, g, xp, gp, d, pf, s1tab, base, sc, win, tmpl, ring;
    SPtrU16 yawidx;
    unsigned lutab;    // shared-memory byte address of the LU step-constant table
    // global
    R *lambda, *mu, *scale_cx, *hx, *gx, *lm_s, *lm_y, *lm_alpha, *lm_ys, *lm_rys, *scr;
    R *Fxy, *Fyaw;                  // row 0 of each factor array
    R *ws;
    // warp group of this trajectory: G warps (1, 2 or 4) of one CTA; warp 0 of the group (the leader) runs the whole algorithm,
    // the others (helpers) only execute the parallel phases the leader posts (samples, gradient accumulation, initScaling)
    int G, wig, barid;
    int *adopt;        // shared-memory state word of this leader slot (two-slot CTAs only; see "adoption" below), else null
    SPtr hring;        // this warp's own factor ring (initScaling sweeps run per warp)
    R *wsw;            // this warp's own initScaling workspace
    int n_evals;
    long long *prof;   // shared-memory phase counters (lane 0 only)
    long long *plast;
};

// phase ids of the in-kernel profiler
enum { PF_FILL = 0, PF_LU, PF_SOLVE, PF_JERK, PF_TABLES, PF_SAMPLES, PF_ACCUM, PF_COMBINE, PF_ADJ, PF_TAIL, PF_TWOLOOP, PF_LS, PF_SCALING,
       PF_DUAL, PF_OTHER, PF_TOTAL };
__device__ __forceinline__ void prof_mark(const Traj &t, int tid, int phase)
{
    if (tid == 0) {
        const long long c = clock64();
        t.prof[phase] += c - *t.plast;
        *t.plast = c;
    }
}

// ---- leader / helper protocol inside a warp group (named barrier 1 + leader warp index, 32*G participants) ----
enum { CMD_SAMPLES = 1, CMD_ACCUM = 2, CMD_SCALE = 3, CMD_EXIT = 4, CMD_REGROUP = 5, CMD_JOIN = 6, CMD_NEXT = 7 };
// Adoption (CTAs that hold two trajectories with two warps each): when a slot finds the launch's queue empty, its two warps join
// the other trajectory's group as helpers 2 and 3, so the slower of the pair runs its parallel phases on the whole CTA.  Per
// leader slot one state word: DONE (no problem) -> RUNNING (problem published) -> (mate asks) JOINREQ -> (leader switches its
// group to the 128-thread barrier) JOINED; -> DONE.  A slot that has been joined takes no further problem.
// The partition of the parallel phases over warps never changes a result bit (every output entry has one owner and a fixed
// summation order), so the solve stays batch-invariant.
enum { AD_RUNNING = 0, AD_JOINREQ = 1, AD_JOINED = 2, AD_DONE = 3 };
#define UALM_BAR_BIG 5
__device__ __forceinline__ void group_bar(const Traj &t)
{
    if (t.G > 1) asm volatile("bar.sync %0, %1;" ::"r"(t.barid), "r"(32 * t.G) : "memory");
    else __syncwarp();
}
// leader: publish the next parallel phase and release the helpers (no-op for a single-warp group)
__device__ __forceinline__ void group_post(const Traj &t, int lane, int cmd)
{
    if (t.G > 1) {
        if (lane == 0) t.sc[SC_CMD] = (R)cmd;
        __syncwarp();
        group_bar(t);
    }
}
// leader of a two-warp group: move the group (its helper and the two waiting joiners) onto the CTA-wide barrier
__device__ __forceinline__ void regroup_now(Traj &t, int lane)
{
    group_post(t, lane, CMD_REGROUP);
    group_bar(t);                       // the helper has read the command word; it may be overwritten now
    t.G = 4; t.barid = UALM_BAR_BIG;
}
__device__ __forceinline__ void maybe_regroup(Traj &t, int lane)
{
    if (t.adopt == nullptr || t.G != 2) return;
    int st = 0;
    if (lane == 0) st = *(volatile int *)t.adopt;
    st = __shfl_sync(0xffffffffu, st, 0);
    if (st == AD_JOINREQ) {
        regroup_now(t, lane);
        if (lane == 0) atomicExch(t.adopt, AD_JOINED);
    }
}

__device__ __forceinline__ R expC2(R tau) // alm_traj_opt.h:232-235
{
    return tau > 0.0 ? ((0.5 * tau + 1.0) * tau + 1.0) : 1.0 / ((0.5 * tau - 1.0) * tau + 1.0);
}
__device__ __forceinline__ R getTtoTauGrad(R tau) // alm_traj_opt.h:244-253
{
    if (tau > 0) return tau + 1.0;
    R denSqrt = (0.5 * tau - 1.0) * tau + 1.0;
    return (1.0 - tau) / (denSqrt * denSqrt);
}
// a yaw cell index wrapped into [0, n)
__device__ __forceinline__ int wrap_index(int c, int n)
{
    while (c > n - 1) c -= n;
    while (c < 0) c += n;
    return c;
}
__device__ __forceinline__ void normSO2(R &yaw) // uneven_map.cpp:64-71
{
    while (yaw < -M_PI) yaw += 2 * M_PI;
    while (yaw > M_PI) yaw -= 2 * M_PI;
}

// The kernel is latency bound and eight warps per SM sit in different phases, so instruction-cache footprint matters
// (L0 ~6 KB, L1.5 32 KB): every large device function is __noinline__ (one copy, called), not inlined per call site.
#define UALM_NOINLINE __noinline__
// returned by value: taking the address of a caller's variable for an out-of-line call would pin that variable (or the whole
// struct it is a member of) in local memory
__device__ UALM_NOINLINE double2 dev_sincos(R x)
{
    R s, c;
    ualm_sincos(x, &s, &c);
    return make_double2(s, c);
}
__device__ UALM_NOINLINE R dev_atan2(R y, R x) { return ualm_atan2(y, x); }
// the same routines inlined (INL: the per-evaluation penalty loop, which has the registers to spare and where four calls per
// sample and their argument moves were a measurable share of the phase) or through the out-of-line copies above
template <bool INL>
__device__ __forceinline__ double2 sincos_sel(R x)
{
    if (!INL) return dev_sincos(x);
    R s, c;
    ualm_sincos(x, &s, &c);
    return make_double2(s, c);
}
template <bool INL>
__device__ __forceinline__ R atan2_sel(R y, R x) { return INL ? ualm_atan2(y, x) : dev_atan2(y, x); }

// IEEE a / b for callers whose numerator is often exactly zero.  The inline fast path of the fp64 division hands a zero (or
// denormal) quotient to an out-of-line slow path, and it does so for the whole warp when a single lane needs it; here a zero
// numerator is replaced by 1 for the division and the signed zero (NaN for b = 0 or NaN) is put back afterwards.
__device__ __forceinline__ R div_nz(R a, R b)
{
    const bool z = (a == 0.0);
    const R q = (z ? 1.0 : a) / b;
    const long long sz = (__double_as_longlong(a) ^ __double_as_longlong(b)) & (long long)0x8000000000000000ull;
    const R zq = (b != b || b == 0.0) ? __longlong_as_double(0x7ff8000000000000ll) : __longlong_as_double(sz);
    return z ? zq : q;
}

// a / b given rb = RN(1/b): q0 = a*rb followed by two residual corrections with FMA returns the correctly rounded quotient
// (Markstein).  Checked bit for bit against IEEE division on 1.6e10 operand pairs on an H100 (tools/microbench/fastdiv.cu).
// Out-of-range quotients and the flagged all-ones divisor (rb = NaN) fall back to the IEEE division.
__device__ __forceinline__ R div_by_recip(R a, R b, R rb)
{
    R q = a * rb;
    R e = fma(-q, b, a);
    q = fma(e, rb, q);
    e = fma(-q, b, a);
    q = fma(e, rb, q);
    const R aq = fabs(q);
    // (the compiler evaluates this division speculatively, so it must stay on the fast path for a zero numerator: div_nz)
    if (!(aq < 1.0e290) || (aq < 1.0e-290 && a != 0.0)) q = div_nz(a, b);
    return q;
}
// the same quotient without the fallback: `bad` collects the cases that need the IEEE division, so that a chain of quotients
// (a sweep block) pays one branch at its end instead of one per row
// With rb = RN(1/b) one correction step already yields the correctly rounded quotient (Markstein's theorem; 0 mismatches in
// 1.6e10 pairs, tools/microbench/fastdiv.cu), so the caller's dependent chain continues from q1 (three dependent fp64
// operations) while the second step only verifies it off the chain: any disagreement raises `bad`.
__device__ __forceinline__ R div_by_recip_flag(R a, R b, R rb, bool &bad)
{
    const R q0 = a * rb;
    const R e0 = fma(-q0, b, a);
    const R q1 = fma(e0, rb, q0);
    const R e1 = fma(-q1, b, a);
    const R q2 = fma(e1, rb, q1);
    const R aq = fabs(q1);
    bad = bad || !(q2 == q1) || !(aq < 1.0e290) || (aq < 1.0e-290 && a != 0.0);
    return q1;
}

// ---------------------------------------------------------------------------------------------
// cp.async (LDGSTS) helpers: 16-byte global -> shared copies that bypass L1 (factors are produced by this warp and
// consumed once per sweep: L2 is the right home)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_l1(const void *p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
__device__ __forceinline__ void cp_async16(unsigned smem_addr, const void *gmem)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(smem_addr), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int NPEND>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(NPEND) : "memory"); }

// ---------------------------------------------------------------------------------------------
// MINCO system matrix entry A(r, r - 6 + q) of a P-piece, uniform-duration system (se2traj.hpp:609-674)
// ---------------------------------------------------------------------------------------------
__device__ UALM_NOINLINE R a_entry(int P, int r, int q, R T1, R T2, R T3, R T4, R T5)
{
    const int n6 = 6 * P;
    const int c = r - 6 + q;
    if (c < 0 || c >= n6 || r >= n6) return 0.0;
    if (r < 3) {
        if (c != r) return 0.0;
        return r == 2 ? 2.0 : 1.0;
    }
    if (r >= n6 - 3) {
        const int e = c - (n6 - 6), tr = r - (n6 - 3);
        if (e < 0) return 0.0;
        if (tr == 0) return e == 0 ? 1.0 : e == 1 ? T1 : e == 2 ? T2 : e == 3 ? T3 : e == 4 ? T4 : T5;
        if (tr == 1) return e == 0 ? 0.0 : e == 1 ? 1.0 : e == 2 ? 2.0 * T1 : e == 3 ? 3.0 * T2 : e == 4 ? 4.0 * T3 : 5.0 * T4;
        return e < 2 ? 0.0 : e == 2 ? 2.0 : e == 3 ? 6.0 * T1 : e == 4 ? 12.0 * T2 : 20.0 * T3;
    }
    const int i = (r - 3) / 6, tt = (r - 3) - 6 * i, e = c - 6 * i;
    switch (tt) {
    case 0: return e == 3 ? 6.0 : e == 4 ? 24.0 * T1 : e == 5 ? 60.0 * T2 : e == 9 ? -6.0 : 0.0;
    case 1: return e == 4 ? 24.0 : e == 5 ? 120.0 * T1 : e == 10 ? -24.0 : 0.0;
    case 2: return e == 0 ? 1.0 : e == 1 ? T1 : e == 2 ? T2 : e == 3 ? T3 : e == 4 ? T4 : e == 5 ? T5 : 0.0;
    case 3: return e == 0 ? 1.0 : e == 1 ? T1 : e == 2 ? T2 : e == 3 ? T3 : e == 4 ? T4 : e == 5 ? T5 : e == 6 ? -1.0 : 0.0;
    case 4: return e == 1 ? 1.0 : e == 2 ? 2.0 * T1 : e == 3 ? 3.0 * T2 : e == 4 ? 4.0 * T3 : e == 5 ? 5.0 * T4 : e == 7 ? -1.0 : 0.0;
    default: return e == 2 ? 2.0 : e == 3 ? 6.0 * T1 : e == 4 ? 12.0 * T2 : e == 5 ? 20.0 * T3 : e == 8 ? -2.0 : 0.0;
    }
}

// ---------------------------------------------------------------------------------------------
// Structure of the MINCO band matrix and of its LU factors (symbolic elimination, period 6 in the row index; the last six
// rows/columns -- the tail position/velocity/acceleration rows -- have their own patterns).  Offsets are relative to the
// pivot: multiplier rows k+o, U columns k+o.  Types 0..5 = k mod 6, types 6..11 = the last six pivots.  The lists are
// supersets of the numerically non-zero entries (exact cancellations make some fill entries 0), so every use keeps the
// reference's numeric `!= 0` test (banded_system.hpp:74,81,83) and stays bit-identical to the dense-band loops.
// ---------------------------------------------------------------------------------------------
__host__ __device__ constexpr int lu_nm(int ty)
{
    return ty == 0 ? 2 : ty == 1 ? 3 : ty == 2 ? 4 : ty == 3 ? 4 : ty == 4 ? 4 : ty == 5 ? 3 : ty == 6 ? 1 : ty == 7 ? 2 : ty == 8 ? 3 : ty == 9 ? 2 : ty == 10 ? 1 : 0;
}
__host__ __device__ constexpr int lu_nu(int ty)
{
    return ty == 3 ? 3 : (ty == 10 ? 1 : (ty == 11 ? 0 : 2));
}
// multiplier row offset l of pivot type ty
__host__ __device__ constexpr int lu_mult(int ty, int l)
{
    return ty == 0 ? (l == 0 ? 5 : 6)
         : ty == 1 ? (l == 0 ? 4 : l == 1 ? 5 : 6)
         : ty == 2 ? (3 + l)
         : ty == 3 ? (2 + l)
         : ty == 4 ? (1 + l)
         : ty == 5 ? (1 + l)
         : ty == 6 ? 3
         : ty == 7 ? (2 + l)
         : ty == 8 ? (1 + l)
         : ty == 9 ? (1 + l)
         : 1;
}
// U column offset c of pivot type ty
__host__ __device__ constexpr int lu_ucol(int ty, int c)
{
    return (ty == 0 || ty == 6) ? (3 + c)
         : (ty == 1 || ty == 7) ? (2 + c)
         : (ty == 2 || ty == 8 || ty == 9) ? (1 + c)
         : ty == 3 ? (c == 2 ? 6 : 1 + c)
         : ty == 4 ? (c == 0 ? 1 : 6)
         : ty == 5 ? (4 + c)
         : 1;
}

// template rows of A: 12 rows x UALM_FW per system: [0..5] junction rows (row index r with (r-3) mod 6 = 0..5), [6..8] head
// rows 0..2, [9..11] tail rows 6P-3..6P-1.  Filled once per evaluation (the durations are uniform, alm_traj_opt.h:257-261).
__device__ __forceinline__ int tmpl_index(int r, int n6)
{
    if (r < 3) return 6 + r;
    if (r >= n6 - 3) return 9 + (r - (n6 - 3));
    return (r - 3) % 6;
}

// Constants of one pivot step per pivot type (0..5 = k mod 6, 6..11 = the last six pivots, 12 = no work) and half-warp lane,
// 16 bytes each: byte offsets into the 12-row window (UALM_WROW doubles per row; the pivot of type ty sits in row ty mod 6) of
//   .x the multiplier entry this lane divides (the pivot itself for the reciprocal lane and for idle lanes),
//   .y the entry this lane updates, .z the pivot-row entry of that update,
//   .w control: bits 0-1 lane holding the update's multiplier, 2 multiplier/reciprocal lane, 3 reciprocal lane, 4 update
//      enabled, 5 factor store enabled, bits 8-14 offset of this lane's factor entry in row k of F, bits 16-18 row offset o of
//      this lane's multiplier L(k+o, k) (0: no multiplier), which also names the right-hand-side row it eliminates.
// Built once per trajectory slot (3.3 KB of shared memory).
#define UALM_WROW 16
__device__ __forceinline__ void sts128(unsigned a, uint4 v)
{
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 lds128(unsigned a)
{
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void lu_build_consts(unsigned tab, int lane)
{
    for (int e = lane; e < 13 * 16; e += 32) {
        const int ty = e >> 4, hl = e & 15;
        uint4 c = make_uint4(8u * 6u, 8u * 6u, 8u * 6u, 0u);
        if (ty < 12) {
            const int tt = ty % 6;
            const int nm = lu_nm(ty), nu = lu_nu(ty);
            int mo = 0, uo = 0, uc = 0, ul = 0;
            if (hl < nm) mo = lu_mult(ty, hl);
            else if (hl == nm) mo = 7;
            if (hl < nm * nu) {
                ul = hl / nu;
                uo = lu_mult(ty, ul);
                uc = lu_ucol(ty, hl - ul * nu);
            }
            const bool act = (mo != 0), isr = (mo == 7), ulane = (hl >= 5 && hl < 12);
            const int o = isr ? 0 : mo;
            const bool upd = (uc != 0) && (ty < 6 || tt + uc < 6);       // the last six pivots: column k + uc must exist
            const int so = act ? (isr ? 13 : o * UALM_FW + 6 - o) : 6 + (ulane ? hl - 5 : 0);
            c.x = 8u * (unsigned)((tt + o) * UALM_WROW + 6 - o);
            c.y = 8u * (unsigned)((tt + uo) * UALM_WROW + 6 + uc - uo);
            c.z = 8u * (unsigned)(tt * UALM_WROW + 6 + uc);
            c.w = (unsigned)ul | (act ? 4u : 0u) | (isr ? 8u : 0u) | (upd ? 16u : 0u) | ((act || ulane) ? 32u : 0u) | ((unsigned)so << 8) |
                  ((unsigned)o << 16);
        }
        sts128(tab + 16u * (unsigned)e, c);
    }
}

// Banded LU without pivoting (banded_system.hpp:66-91) of the xy system (lanes 0..15) and the yaw system (lanes 16..31) in
// lockstep.  Element-wise the update sequence is the reference's; within one pivot step the <=4 multipliers, the reciprocal of
// the pivot and the <=12 updates run on different lanes.  Final factors stream to global memory: F[row][q] = LU(row, row-6+q),
// F[row][13] = RN(1 / LU(row,row)) for the division-free sweeps.
//
// The forward sweep L y = b (banded_system.hpp:96-103) runs inside the factorization, on the right-hand sides in t.cxy (x and
// y columns) and t.cyaw: the lane that forms L(k+o, k) also applies b(k+o) -= L(k+o, k) * b(k), skipped where L(k+o, k) == 0
// as in the reference.  L(k+o, k) is final when pivot step k forms it and b(k) is final after step k-1 (its last update comes
// from row k-1), so every element of b receives the reference's subtractions with the same operands in the same (ascending)
// order.
//
// Six pivots (one period of the structure) form a super-step on a 12-row shared-memory window: rows 0..5 are the pivot rows,
// rows 6..11 the rows below them; after the six steps rows 6..11 move up and fresh template rows enter.  Because the window
// never slides inside a super-step, every operand address of a lane is a constant of (lane, pivot type), read from the table
// of lu_build_consts one step ahead; a pivot step is ~50 instructions without data-dependent branches (a taken branch costs a
// lone warp ~20 cycles) in a loop small enough for the instruction cache (an unrolled super-step measured slower).
__device__ UALM_NOINLINE void lu_dual(Traj &t, int lane)
{
    const int sys = lane >> 4, hl = lane & 15;
    const int P = sys ? t.M : t.N, n6 = 6 * P;
    const unsigned Wb = (t.win + sys * (12 * UALM_WROW)).a;
    const SPtr TM = t.tmpl + sys * (12 * UALM_FW);
    R *F = sys ? t.Fyaw : t.Fxy;
    // right-hand-side columns of this system; the yaw half-warp names its one column twice, so its second store repeats the first
    const unsigned B0 = (sys ? t.cyaw : t.cxy).a, B1 = sys ? 0u : 8u * (unsigned)n6;
    {
        const R T1 = t.sc[sys ? SC_TY1 : SC_TX1], T2 = t.sc[sys ? SC_TY2 : SC_TX2], T3 = t.sc[sys ? SC_TY3 : SC_TX3],
                T4 = t.sc[sys ? SC_TY4 : SC_TX4], T5 = t.sc[sys ? SC_TY5 : SC_TX5];
#pragma unroll 1
        for (int e = hl; e < 12 * 13; e += 16) {
            const int row = e / 13, q = e - 13 * row;
            R v;
            if (row < 6) v = a_entry(4, 9 + row, q, T1, T2, T3, T4, T5);          // junction 1 of a 4-piece system
            else if (row < 9) v = (q == 6) ? (row == 8 ? 2.0 : 1.0) : 0.0;        // head rows
            else v = a_entry(4, 21 + (row - 9), q, T1, T2, T3, T4, T5);          // tail rows of a 4-piece system
            TM[row * UALM_FW + q] = v;
        }
    }
    UALM_SYNC();
    // rows r0 .. r0+5 of A into window rows wr0 .. wr0+5 (entries whose column falls outside the matrix are zero); lane hl < 13
    // owns band column q = hl
    auto fill6 = [&](int r0, int wr0) {
        if (hl < 13) {
#pragma unroll 1
            for (int rr = 0; rr < 6; rr++) {
                const int r = r0 + rr, c = r - 6 + hl;
                R v = 0.0;
                if (r < n6 && c >= 0 && c < n6) v = TM[tmpl_index(r, n6) * UALM_FW + hl];
                sts64(Wb + 8u * (unsigned)((wr0 + rr) * UALM_WROW + hl), v);
            }
        }
    };
    fill6(0, 0);
    fill6(6, 6);
    // this lane's entries of the six interior junction rows in the order they enter the window (row r0 + rr, r0 a multiple of 6)
    R tmv[6];
#pragma unroll
    for (int rr = 0; rr < 6; rr++) tmv[rr] = (hl < 13) ? (R)TM[((rr + 3) % 6) * UALM_FW + hl] : 0.0;
    const bool ulane = (hl >= 5 && hl < 12);
    const int uq = ulane ? hl - 5 : 0;
    UALM_SYNC();
    const int Pmax = t.N > t.M ? t.N : t.M;
    const unsigned tab = t.lutab + 16u * (unsigned)hl;
    R *Fk = F;                     // row k of F
#pragma unroll 1
    for (int j = 0; j < Pmax; j++) {
        // pivot types of this super-step: the last six pivots have their own patterns; a finished system idles on type 12
        const int ty0 = (j >= P) ? 12 : (j == P - 1 ? 6 : 0);
        unsigned ctab = tab + 256u * (unsigned)ty0, apiv = Wb + 8u * 6u, aurow = Wb + 8u * (unsigned)(6 + uq);
        // b(k) of pivot k = 6j + tt; a finished system stays on its last block (no lane eliminates there)
        unsigned abk = B0 + 48u * (unsigned)(j < P ? j : P - 1);
        uint4 cn = lds128(ctab);
#pragma unroll 1
        for (int tt = 0; tt < 6; tt++) {
            const uint4 c = cn;
            if (ty0 != 12) ctab += 256u;
            cn = lds128(ctab);                                   // constants of the next step (tt = 5 reads one entry ahead: unused)
            const bool act = (c.w & 4u) != 0, isr = (c.w & 8u) != 0;
            const unsigned abi = abk + 8u * ((c.w >> 16) & 7u);  // b(k+o)
            const R piv = lds64(apiv);
            const R av = lds64(Wb + c.x);
            const R urow = lds64(aurow);
            const R u = lds64(Wb + c.z);
            const R w = lds64(Wb + c.y);
            const R bk0 = lds64(abk), bk1 = lds64(abk + B1), bi0 = lds64(abi), bi1 = lds64(abi + B1);
            const R a = isr ? 1.0 : av;
            const bool nz = act && (a != 0.0);
            // exact zeros are skipped by the reference (banded_system.hpp:74) and would push the division onto its slow path
            R m = (nz ? a : 1.0) / (act ? piv : 1.0);
            m = nz ? m : (act ? a : 0.0);
            if (act && !isr) sts64(Wb + c.x, m);
            R val = act ? m : urow;
            // a divisor with an all-ones significand is the one case the reciprocal-based division cannot round: flag it
            // (selects, not a branch: the reciprocal lane alone would diverge from the rest of its half-warp)
            const bool ones = (__double_as_longlong(piv) & 0xFFFFFFFFFFFFFll) == 0xFFFFFFFFFFFFFll;
            val = (isr & ones) ? __longlong_as_double(0x7ff8000000000000ll) : val;
            if (c.w & 32u) Fk[(c.w >> 8) & 127u] = val;
            const R mr = __shfl_sync(0xffffffffu, m, (lane & 16) + (int)(c.w & 3u));
            // zero tests on the bit patterns (an fp64 compare has the latency of an fp64 add, and this one sits on the chain)
            const bool unz = ((unsigned long long)__double_as_longlong(u) << 1) != 0ull;
            const bool mnz = ((unsigned long long)__double_as_longlong(mr) << 1) != 0ull;
            if ((c.w & 16u) && unz && mnz) sts64(Wb + c.y, w - mr * u);
            // forward elimination, after the window update so that it does not delay the next pivot (predicated, not a branch)
            const bool fwd = abi != abk && (((unsigned long long)__double_as_longlong(m) << 1) != 0ull);
            sts64_if(fwd, abi, bi0 - m * bk0);
            sts64_if(fwd, abi + B1, bi1 - m * bk1);
            UALM_SYNC();
            Fk += UALM_FW;
            if (ty0 != 12) abk += 8u;
            apiv += 8u * UALM_WROW; aurow += 8u * UALM_WROW;
        }
        // rows 6..11 move up; the next six rows of A enter (each lane moves its own band column: no hazard between lanes)
        if (j + 1 < P && hl < 13) {
            R mv[6];
#pragma unroll
            for (int rr = 0; rr < 6; rr++) mv[rr] = lds64(Wb + 8u * (unsigned)((6 + rr) * UALM_WROW + hl));
#pragma unroll
            for (int rr = 0; rr < 6; rr++) sts64(Wb + 8u * (unsigned)(rr * UALM_WROW + hl), mv[rr]);
            const int r0 = 6 * (j + 1) + 6;
            if (r0 + 5 < n6 - 3) {      // six interior junction rows, every band column inside the matrix
#pragma unroll
                for (int rr = 0; rr < 6; rr++) sts64(Wb + 8u * (unsigned)((6 + rr) * UALM_WROW + hl), tmv[rr]);
            } else {
#pragma unroll 1
                for (int rr = 0; rr < 6; rr++) {
                    const int r = r0 + rr, cc = r - 6 + hl;
                    R v = 0.0;
                    if (r < n6 && cc >= 0 && cc < n6) v = TM[tmpl_index(r, n6) * UALM_FW + hl];
                    sts64(Wb + 8u * (unsigned)((6 + rr) * UALM_WROW + hl), v);
                }
            }
        }
        UALM_SYNC();
    }
}

// ---------------------------------------------------------------------------------------------
// Triangular sweeps (banded_system.hpp:104-145), one block of six rows at a time with the static patterns above and the
// reference's per-element update order (ascending j for the forward sweeps, descending j for the backward ones, then the
// division).  L y = b (banded_system.hpp:96-103) runs inside lu_dual.
//   KIND 1: U x = y      blocks descending, entries F[i][6+d],  then / F[i][6]
//   KIND 2: U^T y = b    blocks ascending,  entries U(i-d,i) = F[i-d][6+d] (the neighbour block's rows), then / F[i][6]
//   KIND 3: L^T x = y    blocks descending, entries L(i+d,i) = F[i+d][6-d]
// Bit d-1 of the mask of row type t (= row mod 6) says whether term d can be non-zero; the last block of a system (tail
// rows) uses the full mask for KIND 3.  Factor blocks arrive through a UALM_RINGB-block cp.async ring per system
// (prefetch distance UALM_RINGB - 2 blocks); the previous block's six results stay in registers, so no window shifting is needed.
// ---------------------------------------------------------------------------------------------
// six 6-bit masks packed per kind (row type t at bits 6t..6t+5)
__host__ __device__ constexpr unsigned long long pack6(int a, int b, int c, int d, int e, int f)
{
    return (unsigned long long)a | ((unsigned long long)b << 6) | ((unsigned long long)c << 12) | ((unsigned long long)d << 18) |
           ((unsigned long long)e << 24) | ((unsigned long long)f << 30);
}
__host__ __device__ constexpr int sweep_mask(int kind, int t)
{
    return (int)(((kind == 1 ? pack6(0x0c, 0x06, 0x03, 0x23, 0x21, 0x18)      // U rows
                 : kind == 2 ? pack6(0x00, 0x00, 0x00, 0x2f, 0x3f, 0x03)      // U columns
                             : pack6(0x30, 0x38, 0x3c, 0x1e, 0x0f, 0x07))     // L columns
                  >> (6 * t)) & 0x3f);
}

template <int KIND, int NCOL, bool FULL, bool EXACT, class BP>
__device__ __forceinline__ bool sweep_rows(SPtr blk, SPtr nb, bool hasnb, BP b0, BP b1, int bst, int row0, const R (&rhs0)[6], const R (&rhs1)[6],
                                           const R (&prev0)[6], const R (&prev1)[6], R (&cur0)[6], R (&cur1)[6])
{
    constexpr bool ASC = (KIND == 2);
    constexpr bool DIV = (KIND == 1 || KIND == 2);
    constexpr bool TR = (KIND == 2 || KIND == 3);   // transposed access: the factor entry lives in the neighbour's row
    bool bad = false;
    // every factor entry of the block first: the shared-memory proxies are ordered (asm volatile), so a load placed after the
    // store of the previous row's result would expose one shared-memory latency per row on the dependent chain
    R fv[6][7], dgv[6], rdgv[6];
#pragma unroll
    for (int t = 0; t < 6; t++) {
        const SPtr f = blk + t * UALM_FW;
#pragma unroll
        for (int d = 6; d >= 1; d--) {
            fv[t][d] = 0.0;
            if (FULL || ((sweep_mask(KIND, t) >> (d - 1)) & 1)) {
                const int tn = ASC ? t - d : t + d;
                const bool incur = ASC ? (tn >= 0) : (tn <= 5);
                const int tq = incur ? tn : (ASC ? tn + 6 : tn - 6);
                // factor entry: KIND 1: U(i,i+d) = F[i][6+d]; KIND 2: U(i-d,i) = F[i-d][6+d]; KIND 3: L(i+d,i) = F[i+d][6-d]
                if (!TR) fv[t][d] = f[6 + d];
                else if (incur) fv[t][d] = blk[tq * UALM_FW + (ASC ? 6 + d : 6 - d)];
                else fv[t][d] = hasnb ? (R)nb[tq * UALM_FW + (ASC ? 6 + d : 6 - d)] : 0.0;
            }
        }
        if (DIV) { dgv[t] = f[6]; rdgv[t] = EXACT ? 0.0 : (R)f[13]; }
    }
#pragma unroll
    for (int tt = 0; tt < 6; tt++) {
        const int t = ASC ? tt : 5 - tt;            // row type processed now
        R v0 = rhs0[t], v1 = rhs1[t];
#pragma unroll
        for (int d = 6; d >= 1; d--) {
            if (FULL || ((sweep_mask(KIND, t) >> (d - 1)) & 1)) {
                // neighbour index: ascending kinds use row i-d, descending kinds row i+d
                const int tn = ASC ? t - d : t + d;
                const bool incur = ASC ? (tn >= 0) : (tn <= 5);
                const int tq = incur ? tn : (ASC ? tn + 6 : tn - 6);
                // the reference skips exact-zero factors (banded_system.hpp:103,112,131,139); subtracting 0 * w instead leaves
                // every value unchanged (at most the sign of an exact zero differs), so no test is needed here
                const R w0 = incur ? cur0[tq] : prev0[tq];
                v0 = v0 - fv[t][d] * w0;
                if (NCOL == 2) {
                    const R w1 = incur ? cur1[tq] : prev1[tq];
                    v1 = v1 - fv[t][d] * w1;
                }
            }
        }
        if (DIV) {
            const R dg = dgv[t];
            if (EXACT) {
                v0 = v0 / dg;
                if (NCOL == 2) v1 = v1 / dg;
            } else {
                v0 = div_by_recip_flag(v0, dg, rdgv[t], bad);
                if (NCOL == 2) v1 = div_by_recip_flag(v1, dg, rdgv[t], bad);
            }
        }
        at(b0, (row0 + t) * bst) = v0;
        cur0[t] = v0;
        if (NCOL == 2) { at(b1, (row0 + t) * bst) = v1; cur1[t] = v1; }
    }
    return bad;
}

template <int KIND, int NCOL, bool FULL, class BP>
__device__ __forceinline__ void sweep_block(SPtr blk, SPtr nb, bool hasnb, BP b0, BP b1, int bst, int row0, R (&prev0)[6], R (&prev1)[6])
{
    constexpr bool DIV = (KIND == 1 || KIND == 2);
    R cur0[6], cur1[6];
    // all right-hand-side entries of the block first: they do not depend on the chain, and issuing them together pays the
    // memory latency once per block instead of once per row (the stores below would otherwise fence them)
    R rhs0[6], rhs1[6];
#pragma unroll
    for (int q = 0; q < 6; q++) {
        rhs0[q] = at(b0, (row0 + q) * bst);
        rhs1[q] = (NCOL == 2) ? (R)at(b1, (row0 + q) * bst) : 0.0;
    }
    // the divisions use the stored reciprocals; a quotient the reciprocal route cannot round (flag) makes the lane redo the
    // block with IEEE divisions -- one branch per block instead of one per row on the dependent chain
    const bool bad = sweep_rows<KIND, NCOL, FULL, false, BP>(blk, nb, hasnb, b0, b1, bst, row0, rhs0, rhs1, prev0, prev1, cur0, cur1);
    if (DIV && bad) sweep_rows<KIND, NCOL, FULL, true, BP>(blk, nb, hasnb, b0, b1, bst, row0, rhs0, rhs1, prev0, prev1, cur0, cur1);
#pragma unroll
    for (int q = 0; q < 6; q++) { prev0[q] = cur0[q]; if (NCOL == 2) prev1[q] = cur1[q]; }
}

// facA/nA: system of the lanes with sel == 0, facB/nB: system of the lanes with sel == 1 (DUAL only).  Each active lane
// solves NCOL right-hand sides.  ringA/ringB: 8 blocks x 6 rows x UALM_FW doubles each.
template <int KIND, int NCOL, bool DUAL, class BP>
__device__ UALM_NOINLINE void sweep(const R *facA, int PA, const R *facB, int PB, SPtr ringA, SPtr ringB, BP b0, BP b1, int bst, int sel,
                                    bool active, int lane, int cstart = 0)
{
    constexpr bool ASC = (KIND == 2);
    constexpr bool LKIND = (KIND == 3);                // the kind whose tail block needs the full pattern
    constexpr int BLK = 6 * UALM_FW;                    // doubles per block (42 x 16 B)
    const int nb = DUAL ? (PA > PB ? PA : PB) : PA;
    auto issue = [&](int c) {
        if (c < PA) {
            const int blk = ASC ? c : PA - 1 - c;
            const R *src = facA + (long long)blk * BLK;
            const SPtr dst = ringA + (c % UALM_RINGB) * BLK;
            for (int p = lane; p < BLK / 2; p += 32) cp_async16(dst.a + 16u * (unsigned)p, src + 2 * p);
        }
        if (DUAL && c < PB) {
            const int blk = ASC ? c : PB - 1 - c;
            const R *src = facB + (long long)blk * BLK;
            const SPtr dst = ringB + (c % UALM_RINGB) * BLK;
            for (int p = lane; p < BLK / 2; p += 32) cp_async16(dst.a + 16u * (unsigned)p, src + 2 * p);
        }
        cp_async_commit();
    };
    R prev0[6] = {0, 0, 0, 0, 0, 0}, prev1[6] = {0, 0, 0, 0, 0, 0};
    const int myP = (DUAL && sel) ? PB : PA;
    const SPtr myring = (DUAL && sel) ? ringB : ringA;
    // cstart (ascending kinds only): blocks before it hold an all-zero right-hand side, whose solution is zero as well
    for (int q = 0; q < UALM_RINGB - 2; q++) issue(cstart + q);
#pragma unroll 1
    for (int c = cstart; c < nb; c++) {
        issue(c + UALM_RINGB - 2);
        cp_async_wait<UALM_RINGB - 2>();
        UALM_SYNC();
        if (active && c < myP) {
            const int blk = ASC ? c : myP - 1 - c;
            const SPtr chunk = myring + (c % UALM_RINGB) * BLK;
            const SPtr nbr = myring + ((c + UALM_RINGB - 1) % UALM_RINGB) * BLK;      // the block processed just before (still in the ring)
            const bool hasnb = c > cstart;
            if (LKIND && blk == myP - 1) sweep_block<KIND, NCOL, true, BP>(chunk, nbr, hasnb, b0, b1, bst, 6 * blk, prev0, prev1);
            else sweep_block<KIND, NCOL, false, BP>(chunk, nbr, hasnb, b0, b1, bst, 6 * blk, prev0, prev1);
        }
        UALM_SYNC();
    }
    cp_async_wait<0>();
}

// x -> T powers, LU of both systems, coefficients c   (alm_traj_opt.cpp:293-299 + se2traj.hpp:595-680)
__device__ UALM_NOINLINE void minco_generate(Traj &t, int lane)
{
    const int N = t.N, M = t.M, nx = 6 * N, ny = 6 * M;
    if (lane == 0) {
        const R tau = t.x[0];
        const R T = expC2(tau);
        const R Tx = T / (R)N, Ty = T / (R)M; // calTfromTau alm_traj_opt.h:257-261
        t.sc[SC_TX1] = Tx; t.sc[SC_TX2] = Tx * Tx; t.sc[SC_TX3] = t.sc[SC_TX2] * Tx; t.sc[SC_TX4] = t.sc[SC_TX2] * t.sc[SC_TX2];
        t.sc[SC_TX5] = t.sc[SC_TX4] * Tx;
        t.sc[SC_TY1] = Ty; t.sc[SC_TY2] = Ty * Ty; t.sc[SC_TY3] = t.sc[SC_TY2] * Ty; t.sc[SC_TY4] = t.sc[SC_TY2] * t.sc[SC_TY2];
        t.sc[SC_TY5] = t.sc[SC_TY4] * Ty;
    }
    // right-hand sides (se2traj.hpp:615-617, 653, 672-674)
    for (int q = lane; q < 2 * nx; q += 32) t.cxy[q] = 0.0;
    for (int q = lane; q < ny; q += 32) t.cyaw[q] = 0.0;
    UALM_SYNC();
    const R *bnd = t.pd->bnd;
    const SPtr Pxy = t.x + 1, Pyaw = t.x + (1 + 2 * (N - 1));
    if (lane < 2) {
        const int d = lane;
        t.cxy[0 + d * nx] = bnd[d + 0]; t.cxy[1 + d * nx] = bnd[d + 2]; t.cxy[2 + d * nx] = bnd[d + 4];
        t.cxy[nx - 3 + d * nx] = bnd[6 + d + 0]; t.cxy[nx - 2 + d * nx] = bnd[6 + d + 2]; t.cxy[nx - 1 + d * nx] = bnd[6 + d + 4];
    }
    if (lane == 2) {
        t.cyaw[0] = bnd[12]; t.cyaw[1] = bnd[13]; t.cyaw[2] = bnd[14];
        t.cyaw[ny - 3] = bnd[15]; t.cyaw[ny - 2] = bnd[16]; t.cyaw[ny - 1] = bnd[17];
    }
    for (int i = lane; i < N - 1; i += 32) {
        t.cxy[6 * i + 5] = Pxy[2 * i];
        t.cxy[6 * i + 5 + nx] = Pxy[2 * i + 1];
    }
    for (int i = lane; i < M - 1; i += 32) t.cyaw[6 * i + 5] = Pyaw[i];
    UALM_SYNC();
    prof_mark(t, lane, PF_FILL);
    lu_dual(t, lane);   // also L y = b on the right-hand sides
    prof_mark(t, lane, PF_LU);
    // U x = y: lanes 0/1: x / y columns against the xy factors; lane 2: the yaw column, all in lockstep
    {
        const SPtr col = lane < 2 ? t.cxy + lane * nx : t.cyaw;
        sweep<1, 1, true, SPtr>(t.Fxy, N, t.Fyaw, M, t.ring, t.ring + UALM_RINGB * 6 * UALM_FW, col, col, 1, lane == 2, lane < 3, lane);
    }
    UALM_SYNC();
    prof_mark(t, lane, PF_SOLVE);
}

// jerk gradient entries on the fly (se2traj.hpp:719-747): dJ/dc(6i+k, col) and dJ/dT(i)
__device__ UALM_NOINLINE R jerk_gc(SPtr c6, int k, R T1, R T2, R T3, R T4, R T5)
{
    const R c3 = c6[3], c4 = c6[4], c5 = c6[5];
    if (k == 5) return 240.0 * c3 * T3 + 720.0 * c4 * T4 + 1440.0 * c5 * T5;
    if (k == 4) return 144.0 * c3 * T2 + 384.0 * c4 * T3 + 720.0 * c5 * T4;
    if (k == 3) return 72.0 * c3 * T1 + 144.0 * c4 * T2 + 240.0 * c5 * T3;
    return 0.0;
}
// per-piece jerk energy and dJ/dT (se2traj.hpp:702-707, 739-744); a = first column block, b = second (or null)
__device__ UALM_NOINLINE void jerk_piece(SPtr a, SPtr b, bool has_b, R T1, R T2, R T3, R T4, R T5, R &e, R &gt)
{
    R d33, d43, d44, d53, d54, d55;
    if (has_b) {
        d33 = a[3] * a[3] + b[3] * b[3]; d43 = a[4] * a[3] + b[4] * b[3]; d44 = a[4] * a[4] + b[4] * b[4];
        d53 = a[5] * a[3] + b[5] * b[3]; d54 = a[5] * a[4] + b[5] * b[4]; d55 = a[5] * a[5] + b[5] * b[5];
    } else {
        d33 = a[3] * a[3]; d43 = a[4] * a[3]; d44 = a[4] * a[4]; d53 = a[5] * a[3]; d54 = a[5] * a[4]; d55 = a[5] * a[5];
    }
    e = 36.0 * d33 * T1 + 144.0 * d43 * T2 + 192.0 * d44 * T3 + 240.0 * d53 * T3 + 720.0 * d54 * T4 + 720.0 * d55 * T5;
    gt = 36.0 * d33 + 288.0 * d43 * T1 + 576.0 * d44 * T2 + 720.0 * d53 * T2 + 2880.0 * d54 * T3 + 3600.0 * d55 * T4;
}

// jerk cost (se2traj.hpp:697-710, 852-855): per-piece energies in parallel (parked in gTxy/gTyaw), summed by lane 0 in
// piece order like the reference's `energy +=` loop.  Leaves sc[SC_JERKRAW].
__device__ UALM_NOINLINE void jerk_cost(Traj &t, int lane)
{
    const int N = t.N, M = t.M, nx = 6 * N;
    for (int q = lane; q < N + M; q += 32) {
        R e, gt;
        if (q < N) { jerk_piece(t.cxy + 6 * q, t.cxy + (6 * q + nx), true, t.sc[SC_TX1], t.sc[SC_TX2], t.sc[SC_TX3], t.sc[SC_TX4], t.sc[SC_TX5], e, gt); t.gTxy[q] = e; }
        else { jerk_piece(t.cyaw + 6 * (q - N), t.cyaw, false, t.sc[SC_TY1], t.sc[SC_TY2], t.sc[SC_TY3], t.sc[SC_TY4], t.sc[SC_TY5], e, gt); t.gTyaw[q - N] = e; }
    }
    UALM_SYNC();
    if (lane == 0) {
        R ex = 0.0, ey = 0.0;
        for (int i = 0; i < N; i++) ex += t.gTxy[i];
        for (int i = 0; i < M; i++) ey += t.gTyaw[i];
        t.sc[SC_JERKRAW] = ex + ey;
    }
    UALM_SYNC();
}

// ---------------------------------------------------------------------------------------------
// UnevenMap::getAllWithGrad  (uneven_map.h:258-377)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool map_in(const DevMap &m, const R pos[3]) // uneven_map.h:437-454
{
    if (pos[0] < m.origin[0] + 1e-4 || pos[1] < m.origin[1] + 1e-4 || pos[2] < m.origin[2] + 1e-4) return false;
    if (pos[0] > m.maxb[0] - 1e-4 || pos[1] > m.maxb[1] - 1e-4 || pos[2] > m.maxb[2] - 1e-4) return false;
    return true;
}

// sc_yaw: sin and cos of pos[2] when the caller already has them (have_sc), else computed here
template <bool INL>
__device__ __forceinline__ void map_get_all_with_grad_impl(const DevMap &m, const R pos[3], R values[7], R grads[7][3], bool have_sc, double2 sc_yaw)
{
    // the map descriptor is a kernel parameter read through a generic pointer: fetch every field once (a re-read after any
    // store costs a long-scoreboard wait, and the corner loop below used to re-read vn[2] sixteen times)
    const int vn0 = m.vn[0], vn1 = m.vn[1], vn2 = m.vn[2];
    const float4 *const cells = m.cells;
    const double *const cells64 = m.cells64;
    const R xy_res = m.xy_res, yaw_res = m.yaw_res, xy_inv = m.xy_inv, yaw_inv = m.yaw_inv, org0 = m.origin[0], org1 = m.origin[1], org2 = m.origin[2];
    R rs[3], rg[4][3];
    const bool in = map_in(m, pos);
    if (!in) {
        for (int r = 0; r < 4; r++) for (int k = 0; k < 3; k++) rg[r][k] = 0.0;
        rs[0] = rs[1] = rs[2] = 0.0;
    } else {
        R pos_m[3] = {pos[0] - 0.5 * xy_res, pos[1] - 0.5 * xy_res, pos[2] - 0.5 * yaw_res};
        normSO2(pos_m[2]);
        int idx[3];
        idx[0] = (int)floor((pos_m[0] - org0) * xy_inv);
        idx[1] = (int)floor((pos_m[1] - org1) * xy_inv);
        idx[2] = (int)floor((pos_m[2] - org2) * yaw_inv);
        R idx_pos[3];
        idx_pos[0] = ((R)idx[0] + 0.5) * xy_res + org0;
        idx_pos[1] = ((R)idx[1] + 0.5) * xy_res + org1;
        idx_pos[2] = ((R)idx[2] + 0.5) * yaw_res + org2;
        R diff[3];
        diff[0] = (pos[0] - idx_pos[0]) * xy_inv;
        diff[1] = (pos[1] - idx_pos[1]) * xy_inv;
        // the eight corner cells: clamped x / y and wrapped yaw indices once, then start the loads now, ahead of the angle
        // difference below, which the loads cannot cross
        int cx[2], cy[2], cw[2];
#pragma unroll
        for (int e = 0; e < 2; e++) {
            cx[e] = max(min(idx[0] + e, vn0 - 1), 0);
            cy[e] = max(min(idx[1] + e, vn1 - 1), 0);
            cw[e] = wrap_index(idx[2] + e, vn2);
        }
        size_t cadr[2][2][2];
#pragma unroll
        for (int x = 0; x < 2; x++)
#pragma unroll
            for (int y = 0; y < 2; y++)
#pragma unroll
                for (int w = 0; w < 2; w++) {
                    const size_t adr = (size_t)cx[x] * vn1 * vn2 + (size_t)cy[y] * vn2 + cw[w];
                    cadr[x][y][w] = adr;
                    prefetch_l1(cells64 ? (const void *)(cells64 + 4 * adr) : (const void *)&cells[adr]);
                }
        {
            R sd, cd;
            { const double2 scv = sincos_sel<INL>(pos[2] - idx_pos[2]); sd = scv.x; cd = scv.y; }
            diff[2] = atan2_sel<INL>(sd, cd) * yaw_inv;
        }
        R v[2][2][2][3];
#pragma unroll
        for (int x = 0; x < 2; x++)
#pragma unroll
            for (int y = 0; y < 2; y++)
#pragma unroll
                for (int w = 0; w < 2; w++) {
                    // inlined (the penalty loop), the addresses are held across the angle difference; the out-of-line copy forms
                    // them again after its two calls: holding eight addresses across the calls took check_kernel from 166 to 205
                    // registers
                    const size_t adr = INL ? cadr[x][y][w] : (size_t)cx[x] * vn1 * vn2 + (size_t)cy[y] * vn2 + wrap_index(idx[2] + w, vn2);
                    if (cells64) {
                        const double2 lo = __ldg((const double2 *)(cells64 + 4 * adr)), hi = __ldg((const double2 *)(cells64 + 4 * adr) + 1);
                        v[x][y][w][0] = lo.y; v[x][y][w][1] = hi.x; v[x][y][w][2] = hi.y;
                    } else {
                        const float4 cell = __ldg(&cells[adr]);
                        v[x][y][w][0] = (R)cell.y; v[x][y][w][1] = (R)cell.z; v[x][y][w][2] = (R)cell.w;
                    }
                }
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const R v00 = v[0][0][0][k] * (1 - diff[0]) + v[1][0][0][k] * diff[0];
            const R v01 = v[0][0][1][k] * (1 - diff[0]) + v[1][0][1][k] * diff[0];
            const R v10 = v[0][1][0][k] * (1 - diff[0]) + v[1][1][0][k] * diff[0];
            const R v11 = v[0][1][1][k] * (1 - diff[0]) + v[1][1][1][k] * diff[0];
            const R v0 = v00 * (1 - diff[1]) + v10 * diff[1];
            const R v1 = v01 * (1 - diff[1]) + v11 * diff[1];
            rs[k] = v0 * (1 - diff[2]) + v1 * diff[2];
            rg[k][2] = (v1 - v0) * yaw_inv;
            rg[k][1] = ((v10 - v00) * (1 - diff[2]) + (v11 - v01) * diff[2]) * xy_inv;
            R g0 = (1 - diff[2]) * (1 - diff[1]) * (v[1][0][0][k] - v[0][0][0][k]);
            g0 += (1 - diff[2]) * diff[1] * (v[1][1][0][k] - v[0][1][0][k]);
            g0 += diff[2] * (1 - diff[1]) * (v[1][0][1][k] - v[0][0][1][k]);
            g0 += diff[2] * diff[1] * (v[1][1][1][k] - v[0][1][1][k]);
            g0 *= xy_inv;
            rg[k][0] = g0;
        }
    }
    const R c = sqrt(1.0 - rs[1] * rs[1] - rs[2] * rs[2]);
    // inside the map, the reference divides by the same square root of the same expression (its `cc`): c, formed once
    if (in) {
#pragma unroll
        for (int k = 0; k < 3; k++) rg[3][k] = div_nz(-(rg[1][k] * rs[1] + rg[2][k] * rs[2]), c);
    }
    const R inv_c = 1.0 / c;
    R syaw, cyaw;
    { const double2 scv = have_sc ? sc_yaw : sincos_sel<INL>(pos[2]); syaw = scv.x; cyaw = scv.y; }
    const R xyaw[2] = {cyaw, syaw};
    const R yyaw[2] = {-syaw, cyaw};
    const R tt = xyaw[0] * rs[1] + xyaw[1] * rs[2];
    const R s = -(yyaw[0] * rs[1] + yyaw[1] * rs[2]);
    const R sqrt_1_t2 = sqrt(1.0 - tt * tt);
    const R inv_sqrt_1_t2 = 1.0 / sqrt_1_t2;
    const R inv_sqrt_1_t2_3 = inv_sqrt_1_t2 * inv_sqrt_1_t2 * inv_sqrt_1_t2;
    R dt[3], ds[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        dt[k] = rg[1][k] * xyaw[0] + rg[2][k] * xyaw[1];
        ds[k] = -(rg[1][k] * yyaw[0] + rg[2][k] * yyaw[1]);
    }
    dt[2] -= s;
    ds[2] += tt;
    values[0] = inv_sqrt_1_t2;
    values[1] = -c * tt * inv_sqrt_1_t2;
    values[2] = sqrt_1_t2 * inv_c;
    values[3] = s * inv_sqrt_1_t2;
    values[4] = c;
    values[5] = inv_c;
    values[6] = rs[0];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        grads[0][k] = tt * inv_sqrt_1_t2_3 * dt[k];
        grads[1][k] = -(tt * inv_sqrt_1_t2 * rg[3][k] + inv_sqrt_1_t2_3 * c * dt[k]);
        grads[2][k] = -inv_c * (tt * inv_sqrt_1_t2 * dt[k] + sqrt_1_t2 * inv_c * rg[3][k]);
        grads[3][k] = inv_sqrt_1_t2 * ds[k] + tt * inv_sqrt_1_t2_3 * s * dt[k];
        grads[4][k] = rg[3][k];
        grads[5][k] = -inv_c * inv_c * rg[3][k];
        grads[6][k] = rg[0][k];
    }
}

__device__ UALM_NOINLINE void map_get_all_with_grad(const DevMap &m, const R pos[3], R values[7], R grads[7][3])
{
    map_get_all_with_grad_impl<false>(m, pos, values, grads, false, make_double2(0.0, 0.0));
}

// kinematics of one constraint sample (alm_traj_opt.cpp:733-817)
struct SampleK {
    R b0[6], b1[6], b2[6], b3[6], y0[6], y1[6], y2[6];
    R pos[2], vel[2], acc[2], jer[2];
    R yaw, dyaw, d2yaw, syaw, cyaw, v_norm, lon_acc, lat_acc;
    R tv[7], tg[7][3];
    R vx, wz, ax, ay, curv_snorm;
    int yaw_idx;
};

// before_map(S) runs once the kinematics are complete and before the map lookup: the penalty loop stores there what it only
// writes out, so that those values are not held in registers across the lookup
template <bool INL, class BeforeMap>
__device__ __forceinline__ void sample_kin_impl(const Traj &t, const DevMap &map, R gravity, int i, R s1, R base_time, SampleK &S, BeforeMap before_map)
{
    const int nx = 6 * t.N;
    const R s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2, s5 = s4 * s1;
    S.b0[0] = 1.0; S.b0[1] = s1; S.b0[2] = s2; S.b0[3] = s3; S.b0[4] = s4; S.b0[5] = s5;
    S.b1[0] = 0.0; S.b1[1] = 1.0; S.b1[2] = 2.0 * s1; S.b1[3] = 3.0 * s2; S.b1[4] = 4.0 * s3; S.b1[5] = 5.0 * s4;
    S.b2[0] = 0.0; S.b2[1] = 0.0; S.b2[2] = 2.0; S.b2[3] = 6.0 * s1; S.b2[4] = 12.0 * s2; S.b2[5] = 20.0 * s3;
    S.b3[0] = 0.0; S.b3[1] = 0.0; S.b3[2] = 0.0; S.b3[3] = 6.0; S.b3[4] = 24.0 * s1; S.b3[5] = 60.0 * s2;
#pragma unroll
    for (int d = 0; d < 2; d++) {
        R p = 0, v = 0, a = 0, j = 0;
#pragma unroll
        for (int k = 0; k < 6; k++) {
            const R c = t.cxy[6 * i + k + d * nx];
            p += c * S.b0[k]; v += c * S.b1[k]; a += c * S.b2[k]; j += c * S.b3[k];
        }
        S.pos[d] = p; S.vel[d] = v; S.acc[d] = a; S.jer[d] = j;
    }
    const R Ty = t.sc[SC_TY1];
    const R now_time = s1 + base_time;
    int yaw_idx = (int)div_by_recip(now_time, Ty, t.sc[SC_RTY]);
    if (yaw_idx >= t.M) yaw_idx = t.M - 1;
    S.yaw_idx = yaw_idx;
    const R sy1 = now_time - (R)yaw_idx * Ty;
    const R sy2 = sy1 * sy1, sy3 = sy2 * sy1, sy4 = sy2 * sy2, sy5 = sy4 * sy1;
    S.y0[0] = 1.0; S.y0[1] = sy1; S.y0[2] = sy2; S.y0[3] = sy3; S.y0[4] = sy4; S.y0[5] = sy5;
    S.y1[0] = 0.0; S.y1[1] = 1.0; S.y1[2] = 2.0 * sy1; S.y1[3] = 3.0 * sy2; S.y1[4] = 4.0 * sy3; S.y1[5] = 5.0 * sy4;
    S.y2[0] = 0.0; S.y2[1] = 0.0; S.y2[2] = 2.0; S.y2[3] = 6.0 * sy1; S.y2[4] = 12.0 * sy2; S.y2[5] = 20.0 * sy3;
    R yaw = 0, dyaw = 0, d2yaw = 0;
#pragma unroll
    for (int k = 0; k < 6; k++) {
        const R c = t.cyaw[6 * yaw_idx + k];
        yaw += c * S.y0[k]; dyaw += c * S.y1[k]; d2yaw += c * S.y2[k];
    }
    S.yaw = yaw; S.dyaw = dyaw; S.d2yaw = d2yaw;
    R se2[3] = {S.pos[0], S.pos[1], yaw};
    normSO2(se2[2]);
    const double2 scv = sincos_sel<INL>(yaw);
    S.syaw = scv.x; S.cyaw = scv.y;
    S.v_norm = sqrt(S.vel[0] * S.vel[0] + S.vel[1] * S.vel[1]);
    S.lon_acc = S.acc[0] * S.cyaw + S.acc[1] * S.syaw;
    S.lat_acc = S.acc[0] * (-S.syaw) + S.acc[1] * S.cyaw;
    before_map(S);
    // the map's sin / cos of the wrapped yaw are the ones above whenever the wrap left the yaw's bits unchanged
    if (INL) map_get_all_with_grad_impl<true>(map, se2, S.tv, S.tg, __double_as_longlong(se2[2]) == __double_as_longlong(yaw), scv);
    else map_get_all_with_grad(map, se2, S.tv, S.tg);
    S.vx = S.v_norm * S.tv[0];
    S.wz = dyaw * S.tv[5];
    S.ax = S.lon_acc * S.tv[0] + gravity * S.tv[1];
    S.ay = S.lat_acc * S.tv[2] + gravity * S.tv[3];
    S.curv_snorm = div_nz(S.wz * S.wz, S.vx * S.vx + UALM_DELTA_SIGL);
}

// out-of-line copy (initScaling) and inlined copy (the per-evaluation penalty loop: keeps the sample state in registers)
__device__ UALM_NOINLINE void sample_kin(const Traj &t, const DevMap &map, R gravity, int i, R s1, R base_time, SampleK &S)
{
    sample_kin_impl<false>(t, map, gravity, i, s1, base_time, S, [](const SampleK &) {});
}

// sample-time tables: s1tab[j] = j-fold accumulated step, base[i] = i-fold accumulated T (alm_traj_opt.cpp:713-714, 987-989)
__device__ UALM_NOINLINE void sample_tables(Traj &t, int lane)
{
    if (lane == 0) {
        const R step = t.sc[SC_TX1] / (R)t.K;
        R s1 = 0.0;
        for (int j = 0; j <= t.K; j++) { t.s1tab[j] = s1; s1 += step; }
    }
    if (lane == 1) {
        R b = 0.0;
        for (int i = 0; i < t.N; i++) { t.base[i] = b; b += t.sc[SC_TX1]; }
    }
    if (lane == 2) {
        const R Ty = t.sc[SC_TY1];
        R r = 1.0 / Ty;
        if ((__double_as_longlong(Ty) & 0xFFFFFFFFFFFFFll) == 0xFFFFFFFFFFFFFll) r = __longlong_as_double(0x7ff8000000000000ll);
        t.sc[SC_RTY] = r;
    }
    UALM_SYNC();
}

// ---------------------------------------------------------------------------------------------
// calConstrainCostGrad, phase A: one lane per sample (alm_traj_opt.cpp:710-964).  Writes hx/gx, the 8 cost
// terms and the per-sample gradients to the scratch; phase B accumulates them in the reference's order.
// ---------------------------------------------------------------------------------------------
// the square of limit `slot` of the problem's row, formed as the reference forms it (max_vel * max_vel)
__device__ __forceinline__ R sq_at(const Traj &t, int slot)
{
    const R v = t.sc[slot];
    return v * v;
}
__device__ UALM_NOINLINE void penalty_samples(Traj &t, const DevMap &map, const DevParams &p, int gtid, int GT)
{
    const int S = t.S, K = t.K;
    const R rho = t.sc[SC_RHO], scale_fx = t.sc[SC_SCALE_FX];
    const R rrho = ((__double_as_longlong(rho) & 0xFFFFFFFFFFFFFll) == 0xFFFFFFFFFFFFFll) ? __longlong_as_double(0x7ff8000000000000ll) : 1.0 / rho;   // RN(1/rho): x / rho below is formed as div_by_recip(x, rho, rrho), bit-identical to the IEEE quotient
    const R step = t.sc[SC_TX1] / (R)K;
    R *scr = t.scr;
    // parameters (kernel-parameter space through a generic pointer) and trajectory pointers (a struct in local memory) once.  The
    // problem's row is read from its slot where it is used (sq_at: the squared limits), which keeps it out of the registers the
    // sample loop holds
    const R gravity = p.gravity;
    R *const lambda_p = t.lambda, *const mu_p = t.mu, *const scale_p = t.scale_cx, *const hx_p = t.hx, *const gx_p = t.gx;
    // piece i and index j of sample s = i (K + 1) + j, carried from one sample of the lane to its next instead of a division per
    // sample
    const int K1 = K + 1;
    int i = gtid / K1, j = gtid - i * K1;
    for (int s = gtid; s < S; s += GT) {
        // the duals and scales of this sample are needed only after the kinematics and the map lookup: start their cache lines
        // now, so that their loads, in one batch after the lookup, find them in L1
        prefetch_l1(lambda_p + s);
        prefetch_l1(mu_p + 6 * (size_t)s); prefetch_l1(mu_p + 6 * (size_t)s + 5);
        prefetch_l1(scale_p + 7 * (size_t)s); prefetch_l1(scale_p + 7 * (size_t)s + 6);
        SampleK q;
        sample_kin_impl<true>(t, map, gravity, i, t.s1tab[j], t.base[i], q, [&](const SampleK &k) {
            t.yawidx[s] = (unsigned short)k.yaw_idx;
            scr[(SF_ACC + 0) * S + s] = k.acc[0]; scr[(SF_ACC + 1) * S + s] = k.acc[1];
            scr[(SF_JER + 0) * S + s] = k.jer[0]; scr[(SF_JER + 1) * S + s] = k.jer[1];
            scr[SF_D2YAW * S + s] = k.d2yaw;
            scr[SF_S1YAW * S + s] = k.y0[1];
        });
        R grad_p[2] = {0, 0}, grad_v[2] = {0, 0}, grad_a[2] = {0, 0}, grad_se2[3] = {0, 0, 0};
        R grad_yaw = 0, grad_dyaw = 0, grad_vx2 = 0, grad_wz = 0, grad_ax = 0, grad_ay = 0, aug_grad = 0;
        const R inv_cos_vphix = q.tv[0], inv_cos_vphiy = q.tv[2], cos_xi = q.tv[4], inv_cos_xi = q.tv[5], sigma = q.tv[6];
        const R vx = q.vx, wz = q.wz, ax = q.ax, ay = q.ay, curv_snorm = q.curv_snorm;
        R sc7[7], mu6[6];
#pragma unroll
        for (int k = 0; k < 7; k++) sc7[k] = scale_p[7 * (size_t)s + k];
        // without scaling, the curvature and surface terms are weighted by fixed factors instead of their scales (the flag is
        // read here, where it is used, rather than held across the loop)
        if (!p.use_scaling) { sc7[4] = UALM_CUR_SCALE; sc7[6] = UALM_SIG_SCALE; }
#pragma unroll
        for (int k = 0; k < 6; k++) mu6[k] = mu_p[6 * (size_t)s + k];
        const R lambda_s = lambda_p[s];
        R *gx6 = gx_p + 6 * (size_t)s;

        R omega;
        if (j == 0 || j == K) omega = 0.5 * t.sc[SC_RHO_TER] * step * scale_fx;
        else omega = t.sc[SC_RHO_TER] * step * scale_fx;
        const R user_cost = omega * sigma * sigma;
        scr[(SF_COST0 + 0) * S + s] = user_cost;
        scr[SF_USER * S + s] = user_cost;
#pragma unroll
        for (int k = 0; k < 3; k++) grad_se2[k] += omega * q.tg[6][k] * sigma * 2.0;

        { // non-holonomic
            const R nonh_lambda = lambda_s;
            const R nhy0 = q.syaw, nhy1 = -q.cyaw;
            const R h = (q.vel[0] * nhy0 + q.vel[1] * nhy1) * sc7[0];
            hx_p[s] = h;
            scr[(SF_COST0 + 1) * S + s] = h * (nonh_lambda + 0.5 * rho * h);
            const R nonh_grad = (rho * h + nonh_lambda) * sc7[0];
            grad_v[0] += nonh_grad * nhy0; grad_v[1] += nonh_grad * nhy1;
            grad_yaw += nonh_grad * (q.vel[0] * q.cyaw + q.vel[1] * q.syaw);
        }
        { // longitude velocity
            const R m_ = mu6[0];
            const R gv = (vx * vx - sq_at(t, SC_MAX_VEL)) * sc7[1];
            gx6[0] = gv;
            if (rho * gv + m_ > 0) {
                scr[(SF_COST0 + 2) * S + s] = gv * (m_ + 0.5 * rho * gv);
                aug_grad = (rho * gv + m_) * sc7[1];
                grad_vx2 += aug_grad;
            } else scr[(SF_COST0 + 2) * S + s] = div_by_recip(-0.5 * m_ * m_, rho, rrho);
        }
        { // longitude acceleration
            const R m_ = mu6[1];
            const R gv = (ax * ax - sq_at(t, SC_MAX_ACC_LON)) * sc7[2];
            gx6[1] = gv;
            if (rho * gv + m_ > 0) {
                scr[(SF_COST0 + 3) * S + s] = gv * (m_ + 0.5 * rho * gv);
                aug_grad = (rho * gv + m_) * sc7[2];
                grad_ax += aug_grad * 2.0 * ax;
            } else scr[(SF_COST0 + 3) * S + s] = div_by_recip(-0.5 * m_ * m_, rho, rrho);
        }
        { // latitude acceleration
            const R m_ = mu6[2];
            const R gv = (ay * ay - sq_at(t, SC_MAX_ACC_LAT)) * sc7[3];
            gx6[2] = gv;
            if (rho * gv + m_ > 0) {
                scr[(SF_COST0 + 4) * S + s] = gv * (m_ + 0.5 * rho * gv);
                aug_grad = (rho * gv + m_) * sc7[3];
                grad_ay += aug_grad * 2.0 * ay;
            } else scr[(SF_COST0 + 4) * S + s] = div_by_recip(-0.5 * m_ * m_, rho, rrho);
        }
        { // curvature
            const R m_ = mu6[3];
            const R gv = (curv_snorm - sq_at(t, SC_MAX_KAP)) * sc7[4];
            gx6[3] = gv;
            if (rho * gv + m_ > 0) {
                const R denominator = 1.0 / (vx * vx + UALM_DELTA_SIGL);
                scr[(SF_COST0 + 5) * S + s] = gv * (m_ + 0.5 * rho * gv);
                aug_grad = (rho * gv + m_) * sc7[4];
                grad_wz += aug_grad * denominator * 2.0 * wz;
                grad_vx2 -= aug_grad * curv_snorm * denominator;
            } else scr[(SF_COST0 + 5) * S + s] = div_by_recip(-0.5 * m_ * m_, rho, rrho);
        }
        { // attitude
            const R m_ = mu6[4];
            const R gv = ((R)t.sc[SC_MIN_CXI] - cos_xi) * sc7[5];
            gx6[4] = gv;
            if (rho * gv + m_ > 0) {
                scr[(SF_COST0 + 6) * S + s] = gv * (m_ + 0.5 * rho * gv);
                const R ag = rho * gv + m_;
#pragma unroll
                for (int k = 0; k < 3; k++) grad_se2[k] -= ag * q.tg[4][k] * sc7[5];
            } else scr[(SF_COST0 + 6) * S + s] = div_by_recip(-0.5 * m_ * m_, rho, rrho);
        }
        { // surface variation
            const R m_ = mu6[5];
            const R gv = (sigma - t.sc[SC_MAX_SIG]) * sc7[6];
            gx6[5] = gv;
            if (rho * gv + m_ > 0) {
                scr[(SF_COST0 + 7) * S + s] = gv * (m_ + 0.5 * rho * gv);
                const R ag = rho * gv + m_;
#pragma unroll
                for (int k = 0; k < 3; k++) grad_se2[k] += ag * q.tg[6][k] * sc7[6];
            } else scr[(SF_COST0 + 7) * S + s] = div_by_recip(-0.5 * m_ * m_, rho, rrho);
        }
        // process with vx, wz, ax (alm_traj_opt.cpp:948-964)
#pragma unroll
        for (int d = 0; d < 2; d++) grad_v[d] += grad_vx2 * inv_cos_vphix * inv_cos_vphix * 2.0 * q.vel[d];
#pragma unroll
        for (int k = 0; k < 3; k++) grad_se2[k] += grad_vx2 * q.v_norm * q.v_norm * 2.0 * inv_cos_vphix * q.tg[0][k];
        grad_dyaw += grad_wz * inv_cos_xi;
#pragma unroll
        for (int k = 0; k < 3; k++) grad_se2[k] += grad_wz * q.dyaw * q.tg[5][k];
        grad_a[0] += grad_ax * inv_cos_vphix * q.cyaw; grad_a[1] += grad_ax * inv_cos_vphix * q.syaw;
        grad_yaw += grad_ax * inv_cos_vphix * q.lat_acc;
#pragma unroll
        for (int k = 0; k < 3; k++) grad_se2[k] += grad_ax * (gravity * q.tg[1][k] + q.tg[0][k] * q.lon_acc);
        grad_a[0] += grad_ay * inv_cos_vphiy * (-q.syaw); grad_a[1] += grad_ay * inv_cos_vphiy * q.cyaw;
        grad_yaw -= grad_ay * inv_cos_vphiy * q.lon_acc;
#pragma unroll
        for (int k = 0; k < 3; k++) grad_se2[k] += grad_ay * (gravity * q.tg[3][k] + q.tg[2][k] * q.lat_acc);
        grad_p[0] += grad_se2[0]; grad_p[1] += grad_se2[1];
        grad_yaw += grad_se2[2];

        scr[(SF_GP + 0) * S + s] = grad_p[0]; scr[(SF_GP + 1) * S + s] = grad_p[1];
        scr[(SF_GV + 0) * S + s] = grad_v[0]; scr[(SF_GV + 1) * S + s] = grad_v[1];
        scr[(SF_GA + 0) * S + s] = grad_a[0]; scr[(SF_GA + 1) * S + s] = grad_a[1];
        scr[SF_GYAW * S + s] = grad_yaw; scr[SF_GDYAW * S + s] = grad_dyaw;
        scr[(SF_VEL + 0) * S + s] = q.vel[0]; scr[(SF_VEL + 1) * S + s] = q.vel[1];
        scr[SF_DYAW * S + s] = q.dyaw;
        for (j += GT; j >= K1; j -= K1) i++;
    }
}

// phase B: accumulate in the reference's order (alm_traj_opt.cpp:825-946 cost; :969-985 gradients).  Homogeneous rounds of
// 32 tasks: (piece, dim) coefficient-gradient blocks, per-piece time gradients, yaw blocks; then the cost chain.
__device__ UALM_NOINLINE void accumulate_tasks(Traj &t, int gtid, int GT)
{
    const int N = t.N, M = t.M, S = t.S, K = t.K, nx = 6 * N;
    const R *scr = t.scr;
    // gdCxy: one task per (piece, dim): 6 accumulators over the K+1 samples of the piece, in sample order; the next sample's
    // scratch values are fetched while the current one is accumulated
    for (int q = gtid; q < 2 * N; q += GT) {
        const int i = q >> 1, d = q & 1;
        R acc[6] = {0, 0, 0, 0, 0, 0};
        const R *pgp = scr + (size_t)(SF_GP + d) * S + i * (K + 1), *pgv = scr + (size_t)(SF_GV + d) * S + i * (K + 1),
                *pga = scr + (size_t)(SF_GA + d) * S + i * (K + 1);
        R gp = pgp[0], gv = pgv[0], ga = pga[0];
#pragma unroll 1
        for (int j = 0; j <= K; j++) {
            const int jn = j < K ? j + 1 : K;
            const R gpn = pgp[jn], gvn = pgv[jn], gan = pga[jn];
            const R s1 = t.s1tab[j];
            const R s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2, s5 = s4 * s1;
            acc[0] += (1.0 * gp + 0.0 * gv + 0.0 * ga);
            acc[1] += (s1 * gp + 1.0 * gv + 0.0 * ga);
            acc[2] += (s2 * gp + (2.0 * s1) * gv + 2.0 * ga);
            acc[3] += (s3 * gp + (3.0 * s2) * gv + (6.0 * s1) * ga);
            acc[4] += (s4 * gp + (4.0 * s3) * gv + (12.0 * s2) * ga);
            acc[5] += (s5 * gp + (5.0 * s4) * gv + (20.0 * s3) * ga);
            gp = gpn; gv = gvn; ga = gan;
        }
#pragma unroll
        for (int k = 0; k < 6; k++) t.gCxy[6 * i + k + d * nx] = acc[k];
    }
    // gdTxy(i): three += per sample (alm_traj_opt.cpp:827, 973-975, 984-985)
    for (int i = gtid; i < N; i += GT) {
        R acc = 0.0;
        R v[16], vn[16];
        auto fetch = [&](int s, R (&o)[16]) {
            o[0] = scr[SF_USER * S + s];
            o[1] = scr[(SF_GP + 0) * S + s]; o[2] = scr[(SF_GP + 1) * S + s];
            o[3] = scr[(SF_GV + 0) * S + s]; o[4] = scr[(SF_GV + 1) * S + s];
            o[5] = scr[(SF_GA + 0) * S + s]; o[6] = scr[(SF_GA + 1) * S + s];
            o[7] = scr[(SF_VEL + 0) * S + s]; o[8] = scr[(SF_VEL + 1) * S + s];
            o[9] = scr[(SF_ACC + 0) * S + s]; o[10] = scr[(SF_ACC + 1) * S + s];
            o[11] = scr[(SF_JER + 0) * S + s]; o[12] = scr[(SF_JER + 1) * S + s];
            o[13] = scr[SF_GYAW * S + s]; o[14] = scr[SF_GDYAW * S + s];
            o[15] = scr[SF_DYAW * S + s];
        };
        fetch(i * (K + 1), v);
        R d2y = scr[SF_D2YAW * S + i * (K + 1)];
#pragma unroll 1
        for (int j = 0; j <= K; j++) {
            const int sn = i * (K + 1) + (j < K ? j + 1 : K);
            fetch(sn, vn);
            const R d2yn = scr[SF_D2YAW * S + sn];
            const R alpha = 1.0 / (R)K * (R)j;
            acc += div_nz(v[0], (R)K);
            acc += ((v[1] * v[7] + v[2] * v[8]) + (v[3] * v[9] + v[4] * v[10]) + (v[5] * v[11] + v[6] * v[12])) * alpha;
            acc += (v[13] * v[15] + v[14] * d2y) * (alpha + (R)i);
#pragma unroll
            for (int q = 0; q < 16; q++) v[q] = vn[q];
            d2y = d2yn;
        }
        t.gTxy[i] = acc;
    }
    // gdCyaw block m and gdTyaw(m): the samples with yaw_idx == m in ascending sample order.  yaw_idx is monotone in the
    // sample index up to rounding at piece boundaries, so only a window around the block's time span is scanned.
    for (int m = gtid; m < M; m += GT) {
        R acc[6] = {0, 0, 0, 0, 0, 0};
        R accT = 0.0;
        const R ratio = (R)(K + 1) * (R)N / (R)M;   // samples per yaw piece
        int lo = (int)((R)m * ratio) - (K + 3), hi = (int)((R)(m + 1) * ratio) + (K + 3);
        if (lo < 0) lo = 0;
        if (hi > S || m == M - 1) hi = S;
        for (int s = lo; s < hi; s++) {
            if (t.yawidx[s] != m) continue;
            const R sy1 = scr[SF_S1YAW * S + s];
            const R sy2 = sy1 * sy1, sy3 = sy2 * sy1, sy4 = sy2 * sy2, sy5 = sy4 * sy1;
            const R gy = scr[SF_GYAW * S + s], gdy = scr[SF_GDYAW * S + s];
            const R gd2 = 0.0;
            acc[0] += (1.0 * gy + 0.0 * gdy + 0.0 * gd2);
            acc[1] += (sy1 * gy + 1.0 * gdy + 0.0 * gd2);
            acc[2] += (sy2 * gy + (2.0 * sy1) * gdy + 2.0 * gd2);
            acc[3] += (sy3 * gy + (3.0 * sy2) * gdy + (6.0 * sy1) * gd2);
            acc[4] += (sy4 * gy + (4.0 * sy3) * gdy + (12.0 * sy2) * gd2);
            acc[5] += (sy5 * gy + (5.0 * sy4) * gdy + (20.0 * sy3) * gd2);
            accT += -(gy * scr[SF_DYAW * S + s] + gdy * scr[SF_D2YAW * S + s]) * (R)m;
        }
#pragma unroll
        for (int k = 0; k < 6; k++) t.gCyaw[6 * m + k] = acc[k];
        t.gTyaw[m] = accT;
    }
}

// the cost chain of calConstrainCostGrad (alm_traj_opt.cpp:825-943) on the leader warp: 8 terms per sample in sample order.
// The terms are fetched 32 samples at a time by all lanes, one block ahead of the chain, and staged sample-major in the LU window
// (idle from the end of minco_generate to the adjoint sweeps).  Every lane then runs the chain on the same values, reading two
// terms per broadcast ld.shared.v2 one sample ahead of the adds.  Handing each term over by shuffle took two SHFL and two moves
// per add, and those instructions competed with the co-resident warps for issue slots.
__device__ UALM_NOINLINE void cost_chain(Traj &t, int lane)
{
    const int S = t.S;
    const R *scr = t.scr;
    const unsigned buf = t.win.a;        // 32 samples x 8 terms
    R cost = 0.0;
    R next[8];
#pragma unroll
    for (int k = 0; k < 8; k++) next[k] = (lane < S) ? scr[(SF_COST0 + k) * S + lane] : 0.0;
    for (int s0 = 0; s0 < S; s0 += 32) {
#pragma unroll
        for (int k = 0; k < 8; k += 2) sts2f64(buf + 64u * lane + 8u * k, next[k], next[k + 1]);
        __syncwarp();
        const int sn = s0 + 32 + lane;
#pragma unroll
        for (int k = 0; k < 8; k++) next[k] = (sn < S) ? scr[(SF_COST0 + k) * S + sn] : 0.0;
        const int cnt = min(32, S - s0);
        R cur[8];
#pragma unroll
        for (int k = 0; k < 8; k += 2) { const double2 v = lds2f64(buf + 8u * k); cur[k] = v.x; cur[k + 1] = v.y; }
#pragma unroll 1
        for (int l = 0; l < cnt; l++) {
            R v[8];
#pragma unroll
            for (int k = 0; k < 8; k++) v[k] = cur[k];
            const unsigned row = buf + 64u * (unsigned)min(l + 1, 31);
#pragma unroll
            for (int k = 0; k < 8; k += 2) { const double2 w = lds2f64(row + 8u * k); cur[k] = w.x; cur[k + 1] = w.y; }
#pragma unroll
            for (int k = 0; k < 8; k++) cost += v[k];
        }
        __syncwarp();                    // every lane has read the block before the next one overwrites it
    }
    if (lane == 0) t.sc[SC_CONSTR] = cost;
}

// gdT(i) += B1 . adj  (se2traj.hpp:763-814); adj = solved adjoint vector (element stride st), Dim columns
template <class AP>
__device__ UALM_NOINLINE R adj_time_term(SPtr c, int cst /*col stride of c*/, AP adj, int ast /*col stride*/, int st, int Dim,
                           int i, int P, R T1, R T2, R T3, R T4)
{
    R s = 0.0;
    if (i < P - 1) {
        for (int d = 0; d < Dim; d++) {
            const SPtr cc = c + (d * cst + 6 * i);
            const R nv = -(cc[1] + 2.0 * T1 * cc[2] + 3.0 * T2 * cc[3] + 4.0 * T3 * cc[4] + 5.0 * T4 * cc[5]);
            const R na = -(2.0 * cc[2] + 6.0 * T1 * cc[3] + 12.0 * T2 * cc[4] + 20.0 * T3 * cc[5]);
            const R nj = -(6.0 * cc[3] + 24.0 * T1 * cc[4] + 60.0 * T2 * cc[5]);
            const R ns = -(24.0 * cc[4] + 120.0 * T1 * cc[5]);
            const R nc = -120.0 * cc[5];
            const R B1[6] = {ns, nc, nv, nv, na, nj};
            for (int r = 0; r < 6; r++) s += B1[r] * at(adj, d * ast + (6 * i + 3 + r) * st);
        }
    } else {
        for (int d = 0; d < Dim; d++) {
            const SPtr cc = c + (d * cst + 6 * (P - 1));
            const R nv = -(cc[1] + 2.0 * T1 * cc[2] + 3.0 * T2 * cc[3] + 4.0 * T3 * cc[4] + 5.0 * T4 * cc[5]);
            const R na = -(2.0 * cc[2] + 6.0 * T1 * cc[3] + 12.0 * T2 * cc[4] + 20.0 * T3 * cc[5]);
            const R nj = -(6.0 * cc[3] + 24.0 * T1 * cc[4] + 60.0 * T2 * cc[5]);
            const R B2[3] = {nv, na, nj};
            for (int r = 0; r < 3; r++) s += B2[r] * at(adj, d * ast + (6 * P - 3 + r) * st);
        }
    }
    return s;
}

// ---------------------------------------------------------------------------------------------
// innerCallback (alm_traj_opt.cpp:280-347): x (smem t.x) -> f (sc[SC_F]) and g (smem t.g)
// ---------------------------------------------------------------------------------------------
__device__ UALM_NOINLINE void evaluate(Traj &t, const DevMap &map, const DevParams &p, int lane)
{
    const int N = t.N, M = t.M, nx = 6 * N, ny = 6 * M;
    t.n_evals++;
    prof_mark(t, lane, PF_OTHER);
    minco_generate(t, lane);
    jerk_cost(t, lane);
    prof_mark(t, lane, PF_JERK);
    sample_tables(t, lane);
    prof_mark(t, lane, PF_TABLES);
    maybe_regroup(t, lane);
    group_post(t, lane, CMD_SAMPLES);
    penalty_samples(t, map, p, lane, 32 * t.G);
    group_bar(t);
    prof_mark(t, lane, PF_SAMPLES);
    if (t.G > 1) {          // helpers sum the gradient entries while the leader runs the sequential cost chain
        group_post(t, lane, CMD_ACCUM);
        cost_chain(t, lane);
        group_bar(t);
    } else {
        accumulate_tasks(t, lane, 32);
        cost_chain(t, lane);
        UALM_SYNC();
    }
    prof_mark(t, lane, PF_ACCUM);
    // combine jerk and constraint gradients (alm_traj_opt.cpp:322-332); the jerk gradient is formed on the fly
    const R scale_fx = t.sc[SC_SCALE_FX];
    {
        const R T1 = t.sc[SC_TX1], T2 = t.sc[SC_TX2], T3 = t.sc[SC_TX3], T4 = t.sc[SC_TX4], T5 = t.sc[SC_TX5];
        for (int q = lane; q < 2 * nx; q += 32) {
            const int d = q >= nx, r = q - d * nx, i = r / 6, k = r - 6 * i;
            R gj = jerk_gc(t.cxy + d * nx + 6 * i, k, T1, T2, T3, T4, T5);
            if (p.use_scaling) gj *= UALM_SCALE_TRICK_JERK;
            t.gCxy[q] = gj * scale_fx + t.gCxy[q];
        }
        for (int i = lane; i < N; i += 32) {
            R e, gj;
            jerk_piece(t.cxy + 6 * i, t.cxy + (6 * i + nx), true, T1, T2, T3, T4, T5, e, gj);
            if (p.use_scaling) gj *= UALM_SCALE_TRICK_JERK;
            t.gTxy[i] = gj * scale_fx + t.gTxy[i];
        }
    }
    {
        const R T1 = t.sc[SC_TY1], T2 = t.sc[SC_TY2], T3 = t.sc[SC_TY3], T4 = t.sc[SC_TY4], T5 = t.sc[SC_TY5];
        for (int q = lane; q < ny; q += 32) {
            const int i = q / 6, k = q - 6 * i;
            R gj = jerk_gc(t.cyaw + 6 * i, k, T1, T2, T3, T4, T5);
            if (p.use_scaling) gj *= UALM_SCALE_TRICK_JERK;
            t.gCyaw[q] = gj * scale_fx + t.gCyaw[q];
        }
        for (int i = lane; i < M; i += 32) {
            R e, gj;
            jerk_piece(t.cyaw + 6 * i, t.cyaw, false, T1, T2, T3, T4, T5, e, gj);
            if (p.use_scaling) gj *= UALM_SCALE_TRICK_JERK;
            t.gTyaw[i] = gj * scale_fx + t.gTyaw[i];
        }
    }
    UALM_SYNC();
    prof_mark(t, lane, PF_COMBINE);
    // calGradCTtoQT (se2traj.hpp:751-816): adjoint solves in place in gCxy / gCyaw
    {
        const SPtr col = lane < 2 ? t.gCxy + lane * nx : t.gCyaw;
        sweep<2, 1, true, SPtr>(t.Fxy, N, t.Fyaw, M, t.ring, t.ring + UALM_RINGB * 6 * UALM_FW, col, col, 1, lane == 2, lane < 3, lane);
        sweep<3, 1, true, SPtr>(t.Fxy, N, t.Fyaw, M, t.ring, t.ring + UALM_RINGB * 6 * UALM_FW, col, col, 1, lane == 2, lane < 3, lane);
    }
    UALM_SYNC();
    prof_mark(t, lane, PF_ADJ);
    for (int q = lane; q < N + M; q += 32) {
        if (q < N) t.gTxy[q] += adj_time_term(t.cxy, nx, t.gCxy, nx, 1, 2, q, N, t.sc[SC_TX1], t.sc[SC_TX2], t.sc[SC_TX3], t.sc[SC_TX4]);
        else t.gTyaw[q - N] += adj_time_term(t.cyaw, ny, t.gCyaw, ny, 1, 1, q - N, M, t.sc[SC_TY1], t.sc[SC_TY2], t.sc[SC_TY3], t.sc[SC_TY4]);
    }
    for (int i = lane; i < N - 1; i += 32) {
        t.g[1 + 2 * i] = t.gCxy[6 * i + 5];
        t.g[1 + 2 * i + 1] = t.gCxy[6 * i + 5 + nx];
    }
    for (int i = lane; i < M - 1; i += 32) t.g[1 + 2 * (N - 1) + i] = t.gCyaw[6 * i + 5];
    UALM_SYNC();
    if (lane == 0) {
        const R tau = t.x[0];
        R jerk_c = t.sc[SC_JERKRAW] * scale_fx;
        if (p.use_scaling) jerk_c *= UALM_SCALE_TRICK_JERK;
        const R rho_T = t.sc[SC_RHO_T];
        const R tau_cost = rho_T * expC2(tau) * scale_fx;
        R sx = 0.0, sy = 0.0;
        for (int i = 0; i < N; i++) sx += t.gTxy[i];
        for (int i = 0; i < M; i++) sy += t.gTyaw[i];
        const R grad_Tsum = rho_T * scale_fx + sx / (R)N + sy / (R)M;
        t.g[0] = grad_Tsum * getTtoTauGrad(tau);
        t.sc[SC_JERK] = jerk_c; t.sc[SC_TAUCOST] = tau_cost;
        t.sc[SC_F] = jerk_c + t.sc[SC_CONSTR] + tau_cost;
    }
    UALM_SYNC();
    prof_mark(t, lane, PF_TAIL);
}

// ---------------------------------------------------------------------------------------------
// canonical 32-lane dot product; result on every lane
// ---------------------------------------------------------------------------------------------
template <class PA, class PB>
__device__ UALM_NOINLINE R lane_dot(PA a, PB b, int n, int lane)
{
    R pacc = 0.0;
    for (int i = lane; i < n; i += 32) pacc += at(a, i) * at(b, i);
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) pacc = pacc + __shfl_xor_sync(0xffffffffu, pacc, off);
    return pacc;
}
__device__ UALM_NOINLINE R lane_absmax(SPtr a, int n, int lane)
{
    R m = 0.0;
    for (int i = lane; i < n; i += 32) m = fmax(m, fabs(a[i]));
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, off));
    return m;
}

struct LbfgsOut { int ret; R f; int iters; int max_bound; int sum_bound; };

// stop = (max_evals > 0 && n_evals >= max_evals) || cancel requested, evaluated where earlyExit is (and by the ALM loop after
// judgeConvergence).  Lane 0 alone reads the problem's stop word (the slot's SC_PROB, set by slot_next); the broadcast keeps the
// decision warp-uniform.
__device__ __forceinline__ bool stop_requested(const Traj &t, const DevParams &p, int lane)
{
    int c = 0;
    if (p.cancel && lane == 0) c = p.cancel[(int)(R)t.sc[SC_PROB]];
    c = __shfl_sync(0xffffffffu, c, 0);
    return (p.max_evals > 0 && t.n_evals >= p.max_evals) || c != 0;
}

// lbfgs_optimize + line_search_lewisoverton (lbfgs.hpp:276-389, 439-722).  All 32 lanes follow the same control flow:
// every scalar the decisions depend on is the result of a warp-uniform reduction or a shared-memory scalar.
__device__ UALM_NOINLINE LbfgsOut lbfgs_optimize(Traj &t, const DevMap &map, const DevParams &p, int lane)
{
    const int n = t.n, m = p.mem_size;
    const R f_dec_coeff = 1.0e-4, s_curv_coeff = 0.9, cautious_factor = 1.0e-6, machine_prec = 1.0e-16;
    const R max_step = 1.0e+20, min_step = p.min_step;
    const int max_linesearch = 64;
    LbfgsOut out; out.ret = 0; out.iters = 0; out.max_bound = 0; out.sum_bound = 0;

    evaluate(t, map, p, lane);
    R fx = t.sc[SC_F];
    if (lane == 0) t.pf[0] = fx;
    for (int q = lane; q < n; q += 32) t.d[q] = -t.g[q];
    UALM_SYNC();
    {
        const R gn = lane_absmax(t.g, n, lane), xn = lane_absmax(t.x, n, lane);
        if (gn / fmax(1.0, xn) < p.g_epsilon) { out.ret = LBFGS_CONVERGENCE; out.f = fx; return out; }
    }
    R step = 1.0 / sqrt(lane_dot(t.d, t.d, n, lane));
    int k = 1, end = 0, bound = 0, ret = 0;
    while (true) {
        for (int q = lane; q < n; q += 32) { t.xp[q] = t.x[q]; t.gp[q] = t.g[q]; }
        UALM_SYNC();
        // ---- line search (lbfgs.hpp:276-389) ----
        int ls;
        {
            int count = 0;
            bool brackt = false, touched = false;
            R stp = step, mu = 0.0, nu = max_step;
            const R dginit = lane_dot(t.gp, t.d, n, lane);
            const R finit = fx;
            if (!(stp > 0.0)) ls = LBFGSERR_INVALIDPARAMETERS;
            else if (0.0 < dginit) ls = LBFGSERR_INCREASEGRADIENT;
            else {
                const R dgtest = f_dec_coeff * dginit, dstest = s_curv_coeff * dginit;
                while (true) {
                    for (int q = lane; q < n; q += 32) t.x[q] = t.xp[q] + stp * t.d[q];
                    UALM_SYNC();
                    evaluate(t, map, p, lane);
                    fx = t.sc[SC_F];
                    ++count;
                    if (isinf(fx) || isnan(fx)) { ls = LBFGSERR_INVALID_FUNCVAL; break; }
                    if (p.past > 0 && fabs(finit - fx) / (fabs(finit) + 1.0) < p.delta / (R)p.past) { ls = count; break; }
                    if (fx > finit + stp * dgtest) {
                        nu = stp;
                        brackt = true;
                    } else {
                        const R dg = lane_dot(t.g, t.d, n, lane);
                        if (dg < dstest) mu = stp;
                        else { ls = count; break; }
                    }
                    if (max_linesearch <= count) { ls = LBFGSERR_MAXIMUMLINESEARCH; break; }
                    if (brackt && (nu - mu) < machine_prec * nu) { ls = LBFGSERR_WIDTHTOOSMALL; break; }
                    if (brackt) stp = 0.5 * (mu + nu);
                    else stp *= 2.0;
                    if (stp < min_step) { ls = LBFGSERR_MINIMUMSTEP; break; }
                    if (stp > max_step) {
                        if (touched) { ls = LBFGSERR_MAXIMUMSTEP; break; }
                        touched = true;
                        stp = max_step;
                    }
                }
            }
            step = stp;
        }
        prof_mark(t, lane, PF_LS);
        if (ls < 0) {
            for (int q = lane; q < n; q += 32) { t.x[q] = t.xp[q]; t.g[q] = t.gp[q]; }
            UALM_SYNC();
            ret = ls;
            break;
        }
        out.iters++;
        {
            const bool stop = stop_requested(t, p, lane);
            if (stop && lane == 0) t.sc[SC_STOPPED] = 1.0;
            if (k > 1000 || stop) { ret = LBFGS_CANCELED; break; } // earlyExit alm_traj_opt.cpp:1016 (k > 1e3)
        }
        {
            const R gn = lane_absmax(t.g, n, lane), xn = lane_absmax(t.x, n, lane);
            if (gn / fmax(1.0, xn) < p.g_epsilon) { ret = LBFGS_CONVERGENCE; break; }
        }
        if (0 < p.past) {
            if (p.past <= k) {
                const R rate = fabs(t.pf[k % p.past] - fx) / fmax(1.0, fabs(fx));
                if (rate < p.delta) { ret = LBFGS_STOP; break; }
            }
            UALM_SYNC();
            if (lane == 0) t.pf[k % p.past] = fx;
            UALM_SYNC();
        }
        if (p.inner_max_iter != 0 && p.inner_max_iter <= k) { ret = LBFGSERR_MAXIMUMITERATION; break; }
        ++k;
        R *sE = t.lm_s + (size_t)end * n, *yE = t.lm_y + (size_t)end * n;
        for (int q = lane; q < n; q += 32) {
            sE[q] = t.x[q] - t.xp[q];
            yE[q] = t.g[q] - t.gp[q];
            t.d[q] = -t.g[q];
        }
        UALM_SYNC();
        const R ys = lane_dot(yE, sE, n, lane);
        const R yy = lane_dot(yE, yE, n, lane);
        const R ss = lane_dot(sE, sE, n, lane);
        const R gpn = lane_dot(t.gp, t.gp, n, lane);
        const R cau = ss * sqrt(gpn) * cautious_factor;
        if (lane == 0) {
            // ys divides one dot product per history step of every later two-loop: keep RN(1/ys) next to it so those quotients are
            // a * RN(1/b) + corrections (div_by_recip) instead of a full division on the dependent chain
            t.lm_ys[end] = ys;
            R r = 1.0 / ys;
            if ((__double_as_longlong(ys) & 0xFFFFFFFFFFFFFll) == 0xFFFFFFFFFFFFFll) r = __longlong_as_double(0x7ff8000000000000ll);
            t.lm_rys[end] = r;
        }
        UALM_SYNC();
        if (ys > cau) {
            ++bound;
            bound = m < bound ? m : bound;
            if (bound > out.max_bound) out.max_bound = bound;
            out.sum_bound += bound;
            end = (end + 1) % m;
            // two-loop recursion (lbfgs.hpp:691-710).  Each lane owns elements lane, lane+32, ... (<= 8 of them) of d in
            // registers; the history vectors of the NEXT step are loaded while the current step's dot product runs.
            R dreg[UALM_NREG], sc_[UALM_NREG], yc_[UALM_NREG], sn_[UALM_NREG], yn_[UALM_NREG];
#pragma unroll
            for (int e = 0; e < UALM_NREG; e++) { const int q = lane + 32 * e; dreg[e] = q < n ? t.d[q] : 0.0; sn_[e] = 0.0; yn_[e] = 0.0; }
            int j = (end + m - 1) % m;
            {
                const R *sj = t.lm_s + (size_t)j * n, *yj = t.lm_y + (size_t)j * n;
#pragma unroll
                for (int e = 0; e < UALM_NREG; e++) { const int q = lane + 32 * e; sc_[e] = q < n ? sj[q] : 0.0; yc_[e] = q < n ? yj[q] : 0.0; }
            }
            R ysj = t.lm_ys[j], rysj = t.lm_rys[j];
            for (int i = 0; i < bound; ++i) {
                const int jn = (j + m - 1) % m;
                R ysn = 0.0, rysn = 0.0;
                if (i + 1 < bound) {
                    const R *sj = t.lm_s + (size_t)jn * n, *yj = t.lm_y + (size_t)jn * n;
#pragma unroll
                    for (int e = 0; e < UALM_NREG; e++) { const int q = lane + 32 * e; if (q < n) { sn_[e] = sj[q]; yn_[e] = yj[q]; } }
                    ysn = t.lm_ys[jn]; rysn = t.lm_rys[jn];
                }
                R pacc = 0.0;
#pragma unroll
                for (int e = 0; e < UALM_NREG; e++) if (lane + 32 * e < n) pacc += sc_[e] * dreg[e];
#pragma unroll
                for (int off = 16; off >= 1; off >>= 1) pacc = pacc + __shfl_xor_sync(0xffffffffu, pacc, off);
                const R a = div_by_recip(pacc, ysj, rysj);
                if (lane == 0) t.lm_alpha[j] = a;
                const R na = -a;
#pragma unroll
                for (int e = 0; e < UALM_NREG; e++) dreg[e] = dreg[e] + na * yc_[e];
                if (i + 1 < bound) {
#pragma unroll
                    for (int e = 0; e < UALM_NREG; e++) { sc_[e] = sn_[e]; yc_[e] = yn_[e]; }
                    j = jn; ysj = ysn; rysj = rysn;
                }
            }
            const R scl = ys / yy;
#pragma unroll
            for (int e = 0; e < UALM_NREG; e++) dreg[e] = dreg[e] * scl;
            UALM_SYNC();
            // second loop walks oldest -> newest starting at the j where the first loop stopped (vectors still in sc_/yc_)
            R alj = t.lm_alpha[j];
            for (int i = 0; i < bound; ++i) {
                const int jn = (j + 1) % m;
                R ysn = 0.0, rysn = 0.0, aln = 0.0;
                if (i + 1 < bound) {
                    const R *sj = t.lm_s + (size_t)jn * n, *yj = t.lm_y + (size_t)jn * n;
#pragma unroll
                    for (int e = 0; e < UALM_NREG; e++) { const int q = lane + 32 * e; if (q < n) { sn_[e] = sj[q]; yn_[e] = yj[q]; } }
                    ysn = t.lm_ys[jn]; rysn = t.lm_rys[jn]; aln = t.lm_alpha[jn];
                }
                R pacc = 0.0;
#pragma unroll
                for (int e = 0; e < UALM_NREG; e++) if (lane + 32 * e < n) pacc += yc_[e] * dreg[e];
#pragma unroll
                for (int off = 16; off >= 1; off >>= 1) pacc = pacc + __shfl_xor_sync(0xffffffffu, pacc, off);
                const R beta = div_by_recip(pacc, ysj, rysj);
                const R cf = alj - beta;
#pragma unroll
                for (int e = 0; e < UALM_NREG; e++) dreg[e] = dreg[e] + cf * sc_[e];
                if (i + 1 < bound) {
#pragma unroll
                    for (int e = 0; e < UALM_NREG; e++) { sc_[e] = sn_[e]; yc_[e] = yn_[e]; }
                    j = jn; ysj = ysn; rysj = rysn; alj = aln;
                }
            }
#pragma unroll
            for (int e = 0; e < UALM_NREG; e++) { const int q = lane + 32 * e; if (q < n) t.d[q] = dreg[e]; }
        }
        UALM_SYNC();
        prof_mark(t, lane, PF_TWOLOOP);
        step = 1.0;
    }
    out.ret = ret;
    out.f = fx;
    return out;
}

// ---------------------------------------------------------------------------------------------
// initScaling (alm_traj_opt.cpp:349-661): one task per constraint (sample x 7), 32 tasks at a time, each lane running
// the reference's adjoint solves on its own interleaved workspace column while the whole warp streams the factors.
// ---------------------------------------------------------------------------------------------
// the per-constraint part of initScaling: GT threads of the warp group take GT constraint samples at a time
__device__ UALM_NOINLINE void scaling_rounds(Traj &t, const DevMap &map, const DevParams &p, int gtid, int GT, int lane)
{
    const int N = t.N, M = t.M, S = t.S, K = t.K, nx = 6 * N, ny = 6 * M;
    const R tau = t.x[0];
    const R dTdtau = getTtoTauGrad(tau);
    const R step = t.sc[SC_TX1] / (R)K;
    const R Tx1 = t.sc[SC_TX1], Tx2 = t.sc[SC_TX2], Tx3 = t.sc[SC_TX3], Tx4 = t.sc[SC_TX4], Tx5 = t.sc[SC_TX5];
    const R Ty1 = t.sc[SC_TY1], Ty2 = t.sc[SC_TY2], Ty3 = t.sc[SC_TY3], Ty4 = t.sc[SC_TY4], Ty5 = t.sc[SC_TY5];
    const int st = 32;
    R *wx = t.wsw + lane;                       // x column: rows 0..nx-1 at stride 32
    R *wy = t.wsw + (size_t)nx * st + lane;     // y column
    R *ww = t.wsw + (size_t)2 * nx * st + lane; // yaw
    R *scr = t.scr;
    const R rho_ter = t.sc[SC_RHO_TER];
    for (int s0 = 0; s0 < S; s0 += GT) {
        const int s = s0 + gtid;
        const bool act = s < S;
        SampleK q;
        int i = 0, j = 0;
        R alpha = 0.0;
        if (act) {
            i = s / (K + 1); j = s - i * (K + 1);
            alpha = 1.0 / (R)K * (R)j;
            sample_kin(t, map, p.gravity, i, t.s1tab[j], t.base[i], q);
            t.yawidx[s] = (unsigned short)q.yaw_idx;
            // user-defined cost -> f gradient pieces (alm_traj_opt.cpp:507-519), parked in the sample scratch
            const R omega = (j == 0 || j == K) ? 0.5 * rho_ter * step : rho_ter * step;
            const R sigma = q.tv[6];
            const R user_cost = omega * sigma * sigma;
            R gs[3];
            for (int k = 0; k < 3; k++) gs[k] = omega * q.tg[6][k] * sigma * 2.0;
            scr[SF_USER * S + s] = user_cost;
            scr[(SF_GP + 0) * S + s] = gs[0]; scr[(SF_GP + 1) * S + s] = gs[1];
            scr[SF_GYAW * S + s] = gs[2];
            scr[(SF_VEL + 0) * S + s] = q.vel[0]; scr[(SF_VEL + 1) * S + s] = q.vel[1];
            scr[SF_DYAW * S + s] = q.dyaw;
            scr[SF_S1YAW * S + s] = q.y0[1];
        }
        for (int ct = 0; ct < 7; ct++) {
            R dTx = 0.0, dTy = 0.0;
            if (act) {
                R grad_p[2] = {0, 0}, grad_v[2] = {0, 0}, grad_a[2] = {0, 0}, grad_se2[3];
                R grad_yaw = 0.0, grad_dyaw = 0.0;
                int usep = 0, usev = 0, usea = 0, usedy = 0;
                const R inv_cos_vphix = q.tv[0], inv_cos_vphiy = q.tv[2], inv_cos_xi = q.tv[5];
                if (ct == 0) { // non-holonomic (521-529)
                    grad_v[0] = q.syaw; grad_v[1] = -q.cyaw;
                    grad_yaw = q.vel[0] * q.cyaw + q.vel[1] * q.syaw;
                    usev = 1;
                } else if (ct == 1) { // longitude velocity (531-544)
                    const R grad_vx2 = 1.0;
                    for (int d = 0; d < 2; d++) grad_v[d] = grad_vx2 * inv_cos_vphix * inv_cos_vphix * 2.0 * q.vel[d];
                    for (int k = 0; k < 3; k++) grad_se2[k] = grad_vx2 * q.v_norm * q.v_norm * 2.0 * inv_cos_vphix * q.tg[0][k];
                    grad_p[0] = grad_se2[0]; grad_p[1] = grad_se2[1]; grad_yaw = grad_se2[2];
                    usep = 1; usev = 1;
                } else if (ct == 2) { // longitude acceleration (546-560)
                    const R grad_ax = 2.0 * q.ax;
                    grad_a[0] = grad_ax * inv_cos_vphix * q.cyaw; grad_a[1] = grad_ax * inv_cos_vphix * q.syaw;
                    grad_yaw = grad_ax * inv_cos_vphix * q.lat_acc;
                    for (int k = 0; k < 3; k++) grad_se2[k] = grad_ax * (p.gravity * q.tg[1][k] + q.tg[0][k] * q.lon_acc);
                    grad_p[0] = grad_se2[0]; grad_p[1] = grad_se2[1]; grad_yaw += grad_se2[2];
                    usep = 1; usea = 1;
                } else if (ct == 3) { // latitude acceleration (562-576)
                    const R grad_ay = 2.0 * q.ay;
                    grad_a[0] = grad_ay * inv_cos_vphiy * (-q.syaw); grad_a[1] = grad_ay * inv_cos_vphiy * q.cyaw;
                    grad_yaw = -grad_ay * inv_cos_vphiy * q.lon_acc;
                    for (int k = 0; k < 3; k++) grad_se2[k] = grad_ay * (p.gravity * q.tg[3][k] + q.tg[2][k] * q.lat_acc);
                    grad_p[0] = grad_se2[0]; grad_p[1] = grad_se2[1]; grad_yaw += grad_se2[2];
                    usep = 1; usea = 1;
                } else if (ct == 4) { // curvature (578-598)
                    const R denominator = 1.0 / (q.vx * q.vx + UALM_DELTA_SIGL);
                    const R grad_wz = denominator * 2.0 * q.wz;
                    const R grad_vx2 = -q.curv_snorm * denominator;
                    grad_dyaw = grad_wz * inv_cos_xi;
                    for (int k = 0; k < 3; k++) grad_se2[k] = grad_wz * q.dyaw * q.tg[5][k];
                    for (int d = 0; d < 2; d++) grad_v[d] = grad_vx2 * inv_cos_vphix * inv_cos_vphix * 2.0 * q.vel[d];
                    for (int k = 0; k < 3; k++) grad_se2[k] += grad_vx2 * q.v_norm * q.v_norm * 2.0 * inv_cos_vphix * q.tg[0][k];
                    grad_p[0] = grad_se2[0]; grad_p[1] = grad_se2[1]; grad_yaw = grad_se2[2];
                    usep = 1; usev = 1; usedy = 1;
                } else if (ct == 5) { // attitude (600-609)
                    for (int k = 0; k < 3; k++) grad_se2[k] = -q.tg[4][k];
                    grad_p[0] = grad_se2[0]; grad_p[1] = grad_se2[1]; grad_yaw = grad_se2[2];
                    usep = 1;
                } else { // surface variation (611-620)
                    for (int k = 0; k < 3; k++) grad_se2[k] = q.tg[6][k];
                    grad_p[0] = grad_se2[0]; grad_p[1] = grad_se2[1]; grad_yaw = grad_se2[2];
                    usep = 1;
                }
                // this constraint's gdC: only block i / block yaw_idx are non-zero
                for (int r = 0; r < nx; r++) { wx[(size_t)r * st] = 0.0; wy[(size_t)r * st] = 0.0; }
                for (int r = 0; r < ny; r++) ww[(size_t)r * st] = 0.0;
                for (int k = 0; k < 6; k++) {
                    R vx_, vy_;
                    if (usep && usev) { vx_ = (q.b0[k] * grad_p[0] + q.b1[k] * grad_v[0]); vy_ = (q.b0[k] * grad_p[1] + q.b1[k] * grad_v[1]); }
                    else if (usep && usea) { vx_ = (q.b0[k] * grad_p[0] + q.b2[k] * grad_a[0]); vy_ = (q.b0[k] * grad_p[1] + q.b2[k] * grad_a[1]); }
                    else if (usep) { vx_ = (q.b0[k] * grad_p[0]); vy_ = (q.b0[k] * grad_p[1]); }
                    else { vx_ = q.b1[k] * grad_v[0]; vy_ = q.b1[k] * grad_v[1]; }
                    wx[(size_t)(6 * i + k) * st] = 0.0 + vx_;
                    wy[(size_t)(6 * i + k) * st] = 0.0 + vy_;
                    R vw;
                    if (usedy) vw = (q.y0[k] * grad_yaw + q.y1[k] * grad_dyaw);
                    else vw = q.y0[k] * grad_yaw;
                    ww[(size_t)(6 * q.yaw_idx + k) * st] = 0.0 + vw;
                }
                // direct time-gradient terms of this constraint
                if (usep && usev) dTx += ((grad_p[0] * q.vel[0] + grad_p[1] * q.vel[1]) + (grad_v[0] * q.acc[0] + grad_v[1] * q.acc[1])) * alpha;
                else if (usep && usea) dTx += ((grad_p[0] * q.vel[0] + grad_p[1] * q.vel[1]) + (grad_a[0] * q.jer[0] + grad_a[1] * q.jer[1])) * alpha;
                else if (usep) dTx += (grad_p[0] * q.vel[0] + grad_p[1] * q.vel[1]) * alpha;
                else dTx += (grad_v[0] * q.acc[0] + grad_v[1] * q.acc[1]) * alpha;
                if (usedy) {
                    dTy += -(grad_yaw * q.dyaw + grad_dyaw * q.d2yaw) * (R)q.yaw_idx;
                    dTx += (grad_yaw * q.dyaw + grad_dyaw * q.d2yaw) * (alpha + (R)i);
                } else {
                    dTy += -(grad_yaw * q.dyaw) * (R)q.yaw_idx;
                    dTx += (grad_yaw * q.dyaw) * (alpha + (R)i);
                }
            }
            UALM_SYNC();
            // adjoint solves (calGradCTtoQT, se2traj.hpp:751-816), all lanes in lockstep; the forward sweeps start at the first
            // block any lane has a non-zero right-hand side in
            int bx0 = act ? i : N - 1, by0 = act ? q.yaw_idx : M - 1;
#pragma unroll
            for (int off = 16; off >= 1; off >>= 1) {
                bx0 = min(bx0, __shfl_xor_sync(0xffffffffu, bx0, off));
                by0 = min(by0, __shfl_xor_sync(0xffffffffu, by0, off));
            }
            sweep<2, 2, false, R *>(t.Fxy, N, nullptr, 0, t.hring, t.hring, wx, wy, st, 0, act, lane, bx0);
            sweep<3, 2, false, R *>(t.Fxy, N, nullptr, 0, t.hring, t.hring, wx, wy, st, 0, act, lane);
            sweep<2, 1, false, R *>(t.Fyaw, M, nullptr, 0, t.hring, t.hring, ww, ww, st, 0, act, lane, by0);
            sweep<3, 1, false, R *>(t.Fyaw, M, nullptr, 0, t.hring, t.hring, ww, ww, st, 0, act, lane);
            if (act) {
                R m1 = 0.0, m2 = 0.0;
                for (int r = 0; r < N - 1; r++) {
                    m1 = fmax(m1, fabs(wx[(size_t)(6 * r + 5) * st]));
                    m1 = fmax(m1, fabs(wy[(size_t)(6 * r + 5) * st]));
                }
                for (int r = 0; r < M - 1; r++) m2 = fmax(m2, fabs(ww[(size_t)(6 * r + 5) * st]));
                R sx = 0.0, sy = 0.0;
                for (int r = 0; r < N; r++) {
                    R gT = (r == i) ? dTx : 0.0;
                    gT += adj_time_term(t.cxy, nx, t.wsw + lane, nx * st, st, 2, r, N, Tx1, Tx2, Tx3, Tx4);
                    sx += gT;
                }
                for (int r = 0; r < M; r++) {
                    R gT = (r == q.yaw_idx) ? dTy : 0.0;
                    gT += adj_time_term(t.cyaw, ny, ww, 0, st, 1, r, M, Ty1, Ty2, Ty3, Ty4);
                    sy += gT;
                }
                const R gdTau = (sx / (R)N + sy / (R)M) * dTdtau;
                t.scale_cx[7 * (size_t)s + ct] = 1.0 / fmax(1.0, fmax(fmax(m1, m2), fabs(gdTau)));
            }
        }
    }
    }

__device__ UALM_NOINLINE void init_scaling(Traj &t, const DevMap &map, const DevParams &p, int lane)
{
    const int N = t.N, M = t.M, S = t.S, K = t.K, nx = 6 * N, ny = 6 * M;
    minco_generate(t, lane);
    sample_tables(t, lane);
    const R tau = t.x[0];
    const R dTdtau = getTtoTauGrad(tau);
    const R step = t.sc[SC_TX1] / (R)K;
    const R Tx1 = t.sc[SC_TX1], Tx2 = t.sc[SC_TX2], Tx3 = t.sc[SC_TX3], Tx4 = t.sc[SC_TX4], Tx5 = t.sc[SC_TX5];
    const R Ty1 = t.sc[SC_TY1], Ty2 = t.sc[SC_TY2], Ty3 = t.sc[SC_TY3], Ty4 = t.sc[SC_TY4], Ty5 = t.sc[SC_TY5];
    R *scr = t.scr;
    group_post(t, lane, CMD_SCALE);
    scaling_rounds(t, map, p, lane, 32 * t.G, lane);
    group_bar(t);
    // ---- f gradient: jerk gradient (formed on the fly) + user cost (alm_traj_opt.cpp:507-519), then adjoint ----
    for (int qq = lane; qq < 2 * N; qq += 32) {
        const int i = qq >> 1, d = qq & 1;
        R acc[6];
        for (int k = 0; k < 6; k++) acc[k] = jerk_gc(t.cxy + d * nx + 6 * i, k, Tx1, Tx2, Tx3, Tx4, Tx5);
        for (int j = 0; j <= K; j++) {
            const int s = i * (K + 1) + j;
            const R s1 = t.s1tab[j];
            const R s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2, s5 = s4 * s1;
            const R gp = scr[(SF_GP + d) * S + s];
            acc[0] += 1.0 * gp; acc[1] += s1 * gp; acc[2] += s2 * gp; acc[3] += s3 * gp; acc[4] += s4 * gp; acc[5] += s5 * gp;
        }
        for (int k = 0; k < 6; k++) t.gCxy[6 * i + k + d * nx] = acc[k];
    }
    for (int i = lane; i < N; i += 32) {
        R e, acc;
        jerk_piece(t.cxy + 6 * i, t.cxy + (6 * i + nx), true, Tx1, Tx2, Tx3, Tx4, Tx5, e, acc);
        for (int j = 0; j <= K; j++) {
            const int s = i * (K + 1) + j;
            const R alpha = 1.0 / (R)K * (R)j;
            acc += div_nz(scr[SF_USER * S + s], (R)K);
            acc += (scr[(SF_GP + 0) * S + s] * scr[(SF_VEL + 0) * S + s] + scr[(SF_GP + 1) * S + s] * scr[(SF_VEL + 1) * S + s]) * alpha;
            acc += (scr[SF_GYAW * S + s] * scr[SF_DYAW * S + s]) * (alpha + (R)i);
        }
        t.gTxy[i] = acc;
    }
    for (int m = lane; m < M; m += 32) {
        R acc[6], e, accT;
        for (int k = 0; k < 6; k++) acc[k] = jerk_gc(t.cyaw + 6 * m, k, Ty1, Ty2, Ty3, Ty4, Ty5);
        jerk_piece(t.cyaw + 6 * m, t.cyaw, false, Ty1, Ty2, Ty3, Ty4, Ty5, e, accT);
        const R ratio = (R)(K + 1) * (R)N / (R)M;
        int lo = (int)((R)m * ratio) - (K + 3), hi = (int)((R)(m + 1) * ratio) + (K + 3);
        if (lo < 0) lo = 0;
        if (hi > S || m == M - 1) hi = S;
        for (int s = lo; s < hi; s++) {
            if (t.yawidx[s] != m) continue;
            const R sy1 = scr[SF_S1YAW * S + s];
            const R sy2 = sy1 * sy1, sy3 = sy2 * sy1, sy4 = sy2 * sy2, sy5 = sy4 * sy1;
            const R gy = scr[SF_GYAW * S + s];
            acc[0] += (1.0 * gy); acc[1] += (sy1 * gy); acc[2] += (sy2 * gy); acc[3] += (sy3 * gy); acc[4] += (sy4 * gy); acc[5] += (sy5 * gy);
            accT += -(gy * scr[SF_DYAW * S + s]) * (R)m;
        }
        for (int k = 0; k < 6; k++) t.gCyaw[6 * m + k] = acc[k];
        t.gTyaw[m] = accT;
    }
    UALM_SYNC();
    {
        const SPtr col = lane < 2 ? t.gCxy + lane * nx : t.gCyaw;
        sweep<2, 1, true, SPtr>(t.Fxy, N, t.Fyaw, M, t.ring, t.ring + UALM_RINGB * 6 * UALM_FW, col, col, 1, lane == 2, lane < 3, lane);
        sweep<3, 1, true, SPtr>(t.Fxy, N, t.Fyaw, M, t.ring, t.ring + UALM_RINGB * 6 * UALM_FW, col, col, 1, lane == 2, lane < 3, lane);
    }
    UALM_SYNC();
    for (int q = lane; q < N + M; q += 32) {
        if (q < N) t.gTxy[q] += adj_time_term(t.cxy, nx, t.gCxy, nx, 1, 2, q, N, Tx1, Tx2, Tx3, Tx4);
        else t.gTyaw[q - N] += adj_time_term(t.cyaw, ny, t.gCyaw, ny, 1, 1, q - N, M, Ty1, Ty2, Ty3, Ty4);
    }
    UALM_SYNC();
    if (lane == 0) {
        R sx = 0.0, sy = 0.0, m1 = 0.0, m2 = 0.0;
        for (int i = 0; i < N; i++) sx += t.gTxy[i];
        for (int i = 0; i < M; i++) sy += t.gTyaw[i];
        const R grad_Tsum_fx = t.sc[SC_RHO_T] + sx / (R)N + sy / (R)M;
        const R gdTau_fx = grad_Tsum_fx * dTdtau;
        for (int i = 0; i < N - 1; i++) { m1 = fmax(m1, fabs(t.gCxy[6 * i + 5])); m1 = fmax(m1, fabs(t.gCxy[6 * i + 5 + nx])); }
        for (int i = 0; i < M - 1; i++) m2 = fmax(m2, fabs(t.gCyaw[6 * i + 5]));
        t.sc[SC_SCALE_FX] = 1.0 / fmax(1.0, fmax(fmax(m1, m2), fabs(gdTau_fx)));
    }
    UALM_SYNC();
}

// ---------------------------------------------------------------------------------------------
// set up the Traj view of one problem
// ---------------------------------------------------------------------------------------------
__device__ UALM_NOINLINE void traj_setup(Traj &t, const BatchPtrs &bp, const DevParams &p, const SmemLayout &L, unsigned sm, unsigned sm_own, int prob, int G, int wig, int leader)
{
    const ProbDesc *pd = bp.desc + prob;
    t.pd = pd; t.N = pd->N; t.M = pd->M; t.n = pd->n; t.S = pd->S; t.K = p.int_K;
    auto S8 = [&](int o) { return SPtr{sm + 8u * (unsigned)o}; };
    t.cxy = S8(L.cxy); t.cyaw = S8(L.cyaw); t.gCxy = S8(L.gCxy); t.gCyaw = S8(L.gCyaw); t.gTxy = S8(L.gTxy); t.gTyaw = S8(L.gTyaw);
    t.x = S8(L.x); t.g = S8(L.g); t.xp = S8(L.xp); t.gp = S8(L.gp); t.d = S8(L.d); t.pf = S8(L.pf); t.s1tab = S8(L.s1tab);
    t.base = S8(L.base); t.sc = S8(L.sc); t.win = S8(L.win); t.tmpl = S8(L.tmpl); t.ring = S8(L.ring);
    t.yawidx = SPtrU16{sm + 8u * (unsigned)L.yawidx};
    t.lutab = sm + 8u * (unsigned)L.lutab;     // filled once per leader slot (lu_build_consts): it does not depend on the problem
    t.lambda = bp.lambda + pd->off_s; t.hx = bp.hx + pd->off_s;
    t.mu = bp.mu + 6 * pd->off_s; t.gx = bp.gx + 6 * pd->off_s;
    t.scale_cx = bp.scale_cx + 7 * pd->off_s;
    t.lm_s = bp.lm_s + pd->off_hist; t.lm_y = bp.lm_y + pd->off_hist;
    t.lm_alpha = bp.lm_aux + pd->off_aux; t.lm_ys = t.lm_alpha + p.mem_size; t.lm_rys = t.lm_ys + p.mem_size;
    t.scr = bp.scratch + pd->off_scr;
    {
        const long long rx = 6 * pd->N + 2 * UALM_FPAD, ry = 6 * pd->M + 2 * UALM_FPAD;
        R *f = bp.fac + pd->off_fac;
        t.Fxy = f + UALM_FPAD * UALM_FW;
        t.Fyaw = f + rx * UALM_FW + UALM_FPAD * UALM_FW;
        (void)ry;
    }
    t.ws = bp.ws_scaling ? bp.ws_scaling + pd->off_ws : nullptr;
    t.G = G; t.wig = wig; t.barid = 1 + leader; t.adopt = nullptr;
    t.hring = SPtr{sm_own + 8u * (unsigned)L.ring};
    t.wsw = t.ws ? t.ws + (size_t)wig * (12 * pd->N + 6 * pd->M) * 32 : nullptr;
    t.n_evals = 0;
    __shared__ long long s_prof_all[UALM_WPB][UALM_NPROF + 1];
    long long *s_prof = s_prof_all[threadIdx.x >> 5];
    const int ln = threadIdx.x & 31;
    if (wig == 0 && ln < 8) t.sc[SC_PP + ln] = pd->pp[ln];   // the leader; its helpers read them after its next post
    if (ln < UALM_NPROF + 1) s_prof[ln] = 0;
    t.prof = s_prof; t.plast = s_prof + UALM_NPROF;
    UALM_SYNC();
    if (ln == 0) { *t.plast = clock64(); s_prof[PF_TOTAL] = -clock64(); }
}

// exit of the ALM loop after judgeConvergence (include/ualm.h, UALM_RET_STOPPED): a stop that fired inside the inner solve that
// just ended, else convergence, else a stop that holds now; -1 = go on (to the max_iter test).  Not inlined: inside solve_kernel
// (255 registers) the test costs a spill
__device__ UALM_NOINLINE int alm_exit(Traj &t, const DevParams &p, int lane, bool converged)
{
    if ((R)t.sc[SC_STOPPED] != 0.0) return UALM_RET_STOPPED;
    if (converged) return 0;
    if (stop_requested(t, p, lane)) return UALM_RET_STOPPED;
    return -1;
}

// =============================================================================================
// kernels (CTA = 4 warp slots; solve_kernel: warp groups per trajectory, the test kernels: one warp per trajectory)
// =============================================================================================

// helper warps of a group: execute the parallel phases the leader posts, nothing else.  Returns the group's next problem
// (CMD_NEXT), -1 (CMD_EXIT) or -2 (CMD_JOIN: the warps join the mate's trajectory)
__device__ UALM_NOINLINE int helper_loop(Traj &t, const DevMap &map, const DevParams &p, int lane)
{
    while (true) {
        group_bar(t);
        const int cmd = (int)(R)t.sc[SC_CMD];
        if (cmd == CMD_EXIT) return -1;
        if (cmd == CMD_JOIN) return -2;
        if (cmd == CMD_REGROUP) { group_bar(t); t.G = 4; t.barid = UALM_BAR_BIG; continue; }
        if (cmd == CMD_NEXT) {
            const int prob = (int)(R)t.sc[SC_PROB];
            group_bar(t);                       // the leader may overwrite the command word after this barrier
            return prob;
        }
        if (cmd == CMD_SAMPLES) penalty_samples(t, map, p, 32 * t.wig + lane, 32 * t.G);
        else if (cmd == CMD_ACCUM) accumulate_tasks(t, 32 * (t.wig - 1) + lane, 32 * (t.G - 1));
        else if (cmd == CMD_SCALE) scaling_rounds(t, map, p, 32 * t.wig + lane, 32 * t.G, lane);
        group_bar(t);
    }
}

// warps of a two-warp group that found the queue empty: serve the mate slot's trajectory `prob` as helpers 2 and 3 until it ends
__device__ UALM_NOINLINE void join_mate(Traj &t, const BatchPtrs &bp, const DevParams &p, const DevMap &map, const SmemLayout &L, unsigned sbase, int mate,
                                        int prob, int wig, int lane)
{
    const unsigned smm = sbase + 8u * (unsigned)(mate * L.total_doubles);
    traj_setup(t, bp, p, L, smm, smm, prob, 4, wig, mate);
    t.barid = UALM_BAR_BIG;
    helper_loop(t, map, p, lane);
}

// leader of a slot between two problems: take the next problem of the launch's queue (largest first) and hand it to the helpers.
// Returns the problem; -1 when the slot is done; -2 when the queue is empty and the group's warps join the mate's trajectory
// (`adopt` = the CTA's two adoption state words, null without adoption; `probs` = the problems the slots published).  A slot
// that has been joined takes no further problem.  A slot of a non-urgent launch under a hold (hold_raised) takes nothing and ends
// as at the end of the queue; the problems it leaves are taken by the next pass of the launch's loop (ualm_api.cu: solve_loop_run)
__device__ UALM_NOINLINE int slot_next(Traj &t, const BatchPtrs &bp, int *adopt, int *probs, int slot, int lane)
{
    bool joined = false;
    if (t.adopt) {                              // end of the slot's last problem
        int old = 0;
        if (lane == 0) old = atomicExch(t.adopt, AD_DONE);
        old = __shfl_sync(0xffffffffu, old, 0);
        if (old == AD_JOINREQ) regroup_now(t, lane);     // the mate's warps already wait on the CTA-wide barrier: release them below
        joined = t.G == 4;
    }
    int next = -1;
    if (!joined) {
        if (lane == 0) {
            const bool held = bp.urgent_slot < 0 && bp.hold && hold_raised(bp.hold) && !((volatile int *)bp.hctl)[1];
            if (!held) {
                const int q = atomicAdd(bp.queue, 1);
                next = q < bp.n_active ? bp.order[q] : -1;
                if (next >= 0 && bp.urgent_slot >= 0 && atomicAdd(bp.hctl, 1) == bp.n_urgent - 1)
                    ((volatile unsigned char *)bp.hold)[bp.urgent_slot] = 0;     // the urgent ticket's last problem is taken
            }
        }
        next = __shfl_sync(0xffffffffu, next, 0);
    }
    if (next >= 0) {
        if (lane == 0) t.sc[SC_PROB] = (R)next;
        group_post(t, lane, CMD_NEXT);
        group_bar(t);                           // the helpers have read the problem
        if (adopt && lane == 0) {               // publish it: from here on the mate may ask to join
            probs[slot] = next;
            __threadfence_block();
            atomicExch(&adopt[slot], AD_RUNNING);
        }
        return next;
    }
    int join = 0;
    if (adopt && !joined && lane == 0) {        // offer this group's warps to the mate's trajectory, if it has one running
        join = atomicCAS(&adopt[1 - slot], AD_RUNNING, AD_JOINREQ) == AD_RUNNING;
        __threadfence_block();                  // probs[1 - slot] is read after this (the mate published it before RUNNING)
    }
    join = __shfl_sync(0xffffffffu, join, 0);
    group_post(t, lane, join ? CMD_JOIN : CMD_EXIT);
    return join ? -2 : -1;
}

// ualm_poll_batch: copy the coefficients and the record of problem `prob`, which this warp has just written to the lane's outputs,
// into the lane's mailbox and raise the problem's flag (ualm_mailbox.h).  Each lane copies the coefficient entries it wrote itself;
// the record was written by lane 0 before the warp barrier that precedes the call.  Nothing without a mailbox (every launch not
// made by ualm_submit_batch*).  Not inlined, like alm_exit, and the test is in here: with it at the call site solve_kernel spilled
// 4 bytes more
__device__ UALM_NOINLINE void publish_problem(const BatchPtrs &bp, int prob, int lane)
{
    if (!bp.mbox.flag) return;
    const ProbDesc *pd = bp.desc + prob;
    const ualm_mbox::Ptrs &mb = bp.mbox;
    const long long ox = pd->off_cxy, oy = pd->off_cyaw;
    const int nxy = 12 * pd->N, nyaw = 6 * pd->M;
    for (int q = lane; q < nxy; q += 32) mb.c_xy[ox + q] = bp.c_xy[ox + q];
    for (int q = lane; q < nyaw; q += 32) mb.c_yaw[oy + q] = bp.c_yaw[oy + q];
    static_assert(sizeof(ualm_result_t) % 8 == 0 && sizeof(ualm_result_t) / 8 <= 32, "the record is copied as one 8-byte word per lane");
    if (lane < (int)(sizeof(ualm_result_t) / 8))
        ((long long *)(mb.res + prob))[lane] = ((const long long *)(bp.results + prob))[lane];
    ualm_mbox::raise_flag_warp(mb, prob, lane);
}

// one problem on a leader slot, from its setup to its result record (`adopt` = the slot's adoption state word, or null).  Not
// inlined: the loop over the queue around it would otherwise add spill to the solve
__device__ UALM_NOINLINE void solve_problem(Traj &t, const BatchPtrs &bp, const DevParams &p, const DevMap &map, const SmemLayout &L, unsigned sm, int slot,
                                            int *adopt, int prob, int lane)
{
    traj_setup(t, bp, p, L, sm, sm, prob, 4 / bp.n_leader_slots, 0, slot);
    const int N = t.N, M = t.M, n = t.n, S = t.S;
    // duals and scales (alm_traj_opt.cpp:193-203)
    for (int q = lane; q < S; q += 32) { t.lambda[q] = 0.0; t.hx[q] = 0.0; }
    for (int q = lane; q < 6 * S; q += 32) { t.mu[q] = 0.0; t.gx[q] = 0.0; }
    for (int q = lane; q < 7 * S; q += 32) t.scale_cx[q] = 1.0;
    for (int q = lane; q < n; q += 32) t.x[q] = bp.x0[t.pd->off_x + q];
    if (lane == 0) { t.sc[SC_SCALE_FX] = 1.0; t.sc[SC_RHO] = p.rho; t.sc[SC_STOPPED] = 0.0; }
    UALM_SYNC();
    if (p.use_scaling) init_scaling(t, map, p, lane);
    prof_mark(t, lane, PF_SCALING);
    t.adopt = adopt;                      // joiners only take part in the evaluation phases

    int ret_code = 0, iter = 0, last = 0, iters_total = 0, max_bound = 0, sum_bound = 0;
    R inner_cost = 0.0, rh = 0.0, rg = 0.0;
    while (true) {
        LbfgsOut lo = lbfgs_optimize(t, map, p, lane);
        inner_cost = lo.f; last = lo.ret; iters_total += lo.iters;
        if (lo.max_bound > max_bound) max_bound = lo.max_bound;
        sum_bound += lo.sum_bound;
        UALM_SYNC();
        if (lo.ret == LBFGS_CONVERGENCE || lo.ret == LBFGS_CANCELED || lo.ret == LBFGS_STOP || lo.ret == LBFGSERR_MAXIMUMITERATION) {
        } else if (lo.ret == LBFGSERR_MAXIMUMLINESEARCH) {
        } else { ret_code = 1; break; }
        // updateDualVars (alm_traj_opt.h:132-138) with hx/gx of the LAST evaluation (Q1), judgeConvergence (:140-151)
        const R rho = t.sc[SC_RHO];
        const R rho_new = fmin((1 + p.gamma) * rho, p.beta);
        R mh = 0.0, mg = 0.0;
        for (int q = lane; q < S; q += 32) {
            const R h = t.hx[q];
            t.lambda[q] += rho * h;
            mh = fmax(mh, fabs(h));
        }
        for (int q = lane; q < 6 * S; q += 32) {
            const R gq = t.gx[q];
            const R mq = fmax(t.mu[q] + rho * gq, 0.0);
            t.mu[q] = mq;
            mg = fmax(mg, fabs(fmax(gq, div_nz(-mq, rho_new))));
        }
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
            mh = fmax(mh, __shfl_xor_sync(0xffffffffu, mh, off));
            mg = fmax(mg, __shfl_xor_sync(0xffffffffu, mg, off));
        }
        rh = mh; rg = mg;
        UALM_SYNC();
        if (lane == 0) t.sc[SC_RHO] = rho_new;
        UALM_SYNC();
        prof_mark(t, lane, PF_DUAL);
        {
            const int e = alm_exit(t, p, lane, fmax(rh, rg) < p.epsilon_con);
            if (e >= 0) { ret_code = e; break; }
        }
        if ((R)(++iter) > p.max_iter) { ret_code = 2; break; }
    }
    // outputs: coefficients / decision vector of the LAST evaluation's MINCO state (Q1), result record
    const int nx = 6 * N, ny = 6 * M;
    for (int q = lane; q < 2 * nx; q += 32) bp.c_xy[t.pd->off_cxy + q] = t.cxy[q];
    for (int q = lane; q < ny; q += 32) bp.c_yaw[t.pd->off_cyaw + q] = t.cyaw[q];
    for (int q = lane; q < n; q += 32) bp.x[t.pd->off_x + q] = t.x[q];
    if (lane == 0) {
        ualm_result_t r;
        r.ret_code = ret_code; r.outer_iters = iter; r.n_evals = t.n_evals; r.n_lbfgs_iters = iters_total; r.last_lbfgs_ret = last;
        r.max_bound = max_bound; r.sum_bound = sum_bound; r.reserved = 0; r.inner_cost = inner_cost; r.jerk_cost = t.sc[SC_JERKRAW];
        R tt = 0.0;
        for (int i = 0; i < N; i++) tt += t.sc[SC_TX1];
        r.total_T = tt; r.res_h = rh; r.res_g = rg; r.scale_fx = t.sc[SC_SCALE_FX]; r.rho_final = t.sc[SC_RHO];
        r.piece_T_xy = t.sc[SC_TX1]; r.piece_T_yaw = t.sc[SC_TY1];
        bp.results[prob] = r;
        bp.piece_T[2 * prob] = t.sc[SC_TX1]; bp.piece_T[2 * prob + 1] = t.sc[SC_TY1];
        if (bp.prof) {
            t.prof[PF_TOTAL] += clock64();
            for (int q = 0; q < UALM_NPROF; q++) bp.prof[(size_t)prob * UALM_NPROF + q] = t.prof[q];
        }
    }
    UALM_SYNC();
    publish_problem(bp, prob, lane);
}

// full solve: optimizeSE2Traj (alm_traj_opt.cpp:168-278).  Each leader slot of a CTA solves problems from the launch's queue until
// it is empty, so a slot whose trajectory ends early takes the next one instead of idling until its CTA's slowest trajectory ends.
// Every buffer a problem reads or writes is its own (ProbDesc offsets) and the slot's shared memory is set up again per problem,
// so which slot solves which problem, and when, changes no result bit.
__global__ void __launch_bounds__(UALM_THREADS * UALM_WPB) solve_kernel(const __grid_constant__ BatchPtrs bp, const __grid_constant__ DevParams p, const __grid_constant__ DevMap map,
        const __grid_constant__ SmemLayout L)
{
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int G = UALM_WPB / bp.n_leader_slots, slot = w / G, wig = w - slot * G;   // group size, leader slot, warp in group
    __shared__ int s_adopt[2], s_prob[2];
    const bool adoptable = (bp.n_leader_slots == 2 && bp.adopt);
    if (adoptable) {
        if (threadIdx.x < 2) s_adopt[threadIdx.x] = AD_DONE;
        __syncthreads();
    }
    const unsigned sbase = (unsigned)__cvta_generic_to_shared(ualm_smem);
    const unsigned sm = sbase + 8u * (unsigned)(slot * L.total_doubles);
    Traj t;
    t.G = G; t.barid = 1 + slot; t.sc = SPtr{sm + 8u * (unsigned)L.sc}; t.adopt = nullptr;   // the group before its first problem
    if (wig > 0) {
        // a helper's own shared memory is just a factor ring behind the leader slots (ring wig - 1 in a four-warp group, the slot's
        // in a two-warp group); traj_setup adds L.ring to sm_own
        const int hring = G == 4 ? wig - 1 : slot;
        const unsigned sm_own = sbase + 8u * (unsigned)(bp.n_leader_slots * L.total_doubles + hring * (2 * UALM_RINGB * 6 * UALM_FW)) - 8u * (unsigned)L.ring;
        int prob;
        while ((prob = helper_loop(t, map, p, lane)) >= 0) traj_setup(t, bp, p, L, sm, sm_own, prob, G, wig, slot);
        if (prob == -2) join_mate(t, bp, p, map, L, sbase, 1 - slot, ((volatile int *)s_prob)[1 - slot], 3, lane);
        return;
    }
    lu_build_consts(sm + 8u * (unsigned)L.lutab, lane);
    int *const adopt = adoptable ? s_adopt : nullptr;
    int prob;
    while ((prob = slot_next(t, bp, adopt, s_prob, slot, lane)) >= 0) solve_problem(t, bp, p, map, L, sm, slot, adopt ? adopt + slot : nullptr, prob, lane);
    if (prob == -2) join_mate(t, bp, p, map, L, sbase, 1 - slot, ((volatile int *)s_prob)[1 - slot], 2, lane);
}

// the two ends of a pass of a solve launch's loop (ualm_api.cu: solve_loop_run).  The gate holds a non-urgent launch back while a hold
// is raised.  hctl[2] sums the microseconds the gates of the lane's solve have waited (all passes, all launches); when the sum reaches
// UALM_HOLD_BOUND_NS the gate marks the solve as taking no further hold (hctl[1]) and lets it go, so the solve waits at most that long
// in all.  The control kernel repeats the pass while the launch's queue has problems no slot took
__global__ void hold_gate_kernel(const unsigned char *hold, int *hctl, int urgent)
{
    if (urgent || ((volatile int *)hctl)[1]) return;
    const long long budget = (long long)(UALM_HOLD_BOUND_NS / 1000ull) - ((volatile int *)hctl)[2];
    unsigned long long t0, now;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    now = t0;
    bool bound = budget <= 0;
    while (!bound && hold_raised(hold)) {
        __nanosleep(4000);
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
        bound = (long long)((now - t0) / 1000ull) >= budget;
    }
    atomicAdd(hctl + 2, (int)((now - t0) / 1000ull));
    if (bound) ((volatile int *)hctl)[1] = 1;
}
__global__ void solve_loop_ctrl_kernel(cudaGraphConditionalHandle h, const int *queue, int n_active)
{
    cudaGraphSetConditional(h, *(const volatile int *)queue < n_active ? 1u : 0u);
}

// one innerCallback evaluation per problem at caller-provided x / duals (kernel-level parity)
__global__ void __launch_bounds__(UALM_THREADS * UALM_WPB) eval_kernel(const __grid_constant__ BatchPtrs bp, const __grid_constant__ DevParams p, const __grid_constant__ DevMap map,
        const __grid_constant__ SmemLayout L, R rho)
{
    const int lane = threadIdx.x & 31, wslot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);   // 1 .. UALM_WPB warps per CTA
    if (wslot >= bp.n_active) return;   // whole warp exits; warps never synchronise with each other
    const unsigned sm = (unsigned)__cvta_generic_to_shared(ualm_smem) + 8u * (unsigned)((threadIdx.x >> 5) * L.total_doubles);
    const int prob = bp.order[wslot];
    Traj t;
    lu_build_consts(sm + 8u * (unsigned)L.lutab, lane);
    traj_setup(t, bp, p, L, sm, sm, prob, 1, 0, threadIdx.x >> 5);
    for (int q = lane; q < t.n; q += 32) t.x[q] = bp.x0[t.pd->off_x + q];
    if (lane == 0) { t.sc[SC_SCALE_FX] = bp.scale_fx_io[prob]; t.sc[SC_RHO] = rho; }
    UALM_SYNC();
    evaluate(t, map, p, lane);
    const int nx = 6 * t.N, ny = 6 * t.M;
    for (int q = lane; q < t.n; q += 32) bp.grad_out[t.pd->off_x + q] = t.g[q];
    for (int q = lane; q < 2 * nx; q += 32) bp.c_xy[t.pd->off_cxy + q] = t.cxy[q];
    for (int q = lane; q < ny; q += 32) bp.c_yaw[t.pd->off_cyaw + q] = t.cyaw[q];
    if (lane == 0) bp.f_out[prob] = t.sc[SC_F];
}

// initScaling per problem at x0
__global__ void __launch_bounds__(UALM_THREADS * UALM_WPB) scaling_kernel(const __grid_constant__ BatchPtrs bp, const __grid_constant__ DevParams p, const __grid_constant__ DevMap map,
        const __grid_constant__ SmemLayout L)
{
    const int lane = threadIdx.x & 31, wslot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);   // 1 .. UALM_WPB warps per CTA
    if (wslot >= bp.n_active) return;   // whole warp exits; warps never synchronise with each other
    const unsigned sm = (unsigned)__cvta_generic_to_shared(ualm_smem) + 8u * (unsigned)((threadIdx.x >> 5) * L.total_doubles);
    const int prob = bp.order[wslot];
    Traj t;
    lu_build_consts(sm + 8u * (unsigned)L.lutab, lane);
    traj_setup(t, bp, p, L, sm, sm, prob, 1, 0, threadIdx.x >> 5);
    for (int q = lane; q < t.n; q += 32) t.x[q] = bp.x0[t.pd->off_x + q];
    if (lane == 0) { t.sc[SC_SCALE_FX] = 1.0; t.sc[SC_RHO] = p.rho; }
    UALM_SYNC();
    init_scaling(t, map, p, lane);
    if (lane == 0) bp.scale_fx_io[prob] = t.sc[SC_SCALE_FX];
}

// the penalty-sampling phase alone (calConstrainCostGrad, alm_traj_opt.cpp:663-991) for roofline timing:
// MINCO state is generated once, then `reps` sampling + accumulation passes are run.
__global__ void __launch_bounds__(UALM_THREADS * UALM_WPB) penalty_only_kernel(const __grid_constant__ BatchPtrs bp, const __grid_constant__ DevParams p, const __grid_constant__ DevMap map,
        const __grid_constant__ SmemLayout L, int reps)
{
    const int lane = threadIdx.x & 31, wslot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);   // 1 .. UALM_WPB warps per CTA
    if (wslot >= bp.n_active) return;   // whole warp exits; warps never synchronise with each other
    const unsigned sm = (unsigned)__cvta_generic_to_shared(ualm_smem) + 8u * (unsigned)((threadIdx.x >> 5) * L.total_doubles);
    const int prob = bp.order[wslot];
    Traj t;
    lu_build_consts(sm + 8u * (unsigned)L.lutab, lane);
    traj_setup(t, bp, p, L, sm, sm, prob, 1, 0, threadIdx.x >> 5);
    for (int q = lane; q < t.n; q += 32) t.x[q] = bp.x0[t.pd->off_x + q];
    if (lane == 0) { t.sc[SC_SCALE_FX] = 1.0; t.sc[SC_RHO] = p.rho; }
    UALM_SYNC();
    minco_generate(t, lane);
    sample_tables(t, lane);
    for (int r = 0; r < reps; r++) {
        penalty_samples(t, map, p, lane, 32);
        UALM_SYNC();
        accumulate_tasks(t, lane, 32);
        cost_chain(t, lane);
        UALM_SYNC();
    }
    if (lane == 0) bp.f_out[prob] = t.sc[SC_CONSTR];
}

// ---------------------------------------------------------------------------------------------
// Sampling a trajectory as the reference does: its duration, its sample times t = 0, dt, 2dt.. and its value at a time.  The scan,
// the replan build and the hand-over to the MPC all sample through these helpers, so their samples are the same bits.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int locate_piece(int P, R dur, R &t)   // PolyTrajectory::locatePieceIdx (se2traj.hpp:343-361), uniform durations
{
    int idx;
    for (idx = 0; idx < P && t > dur; idx++) t -= dur;
    if (idx == P) { idx--; t += dur; }
    return idx;
}
__device__ __forceinline__ void piece_eval(const R *c, R t, R &v, R &dv, R &ddv)   // Piece::getValue / getDotValue / getDDotValue (se2traj.hpp:106-150)
{
    v = 0.0; dv = 0.0; ddv = 0.0;
    R tn = 1.0;
    for (int k = 0; k <= 5; k++) { v += tn * c[k]; tn *= t; }
    tn = 1.0;
    int n = 1;
    for (int k = 1; k <= 5; k++) { dv += (R)n * tn * c[k]; tn *= t; n++; }
    tn = 1.0;
    int m = 1; n = 2;
    for (int k = 2; k <= 5; k++) { ddv += (R)(m * n) * tn * c[k]; tn *= t; m++; n++; }
}
// PolyTrajectory::getTotalDuration (se2traj.hpp:291-300) of the xy and the yaw part, each summed piece by piece; an SE2 trajectory
// lasts the smaller (:415-418).  A diverged solve can leave an astronomically long (or non-finite) duration, over which the
// reference's scan would run (almost) forever: such a trajectory is not scanned.  The host validates replan input with the same sums
struct TrajDur {
    R xy, yaw, total;
    __host__ __device__ __forceinline__ bool scannable(R dt) const { return total / dt < 4.0e6; }
};
__host__ __device__ __forceinline__ TrajDur traj_duration(int N, int M, R Tx, R Ty)
{
    TrajDur d{0.0, 0.0, 0.0};
    for (int i = 0; i < N; i++) d.xy += Tx;
    for (int i = 0; i < M; i++) d.yaw += Ty;
    d.total = d.xy < d.yaw ? d.xy : d.yaw;
    return d;
}
// The lane's sample time in the chunk of 32 that starts at tbase, which moves on to the next chunk's start.  The reference forms its
// samples by t += dt: every lane makes the same 32 additions, so each sample is bit for bit the sequential loop's
__device__ __forceinline__ R chunk_time(R &tbase, R dt, int lane)
{
    R tm = 0.0, tt = tbase;
    for (int i = 0; i < 32; i++) { if (i == lane) tm = tt; tt = tt + dt; }
    tbase = tt;
    return tm;
}
// Position, velocity and acceleration of the xy part at time txy and the yaw part at time tyaw (PolyTrajectory::getValue / getVel /
// getAcc, se2traj.hpp:363-391).  ip, tl and iy, ty locate the pieces, for a second trajectory of the same piece durations
struct SE2Eval { R x, y, yaw, vx, vy, dyaw, ax, ay, ddyaw; int ip, iy; R tl, ty; };
__device__ __forceinline__ SE2Eval se2_eval(const R *cxy, const R *cyaw, int N, int M, R Tx, R Ty, R txy, R tyaw)
{
    SE2Eval e;
    e.tl = txy;
    e.ip = locate_piece(N, Tx, e.tl);
    piece_eval(cxy + 6 * e.ip, e.tl, e.x, e.vx, e.ax);
    piece_eval(cxy + 6 * N + 6 * e.ip, e.tl, e.y, e.vy, e.ay);
    e.ty = tyaw;
    e.iy = locate_piece(M, Ty, e.ty);
    piece_eval(cyaw + 6 * e.iy, e.ty, e.yaw, e.dyaw, e.ddyaw);
    return e;
}

// ---------------------------------------------------------------------------------------------
// Post-solve quality scan (SURVEY 8f-4): ALMTrajOpt::getMaxVxAxAyCurAttSig (alm_traj_opt.h:170-229) and
// SE2Trajectory::getNonHolError (se2traj.hpp:551-561), one warp per trajectory, one lane per sample time.  The reference keeps "the
// first sample with the largest |value|": every lane keeps its own slice, the warp reduces by (|value|, earliest sample), and the
// non-holonomic error is summed in sample order -- bit-identical to the sequential loops (oracle: orc_feasibility).
// ---------------------------------------------------------------------------------------------
struct AbsMax {   // "if (fabs(best) < fabs(v)) best = v" over samples in time order
    R val; int idx;
    __device__ __forceinline__ void init() { val = 0.0; idx = 0x7fffffff; }
    __device__ __forceinline__ void see(R v, int k) { if (fabs(val) < fabs(v)) { val = v; idx = k; } }
    __device__ __forceinline__ void reduce()
    {
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
            const R ov = __shfl_xor_sync(0xffffffffu, val, off);
            const int oi = __shfl_xor_sync(0xffffffffu, idx, off);
            if (fabs(val) < fabs(ov) || (fabs(val) == fabs(ov) && oi < idx)) { val = ov; idx = oi; }
        }
    }
};
// The values of one sample at time tm < the trajectory's duration: vx, ax, ay, cur, att and sig of getMaxVxAxAyCurAttSig and the
// term getNonHolError sums
struct FeasSample { R vx, ax, ay, cur, att, sig, term; };
__device__ __forceinline__ FeasSample feas_sample(const DevMap &map, R gravity, const R *cxy, const R *cyaw, int N, int M, R Tx, R Ty, R tm)
{
    const SE2Eval e = se2_eval(cxy, cyaw, N, M, Tx, Ty, tm, tm);
    R se2[3] = {e.x, e.y, e.yaw};
    normSO2(se2[2]);                                  // getNormSE2Pos (se2traj.hpp:433-443)
    R tv[7], tg[7][3];
    map_get_all_with_grad(map, se2, tv, tg);          // values as getTerrainVariables (uneven_map.h:221-256)
    const double2 sc = dev_sincos(e.yaw);
    const R sy_ = sc.x, cy_ = sc.y;
    const R vnorm = sqrt(e.vx * e.vx + e.vy * e.vy);
    const R lon = e.ax * cy_ + e.ay * sy_;
    const R lat = -e.ax * sy_ + e.ay * cy_;
    FeasSample s;
    s.vx = vnorm * tv[0];
    s.ax = lon * tv[0] + gravity * tv[1];
    s.ay = lat * tv[2] + gravity * tv[3];
    const R wz = e.dyaw * tv[5];
    s.cur = wz / sqrt(s.vx * s.vx + UALM_DELTA_SIGL);
    s.att = -1.0 / tv[5];
    s.sig = tv[6];
    s.term = fabs(e.vx * sy_ + e.vy * (-cy_));
    return s;
}
// The scan of solved trajectories (ualm_feasibility_batch, t_from null) and of trajectories the caller holds
// (ualm_check_trajectories), restricted to the samples t >= t_from of the sequence t = 0, dt, 2dt.. (not restarted at t_from, so
// every kept sample is bit for bit the full scan's), with the time of the first kept sample that breaks each of six limits; a first
// violation is the earliest set lane of its ballot in the first chunk that has one.  Oracle: tests/check_oracle.cpp.
// out[16 * problem + ...] = {max_vx, max_ax, max_ay, max_cur, max_att, max_sig, nonhol_error, samples, T_xy piece, T_yaw piece} over
// the kept samples, then the first-violation times of |vx| > max_vel, |ax| > max_acc_lon, |ay| > max_acc_lat, |cur| > max_kap,
// att > -min_cxi, sig > max_sig (-1: none).  Not scanned (over the compiled limits, or more than 4e6 samples): zeros, a sample count
// of -1, no violation, and the piece durations of a trajectory within the limits
struct CheckPtrs {
    const ProbDesc *desc;          // N, M, off_cxy, off_cyaw, the six limits at pp[2..7]; S == 0 marks a problem over the compiled limits
    const R *c_xy, *c_yaw, *piece_T;
    const R *t_from;               // null: 0 for every problem
    R *out;
};
// idx: the n problems to scan, those of one environment, whose grid and gravity this launch carries
__global__ void __launch_bounds__(UALM_THREADS * UALM_WPB) check_kernel(const __grid_constant__ CheckPtrs a, const __grid_constant__ DevMap map, R gravity,
        R dt, const int *idx, int n)
{
    const int lane = threadIdx.x & 31, w = blockIdx.x * UALM_WPB + (threadIdx.x >> 5);
    if (w >= n) return;         // whole warp exits
    const int prob = idx[w];
    const ProbDesc *pd = a.desc + prob;
    R *o = a.out + 16 * (size_t)prob;
    if (pd->S == 0) {
        if (lane < 16) o[lane] = lane == 7 || lane >= 10 ? -1.0 : 0.0;
        return;
    }
    const R Tx = a.piece_T[2 * prob], Ty = a.piece_T[2 * prob + 1];
    const int N = pd->N, M = pd->M;
    const TrajDur d = traj_duration(N, M, Tx, Ty);
    if (!d.scannable(dt)) {
        if (lane < 16) o[lane] = lane == 7 || lane >= 10 ? -1.0 : lane == 8 ? Tx : lane == 9 ? Ty : 0.0;
        return;
    }
    const R *cxy = a.c_xy + pd->off_cxy, *cyaw = a.c_yaw + pd->off_cyaw, *lim = pd->pp + 2;
    const R max_vel = lim[0], max_acc_lon = lim[1], max_acc_lat = lim[2], max_kap = lim[3], min_cxi = lim[4], max_sig = lim[5];
    const R t0 = a.t_from ? a.t_from[prob] : 0.0;
    AbsMax mvx, max_, may, mcur;
    mvx.init(); max_.init(); may.init(); mcur.init();
    R matt = -1.0, msig = 0.0, err = 0.0;
    R first[6] = {-1.0, -1.0, -1.0, -1.0, -1.0, -1.0};   // the same on every lane
    unsigned found = 0;
    long long count = 0;
    R tbase = 0.0;
    for (int kbase = 0;; kbase += 32) {
        const R tm = chunk_time(tbase, dt, lane);
        const bool valid = tm < d.total, kept = valid && tm >= t0;
        R term = 0.0;
        unsigned viol = 0;
        if (kept) {
            const FeasSample s = feas_sample(map, gravity, cxy, cyaw, N, M, Tx, Ty, tm);
            const int k = kbase + lane;
            max_.see(s.ax, k); may.see(s.ay, k); mvx.see(s.vx, k); mcur.see(s.cur, k);
            if (matt < s.att) matt = s.att;
            if (msig < s.sig) msig = s.sig;
            term = s.term;
            viol = (fabs(s.vx) > max_vel ? 1u : 0u) | (fabs(s.ax) > max_acc_lon ? 2u : 0u) | (fabs(s.ay) > max_acc_lat ? 4u : 0u) |
                   (fabs(s.cur) > max_kap ? 8u : 0u) | (s.att > -min_cxi ? 16u : 0u) | (s.sig > max_sig ? 32u : 0u);
        }
        const unsigned km = __ballot_sync(0xffffffffu, kept);   // the kept lanes are contiguous: t grows with the lane
        for (unsigned m = km; m; m &= m - 1) err += __shfl_sync(0xffffffffu, term, __ffs(m) - 1);
        count += __popc(km);
#pragma unroll
        for (int q = 0; q < 6; q++) {
            const unsigned vm = __ballot_sync(0xffffffffu, (viol >> q) & 1u);
            const R tv = __shfl_sync(0xffffffffu, tm, vm ? __ffs(vm) - 1 : 0);
            if (vm && !((found >> q) & 1u)) { first[q] = tv; found |= 1u << q; }
        }
        if (__popc(__ballot_sync(0xffffffffu, valid)) < 32) break;
    }
    mvx.reduce(); max_.reduce(); may.reduce(); mcur.reduce();
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        const R oa = __shfl_xor_sync(0xffffffffu, matt, off), os = __shfl_xor_sync(0xffffffffu, msig, off);
        if (matt < oa) matt = oa;
        if (msig < os) msig = os;
    }
    if (lane == 0) {
        o[0] = mvx.val; o[1] = max_.val; o[2] = may.val; o[3] = mcur.val; o[4] = matt; o[5] = msig; o[6] = err; o[7] = (R)count; o[8] = Tx; o[9] = Ty;
        for (int q = 0; q < 6; q++) o[10 + q] = first[q];
    }
}

// ---------------------------------------------------------------------------------------------
// Replanned problems of trajectories the caller holds (ualm_submit_replan): the state at tau = t_from, then PlanManager's resampler
// (resample_stream.h) over the polyline {the point at tau, the samples tau < t < duration of the reference's sequence
// t = 0, dt, 2dt.., the goal of the original problem}.  One warp per row:
// each chunk the lanes evaluate 32 sample times, then every lane runs the sequential resampler on the same points broadcast by
// shuffle, and lane 0 writes.  Waypoints past the compiled limits are counted, not formed; such a row's inner points are zeros.  The
// stream is bounded (ualm_rs_push), so a row's serial work is bounded whatever its lengths and yaws.
// Oracle: tests/replan_oracle.cpp.
// out[UALM_REPLAN_STRIDE * row + ...] = bnd' (18) | total_time | N' | M' | inner xy (2 (UALM_NMAX - 1)) | inner yaw (UALM_MMAX - 1)
// ---------------------------------------------------------------------------------------------
static_assert(UALM_REPLAN_INNER_XY == 2 * (UALM_NMAX - 1) && UALM_REPLAN_INNER_YAW == UALM_MMAX - 1, "ualm.h's replan strides");
#define UALM_REPLAN_STRIDE (21 + UALM_REPLAN_INNER_XY + UALM_REPLAN_INNER_YAW)
struct ReplanPtrs {
    const ProbDesc *desc;          // N, M, off_cxy, off_cyaw of the trajectory
    const R *c_xy, *c_yaw, *piece_T, *bnd, *t_from;
    R *out;
};
struct ReplanParams { R dt, piece_len, yaw_piece_times, mean_vel, init_time_times; };
// the host has checked N, M >= 1, 0 <= t_from < duration and duration / dt < 4e6 for every row
__global__ void __launch_bounds__(UALM_THREADS * UALM_WPB) replan_kernel(const __grid_constant__ ReplanPtrs a, const __grid_constant__ ReplanParams rp, int n)
{
    const int lane = threadIdx.x & 31, w = blockIdx.x * UALM_WPB + (threadIdx.x >> 5);
    if (w >= n) return;         // whole warp exits
    const ProbDesc *pd = a.desc + w;
    const int N = pd->N, M = pd->M;
    const R *cxy = a.c_xy + pd->off_cxy, *cyaw = a.c_yaw + pd->off_cyaw, *bnd = a.bnd + 18 * (size_t)w;
    const R Tx = a.piece_T[2 * w], Ty = a.piece_T[2 * w + 1], t0 = a.t_from[w];
    R *o = a.out + UALM_REPLAN_STRIDE * (size_t)w, *oxy = o + 21, *oyaw = oxy + UALM_REPLAN_INNER_XY;
    for (int q = lane; q < UALM_REPLAN_INNER_XY + UALM_REPLAN_INNER_YAW; q += 32) oxy[q] = 0.0;
    __syncwarp();
    const R total = traj_duration(N, M, Tx, Ty).total;
    const SE2Eval st = se2_eval(cxy, cyaw, N, M, Tx, Ty, t0, t0);     // the start state (every lane)
    R *wxy = lane == 0 ? oxy : nullptr, *wyaw = lane == 0 ? oyaw : nullptr;
    UalmResampleStream s;
    ualm_rs_init(s, rp.piece_len, rp.yaw_piece_times);
    ualm_rs_push(s, st.x, st.y, st.yaw, wxy, UALM_NMAX - 1, wyaw, UALM_MMAX - 1);
    R tbase = 0.0;
    while (true) {
        const R tm = chunk_time(tbase, rp.dt, lane);
        const bool valid = tm < total, kept = valid && tm > t0;
        R x = 0.0, y = 0.0, h = 0.0;
        if (kept) {
            const SE2Eval e = se2_eval(cxy, cyaw, N, M, Tx, Ty, tm, tm);
            x = e.x; y = e.y; h = e.yaw;
        }
        const unsigned km = __ballot_sync(0xffffffffu, kept);   // the kept lanes are contiguous: t grows with the lane
        for (unsigned m = km; m; m &= m - 1) {
            const int l = __ffs(m) - 1;
            const R bx = __shfl_sync(0xffffffffu, x, l), by = __shfl_sync(0xffffffffu, y, l), bh = __shfl_sync(0xffffffffu, h, l);
            ualm_rs_push(s, bx, by, bh, wxy, UALM_NMAX - 1, wyaw, UALM_MMAX - 1);
        }
        if (__popc(__ballot_sync(0xffffffffu, valid)) < 32) break;
    }
    ualm_rs_push(s, bnd[6], bnd[7], bnd[15], wxy, UALM_NMAX - 1, wyaw, UALM_MMAX - 1);   // the goal: end_xy's position, end_yaw's angle
    // cut short (resample_stream.h: a huge or non-finite length or yaw): over the limits, N' = M' = UALM_RS_MAX_WAYPOINTS + 2
    const long long Nn = s.cut ? UALM_RS_MAX_WAYPOINTS + 2 : s.nxy + 1, Mn = s.cut ? UALM_RS_MAX_WAYPOINTS + 2 : s.nyaw + 1;
    if (Nn > UALM_NMAX || Mn > UALM_MMAX) {      // over the limits: the waypoints written before the count passed them go
        __syncwarp();
        for (int q = lane; q < UALM_REPLAN_INNER_XY + UALM_REPLAN_INNER_YAW; q += 32) oxy[q] = 0.0;
    }
    if (lane == 0) {
        const R head[18] = {st.x, st.y, st.vx, st.vy, st.ax, st.ay, bnd[6], bnd[7], bnd[8], bnd[9], bnd[10], bnd[11], st.yaw, st.dyaw, st.ddyaw,
                            bnd[15], bnd[16], bnd[17]};
        for (int k = 0; k < 18; k++) o[k] = head[k];
        o[18] = ualm_rs_total_time(s, rp.mean_vel, rp.init_time_times);
        o[19] = (R)Nn; o[20] = (R)Mn;
    }
}

// ---------------------------------------------------------------------------------------------
// SURVEY 8f-3: the hand-over to the MPC, for the whole batch on the device.
//   (1) the SE2Traj message PlanManager publishes (plan_manager.cpp:151-185, msg/SE2Traj.msg:1-9): start point of every piece
//       (Piece::getValue(0), se2traj.hpp:106-118), the end point (PolyTrajectory::getValue(total), :363-368) and the piece durations;
//   (2) the trajectory the MPC then tracks: TrajAnalyzer::setTraj (traj_anal.hpp:125-181) feeds those points, the message's (zero)
//       boundary velocity / acceleration and zero tail derivatives to its own MinJerkOpt::generate (minco_traj.hpp:365-444 -- the same
//       banded LU without pivoting as the back-end's, banded_system.hpp:66-118, restated here operation for operation);
//   (3) how far (2) is from the planned spline (the back-end plans with a boundary speed of init_sig_vel, plan_manager.cpp:93-94,
//       which the message does not carry): the largest position / yaw deviation over t = 0, dt, 2dt, .. and where it occurs.
// One warp per problem: lane 0 solves the xy system (one factorization, two right-hand sides), lane 1 the yaw system, every lane
// takes a slice of the samples of (3).  band: scratch, 13 * (6N + 6M) doubles per problem at 13 * (off_cxy / 2 + off_cyaw).
// The same kernel serves a lane's solved batch (ualm_mpc_export_batch) and trajectories the caller holds (ualm_mpc_export_trajectories).
// dev[4 * problem + ..] = {max |p_plan - p_mpc|, its time, max |yaw_plan - yaw_mpc|, its time}
// ---------------------------------------------------------------------------------------------
struct BandView {      // BandedSystem storage (banded_system.hpp:25-64): entry (i, j) at [(i - j + 6) * n + j]
    R *d; int n;
    __device__ __forceinline__ R &operator()(int i, int j) const { return d[(size_t)(i - j + 6) * n + j]; }
};
// MinJerkOpt::generate for Dim right-hand sides sharing one matrix (minco_traj.hpp:365-444 == se2traj.hpp:595-680); c: 6P x Dim
// column-major (column stride 6P); point i of column d at pts[i * pst + d * cst]; all pieces last T
__device__ void mpc_minco_serial(BandView A, int P, int Dim, R T, const R *pts, int pst, int cst, const R *v0, const R *a0, R *c)
{
    const int n = 6 * P;
    for (int q = 0; q < 13 * n; q++) A.d[q] = 0.0;
    for (int q = 0; q < n * Dim; q++) c[q] = 0.0;
    const R T1 = T, T2 = T1 * T1, T3 = T2 * T1, T4 = T2 * T2, T5 = T4 * T1;
    A(0, 0) = 1.0; A(1, 1) = 1.0; A(2, 2) = 2.0;
    for (int d = 0; d < Dim; d++) { c[0 + d * n] = pts[d * cst]; c[1 + d * n] = v0[d]; c[2 + d * n] = a0[d]; }
    for (int i = 0; i < P - 1; i++) {
        const int r = 6 * i;
        A(r + 3, r + 3) = 6.0; A(r + 3, r + 4) = 24.0 * T1; A(r + 3, r + 5) = 60.0 * T2; A(r + 3, r + 9) = -6.0;
        A(r + 4, r + 4) = 24.0; A(r + 4, r + 5) = 120.0 * T1; A(r + 4, r + 10) = -24.0;
        A(r + 5, r) = 1.0; A(r + 5, r + 1) = T1; A(r + 5, r + 2) = T2; A(r + 5, r + 3) = T3; A(r + 5, r + 4) = T4; A(r + 5, r + 5) = T5;
        A(r + 6, r) = 1.0; A(r + 6, r + 1) = T1; A(r + 6, r + 2) = T2; A(r + 6, r + 3) = T3; A(r + 6, r + 4) = T4; A(r + 6, r + 5) = T5;
        A(r + 6, r + 6) = -1.0;
        A(r + 7, r + 1) = 1.0; A(r + 7, r + 2) = 2.0 * T1; A(r + 7, r + 3) = 3.0 * T2; A(r + 7, r + 4) = 4.0 * T3; A(r + 7, r + 5) = 5.0 * T4;
        A(r + 7, r + 7) = -1.0;
        A(r + 8, r + 2) = 2.0; A(r + 8, r + 3) = 6.0 * T1; A(r + 8, r + 4) = 12.0 * T2; A(r + 8, r + 5) = 20.0 * T3; A(r + 8, r + 8) = -2.0;
        for (int d = 0; d < Dim; d++) c[r + 5 + d * n] = pts[(i + 1) * pst + d * cst];
    }
    A(n - 3, n - 6) = 1.0; A(n - 3, n - 5) = T1; A(n - 3, n - 4) = T2; A(n - 3, n - 3) = T3; A(n - 3, n - 2) = T4; A(n - 3, n - 1) = T5;
    A(n - 2, n - 5) = 1.0; A(n - 2, n - 4) = 2.0 * T1; A(n - 2, n - 3) = 3.0 * T2; A(n - 2, n - 2) = 4.0 * T3; A(n - 2, n - 1) = 5.0 * T4;
    A(n - 1, n - 4) = 2.0; A(n - 1, n - 3) = 6.0 * T1; A(n - 1, n - 2) = 12.0 * T2; A(n - 1, n - 1) = 20.0 * T3;
    for (int d = 0; d < Dim; d++) c[n - 3 + d * n] = pts[P * pst + d * cst];   // tail velocity / acceleration stay zero (traj_anal.hpp:162-163)
    // factorizeLU (banded_system.hpp:66-91): no pivoting, exact-zero multipliers skipped
    for (int k = 0; k <= n - 2; k++) {
        const int iM = min(k + 6, n - 1), jM = min(k + 6, n - 1);
        R cVl = A(k, k);
        for (int i = k + 1; i <= iM; i++) if (A(i, k) != 0.0) A(i, k) /= cVl;
        for (int j = k + 1; j <= jM; j++) {
            cVl = A(k, j);
            if (cVl != 0.0)
                for (int i = k + 1; i <= iM; i++) if (A(i, k) != 0.0) A(i, j) -= A(i, k) * cVl;
        }
    }
    // solve (banded_system.hpp:96-118)
    for (int j = 0; j <= n - 1; j++) {
        const int iM = min(j + 6, n - 1);
        for (int i = j + 1; i <= iM; i++)
            if (A(i, j) != 0.0) for (int d = 0; d < Dim; d++) c[i + d * n] -= A(i, j) * c[j + d * n];
    }
    for (int j = n - 1; j >= 0; j--) {
        for (int d = 0; d < Dim; d++) c[j + d * n] /= A(j, j);
        const int iM = max(0, j - 6);
        for (int i = iM; i <= j - 1; i++)
            if (A(i, j) != 0.0) for (int d = 0; d < Dim; d++) c[i + d * n] -= A(i, j) * c[j + d * n];
    }
}
// the message's boundary derivatives: row `prob` of init_rows, 6 doubles {v_x, v_y, v_yaw, a_x, a_y, a_yaw} per problem (each robot
// its own start state), or `init` for every problem when init_rows is null
struct MpcOut { R *pos_pts, *posT_pts, *angle_pts, *angleT_pts, *c_mpc_xy, *c_mpc_yaw, *dev, *band; const R *init_rows; R init[6]; };
__global__ void __launch_bounds__(UALM_THREADS * UALM_WPB) mpc_export_kernel(const __grid_constant__ BatchPtrs bp, R dt, const __grid_constant__ MpcOut o)
{
    const int lane = threadIdx.x & 31, prob = blockIdx.x * UALM_WPB + (threadIdx.x >> 5);
    if (prob >= bp.B) return;
    const ProbDesc *pd = bp.desc + prob;
    const int N = pd->N, M = pd->M, nx = 6 * N;
    const long long sN = pd->off_cxy / 12, sM = pd->off_cyaw / 6;         // pieces of the problems before this one
    R *pp = o.pos_pts + 2 * (sN + prob), *pt = o.posT_pts + sN, *ap = o.angle_pts + (sM + prob), *at = o.angleT_pts + sM;
    R *mxy = o.c_mpc_xy + pd->off_cxy, *myaw = o.c_mpc_yaw + pd->off_cyaw;
    R *dv = o.dev + 4 * (size_t)prob;
    if (pd->S == 0) {            // over the compiled limits: not solved
        for (int q = lane; q < 2 * (N + 1); q += 32) pp[q] = 0.0;
        for (int q = lane; q < N; q += 32) pt[q] = 0.0;
        for (int q = lane; q <= M; q += 32) ap[q] = 0.0;
        for (int q = lane; q < M; q += 32) at[q] = 0.0;
        for (int q = lane; q < 12 * N; q += 32) mxy[q] = 0.0;
        for (int q = lane; q < 6 * M; q += 32) myaw[q] = 0.0;
        if (lane < 4) dv[lane] = 0.0;
        return;
    }
    const R *cxy = bp.c_xy + pd->off_cxy, *cyaw = bp.c_yaw + pd->off_cyaw;
    const R Tx = bp.piece_T[2 * prob], Ty = bp.piece_T[2 * prob + 1];
    const TrajDur d = traj_duration(N, M, Tx, Ty);
    // (1) the message: piece start points are the constant coefficients (getValue(0) only adds exact zeros to them); the end point is
    // PolyTrajectory::getValue at the summed duration
    for (int i = lane; i < N; i += 32) { pp[2 * i] = cxy[6 * i]; pp[2 * i + 1] = cxy[nx + 6 * i]; pt[i] = Tx; }
    for (int i = lane; i < M; i += 32) { ap[i] = cyaw[6 * i]; at[i] = Ty; }
    if (lane == 0) {
        const SE2Eval e = se2_eval(cxy, cyaw, N, M, Tx, Ty, d.xy, d.yaw);
        pp[2 * N] = e.x; pp[2 * N + 1] = e.y; ap[M] = e.yaw;
    }
    __syncwarp();
    // (2) the MPC's own MINCO over the message
    R *band = o.band + 13 * (pd->off_cxy / 2 + pd->off_cyaw);
    const R *init = o.init_rows ? o.init_rows + 6 * (size_t)prob : o.init;
    if (lane == 0) mpc_minco_serial(BandView{band, nx}, N, 2, Tx, pp, 2, 1, init, init + 3, mxy);
    if (lane == 1) mpc_minco_serial(BandView{band + 13 * nx, 6 * M}, M, 1, Ty, ap, 1, 0, init + 2, init + 5, myaw);
    __syncwarp();
    // (3) planned against tracked, over the shorter of the two durations like every scan of the reference (se2traj.hpp:415-418)
    if (!d.scannable(dt)) {
        if (lane == 0) { dv[0] = -1.0; dv[1] = 0.0; dv[2] = -1.0; dv[3] = 0.0; }
        return;
    }
    R bp_ = 0.0, bpt = 0.0, by_ = 0.0, byt = 0.0;
    R tbase = 0.0;
    while (true) {
        const R tm = chunk_time(tbase, dt, lane);
        const bool valid = tm < d.total;
        if (valid) {
            const SE2Eval e = se2_eval(cxy, cyaw, N, M, Tx, Ty, tm, tm);
            R qx, qy, yb, d1, d2;      // the tracked trajectory, whose pieces last as long as the planned one's
            piece_eval(mxy + 6 * e.ip, e.tl, qx, d1, d2); piece_eval(mxy + nx + 6 * e.ip, e.tl, qy, d1, d2);
            piece_eval(myaw + 6 * e.iy, e.ty, yb, d1, d2);
            const R ep = sqrt((e.x - qx) * (e.x - qx) + (e.y - qy) * (e.y - qy)), ey = fabs(e.yaw - yb);
            if (bp_ < ep) { bp_ = ep; bpt = tm; }
            if (by_ < ey) { by_ = ey; byt = tm; }
        }
        if (__popc(__ballot_sync(0xffffffffu, valid)) < 32) break;
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {      // largest value, earliest time among equals
        const R op = __shfl_xor_sync(0xffffffffu, bp_, off), opt = __shfl_xor_sync(0xffffffffu, bpt, off);
        const R oy = __shfl_xor_sync(0xffffffffu, by_, off), oyt = __shfl_xor_sync(0xffffffffu, byt, off);
        if (bp_ < op || (bp_ == op && opt < bpt)) { bp_ = op; bpt = opt; }
        if (by_ < oy || (by_ == oy && oyt < byt)) { by_ = oy; byt = oyt; }
    }
    if (lane == 0) { dv[0] = bp_; dv[1] = bpt; dv[2] = by_; dv[3] = byt; }
}

// fixed-stride result records for the multi-GPU all-gather
__global__ void pack_records_kernel(BatchPtrs bp, int B, R *rec, int stride)
{
    const int b = blockIdx.x;
    if (b >= B) return;
    const ProbDesc *pd = bp.desc + b;
    R *o = rec + (size_t)b * stride;
    const ualm_result_t r = bp.results[b];
    if (threadIdx.x == 0) {
        o[0] = r.ret_code; o[1] = r.outer_iters; o[2] = r.n_evals; o[3] = r.n_lbfgs_iters; o[4] = r.inner_cost; o[5] = r.jerk_cost;
        o[6] = r.total_T; o[7] = r.res_h; o[8] = r.res_g; o[9] = pd->N; o[10] = pd->M; o[11] = 0.0;
    }
    const int ncx = 12 * pd->N, ncy = 6 * pd->M;
    for (int q = threadIdx.x; q < stride - 12; q += blockDim.x) {
        R v = 0.0;
        if (q < ncx) v = bp.c_xy[pd->off_cxy + q];
        else if (q < ncx + ncy) v = bp.c_yaw[pd->off_cyaw + q - ncx];
        o[12 + q] = v;
    }
}

} // namespace ualm
