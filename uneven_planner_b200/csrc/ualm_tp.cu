// ualm_tp.cu -- host side of the throughput engine (precision 32 / 65 of include/ualm.h): slot pool, admission of batches,
// the device-side round loop of every group (one CUDA graph per group: ka -> [ks] -> kb per round, continuous batching across the
// batches in flight) and result gathering.
// Kernels: ualm_tp_kernels.cuh, ualm_tp_samples.cuh.  Compiled with FMA contraction ON (its own translation unit).
#include "ualm_tp_samples.cuh"
#include "ualm_tp_host.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

namespace ualm_tp {

#define TP_LANES TP_MAXLANES

#define TCK(call)                                                                                       \
    do {                                                                                                \
        cudaError_t e_ = (call);                                                                        \
        if (e_ != cudaSuccess) { if (err) *err = std::string(#call) + ": " + cudaGetErrorString(e_); return UALM_ENOCUDA; } \
    } while (0)

// device buffer, grown only.  Stream-ordered allocation: cudaFree would wait for the whole device, and so hold the admission of a
// batch until every other batch in flight had finished its round loop.  A buffer is only grown or released when no queued work
// uses it (the host synchronised that work), and the allocation is complete before ensure returns
template <class T>
struct Buf {
    T *p = nullptr;
    size_t cap = 0;
    cudaError_t ensure(size_t n)
    {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFreeAsync(p, cudaStreamPerThread);
        p = nullptr; cap = 0;
        cudaError_t e = cudaMallocAsync((void **)&p, std::max<size_t>(n, 1) * sizeof(T), cudaStreamPerThread);
        if (e == cudaSuccess) e = cudaStreamSynchronize(cudaStreamPerThread);
        if (e == cudaSuccess) cap = n;
        return e;
    }
    void release() { if (p) cudaFreeAsync(p, cudaStreamPerThread); p = nullptr; cap = 0; }
};

static_assert(TP_SUBGROUPS >= UALM_MAX_ENVS, "a lane runs the problems of environment k in its group k: one group per environment");
// the C ABI skips the problems over its compiled limits (UALM_NMAX / UALM_MMAX of ualm_kernels.cuh, which this unit does not include);
// the engine's strides must be those same limits, which ualm.h states as the inner points of a replanned row
static_assert(2 * (TP_NMAX - 1) == UALM_REPLAN_INNER_XY && TP_MMAX - 1 == UALM_REPLAN_INNER_YAW, "TP_NMAX / TP_MMAX must be the compiled limits of ualm.h");

struct TpLane {
    bool have_batch = false, in_flight = false, collected = false;
    int mode = 0;
    const BatchLayout *lay = nullptr;     // the uploaded batch's layout, owned by the context (tp_upload)
    std::vector<int> slots;
    std::vector<AdmitDesc> ad;
    std::vector<GatherDesc> gd;
    Buf<AdmitDesc> d_ad;
    Buf<GatherDesc> d_gd;
    Buf<GatherDesc> d_gdg;            // a submitted batch in several groups: d_gd once per group, other groups' problems without slot
    Buf<double> d_x0, d_xev, d_cxy, d_cyaw, d_xout, d_f, d_grad, d_hx, d_gx, d_sfx, d_scx, d_lam, d_mu, d_scin, d_sfin;
    Buf<long long> d_offs;
    Buf<ualm_result_t> d_res;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    int launches = 0;
    double rho_eval = 1.0;
    bool has_lam = false, has_mu = false, has_scx = false, has_sfx = false, has_xev = false;   // has_xev: admit from d_xev, not d_x0
    // a submitted batch (ualm_submit_batch): its problems go to the mailbox as they finish (tp_poll); d_pub = published already
    bool publish = false;
    ualm_mbox::Mailbox mbox;
    Buf<int> d_pub;
    // stop words, one per problem (TpPool::stop), and their pinned host mirror (grows only): cleared at admission on the engine's
    // stream, raised by copying the whole mirror on the cancel stream while the lane's loops run (tp_cancel, tp_collect's deadline)
    Buf<int> d_stop;
    int *h_stop = nullptr;
    size_t h_stop_cap = 0;
};

struct TpEngine {
    int device = 0, precision = 32;
    bool f32() const { return precision == 32; }
    size_t esz() const { return precision == 32 ? 4 : 8; }
    cudaStream_t stream = nullptr;
    cudaStream_t cstream = nullptr;       // stop-word raises: no group loop occupies it, so a raise reaches the rounds running
    cudaEvent_t evA = nullptr, evB = nullptr;
    // environments (ualm_select_env): parameters, grid and its TMA descriptor of each; group g runs with those of genv[g]
    bool have_params[UALM_MAX_ENVS] = {};
    TpParams p[UALM_MAX_ENVS];
    TpMap map[UALM_MAX_ENVS];
    CUtensorMap tmap[UALM_MAX_ENVS];
    bool have_tmap[UALM_MAX_ENVS] = {};
    int genv[TP_NGROUPS] = {};
    int max_evals = 0;
    int use_tma = 0;              // map corners of kb_kernel: 0 = direct gather through L1 (default: measured faster), 1 = TMA-staged tiles (UALM_TP_TMA=1)
    // (the grids themselves belong to the context, which keeps every version a batch in flight was admitted with: tp_bind_map)
    // pool
    TpPool E;
    int capacity = 0;
    std::vector<int> free_slots;
    int live = 0;                 // slots admitted and not yet freed
    // groups: every batch in flight is split into TP_SUBGROUPS groups (group = lane * TP_SUBGROUPS + k); each group has its own
    // stream, active list and round loop (a CUDA graph launched at admission), so ka of one group overlaps kb of another and a slow
    // trajectory only holds up the rounds of its own group
    cudaStream_t gstream[TP_NGROUPS] = {};
    cudaEvent_t gev[TP_NGROUPS] = {};
    // an urgent ticket (ualm_set_urgent): its admission on ustream and its group loops on ugstream[g], all of the greatest priority and
    // made at their first use (a stream made earlier changes which hardware queue every later stream shares); each is ordered after the
    // work queued on the stream it stands in for, and that stream waits for it, so everything that waits for or queries the engine's
    // own streams sees the urgent work
    cudaStream_t ustream = nullptr, ugstream[TP_NGROUPS] = {};
    cudaEvent_t uev = nullptr;
    // the round loop of each group (launch_loop), one per variant (with / without ks_kernel in the first round, with / without
    // publish_kernel): its graph keeps its conditional node and handle for the engine's life, and every admission replaces the other
    // nodes and updates the executable graph in place.  Destroying an executable graph waits for the device, which would hold the
    // admission until every other batch in flight had finished
    struct Loop { cudaGraph_t G = nullptr, body = nullptr; cudaGraphNode_t cond = nullptr; cudaGraphConditionalHandle h = 0; cudaGraphExec_t exec = nullptr; };
    Loop loops[TP_NGROUPS][4];
    int glive[TP_NGROUPS] = {};           // slots admitted and not yet freed, per group
    Buf<GroupLoop> gloop;                 // [TP_NGROUPS] rounds / launches / round-cap error of each group's loop since its admission
    GroupLoop *h_gloop = nullptr;         // pinned, TP_SUBGROUPS entries
    cudaStream_t capstream = nullptr;     // graph capture only
    int sg = 1;                           // subgroups per batch in use (UALM_TP_SUBGROUPS, <= TP_SUBGROUPS); 1 measured best: the batches in flight already are the groups
    int Nmax_live = 1, Mmax_live = 1;
    Buf<TpState> st;
    Buf<int> active, n_active, remaining;
    Buf<double> vec, cd, gw, kb_cost, lm_ys, lm_alpha, wf, wt;
    Buf<unsigned char> cr, gdc, gdt, dual, hs, hy, wway;
    Buf<long long> wf_off, wway_off, kprof;
    int *h_remaining = nullptr;   // pinned
    TpLane lanes[TP_LANES];
    int chunk = 8;
    int ka_warps = 1;             // warps (= trajectories) per ka_kernel CTA: 1, 2 or 4 (UALM_TP_KA_WARPS); 1 measured best by ~1 %: no warp waits for a CTA mate
    bool prof = false;            // developer profile (UALM_TP_PROFILE=1): in-kernel phase cycle counters, printed at destroy
};

// The columns of A(1)^-1 a MINCO right-hand side can excite, for every piece count (ualm_tp_kernels.cuh: w_tables_kernel).  The LU
// factors they are solved with are scratch
static int build_tables(TpEngine *e, std::string *err)
{
    const int Pmax = TP_MMAX;
    std::vector<int> lu_off(Pmax + 1, 0);
    std::vector<long long> wf_off(Pmax + 1, 0), w_off(Pmax + 1, 0);
    size_t lu_tot = 0, wf_tot = 0, w_tot = 0;
    for (int P = 1; P <= Pmax; P++) {
        lu_off[P] = (int)(lu_tot + (size_t)TP_FPAD * TP_FW);
        lu_tot += (size_t)(6 * P + 2 * TP_FPAD) * TP_FW;
        wf_off[P] = (long long)wf_tot;
        wf_tot += (size_t)(P + 5) * 6 * P;
        w_off[P] = (long long)w_tot;
        w_tot += (size_t)std::max(P - 1, 0) * 6 * P;
    }
    Buf<double> lu;
    Buf<int> d_lu_off;
    TCK(lu.ensure(lu_tot));
    TCK(d_lu_off.ensure(Pmax + 1));
    TCK(e->wf_off.ensure(Pmax + 1));
    TCK(e->wway_off.ensure(Pmax + 1));
    TCK(e->wf.ensure(wf_tot));
    TCK(e->wt.ensure(w_tot));
    TCK(e->wway.ensure(w_tot * e->esz()));
    TCK(cudaMemcpyAsync(d_lu_off.p, lu_off.data(), sizeof(int) * (Pmax + 1), cudaMemcpyHostToDevice, e->stream));
    TCK(cudaMemcpyAsync(e->wf_off.p, wf_off.data(), sizeof(long long) * (Pmax + 1), cudaMemcpyHostToDevice, e->stream));
    TCK(cudaMemcpyAsync(e->wway_off.p, w_off.data(), sizeof(long long) * (Pmax + 1), cudaMemcpyHostToDevice, e->stream));
    lu_tables_kernel<<<(Pmax + 31) / 32, 32, 0, e->stream>>>(lu.p, d_lu_off.p, Pmax);
    TCK(cudaGetLastError());
    const int tpb = 32, gx = (Pmax + 5 + tpb - 1) / tpb;
    dim3 grid(gx, Pmax);
    if (e->f32()) w_tables_kernel<float><<<grid, tpb, 0, e->stream>>>(lu.p, d_lu_off.p, e->wf.p, e->wf_off.p, e->wt.p, (float *)e->wway.p, e->wway_off.p, Pmax);
    else w_tables_kernel<double><<<grid, tpb, 0, e->stream>>>(lu.p, d_lu_off.p, e->wf.p, e->wf_off.p, e->wt.p, (double *)e->wway.p, e->wway_off.p, Pmax);
    TCK(cudaGetLastError());
    TCK(cudaStreamSynchronize(e->stream));
    lu.release();
    d_lu_off.release();
    return UALM_OK;
}

int tp_create(TpEngine **out, int device, int precision, std::string *err)
{
    if (precision != 32 && precision != 65) { if (err) *err = "throughput engine: precision must be 32 or 65"; return UALM_EINVAL; }
    int ndev = 0;
    cudaError_t ce = cudaGetDeviceCount(&ndev);
    if (ce != cudaSuccess || ndev <= 0) { if (err) *err = std::string("no CUDA device: ") + cudaGetErrorString(ce); return UALM_ENOCUDA; }
    if (device < 0 || device >= ndev) { if (err) *err = "device ordinal out of range"; return UALM_EINVAL; }
    TCK(cudaSetDevice(device));
    TpEngine *e = new TpEngine();
    e->device = device; e->precision = precision;
    if (const char *s = getenv("UALM_TP_TMA")) e->use_tma = atoi(s) ? 1 : 0;
    if (const char *s = getenv("UALM_TP_NOTMA")) { if (atoi(s)) e->use_tma = 0; }
    if (const char *s = getenv("UALM_TP_CHUNK")) e->chunk = std::max(1, atoi(s));
    if (const char *s = getenv("UALM_TP_KA_WARPS")) { const int w = atoi(s); if (w == 1 || w == 2 || w == 4) e->ka_warps = w; }
    if (const char *s = getenv("UALM_TP_PROFILE")) e->prof = atoi(s) != 0;
    if (const char *s = getenv("UALM_TP_SUBGROUPS")) e->sg = std::min(TP_SUBGROUPS, std::max(1, atoi(s)));
    memset(&e->E, 0, sizeof(e->E));
    auto failed = [&](int rc) { tp_destroy(e); return rc; };
    // group streams first and group-major, so the first groups of up to eight lanes, whose loops run side by side, are created one
    // after another: CUDA multiplexes streams onto its hardware queues (CUDA_DEVICE_MAX_CONNECTIONS, 8 by default), and a long loop
    // must not share a queue with another lane's loop (a precaution; not measured on its own)
    for (int k = 0; k < TP_SUBGROUPS; k++)
        for (int lane = 0; lane < TP_LANES; lane++) {
            const int g = lane * TP_SUBGROUPS + k;
            if (cudaStreamCreateWithFlags(&e->gstream[g], cudaStreamNonBlocking) != cudaSuccess || cudaEventCreateWithFlags(&e->gev[g], cudaEventDisableTiming) != cudaSuccess) {
                if (err) *err = "group stream creation failed";
                return failed(UALM_ENOCUDA);
            }
        }
    if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess || cudaStreamCreateWithFlags(&e->cstream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&e->capstream, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreate(&e->evA) != cudaSuccess ||
        cudaEventCreate(&e->evB) != cudaSuccess || cudaMallocHost(&e->h_remaining, sizeof(int) * TP_MAX_TICKETS) != cudaSuccess ||
        cudaMallocHost(&e->h_gloop, sizeof(GroupLoop) * TP_SUBGROUPS) != cudaSuccess) {
        if (err) *err = "throughput engine: stream / event / pinned allocation failed";
        return failed(UALM_ENOCUDA);
    }
    for (auto &l : e->lanes)
        if (cudaEventCreate(&l.ev0) != cudaSuccess || cudaEventCreate(&l.ev1) != cudaSuccess) { if (err) *err = "event creation failed"; return failed(UALM_ENOCUDA); }
    if (e->remaining.ensure(TP_MAX_TICKETS) != cudaSuccess || e->n_active.ensure(TP_NGROUPS) != cudaSuccess || e->gloop.ensure(TP_NGROUPS) != cudaSuccess) {
        if (err) *err = "allocation failed";
        return failed(UALM_ENOCUDA);
    }
    cudaMemsetAsync(e->remaining.p, 0, sizeof(int) * TP_MAX_TICKETS, e->stream);
    cudaMemsetAsync(e->n_active.p, 0, sizeof(int) * TP_NGROUPS, e->stream);
    cudaMemsetAsync(e->gloop.p, 0, sizeof(GroupLoop) * TP_NGROUPS, e->stream);
    int rc = build_tables(e, err);
    if (rc) return failed(rc);
    *out = e;
    return UALM_OK;
}

void tp_destroy(TpEngine *e)
{
    if (!e) return;
    cudaSetDevice(e->device);
    cudaDeviceSynchronize();
    if (e->prof && e->kprof.p) {
        long long h[32];
        cudaMemcpy(h, e->kprof.p, sizeof(h), cudaMemcpyDeviceToHost);
        const char *nm[KP_N] = {"finish:pre", "finish:gradient-tables", "finish:post", "advance:line-search", "advance:post-ls", "two-loop", "alm-update", "forward:pre",
                                "forward:coefficient-tables", "forward:post", "(unused)", "warps"};
        long long tot = 0;
        for (int q = 0; q < KP_WARPS; q++) tot += h[q];
        fprintf(stderr, "[ualm-tp] ka phases (SM cycles per warp-round, %lld warp-rounds):", h[KP_WARPS]);
        for (int q = 0; q < KP_WARPS; q++) fprintf(stderr, " %s %.0f (%.0f%%);", nm[q], (double)h[q] / std::max(1ll, h[KP_WARPS]), 100.0 * h[q] / std::max(1ll, tot));
        fprintf(stderr, " total %.0f\n", (double)tot / std::max(1ll, h[KP_WARPS]));
        const char *nb[7] = {"setup", "spline+stencil", "tile issue+wait", "terrain+penalties", "barrier", "reductions", "final"};
        long long tb = 0;
        for (int q = 0; q < 7; q++) tb += h[16 + q];
        fprintf(stderr, "[ualm-tp] kb phases (SM cycles of thread 0 per CTA, %lld CTAs):", h[16 + 7]);
        for (int q = 0; q < 7; q++) fprintf(stderr, " %s %.0f (%.0f%%);", nb[q], (double)h[16 + q] / std::max(1ll, h[16 + 7]), 100.0 * h[16 + q] / std::max(1ll, tb));
        fprintf(stderr, " total %.0f\n", (double)tb / std::max(1ll, h[16 + 7]));
        e->kprof.release();
    }
    for (int g = 0; g < TP_NGROUPS; g++) {
        for (auto &L : e->loops[g]) {
            if (L.exec) cudaGraphExecDestroy(L.exec);
            if (L.G) cudaGraphDestroy(L.G);
        }
        if (e->gstream[g]) cudaStreamDestroy(e->gstream[g]);
        if (e->ugstream[g]) cudaStreamDestroy(e->ugstream[g]);
        if (e->gev[g]) cudaEventDestroy(e->gev[g]);
    }
    if (e->ustream) cudaStreamDestroy(e->ustream);
    if (e->uev) cudaEventDestroy(e->uev);
    for (auto &l : e->lanes) {
        l.d_ad.release(); l.d_gd.release(); l.d_gdg.release(); l.d_x0.release(); l.d_xev.release(); l.d_cxy.release(); l.d_cyaw.release(); l.d_xout.release(); l.d_f.release(); l.d_grad.release();
        l.d_hx.release(); l.d_gx.release(); l.d_sfx.release(); l.d_scx.release(); l.d_lam.release(); l.d_mu.release(); l.d_scin.release(); l.d_sfin.release();
        l.d_offs.release(); l.d_res.release(); l.d_pub.release(); l.mbox.release(); l.d_stop.release();
        if (l.h_stop) cudaFreeHost(l.h_stop);
        if (l.ev0) cudaEventDestroy(l.ev0);
        if (l.ev1) cudaEventDestroy(l.ev1);
    }
    e->st.release(); e->active.release(); e->n_active.release(); e->remaining.release(); e->vec.release(); e->cd.release(); e->gw.release();
    e->kb_cost.release(); e->lm_ys.release(); e->lm_alpha.release(); e->cr.release(); e->gdc.release(); e->gdt.release(); e->dual.release();
    e->hs.release(); e->hy.release(); e->wway.release(); e->wf.release(); e->wt.release(); e->wf_off.release(); e->wway_off.release();
    e->gloop.release();
    if (e->h_remaining) cudaFreeHost(e->h_remaining);
    if (e->h_gloop) cudaFreeHost(e->h_gloop);
    if (e->evA) cudaEventDestroy(e->evA);
    if (e->evB) cudaEventDestroy(e->evB);
    if (e->stream) cudaStreamDestroy(e->stream);
    if (e->cstream) cudaStreamDestroy(e->cstream);
    if (e->capstream) cudaStreamDestroy(e->capstream);
    cudaStreamSynchronize(cudaStreamPerThread);      // the buffers' frees
    delete e;
}

// the pool strides are sized by the largest int_K and mem_size over the bound environments
static int max_K(const TpEngine *e)
{
    int K = 1;
    for (int v = 0; v < UALM_MAX_ENVS; v++) if (e->have_params[v]) K = std::max(K, e->p[v].int_K);
    return K;
}
static int max_m(const TpEngine *e)
{
    int m = 1;
    for (int v = 0; v < UALM_MAX_ENVS; v++) if (e->have_params[v]) m = std::max(m, e->p[v].mem_size);
    return m;
}

int tp_set_params(TpEngine *e, int env, const ualm_params_t *p, std::string *err)
{
    if (p->int_K < 1 || p->int_K > TP_KB_THREADS - 1) { if (err) *err = "int_K out of range [1,127] on the throughput path"; return UALM_ELIMIT; }
    TpParams &d = e->p[env];
    d.use_scaling = p->use_scaling; d.rho = p->rho;
    d.beta = p->beta; d.gamma = p->gamma; d.epsilon_con = p->epsilon_con; d.max_iter = p->max_iter; d.g_epsilon = p->g_epsilon;
    d.min_step = p->min_step; d.delta = p->delta; d.inner_max_iter = (int)p->inner_max_iter; d.mem_size = p->mem_size; d.past = p->past;
    d.int_K = p->int_K; d.gravity = p->gravity; d.max_evals = e->max_evals;
    e->have_params[env] = true;
    // the pool strides depend on the largest int_K and mem_size: it is rebuilt at the next admission.  The uploaded batches' sample
    // offsets depend on int_K: they are invalidated, as on the parity path (upload again)
    e->capacity = 0; e->free_slots.clear(); e->live = 0;
    for (int g = 0; g < TP_NGROUPS; g++) e->glive[g] = 0;
    for (auto &l : e->lanes) { l.collected = false; l.have_batch = false; }
    return UALM_OK;
}

void tp_set_budget(TpEngine *e, int max_evals)
{
    e->max_evals = max_evals;
    for (auto &p : e->p) p.max_evals = max_evals;
}

void tp_bind_map(TpEngine *e, int env, const ualm_map_geom_t *g, const float4 *cells)
{
    TpMap &m = e->map[env];
    m.cells = cells;
    for (int k = 0; k < 3; k++) { m.vn[k] = g->voxel_num[k]; m.origin[k] = g->origin[k]; m.maxb[k] = g->max_boundary[k]; }
    m.xy_res = g->xy_resolution; m.yaw_res = g->yaw_resolution; m.xy_inv = 1.0 / g->xy_resolution; m.yaw_inv = 1.0 / g->yaw_resolution;
    // TMA descriptor of the grid: a 3-D float tensor {4 * Yaw, Y, X} (innermost first), box = 8 yaw layers x 8 x 8 cells
    e->have_tmap[env] = false;
    memset(&e->tmap[env], 0, sizeof(e->tmap[env]));
    typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                 CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess && fn && qres == cudaDriverEntryPointSuccess) {
        const cuuint64_t dims[3] = {(cuuint64_t)4 * g->voxel_num[2], (cuuint64_t)g->voxel_num[1], (cuuint64_t)g->voxel_num[0]};
        const cuuint64_t strides[2] = {(cuuint64_t)16 * g->voxel_num[2], (cuuint64_t)16 * g->voxel_num[2] * g->voxel_num[1]};
        const cuuint32_t box[3] = {4 * TP_TILE, TP_TILE, TP_TILE};
        const cuuint32_t estr[3] = {1, 1, 1};
        const CUresult r = ((EncodeFn)fn)(&e->tmap[env], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void *)cells, dims, strides, box, estr,
                                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        e->have_tmap[env] = (r == CUDA_SUCCESS) && g->voxel_num[2] >= TP_TILE && g->voxel_num[1] >= TP_TILE && g->voxel_num[0] >= TP_TILE;
    }
    if (getenv("UALM_DEBUG"))
        fprintf(stderr, "[ualm-tp] env %d: tensor map %s, TMA staging %s\n", env, e->have_tmap[env] ? "encoded" : "unavailable", (e->have_tmap[env] && e->use_tma) ? "on" : "off");
}

// (re)allocate the pool for `cap` slots with the current parameters; only when nothing is resident
static int pool_alloc(TpEngine *e, int cap, std::string *err)
{
    const int K = max_K(e), m = max_m(e);
    const size_t Smax = (size_t)TP_NMAX * (K + 1), es = e->esz();
    TCK(e->st.ensure(cap)); TCK(e->active.ensure((size_t)cap * TP_NGROUPS));
    TCK(e->vec.ensure((size_t)cap * 5 * TP_NVAR)); TCK(e->cd.ensure((size_t)cap * TP_CSTRIDE)); TCK(e->gw.ensure((size_t)cap * TP_CSTRIDE));
    TCK(e->kb_cost.ensure(cap)); TCK(e->lm_ys.ensure((size_t)cap * m)); TCK(e->lm_alpha.ensure((size_t)cap * m));
    if (e->f32()) TCK(e->cr.ensure((size_t)cap * TP_CSTRIDE * es));
    TCK(e->gdc.ensure((size_t)cap * TP_CSTRIDE * es)); TCK(e->gdt.ensure((size_t)cap * TP_TSTRIDE * es));
    TCK(e->dual.ensure((size_t)cap * TP_NDUAL * Smax * es));
    TCK(e->hs.ensure((size_t)cap * m * TP_NVAR * es)); TCK(e->hy.ensure((size_t)cap * m * TP_NVAR * es));
    TCK(cudaMemsetAsync(e->st.p, 0, sizeof(TpState) * cap, e->stream));     // every slot PH_FREE
    TCK(cudaMemsetAsync(e->n_active.p, 0, sizeof(int) * TP_NGROUPS, e->stream));
    TCK(cudaStreamSynchronize(e->stream));
    TpPool &E = e->E;
    E.capacity = cap; E.m = m; E.K = K; E.Smax = (int)Smax; E.use_tma = e->use_tma;
    E.st = e->st.p; E.active = e->active.p; E.n_active = e->n_active.p; E.remaining = e->remaining.p;
    E.vec = e->vec.p; E.cd = e->cd.p; E.gw = e->gw.p; E.cr = e->f32() ? (void *)e->cr.p : (void *)e->cd.p; E.gdc = e->gdc.p; E.gdt = e->gdt.p;
    E.kb_cost = e->kb_cost.p; E.dual = e->dual.p; E.hs = e->hs.p; E.hy = e->hy.p; E.lm_ys = e->lm_ys.p; E.lm_alpha = e->lm_alpha.p;
    E.wf = e->wf.p; E.wf_off = e->wf_off.p; E.wt = e->wt.p; E.wway = e->wway.p; E.wway_off = e->wway_off.p;
    E.prof = nullptr;
    if (e->prof) { TCK(e->kprof.ensure(32)); TCK(cudaMemsetAsync(e->kprof.p, 0, 32 * sizeof(long long), e->stream)); E.prof = e->kprof.p; }
    e->capacity = cap;
    e->free_slots.clear();
    for (int s = cap - 1; s >= 0; s--) e->free_slots.push_back(s);
    e->live = 0;
    for (int g = 0; g < TP_NGROUPS; g++) e->glive[g] = 0;
    if (getenv("UALM_DEBUG")) fprintf(stderr, "[ualm-tp] pool of %d slots allocated (%.2f MB per slot)\n", cap,
                                      (double)((size_t)5 * TP_NVAR * 8 + 3 * TP_CSTRIDE * 8 + TP_NDUAL * Smax * es + 2 * (size_t)m * TP_NVAR * es) / 1e6);
    return UALM_OK;
}

int tp_upload(TpEngine *e, int lane, const BatchLayout &L, const double *bnd, const double *total_time, std::string *err)
{
    TpLane &l = e->lanes[lane];
    l.have_batch = false; l.collected = false; l.lay = &L;
    TCK(cudaSetDevice(e->device));
    const int B = L.B;
    l.ad.assign(B, AdmitDesc()); l.gd.assign(B, GatherDesc());
    for (int b = 0; b < B; b++) {
        AdmitDesc &a = l.ad[b];
        GatherDesc &g = l.gd[b];
        a.slot = -1; a.N = L.N[b]; a.M = L.M[b]; a.ticket = lane; a.index = b; a.mode = L.skip[b] ? -1 : 0; a.off_x = L.off_x[b]; a.total_time = total_time[b];
        for (int k = 0; k < 18; k++) a.bnd[k] = bnd[(size_t)b * 18 + k];
        for (int k = 0; k < 8; k++) a.pp[k] = L.pp[8 * (size_t)b + k];
        g.slot = -1; g.N = L.N[b]; g.M = L.M[b]; g.off_cxy = L.off_cxy[b]; g.off_cyaw = L.off_cyaw[b]; g.off_x = L.off_x[b]; g.off_s = L.off_s[b];
    }
    TCK(l.d_ad.ensure(B)); TCK(l.d_gd.ensure(B)); TCK(l.d_x0.ensure(L.tot_x)); TCK(l.d_cxy.ensure(L.tot_cxy)); TCK(l.d_cyaw.ensure(L.tot_cyaw));
    TCK(l.d_res.ensure(B)); TCK(l.d_offs.ensure(B));
    if (L.tot_x > 0) {
        TCK(cudaMemcpyAsync(l.d_x0.p, L.x0.data(), sizeof(double) * L.tot_x, cudaMemcpyHostToDevice, e->stream));
        TCK(cudaStreamSynchronize(e->stream));
    }
    l.have_batch = true; l.mode = 0;
    return UALM_OK;
}

static int start_loops(TpEngine *e, int lane, bool publish, std::string *err, bool urgent = false);

// admission of the lane's uploaded batch into the pool; loops: launch its groups' round loops (tp_time_penalty launches them itself
// after its own rounds)
static int admit_impl(TpEngine *e, int lane, int mode, bool single_group, bool publish, bool loops, std::string *err, bool urgent = false)
{
    TpLane &l = e->lanes[lane];
    if (!l.have_batch) { if (err) *err = "set_params, set_map and upload must precede the solve"; return UALM_ESTATE; }
    if (l.in_flight) { if (err) *err = "lane already in flight"; return UALM_ESTATE; }
    const BatchLayout &L = *l.lay;
    TCK(cudaSetDevice(e->device));
    const cudaStream_t as = urgent ? e->ustream : e->stream;     // (tp_admit made ustream and ordered it after the engine's stream)
    const int need = L.n_active;
    // the pool grows only while nothing is resident; it is sized for TP_LANES batches of this size in flight (fewer when that
    // would take more than three quarters of the free device memory: 8 x 8192 float slots take ~43 GB of an 80 GB H100)
    int mult = TP_LANES;
    {
        size_t free_b = 0, total_b = 0;
        TCK(cudaMemGetInfo(&free_b, &total_b));
        const double per_slot = 5.0 * TP_NVAR * 8 + 3.0 * TP_CSTRIDE * 8 + (double)TP_NDUAL * TP_NMAX * (max_K(e) + 1) * e->esz() + 2.0 * max_m(e) * TP_NVAR * e->esz();
        while (mult > 1 && per_slot * mult * need > 0.75 * free_b) mult /= 2;
    }
    if (e->live == 0 && e->capacity < mult * need) {
        int cap = std::max(1024, e->capacity);
        while (cap < mult * need) cap *= 2;
        if (const char *s = getenv("UALM_TP_CAPACITY")) cap = std::max(cap, atoi(s));
        int rc = pool_alloc(e, cap, err);
        if (rc) return rc;
    }
    if ((int)e->free_slots.size() < need) { if (err) *err = "throughput pool exhausted: collect a batch in flight first (the pool grows only when idle)"; return UALM_ELIMIT; }
    // the lane's stop words: no request of its previous batch carries over (nothing raises them while the lane is not in flight, and
    // the raises of its previous batch were complete when that batch was collected)
    {
        const size_t nw = (size_t)std::max(L.B, 1);
        TCK(l.d_stop.ensure(nw));
        if (l.h_stop_cap < nw) {         // (in powers of two: freeing pinned memory waits for the device)
            size_t c = 1024;
            while (c < nw) c *= 2;
            if (l.h_stop) cudaFreeHost(l.h_stop);
            l.h_stop = nullptr; l.h_stop_cap = 0;
            TCK(cudaMallocHost(&l.h_stop, sizeof(int) * c));
            l.h_stop_cap = c;
        }
        memset(l.h_stop, 0, sizeof(int) * l.h_stop_cap);
        TCK(cudaMemsetAsync(l.d_stop.p, 0, sizeof(int) * nw, as));
        e->E.stop[lane] = l.d_stop.p;
    }
    l.slots.clear();
    std::vector<ualm_result_t> res0(L.B);
    int k = 0;
    for (int b = 0; b < L.B; b++) {
        memset(&res0[b], 0, sizeof(ualm_result_t));
        if (L.skip[b]) { l.ad[b].slot = -1; l.gd[b].slot = -1; l.ad[b].mode = -1; res0[b].ret_code = UALM_ELIMIT; continue; }
        const int s = e->free_slots.back();
        e->free_slots.pop_back();
        l.slots.push_back(s);
        // a batch of one environment is dealt over the lane's e->sg groups; in a mixed batch group k runs environment k
        const int g = lane * TP_SUBGROUPS + (L.mixed() ? L.env[b] : single_group ? 0 : k % e->sg);
        l.ad[b].slot = s; l.ad[b].mode = mode; l.ad[b].group = g; l.gd[b].slot = s;
        e->glive[g]++;
        e->genv[g] = L.env[b];
        k++;
    }
    e->live += (int)l.slots.size();
    e->Nmax_live = std::max(e->Nmax_live, L.Nmax); e->Mmax_live = std::max(e->Mmax_live, L.Mmax);
    // compact descriptors of the admitted problems only (skipped ones keep their UALM_ELIMIT record), grouped by environment: one
    // admit_kernel launch per environment, with its own use_scaling and int_K.  offs: sample offsets in the caller's dual arrays
    std::vector<AdmitDesc> ad;
    std::vector<long long> offs;
    int eoff[UALM_MAX_ENVS + 1];
    for (int v = 0; v < UALM_MAX_ENVS; v++) {
        eoff[v] = (int)ad.size();
        for (int q = L.eoff[v]; q < L.eoff[v + 1]; q++)
            if (!L.skip[L.eidx[q]]) { ad.push_back(l.ad[L.eidx[q]]); offs.push_back(L.off_s[L.eidx[q]]); }
    }
    eoff[UALM_MAX_ENVS] = (int)ad.size();
    const int BA = (int)ad.size();
    TCK(cudaEventRecord(l.ev0, as));
    l.launches = 0;
    TCK(cudaMemcpyAsync(l.d_res.p, res0.data(), sizeof(ualm_result_t) * L.B, cudaMemcpyHostToDevice, as));
    if (BA < L.B) {
        TCK(cudaMemsetAsync(l.d_cxy.p, 0, sizeof(double) * L.tot_cxy, as));
        TCK(cudaMemsetAsync(l.d_cyaw.p, 0, sizeof(double) * L.tot_cyaw, as));
    }
    if (BA > 0) {
        TCK(cudaMemcpyAsync(l.d_ad.p, ad.data(), sizeof(AdmitDesc) * BA, cudaMemcpyHostToDevice, as));
        TCK(cudaMemcpyAsync(l.d_offs.p, offs.data(), sizeof(long long) * BA, cudaMemcpyHostToDevice, as));
        TCK(cudaMemcpyAsync(l.d_gd.p, l.gd.data(), sizeof(GatherDesc) * L.B, cudaMemcpyHostToDevice, as));
        std::vector<GatherDesc> gdg;
        int ngroups = 0;
        for (int q = 0; q < TP_SUBGROUPS; q++) ngroups += e->glive[lane * TP_SUBGROUPS + q] > 0;
        if (publish && ngroups > 1) {    // per group: start_loops
            gdg.resize((size_t)TP_SUBGROUPS * L.B);
            for (int q = 0; q < TP_SUBGROUPS; q++)
                for (int b = 0; b < L.B; b++) {
                    GatherDesc &d = gdg[(size_t)q * L.B + b];
                    d = l.gd[b];
                    if (l.ad[b].slot < 0 || l.ad[b].group != lane * TP_SUBGROUPS + q) d.slot = -1;
                }
            TCK(l.d_gdg.ensure(gdg.size()));
            TCK(cudaMemcpyAsync(l.d_gdg.p, gdg.data(), sizeof(GatherDesc) * gdg.size(), cudaMemcpyHostToDevice, as));
        }
        TCK(cudaMemsetAsync(e->gloop.p + lane * TP_SUBGROUPS, 0, sizeof(GroupLoop) * TP_SUBGROUPS, as));
        e->h_remaining[lane] = BA;
        TCK(cudaMemcpyAsync(e->remaining.p + lane, e->h_remaining + lane, sizeof(int), cudaMemcpyHostToDevice, as));
        const double *x0 = l.has_xev ? l.d_xev.p : l.d_x0.p;
        const double *lam = l.has_lam ? l.d_lam.p : nullptr, *mu = l.has_mu ? l.d_mu.p : nullptr, *scx = l.has_scx ? l.d_scin.p : nullptr,
                     *sfx = l.has_sfx ? l.d_sfin.p : nullptr;
        for (int v = 0; v < UALM_MAX_ENVS; v++) {
            const int n = eoff[v + 1] - eoff[v];
            if (n == 0) continue;
            const TpParams &p = e->p[v];
            if (e->f32()) admit_kernel<float><<<n, 128, 0, as>>>(e->E, l.d_ad.p + eoff[v], x0, n, p.use_scaling, p.int_K, lam, mu, scx, sfx, l.rho_eval, l.d_offs.p + eoff[v]);
            else admit_kernel<double><<<n, 128, 0, as>>>(e->E, l.d_ad.p + eoff[v], x0, n, p.use_scaling, p.int_K, lam, mu, scx, sfx, l.rho_eval, l.d_offs.p + eoff[v]);
            TCK(cudaGetLastError());
            l.launches++;
        }
        // host-synchronised: ad / offs / res0 / gdg are stack-local staging vectors, and the lane's group loops start after the
        // admission (which also cleared the lane's stop words: a raise on the cancel stream lands after that clear)
        TCK(cudaStreamSynchronize(as));
    } else {
        e->h_remaining[lane] = 0;
        TCK(cudaStreamSynchronize(as));
    }
    l.in_flight = true; l.collected = false; l.mode = mode; l.publish = publish;
    return loops ? start_loops(e, lane, publish, err, urgent) : UALM_OK;
}

// the engine's priority stream for urgent work: *s, made at its first use
static int priority_stream(cudaStream_t *s, std::string *err)
{
    if (!*s) {
        int least = 0, greatest = 0;
        TCK(cudaDeviceGetStreamPriorityRange(&least, &greatest));
        TCK(cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, greatest));
    }
    return UALM_OK;
}

int tp_admit(TpEngine *e, int lane, std::string *err, bool publish, bool urgent)
{
    TpLane &l = e->lanes[lane];
    if (publish && l.have_batch && !l.in_flight) {      // (admit_impl refuses the other cases)
        const BatchLayout &L = *l.lay;
        TCK(cudaSetDevice(e->device));
        TCK(l.mbox.begin(L.B, L.N.data(), L.M.data(), L.skip.data()));
        TCK(l.d_pub.ensure(L.B));
        if (L.B > 0) TCK(cudaMemsetAsync(l.d_pub.p, 0, sizeof(int) * L.B, e->stream));   // ordered before admission's synchronise
    }
    if (urgent) {
        TCK(cudaSetDevice(e->device));
        if (int rc = priority_stream(&e->ustream, err)) return rc;
        if (!e->uev) TCK(cudaEventCreateWithFlags(&e->uev, cudaEventDisableTiming));
        TCK(cudaEventRecord(e->uev, e->stream));
        TCK(cudaStreamWaitEvent(e->ustream, e->uev, 0));
    }
    return admit_impl(e, lane, 0, false, publish, true, err, urgent);
}

static size_t kb_smem_bytes(TpEngine *e, bool tma)
{
    const size_t es = e->esz();
    const size_t arrays = 2 * (size_t)(TP_KB_THREADS / 32) * (TP_MAXPPC * 13 + TP_YCAP * 7) * es;      // two ChunkPart<R> tables
    const size_t coef = ((size_t)12 * e->Nmax_live + (size_t)6 * e->Mmax_live * 2 + e->Mmax_live) * es;
    return (tma ? (size_t)TP_MAXPPC * TP_TILE_BYTES : 0) + ((arrays + 15) & ~(size_t)15) + coef + 64;
}
static size_t ks_smem_bytes(TpEngine *e)
{
    const size_t es = e->esz();
    const size_t arrays = (size_t)(TP_KB_THREADS / 32) * (TP_MAXPPC * 13 + TP_YCAP * 7) * es;      // ChunkPart<R>
    const size_t coef = ((size_t)12 * e->Nmax_live * 3 + (size_t)6 * e->Mmax_live * 3 + e->Nmax_live + e->Mmax_live) * es;
    return ((arrays + 15) & ~(size_t)15) + coef + 64;
}
// ka_kernel's shared memory per warp: the C^-1 dcost/dc vector (12 N + 6 M doubles of the largest live problem), aliased by the
// right-hand sides of the forward pass and by the two-loop's history ring (TP_HRING slots x {s, y} x n elements)
static void ka_layout(TpEngine *e)
{
    const int nmax = 1 + 2 * (e->Nmax_live - 1) + (e->Mmax_live - 1);
    const int hstride = (int)(((size_t)nmax * e->esz() + 15) / 16 * 16 / e->esz());
    const size_t col = ((size_t)12 * e->Nmax_live + 6 * e->Mmax_live) * 8, hist = (((size_t)TP_HRING * 2 * hstride * e->esz()) + 15) & ~(size_t)15;
    e->E.ka_hist_bytes = (int)hist;                                             // behind the ring: 1 / ys and alpha of the two-loop (2 m doubles)
    e->E.ka_col_bytes = (int)((std::max(col, hist + 2 * (size_t)max_m(e) * 8) + 15) & ~(size_t)15);
    e->E.ka_hist_stride = hstride;
}
static size_t ka_smem_bytes(TpEngine *e) { return (size_t)e->ka_warps * e->E.ka_col_bytes; }

// one round of group g on stream st: ka -> [ks] -> kb, with the parameters, grid and TMA descriptor of the group's environment
template <class R>
static int launch_round(TpEngine *e, int g, cudaStream_t st, bool with_ks, bool tma, std::string *err)
{
    const int upper = e->glive[g], v = e->genv[g];
    ka_kernel<R><<<(upper + e->ka_warps - 1) / e->ka_warps, 32 * e->ka_warps, ka_smem_bytes(e), st>>>(e->E, e->p[v], g);
    if (with_ks) ks_kernel<R><<<upper, TP_KB_THREADS, ks_smem_bytes(e), st>>>(e->E, e->p[v], e->map[v], g);
    if (tma && e->have_tmap[v]) kb_kernel<R, true><<<upper, TP_KB_THREADS, kb_smem_bytes(e, true), st>>>(e->E, e->p[v], e->map[v], e->tmap[v], g);
    else kb_kernel<R, false><<<upper, TP_KB_THREADS, kb_smem_bytes(e, false), st>>>(e->E, e->p[v], e->map[v], e->tmap[v], g);
    TCK(cudaGetLastError());
    return UALM_OK;
}

template <class R>
static int set_attrs(TpEngine *e, std::string *err)
{
    static size_t done_kb[2][2] = {{0, 0}, {0, 0}}, done_ks[2] = {0, 0}, done_ka[2] = {0, 0};
    const int pi = sizeof(R) == 4 ? 0 : 1;
    ka_layout(e);
    const size_t a = kb_smem_bytes(e, true), b = kb_smem_bytes(e, false), c = ks_smem_bytes(e), d = ka_smem_bytes(e);
    if (a > 227 * 1024 || c > 227 * 1024 || d > 227 * 1024) { if (err) *err = "problem too large for shared memory"; return UALM_ELIMIT; }
    if (d > done_ka[pi]) { TCK(cudaFuncSetAttribute(ka_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)d)); done_ka[pi] = d; }
    if (a > done_kb[pi][1]) { TCK(cudaFuncSetAttribute(kb_kernel<R, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)a)); done_kb[pi][1] = a; }
    if (b > done_kb[pi][0]) { TCK(cudaFuncSetAttribute(kb_kernel<R, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)b)); done_kb[pi][0] = b; }
    if (c > done_ks[pi]) { TCK(cudaFuncSetAttribute(ks_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c)); done_ks[pi] = c; }
    return UALM_OK;
}

// The round loop of group g as one CUDA graph, launched on the group's stream:
//     compact -> the first round (with ks_kernel when the problems start with initScaling)
//     WHILE { chunk rounds -> compact -> [publish_kernel] -> loop_ctrl_kernel }
// The body runs at least once and repeats until the group has no trajectory left to run.  Rounds are per-trajectory lockstep steps,
// and compaction and publication only change which slots are listed and when results are copied out, so the loop computes what
// host-queued rounds compute.  Everything a kernel reads from the engine is fixed at capture: the grids by glive[g], which stays
// until the lane is collected; the pool's shared-memory layout and sizes by the maxima live now, which cover this batch; parameters
// and budget cannot change while a batch is in flight; a map grid replaced meanwhile (ualm_update_map) changes e->map only for later
// captures, and the context keeps the version captured here allocated until the lane is admitted again.  pub_gd: the descriptors
// publish_kernel walks (null: no publication)
template <class R>
static int launch_loop(TpEngine *e, int g, bool with_ks, const GatherDesc *pub_gd, int *launches, std::string *err, bool urgent)
{
    TpLane &l = e->lanes[g / TP_SUBGROUPS];
    TpEngine::Loop &L = e->loops[g][(with_ks ? 2 : 0) + (pub_gd ? 1 : 0)];
    cudaStream_t cs = e->capstream;
    const bool tma = e->use_tma;          // (for the environments whose grid has a tensor map)
    const int body_launches = 2 * e->chunk + 2 + (pub_gd ? 1 : 0);
    int rc = UALM_OK;
    auto check = [&](cudaError_t ce, const char *what) {
        if (ce != cudaSuccess && rc == UALM_OK) { if (err) *err = std::string(what) + ": " + cudaGetErrorString(ce); rc = UALM_ENOCUDA; }
        return rc == UALM_OK;
    };
    auto clear = [&](cudaGraph_t G, cudaGraphNode_t keep) {         // every node of G but `keep`
        size_t n = 0;
        if (!check(cudaGraphGetNodes(G, nullptr, &n), "cudaGraphGetNodes")) return false;
        std::vector<cudaGraphNode_t> nodes(n);
        if (n && !check(cudaGraphGetNodes(G, nodes.data(), &n), "cudaGraphGetNodes")) return false;
        for (cudaGraphNode_t v : nodes)
            if (v != keep && !check(cudaGraphDestroyNode(v), "cudaGraphDestroyNode")) return false;
        return true;
    };
    if (!L.G) {
        cudaGraphNodeParams cp = {};
        cp.type = cudaGraphNodeTypeConditional;
        cp.conditional.type = cudaGraphCondTypeWhile;
        cp.conditional.size = 1;
        if (!check(cudaGraphCreate(&L.G, 0), "cudaGraphCreate") ||
            !check(cudaGraphConditionalHandleCreate(&L.h, L.G, 1, cudaGraphCondAssignDefault), "cudaGraphConditionalHandleCreate"))
            return rc;
        cp.conditional.handle = L.h;
        if (!check(cudaGraphAddNode(&L.cond, L.G, nullptr, 0, &cp), "cudaGraphAddNode(conditional)")) return rc;
        L.body = cp.conditional.phGraph_out[0];
    } else if (!clear(L.G, L.cond) || !clear(L.body, nullptr)) {
        return rc;
    }
    // prologue, then the edge from its last node to the conditional node
    std::vector<cudaGraphNode_t> tail;
    if (!check(cudaStreamBeginCaptureToGraph(cs, L.G, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal), "cudaStreamBeginCaptureToGraph")) return rc;
    compact_kernel<<<1, 1024, 0, cs>>>(e->E, e->capacity, g);
    rc = launch_round<R>(e, g, cs, with_ks, tma, err);
    {
        cudaStreamCaptureStatus cst;
        const cudaGraphNode_t *deps = nullptr;
        size_t nd = 0;
        if (check(cudaStreamGetCaptureInfo(cs, &cst, nullptr, nullptr, &deps, &nd), "cudaStreamGetCaptureInfo")) tail.assign(deps, deps + nd);
    }
    cudaGraph_t captured = nullptr;
    check(cudaStreamEndCapture(cs, &captured), "cudaStreamEndCapture");
    for (cudaGraphNode_t v : tail)
        if (!check(cudaGraphAddDependencies(L.G, &v, &L.cond, 1), "cudaGraphAddDependencies")) break;
    if (rc) return rc;
    // body
    if (!check(cudaStreamBeginCaptureToGraph(cs, L.body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal), "cudaStreamBeginCaptureToGraph")) return rc;
    for (int r = 0; r < e->chunk && rc == UALM_OK; r++) rc = launch_round<R>(e, g, cs, false, tma, err);
    if (rc == UALM_OK) {
        compact_kernel<<<1, 1024, 0, cs>>>(e->E, e->capacity, g);
        if (pub_gd) publish_kernel<R><<<l.lay->B, 128, 0, cs>>>(e->E, pub_gd, l.lay->B, l.d_pub.p, l.mbox.device());
        loop_ctrl_kernel<<<1, 1, 0, cs>>>(L.h, e->n_active.p, e->gloop.p, g, e->chunk, body_launches);
        check(cudaGetLastError(), "loop body launch");
    }
    check(cudaStreamEndCapture(cs, &captured), "cudaStreamEndCapture");
    if (rc) return rc;
    // the same graph with new kernel arguments and grids: updated in place (the previous batch of this group has finished)
    if (L.exec) {
        cudaGraphExecUpdateResultInfo info;
        if (cudaGraphExecUpdate(L.exec, L.G, &info) != cudaSuccess) {
            cudaGetLastError();
            cudaGraphExecDestroy(L.exec);
            L.exec = nullptr;
            if (getenv("UALM_DEBUG")) fprintf(stderr, "[ualm-tp] group %d: loop graph re-instantiated (update result %d)\n", g, (int)info.result);
        }
    }
    if (!L.exec && !check(cudaGraphInstantiate(&L.exec, L.G, 0), "cudaGraphInstantiate")) return rc;
    // an urgent ticket's loop: on the group's priority stream, between two joins with the group's stream (the graph's kernel nodes
    // take the priority of the stream it is launched into)
    cudaStream_t ls = e->gstream[g];
    if (urgent) {
        if (int prc = priority_stream(&e->ugstream[g], err)) return prc;
        if (!check(cudaEventRecord(e->gev[g], e->gstream[g]), "cudaEventRecord") || !check(cudaStreamWaitEvent(e->ugstream[g], e->gev[g], 0), "cudaStreamWaitEvent"))
            return rc;
        ls = e->ugstream[g];
    }
    if (check(cudaGraphLaunch(L.exec, ls), "cudaGraphLaunch")) *launches += 3 + (with_ks ? 1 : 0);   // the prologue's; loop_ctrl_kernel counts the body's
    if (urgent && rc == UALM_OK && check(cudaEventRecord(e->gev[g], ls), "cudaEventRecord")) check(cudaStreamWaitEvent(e->gstream[g], e->gev[g], 0), "cudaStreamWaitEvent");
    return rc;
}

// launch the round loop of every live group of `lane` (after its admission); publish: its problems go to the mailbox as they end
static int start_loops(TpEngine *e, int lane, bool publish, std::string *err, bool urgent)
{
    TpLane &l = e->lanes[lane];
    int rc = e->f32() ? set_attrs<float>(e, err) : set_attrs<double>(e, err);
    if (rc) return rc;
    int ngroups = 0;
    for (int q = 0; q < TP_SUBGROUPS; q++) ngroups += e->glive[lane * TP_SUBGROUPS + q] > 0;
    for (int q = 0; q < TP_SUBGROUPS && rc == UALM_OK; q++) {
        const int g = lane * TP_SUBGROUPS + q;
        if (e->glive[g] <= 0) continue;
        // each group publishes only its own problems: a slot of another group may be in the middle of its round
        const GatherDesc *pub = !publish ? nullptr : ngroups > 1 ? l.d_gdg.p + (size_t)q * l.lay->B : l.d_gd.p;
        const bool with_ks = (l.mode == 0 && e->p[e->genv[g]].use_scaling) || l.mode == 2;
        rc = e->f32() ? launch_loop<float>(e, g, with_ks, pub, &l.launches, err, urgent) : launch_loop<double>(e, g, with_ks, pub, &l.launches, err, urgent);
    }
    return rc;
}

// raise the stop words idx[0, n) of lane l's batch (idx = null: all B): set them in the mirror, then copy the whole mirror on the
// cancel stream, which no group loop occupies, so the copy lands while the lane's rounds run (ka_kernel's stop test takes a raise
// that lands in the middle of a round).  Admission cleared the words and synchronised before the loops started, so the copy is
// ordered after the clear; words only go from 0 to 1 while the batch runs, so the copy never lowers one
static int raise_stop(TpEngine *e, TpLane &l, int n, const int32_t *idx, std::string *err)
{
    const int B = l.lay->B;
    if (idx) for (int k = 0; k < n; k++) l.h_stop[idx[k]] = 1;
    else for (int b = 0; b < B; b++) l.h_stop[b] = 1;
    if (B > 0) TCK(cudaMemcpyAsync(l.d_stop.p, l.h_stop, sizeof(int) * B, cudaMemcpyHostToDevice, e->cstream));
    return UALM_OK;
}

int tp_cancel(TpEngine *e, int lane, int n, const int32_t *idx, std::string *err)
{
    TpLane &l = e->lanes[lane];
    if (!l.in_flight || !l.publish) { if (err) *err = "ticket is not in flight"; return UALM_ESTATE; }
    for (int k = 0; k < n; k++)
        if (idx[k] < 0 || idx[k] >= l.lay->B) { if (err) *err = "problem index out of range [0, B)"; return UALM_EINVAL; }
    if (n == 0) return UALM_OK;
    TCK(cudaSetDevice(e->device));
    return raise_stop(e, l, n, idx, err);
}

// whether the round loops of the lane's groups have all ended (a failed launch or loop is reported, not waited out)
static int loops_done(TpEngine *e, int lane, bool *done, std::string *err)
{
    *done = true;
    for (int q = 0; q < TP_SUBGROUPS; q++) {
        const cudaError_t s = cudaStreamQuery(e->gstream[lane * TP_SUBGROUPS + q]);
        if (s == cudaErrorNotReady) *done = false;
        else TCK(s);
    }
    return UALM_OK;
}

int tp_collect(TpEngine *e, int lane, std::string *err, double timeout_ms)
{
    TpLane &l = e->lanes[lane];
    if (l.collected) return UALM_OK;
    if (!l.in_flight) { if (err) *err = "nothing in flight on this lane"; return UALM_ESTATE; }
    const BatchLayout &L = *l.lay;
    TCK(cudaSetDevice(e->device));
    if (timeout_ms >= 0.0) {
        // deadline: yield-poll the lane's loops until it has passed, then raise every stop word of the batch and let the loops drain
        // (every trajectory still running stops at its next stop test)
        const auto t0 = std::chrono::steady_clock::now();
        while (true) {
            bool done = false;
            if (int rc = loops_done(e, lane, &done, err)) return rc;
            if (done) break;
            if (std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() >= timeout_ms) {
                if (int rc = raise_stop(e, l, 0, nullptr, err)) return rc;
                break;
            }
            std::this_thread::yield();
        }
    }
    for (int q = 0; q < TP_SUBGROUPS; q++) TCK(cudaStreamSynchronize(e->gstream[lane * TP_SUBGROUPS + q]));
    // a raise the batch outran may still be queued: it lands before the lane's next clear, and the mirror is free again
    TCK(cudaStreamSynchronize(e->cstream));
    TCK(cudaMemcpyAsync(e->h_gloop, e->gloop.p + lane * TP_SUBGROUPS, sizeof(GroupLoop) * TP_SUBGROUPS, cudaMemcpyDeviceToHost, e->stream));
    TCK(cudaStreamSynchronize(e->stream));
    for (int q = 0; q < TP_SUBGROUPS; q++) {
        if (e->h_gloop[q].err) { if (err) *err = "throughput engine: a trajectory did not terminate"; return UALM_ENOCUDA; }
        l.launches += e->h_gloop[q].launches;
    }
    // gather the batch's results into the lane's packed device outputs, free its slots
    const bool ev = l.mode != 0;
    if (L.B > 0 && !l.slots.empty()) {
        if (ev) {
            TCK(l.d_f.ensure(L.B)); TCK(l.d_grad.ensure(L.tot_x)); TCK(l.d_hx.ensure(L.tot_s)); TCK(l.d_gx.ensure(6 * L.tot_s)); TCK(l.d_sfx.ensure(L.B));
            TCK(l.d_scx.ensure(7 * L.tot_s));
        }
        TCK(l.d_xout.ensure(L.tot_x));
#define GATHER(R)                                                                                                                                          \
        gather_kernel<R><<<L.B, 128, 0, e->stream>>>(e->E, l.d_gd.p, L.B, l.d_res.p, l.d_cxy.p, l.d_cyaw.p, l.d_xout.p, ev ? l.d_f.p : nullptr,            \
                                                     ev ? l.d_grad.p : nullptr, ev ? l.d_hx.p : nullptr, ev ? l.d_gx.p : nullptr, ev ? l.d_sfx.p : nullptr,    \
                                                     ev ? l.d_scx.p : nullptr)
        if (e->f32()) GATHER(float); else GATHER(double);
#undef GATHER
        TCK(cudaGetLastError());
        free_kernel<<<(L.B + 127) / 128, 128, 0, e->stream>>>(e->E, l.d_gd.p, L.B);
        TCK(cudaGetLastError());
        l.launches += 2;
    }
    TCK(cudaEventRecord(l.ev1, e->stream));
    TCK(cudaStreamSynchronize(e->stream));
    for (int s : l.slots) e->free_slots.push_back(s);
    e->live -= (int)l.slots.size();
    l.slots.clear();
    for (int q = 0; q < TP_SUBGROUPS; q++) e->glive[lane * TP_SUBGROUPS + q] = 0;
    l.in_flight = false; l.collected = true; l.publish = false;
    return UALM_OK;
}

int tp_poll(TpEngine *e, int lane, double wait_ms, int32_t *idx, int *n_new, int *n_pending, ualm_result_t *results, double *c_xy, double *c_yaw,
            std::string *err)
{
    TpLane &l = e->lanes[lane];
    if (!l.in_flight || !l.publish) { if (err) *err = "ticket is not in flight"; return UALM_ESTATE; }
    TCK(cudaSetDevice(e->device));
    const auto t0 = std::chrono::steady_clock::now();
    int n = 0;
    while (true) {
        n = l.mbox.collect(idx, results, c_xy, c_yaw);       // the group loops publish into the mailbox as problems finish
        if (n > 0 || l.mbox.pending() == 0 || wait_ms == 0.0) break;
        bool done = false;
        if (int rc = loops_done(e, lane, &done, err)) return rc;
        if (std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() >= wait_ms) break;
        std::this_thread::yield();
    }
    *n_new = n;
    *n_pending = l.mbox.pending();
    return UALM_OK;
}

int tp_download(TpEngine *e, int lane, ualm_result_t *results, double *c_xy, double *c_yaw, std::string *err)
{
    TpLane &l = e->lanes[lane];
    if (!l.collected) { int rc = tp_collect(e, lane, err); if (rc) return rc; }
    const BatchLayout &L = *l.lay;
    TCK(cudaSetDevice(e->device));
    if (L.B > 0) {
        if (results) TCK(cudaMemcpyAsync(results, l.d_res.p, sizeof(ualm_result_t) * L.B, cudaMemcpyDeviceToHost, e->stream));
        if (c_xy) TCK(cudaMemcpyAsync(c_xy, l.d_cxy.p, sizeof(double) * L.tot_cxy, cudaMemcpyDeviceToHost, e->stream));
        if (c_yaw) TCK(cudaMemcpyAsync(c_yaw, l.d_cyaw.p, sizeof(double) * L.tot_cyaw, cudaMemcpyDeviceToHost, e->stream));
    }
    TCK(cudaStreamSynchronize(e->stream));
    return UALM_OK;
}

__global__ void tp_pack_records_kernel(const ualm_result_t *res, const GatherDesc *gd, const double *c_xy, const double *c_yaw, int B, double *rec, int stride)
{
    const int b = blockIdx.x;
    if (b >= B) return;
    const GatherDesc g = gd[b];
    double *o = rec + (size_t)b * stride;
    const ualm_result_t r = res[b];
    if (threadIdx.x == 0) {
        o[0] = r.ret_code; o[1] = r.outer_iters; o[2] = r.n_evals; o[3] = r.n_lbfgs_iters; o[4] = r.inner_cost; o[5] = r.jerk_cost;
        o[6] = r.total_T; o[7] = r.res_h; o[8] = r.res_g; o[9] = g.N; o[10] = g.M; o[11] = 0.0;
    }
    const int ncx = 12 * g.N, ncy = 6 * g.M;
    for (int q = threadIdx.x; q < stride - 12; q += blockDim.x) {
        double v = 0.0;
        if (q < ncx) v = c_xy[g.off_cxy + q];
        else if (q < ncx + ncy) v = c_yaw[g.off_cyaw + q - ncx];
        o[12 + q] = v;
    }
}

int tp_pack_records(TpEngine *e, int lane, double *d_records, int stride, std::string *err)
{
    TpLane &l = e->lanes[lane];
    if (!l.collected) { int rc = tp_collect(e, lane, err); if (rc) return rc; }
    const BatchLayout &L = *l.lay;
    if (stride < 12 + 12 * L.Nmax + 6 * L.Mmax) { if (err) *err = "record stride too small"; return UALM_EINVAL; }
    if (L.B > 0) {
        tp_pack_records_kernel<<<L.B, 128, 0, e->stream>>>(l.d_res.p, l.d_gd.p, l.d_cxy.p, l.d_cyaw.p, L.B, d_records, stride);
        TCK(cudaGetLastError());
    }
    TCK(cudaStreamSynchronize(e->stream));
    return UALM_OK;
}

bool tp_lane_in_flight(TpEngine *e, int lane) { return e->lanes[lane].in_flight; }
bool tp_lane_collected(TpEngine *e, int lane) { return e->lanes[lane].collected; }

int tp_last_solve(TpEngine *e, int lane, float *ms, int *launches)
{
    TpLane &l = e->lanes[lane];
    if (!l.collected) return UALM_ESTATE;
    float t = 0.f;
    cudaEventElapsedTime(&t, l.ev0, l.ev1);
    if (ms) *ms = t;
    if (launches) *launches = l.launches;
    return UALM_OK;
}

int tp_mark_begin(TpEngine *e, std::string *err)
{
    TCK(cudaSetDevice(e->device));
    TCK(cudaEventRecord(e->evA, e->stream));
    return UALM_OK;
}
int tp_mark_end(TpEngine *e, float *ms, std::string *err)
{
    TCK(cudaSetDevice(e->device));
    for (int g = 0; g < TP_NGROUPS; g++) { TCK(cudaEventRecord(e->gev[g], e->gstream[g])); TCK(cudaStreamWaitEvent(e->stream, e->gev[g], 0)); }
    TCK(cudaEventRecord(e->evB, e->stream));
    TCK(cudaEventSynchronize(e->evB));
    TCK(cudaEventElapsedTime(ms, e->evA, e->evB));
    return UALM_OK;
}

static int put(TpEngine *e, Buf<double> &dst, const double *src, size_t n, bool &has, std::string *err)
{
    has = src != nullptr;
    if (!src || n == 0) return UALM_OK;
    TCK(dst.ensure(n));
    TCK(cudaMemcpyAsync(dst.p, src, n * sizeof(double), cudaMemcpyHostToDevice, e->stream));
    return UALM_OK;
}

int tp_eval(TpEngine *e, int lane, const double *x, const double *lambda, const double *mu, const double *scale_cx, const double *scale_fx, double rho,
            double *f, double *grad, double *hx, double *gx, double *c_xy, double *c_yaw, std::string *err)
{
    TpLane &l = e->lanes[lane];
    if (!l.have_batch) { if (err) *err = "upload and set_map first"; return UALM_ESTATE; }
    const BatchLayout &L = *l.lay;
    if (L.n_active != L.B) { if (err) *err = "batch holds problems over the compiled limits"; return UALM_ELIMIT; }
    TCK(cudaSetDevice(e->device));
    // the evaluation point goes to its own buffer: d_x0 keeps the uploaded initial guesses, which ualm_init_scaling_batch and a
    // later solve of the resident batch start from
    const bool xev = x && L.tot_x > 0;
    if (xev) {
        TCK(l.d_xev.ensure(L.tot_x));
        TCK(cudaMemcpyAsync(l.d_xev.p, x, sizeof(double) * L.tot_x, cudaMemcpyHostToDevice, e->stream));
    }
    int rc;
    if ((rc = put(e, l.d_lam, lambda, L.tot_s, l.has_lam, err))) return rc;
    if ((rc = put(e, l.d_mu, mu, 6 * L.tot_s, l.has_mu, err))) return rc;
    if ((rc = put(e, l.d_scin, scale_cx, 7 * L.tot_s, l.has_scx, err))) return rc;
    if ((rc = put(e, l.d_sfin, scale_fx, L.B, l.has_sfx, err))) return rc;
    l.rho_eval = rho;
    l.has_xev = xev;
    rc = admit_impl(e, lane, 1, false, false, true, err);
    l.has_lam = l.has_mu = l.has_scx = l.has_sfx = l.has_xev = false;
    if (rc) return rc;
    if ((rc = tp_collect(e, lane, err))) return rc;
    if (L.B > 0) {
        if (f) TCK(cudaMemcpyAsync(f, l.d_f.p, sizeof(double) * L.B, cudaMemcpyDeviceToHost, e->stream));
        if (grad) TCK(cudaMemcpyAsync(grad, l.d_grad.p, sizeof(double) * L.tot_x, cudaMemcpyDeviceToHost, e->stream));
        if (hx) TCK(cudaMemcpyAsync(hx, l.d_hx.p, sizeof(double) * L.tot_s, cudaMemcpyDeviceToHost, e->stream));
        if (gx) TCK(cudaMemcpyAsync(gx, l.d_gx.p, sizeof(double) * 6 * L.tot_s, cudaMemcpyDeviceToHost, e->stream));
        if (c_xy) TCK(cudaMemcpyAsync(c_xy, l.d_cxy.p, sizeof(double) * L.tot_cxy, cudaMemcpyDeviceToHost, e->stream));
        if (c_yaw) TCK(cudaMemcpyAsync(c_yaw, l.d_cyaw.p, sizeof(double) * L.tot_cyaw, cudaMemcpyDeviceToHost, e->stream));
    }
    TCK(cudaStreamSynchronize(e->stream));
    l.collected = false;           // the lane holds evaluation outputs, not a solve
    return UALM_OK;
}

int tp_init_scaling(TpEngine *e, int lane, double *scale_fx, double *scale_cx, std::string *err)
{
    TpLane &l = e->lanes[lane];
    if (!l.have_batch) { if (err) *err = "upload and set_map first"; return UALM_ESTATE; }
    const BatchLayout &L = *l.lay;
    if (L.n_active != L.B) { if (err) *err = "batch holds problems over the compiled limits"; return UALM_ELIMIT; }
    TCK(cudaSetDevice(e->device));
    int rc = admit_impl(e, lane, 2, false, false, true, err);
    if (rc) return rc;
    if ((rc = tp_collect(e, lane, err))) return rc;
    if (L.B > 0) {
        if (scale_fx) TCK(cudaMemcpyAsync(scale_fx, l.d_sfx.p, sizeof(double) * L.B, cudaMemcpyDeviceToHost, e->stream));
        if (scale_cx) TCK(cudaMemcpyAsync(scale_cx, l.d_scx.p, sizeof(double) * 7 * L.tot_s, cudaMemcpyDeviceToHost, e->stream));
    }
    TCK(cudaStreamSynchronize(e->stream));
    l.collected = false;
    return UALM_OK;
}

int tp_time_penalty(TpEngine *e, int lane, int reps, int use_tma, float *ms_per_launch, double *algorithmic_bytes, std::string *err)
{
    TpLane &l = e->lanes[lane];
    if (!l.have_batch) { if (err) *err = "upload and set_map first"; return UALM_ESTATE; }
    const BatchLayout &L = *l.lay;
    if (L.mixed()) { if (err) *err = "ualm_time_penalty_kernel: the uploaded batch mixes environments"; return UALM_EINVAL; }
    if (l.in_flight || e->live > 0) { if (err) *err = "ualm_time_penalty_kernel needs an idle pool"; return UALM_ESTATE; }
    if (ms_per_launch) *ms_per_launch = 0.f;
    if (algorithmic_bytes) *algorithmic_bytes = 0.0;
    if (L.B == 0) return UALM_OK;
    TCK(cudaSetDevice(e->device));
    const int v = L.env[0];
    // admit as single evaluations (initial guess, zero duals, unit scales), run the forward half of a round, then time kb alone
    l.has_lam = l.has_mu = l.has_scx = l.has_sfx = false; l.rho_eval = e->p[v].rho;
    int rc = admit_impl(e, lane, 1, true, false, false, err);
    if (rc) return rc;
    rc = e->f32() ? set_attrs<float>(e, err) : set_attrs<double>(e, err);
    if (rc) return rc;
    const int g = lane * TP_SUBGROUPS;
    cudaStream_t st = e->gstream[g];
    compact_kernel<<<1, 1024, 0, st>>>(e->E, e->capacity, g);
    const int upper = e->glive[g];
    const bool tma = e->have_tmap[v] && use_tma;
    if (e->f32()) ka_kernel<float><<<(upper + e->ka_warps - 1) / e->ka_warps, 32 * e->ka_warps, ka_smem_bytes(e), st>>>(e->E, e->p[v], g);
    else ka_kernel<double><<<(upper + e->ka_warps - 1) / e->ka_warps, 32 * e->ka_warps, ka_smem_bytes(e), st>>>(e->E, e->p[v], g);
    auto kb = [&]() {
        if (e->f32()) {
            if (tma) kb_kernel<float, true><<<upper, TP_KB_THREADS, kb_smem_bytes(e, true), st>>>(e->E, e->p[v], e->map[v], e->tmap[v], g);
            else kb_kernel<float, false><<<upper, TP_KB_THREADS, kb_smem_bytes(e, false), st>>>(e->E, e->p[v], e->map[v], e->tmap[v], g);
        } else {
            if (tma) kb_kernel<double, true><<<upper, TP_KB_THREADS, kb_smem_bytes(e, true), st>>>(e->E, e->p[v], e->map[v], e->tmap[v], g);
            else kb_kernel<double, false><<<upper, TP_KB_THREADS, kb_smem_bytes(e, false), st>>>(e->E, e->p[v], e->map[v], e->tmap[v], g);
        }
    };
    kb();    // warm-up
    TCK(cudaEventRecord(e->evA, st));
    for (int r = 0; r < reps; r++) kb();
    TCK(cudaEventRecord(e->evB, st));
    TCK(cudaGetLastError());
    TCK(cudaEventSynchronize(e->evB));
    float ms = 0.f;
    TCK(cudaEventElapsedTime(&ms, e->evA, e->evB));
    if (ms_per_launch) *ms_per_launch = ms / reps;
    if (algorithmic_bytes) {
        // SURVEY 8d: per trajectory per evaluation S * 45 e + (25 N + 13 M) e, e = element size of the sample data
        double bytes = 0;
        const double es = (double)e->esz();
        for (int b = 0; b < L.B; b++) bytes += (double)L.N[b] * (e->p[v].int_K + 1) * 45 * es + (25.0 * L.N[b] + 13.0 * L.M[b]) * es;
        *algorithmic_bytes = bytes;
    }
    // finish the evaluations (the group's loop, queued behind the timed launches) and release the slots
    rc = start_loops(e, lane, false, err);
    if (rc == UALM_OK) rc = tp_collect(e, lane, err);
    l.collected = false;
    return rc;
}

int tp_lane_outputs(TpEngine *e, int lane, const ualm_result_t **d_res, const double **d_cxy, const double **d_cyaw)
{
    TpLane &l = e->lanes[lane];
    if (!l.collected) return UALM_ESTATE;
    *d_res = l.d_res.p; *d_cxy = l.d_cxy.p; *d_cyaw = l.d_cyaw.p;
    return UALM_OK;
}

} // namespace ualm_tp
