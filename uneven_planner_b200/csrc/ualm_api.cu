// ualm_api.cu -- the extern "C" layer declared in include/ualm.h: context, uploads, kernel launches.
// Host code is thin: it packs descriptors, sizes shared memory from the batch maxima and launches the
// per-trajectory kernels of ualm_kernels.cuh.  There is NO CPU fallback: every compute entry point needs a CUDA
// device and returns UALM_ENOCUDA otherwise.
#include "ualm_kernels.cuh"
#include "map_prep.h"
#include "ualm_tp_host.h"

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <numeric>
#include <string>
#include <thread>
#include <vector>

using namespace ualm;

static thread_local std::string g_err;
static int fail(int code, const std::string &msg)
{
    g_err = msg;
    return code;
}
#define CK(call)                                                                                             \
    do {                                                                                                     \
        cudaError_t e_ = (call);                                                                             \
        if (e_ != cudaSuccess) return fail(UALM_ENOCUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
    } while (0)

template <class T>
struct DevBuf {
    T *p = nullptr;
    size_t cap = 0;
    cudaError_t ensure(size_t n)
    {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        cudaError_t e = cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T));
        if (e == cudaSuccess) cap = n;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

// One version of an environment's map grid: its device buffer ([X][Y][Yaw] float4, or 4 doubles per cell from ualm_set_map_f64) and
// the DevMap that points into it.  The environment holds its current version, and every lane holds the versions its last launch read
// until its next launch or its release, so ualm_update_map* never changes a grid that queued work or a later scan of that work reads.
// The buffer is freed on the context's free stream, which waits for the completion of every lane that let go of a version (lane_hold),
// so the last holder's release frees it without a host or device-wide wait.
struct MapVer {
    cudaStream_t fs = nullptr;
    void *p = nullptr;
    size_t bytes = 0;
    DevMap dm = {};
    ualm_map_geom_t geom = {};           // the geometry dm was set from (the geometry of a ualm_update_map_window* copy)
    ~MapVer() { if (p) cudaFreeAsync(p, fs); }
};
typedef std::shared_ptr<MapVer> MapRef;

// One in-flight batch ("lane"): its own device buffers, launch plan, streams and events.  A context owns up to UALM_MAX_LANES of
// them so that several batches can be resident and running at once (the stragglers of batch k drain while batch k+1 fills the
// SMs they left: ualm_submit_batch / ualm_wait_batch, or ualm_select_lane + the three-step calls).
#define UALM_MAX_LANES 16
struct Lane {
    bool made = false;
    cudaStream_t stream = nullptr, own_stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    bool have_batch = false, solved = false, in_flight = false;
    // the lane's uploaded batch, on both paths (the throughput engine reads it too: tp_upload)
    BatchLayout batch;
    std::vector<ProbDesc> desc;
    std::vector<int> order;              // launch order over the ACTIVE problems (largest first)
    // the one-warp-per-problem kernels run once per environment present, over its slice of d_eidx (batch.eidx)
    DevBuf<int> d_eidx;
    SmemLayout eL[UALM_MAX_ENVS];        // their layouts (maxima over the environment's problems)
    size_t esmem[UALM_MAX_ENVS] = {};    // dynamic shared memory of one of their CTAs: ewpb slots of eL
    int ewpb[UALM_MAX_ENVS] = {};        // their warps per CTA
    long long tot_hist = 0, tot_scr = 0, tot_fac = 0, tot_ws = 0;
    DevBuf<ProbDesc> d_desc;
    DevBuf<int> d_order;
    std::vector<int> group;      // warps per problem (1, 2 or 4)
    // one solve launch: the problems order[r0, r1) of one group size and one environment, taken from a work queue by grid CTAs
    struct GClass { int G = 1, n_ctas = 0, grid = 0, r0 = 0, r1 = 0, occ = 1, env = 0; size_t smem = 0; SmemLayout L; };
    std::vector<GClass> cls;
    DevBuf<int> d_queue;         // one work counter per launch, then the lane's three hold words (BatchPtrs::hctl); zeroed before the launches
    // each launch runs as a CUDA graph: WHILE (problems of its queue untaken) { hold_gate_kernel -> solve_kernel -> solve_loop_ctrl_kernel }
    // (solve_loop_run), one per launch index, built at its first use and updated in place after
    struct SolveLoop { cudaGraph_t G = nullptr; cudaGraphNode_t gate = nullptr, solve = nullptr, ctrl = nullptr; cudaGraphConditionalHandle h = 0; cudaGraphExec_t exec = nullptr; };
    std::vector<SolveLoop> loops;
    std::vector<cudaGraphExec_t> retired;    // executable graphs an update could not reuse, destroyed at release
    enum { NAUX = 7 };
    cudaStream_t aux[NAUX] = {};
    cudaEvent_t evs[NAUX + 1] = {};
    // an urgent ticket's launches (ualm_set_urgent): streams of the greatest priority, made at the lane's first urgent ticket (a stream
    // made earlier changes which hardware queue every later stream shares)
    cudaStream_t ustream[NAUX + 1] = {};
    DevBuf<double> d_x0, d_x, d_xev, d_lambda, d_mu, d_scale_cx, d_hx, d_gx, d_lm_s, d_lm_y, d_lm_aux, d_fac, d_scr, d_ws, d_cxy, d_cyaw, d_f, d_grad, d_sfx;
    DevBuf<ualm_result_t> d_res;
    DevBuf<long long> d_prof;
    DevBuf<double> d_pieceT, d_feas;
    float last_ms = 0.f;
    int last_launches = 0;
    // stop words of the lane's solves, one per problem (ualm_cancel_problems, ualm_wait_batch_for), in device memory: cleared on the
    // lane stream before every solve launch (ev_clear marks that), raised while the kernels run by copying the whole pinned mirror
    // h_stop (grows only, like the mailbox) on the context's cancel stream after ev_clear.  Words only go from 0 to 1 during a batch
    // and only the host writes them, so a copy of the whole mirror never lowers a word.  (A word in mapped pinned host memory, read
    // over PCIe at every stop test, made the bench step 5 % slower on an H100 80GB HBM3 at a 400 W power limit.)
    DevBuf<int> d_stop;
    int *h_stop = nullptr;
    size_t h_stop_cap = 0;
    bool raised = false;                 // a raise copy of the batch in flight may still be queued on the cancel stream
    cudaEvent_t ev_clear = nullptr;
    ualm_mbox::Mailbox mbox;             // results of a submitted batch as its problems finish (ualm_poll_batch)
    MapRef vref[UALM_MAX_ENVS];          // the grid versions the lane's last launch read, per environment of its batch (lane_hold)
    void release()
    {
        for (auto &r : vref) r.reset();
        d_stop.release();
        if (h_stop) cudaFreeHost(h_stop);
        h_stop = nullptr; h_stop_cap = 0;
        mbox.release();
        d_desc.release(); d_order.release(); d_queue.release(); d_eidx.release();
        DevBuf<double> *bufs[] = {&d_x0, &d_x, &d_xev, &d_lambda, &d_mu, &d_scale_cx, &d_hx, &d_gx, &d_lm_s, &d_lm_y, &d_lm_aux, &d_fac,
                                  &d_scr, &d_ws, &d_cxy, &d_cyaw, &d_f, &d_grad, &d_sfx};
        for (auto *b : bufs) b->release();
        d_res.release(); d_prof.release(); d_pieceT.release(); d_feas.release();
        for (auto &g : loops) {
            if (g.exec) cudaGraphExecDestroy(g.exec);
            if (g.G) cudaGraphDestroy(g.G);
        }
        loops.clear();
        for (auto x : retired) cudaGraphExecDestroy(x);
        retired.clear();
        for (auto &s : ustream) if (s) cudaStreamDestroy(s);
        for (auto &s : ustream) s = nullptr;
        if (!made) return;
        for (int q = 0; q < NAUX; q++) if (aux[q]) cudaStreamDestroy(aux[q]);
        for (int q = 0; q < NAUX + 1; q++) if (evs[q]) cudaEventDestroy(evs[q]);
        if (ev0) cudaEventDestroy(ev0);
        if (ev1) cudaEventDestroy(ev1);
        if (ev_clear) cudaEventDestroy(ev_clear);
        if (own_stream) cudaStreamDestroy(own_stream);
        made = false;
    }
};

// One environment: a parameter set and a map grid (ualm_select_env).  The kernels take both as per-launch grid constants.
struct Env {
    bool have_params = false, have_map = false;
    ualm_params_t hp;
    DevParams dp;
    MapRef map;                          // the current grid version: what every launch from now on reads
};

struct ualm_ctx {
    int device = 0, precision = 64;
    ualm_tp::TpEngine *tp = nullptr;     // precision 32 / 65: the throughput engine (ualm_tp.cu) behind the same entry points
    Env envs[UALM_MAX_ENVS];
    int sel_env = 0;                     // the environment ualm_set_params / ualm_set_map bind (ualm_select_env)
    int max_evals = 0;                   // ualm_set_budget
    Lane lanes[UALM_MAX_LANES];
    Lane *b = nullptr;            // the selected lane (ualm_select_lane; lane 0 by default)
    int cur = 0, next_submit = 0;
    int group_mode = 1;
    bool profile = false;
    // pipeline timing (ualm_mark_begin / ualm_mark_end): events on the lanes' own streams, joined on `join`
    cudaStream_t join = nullptr;
    cudaEvent_t evA = nullptr, evB = nullptr;
    // raises of the lanes' stop words (ualm_cancel_problems, ualm_wait_batch_for): copies go through the copy engines, so they do
    // not wait for free SMs
    cudaStream_t cancel = nullptr;
    // grid versions: allocated, filled and built on `mstream`, freed on `fstream` (MapVer).  No solve runs on either, so an update
    // never waits for one, and fstream's waits for lanes never hold up an update.  They come from a memory pool of their own, so a
    // freed grid shares no pool block with other buffers and goes back to the device at the next synchronisation
    cudaStream_t mstream = nullptr, fstream = nullptr;
    cudaMemPool_t mpool = nullptr;
    // pinned staging of ualm_update_map_window*'s grid copy (map_copy_ce), allocated at the first window
    static constexpr size_t STAGE_BYTES = 8u << 20;
    void *h_stage = nullptr;
    // ualm_check_trajectories and ualm_submit_replan's build: a stream no solve occupies, at the greatest priority, so its CTAs go ahead
    // of queued lane launches when SM slots free up; cdone marks the end of a check's kernels, which the free stream waits for before the grids it read can go.
    // Both are made at the first check, not at creation: streams share the device's hardware queues in creation order, and with one
    // more stream made before the throughput engine's, its cancels right after a submit came too late (tests/test_gpu_cancel.py)
    cudaStream_t cstream = nullptr;
    cudaEvent_t cdone = nullptr;
    // their inputs and outputs: one grow-only block, allocated and replaced in stream order on cstream (a block freed at every call would
    // go back to the device at that call's synchronisation and be mapped again at the next)
    void *cbuf = nullptr;
    size_t cbuf_bytes = 0;
    // urgent work (ualm_set_urgent).  d_hold: the hold bytes the solve launches read (BatchPtrs::hold), byte q < UALM_MAX_LANES raised by
    // lane q's urgent ticket, byte UALM_MAX_LANES by an urgent check or replan build; raised and lowered by copies from h_hold = {0, 1}
    // (pinned), which need no SM
    bool urgent = false;
    unsigned char *d_hold = nullptr, *h_hold = nullptr;
};
static_assert(UALM_MAX_LANES + 1 <= UALM_HOLD_BYTES, "one hold byte per lane and one for the check stream");

static int lane_make(ualm_ctx *c, Lane &l)
{
    if (l.made) return UALM_OK;
    l.made = true;     // release() cleans up whatever was created if one of the calls below fails
    CK(cudaStreamCreateWithFlags(&l.own_stream, cudaStreamNonBlocking));
    l.stream = l.own_stream;
    for (int q = 0; q < Lane::NAUX; q++) CK(cudaStreamCreateWithFlags(&l.aux[q], cudaStreamNonBlocking));
    for (int q = 0; q < Lane::NAUX + 1; q++) CK(cudaEventCreateWithFlags(&l.evs[q], cudaEventDisableTiming));
    CK(cudaEventCreate(&l.ev0));
    CK(cudaEventCreate(&l.ev1));
    CK(cudaEventCreateWithFlags(&l.ev_clear, cudaEventDisableTiming));
    (void)c;
    return UALM_OK;
}

extern "C" const char *ualm_last_error(void) { return g_err.c_str(); }

// throughput contexts forward to the engine; its error text lands in the same thread-local message
#define TP_CALL(expr)                                  \
    do {                                               \
        std::string em_;                               \
        std::string *err = &em_;                       \
        const int rc_ = (expr);                        \
        if (rc_ != UALM_OK) g_err = em_;               \
        return rc_;                                    \
    } while (0)
#define TP_UNSUPPORTED(name) return fail(UALM_EINVAL, name " is an entry point of the parity path (precision 64) only")

extern "C" int ualm_create(ualm_ctx_t **out, int device, int precision)
{
    if (!out) return fail(UALM_EINVAL, "ctx out pointer is NULL");
    if (precision != 64 && precision != 65 && precision != 32)
        return fail(UALM_EINVAL, "precision must be 64 (bit-reproducible double), 65 (throughput path in double) or 32 (throughput path in float)");
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev <= 0) return fail(UALM_ENOCUDA, std::string("no CUDA device: ") + cudaGetErrorString(e));
    if (device < 0 || device >= ndev) return fail(UALM_EINVAL, "device ordinal out of range");
    CK(cudaSetDevice(device));
    ualm_ctx *c = new ualm_ctx();
    c->device = device; c->precision = precision;
    if (const char *e = getenv("UALM_GROUPS")) c->group_mode = atoi(e);   // 0 = one warp per trajectory everywhere (developer switch)
    c->b = &c->lanes[0];
    cudaMemPoolProps pp = {};
    pp.allocType = cudaMemAllocationTypePinned;
    pp.location.type = cudaMemLocationTypeDevice;
    pp.location.id = device;
    if (cudaStreamCreateWithFlags(&c->mstream, cudaStreamNonBlocking) != cudaSuccess || cudaStreamCreateWithFlags(&c->fstream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaMemPoolCreate(&c->mpool, &pp) != cudaSuccess) {
        ualm_destroy(c);
        return fail(UALM_ENOCUDA, "context map streams");
    }
    if (precision != 64) {
        std::string em;
        const int rc = ualm_tp::tp_create(&c->tp, device, precision, &em);
        if (rc != UALM_OK) { ualm_destroy(c); return fail(rc, em); }
        *out = c;
        return UALM_OK;
    }
    int rc = lane_make(c, c->lanes[0]);
    if (rc == UALM_OK) {
        cudaError_t e1 = cudaStreamCreateWithFlags(&c->join, cudaStreamNonBlocking);
        if (e1 == cudaSuccess) e1 = cudaStreamCreateWithFlags(&c->cancel, cudaStreamNonBlocking);
        if (e1 == cudaSuccess) e1 = cudaEventCreate(&c->evA);
        if (e1 == cudaSuccess) e1 = cudaEventCreate(&c->evB);
        if (e1 == cudaSuccess) e1 = cudaMalloc(&c->d_hold, UALM_HOLD_BYTES);
        if (e1 == cudaSuccess) e1 = cudaMemset(c->d_hold, 0, UALM_HOLD_BYTES);
        if (e1 == cudaSuccess) e1 = cudaHostAlloc(&c->h_hold, 2, cudaHostAllocDefault);
        if (e1 == cudaSuccess) { c->h_hold[0] = 0; c->h_hold[1] = 1; }
        if (e1 != cudaSuccess) rc = fail(UALM_ENOCUDA, std::string("context streams/events: ") + cudaGetErrorString(e1));
    }
    if (rc != UALM_OK) { const std::string keep = g_err; ualm_destroy(c); g_err = keep; return rc; }   // no leak on a failed create
    *out = c;
    return UALM_OK;
}

extern "C" int ualm_destroy(ualm_ctx_t *c)
{
    if (!c) return UALM_OK;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    if (c->tp) { ualm_tp::tp_destroy(c->tp); c->tp = nullptr; }
    for (auto &v : c->envs) v.map.reset();
    for (auto &l : c->lanes) l.release();
    if (c->fstream) { cudaStreamSynchronize(c->fstream); cudaStreamDestroy(c->fstream); }     // the grids' frees
    if (c->mstream) cudaStreamDestroy(c->mstream);
    if (c->mpool) cudaMemPoolDestroy(c->mpool);
    if (c->h_stage) cudaFreeHost(c->h_stage);
    if (c->cbuf) { cudaFreeAsync(c->cbuf, c->cstream); cudaStreamSynchronize(c->cstream); }
    if (c->cstream) cudaStreamDestroy(c->cstream);
    if (c->cdone) cudaEventDestroy(c->cdone);
    if (c->join) cudaStreamDestroy(c->join);
    if (c->cancel) cudaStreamDestroy(c->cancel);
    if (c->evA) cudaEventDestroy(c->evA);
    if (c->evB) cudaEventDestroy(c->evB);
    if (c->d_hold) cudaFree(c->d_hold);
    if (c->h_hold) cudaFreeHost(c->h_hold);
    delete c;
    return UALM_OK;
}

extern "C" int ualm_select_lane(ualm_ctx_t *c, int lane)
{
    if (!c) return fail(UALM_EINVAL, "null ctx");
    if (lane < 0 || lane >= UALM_MAX_LANES) return fail(UALM_EINVAL, "lane out of range [0, UALM_MAX_LANES)");
    CK(cudaSetDevice(c->device));
    if (!c->tp) {
        int rc = lane_make(c, c->lanes[lane]);
        if (rc) return rc;
    }
    c->cur = lane; c->b = &c->lanes[lane];
    return UALM_OK;
}

extern "C" int ualm_max_lanes(void) { return UALM_MAX_LANES; }

// all work of the selected lane on a caller-owned stream.  The handle is taken literally: NULL is the legacy default stream
// (what torch.cuda.current_stream().cuda_stream is when torch runs on its default stream); ualm_reset_stream restores the
// lane's own non-blocking stream.
extern "C" int ualm_set_stream(ualm_ctx_t *c, void *s)
{
    if (!c) return fail(UALM_EINVAL, "null ctx");
    if (c->tp) TP_UNSUPPORTED("ualm_set_stream");
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->b->stream));
    c->b->stream = (cudaStream_t)s;
    return UALM_OK;
}
extern "C" int ualm_reset_stream(ualm_ctx_t *c)
{
    if (!c) return fail(UALM_EINVAL, "null ctx");
    if (c->tp) return UALM_OK;
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->b->stream));
    c->b->stream = c->b->own_stream;
    return UALM_OK;
}

static bool lane_in_flight(ualm_ctx *c, int q) { return c->tp ? ualm_tp::tp_lane_in_flight(c->tp, q) : c->lanes[q].in_flight; }

// binding is refused while a batch is in flight, on the parity lanes and on the throughput engine's
static int lanes_idle(ualm_ctx *c, const char *what)
{
    for (int q = 0; q < UALM_MAX_LANES; q++)
        if (lane_in_flight(c, q))
            return fail(UALM_ESTATE, std::string(what) + " while a submitted batch is in flight (ualm_wait_batch first)");
    return UALM_OK;
}

extern "C" int ualm_set_params(ualm_ctx_t *c, const ualm_params_t *p)
{
    if (!c || !p) return fail(UALM_EINVAL, "null argument");
    if (p->int_K < 1 || p->int_K > 128) return fail(UALM_ELIMIT, "int_K out of range [1,128]");
    if (p->mem_size < 1 || p->mem_size > 1024) return fail(UALM_ELIMIT, "mem_size out of range [1,1024]");
    if (p->past < 0 || p->past > 16) return fail(UALM_ELIMIT, "past out of range [0,16]");
    if (int rc = lanes_idle(c, "ualm_set_params")) return rc;
    // the throughput engine has its own limits (int_K <= 127): the context's copy and its flag change only once it has accepted them,
    // so a refused binding leaves the environment as it was
    if (c->tp) {
        std::string em;
        if (int rc = ualm_tp::tp_set_params(c->tp, c->sel_env, p, &em)) return fail(rc, em);
    }
    // int_K, mem_size and past are baked into the resident batches' descriptors, buffer sizes and shared-memory layouts: a
    // parameter change invalidates every uploaded batch (it must be uploaded again before the next solve / eval call)
    for (auto &l : c->lanes) { l.have_batch = false; l.solved = false; }
    Env &v = c->envs[c->sel_env];
    v.hp = *p;
    DevParams &d = v.dp;
    d.use_scaling = p->use_scaling; d.rho = p->rho;
    d.beta = p->beta; d.gamma = p->gamma; d.epsilon_con = p->epsilon_con; d.max_iter = p->max_iter; d.g_epsilon = p->g_epsilon;
    d.min_step = p->min_step; d.delta = p->delta; d.inner_max_iter = (int)p->inner_max_iter; d.mem_size = p->mem_size; d.past = p->past;
    d.int_K = p->int_K; d.gravity = p->gravity;
    v.have_params = true;
    return UALM_OK;
}

extern "C" int ualm_select_env(ualm_ctx_t *c, int env)
{
    if (!c) return fail(UALM_EINVAL, "null ctx");
    if (env < 0 || env >= UALM_MAX_ENVS) return fail(UALM_EINVAL, "env out of range [0, UALM_MAX_ENVS)");
    c->sel_env = env;
    return UALM_OK;
}

static void map_geometry_set(MapVer &v, const ualm_map_geom_t *g)
{
    DevMap &m = v.dm;
    v.geom = *g;
    for (int k = 0; k < 3; k++) { m.vn[k] = g->voxel_num[k]; m.origin[k] = g->origin[k]; m.maxb[k] = g->max_boundary[k]; }
    m.xy_res = g->xy_resolution; m.yaw_res = g->yaw_resolution;
    m.xy_inv = 1.0 / g->xy_resolution; m.yaw_inv = 1.0 / g->yaw_resolution; // uneven_map.cpp:104-105
}

static size_t map_ncell(const ualm_map_geom_t *g) { return (size_t)g->voxel_num[0] * g->voxel_num[1] * g->voxel_num[2]; }
// the cell box {ix0, iy0, nx, ny} of the whole grid
static int4 map_box_all(const ualm_map_geom_t *g) { return make_int4(0, 0, g->voxel_num[0], g->voxel_num[1]); }

// a new grid version of `bytes` bytes, allocated on the map stream (usable once that stream is synchronised)
static int map_version_new(ualm_ctx *c, size_t bytes, MapRef *out)
{
    MapRef v = std::make_shared<MapVer>();
    v->fs = c->fstream;
    const cudaError_t e = cudaMallocFromPoolAsync(&v->p, std::max<size_t>(bytes, 1), c->mpool, c->mstream);
    if (e != cudaSuccess) {
        v->p = nullptr;
        cudaGetLastError();      // an allocation failure is not sticky: clear it, so no later launch check reports it
        return fail(UALM_ENOCUDA, std::string("grid allocation: ") + cudaGetErrorString(e));
    }
    v->bytes = bytes;
    *out = std::move(v);
    return UALM_OK;
}

// ualm_set_map / ualm_set_map_f64: the host grid into the selected environment's CURRENT version, in place, so a lane that holds it
// reads the new cells (ualm_set_map's contract).  The caller refused a batch in flight and synchronised the device
static int map_write_current(ualm_ctx *c, const ualm_map_geom_t *g, const void *cells, size_t bytes, bool f64)
{
    Env &v = c->envs[c->sel_env];
    v.have_map = false;         // until the copy below is complete (a failed copy leaves the environment unbound, not half bound)
    if (!v.map) {
        if (int rc = map_version_new(c, bytes, &v.map)) return rc;
    } else if (v.map->bytes < bytes) {       // grown in place: the lanes that hold this version see the new buffer
        CK(cudaFreeAsync(v.map->p, c->mstream));
        v.map->p = nullptr; v.map->bytes = 0;
        CK(cudaMallocFromPoolAsync(&v.map->p, bytes, c->mpool, c->mstream));
        v.map->bytes = bytes;
    }
    CK(cudaMemcpyAsync(v.map->p, cells, bytes, cudaMemcpyHostToDevice, c->mstream));
    CK(cudaStreamSynchronize(c->mstream));
    DevMap &m = v.map->dm;
    m.cells = f64 ? nullptr : (const float4 *)v.map->p;
    m.cells64 = f64 ? (const double *)v.map->p : nullptr;
    map_geometry_set(*v.map, g);
    if (c->tp) ualm_tp::tp_bind_map(c->tp, c->sel_env, g, m.cells);
    v.have_map = true;
    return UALM_OK;
}

// ualm_update_map*: the complete float4 version nv becomes the selected environment's current grid.  The version it replaces is freed
// once no lane holds it any more
static void map_install(ualm_ctx *c, const ualm_map_geom_t *g, MapRef nv)
{
    Env &v = c->envs[c->sel_env];
    nv->dm.cells = (const float4 *)nv->p;
    nv->dm.cells64 = nullptr;
    map_geometry_set(*nv, g);
    if (c->tp) ualm_tp::tp_bind_map(c->tp, c->sel_env, g, nv->dm.cells);
    v.map = std::move(nv);
    v.have_map = true;
}

// lane l launches its batch: it holds the current versions of the batch's environments from now on, and lets go of the versions of
// its previous launch.  That launch may still run (ualm_solve_resident twice on one lane), so the free stream first waits for its
// completion: whatever only it held is freed after it.  A throughput lane is relaunched only once collected (ctx lanes not made)
static int lane_hold(ualm_ctx *c, Lane &l)
{
    if (l.made) CK(cudaStreamWaitEvent(c->fstream, l.ev1, 0));
    for (int e = 0; e < UALM_MAX_ENVS; e++) l.vref[e] = (l.batch.env_mask >> e) & 1u ? c->envs[e].map : nullptr;
    return UALM_OK;
}

extern "C" int ualm_set_map(ualm_ctx_t *c, const ualm_map_geom_t *g, const float *cells)
{
    if (!c || !g || !cells) return fail(UALM_EINVAL, "null argument");
    if (int rc = lanes_idle(c, "ualm_set_map")) return rc;
    CK(cudaSetDevice(c->device));
    CK(cudaDeviceSynchronize());
    return map_write_current(c, g, cells, map_ncell(g) * sizeof(float4), false);
}

// the reference's own grid: UnevenMap::map_buffer is RXS2 {double z, sigma; Vector2d zb} = 4 doubles per cell (uneven_map.h:36-64)
extern "C" int ualm_set_map_f64(ualm_ctx_t *c, const ualm_map_geom_t *g, const double *cells, int repack_to_float)
{
    if (!c || !g || !cells) return fail(UALM_EINVAL, "null argument");
    if (int rc = lanes_idle(c, "ualm_set_map_f64")) return rc;
    CK(cudaSetDevice(c->device));
    CK(cudaDeviceSynchronize());
    const size_t ncell = map_ncell(g);
    if (repack_to_float || c->tp) {      // the throughput path always reads the float4 grid
        std::vector<float> f(4 * ncell);
        for (size_t q = 0; q < 4 * ncell; q++) f[q] = (float)cells[q];
        return ualm_set_map(c, g, f.data());
    }
    return map_write_current(c, g, cells, 4 * ncell * sizeof(double), true);
}

// Per device: the dynamic shared memory a CTA of every parity kernel may use (the opt-in per-block maximum, 227 KB on an H100,
// less the largest static shared memory of those kernels), and how far their dynamic shared-memory attribute has been raised.  The
// attribute belongs to the function on the current device, so it is kept per device, and only ever raised (kernels of another
// lane or context on the same device may be in flight with a larger size)
struct SmemDev { size_t cap = 0, raised = 0; };
static std::mutex g_smem_mu;
static std::vector<SmemDev> g_smem;

static int smem_dev(ualm_ctx *c, SmemDev **out)
{
    if ((size_t)c->device >= g_smem.size()) g_smem.resize(c->device + 1);
    SmemDev &s = g_smem[c->device];
    if (!s.cap) {
        CK(cudaSetDevice(c->device));
        int optin = 0;
        CK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
        size_t stat = 0;
        const void *ks[] = {(const void *)solve_kernel, (const void *)eval_kernel, (const void *)scaling_kernel, (const void *)penalty_only_kernel};
        for (const void *k : ks) {
            cudaFuncAttributes fa;
            CK(cudaFuncGetAttributes(&fa, k));
            stat = std::max(stat, fa.sharedSizeBytes);
        }
        if ((size_t)optin <= stat) return fail(UALM_ENOCUDA, "device has too little shared memory per block");
        s.cap = (size_t)optin - stat;
    }
    *out = &s;
    return UALM_OK;
}

static int smem_cap(ualm_ctx *c, size_t *cap)
{
    std::lock_guard<std::mutex> g(g_smem_mu);
    SmemDev *s;
    if (int rc = smem_dev(c, &s)) return rc;
    *cap = s->cap;
    return UALM_OK;
}

// the parity kernels' attribute on the context's device raised to at least `bytes` (at most the device's cap)
static int smem_raise(ualm_ctx *c, size_t bytes)
{
    std::lock_guard<std::mutex> g(g_smem_mu);
    SmemDev *s;
    if (int rc = smem_dev(c, &s)) return rc;
    if (bytes <= s->raised) return UALM_OK;
    CK(cudaSetDevice(c->device));
    CK(cudaFuncSetAttribute(solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    CK(cudaFuncSetAttribute(eval_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    CK(cudaFuncSetAttribute(scaling_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    CK(cudaFuncSetAttribute(penalty_only_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    s->raised = bytes;
    return UALM_OK;
}

// one trajectory slot of layout L fits four to a CTA of `cap` bytes (a one-warp solve launch)
static bool fits_four(const SmemLayout &L, size_t cap) { return (size_t)UALM_WPB * L.total_doubles * sizeof(double) <= cap; }

// the one-warp-per-problem layout of every environment present in the lane's batch (sized by that environment's maxima), and how
// many of those warps share a CTA: up to UALM_WPB, as many as a CTA's shared memory holds (eval_kernel, scaling_kernel and
// penalty_only_kernel take their warps per CTA from blockDim)
static int prepare_launch(ualm_ctx *c)
{
    Lane *b = c->b;
    const BatchLayout &L = b->batch;
    size_t cap = 0;
    if (int rc = smem_cap(c, &cap)) return rc;
    for (int e = 0; e < UALM_MAX_ENVS; e++) {
        if (L.eoff[e + 1] == L.eoff[e]) continue;
        int Nm = 1, Mm = 1, nm = 1, Sm = 1;
        for (int q = L.eoff[e]; q < L.eoff[e + 1]; q++) {
            const ProbDesc &d = b->desc[L.eidx[q]];
            if (L.skip[L.eidx[q]]) continue;
            Nm = std::max(Nm, d.N); Mm = std::max(Mm, d.M); nm = std::max(nm, d.n); Sm = std::max(Sm, d.S);
        }
        const DevParams &dp = c->envs[e].dp;
        b->eL[e] = make_layout(Nm, Mm, nm, dp.mem_size, dp.past, dp.int_K, Sm);
        const size_t slot = (size_t)b->eL[e].total_doubles * sizeof(double);
        b->ewpb[e] = (int)std::min<size_t>(UALM_WPB, cap / slot);
        // within the compiled limits (N <= 64, M <= 128, int_K <= 128, past <= 16) a slot is under 64 KB: three fit at least
        if (b->ewpb[e] < 1) return fail(UALM_ELIMIT, "problem too large for shared memory (N/M/int_K too big)");
        b->esmem[e] = slot * b->ewpb[e];
        if (int rc = smem_raise(c, b->esmem[e])) return rc;
    }
    return UALM_OK;
}

static int env_bound(ualm_ctx *c, int e)
{
    if (!c->envs[e].have_params || !c->envs[e].have_map)
        return fail(UALM_ESTATE, "environment " + std::to_string(e) + " has no parameters or no map grid bound (ualm_select_env + ualm_set_params / ualm_set_map)");
    return UALM_OK;
}
// env[B] (NULL = all 0): every index in range and every environment used fully bound, checked before anything is touched
static int check_envs(ualm_ctx *c, int B, const int32_t *env)
{
    for (int b = 0; b < (env ? B : 1); b++) {
        const int e = env ? env[b] : 0;
        if (e < 0 || e >= UALM_MAX_ENVS) return fail(UALM_EINVAL, "env index out of range [0, UALM_MAX_ENVS)");
        if (int rc = env_bound(c, e)) return rc;
    }
    return UALM_OK;
}
// every environment of an uploaded batch still bound (a failed ualm_set_map leaves its environment unbound)
static int check_envs(ualm_ctx *c, const BatchLayout &L)
{
    for (int e = 0; e < UALM_MAX_ENVS; e++)
        if ((L.env_mask >> e) & 1u)
            if (int rc = env_bound(c, e)) return rc;
    return UALM_OK;
}

// the compiled limits (n <= 256: the L-BFGS register tile, UALM_NREG in ualm_kernels.cuh): a problem over them is not solved or
// scanned, its record says UALM_ELIMIT, and the rest of its batch runs
static bool over_limits(int N, int M) { return N > UALM_NMAX || M > UALM_MMAX; }

// the problems of env[B] (NULL = all 0) grouped by environment, ascending within one: environment e at idx[off[e], off[e + 1])
static void group_by_env(int B, const int32_t *env, std::vector<int> &idx, int off[UALM_MAX_ENVS + 1])
{
    idx.clear();
    for (int e = 0; e < UALM_MAX_ENVS; e++) {
        off[e] = (int)idx.size();
        for (int b = 0; b < B; b++) if ((env ? env[b] : 0) == e) idx.push_back(b);
    }
    off[UALM_MAX_ENVS] = (int)idx.size();
}

// pp[B] (NULL = none): every field of every row finite
static_assert(sizeof(ualm_problem_params_t) == 8 * sizeof(double), "eight doubles, the first eight members of ualm_params_t");
static int check_pp(int B, const ualm_problem_params_t *pp)
{
    for (int b = 0; pp && b < B; b++)
        for (int k = 0; k < 8; k++)
            if (!std::isfinite((&pp[b].rho_T)[k])) return fail(UALM_EINVAL, "problem parameter row " + std::to_string(b) + " has a non-finite field");
    return UALM_OK;
}

// the layout of a batch (BatchLayout) for either path, from the arguments of ualm_upload_pp; every argument is checked first
static int batch_layout(ualm_ctx *c, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time, const double *inner_xy,
                        const double *inner_yaw, const int32_t *env, const ualm_problem_params_t *pp, BatchLayout *out)
{
    if (!c || B < 0 || (B > 0 && (!N || !M || !bnd || !total_time))) return fail(UALM_EINVAL, "bad argument");
    if (int rc = check_pp(B, pp)) return rc;
    if (int rc = check_envs(c, B, env)) return rc;
    long long need_xy = 0, need_yaw = 0;
    for (int b = 0; b < B; b++) {
        if (N[b] < 1 || M[b] < 1) return fail(UALM_EINVAL, "piece counts must be >= 1");
        if (!(total_time[b] > 0.0) || !std::isfinite(total_time[b])) return fail(UALM_EINVAL, "total_time must be finite and > 0");
        need_xy += 2LL * (N[b] - 1); need_yaw += M[b] - 1;
    }
    if ((need_xy > 0 && !inner_xy) || (need_yaw > 0 && !inner_yaw)) return fail(UALM_EINVAL, "inner waypoint arrays are NULL but N > 1 or M > 1");
    BatchLayout &L = *out;
    L = BatchLayout();
    L.B = B; L.N.assign(N, N + B); L.M.assign(M, M + B); L.env.assign(B, 0);
    if (env) L.env.assign(env, env + B);
    L.n.assign(B, 0); L.S.assign(B, 0); L.skip.assign(B, 0);
    L.off_x.assign(B, 0); L.off_s.assign(B, 0); L.off_cxy.assign(B, 0); L.off_cyaw.assign(B, 0);
    L.pp.resize(8 * (size_t)B);
    for (int b = 0; b < B; b++)
        memcpy(&L.pp[8 * (size_t)b], pp ? (const double *)&pp[b] : &c->envs[L.env[b]].hp.rho_T, 8 * sizeof(double));
    long long oixy = 0, oiyaw = 0;
    for (int b = 0; b < B; b++) {
        L.off_x[b] = L.tot_x; L.off_s[b] = L.tot_s; L.off_cxy[b] = L.tot_cxy; L.off_cyaw[b] = L.tot_cyaw;
        L.tot_cxy += 12LL * N[b]; L.tot_cyaw += 6LL * M[b];
        L.env_mask |= 1u << L.env[b];
        const long long nxy = 2LL * (N[b] - 1), nyaw = M[b] - 1;
        if (over_limits(N[b], M[b])) { L.skip[b] = 1; oixy += nxy; oiyaw += nyaw; continue; }
        L.n[b] = 1 + 2 * (N[b] - 1) + (M[b] - 1); L.S[b] = N[b] * (c->envs[L.env[b]].dp.int_K + 1);
        // x = [tau | Pxy | Pyaw]  (alm_traj_opt.cpp:205-216); logC2 (alm_traj_opt.h:238-241) is two IEEE ops + sqrt
        const double T = total_time[b];
        L.x0.push_back(T > 1.0 ? (std::sqrt(2.0 * T - 1.0) - 1.0) : (1.0 - std::sqrt(2.0 / T - 1.0)));
        L.x0.insert(L.x0.end(), inner_xy + oixy, inner_xy + oixy + nxy);
        L.x0.insert(L.x0.end(), inner_yaw + oiyaw, inner_yaw + oiyaw + nyaw);
        oixy += nxy; oiyaw += nyaw;
        L.tot_x += L.n[b]; L.tot_s += L.S[b];
        L.Nmax = std::max(L.Nmax, N[b]); L.Mmax = std::max(L.Mmax, M[b]);
        L.n_active++;
    }
    group_by_env(B, L.env.data(), L.eidx, L.eoff);
    return UALM_OK;
}

static BatchPtrs batch_ptrs(ualm_ctx *c)
{
    Lane *l = c->b;
    BatchPtrs b;
    b.B = l->batch.B;
    b.n_active = l->batch.n_active;
    b.queue = nullptr;
    b.n_leader_slots = 4;
    b.adopt = getenv("UALM_NOADOPT") ? 0 : 1;
    b.desc = l->d_desc.p; b.order = l->d_order.p; b.x0 = l->d_x0.p; b.x = l->d_x.p;
    b.lambda = l->d_lambda.p; b.mu = l->d_mu.p; b.scale_cx = l->d_scale_cx.p; b.hx = l->d_hx.p; b.gx = l->d_gx.p;
    b.lm_s = l->d_lm_s.p; b.lm_y = l->d_lm_y.p; b.lm_aux = l->d_lm_aux.p; b.fac = l->d_fac.p; b.scratch = l->d_scr.p; b.ws_scaling = l->d_ws.p;
    b.c_xy = l->d_cxy.p; b.c_yaw = l->d_cyaw.p; b.results = l->d_res.p; b.piece_T = l->d_pieceT.p; b.f_out = l->d_f.p; b.grad_out = l->d_grad.p;
    b.scale_fx_io = l->d_sfx.p;
    b.prof = c->profile ? l->d_prof.p : nullptr;
    b.mbox = ualm_mbox::Ptrs{};
    b.hold = nullptr; b.hctl = nullptr; b.urgent_slot = -1; b.n_urgent = 0;
    return b;
}

// launch(e, bp, count) once per environment present in the selected lane's batch, with bp.order / bp.n_active set to that
// environment's problems (eval_kernel, scaling_kernel and penalty_only_kernel map their warps to problems through them)
template <class F>
static int per_env(ualm_ctx *c, F launch)
{
    Lane *l = c->b;
    for (int e = 0; e < UALM_MAX_ENVS; e++) {
        const int cnt = l->batch.eoff[e + 1] - l->batch.eoff[e];
        if (cnt == 0) continue;
        BatchPtrs bp = batch_ptrs(c);
        bp.order = l->d_eidx.p + l->batch.eoff[e];
        bp.n_active = cnt;
        launch(e, bp, cnt);
        CK(cudaGetLastError());
    }
    return UALM_OK;
}

extern "C" int ualm_upload(ualm_ctx_t *c, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                           const double *inner_xy, const double *inner_yaw)
{
    return ualm_upload_pp(c, B, N, M, bnd, total_time, inner_xy, inner_yaw, nullptr, nullptr);
}

// ualm_upload_pp; `before_device` (parity path, may be empty) runs after every host-side allocation and free of the upload and before
// its first device operation: ualm_submit_batch_env raises an urgent ticket's hold there, where nothing of the call waits for the device
// any more
static int upload_env(ualm_ctx *c, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time, const double *inner_xy,
                      const double *inner_yaw, const int32_t *env, const ualm_problem_params_t *pp, const std::function<int()> &before_device)
{
    // validate everything before touching the lane; the lane holds no batch until this call has fully succeeded
    BatchLayout lay;
    if (int rc = batch_layout(c, B, N, M, bnd, total_time, inner_xy, inner_yaw, env, pp, &lay)) return rc;
    if (lane_in_flight(c, c->cur)) return fail(UALM_ESTATE, "ualm_upload into a lane whose submitted batch is still in flight");
    Lane *l = c->b;
    l->have_batch = false; l->solved = false;
    l->batch = std::move(lay);
    const BatchLayout &L = l->batch;
    if (c->tp) TP_CALL(ualm_tp::tp_upload(c->tp, c->cur, L, bnd, total_time, err));
    CK(cudaSetDevice(c->device));
    l->desc.assign(B, ProbDesc()); l->order.clear(); l->group.assign(B, 1);
    for (int b = 0; b < B; b++) {
        ProbDesc &d = l->desc[b];
        d.N = L.N[b]; d.M = L.M[b]; d.n = L.n[b]; d.S = L.S[b];
        if (!L.skip[b]) l->order.push_back(b);
    }
    const int BA = L.n_active;
    // launch order: most samples first (longest-processing-time-first keeps the tail short)
    std::stable_sort(l->order.begin(), l->order.end(), [&](int a, int b2) { return l->desc[a].S > l->desc[b2].S; });
    // a problem whose own layout does not fit four to a CTA (N, M and int_K near their limits) is solved by a group of two or four
    // warps (a G=4 CTA holds one slot, a G=2 CTA two): these "wide" problems go first, so the group-size ranges below give them one
    size_t cap = 0;
    if (int rc = smem_cap(c, &cap)) return rc;
    const long long n_wide = std::stable_partition(l->order.begin(), l->order.end(), [&](int b2) {
        const ProbDesc &d = l->desc[b2];
        const DevParams &ep = c->envs[L.env[b2]].dp;
        return !fits_four(make_layout(d.N, d.M, d.n, ep.mem_size, ep.past, ep.int_K, d.S), cap);
    }) - l->order.begin();
    int rc0 = prepare_launch(c);
    if (rc0) return rc0;
    // Warp groups and launches.  Problems are sorted by size; the largest get 4 or 2 warps (helpers for the parallel phases) as
    // far as the whole batch still fits on the device at once.  Every (group size, environment) range of the order is one launch
    // with its own shared-memory layout sized by the range's maxima: a G=4 CTA holds one trajectory slot + 3 helper rings, a G=2
    // CTA two slots + 2 rings, a G=1 CTA four slots.  The slots of a launch take its problems largest first from one work queue
    // (solve_kernel), so a slot whose trajectory ends early starts the next one; the grid is what the device holds at once, or
    // fewer CTAs when the range is smaller.  The launches run concurrently on separate streams.
    {
        int dev_sms = 0;
        CK(cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, c->device));
        const int RINGD = 2 * UALM_RINGB * 6 * UALM_FW;
        int occ0 = 1;   // CTAs per SM the register file allows (shared memory is checked per class below)
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ0, solve_kernel, UALM_THREADS * UALM_WPB, 16 * 1024));
        if (getenv("UALM_DEBUG")) {
            cudaFuncAttributes fa;
            CK(cudaFuncGetAttributes(&fa, solve_kernel));
            fprintf(stderr, "[ualm] solve_kernel: %d regs/thread, %zu B local, %zu B static smem, %d CTAs/SM by registers\n", fa.numRegs, fa.localSizeBytes,
                    fa.sharedSizeBytes, occ0);
        }
        const long long W = 4LL * occ0 * dev_sms;   // warp slots on the device
        std::vector<Lane::GClass> best;
        std::vector<int> best_ord;
        for (int attempt = 0; attempt < 32; attempt++) {
            // Policy: helpers shorten the latency of a trajectory without adding to the L2-resident working set, while more
            // resident trajectories thrash the L2.  So: everything that fits gets 4 warps; beyond that 2 warps per trajectory,
            // run in waves (on an H100, 1024 problems with 3 batches in flight: 4.7 % faster than giving the largest tenth 4 warps,
            // 8 % faster than single warps; tools/gpu_policy_dev.py).
            long long K4 = 0, K2 = 0;
            if (c->group_mode) {
                if (4LL * BA <= W) K4 = BA;
                else if (2LL * BA <= W) { K4 = std::min<long long>(BA, (W - 2LL * BA) / 2); K2 = (BA - K4) & ~1LL; }
                else K2 = BA & ~1LL;
                if (attempt > 0) { K4 = (long long)(K4 * std::pow(0.8, attempt)); K2 = std::min<long long>(BA - K4, K2) & ~1LL; }
            }
            const bool forced = getenv("UALM_F4") || getenv("UALM_F2");   // developer override: fractions of the batch
            if (forced) {
                K4 = (long long)(BA * (getenv("UALM_F4") ? atof(getenv("UALM_F4")) : 0.0));
                K2 = std::min<long long>(BA - K4, (long long)(BA * (getenv("UALM_F2") ? atof(getenv("UALM_F2")) : 0.0))) & ~1LL;
            }
            if (K4 + K2 < n_wide) {
                if (!c->group_mode && !forced)
                    return fail(UALM_ELIMIT, "UALM_GROUPS=0: a problem's shared-memory layout does not fit four one-warp slots per CTA (N/M/int_K too big)");
                K2 = n_wide - K4;
            }
            // rank ranges per group size; within one, the problems of each environment (a launch holds one: its parameters and grid
            // are the launch's grid constants)
            std::vector<Lane::GClass> cls;
            std::vector<int> ord = l->order;
            const long long lim[4] = {0, K4, K4 + K2, BA};
            for (int gi = 0; gi < 3; gi++) {
                const int G = gi == 0 ? 4 : gi == 1 ? 2 : 1;
                if (lim[gi + 1] <= lim[gi]) continue;
                std::stable_sort(ord.begin() + lim[gi], ord.begin() + lim[gi + 1], [&](int x, int y) { return L.env[x] < L.env[y]; });
                for (long long a = lim[gi], b2; a < lim[gi + 1]; a = b2) {
                    const int ce = L.env[ord[a]];
                    const DevParams &ep = c->envs[ce].dp;
                    Lane::GClass cl;
                    cl.G = G; cl.env = ce; cl.r0 = (int)a;
                    // the range's problems of one environment; a one-warp launch also ends before a problem that would take the
                    // layout of its maxima past four slots per CTA (each problem of that range fits alone: the wide ones come first)
                    int Nm = 1, Mm = 1, nm = 1, Sm = 1;
                    for (b2 = a; b2 < lim[gi + 1] && L.env[ord[b2]] == ce; b2++) {
                        const ProbDesc &d = l->desc[ord[b2]];
                        const int N2 = std::max(Nm, d.N), M2 = std::max(Mm, d.M), n2 = std::max(nm, d.n), S2 = std::max(Sm, d.S);
                        if (G == 1 && b2 > a && !fits_four(make_layout(N2, M2, n2, ep.mem_size, ep.past, ep.int_K, S2), cap)) break;
                        Nm = N2; Mm = M2; nm = n2; Sm = S2;
                    }
                    cl.r1 = (int)b2;
                    cl.L = make_layout(Nm, Mm, nm, ep.mem_size, ep.past, ep.int_K, Sm);
                    const int per = 4 / G;                         // trajectory slots per CTA
                    cl.smem = ((size_t)per * cl.L.total_doubles + (size_t)(4 - per) * RINGD) * sizeof(double);
                    if (int rc = smem_raise(c, cl.smem)) return rc;
                    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cl.occ, solve_kernel, UALM_THREADS * UALM_WPB, cl.smem));
                    cl.n_ctas = (int)((b2 - a + per - 1) / per);
                    cl.grid = (int)std::min<long long>(cl.n_ctas, (long long)std::max(cl.occ, 1) * dev_sms);
                    cls.push_back(cl);
                }
            }
            double sm_need = 0.0;
            for (auto &cl : cls) sm_need += (double)cl.n_ctas / std::max(cl.occ, 1);
            best = cls;
            best_ord = ord;
            // multi-wave batches need not fit at once; batches meant to be fully resident must
            if (forced || 2LL * BA > W || sm_need <= 0.98 * dev_sms || attempt >= 12) break;
        }
        l->cls = best;
        l->order = best_ord;
        for (auto &cl : l->cls) {
            for (int r = cl.r0; r < cl.r1; r++) l->group[l->order[r]] = cl.G;
            if (getenv("UALM_DEBUG"))
                fprintf(stderr, "[ualm] launch G=%d env %d: problems [%d,%d), %d CTAs, smem %zu B, %d CTAs/SM\n", cl.G, cl.env, cl.r0, cl.r1, cl.grid,
                        cl.smem, cl.occ);
        }
    }
    // the offsets of the parity path's own buffers (the layout has those of x, the samples and the coefficients)
    long long oh = 0, oscr = 0, ofac = 0, ows = 0, oaux = 0;
    std::vector<ualm_result_t> res0(B);
    for (int b = 0; b < B; b++) {
        ProbDesc &d = l->desc[b];
        const int m = c->envs[L.env[b]].dp.mem_size;
        d.off_x = L.off_x[b]; d.off_s = L.off_s[b]; d.off_cxy = L.off_cxy[b]; d.off_cyaw = L.off_cyaw[b];
        d.off_hist = oh; d.off_scr = oscr; d.off_fac = ofac; d.off_ws = ows;
        d.off_aux = oaux; oaux += 3LL * m;
        for (int k = 0; k < 18; k++) d.bnd[k] = bnd[(size_t)b * 18 + k];
        for (int k = 0; k < 8; k++) d.pp[k] = L.pp[8 * (size_t)b + k];
        d.total_time = total_time[b];
        memset(&res0[b], 0, sizeof(ualm_result_t));
        if (L.skip[b]) { res0[b].ret_code = UALM_ELIMIT; continue; }
        oh += (long long)m * d.n; oscr += (long long)UALM_NFIELD * d.S;
        ofac += 1LL * UALM_FW * ((6 * d.N + 2 * UALM_FPAD) + (6 * d.M + 2 * UALM_FPAD));
        ows += (long long)(12 * d.N + 6 * d.M) * 32 * l->group[b];
    }
    l->tot_hist = oh; l->tot_scr = oscr; l->tot_fac = ofac; l->tot_ws = ows;
    const long long ox = L.tot_x, os = L.tot_s, ocx = L.tot_cxy, ocy = L.tot_cyaw;
    CK(l->d_desc.ensure(B)); CK(l->d_order.ensure(BA)); CK(l->d_queue.ensure(l->cls.size() + 3)); CK(l->d_x0.ensure(ox)); CK(l->d_x.ensure(ox)); CK(l->d_grad.ensure(ox));
    CK(l->d_lambda.ensure(os)); CK(l->d_hx.ensure(os)); CK(l->d_mu.ensure(6 * os)); CK(l->d_gx.ensure(6 * os)); CK(l->d_scale_cx.ensure(7 * os));
    CK(l->d_lm_s.ensure(oh)); CK(l->d_lm_y.ensure(oh)); CK(l->d_scr.ensure(oscr));
    CK(l->d_ws.ensure(ows)); CK(l->d_fac.ensure(ofac)); CK(l->d_lm_aux.ensure((size_t)std::max(oaux, 1LL)));
    CK(l->d_eidx.ensure(B));
    CK(l->d_stop.ensure((size_t)std::max(B, 1)));
    CK(l->d_prof.ensure((size_t)std::max(B, 1) * UALM_NPROF));
    CK(l->d_pieceT.ensure((size_t)std::max(B, 1) * 2)); CK(l->d_feas.ensure((size_t)std::max(B, 1) * 16));
    CK(l->d_cxy.ensure(ocx)); CK(l->d_cyaw.ensure(ocy)); CK(l->d_res.ensure(B)); CK(l->d_f.ensure(B)); CK(l->d_sfx.ensure(B));
    if (before_device) if (int rc = before_device()) return rc;
    // factor arrays: entries outside the band-in-matrix positions (and the pad rows) are never written and must read 0
    if (ofac > 0) CK(cudaMemsetAsync(l->d_fac.p, 0, sizeof(double) * ofac, l->stream));
    if (B > 0) {
        CK(cudaMemcpyAsync(l->d_desc.p, l->desc.data(), sizeof(ProbDesc) * B, cudaMemcpyHostToDevice, l->stream));
        if (BA > 0) CK(cudaMemcpyAsync(l->d_order.p, l->order.data(), sizeof(int) * BA, cudaMemcpyHostToDevice, l->stream));
        CK(cudaMemcpyAsync(l->d_eidx.p, L.eidx.data(), sizeof(int) * B, cudaMemcpyHostToDevice, l->stream));
        if (ox > 0) CK(cudaMemcpyAsync(l->d_x0.p, L.x0.data(), sizeof(double) * ox, cudaMemcpyHostToDevice, l->stream));
        // records of skipped problems (the kernels overwrite the others), zero coefficients and durations for them
        CK(cudaMemcpyAsync(l->d_res.p, res0.data(), sizeof(ualm_result_t) * B, cudaMemcpyHostToDevice, l->stream));
        if (BA < B) {
            CK(cudaMemsetAsync(l->d_cxy.p, 0, sizeof(double) * ocx, l->stream));
            CK(cudaMemsetAsync(l->d_cyaw.p, 0, sizeof(double) * ocy, l->stream));
            CK(cudaMemsetAsync(l->d_pieceT.p, 0, sizeof(double) * 2 * B, l->stream));
        }
        CK(cudaStreamSynchronize(l->stream)); // res0 is a stack-local staging vector
    }
    l->have_batch = true; l->solved = false;
    return UALM_OK;
}
extern "C" int ualm_upload_env(ualm_ctx_t *c, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                               const double *inner_xy, const double *inner_yaw, const int32_t *env)
{
    return ualm_upload_pp(c, B, N, M, bnd, total_time, inner_xy, inner_yaw, env, nullptr);
}
extern "C" int ualm_upload_pp(ualm_ctx_t *c, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                              const double *inner_xy, const double *inner_yaw, const int32_t *env, const ualm_problem_params_t *pp)
{
    return upload_env(c, B, N, M, bnd, total_time, inner_xy, inner_yaw, env, pp, {});
}

// raise (1) or lower (0) hold byte `slot` (ualm_ctx::d_hold) in the order of stream st
static int hold_set(ualm_ctx *c, int slot, int v, cudaStream_t st)
{
    CK(cudaMemcpyAsync(c->d_hold + slot, c->h_hold + v, 1, cudaMemcpyHostToDevice, st));
    return UALM_OK;
}

// the lane's greatest-priority streams (Lane::ustream), made at its first urgent ticket
static int lane_priority_streams(Lane &l)
{
    if (!l.ustream[0]) {
        int least = 0, greatest = 0;
        CK(cudaDeviceGetStreamPriorityRange(&least, &greatest));
        for (auto &s : l.ustream) CK(cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, greatest));
    }
    return UALM_OK;
}

// lowers a hold on every exit of a call that raised it, unless the raise is handed on (armed = false)
struct HoldGuard {
    ualm_ctx *c;
    int slot;
    cudaStream_t st;
    bool armed;
    ~HoldGuard() { if (armed) cudaMemcpyAsync(c->d_hold + slot, c->h_hold, 1, cudaMemcpyHostToDevice, st); }
};

// launch ci of the selected lane's solve on stream st: its loop graph (Lane::SolveLoop) with this launch's arguments.  The handle
// starts every graph launch at 1, so the body runs at least once; without a hold it runs exactly once.  A graph is updated in place,
// never destroyed while the device may run it: destroying an executable graph waits for the device
static int solve_loop_run(Lane &l, size_t ci, const BatchPtrs &bp, const DevParams &dp, const DevMap &dm, const Lane::GClass &cl, cudaStream_t st)
{
    if (l.loops.size() <= ci) l.loops.resize(ci + 1);
    Lane::SolveLoop &g = l.loops[ci];
    BatchPtrs a_bp = bp;
    DevParams a_dp = dp;
    DevMap a_dm = dm;
    SmemLayout a_L = cl.L;
    unsigned char *a_hold = bp.hold;
    int *a_hctl = bp.hctl, a_urgent = bp.urgent_slot >= 0, a_n = bp.n_active;
    const int *a_queue = bp.queue;
    if (!g.G) CK(cudaGraphCreate(&g.G, 0));
    if (!g.h) CK(cudaGraphConditionalHandleCreate(&g.h, g.G, 1, cudaGraphCondAssignDefault));
    cudaGraphConditionalHandle a_h = g.h;
    void *gate_args[] = {&a_hold, &a_hctl, &a_urgent};
    void *solve_args[] = {&a_bp, &a_dp, &a_dm, &a_L};
    void *ctrl_args[] = {&a_h, &a_queue, &a_n};
    cudaKernelNodeParams gp = {}, sp = {}, cp = {};
    gp.func = (void *)hold_gate_kernel; gp.gridDim = dim3(1); gp.blockDim = dim3(1); gp.kernelParams = gate_args;
    sp.func = (void *)solve_kernel; sp.gridDim = dim3(cl.grid); sp.blockDim = dim3(UALM_THREADS * UALM_WPB); sp.sharedMemBytes = (unsigned)cl.smem;
    sp.kernelParams = solve_args;
    cp.func = (void *)solve_loop_ctrl_kernel; cp.gridDim = dim3(1); cp.blockDim = dim3(1); cp.kernelParams = ctrl_args;
    if (!g.gate) {
        cudaGraphNodeParams wp = {};
        wp.type = cudaGraphNodeTypeConditional;
        wp.conditional.handle = g.h;
        wp.conditional.type = cudaGraphCondTypeWhile;
        wp.conditional.size = 1;
        cudaGraphNode_t wn;
        CK(cudaGraphAddNode(&wn, g.G, nullptr, 0, &wp));
        const cudaGraph_t body = wp.conditional.phGraph_out[0];
        CK(cudaGraphAddKernelNode(&g.gate, body, nullptr, 0, &gp));
        CK(cudaGraphAddKernelNode(&g.solve, body, &g.gate, 1, &sp));
        CK(cudaGraphAddKernelNode(&g.ctrl, body, &g.solve, 1, &cp));
    } else {
        CK(cudaGraphKernelNodeSetParams(g.gate, &gp));
        CK(cudaGraphKernelNodeSetParams(g.solve, &sp));
        CK(cudaGraphKernelNodeSetParams(g.ctrl, &cp));
    }
    if (g.exec) {
        cudaGraphExecUpdateResultInfo info;
        if (cudaGraphExecUpdate(g.exec, g.G, &info) != cudaSuccess) {     // kept until the lane's release: destroying it would wait
            cudaGetLastError();                                             // for the device, possibly under a hold this call raised
            l.retired.push_back(g.exec);
            g.exec = nullptr;
        }
    }
    if (!g.exec) CK(cudaGraphInstantiate(&g.exec, g.G, 0));
    CK(cudaGraphLaunch(g.exec, st));
    return UALM_OK;
}

// the solve launches of the selected lane's batch; `publish`: every problem also goes to the lane's mailbox as it ends (submit only);
// `urgent`: an urgent ticket (ualm_set_urgent) that has raised the lane's hold byte (ualm_submit_batch_env); its launches run on the lane's
// greatest-priority streams and ignore holds, and the take of its last problem lowers the byte (slot_next)
static int solve_launch(ualm_ctx *c, bool publish, bool urgent = false)
{
    Lane *l = c->b;
    if (!l->have_batch) return fail(UALM_ESTATE, "set_params, set_map and upload must precede solve");
    if (int rc = check_envs(c, l->batch)) return rc;
    CK(cudaSetDevice(c->device));
    if (int rc = lane_hold(c, *l)) return rc;
    if (urgent) if (int rc = lane_priority_streams(*l)) return rc;
    l->last_launches = 0;
    // no stop request carries over: the words are cleared before the solve, and raises are queued after ev_clear
    if (l->h_stop) memset(l->h_stop, 0, sizeof(int) * l->h_stop_cap);
    CK(cudaMemsetAsync(l->d_stop.p, 0, sizeof(int) * std::max(l->batch.B, 1), l->stream));
    CK(cudaEventRecord(l->ev_clear, l->stream));
    // every launch's queue full, the lane's hold words zero
    CK(cudaMemsetAsync(l->d_queue.p, 0, sizeof(int) * (l->cls.size() + 3), l->stream));
    CK(cudaEventRecord(l->ev0, l->stream));
    if (l->batch.n_active > 0) {
        // the launches run concurrently: launch 0 on the lane stream, the others on auxiliary streams (an urgent ticket's: on the
        // lane's priority streams, joined back to the lane stream)
        const int last = Lane::NAUX;
        const cudaStream_t base = urgent ? l->ustream[last] : l->stream;
        CK(cudaEventRecord(l->evs[last], l->stream));
        if (urgent) CK(cudaStreamWaitEvent(base, l->evs[last], 0));
        for (size_t ci = 0; ci < l->cls.size(); ci++) {
            auto &cl = l->cls[ci];
            if (cl.grid == 0) continue;
            const int ai = (int)((ci - 1) % Lane::NAUX);
            cudaStream_t st = ci == 0 ? base : urgent ? l->ustream[ai] : l->aux[ai];
            if (ci > 0) CK(cudaStreamWaitEvent(st, l->evs[last], 0));
            BatchPtrs bp = batch_ptrs(c);
            bp.queue = l->d_queue.p + ci;
            bp.order = l->d_order.p + cl.r0;
            bp.n_active = cl.r1 - cl.r0;
            bp.n_leader_slots = 4 / cl.G;
            if (publish) bp.mbox = l->mbox.device();
            bp.hold = c->d_hold;
            bp.hctl = l->d_queue.p + l->cls.size();
            bp.urgent_slot = urgent ? c->cur : -1;
            bp.n_urgent = l->batch.n_active;
            // the launch's environment: its parameters and grid are the launch's grid constants, the solve reads them as before
            DevParams dp = c->envs[cl.env].dp;
            dp.cancel = l->d_stop.p;
            dp.max_evals = c->max_evals;
            if (int rc = solve_loop_run(*l, ci, bp, dp, l->vref[cl.env]->dm, cl, st)) return rc;
            l->last_launches++;
            if (ci > 0) { CK(cudaEventRecord(l->evs[ai], st)); CK(cudaStreamWaitEvent(base, l->evs[ai], 0)); }
        }
        if (urgent) { CK(cudaEventRecord(l->evs[last], base)); CK(cudaStreamWaitEvent(l->stream, l->evs[last], 0)); }
    }
    CK(cudaEventRecord(l->ev1, l->stream));
    l->solved = true;
    return UALM_OK;
}

extern "C" int ualm_solve_resident(ualm_ctx_t *c)
{
    if (!c) return fail(UALM_EINVAL, "null ctx");
    if (c->tp) {     // joins the pool of running trajectories; its rounds run on the device, ualm_sync waits
        if (int rc = check_envs(c, c->b->batch)) return rc;
        std::string em;
        if (int rc = ualm_tp::tp_admit(c->tp, c->cur, &em)) return fail(rc, em);
        return lane_hold(c, *c->b);
    }
    return solve_launch(c, false);
}

extern "C" int ualm_sync(ualm_ctx_t *c)
{
    if (!c) return fail(UALM_EINVAL, "null ctx");
    if (c->tp) {
        if (!ualm_tp::tp_lane_in_flight(c->tp, c->cur)) return UALM_OK;
        TP_CALL(ualm_tp::tp_collect(c->tp, c->cur, err));
    }
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->b->stream));
    return UALM_OK;
}

extern "C" int ualm_last_solve_ms(ualm_ctx_t *c, float *ms, int *launches)
{
    if (c && c->tp) return ualm_tp::tp_last_solve(c->tp, c->cur, ms, launches) == UALM_OK ? UALM_OK : fail(UALM_ESTATE, "no collected solve to time");
    if (!c || !c->b->solved) return fail(UALM_ESTATE, "no solve to time");
    Lane *l = c->b;
    CK(cudaEventSynchronize(l->ev1));
    CK(cudaEventElapsedTime(&l->last_ms, l->ev0, l->ev1));
    if (ms) *ms = l->last_ms;
    if (launches) *launches = l->last_launches;
    return UALM_OK;
}

// pipeline timing over several lanes: begin = an event on the selected lane's stream (record it before the first launch of the
// timed region); end = an event on a join stream that waits for the last solve of every lane
extern "C" int ualm_mark_begin(ualm_ctx_t *c)
{
    if (!c) return fail(UALM_EINVAL, "null ctx");
    if (c->tp) TP_CALL(ualm_tp::tp_mark_begin(c->tp, err));
    CK(cudaSetDevice(c->device));
    CK(cudaEventRecord(c->evA, c->b->stream));
    return UALM_OK;
}
extern "C" int ualm_mark_end(ualm_ctx_t *c, float *ms)
{
    if (!c || !ms) return fail(UALM_EINVAL, "null argument");
    if (c->tp) TP_CALL(ualm_tp::tp_mark_end(c->tp, ms, err));
    CK(cudaSetDevice(c->device));
    for (auto &l : c->lanes)
        if (l.made && l.solved) CK(cudaStreamWaitEvent(c->join, l.ev1, 0));
    CK(cudaEventRecord(c->evB, c->join));
    CK(cudaEventSynchronize(c->evB));
    CK(cudaEventElapsedTime(ms, c->evA, c->evB));
    return UALM_OK;
}

extern "C" int ualm_download(ualm_ctx_t *c, ualm_result_t *results, double *c_xy, double *c_yaw)
{
    if (c && c->tp) {
        if (!ualm_tp::tp_lane_in_flight(c->tp, c->cur) && !ualm_tp::tp_lane_collected(c->tp, c->cur)) return fail(UALM_ESTATE, "nothing solved");
        TP_CALL(ualm_tp::tp_download(c->tp, c->cur, results, c_xy, c_yaw, err));
    }
    if (!c || !c->b->solved) return fail(UALM_ESTATE, "nothing solved");
    Lane *l = c->b;
    const BatchLayout &L = l->batch;
    CK(cudaSetDevice(c->device));
    if (L.B > 0) {
        if (results) CK(cudaMemcpyAsync(results, l->d_res.p, sizeof(ualm_result_t) * L.B, cudaMemcpyDeviceToHost, l->stream));
        if (c_xy) CK(cudaMemcpyAsync(c_xy, l->d_cxy.p, sizeof(double) * L.tot_cxy, cudaMemcpyDeviceToHost, l->stream));
        if (c_yaw) CK(cudaMemcpyAsync(c_yaw, l->d_cyaw.p, sizeof(double) * L.tot_cyaw, cudaMemcpyDeviceToHost, l->stream));
    }
    CK(cudaStreamSynchronize(l->stream));
    return UALM_OK;
}

extern "C" int ualm_solve_batch(ualm_ctx_t *c, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                                const double *inner_xy, const double *inner_yaw, ualm_result_t *results, double *c_xy, double *c_yaw)
{
    return ualm_solve_batch_env(c, B, N, M, bnd, total_time, inner_xy, inner_yaw, nullptr, results, c_xy, c_yaw);
}
extern "C" int ualm_solve_batch_env(ualm_ctx_t *c, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                                    const double *inner_xy, const double *inner_yaw, const int32_t *env, ualm_result_t *results, double *c_xy,
                                    double *c_yaw)
{
    return ualm_solve_batch_pp(c, B, N, M, bnd, total_time, inner_xy, inner_yaw, env, nullptr, results, c_xy, c_yaw);
}
extern "C" int ualm_solve_batch_pp(ualm_ctx_t *c, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                                   const double *inner_xy, const double *inner_yaw, const int32_t *env, const ualm_problem_params_t *pp,
                                   ualm_result_t *results, double *c_xy, double *c_yaw)
{
    int rc = ualm_upload_pp(c, B, N, M, bnd, total_time, inner_xy, inner_yaw, env, pp);
    if (rc) return rc;
    rc = ualm_solve_resident(c);
    if (rc) return rc;
    return ualm_download(c, results, c_xy, c_yaw);
}

// ---- pipelined batches: submit returns as soon as the batch is uploaded and its kernels are queued; several batches (one per
// lane, round robin) run concurrently, so the slow tail of one batch overlaps the bulk of the next ----
extern "C" int ualm_submit_batch(ualm_ctx_t *c, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                                 const double *inner_xy, const double *inner_yaw, int depth, int *ticket)
{
    return ualm_submit_batch_env(c, B, N, M, bnd, total_time, inner_xy, inner_yaw, nullptr, depth, ticket);
}
extern "C" int ualm_submit_batch_env(ualm_ctx_t *c, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                                     const double *inner_xy, const double *inner_yaw, const int32_t *env, int depth, int *ticket)
{
    return ualm_submit_batch_pp(c, B, N, M, bnd, total_time, inner_xy, inner_yaw, env, nullptr, depth, ticket);
}
extern "C" int ualm_submit_batch_pp(ualm_ctx_t *c, int B, const int32_t *N, const int32_t *M, const double *bnd, const double *total_time,
                                    const double *inner_xy, const double *inner_yaw, const int32_t *env, const ualm_problem_params_t *pp, int depth,
                                    int *ticket)
{
    if (!c || !ticket) return fail(UALM_EINVAL, "null argument");
    if (int rc = check_pp(B, pp)) return rc;
    if (depth < 1 || depth > UALM_MAX_LANES) return fail(UALM_EINVAL, "depth out of range [1, UALM_MAX_LANES]");
    const int lane = c->next_submit % depth;
    if (lane_in_flight(c, lane)) return fail(UALM_ESTATE, "all lanes of this depth are in flight: ualm_wait_batch the oldest ticket first");
    const int keep = c->cur;
    int rc = ualm_select_lane(c, lane);
    Lane &l = c->lanes[lane];
    // an urgent ticket with a problem to solve raises the lane's hold byte on the lane stream once the upload has made every host-side
    // allocation and free (they can wait for the device, and under a raised hold the device would wait for this call) and before its
    // device work, which needs SM slots too.  The same holds for the mailbox, the stop words' mirror and the priority streams, made
    // there first.  Every refusal after the raise lowers it; after a solve_launch the launches' last take lowers it
    bool urgent = false;
    HoldGuard guard{c, lane, l.stream, false};
    auto before_device = [&]() -> int {
        cudaError_t e = l.mbox.begin(B, N, M, l.batch.skip.data());
        if (e != cudaSuccess) return fail(UALM_ENOCUDA, std::string("result mailbox: ") + cudaGetErrorString(e));
        if (l.h_stop_cap < (size_t)std::max(B, 1)) {      // the stop words' host mirror (solve_launch clears it)
            if (l.h_stop) cudaFreeHost(l.h_stop);
            l.h_stop = nullptr; l.h_stop_cap = 0;
            e = cudaHostAlloc(&l.h_stop, sizeof(int) * std::max(B, 1), cudaHostAllocDefault);
            if (e != cudaSuccess) return fail(UALM_ENOCUDA, std::string("stop words: ") + cudaGetErrorString(e));
            l.h_stop_cap = (size_t)std::max(B, 1);
        }
        urgent = c->urgent && l.batch.n_active > 0;
        if (!urgent) return UALM_OK;
        if (int r = lane_priority_streams(l)) return r;
        if (int r = hold_set(c, lane, 1, l.stream)) return r;
        guard.armed = true;
        return UALM_OK;
    };
    if (!rc) rc = upload_env(c, B, N, M, bnd, total_time, inner_xy, inner_yaw, env, pp, before_device);
    if (!rc && c->tp) {
        std::string em;
        rc = ualm_tp::tp_admit(c->tp, lane, &em, true, c->urgent);
        rc = rc ? fail(rc, em) : lane_hold(c, l);
    } else if (!rc) {
        rc = solve_launch(c, true, urgent);
        if (!rc) { l.in_flight = true; guard.armed = false; }
    }
    if (!rc) { *ticket = lane; c->next_submit = (lane + 1) % depth; }
    c->cur = keep; c->b = &c->lanes[keep];
    return rc;
}
extern "C" int ualm_wait_batch(ualm_ctx_t *c, int ticket, ualm_result_t *results, double *c_xy, double *c_yaw)
{
    if (!c || ticket < 0 || ticket >= UALM_MAX_LANES) return fail(UALM_EINVAL, "bad ticket");
    if (c->tp) {
        if (!ualm_tp::tp_lane_in_flight(c->tp, ticket)) return fail(UALM_ESTATE, "ticket is not in flight");
        TP_CALL(ualm_tp::tp_download(c->tp, ticket, results, c_xy, c_yaw, err));
    }
    if (!c->lanes[ticket].in_flight) return fail(UALM_ESTATE, "ticket is not in flight");
    const int keep = c->cur;
    c->cur = ticket; c->b = &c->lanes[ticket];
    int rc = ualm_download(c, results, c_xy, c_yaw);
    // a raise that the batch outran may still be queued: it lands before the lane's next clear, and the mirror is free again
    if (c->lanes[ticket].raised) {
        const cudaError_t e = cudaStreamSynchronize(c->cancel);
        if (!rc && e != cudaSuccess) rc = fail(UALM_ENOCUDA, std::string("cudaStreamSynchronize(cancel): ") + cudaGetErrorString(e));
        c->lanes[ticket].raised = false;
    }
    c->lanes[ticket].in_flight = false;
    c->cur = keep; c->b = &c->lanes[keep];
    return rc;
}

// raise the stop words idx[0, n) of parity lane `l` (idx = null: all B), in the host mirror and then by one H2D copy of the whole
// mirror on the cancel stream, ordered after the clear of the lane's current batch
static int raise_stop(ualm_ctx *c, Lane &l, int n, const int32_t *idx)
{
    const int B = l.batch.B;
    if (idx) for (int k = 0; k < n; k++) l.h_stop[idx[k]] = 1;
    else for (int b = 0; b < B; b++) l.h_stop[b] = 1;
    if (B == 0) return UALM_OK;
    CK(cudaStreamWaitEvent(c->cancel, l.ev_clear, 0));
    CK(cudaMemcpyAsync(l.d_stop.p, l.h_stop, sizeof(int) * B, cudaMemcpyHostToDevice, c->cancel));
    l.raised = true;
    return UALM_OK;
}

// deadline-bounded wait: poll the lane's completion until the timeout, then raise every stop word of its batch and wait for the
// batch to drain (every problem still running stops at its next stop test, include/ualm.h UALM_RET_STOPPED)
extern "C" int ualm_wait_batch_for(ualm_ctx_t *c, int ticket, double timeout_ms, ualm_result_t *results, double *c_xy, double *c_yaw)
{
    if (!c || ticket < 0 || ticket >= UALM_MAX_LANES) return fail(UALM_EINVAL, "bad ticket");
    if (!(timeout_ms >= 0.0)) return fail(UALM_EINVAL, "timeout_ms must be >= 0");
    if (c->tp) {
        if (!ualm_tp::tp_lane_in_flight(c->tp, ticket)) return fail(UALM_ESTATE, "ticket is not in flight");
        std::string em;
        const int rc = ualm_tp::tp_collect(c->tp, ticket, &em, timeout_ms);
        if (rc) return fail(rc, em);
        TP_CALL(ualm_tp::tp_download(c->tp, ticket, results, c_xy, c_yaw, err));
    }
    Lane &l = c->lanes[ticket];
    if (!l.in_flight) return fail(UALM_ESTATE, "ticket is not in flight");
    CK(cudaSetDevice(c->device));
    const auto t0 = std::chrono::steady_clock::now();
    while (true) {
        const cudaError_t q = cudaEventQuery(l.ev1);
        if (q == cudaSuccess) break;
        if (q != cudaErrorNotReady) CK(q);
        if (std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() >= timeout_ms) {
            if (int rc = raise_stop(c, l, 0, nullptr)) return rc;
            break;
        }
        std::this_thread::yield();
    }
    return ualm_wait_batch(c, ticket, results, c_xy, c_yaw);
}

// the problems of a submitted batch that have finished since the last poll of the ticket: read from the lane's mailbox, which the
// solve fills as each problem ends (ualm_mailbox.h).  wait_ms > 0: yield-poll the flags until one is new or the time is up
extern "C" int ualm_poll_batch(ualm_ctx_t *c, int ticket, double wait_ms, int32_t *idx, int *n_new, int *n_pending, ualm_result_t *results,
                               double *c_xy, double *c_yaw)
{
    if (!c || ticket < 0 || ticket >= UALM_MAX_LANES) return fail(UALM_EINVAL, "bad ticket");
    if (!(wait_ms >= 0.0)) return fail(UALM_EINVAL, "wait_ms must be >= 0");
    if (!idx || !n_new || !n_pending) return fail(UALM_EINVAL, "null argument");
    if (c->tp) TP_CALL(ualm_tp::tp_poll(c->tp, ticket, wait_ms, idx, n_new, n_pending, results, c_xy, c_yaw, err));
    Lane &l = c->lanes[ticket];
    if (!l.in_flight) return fail(UALM_ESTATE, "ticket is not in flight");
    CK(cudaSetDevice(c->device));
    const auto t0 = std::chrono::steady_clock::now();
    int n = 0;
    while (true) {
        n = l.mbox.collect(idx, results, c_xy, c_yaw);
        if (n > 0 || l.mbox.pending() == 0 || wait_ms == 0.0) break;
        const cudaError_t q = cudaEventQuery(l.ev1);     // a failed launch is reported, not waited out
        if (q != cudaSuccess && q != cudaErrorNotReady) CK(q);
        if (std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() >= wait_ms) break;
        std::this_thread::yield();
    }
    *n_new = n;
    *n_pending = l.mbox.pending();
    return UALM_OK;
}

// stop the problems idx[0, n) of a submitted batch at their next stop test: their words in the lane's host mirror, then the mirror to
// the device on a stream no solve occupies (the copy engines serve it while the kernels hold the SMs): the context's cancel stream on
// the parity path, the engine's on the throughput path.  Everything is checked before a word is raised
extern "C" int ualm_cancel_problems(ualm_ctx_t *c, int ticket, int n, const int32_t *idx)
{
    if (!c || ticket < 0 || ticket >= UALM_MAX_LANES) return fail(UALM_EINVAL, "bad ticket");
    if (n < 0) return fail(UALM_EINVAL, "n must be >= 0");
    if (n > 0 && !idx) return fail(UALM_EINVAL, "null idx");
    if (c->tp) TP_CALL(ualm_tp::tp_cancel(c->tp, ticket, n, idx, err));
    Lane &l = c->lanes[ticket];
    if (!l.in_flight) return fail(UALM_ESTATE, "ticket is not in flight");
    for (int k = 0; k < n; k++)
        if (idx[k] < 0 || idx[k] >= l.batch.B) return fail(UALM_EINVAL, "problem index out of range [0, B)");
    if (n == 0) return UALM_OK;
    CK(cudaSetDevice(c->device));
    return raise_stop(c, l, n, idx);
}

extern "C" int ualm_set_urgent(ualm_ctx_t *c, int urgent)
{
    if (!c) return fail(UALM_EINVAL, "null ctx");
    if (urgent != 0 && urgent != 1) return fail(UALM_EINVAL, "urgent must be 0 or 1");
    c->urgent = urgent == 1;
    return UALM_OK;
}

extern "C" int ualm_set_budget(ualm_ctx_t *c, int32_t max_evals)
{
    if (!c) return fail(UALM_EINVAL, "null ctx");
    if (max_evals < 0) return fail(UALM_EINVAL, "max_evals must be >= 0 (0 = no budget)");
    if (int rc = lanes_idle(c, "ualm_set_budget")) return rc;
    if (c->tp) ualm_tp::tp_set_budget(c->tp, max_evals);
    c->max_evals = max_evals;
    return UALM_OK;
}

// ---- one host process, several GPUs: contexts on different devices (same params and map set on each), the batch dealt over
// them (cost-sorted snake, like uneven_planner_b200/distributed.py), solved concurrently, results scattered back in problem order.
// No collective: a single host gathers by D2H copies.  (The one-process-per-GPU variant with an NCCL all-gather of result
// records is ualm_pack_records_device + the caller's communicator.) ----
extern "C" int ualm_solve_batch_multi(ualm_ctx_t **ctxs, int nctx, int B, const int32_t *N, const int32_t *M, const double *bnd,
                                      const double *total_time, const double *inner_xy, const double *inner_yaw, ualm_result_t *results,
                                      double *c_xy, double *c_yaw)
{
    return ualm_solve_batch_multi_env(ctxs, nctx, B, N, M, bnd, total_time, inner_xy, inner_yaw, nullptr, results, c_xy, c_yaw);
}
extern "C" int ualm_solve_batch_multi_env(ualm_ctx_t **ctxs, int nctx, int B, const int32_t *N, const int32_t *M, const double *bnd,
                                          const double *total_time, const double *inner_xy, const double *inner_yaw, const int32_t *env,
                                          ualm_result_t *results, double *c_xy, double *c_yaw)
{
    return ualm_solve_batch_multi_pp(ctxs, nctx, B, N, M, bnd, total_time, inner_xy, inner_yaw, env, nullptr, results, c_xy, c_yaw);
}
extern "C" int ualm_solve_batch_multi_pp(ualm_ctx_t **ctxs, int nctx, int B, const int32_t *N, const int32_t *M, const double *bnd,
                                         const double *total_time, const double *inner_xy, const double *inner_yaw, const int32_t *env,
                                         const ualm_problem_params_t *pp, ualm_result_t *results, double *c_xy, double *c_yaw)
{
    if (!ctxs || nctx < 1 || B < 0) return fail(UALM_EINVAL, "bad argument");
    for (int r = 0; r < nctx; r++) if (!ctxs[r]) return fail(UALM_EINVAL, "null ctx in list");
    if (B == 0) return UALM_OK;
    if (!N || !M || !bnd || !total_time) return fail(UALM_EINVAL, "null argument");
    BatchLayout L;       // checked against ctxs[0], the coefficient offsets of the whole batch
    if (int rc = batch_layout(ctxs[0], B, N, M, bnd, total_time, inner_xy, inner_yaw, env, pp, &L)) return rc;
    for (int r = 1; r < nctx; r++) if (int rc = check_envs(ctxs[r], B, env)) return rc;
    std::vector<long long> oxy(B + 1, 0), oyw(B + 1, 0);
    for (int b = 0; b < B; b++) { oxy[b + 1] = oxy[b] + 2LL * (N[b] - 1); oyw[b + 1] = oyw[b] + (M[b] - 1); }
    std::vector<int> ord(B);
    std::iota(ord.begin(), ord.end(), 0);
    std::stable_sort(ord.begin(), ord.end(), [&](int a, int b2) { return N[a] > N[b2]; });
    std::vector<std::vector<int>> shard(nctx);
    for (int pos = 0; pos < B; pos++) {
        const int rnd = pos / nctx, k = pos % nctx;
        shard[(rnd % 2 == 0) ? k : nctx - 1 - k].push_back(ord[pos]);
    }
    for (auto &s : shard) std::sort(s.begin(), s.end());
    struct Sub { std::vector<int32_t> N, M, E; std::vector<ualm_problem_params_t> P; std::vector<double> bnd, T, ixy, iyw, cxy, cyw; std::vector<ualm_result_t> res; };
    std::vector<Sub> sub(nctx);
    for (int r = 0; r < nctx; r++) {
        Sub &s = sub[r];
        for (int b : shard[r]) {
            s.N.push_back(N[b]); s.M.push_back(M[b]); s.T.push_back(total_time[b]); s.E.push_back(env ? env[b] : 0);
            if (pp) s.P.push_back(pp[b]);
            s.bnd.insert(s.bnd.end(), bnd + 18 * (size_t)b, bnd + 18 * (size_t)b + 18);
            if (oxy[b + 1] > oxy[b]) s.ixy.insert(s.ixy.end(), inner_xy + oxy[b], inner_xy + oxy[b + 1]);
            if (oyw[b + 1] > oyw[b]) s.iyw.insert(s.iyw.end(), inner_yaw + oyw[b], inner_yaw + oyw[b + 1]);
        }
        long long ncx = 0, ncy = 0;
        for (int b : shard[r]) { ncx += 12LL * N[b]; ncy += 6LL * M[b]; }
        s.cxy.assign(ncx, 0.0); s.cyw.assign(ncy, 0.0); s.res.resize(shard[r].size());
        if (s.ixy.empty()) s.ixy.push_back(0.0);
        if (s.iyw.empty()) s.iyw.push_back(0.0);
    }
    // upload + launch everywhere first (asynchronous per device), then collect
    for (int r = 0; r < nctx; r++) {
        if (shard[r].empty()) continue;
        int rc = ualm_upload_pp(ctxs[r], (int)shard[r].size(), sub[r].N.data(), sub[r].M.data(), sub[r].bnd.data(), sub[r].T.data(), sub[r].ixy.data(),
                                sub[r].iyw.data(), sub[r].E.data(), pp ? sub[r].P.data() : nullptr);
        if (!rc) rc = ualm_solve_resident(ctxs[r]);
        if (rc) return rc;
    }
    for (int r = 0; r < nctx; r++) {
        if (shard[r].empty()) continue;
        int rc = ualm_download(ctxs[r], sub[r].res.data(), sub[r].cxy.data(), sub[r].cyw.data());
        if (rc) return rc;
        long long px = 0, py = 0;
        for (size_t q = 0; q < shard[r].size(); q++) {
            const int b = shard[r][q];
            if (results) results[b] = sub[r].res[q];
            if (c_xy) memcpy(c_xy + L.off_cxy[b], sub[r].cxy.data() + px, sizeof(double) * 12 * N[b]);
            if (c_yaw) memcpy(c_yaw + L.off_cyaw[b], sub[r].cyw.data() + py, sizeof(double) * 6 * M[b]);
            px += 12LL * N[b]; py += 6LL * M[b];
        }
    }
    return UALM_OK;
}

extern "C" int ualm_pack_records_device(ualm_ctx_t *c, double *d_records, int stride)
{
    if (c && c->tp) {
        if (!d_records) return fail(UALM_EINVAL, "null buffer");
        TP_CALL(ualm_tp::tp_pack_records(c->tp, c->cur, d_records, stride, err));
    }
    if (!c || !c->b->solved || !d_records) return fail(UALM_ESTATE, "nothing solved / null buffer");
    Lane *l = c->b;
    if (stride < 12 + 12 * l->batch.Nmax + 6 * l->batch.Mmax) return fail(UALM_EINVAL, "record stride too small");
    CK(cudaSetDevice(c->device));
    if (l->batch.B > 0) {
        pack_records_kernel<<<l->batch.B, 128, 0, l->stream>>>(batch_ptrs(c), l->batch.B, d_records, stride);
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(l->stream));
    return UALM_OK;
}
// the same without the host-side wait (pipelined callers synchronise the lane themselves before reading the records)
extern "C" int ualm_pack_records_device_async(ualm_ctx_t *c, double *d_records, int stride)
{
    if (c && c->tp) return ualm_pack_records_device(c, d_records, stride);     // the engine gathers a batch only once it is complete
    if (!c || !c->b->solved || !d_records) return fail(UALM_ESTATE, "nothing solved / null buffer");
    Lane *l = c->b;
    if (stride < 12 + 12 * l->batch.Nmax + 6 * l->batch.Mmax) return fail(UALM_EINVAL, "record stride too small");
    CK(cudaSetDevice(c->device));
    if (l->batch.B > 0) {
        pack_records_kernel<<<l->batch.B, 128, 0, l->stream>>>(batch_ptrs(c), l->batch.B, d_records, stride);
        CK(cudaGetLastError());
    }
    return UALM_OK;
}

// upload an optional host array (or a constant fill) into a device buffer
static int put(ualm_ctx *c, double *dst, const double *src, size_t n, double fill)
{
    if (n == 0) return UALM_OK;
    if (src) { CK(cudaMemcpyAsync(dst, src, n * sizeof(double), cudaMemcpyHostToDevice, c->b->stream)); }
    else {
        std::vector<double> tmp(n, fill);
        CK(cudaMemcpyAsync(dst, tmp.data(), n * sizeof(double), cudaMemcpyHostToDevice, c->b->stream));
        CK(cudaStreamSynchronize(c->b->stream));
    }
    return UALM_OK;
}

extern "C" int ualm_eval_batch(ualm_ctx_t *c, const double *x, const double *lambda, const double *mu, const double *scale_cx,
                               const double *scale_fx, double rho, double *f, double *grad, double *hx, double *gx, double *c_xy,
                               double *c_yaw)
{
    if (c && c->tp) TP_CALL(ualm_tp::tp_eval(c->tp, c->cur, x, lambda, mu, scale_cx, scale_fx, rho, f, grad, hx, gx, c_xy, c_yaw, err));
    if (!c || !c->b->have_batch) return fail(UALM_ESTATE, "upload and set_map first");
    Lane *l = c->b;
    const BatchLayout &L = l->batch;
    if (L.n_active != L.B) return fail(UALM_ELIMIT, "ualm_eval_batch: the uploaded batch holds problems over the compiled limits");
    CK(cudaSetDevice(c->device));
    int rc;
    // the evaluation point goes to its own buffer: d_x0 keeps the uploaded initial guesses, which ualm_init_scaling_batch and a
    // later solve of the resident batch start from
    if (x) {
        CK(l->d_xev.ensure(L.tot_x));
        if ((rc = put(c, l->d_xev.p, x, L.tot_x, 0.0))) return rc;
    }
    if ((rc = put(c, l->d_lambda.p, lambda, L.tot_s, 0.0))) return rc;
    if ((rc = put(c, l->d_mu.p, mu, 6 * L.tot_s, 0.0))) return rc;
    if ((rc = put(c, l->d_scale_cx.p, scale_cx, 7 * L.tot_s, 1.0))) return rc;
    if ((rc = put(c, l->d_sfx.p, scale_fx, L.B, 1.0))) return rc;
    if (L.B > 0) {
        if ((rc = per_env(c, [&](int e, const BatchPtrs &bp, int cnt) {
                 BatchPtrs be = bp;
                 if (x) be.x0 = l->d_xev.p;
                 const int wpb = l->ewpb[e];
                 eval_kernel<<<(cnt + wpb - 1) / wpb, UALM_THREADS * wpb, l->esmem[e], l->stream>>>(be, c->envs[e].dp, c->envs[e].map->dm, l->eL[e], rho);
             })))
            return rc;
        if (f) CK(cudaMemcpyAsync(f, l->d_f.p, sizeof(double) * L.B, cudaMemcpyDeviceToHost, l->stream));
        if (grad) CK(cudaMemcpyAsync(grad, l->d_grad.p, sizeof(double) * L.tot_x, cudaMemcpyDeviceToHost, l->stream));
        if (hx) CK(cudaMemcpyAsync(hx, l->d_hx.p, sizeof(double) * L.tot_s, cudaMemcpyDeviceToHost, l->stream));
        if (gx) CK(cudaMemcpyAsync(gx, l->d_gx.p, sizeof(double) * 6 * L.tot_s, cudaMemcpyDeviceToHost, l->stream));
        if (c_xy) CK(cudaMemcpyAsync(c_xy, l->d_cxy.p, sizeof(double) * L.tot_cxy, cudaMemcpyDeviceToHost, l->stream));
        if (c_yaw) CK(cudaMemcpyAsync(c_yaw, l->d_cyaw.p, sizeof(double) * L.tot_cyaw, cudaMemcpyDeviceToHost, l->stream));
    }
    CK(cudaStreamSynchronize(l->stream));
    return UALM_OK;
}

extern "C" int ualm_init_scaling_batch(ualm_ctx_t *c, double *scale_fx, double *scale_cx)
{
    if (c && c->tp) TP_CALL(ualm_tp::tp_init_scaling(c->tp, c->cur, scale_fx, scale_cx, err));
    if (!c || !c->b->have_batch) return fail(UALM_ESTATE, "upload and set_map first");
    Lane *l = c->b;
    const BatchLayout &L = l->batch;
    if (L.n_active != L.B) return fail(UALM_ELIMIT, "ualm_init_scaling_batch: the uploaded batch holds problems over the compiled limits");
    CK(cudaSetDevice(c->device));
    if (L.B > 0) {
        if (int rc = per_env(c, [&](int e, const BatchPtrs &bp, int cnt) {
                const int wpb = l->ewpb[e];
                scaling_kernel<<<(cnt + wpb - 1) / wpb, UALM_THREADS * wpb, l->esmem[e], l->stream>>>(bp, c->envs[e].dp, c->envs[e].map->dm, l->eL[e]);
            }))
            return rc;
        if (scale_fx) CK(cudaMemcpyAsync(scale_fx, l->d_sfx.p, sizeof(double) * L.B, cudaMemcpyDeviceToHost, l->stream));
        if (scale_cx) CK(cudaMemcpyAsync(scale_cx, l->d_scale_cx.p, sizeof(double) * 7 * L.tot_s, cudaMemcpyDeviceToHost, l->stream));
    }
    CK(cudaStreamSynchronize(l->stream));
    return UALM_OK;
}

extern "C" int ualm_time_penalty_kernel(ualm_ctx_t *c, int reps, float *ms_per_launch, double *algorithmic_bytes)
{
    if (reps < 1) return fail(UALM_EINVAL, "reps < 1");
    if (c && c->tp) TP_CALL(ualm_tp::tp_time_penalty(c->tp, c->cur, reps, (getenv("UALM_TP_TMA") && atoi(getenv("UALM_TP_TMA"))) ? 1 : 0, ms_per_launch, algorithmic_bytes, err));
    if (!c || !c->b->have_batch) return fail(UALM_ESTATE, "upload and set_map first");
    Lane *l = c->b;
    const BatchLayout &L = l->batch;
    if (L.n_active != L.B) return fail(UALM_ELIMIT, "ualm_time_penalty_kernel: the uploaded batch holds problems over the compiled limits");
    if (L.mixed()) return fail(UALM_EINVAL, "ualm_time_penalty_kernel: the uploaded batch mixes environments");
    if (ms_per_launch) *ms_per_launch = 0.f;
    if (algorithmic_bytes) *algorithmic_bytes = 0.0;
    if (L.B == 0) return UALM_OK;
    CK(cudaSetDevice(c->device));
    int rc;
    if ((rc = put(c, l->d_lambda.p, nullptr, L.tot_s, 0.0))) return rc;
    if ((rc = put(c, l->d_mu.p, nullptr, 6 * L.tot_s, 0.0))) return rc;
    if ((rc = put(c, l->d_scale_cx.p, nullptr, 7 * L.tot_s, 1.0))) return rc;
    const int e = L.env[0];
    const BatchPtrs bp = batch_ptrs(c);
    const int wpb = l->ewpb[e];
    penalty_only_kernel<<<(L.B + wpb - 1) / wpb, UALM_THREADS * wpb, l->esmem[e], l->stream>>>(bp, c->envs[e].dp, c->envs[e].map->dm, l->eL[e], 1); // warm-up
    CK(cudaEventRecord(l->ev0, l->stream));
    penalty_only_kernel<<<(L.B + wpb - 1) / wpb, UALM_THREADS * wpb, l->esmem[e], l->stream>>>(bp, c->envs[e].dp, c->envs[e].map->dm, l->eL[e], reps);
    CK(cudaEventRecord(l->ev1, l->stream));
    CK(cudaGetLastError());
    CK(cudaEventSynchronize(l->ev1));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, l->ev0, l->ev1));
    if (ms_per_launch) *ms_per_launch = ms / reps;
    if (algorithmic_bytes) {
        // SURVEY 8d: per trajectory per evaluation S*45e + (25N + 13M)e
        double bytes = 0;
        for (auto &d : l->desc) bytes += (double)d.S * 45 * 8 + (25.0 * d.N + 13.0 * d.M) * 8;
        *algorithmic_bytes = bytes;
    }
    return UALM_OK;
}

// developer aid: per-phase SM cycle counters of the last solve (thread 0 of every CTA), summed over the batch.
// enable != 0 turns collection on for subsequent solves; out16 (may be NULL) receives the sums of the last solve.
extern "C" int ualm_profile(ualm_ctx_t *c, int enable, long long *out16)
{
    if (!c) return fail(UALM_EINVAL, "null ctx");
    if (c->tp) TP_UNSUPPORTED("ualm_profile");
    Lane *l = c->b;
    CK(cudaSetDevice(c->device));
    if (out16 && c->profile && l->solved && l->batch.B > 0) {
        std::vector<long long> h((size_t)l->batch.B * UALM_NPROF);
        CK(cudaMemcpyAsync(h.data(), l->d_prof.p, h.size() * sizeof(long long), cudaMemcpyDeviceToHost, l->stream));
        CK(cudaStreamSynchronize(l->stream));
        if (enable == 2) { // raw: out16 has room for B x 16 values, rows in problem order
            for (size_t q = 0; q < h.size(); q++) out16[q] = h[q];
        } else {
            for (int q = 0; q < UALM_NPROF; q++) out16[q] = 0;
            for (int b = 0; b < l->batch.B; b++) if (!l->batch.skip[b]) for (int q = 0; q < UALM_NPROF; q++) out16[q] += h[(size_t)b * UALM_NPROF + q];
        }
    }
    c->profile = enable != 0;
    return UALM_OK;
}

namespace ualm {
__global__ void piece_T_from_results(const ualm_result_t *res, int B, double *piece_T)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B) { piece_T[2 * b] = res[b].piece_T_xy; piece_T[2 * b + 1] = res[b].piece_T_yaw; }
}
} // namespace ualm

// descriptors of a scan over B trajectories of N[b] / M[b] pieces whose coefficients are packed in problem order; S == 0 marks a problem
// over the compiled limits, which is not scanned.  pp[2..7] carry the six limits check_kernel tests: `limits` when given, else the
// problem's parameter row (rows: 8 doubles each, as ualm_problem_params_t; null = none), else its environment's
static_assert(sizeof(ualm_limits_t) == 6 * sizeof(double), "ualm_problem_params_t's six limits, in its order");
static std::vector<ProbDesc> scan_descs(const ualm_ctx *c, int B, const int32_t *N, const int32_t *M, const int32_t *env, const double *rows,
                                        const ualm_limits_t *limits)
{
    std::vector<ProbDesc> desc(B);
    long long ocx = 0, ocy = 0;
    for (int b = 0; b < B; b++) {
        memset(&desc[b], 0, sizeof(ProbDesc));
        desc[b].N = N[b]; desc[b].M = M[b]; desc[b].off_cxy = ocx; desc[b].off_cyaw = ocy;
        desc[b].S = over_limits(N[b], M[b]) ? 0 : 1;
        memcpy(desc[b].pp, rows ? rows + 8 * (size_t)b : &c->envs[env ? env[b] : 0].hp.rho_T, 8 * sizeof(double));
        if (limits) memcpy(desc[b].pp + 2, limits, sizeof(ualm_limits_t));
        ocx += 12LL * N[b]; ocy += 6LL * M[b];
    }
    return desc;
}

// a collected throughput batch as the BatchPtrs of the scans (feasibility, MPC export): descriptors of the lane's layout and piece
// durations from the records, in device buffers this object owns, with the scan's index list and rows
struct TpScan {
    DevBuf<ProbDesc> desc;
    DevBuf<double> pt, feas;
    DevBuf<int> idx;
    BatchPtrs bp;
    ~TpScan() { desc.release(); pt.release(); feas.release(); idx.release(); }
};
// what: the entry point, for the refusal of a lane with no collected batch
static int tp_scan(ualm_ctx *c, const char *what, TpScan &s)
{
    const ualm_result_t *d_res; const double *d_cxy, *d_cyaw;
    if (ualm_tp::tp_lane_outputs(c->tp, c->cur, &d_res, &d_cxy, &d_cyaw) != UALM_OK)
        return fail(UALM_ESTATE, std::string(what) + " needs a solved, collected batch (ualm_sync / ualm_download first)");
    CK(cudaSetDevice(c->device));
    const BatchLayout &L = c->b->batch;
    if (L.B == 0) return UALM_OK;
    const std::vector<ProbDesc> desc = scan_descs(c, L.B, L.N.data(), L.M.data(), L.env.data(), L.pp.data(), nullptr);
    CK(s.desc.ensure(L.B)); CK(s.pt.ensure(2 * (size_t)L.B));
    CK(cudaMemcpy(s.desc.p, desc.data(), sizeof(ProbDesc) * L.B, cudaMemcpyHostToDevice));
    piece_T_from_results<<<(L.B + 127) / 128, 128>>>(d_res, L.B, s.pt.p);
    memset(&s.bp, 0, sizeof(s.bp));
    s.bp.B = L.B; s.bp.desc = s.desc.p; s.bp.c_xy = const_cast<double *>(d_cxy); s.bp.c_yaw = const_cast<double *>(d_cyaw); s.bp.piece_T = s.pt.p;
    return UALM_OK;
}

// check_kernel once per environment present: over its problems d_idx[eoff[e], eoff[e + 1]), against grid version maps[e] with its gravity
static int scan_launch(ualm_ctx *c, const CheckPtrs &a, const int *d_idx, const int *eoff, const MapRef *maps, double dt, cudaStream_t st)
{
    for (int e = 0; e < UALM_MAX_ENVS; e++) {
        const int cnt = eoff[e + 1] - eoff[e];
        if (cnt == 0) continue;
        check_kernel<<<(cnt + UALM_WPB - 1) / UALM_WPB, UALM_THREADS * UALM_WPB, 0, st>>>(a, maps[e]->dm, c->envs[e].dp.gravity, dt, d_idx + eoff[e], cnt);
        CK(cudaGetLastError());
    }
    return UALM_OK;
}

// the scan of the lane's solved batch, every sample, on the grid versions it was solved on.  A problem over the compiled limits was
// not solved: its row is zeros
extern "C" int ualm_feasibility_batch(ualm_ctx_t *c, double dt, double *out10)
{
    if (!c || !out10 || !(dt > 0.0)) return fail(UALM_EINVAL, "null argument or dt <= 0");
    Lane *l = c->b;
    const BatchLayout &L = l->batch;
    TpScan s;
    CheckPtrs a{};
    const int *d_idx;
    cudaStream_t st;
    if (c->tp) {
        if (int rc = tp_scan(c, "ualm_feasibility_batch", s)) return rc;
        if (L.B == 0) return UALM_OK;
        CK(s.feas.ensure(16 * (size_t)L.B)); CK(s.idx.ensure(L.B));
        CK(cudaMemcpy(s.idx.p, L.eidx.data(), sizeof(int) * L.B, cudaMemcpyHostToDevice));
        a.desc = s.bp.desc; a.c_xy = s.bp.c_xy; a.c_yaw = s.bp.c_yaw; a.piece_T = s.bp.piece_T; a.out = s.feas.p;
        d_idx = s.idx.p; st = 0;
    } else {
        if (!l->have_batch || !l->solved) return fail(UALM_ESTATE, "ualm_feasibility_batch needs a solved resident batch");
        CK(cudaSetDevice(c->device));
        if (L.B == 0) return UALM_OK;
        const BatchPtrs bp = batch_ptrs(c);
        a.desc = bp.desc; a.c_xy = bp.c_xy; a.c_yaw = bp.c_yaw; a.piece_T = bp.piece_T; a.out = l->d_feas.p;
        d_idx = l->d_eidx.p; st = l->stream;
    }
    for (int e = 0; e < UALM_MAX_ENVS; e++)
        if (((L.env_mask >> e) & 1u) && !l->vref[e]) return fail(UALM_ESTATE, "ualm_feasibility_batch: the batch was not solved by a launch of this context");
    if (int rc = scan_launch(c, a, d_idx, L.eoff, l->vref, dt, st)) return rc;
    CK(cudaMemcpy2DAsync(out10, 10 * sizeof(double), a.out, 16 * sizeof(double), 10 * sizeof(double), L.B, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (int b = 0; b < L.B; b++) if (L.skip[b]) memset(out10 + 10 * (size_t)b, 0, 10 * sizeof(double));
    return UALM_OK;
}

// the check stream (ualm_ctx::cstream), made at first use
static int check_stream(ualm_ctx *c)
{
    if (!c->cstream) {
        int least = 0, greatest = 0;
        CK(cudaDeviceGetStreamPriorityRange(&least, &greatest));
        CK(cudaStreamCreateWithPriority(&c->cstream, cudaStreamNonBlocking, greatest));
    }
    return UALM_OK;
}
// cbuf of at least `bytes`, grown in stream order on the check stream: the old block is freed behind the work that used it
static int check_block(ualm_ctx *c, size_t bytes)
{
    if (c->cbuf_bytes < bytes) {
        if (c->cbuf) CK(cudaFreeAsync(c->cbuf, c->cstream));
        c->cbuf = nullptr; c->cbuf_bytes = 0;
        CK(cudaMallocAsync(&c->cbuf, bytes, c->cstream));
        c->cbuf_bytes = bytes;
    }
    return UALM_OK;
}

// Trajectories the caller holds (ualm_check_trajectories, ualm_submit_replan, ualm_mpc_export_trajectories), in the layouts
// ualm_wait_batch returns
struct Held {
    int B;
    const int32_t *N, *M;
    const double *piece_T, *c_xy, *c_yaw, *t_from;     // t_from: null = 0 for every row (the check only)
    long long ncx = 0, ncy = 0;                          // coefficients, 12 N and 6 M summed (held_counts)
};
// every row has N, M >= 1; counts the coefficients
static int held_counts(const char *what, Held &h)
{
    for (int b = 0; b < h.B; b++) {
        if (h.N[b] < 1 || h.M[b] < 1) return fail(UALM_EINVAL, std::string(what) + ": piece counts must be >= 1");
        h.ncx += 12LL * h.N[b]; h.ncy += 6LL * h.M[b];
    }
    return UALM_OK;
}
// h staged on the check stream in the context's block, grown in stream order: out (nout doubles) | piece_T 2B | t_from B | rows, rw
// per problem (when given: a replan's bnd, 18; the MPC's boundary derivatives, 6) | c_xy | c_yaw, then the descriptors, then B ints of
// idx (when given).  Under urgent work the hold of the check stream (urgent: unarmed, on that stream) is raised before the copies; the
// caller lowers it behind its kernel (hold_lower), `urgent` on any earlier exit.  a: the block as check_kernel reads it
struct Staged { CheckPtrs a; double *rows; int *idx; };
static int stage_held(ualm_ctx *c, const Held &h, const std::vector<ProbDesc> &desc, size_t nout, const double *rows, int rw, const std::vector<int> *idx,
                      HoldGuard &urgent, Staged &s)
{
    const int B = h.B;
    const cudaStream_t st = c->cstream;
    if (c->urgent && c->d_hold) {     // (parity path: the throughput path has no hold)
        if (int rc = hold_set(c, UALM_MAX_LANES, 1, st)) return rc;
        urgent.armed = true;
    }
    const size_t nrows = rows ? (size_t)rw * B : 0, nd = nout + 3 * (size_t)B + nrows + (size_t)h.ncx + (size_t)h.ncy;
    if (int rc = check_block(c, sizeof(double) * nd + sizeof(ProbDesc) * B + (idx ? sizeof(int) * B : 0))) return rc;
    double *d_out = (double *)c->cbuf, *d_pt = d_out + nout, *d_tf = d_pt + 2 * (size_t)B, *d_rows = d_tf + B, *d_cxy = d_rows + nrows,
           *d_cyaw = d_cxy + h.ncx;
    ProbDesc *d_desc = (ProbDesc *)(d_out + nd);
    int *d_idx = (int *)(d_desc + B);
    CK(cudaMemcpyAsync(d_pt, h.piece_T, sizeof(double) * 2 * B, cudaMemcpyHostToDevice, st));
    if (h.t_from) CK(cudaMemcpyAsync(d_tf, h.t_from, sizeof(double) * B, cudaMemcpyHostToDevice, st));
    if (rows) CK(cudaMemcpyAsync(d_rows, rows, sizeof(double) * nrows, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_cxy, h.c_xy, sizeof(double) * h.ncx, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_cyaw, h.c_yaw, sizeof(double) * h.ncy, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_desc, desc.data(), sizeof(ProbDesc) * B, cudaMemcpyHostToDevice, st));
    if (idx) CK(cudaMemcpyAsync(d_idx, idx->data(), sizeof(int) * B, cudaMemcpyHostToDevice, st));
    s.a.desc = d_desc; s.a.c_xy = d_cxy; s.a.c_yaw = d_cyaw; s.a.piece_T = d_pt; s.a.t_from = h.t_from ? d_tf : nullptr; s.a.out = d_out;
    s.rows = rows ? d_rows : nullptr;
    s.idx = idx ? d_idx : nullptr;
    return UALM_OK;
}
// lowers a raised hold in the order of its stream, here rather than on exit
static int hold_lower(HoldGuard &g)
{
    if (!g.armed) return UALM_OK;
    g.armed = false;
    return hold_set(g.c, g.slot, 0, g.st);
}

// check_kernel over host trajectories, on the context's check stream, against each environment's grid version current at the call.
// The context's block (cbuf) grows in stream order on that stream, and the versions are let go only after cdone (as lane_hold lets
// go), so nothing here waits for a batch in flight
extern "C" int ualm_check_trajectories(ualm_ctx_t *c, int B, const int32_t *N, const int32_t *M, const double *piece_T, const double *c_xy,
                                       const double *c_yaw, const int32_t *env, const double *t_from, double dt, const ualm_limits_t *limits,
                                       double *out16)
{
    return ualm_check_trajectories_pp(c, B, N, M, piece_T, c_xy, c_yaw, env, nullptr, t_from, dt, limits, out16);
}
extern "C" int ualm_check_trajectories_pp(ualm_ctx_t *c, int B, const int32_t *N, const int32_t *M, const double *piece_T, const double *c_xy,
                                          const double *c_yaw, const int32_t *env, const ualm_problem_params_t *pp, const double *t_from, double dt,
                                          const ualm_limits_t *limits, double *out16)
{
    if (!c || B < 0 || (B > 0 && (!N || !M || !piece_T || !c_xy || !c_yaw || !out16))) return fail(UALM_EINVAL, "ualm_check_trajectories: null argument or B < 0");
    if (!(dt > 0.0)) return fail(UALM_EINVAL, "ualm_check_trajectories: dt must be > 0");
    Held held{B, N, M, piece_T, c_xy, c_yaw, t_from};
    if (int rc = held_counts("ualm_check_trajectories", held)) return rc;
    for (int b = 0; t_from && b < B; b++)
        if (!(t_from[b] >= 0.0)) return fail(UALM_EINVAL, "ualm_check_trajectories: t_from must be >= 0 (and not NaN)");
    if (int rc = check_pp(B, pp)) return rc;
    if (B == 0) return UALM_OK;
    if (int rc = check_envs(c, B, env)) return rc;
    CK(cudaSetDevice(c->device));
    if (int rc = check_stream(c)) return rc;
    if (!c->cdone) CK(cudaEventCreateWithFlags(&c->cdone, cudaEventDisableTiming));
    // problems grouped by environment, and the grid version each environment has now
    std::vector<int> idx;
    int off[UALM_MAX_ENVS + 1];
    group_by_env(B, env, idx, off);
    MapRef hold[UALM_MAX_ENVS];
    for (int e = 0; e < UALM_MAX_ENVS; e++) if (off[e + 1] > off[e]) hold[e] = c->envs[e].map;
    const std::vector<ProbDesc> desc = scan_descs(c, B, N, M, env, pp ? &pp[0].rho_T : nullptr, limits);
    // declared after hold: on every exit cdone is recorded behind the kernels before the versions are let go
    struct Done {
        ualm_ctx *c;
        ~Done() { if (cudaEventRecord(c->cdone, c->cstream) == cudaSuccess) cudaStreamWaitEvent(c->fstream, c->cdone, 0); }
    } done{c};
    HoldGuard urgent{c, UALM_MAX_LANES, c->cstream, false};
    Staged s;
    if (int rc = stage_held(c, held, desc, 16 * (size_t)B, nullptr, 0, &idx, urgent, s)) return rc;
    if (int rc = scan_launch(c, s.a, s.idx, off, hold, dt, c->cstream)) return rc;
    if (int rc = hold_lower(urgent)) return rc;
    CK(cudaMemcpyAsync(out16, s.a.out, sizeof(double) * 16 * B, cudaMemcpyDeviceToHost, c->cstream));
    CK(cudaStreamSynchronize(c->cstream));
    return UALM_OK;
}

// replan_kernel on the check stream (it reads no grid, so no version is held), then the built arrays go through ualm_submit_batch_env.
// Every refusal but one is decided before the build; that one (a polyline whose length gives no usable total_time) is decided before any
// output is written or lane taken
extern "C" int ualm_submit_replan(ualm_ctx_t *c, int B, const int32_t *N, const int32_t *M, const double *piece_T, const double *c_xy,
                                  const double *c_yaw, const double *bnd, const int32_t *env, const double *t_from, double dt,
                                  const ualm_resample_params_t *rp, int depth, int *ticket, int32_t *N_out, int32_t *M_out, double *bnd_out,
                                  double *total_time_out, double *inner_xy_out, double *inner_yaw_out)
{
    return ualm_submit_replan_pp(c, B, N, M, piece_T, c_xy, c_yaw, bnd, env, nullptr, t_from, dt, rp, depth, ticket, N_out, M_out, bnd_out,
                                 total_time_out, inner_xy_out, inner_yaw_out);
}
extern "C" int ualm_submit_replan_pp(ualm_ctx_t *c, int B, const int32_t *N, const int32_t *M, const double *piece_T, const double *c_xy,
                                     const double *c_yaw, const double *bnd, const int32_t *env, const ualm_problem_params_t *pp, const double *t_from,
                                     double dt, const ualm_resample_params_t *rp, int depth, int *ticket, int32_t *N_out, int32_t *M_out,
                                     double *bnd_out, double *total_time_out, double *inner_xy_out, double *inner_yaw_out)
{
    if (!c || !ticket || B < 0 || (B > 0 && (!N || !M || !piece_T || !c_xy || !c_yaw || !bnd || !t_from || !N_out || !M_out || !bnd_out || !total_time_out)))
        return fail(UALM_EINVAL, "ualm_submit_replan: null argument or B < 0");
    if (!(dt > 0.0)) return fail(UALM_EINVAL, "ualm_submit_replan: dt must be > 0");
    if (depth < 1 || depth > UALM_MAX_LANES) return fail(UALM_EINVAL, "ualm_submit_replan: depth out of range [1, UALM_MAX_LANES]");
    if (int rc = check_pp(B, pp)) return rc;
    const ualm_resample_params_t r = rp ? *rp : ualm_resample_params_t{0.3, 2.0, 0.5, 1.2, 0.0};   // run_*.yaml manager/*
    if (!(r.piece_len > 0.0) || !(r.yaw_piece_times > 0.0) || !(r.mean_vel > 0.0) || !(r.init_time_times > 0.0))
        return fail(UALM_EINVAL, "ualm_submit_replan: piece_len, yaw_piece_times, mean_vel and init_time_times must be > 0");
    Held held{B, N, M, piece_T, c_xy, c_yaw, t_from};
    if (int rc = held_counts("ualm_submit_replan", held)) return rc;
    for (int b = 0; b < B; b++) {
        const TrajDur d = traj_duration(N[b], M[b], piece_T[2 * b], piece_T[2 * b + 1]);    // replan_kernel's duration
        if (!(t_from[b] >= 0.0) || !(t_from[b] < d.total)) return fail(UALM_EINVAL, "ualm_submit_replan: t_from must be in [0, the trajectory's duration)");
        if (!d.scannable(dt)) return fail(UALM_EINVAL, "ualm_submit_replan: duration / dt must be < 4e6");
        if (!std::isfinite(piece_T[2 * b]) || !std::isfinite(piece_T[2 * b + 1])) return fail(UALM_EINVAL, "ualm_submit_replan: piece_T must be finite");
        for (int k : {6, 7, 8, 9, 10, 11, 15, 16, 17})      // the goal entries bnd' takes
            if (!std::isfinite(bnd[18 * (size_t)b + k])) return fail(UALM_EINVAL, "ualm_submit_replan: the goal entries of bnd must be finite");
    }
    // a diverged solve's coefficients: refused, not sampled
    for (long long q = 0; q < held.ncx; q++) if (!std::isfinite(c_xy[q])) return fail(UALM_EINVAL, "ualm_submit_replan: c_xy must be finite");
    for (long long q = 0; q < held.ncy; q++) if (!std::isfinite(c_yaw[q])) return fail(UALM_EINVAL, "ualm_submit_replan: c_yaw must be finite");
    if (B == 0) return ualm_submit_batch_pp(c, 0, N_out, M_out, bnd_out, total_time_out, nullptr, nullptr, env, pp, depth, ticket);
    if (int rc = check_envs(c, B, env)) return rc;
    if (lane_in_flight(c, c->next_submit % depth)) return fail(UALM_ESTATE, "all lanes of this depth are in flight: ualm_wait_batch the oldest ticket first");
    CK(cudaSetDevice(c->device));
    if (int rc = check_stream(c)) return rc;
    const std::vector<ProbDesc> desc = scan_descs(c, B, N, M, env, nullptr, nullptr);      // (replan_kernel reads neither S nor the limits)
    const size_t nout = (size_t)UALM_REPLAN_STRIDE * B;
    const cudaStream_t st = c->cstream;
    // urgent: the hold is lowered behind the build's kernel before any refusal can follow; the ticket is urgent by itself
    // (ualm_submit_batch_env)
    HoldGuard urgent{c, UALM_MAX_LANES, st, false};
    Staged s;
    if (int rc = stage_held(c, held, desc, nout, bnd, 18, nullptr, urgent, s)) return rc;
    ReplanPtrs a;
    a.desc = s.a.desc; a.c_xy = s.a.c_xy; a.c_yaw = s.a.c_yaw; a.piece_T = s.a.piece_T; a.bnd = s.rows; a.t_from = s.a.t_from; a.out = s.a.out;
    const ReplanParams p{dt, r.piece_len, r.yaw_piece_times, r.mean_vel, r.init_time_times};
    replan_kernel<<<(B + UALM_WPB - 1) / UALM_WPB, UALM_THREADS * UALM_WPB, 0, st>>>(a, p, B);
    CK(cudaGetLastError());
    if (int rc = hold_lower(urgent)) return rc;
    std::vector<double> h(nout);
    CK(cudaMemcpyAsync(h.data(), s.a.out, sizeof(double) * nout, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    // the one refusal after the build, before any output: a polyline of zero or non-finite length (a robot already at its goal, or
    // coordinates so large that their squares overflow) has no total_time ualm_submit_batch_env would take
    for (int b = 0; b < B; b++) {
        const double T = h[(size_t)UALM_REPLAN_STRIDE * b + 18];
        if (!(T > 0.0) || !std::isfinite(T)) return fail(UALM_EINVAL, "ualm_submit_replan: row " + std::to_string(b) + "'s polyline has zero or non-finite length");
    }
    // the outputs, and the packed inner arrays ualm_submit_batch_env takes (a row over the limits: zeros, never read).  The stream's
    // bound keeps N', M' <= UALM_RS_MAX_WAYPOINTS + 2
    long long pxy = 0, pyaw = 0;
    for (int b = 0; b < B; b++) {
        const double *o = &h[(size_t)UALM_REPLAN_STRIDE * b];
        N_out[b] = (int32_t)o[19]; M_out[b] = (int32_t)o[20];
        memcpy(bnd_out + 18 * (size_t)b, o, sizeof(double) * 18);
        total_time_out[b] = o[18];
        if (inner_xy_out) memcpy(inner_xy_out + (size_t)UALM_REPLAN_INNER_XY * b, o + 21, sizeof(double) * UALM_REPLAN_INNER_XY);
        if (inner_yaw_out) memcpy(inner_yaw_out + (size_t)UALM_REPLAN_INNER_YAW * b, o + 21 + UALM_REPLAN_INNER_XY, sizeof(double) * UALM_REPLAN_INNER_YAW);
        pxy += 2LL * (N_out[b] - 1); pyaw += M_out[b] - 1;
    }
    std::vector<double> ixy((size_t)pxy, 0.0), iyaw((size_t)pyaw, 0.0);
    pxy = pyaw = 0;
    for (int b = 0; b < B; b++) {
        const double *o = &h[(size_t)UALM_REPLAN_STRIDE * b];
        const long long nxy = 2LL * (N_out[b] - 1), nyaw = M_out[b] - 1;
        if (!over_limits(N_out[b], M_out[b])) {
            memcpy(ixy.data() + pxy, o + 21, sizeof(double) * nxy);
            memcpy(iyaw.data() + pyaw, o + 21 + UALM_REPLAN_INNER_XY, sizeof(double) * nyaw);
        }
        pxy += nxy; pyaw += nyaw;
    }
    return ualm_submit_batch_pp(c, B, N_out, M_out, bnd_out, total_time_out, ixy.data(), iyaw.data(), env, pp, depth, ticket);
}

// ---------------------------------------------------------------------------------------------
// SURVEY 8f-3: SE2Traj message + the MPC side's MINCO re-solve + planned-vs-tracked deviation for a solved batch (mpc_export_kernel)
// ---------------------------------------------------------------------------------------------
// doubles of mpc_export_run's device block for B problems of sN xy and sM yaw pieces in all: the seven outputs, then the band scratch
static size_t mpc_export_doubles(int B, long long sN, long long sM)
{
    return 2 * (size_t)(sN + B) + (size_t)sN + (size_t)(sM + B) + (size_t)sM + 12 * (size_t)sN + 6 * (size_t)sM + 4 * (size_t)B +
           13 * (6 * (size_t)sN + 6 * (size_t)sM);
}
// mpc_export_kernel over bp's B problems on stream st, its outputs and scratch in `block` (mpc_export_doubles), then the outputs to the
// host.  The boundary derivatives: d_init_rows (device, 6 per problem, MpcOut) when given, else init_v / init_a for every problem
// (null = zero).  `urgent` is lowered behind the kernel, before the copies
static int mpc_export_run(const BatchPtrs &bp, long long sN, long long sM, double dt, const double *init_v, const double *init_a,
                          const double *d_init_rows, double *block, double *pos_pts, double *posT_pts, double *angle_pts, double *angleT_pts,
                          double *c_mpc_xy, double *c_mpc_yaw, double *dev4, cudaStream_t st, HoldGuard &urgent)
{
    const int B = bp.B;
    const size_t n_pp = 2 * (size_t)(sN + B), n_pt = (size_t)sN, n_ap = (size_t)(sM + B), n_at = (size_t)sM, n_cx = 12 * (size_t)sN, n_cy = 6 * (size_t)sM, n_dv = 4 * (size_t)B;
    MpcOut o;
    double *q = block;
    o.pos_pts = q; q += n_pp; o.posT_pts = q; q += n_pt; o.angle_pts = q; q += n_ap; o.angleT_pts = q; q += n_at;
    o.c_mpc_xy = q; q += n_cx; o.c_mpc_yaw = q; q += n_cy; o.dev = q; q += n_dv; o.band = q;
    o.init_rows = d_init_rows;
    for (int k = 0; k < 3; k++) { o.init[k] = init_v ? init_v[k] : 0.0; o.init[3 + k] = init_a ? init_a[k] : 0.0; }
    mpc_export_kernel<<<(B + UALM_WPB - 1) / UALM_WPB, UALM_THREADS * UALM_WPB, 0, st>>>(bp, dt, o);
    CK(cudaGetLastError());
    if (int rc = hold_lower(urgent)) return rc;
    struct { double *h; const double *d; size_t n; } cp[7] = {{pos_pts, o.pos_pts, n_pp}, {posT_pts, o.posT_pts, n_pt}, {angle_pts, o.angle_pts, n_ap},
        {angleT_pts, o.angleT_pts, n_at}, {c_mpc_xy, o.c_mpc_xy, n_cx}, {c_mpc_yaw, o.c_mpc_yaw, n_cy}, {dev4, o.dev, n_dv}};
    for (auto &e : cp) if (e.h && e.n) CK(cudaMemcpyAsync(e.h, e.d, sizeof(double) * e.n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return UALM_OK;
}
// the lane form: its block from cudaMalloc, freed on return
static int mpc_export_lane(ualm_ctx *c, const BatchPtrs &bp, const BatchLayout &L, double dt, const double *init_v, const double *init_a, double *pos_pts,
                           double *posT_pts, double *angle_pts, double *angleT_pts, double *c_mpc_xy, double *c_mpc_yaw, double *dev4, cudaStream_t st)
{
    long long sN = 0, sM = 0;
    for (int b = 0; b < L.B; b++) { sN += L.N[b]; sM += L.M[b]; }
    struct Tmp { DevBuf<double> buf; ~Tmp() { buf.release(); } } t;
    CK(t.buf.ensure(mpc_export_doubles(L.B, sN, sM)));
    HoldGuard none{c, UALM_MAX_LANES, st, false};
    return mpc_export_run(bp, sN, sM, dt, init_v, init_a, nullptr, t.buf.p, pos_pts, posT_pts, angle_pts, angleT_pts, c_mpc_xy, c_mpc_yaw, dev4, st, none);
}

extern "C" int ualm_mpc_export_batch(ualm_ctx_t *c, double dt, const double *init_v, const double *init_a, double *pos_pts, double *posT_pts, double *angle_pts,
                                     double *angleT_pts, double *c_mpc_xy, double *c_mpc_yaw, double *dev4)
{
    if (!c || !(dt > 0.0)) return fail(UALM_EINVAL, "null ctx or dt <= 0");
    const BatchLayout &L = c->b->batch;
    if (c->tp) {     // (the hand-over reads no parameter and no grid)
        TpScan s;
        if (int rc = tp_scan(c, "ualm_mpc_export_batch", s)) return rc;
        if (L.B == 0) return UALM_OK;
        return mpc_export_lane(c, s.bp, L, dt, init_v, init_a, pos_pts, posT_pts, angle_pts, angleT_pts, c_mpc_xy, c_mpc_yaw, dev4, 0);
    }
    Lane *l = c->b;
    if (!l->have_batch || !l->solved) return fail(UALM_ESTATE, "ualm_mpc_export_batch needs a solved resident batch");
    CK(cudaSetDevice(c->device));
    if (L.B == 0) return UALM_OK;
    return mpc_export_lane(c, batch_ptrs(c), L, dt, init_v, init_a, pos_pts, posT_pts, angle_pts, angleT_pts, c_mpc_xy, c_mpc_yaw, dev4, l->stream);
}

// the held form: the records staged on the check stream (stage_held), the kernel's outputs and scratch at the front of the check block,
// each row's boundary derivatives behind them.  Reads no grid, parameter, lane or record of the context, so nothing waits for a batch
// in flight: the block grows in stream order and the call synchronises the check stream only
extern "C" int ualm_mpc_export_trajectories(ualm_ctx_t *c, int B, const int32_t *N, const int32_t *M, const double *piece_T, const double *c_xy,
                                            const double *c_yaw, const double *init_v, const double *init_a, double dt, double *pos_pts,
                                            double *posT_pts, double *angle_pts, double *angleT_pts, double *c_mpc_xy, double *c_mpc_yaw, double *dev4)
{
    if (!c || B < 0 || (B > 0 && (!N || !M || !piece_T || !c_xy || !c_yaw)))
        return fail(UALM_EINVAL, "ualm_mpc_export_trajectories: null argument or B < 0");
    if (!(dt > 0.0)) return fail(UALM_EINVAL, "ualm_mpc_export_trajectories: dt must be > 0");
    Held held{B, N, M, piece_T, c_xy, c_yaw, nullptr};
    if (int rc = held_counts("ualm_mpc_export_trajectories", held)) return rc;
    for (int b = 0; b < B; b++) {
        for (const double *v : {init_v, init_a})
            for (int k = 0; v && k < 3; k++)
                if (!std::isfinite(v[3 * (size_t)b + k])) return fail(UALM_EINVAL, "ualm_mpc_export_trajectories: init_v and init_a must be finite");
        // a record ualm_poll_batch has not filled yet (zero durations); +inf is a diverged solve, exported as the lane form exports it
        if (!over_limits(N[b], M[b]) && (!(piece_T[2 * b] > 0.0) || !(piece_T[2 * b + 1] > 0.0)))
            return fail(UALM_EINVAL, "ualm_mpc_export_trajectories: piece_T must be > 0 (row " + std::to_string(b) + ")");
    }
    if (B == 0) return UALM_OK;
    CK(cudaSetDevice(c->device));
    if (int rc = check_stream(c)) return rc;
    std::vector<double> rows;
    if (init_v || init_a) {
        rows.assign(6 * (size_t)B, 0.0);
        for (int b = 0; b < B; b++)
            for (int k = 0; k < 3; k++) {
                if (init_v) rows[6 * (size_t)b + k] = init_v[3 * (size_t)b + k];
                if (init_a) rows[6 * (size_t)b + 3 + k] = init_a[3 * (size_t)b + k];
            }
    }
    const long long sN = held.ncx / 12, sM = held.ncy / 6;
    const std::vector<ProbDesc> desc = scan_descs(c, B, N, M, nullptr, nullptr, nullptr);    // (the kernel reads N, M, S and the offsets)
    HoldGuard urgent{c, UALM_MAX_LANES, c->cstream, false};
    Staged s;
    if (int rc = stage_held(c, held, desc, mpc_export_doubles(B, sN, sM), rows.empty() ? nullptr : rows.data(), 6, nullptr, urgent, s)) return rc;
    BatchPtrs bp;
    memset(&bp, 0, sizeof(bp));
    bp.B = B; bp.desc = s.a.desc; bp.c_xy = const_cast<double *>(s.a.c_xy); bp.c_yaw = const_cast<double *>(s.a.c_yaw);
    bp.piece_T = const_cast<double *>(s.a.piece_T);
    return mpc_export_run(bp, sN, sM, dt, nullptr, nullptr, s.rows, s.a.out, pos_pts, posT_pts, angle_pts, angleT_pts, c_mpc_xy, c_mpc_yaw, dev4,
                          c->cstream, urgent);
}

// ---------------------------------------------------------------------------------------------
// UnevenMap construction on the device (SURVEY 8f-1).  HBM-bound gather: one thread per cell, yaw fastest so that the 64
// threads of a CTA share (x, y) and read the same few cloud bins through L1.  A launch covers the cell columns
// [box.x, box.x + box.z) x [box.y, box.y + box.w), all yaw layers, and writes them at their places in the whole grid `cells`:
// blockIdx.y is the x row of the box, whose ny * Yaw cells are contiguous in the grid.  The thread's cell and address are plain
// functions of its indices and the parameters, so neither holds a register across ualm_map_cell.
// ---------------------------------------------------------------------------------------------
namespace ualm {
__global__ void __launch_bounds__(64) map_build_kernel(UalmMapPrep prep, ualm_map_geom_t geom, int4 box, float4 *cells)
{
    const int W = geom.voxel_num[2], Y = geom.voxel_num[1];
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;      // cell k of the box's x row
    if (k >= (long long)box.w * W) return;
    const int w = (int)(k % W), y = box.y + (int)(k / W), x = box.x + (int)blockIdx.y;
    float o[4];
    ualm_map_cell(prep, geom, x, y, w, o);
    cells[((long long)x * Y + box.y) * W + k] = make_float4(o[0], o[1], o[2], o[3]);
}
} // namespace ualm

// map_build_kernel on stream st: UnevenMap::init's preprocessing of the cloud on the host (cropped about g's centre), then the cells
// of the cell boxes boxes[0 .. nbox) ({ix0, iy0, nx, ny}, all yaw layers; empty boxes are skipped) into their places in the whole-grid
// device buffer dst; the rest of dst is not touched (scratch allocated and freed on st).  cells_out (optional): the boxes' cells to the
// host one box after the other, each [nx][ny][yaw] float4; kernel_ms (optional): CUDA-event time of the kernels.  Returns once st has
// completed the work
static int map_build_on(cudaStream_t st, const float *pin, int64_t npts, const ualm_map_geom_t *g, const int4 *boxes, int nbox, double ex,
                        double ey, double ez, int iter_num, float4 *dst, float *cells_out, float *kernel_ms)
{
    UalmMapHostPrep prep;
    ualm_map_preprocess(pin, npts, ex, ey, ez, ualm_map_centre(*g, 0), ualm_map_centre(*g, 1), prep);
    UalmMapPrep view = prep.view(ex, ey, ez, iter_num);
    // scratch and events are released on every exit path (CK returns on the first CUDA error)
    struct Scratch {
        cudaStream_t st;
        float *pts = nullptr; int *start = nullptr;
        cudaEvent_t e0 = nullptr, e1 = nullptr;
        ~Scratch()
        {
            if (pts) cudaFreeAsync(pts, st);
            if (start) cudaFreeAsync(start, st);
            if (e0) cudaEventDestroy(e0);
            if (e1) cudaEventDestroy(e1);
        }
    } sc{st};
    CK(cudaMallocAsync(&sc.pts, sizeof(float) * std::max<size_t>(prep.pts.size(), 3), st));
    CK(cudaMallocAsync(&sc.start, sizeof(int) * std::max<size_t>(prep.start.size(), 1), st));
    CK(cudaEventCreate(&sc.e0)); CK(cudaEventCreate(&sc.e1));
    if (!prep.pts.empty()) CK(cudaMemcpyAsync(sc.pts, prep.pts.data(), sizeof(float) * prep.pts.size(), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(sc.start, prep.start.data(), sizeof(int) * prep.start.size(), cudaMemcpyHostToDevice, st));
    view.pts = sc.pts; view.start = sc.start;
    CK(cudaEventRecord(sc.e0, st));
    for (int b = 0; b < nbox; b++) {
        const int4 box = boxes[b];
        const long long row = (long long)box.w * g->voxel_num[2];        // cells per x row of the box
        for (int x0 = 0; x0 < box.z && row > 0; x0 += 65535) {          // gridDim.y <= 65535 x rows per launch
            const int4 part = make_int4(box.x + x0, box.y, std::min(65535, box.z - x0), box.w);
            map_build_kernel<<<dim3((unsigned)((row + 63) / 64), (unsigned)part.z), 64, 0, st>>>(view, *g, part, dst);
            CK(cudaGetLastError());
        }
    }
    CK(cudaEventRecord(sc.e1, st));
    const size_t col = sizeof(float4) * g->voxel_num[2], pitch = col * g->voxel_num[1];
    for (int b = 0; b < nbox && cells_out; b++) {
        const int4 box = boxes[b];
        if (box.z <= 0 || box.w <= 0) continue;
        CK(cudaMemcpy2DAsync(cells_out, col * box.w, (const char *)dst + pitch * box.x + col * box.y, pitch, col * box.w, box.z,
                             cudaMemcpyDeviceToHost, st));
        cells_out += 4 * (size_t)box.z * box.w * g->voxel_num[2];
    }
    CK(cudaStreamSynchronize(st));
    if (kernel_ms) CK(cudaEventElapsedTime(kernel_ms, sc.e0, sc.e1));
    return UALM_OK;
}

extern "C" int ualm_map_build_device(ualm_ctx_t *c, const float *pin, int64_t npts, const ualm_map_geom_t *g, double ex, double ey, double ez,
                                     int iter_num, float *cells, float *kernel_ms)
{
    if (!c || !pin || !g || !cells || npts < 0) return fail(UALM_EINVAL, "null argument");
    CK(cudaSetDevice(c->device));
    struct Scratch { DevBuf<float4> cells; ~Scratch() { cells.release(); } } sc;
    CK(sc.cells.ensure(map_ncell(g)));
    const int4 all = map_box_all(g);
    return map_build_on(c->b->stream, pin, npts, g, &all, 1, ex, ey, ez, iter_num, sc.cells.p, cells, kernel_ms);
}

// ---------------------------------------------------------------------------------------------
// Grid updates while batches are in flight: a new version is filled (or built) on the map stream, which no solve occupies, and made
// current once complete.  Work launched before keeps the version it was launched with (MapVer, lane_hold)
// ---------------------------------------------------------------------------------------------
static int map_geom_check(const ualm_map_geom_t *g)
{
    for (int k = 0; k < 3; k++)
        if (g->voxel_num[k] <= 0) return fail(UALM_EINVAL, "voxel_num must be > 0 in every dimension");
    return UALM_OK;
}

extern "C" int ualm_update_map(ualm_ctx_t *c, const ualm_map_geom_t *g, const float *cells)
{
    if (!c || !g || !cells) return fail(UALM_EINVAL, "null argument");
    if (int rc = map_geom_check(g)) return rc;
    CK(cudaSetDevice(c->device));
    const size_t bytes = map_ncell(g) * sizeof(float4);
    MapRef nv;
    if (int rc = map_version_new(c, bytes, &nv)) return rc;
    const cudaError_t e = cudaMemcpyAsync(nv->p, cells, bytes, cudaMemcpyHostToDevice, c->mstream);
    const cudaError_t s = cudaStreamSynchronize(c->mstream);       // complete on return; also before a failed version is freed
    if (e != cudaSuccess || s != cudaSuccess) return fail(UALM_ENOCUDA, std::string("ualm_update_map: ") + cudaGetErrorString(e != cudaSuccess ? e : s));
    map_install(c, g, std::move(nv));
    return UALM_OK;
}

extern "C" int ualm_update_map_from_cloud(ualm_ctx_t *c, const float *pts, int64_t npts, const ualm_map_geom_t *g, double ex, double ey, double ez,
                                          int iter_num, float *cells_out, float *kernel_ms)
{
    if (!c || !pts || !g || npts < 0) return fail(UALM_EINVAL, "null argument or npts < 0");
    if (int rc = map_geom_check(g)) return rc;
    CK(cudaSetDevice(c->device));
    MapRef nv;
    if (int rc = map_version_new(c, map_ncell(g) * sizeof(float4), &nv)) return rc;
    const int4 all = map_box_all(g);
    if (int rc = map_build_on(c->mstream, pts, npts, g, &all, 1, ex, ey, ez, iter_num, (float4 *)nv->p, cells_out, kernel_ms)) {
        cudaStreamSynchronize(c->mstream);      // before the version is freed
        return rc;
    }
    map_install(c, g, std::move(nv));
    return UALM_OK;
}

// dst <- src (device, `rows` rows of `width` bytes, `dpitch` / `spitch` bytes apart) on the map stream through the copy engines only:
// blocks of rows go to the pinned staging buffer and back, a row wider than the buffer in pieces.  A device-to-device cudaMemcpyAsync
// runs as a copy kernel, which on the parity path waits for the solve's SMs like any kernel (the driver ignored cudaMemcpyBatchAsync's
// cudaMemcpyFlagPreferOverlapWithCompute hint there: DESIGN.md section 3h).  The staging buffer is allocated once per context
// (cudaFreeHost would synchronise the device) and reused in stream order
static cudaError_t map_copy_ce(ualm_ctx *c, void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, size_t rows)
{
    if (!c->h_stage) {
        const cudaError_t e = cudaHostAlloc(&c->h_stage, ualm_ctx::STAGE_BYTES, cudaHostAllocDefault);
        if (e != cudaSuccess) { c->h_stage = nullptr; return e; }
    }
    for (size_t o = 0; o < width; o += ualm_ctx::STAGE_BYTES) {
        const size_t w = std::min(ualm_ctx::STAGE_BYTES, width - o), k = ualm_ctx::STAGE_BYTES / w;     // k >= 1 rows per block
        for (size_t r = 0; r < rows; r += k) {
            const size_t n = std::min(k, rows - r);
            cudaError_t e = cudaMemcpy2DAsync(c->h_stage, w, (const char *)src + r * spitch + o, spitch, w, n, cudaMemcpyDeviceToHost, c->mstream);
            if (e == cudaSuccess) e = cudaMemcpy2DAsync((char *)dst + r * dpitch + o, dpitch, c->h_stage, w, w, n, cudaMemcpyHostToDevice, c->mstream);
            if (e != cudaSuccess) return e;
        }
    }
    return cudaSuccess;
}

// ualm_update_map_window*: a new version that starts as a copy (map_copy_ce) of the selected environment's current one, with the
// cell box {ix0, iy0, nx, ny} (all yaw layers) written over it by write(geometry, new cells) on the map stream, made current once
// complete.  The geometry stays the current version's
template <class F>
static int map_window_update(ualm_ctx *c, int ix0, int iy0, int nx, int ny, const char *what, F write)
{
    if (nx <= 0 || ny <= 0) return fail(UALM_EINVAL, std::string(what) + ": nx and ny must be > 0");
    const Env &v = c->envs[c->sel_env];
    if (!v.have_map || !v.map) return fail(UALM_ESTATE, std::string(what) + ": the selected environment has no map grid bound");
    if (!v.map->dm.cells) return fail(UALM_ESTATE, std::string(what) + ": the selected environment holds a double grid (ualm_set_map_f64); a window needs the float grid");
    const MapRef cur = v.map;          // held until the copy below is complete
    const ualm_map_geom_t g = cur->geom;
    if (ix0 < 0 || iy0 < 0 || (long long)ix0 + nx > g.voxel_num[0] || (long long)iy0 + ny > g.voxel_num[1])
        return fail(UALM_EINVAL, std::string(what) + ": the box is outside the grid's voxel_num");
    CK(cudaSetDevice(c->device));
    const size_t pitch = sizeof(float4) * g.voxel_num[1] * g.voxel_num[2];      // one x row of the grid
    MapRef nv;
    if (int rc = map_version_new(c, pitch * g.voxel_num[0], &nv)) return rc;
    const cudaError_t e = map_copy_ce(c, nv->p, pitch, cur->p, pitch, pitch, g.voxel_num[0]);
    const int rc = e != cudaSuccess ? fail(UALM_ENOCUDA, std::string(what) + ": " + cudaGetErrorString(e)) : write(g, (float4 *)nv->p);
    const cudaError_t s = cudaStreamSynchronize(c->mstream);       // complete on return; also before a failed version is freed
    if (rc) return rc;
    if (s != cudaSuccess) return fail(UALM_ENOCUDA, std::string(what) + ": " + cudaGetErrorString(s));
    map_install(c, &g, std::move(nv));
    return UALM_OK;
}

extern "C" int ualm_update_map_window(ualm_ctx_t *c, int ix0, int iy0, int nx, int ny, const float *cells)
{
    if (!c || !cells) return fail(UALM_EINVAL, "null argument");
    // one strided host-to-device copy: x row k of the box is ny*W float4, contiguous in the host array and one grid row apart in the
    // new version.  Copy engines only, so it needs no free SM
    return map_window_update(c, ix0, iy0, nx, ny, "ualm_update_map_window", [&](const ualm_map_geom_t &g, float4 *dst) {
        const size_t col = sizeof(float4) * g.voxel_num[2], pitch = col * g.voxel_num[1];
        CK(cudaMemcpy2DAsync((char *)dst + pitch * ix0 + col * iy0, pitch, cells, col * ny, col * ny, nx, cudaMemcpyHostToDevice, c->mstream));
        return UALM_OK;
    });
}

extern "C" int ualm_update_map_window_from_cloud(ualm_ctx_t *c, const float *pts, int64_t npts, int ix0, int iy0, int nx, int ny, double ex, double ey,
                                                 double ez, int iter_num, float *cells_out, float *kernel_ms)
{
    if (!c || !pts || npts < 0) return fail(UALM_EINVAL, "null argument or npts < 0");
    return map_window_update(c, ix0, iy0, nx, ny, "ualm_update_map_window_from_cloud", [&](const ualm_map_geom_t &g, float4 *dst) {
        const int4 box = make_int4(ix0, iy0, nx, ny);
        return map_build_on(c->mstream, pts, npts, &g, &box, 1, ex, ey, ez, iter_num, dst, cells_out, kernel_ms);
    });
}

// The cell boxes {ix0, iy0, nx, ny} of grid g moved by (dx, dy) cells whose cells have no source before the move: box[0] = A, the x
// strip; box[1] = B, the y strip over the x columns not in A.  An empty box is {0, 0, 0, 0}
static void map_shift_boxes(const ualm_map_geom_t &g, int dx, int dy, int4 box[2])
{
    const long long X = g.voxel_num[0], Y = g.voxel_num[1];
    const long long ax = std::min<long long>(std::llabs((long long)dx), X), ay = std::min<long long>(std::llabs((long long)dy), Y);
    box[0] = ax == 0 ? make_int4(0, 0, 0, 0) : make_int4(dx > 0 ? (int)(X - ax) : 0, 0, (int)ax, (int)Y);
    box[1] = ay == 0 || ax == X ? make_int4(0, 0, 0, 0) : make_int4(dx < 0 ? (int)ax : 0, dy > 0 ? (int)(Y - ay) : 0, (int)(X - ax), (int)ay);
}

// ualm_shift_map*: a new version with the selected environment's current geometry moved by (dx, dy) cells, whose overlap with the current
// version is copied over (map_copy_ce) and whose uncovered boxes A and B (map_shift_boxes) are written by write(moved geometry, boxes,
// new cells) on the map stream, made current once complete
template <class F>
static int map_shift_update(ualm_ctx *c, int dx, int dy, const char *what, F write)
{
    if (dx == 0 && dy == 0) return fail(UALM_EINVAL, std::string(what) + ": dx and dy are both 0");
    const Env &v = c->envs[c->sel_env];
    if (!v.have_map || !v.map) return fail(UALM_ESTATE, std::string(what) + ": the selected environment has no map grid bound");
    if (!v.map->dm.cells) return fail(UALM_ESTATE, std::string(what) + ": the selected environment holds a double grid (ualm_set_map_f64); a shift needs the float grid");
    const MapRef cur = v.map;          // held until the copy below is complete
    ualm_map_geom_t g = cur->geom;
    g.origin[0] = g.origin[0] + dx * g.xy_resolution; g.max_boundary[0] = g.max_boundary[0] + dx * g.xy_resolution;
    g.origin[1] = g.origin[1] + dy * g.xy_resolution; g.max_boundary[1] = g.max_boundary[1] + dy * g.xy_resolution;
    int4 box[2];
    map_shift_boxes(g, dx, dy, box);
    CK(cudaSetDevice(c->device));
    const long long X = g.voxel_num[0], Y = g.voxel_num[1];
    const size_t col = sizeof(float4) * g.voxel_num[2], pitch = col * Y;
    MapRef nv;
    if (int rc = map_version_new(c, pitch * X, &nv)) return rc;
    cudaError_t e = cudaSuccess;
    // the overlap: new columns [x0, x0 + nxo) x [y0, y0 + nyo) from old (x + dx, y + dy); each x row of it is nyo * W float4, contiguous
    // in both versions and one grid row apart
    const long long nxo = X - std::min<long long>(std::llabs((long long)dx), X), nyo = Y - std::min<long long>(std::llabs((long long)dy), Y);
    if (nxo > 0 && nyo > 0) {
        const long long x0 = std::max(0, -dx), y0 = std::max(0, -dy);
        e = map_copy_ce(c, (char *)nv->p + pitch * x0 + col * y0, pitch, (const char *)cur->p + pitch * (x0 + dx) + col * (y0 + dy), pitch,
                        col * nyo, nxo);
    }
    const int rc = e != cudaSuccess ? fail(UALM_ENOCUDA, std::string(what) + ": " + cudaGetErrorString(e)) : write(g, box, (float4 *)nv->p);
    const cudaError_t s = cudaStreamSynchronize(c->mstream);       // complete on return; also before a failed version is freed
    if (rc) return rc;
    if (s != cudaSuccess) return fail(UALM_ENOCUDA, std::string(what) + ": " + cudaGetErrorString(s));
    map_install(c, &g, std::move(nv));
    return UALM_OK;
}

extern "C" int ualm_shift_map(ualm_ctx_t *c, int dx, int dy, const float *cells)
{
    if (!c || !cells) return fail(UALM_EINVAL, "null argument");
    // A then B from the host array, one strided host-to-device copy each (as a window's): copy engines only
    return map_shift_update(c, dx, dy, "ualm_shift_map", [&](const ualm_map_geom_t &g, const int4 *box, float4 *dst) {
        const size_t col = sizeof(float4) * g.voxel_num[2], pitch = col * g.voxel_num[1];
        const char *src = (const char *)cells;
        for (int b = 0; b < 2; b++) {
            if (box[b].z <= 0 || box[b].w <= 0) continue;
            CK(cudaMemcpy2DAsync((char *)dst + pitch * box[b].x + col * box[b].y, pitch, src, col * box[b].w, col * box[b].w, box[b].z,
                                 cudaMemcpyHostToDevice, c->mstream));
            src += col * box[b].w * box[b].z;
        }
        return UALM_OK;
    });
}

extern "C" int ualm_shift_map_from_cloud(ualm_ctx_t *c, const float *pts, int64_t npts, int dx, int dy, double ex, double ey, double ez, int iter_num,
                                         float *cells_out, float *kernel_ms)
{
    if (!c || !pts || npts < 0) return fail(UALM_EINVAL, "null argument or npts < 0");
    return map_shift_update(c, dx, dy, "ualm_shift_map_from_cloud", [&](const ualm_map_geom_t &g, const int4 *box, float4 *dst) {
        return map_build_on(c->mstream, pts, npts, &g, box, 2, ex, ey, ez, iter_num, dst, cells_out, kernel_ms);
    });
}
