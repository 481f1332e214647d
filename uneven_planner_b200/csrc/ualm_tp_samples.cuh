// ualm_tp_samples.cuh -- the per-constraint-sample kernels of the throughput path: kb_kernel (calConstrainCostGrad,
// alm_traj_opt.cpp:663-991) and ks_kernel (initScaling, alm_traj_opt.cpp:349-661), with UnevenMap::getAllWithGrad
// (uneven_map.h:258-377) evaluated from map tiles that TMA stages into shared memory.  One CTA per trajectory, one thread per sample.
#pragma once

#include "ualm_tp_kernels.cuh"
#include "ualm_mailbox.h"

namespace ualm_tp {

__device__ __forceinline__ void sincos_(float x, float &s, float &c) { sincosf(x, &s, &c); }
__device__ __forceinline__ void sincos_(double x, double &s, double &c) { sincos(x, &s, &c); }
__device__ __forceinline__ float sqrt_(float x) { return sqrtf(x); }
__device__ __forceinline__ double sqrt_(double x) { return sqrt(x); }
__device__ __forceinline__ float rint_(float x) { return rintf(x); }
__device__ __forceinline__ double rint_(double x) { return rint(x); }
__device__ __forceinline__ float floor_(float x) { return floorf(x); }
__device__ __forceinline__ double floor_(double x) { return floor(x); }
__device__ __forceinline__ float abs_(float x) { return fabsf(x); }
__device__ __forceinline__ double abs_(double x) { return fabs(x); }
__device__ __forceinline__ float max_(float a, float b) { return fmaxf(a, b); }
__device__ __forceinline__ double max_(double a, double b) { return fmax(a, b); }

// ---- mbarrier / TMA (cp.async.bulk.tensor) primitives ----
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("{ .reg .b64 st; mbarrier.arrive.shared::cta.b64 st, [%0]; }" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, unsigned bytes)
{
    asm volatile("{ .reg .b64 st; mbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1; }" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity)
{
    asm volatile(
        "{ .reg .pred p;\n"
        "WAIT_%=: mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=: }" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// 3-D box load: coordinates (innermost first) = {4 * yaw cell, y cell, x cell}
__device__ __forceinline__ void tma_load_tile(void *dst, const CUtensorMap *tm, int c0, int c1, int c2, uint64_t *bar)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

// shared-memory view of the staged tiles of one chunk: tile t covers cells [org[t], org[t] + TP_TILE) in x, y and yaw
struct TileSet {
    const float4 *tiles;     // [ppc][8][8][8]
    const int *org;          // [ppc][4]   x0, y0, w0, valid
};

template <class R>
struct Kin {              // kinematics + terrain of one constraint sample (alm_traj_opt.cpp:733-817)
    R b0[6], b1[6], b2[6];
    R vel[2], acc[2], jer[2];
    R yaw, dyaw, d2yaw, syaw, cyaw, v_norm, lon_acc, lat_acc;
    R sy1;
    R tv[7], tg[7][3];
    R vx, wz, ax, ay, curv_snorm;
    int yaw_idx;
};

// UnevenMap::getAllWithGrad (uneven_map.h:318-377 on top of getTerrainWithGradI :258-315).  pos = (x, y, yaw normalised to [-pi, pi]);
// sy / cy = sin / cos of the yaw.  Corner cells come from the tile when it holds them, else from global memory.
template <class R>
__device__ __forceinline__ void map_query(const TpMap &m, R px, R py, R pw, R syaw, R cyaw, const float4 *tile, int tx0, int ty0, int tw0, bool has_tile,
                                          R tv[7], R tg[7][3])
{
    R rs[3] = {0, 0, 0}, rg[4][3];
#pragma unroll
    for (int r = 0; r < 4; r++)
#pragma unroll
        for (int k = 0; k < 3; k++) rg[r][k] = 0;
    const bool in = !(px < (R)(m.origin[0] + 1e-4) || py < (R)(m.origin[1] + 1e-4) || pw < (R)(m.origin[2] + 1e-4) || px > (R)(m.maxb[0] - 1e-4) ||
                      py > (R)(m.maxb[1] - 1e-4) || pw > (R)(m.maxb[2] - 1e-4));
    if (in) {
        const R xy_res = (R)m.xy_res, yaw_res = (R)m.yaw_res, xy_inv = (R)m.xy_inv, yaw_inv = (R)m.yaw_inv;
        const R o0 = (R)m.origin[0], o1 = (R)m.origin[1], o2 = (R)m.origin[2];
        const R twopi = (R)6.283185307179586476925;
        R pm2 = pw - (R)0.5 * yaw_res;
        pm2 -= twopi * rint_(pm2 / twopi);                          // normSO2
        const int i0 = (int)floor_((px - (R)0.5 * xy_res - o0) * xy_inv), i1 = (int)floor_((py - (R)0.5 * xy_res - o1) * xy_inv),
                  i2 = (int)floor_((pm2 - o2) * yaw_inv);
        const R d0 = (px - (((R)i0 + (R)0.5) * xy_res + o0)) * xy_inv, d1 = (py - (((R)i1 + (R)0.5) * xy_res + o1)) * xy_inv;
        R dw = pw - (((R)i2 + (R)0.5) * yaw_res + o2);
        dw -= twopi * rint_(dw / twopi);                             // = atan2(sin, cos) of the difference (uneven_map.h:284)
        const R d2 = dw * yaw_inv;
        R v[2][2][2][3];
#pragma unroll
        for (int x = 0; x < 2; x++)
#pragma unroll
            for (int y = 0; y < 2; y++)
#pragma unroll
                for (int w = 0; w < 2; w++) {
                    int c0 = max(min(i0 + x, m.vn[0] - 1), 0), c1 = max(min(i1 + y, m.vn[1] - 1), 0), c2 = i2 + w;
                    if (c2 >= m.vn[2]) c2 -= m.vn[2];
                    if (c2 < 0) c2 += m.vn[2];
                    const unsigned ux = (unsigned)(c0 - tx0), uy = (unsigned)(c1 - ty0), uw = (unsigned)(c2 - tw0);
                    float4 cell;
                    if (has_tile && ux < TP_TILE && uy < TP_TILE && uw < TP_TILE) cell = tile[(ux * TP_TILE + uy) * TP_TILE + uw];
                    else cell = __ldg(&m.cells[((size_t)c0 * m.vn[1] + c1) * m.vn[2] + c2]);
                    v[x][y][w][0] = (R)cell.y; v[x][y][w][1] = (R)cell.z; v[x][y][w][2] = (R)cell.w;
                }
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const R v00 = v[0][0][0][k] * (1 - d0) + v[1][0][0][k] * d0, v01 = v[0][0][1][k] * (1 - d0) + v[1][0][1][k] * d0;
            const R v10 = v[0][1][0][k] * (1 - d0) + v[1][1][0][k] * d0, v11 = v[0][1][1][k] * (1 - d0) + v[1][1][1][k] * d0;
            const R v0 = v00 * (1 - d1) + v10 * d1, v1 = v01 * (1 - d1) + v11 * d1;
            rs[k] = v0 * (1 - d2) + v1 * d2;
            rg[k][2] = (v1 - v0) * yaw_inv;
            rg[k][1] = ((v10 - v00) * (1 - d2) + (v11 - v01) * d2) * xy_inv;
            R g0 = (1 - d2) * (1 - d1) * (v[1][0][0][k] - v[0][0][0][k]);
            g0 += (1 - d2) * d1 * (v[1][1][0][k] - v[0][1][0][k]);
            g0 += d2 * (1 - d1) * (v[1][0][1][k] - v[0][0][1][k]);
            g0 += d2 * d1 * (v[1][1][1][k] - v[0][1][1][k]);
            rg[k][0] = g0 * xy_inv;
        }
        const R cc = sqrt_((R)1 - rs[1] * rs[1] - rs[2] * rs[2]);
#pragma unroll
        for (int k = 0; k < 3; k++) rg[3][k] = -(rg[1][k] * rs[1] + rg[2][k] * rs[2]) / cc;
    }
    const R c = sqrt_((R)1 - rs[1] * rs[1] - rs[2] * rs[2]);
    const R inv_c = (R)1 / c;
    const R tt = cyaw * rs[1] + syaw * rs[2];
    const R s = -(-syaw * rs[1] + cyaw * rs[2]);
    const R sq = sqrt_((R)1 - tt * tt);
    const R isq = (R)1 / sq, isq3 = isq * isq * isq;
    R dt[3], ds[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        dt[k] = rg[1][k] * cyaw + rg[2][k] * syaw;
        ds[k] = -(rg[1][k] * (-syaw) + rg[2][k] * cyaw);
    }
    dt[2] -= s;
    ds[2] += tt;
    tv[0] = isq; tv[1] = -c * tt * isq; tv[2] = sq * inv_c; tv[3] = s * isq; tv[4] = c; tv[5] = inv_c; tv[6] = rs[0];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        tg[0][k] = tt * isq3 * dt[k];
        tg[1][k] = -(tt * isq * rg[3][k] + isq3 * c * dt[k]);
        tg[2][k] = -inv_c * (tt * isq * dt[k] + sq * inv_c * rg[3][k]);
        tg[3][k] = isq * ds[k] + tt * isq3 * s * dt[k];
        tg[4][k] = rg[3][k];
        tg[5][k] = -inv_c * inv_c * rg[3][k];
        tg[6][k] = rg[0][k];
    }
}

// spline part of the kinematics: basis, position .. jerk, yaw piece, yaw .. d2yaw, and the map cell of the sample
template <class R>
__device__ __forceinline__ void kin_spline(const R *cx6, const R *cy6, const R *cyaw_all, int M, R s1, R base_time, R Ty, Kin<R> &q, R pos[2])
{
    const R s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2, s5 = s4 * s1;
    q.b0[0] = 1; q.b0[1] = s1; q.b0[2] = s2; q.b0[3] = s3; q.b0[4] = s4; q.b0[5] = s5;
    q.b1[0] = 0; q.b1[1] = 1; q.b1[2] = 2 * s1; q.b1[3] = 3 * s2; q.b1[4] = 4 * s3; q.b1[5] = 5 * s4;
    q.b2[0] = 0; q.b2[1] = 0; q.b2[2] = 2; q.b2[3] = 6 * s1; q.b2[4] = 12 * s2; q.b2[5] = 20 * s3;
    const R b3[6] = {0, 0, 0, 6, 24 * s1, 60 * s2};
#pragma unroll
    for (int d = 0; d < 2; d++) {
        const R *c = d ? cy6 : cx6;
        R p = 0, v = 0, a = 0, j = 0;
#pragma unroll
        for (int k = 0; k < 6; k++) { p += c[k] * q.b0[k]; v += c[k] * q.b1[k]; a += c[k] * q.b2[k]; j += c[k] * b3[k]; }
        pos[d] = p; q.vel[d] = v; q.acc[d] = a; q.jer[d] = j;
    }
    const R now_time = s1 + base_time;
    int yi = (int)(now_time / Ty);                                  // alm_traj_opt.cpp:749-755
    if (yi >= M) yi = M - 1;
    q.yaw_idx = yi;
    const R y1 = now_time - (R)yi * Ty;
    q.sy1 = y1;
    const R y2 = y1 * y1, y3 = y2 * y1, y4 = y2 * y2, y5 = y4 * y1;
    const R *c = cyaw_all + 6 * yi;
    q.yaw = c[0] + c[1] * y1 + c[2] * y2 + c[3] * y3 + c[4] * y4 + c[5] * y5;
    q.dyaw = c[1] + 2 * c[2] * y1 + 3 * c[3] * y2 + 4 * c[4] * y3 + 5 * c[5] * y4;
    q.d2yaw = 2 * c[2] + 6 * c[3] * y1 + 12 * c[4] * y2 + 20 * c[5] * y3;
    sincos_(q.yaw, q.syaw, q.cyaw);
    q.v_norm = sqrt_(q.vel[0] * q.vel[0] + q.vel[1] * q.vel[1]);
    q.lon_acc = q.acc[0] * q.cyaw + q.acc[1] * q.syaw;
    q.lat_acc = -q.acc[0] * q.syaw + q.acc[1] * q.cyaw;
}
template <class R>
__device__ __forceinline__ void kin_terrain(const TpMap &map, R gravity, const R pos[2], R yawn, const float4 *tile, int tx0, int ty0, int tw0, bool has_tile, Kin<R> &q)
{
    map_query<R>(map, pos[0], pos[1], yawn, q.syaw, q.cyaw, tile, tx0, ty0, tw0, has_tile, q.tv, q.tg);
    q.vx = q.v_norm * q.tv[0];
    q.wz = q.dyaw * q.tv[5];
    q.ax = q.lon_acc * q.tv[0] + gravity * q.tv[1];
    q.ay = q.lat_acc * q.tv[2] + gravity * q.tv[3];
    q.curv_snorm = q.wz * q.wz / (q.vx * q.vx + (R)TP_DELTA_SIGL);
}
template <class R>
__device__ __forceinline__ R norm_yaw(R yaw)
{
    const R twopi = (R)6.283185307179586476925;
    return yaw - twopi * rint_(yaw / twopi);
}
// lower-corner cell of the trilinear stencil of pose (x, y, normalised yaw); false when the pose is outside the map
template <class R>
__device__ __forceinline__ bool stencil_cell(const TpMap &m, R px, R py, R pw, int &i0, int &i1, int &i2)
{
    if (px < (R)(m.origin[0] + 1e-4) || py < (R)(m.origin[1] + 1e-4) || pw < (R)(m.origin[2] + 1e-4) || px > (R)(m.maxb[0] - 1e-4) ||
        py > (R)(m.maxb[1] - 1e-4) || pw > (R)(m.maxb[2] - 1e-4)) return false;
    const R twopi = (R)6.283185307179586476925;
    R pm2 = pw - (R)0.5 * (R)m.yaw_res;
    pm2 -= twopi * rint_(pm2 / twopi);
    i0 = (int)floor_((px - (R)0.5 * (R)m.xy_res - (R)m.origin[0]) * (R)m.xy_inv);
    i1 = (int)floor_((py - (R)0.5 * (R)m.xy_res - (R)m.origin[1]) * (R)m.xy_inv);
    i2 = (int)floor_((pm2 - (R)m.origin[2]) * (R)m.yaw_inv);
    i0 = max(min(i0, m.vn[0] - 1), 0); i1 = max(min(i1, m.vn[1] - 1), 0);
    if (i2 < 0) i2 = 0;
    return true;
}

#define TP_YCAP 32           // yaw pieces per sample chunk that take the deterministic path (relative to the chunk's first one)
// Reduction of the per-sample gradient products onto the control points (alm_traj_opt.cpp:969-985, 827), without atomics on the
// common path: every thread forms its own contributions (basis x gradient), a segmented warp-shuffle reduction sums them per
// piece (xy coefficients, xy time gradient) resp. per yaw piece (yaw coefficients, yaw time gradient), the run heads park the
// per-warp partial sums in shared memory, and after one barrier a fixed-order sum over the warps writes the result.  The order of
// every sum is fixed by the sample index, so a trajectory's result does not depend on what else runs.
template <class R>
struct ChunkPart {
    R xy[TP_KB_THREADS / 32][TP_MAXPPC][13];   // per warp, per piece of the chunk: 12 coefficient-gradient sums + the time-gradient sum
    R yw[TP_KB_THREADS / 32][TP_YCAP][7];      // per warp, per yaw piece (index - ybase): 6 coefficient-gradient sums + the time-gradient sum
};
template <class R>
__device__ __forceinline__ void chunk_part_zero(ChunkPart<R> &P, int tid)
{
    R *z = &P.xy[0][0][0];
    for (int q = tid; q < (int)(sizeof(ChunkPart<R>) / sizeof(R)); q += TP_KB_THREADS) z[q] = 0;
}
// all 32 lanes of every warp call this (lanes without a sample pass on = false)
template <class R>
__device__ __forceinline__ void chunk_scatter(ChunkPart<R> &P, bool on, int pl, int yrel, R (&cx)[13], R (&cw)[7], R *accY, R *accTy, int ybase, int M)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int k1 = on ? pl : -1, k2 = on ? yrel : -1;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const int o1 = __shfl_down_sync(0xffffffffu, k1, off), o2 = __shfl_down_sync(0xffffffffu, k2, off);
        const bool t1 = (lane + off < 32) && o1 == k1, t2 = (lane + off < 32) && o2 == k2;
#pragma unroll
        for (int e = 0; e < 13; e++) { const R v = __shfl_down_sync(0xffffffffu, cx[e], off); if (t1) cx[e] += v; }
#pragma unroll
        for (int e = 0; e < 7; e++) { const R v = __shfl_down_sync(0xffffffffu, cw[e], off); if (t2) cw[e] += v; }
    }
    const int p1 = __shfl_up_sync(0xffffffffu, k1, 1), p2 = __shfl_up_sync(0xffffffffu, k2, 1);
    if (on && (lane == 0 || p1 != k1)) {
#pragma unroll
        for (int e = 0; e < 13; e++) P.xy[warp][pl][e] = cx[e];
    }
    const bool head2 = on && (lane == 0 || p2 != k2);
    const unsigned heads2 = __ballot_sync(0xffffffffu, head2);
    if (head2) {
        // two runs of one yaw piece inside a warp only happen when rounding swaps two samples at a piece boundary (two addends commute):
        // the common, unique run head stores; only such twins add atomically (the table is zeroed before every chunk)
        const unsigned same = __match_any_sync(heads2, k2);
        if (yrel < TP_YCAP) {
            if ((same & (same - 1u)) == 0u) {
#pragma unroll
                for (int e = 0; e < 7; e++) P.yw[warp][yrel][e] = cw[e];
            } else {
#pragma unroll
                for (int e = 0; e < 7; e++) atomicAdd(&P.yw[warp][yrel][e], cw[e]);
            }
        } else {           // more yaw pieces per chunk than the table holds (M >> N): straight onto the accumulators
            const int m = ybase + yrel;
            if (m < M) {
#pragma unroll
                for (int e = 0; e < 6; e++) atomicAdd(&accY[6 * m + e], cw[e]);
                atomicAdd(&accTy[m], cw[6]);
            }
        }
    }
}
// after a barrier: fixed-order sums over the warps
template <class R>
__device__ __forceinline__ void chunk_gather(const ChunkPart<R> &P, int p0, int np, int N, int M, int ybase, R *gdc_xy, R *gdt_xy, R *accY, R *accTy, int tid)
{
    const int nx = 6 * N;
    for (int t = tid; t < np * 13; t += TP_KB_THREADS) {
        const int pl = t / 13, e = t - 13 * pl;
        R s = 0;
#pragma unroll
        for (int w = 0; w < TP_KB_THREADS / 32; w++) s += P.xy[w][pl][e];
        if (e < 12) gdc_xy[(e / 6) * nx + 6 * (p0 + pl) + (e % 6)] = s;
        else gdt_xy[p0 + pl] = s;
    }
    for (int t = tid; t < TP_YCAP * 7; t += TP_KB_THREADS) {
        const int yr = t / 7, e = t - 7 * yr, m = ybase + yr;
        if (m >= M) continue;
        R s = 0;
#pragma unroll
        for (int w = 0; w < TP_KB_THREADS / 32; w++) s += P.yw[w][yr][e];
        if (e < 6) accY[6 * m + e] += s; else accTy[m] += s;
    }
}

struct KbShared {     // fixed part of kb_kernel's shared memory; the dynamic part follows (coefficients, yaw accumulators, tiles)
    uint64_t bar;
    int org[TP_MAXPPC][4];
};

// ---------------------------------------------------------------------------------------------------------------------
// kb_kernel: calConstrainCostGrad for every active trajectory (one CTA each)
// ---------------------------------------------------------------------------------------------------------------------
template <class R, bool TMA>
__global__ void __launch_bounds__(TP_KB_THREADS) kb_kernel(const __grid_constant__ TpPool E, const __grid_constant__ TpParams p, const __grid_constant__ TpMap map,
                                                           const __grid_constant__ CUtensorMap tmap, int group)
{
    if ((int)blockIdx.x >= E.n_active[group]) return;
    const int slot = E.active[(size_t)group * E.capacity + blockIdx.x];
    const TpState *st = E.st + slot;
    const int ph = st->phase;
    if (ph != PH_REQ_FIRST && ph != PH_REQ_LS && ph != PH_REQ_EVALONLY) return;
    const int N = st->N, M = st->M, S = st->S, K = p.int_K, K1 = K + 1, nx = 6 * N, ny = 6 * M, tid = threadIdx.x;
    extern __shared__ __align__(128) unsigned char kb_smem[];
    // layout: tiles (128-byte aligned, first) | ChunkPart | c_xy (12N) | c_yaw (6M) | accY (6M) | accTy (M)
    float4 *tiles = (float4 *)kb_smem;
    ChunkPart<R> *Pbuf = (ChunkPart<R> *)(kb_smem + (TMA ? TP_MAXPPC * TP_TILE_BYTES : 0));      // two tables: chunk k scatters into one while the other is zeroed
    R *cxy = (R *)(Pbuf + 2);
    R *cyaw = cxy + 12 * N;
    R *accY = cyaw + ny;
    R *accTy = accY + ny;
    __shared__ KbShared sh;
    __shared__ double s_cost[TP_KB_THREADS / 32];
    const R *cr = (const R *)E.cr + (size_t)slot * TP_CSTRIDE;
    for (int q = tid; q < 2 * nx; q += TP_KB_THREADS) cxy[q] = cr[q];
    for (int q = tid; q < ny; q += TP_KB_THREADS) { cyaw[q] = cr[TP_CYAW + q]; accY[q] = 0; }
    for (int q = tid; q < M; q += TP_KB_THREADS) accTy[q] = 0;
    if (TMA && tid == 0) { mbar_init(&sh.bar, TP_MAXPPC); mbar_fence_init(); }   // every chunk: TP_MAXPPC arrivals (one per piece slot)
    const int ppc = max(1, min(TP_MAXPPC, TP_KB_THREADS / K1));
    const R Tx = (R)st->Tx, Ty = (R)st->Ty, step = Tx / (R)K, rho = (R)st->rho, scale_fx = (R)st->scale_fx;
    // the limits and rho_ter are the slot's (its problem's row), formed in double and then cast
    const double *pp = st->pp;
    const R gravity = (R)p.gravity, rho_ter = (R)pp[1], min_cxi = (R)pp[6], max_sig = (R)pp[7];
    const R max_vel2 = (R)(pp[2] * pp[2]), max_alon2 = (R)(pp[3] * pp[3]), max_alat2 = (R)(pp[4] * pp[4]), max_kap2 = (R)(pp[5] * pp[5]);
    const bool use_scaling = p.use_scaling != 0;
    R *du = (R *)E.dual + (size_t)slot * TP_NDUAL * E.Smax;
    R *gdc = (R *)E.gdc + (size_t)slot * TP_CSTRIDE;
    R *gdt = (R *)E.gdt + (size_t)slot * TP_TSTRIDE;
    double cost_acc = 0.0;
    unsigned parity = 0;
    KProf kp;
    kp.start(E.prof ? E.prof + 16 : nullptr, tid);       // developer profile: phases of thread 0
    if (kp.p) atomicAdd((unsigned long long *)&kp.p[7], 1ull);
    if (tid < TP_MAXPPC) { sh.org[tid][0] = sh.org[tid][1] = sh.org[tid][2] = 0x7fffffff; sh.org[tid][3] = 0; }
    chunk_part_zero(Pbuf[0], tid);
    __syncthreads();
    kp.mark(0);
    int it = 0;
    for (int p0 = 0; p0 < N; p0 += ppc, it++) {
        const int np = min(ppc, N - p0), ns = np * K1;
        ChunkPart<R> &P = Pbuf[it & 1];
        const int ybase = max(0, min((int)((R)p0 * Tx / Ty), M - 1) - 1);     // yaw piece of the chunk's first sample, one spare for rounding
        {
            const int qb = 0, q = tid;       // one pass: ns <= TP_KB_THREADS (int_K <= 127 on this path)
            const bool on = q < ns;
            R cx[13], cw[7], cost = 0;
#pragma unroll
            for (int e = 0; e < 13; e++) cx[e] = 0;
#pragma unroll
            for (int e = 0; e < 7; e++) cw[e] = 0;
            Kin<R> kq;
            kq.yaw_idx = 0;
            R pos[2] = {0, 0}, yawn = 0;
            int pl = 0, j = 0, i = 0, s = 0;
            int ci0 = 0, ci1 = 0, ci2 = 0;
            bool inmap = false;
            R lam = 0, mu6[6] = {0, 0, 0, 0, 0, 0}, sc7[7] = {1, 1, 1, 1, 1, 1, 1};
            if (on) {
                pl = q / K1; j = q - pl * K1; i = p0 + pl; s = i * K1 + j;
                // duals and scales of this sample (coalesced SoA): in flight while the spline is evaluated and the tiles arrive
                lam = du[s];
#pragma unroll
                for (int t = 0; t < 6; t++) mu6[t] = du[(1 + t) * S + s];
#pragma unroll
                for (int t = 0; t < 7; t++) sc7[t] = du[(7 + t) * S + s];
                kin_spline<R>(cxy + 6 * i, cxy + nx + 6 * i, cyaw, M, (R)j * step, (R)i * Tx, Ty, kq, pos);
                yawn = norm_yaw(kq.yaw);
                inmap = stencil_cell<R>(map, pos[0], pos[1], yawn, ci0, ci1, ci2);
                if (TMA && inmap && qb == 0) { atomicMin(&sh.org[pl][0], ci0); atomicMin(&sh.org[pl][1], ci1); atomicMin(&sh.org[pl][2], ci2); }
            }
            if (qb == 0) kp.mark(1);
            if (TMA && qb == 0) {
                __syncthreads();
                if (tid < TP_MAXPPC) {    // one elected thread per piece slot issues its tile (or just arrives)
                    if (tid < np && sh.org[tid][0] != 0x7fffffff) {
                        sh.org[tid][3] = 1;
                        mbar_arrive_expect_tx(&sh.bar, TP_TILE_BYTES);
                        tma_load_tile(tiles + (size_t)tid * (TP_TILE_BYTES / 16), &tmap, 4 * sh.org[tid][2], sh.org[tid][1], sh.org[tid][0], &sh.bar);
                    } else mbar_arrive(&sh.bar);
                }
                __syncthreads();
                mbar_wait(&sh.bar, parity);
                kp.mark(2);
            }
            if (on) {
                const bool has_tile = TMA && qb == 0 && sh.org[pl][3];
                kin_terrain<R>(map, gravity, pos, yawn, tiles + (size_t)pl * (TP_TILE_BYTES / 16), sh.org[pl][0], sh.org[pl][1], sh.org[pl][2], has_tile, kq);
                // ---- the seven penalty terms (alm_traj_opt.cpp:819-946) ----
                R grad_p[2] = {0, 0}, grad_v[2] = {0, 0}, grad_a[2] = {0, 0}, grad_se2[3] = {0, 0, 0};
                R grad_yaw = 0, grad_dyaw = 0, grad_vx2 = 0, grad_wz = 0, grad_ax = 0, grad_ay = 0;
                const R icx = kq.tv[0], icy = kq.tv[2], cos_xi = kq.tv[4], inv_cos_xi = kq.tv[5], sigma = kq.tv[6];
                const R omega = ((j == 0 || j == K) ? (R)0.5 : (R)1) * rho_ter * step * scale_fx;
                const R user_cost = omega * sigma * sigma;
                cost = user_cost;
#pragma unroll
                for (int k = 0; k < 3; k++) grad_se2[k] += omega * kq.tg[6][k] * sigma * 2;
                {   // non-holonomic equality
                    const R h = (kq.vel[0] * kq.syaw - kq.vel[1] * kq.cyaw) * sc7[0];
                    du[14 * S + s] = h;
                    cost += h * (lam + (R)0.5 * rho * h);
                    const R g = (rho * h + lam) * sc7[0];
                    grad_v[0] += g * kq.syaw; grad_v[1] -= g * kq.cyaw;
                    grad_yaw += g * (kq.vel[0] * kq.cyaw + kq.vel[1] * kq.syaw);
                }
                const R hr = (R)0.5 / rho;
                {   // longitudinal velocity
                    const R gv = (kq.vx * kq.vx - max_vel2) * sc7[1];
                    du[15 * S + s] = gv;
                    if (rho * gv + mu6[0] > 0) { cost += gv * (mu6[0] + (R)0.5 * rho * gv); grad_vx2 += (rho * gv + mu6[0]) * sc7[1]; }
                    else cost -= mu6[0] * mu6[0] * hr;
                }
                {   // longitudinal acceleration
                    const R gv = (kq.ax * kq.ax - max_alon2) * sc7[2];
                    du[16 * S + s] = gv;
                    if (rho * gv + mu6[1] > 0) { cost += gv * (mu6[1] + (R)0.5 * rho * gv); grad_ax += (rho * gv + mu6[1]) * sc7[2] * 2 * kq.ax; }
                    else cost -= mu6[1] * mu6[1] * hr;
                }
                {   // lateral acceleration
                    const R gv = (kq.ay * kq.ay - max_alat2) * sc7[3];
                    du[17 * S + s] = gv;
                    if (rho * gv + mu6[2] > 0) { cost += gv * (mu6[2] + (R)0.5 * rho * gv); grad_ay += (rho * gv + mu6[2]) * sc7[3] * 2 * kq.ay; }
                    else cost -= mu6[2] * mu6[2] * hr;
                }
                {   // curvature
                    const R scl = use_scaling ? sc7[4] : (R)TP_CUR_SCALE;
                    const R gv = (kq.curv_snorm - max_kap2) * scl;
                    du[18 * S + s] = gv;
                    if (rho * gv + mu6[3] > 0) {
                        const R den = (R)1 / (kq.vx * kq.vx + (R)TP_DELTA_SIGL);
                        cost += gv * (mu6[3] + (R)0.5 * rho * gv);
                        const R ag = (rho * gv + mu6[3]) * scl;
                        grad_wz += ag * den * 2 * kq.wz;
                        grad_vx2 -= ag * kq.curv_snorm * den;
                    } else cost -= mu6[3] * mu6[3] * hr;
                }
                {   // attitude
                    const R gv = (min_cxi - cos_xi) * sc7[5];
                    du[19 * S + s] = gv;
                    if (rho * gv + mu6[4] > 0) {
                        cost += gv * (mu6[4] + (R)0.5 * rho * gv);
                        const R ag = (rho * gv + mu6[4]) * sc7[5];
#pragma unroll
                        for (int k = 0; k < 3; k++) grad_se2[k] -= ag * kq.tg[4][k];
                    } else cost -= mu6[4] * mu6[4] * hr;
                }
                {   // surface variation
                    const R scl = use_scaling ? sc7[6] : (R)TP_SIG_SCALE;
                    const R gv = (sigma - max_sig) * scl;
                    du[20 * S + s] = gv;
                    if (rho * gv + mu6[5] > 0) {
                        cost += gv * (mu6[5] + (R)0.5 * rho * gv);
                        const R ag = (rho * gv + mu6[5]) * scl;
#pragma unroll
                        for (int k = 0; k < 3; k++) grad_se2[k] += ag * kq.tg[6][k];
                    } else cost -= mu6[5] * mu6[5] * hr;
                }
                // chain rule through vx, wz, ax, ay (alm_traj_opt.cpp:948-964)
#pragma unroll
                for (int d = 0; d < 2; d++) grad_v[d] += grad_vx2 * icx * icx * 2 * kq.vel[d];
#pragma unroll
                for (int k = 0; k < 3; k++)
                    grad_se2[k] += grad_vx2 * kq.v_norm * kq.v_norm * 2 * icx * kq.tg[0][k] + grad_wz * kq.dyaw * kq.tg[5][k] +
                                   grad_ax * (gravity * kq.tg[1][k] + kq.tg[0][k] * kq.lon_acc) + grad_ay * (gravity * kq.tg[3][k] + kq.tg[2][k] * kq.lat_acc);
                grad_dyaw += grad_wz * inv_cos_xi;
                grad_a[0] += grad_ax * icx * kq.cyaw - grad_ay * icy * kq.syaw;
                grad_a[1] += grad_ax * icx * kq.syaw + grad_ay * icy * kq.cyaw;
                grad_yaw += grad_ax * icx * kq.lat_acc - grad_ay * icy * kq.lon_acc + grad_se2[2];
                grad_p[0] += grad_se2[0]; grad_p[1] += grad_se2[1];
                // products for the reductions; direct time-gradient terms (alm_traj_opt.cpp:827, 973-975, 984-985; Q3: user_cost / K)
                const R alpha = (R)j / (R)K;
                const R ydot = grad_yaw * kq.dyaw + grad_dyaw * kq.d2yaw;
                // this sample's contributions: basis x gradient (alm_traj_opt.cpp:969-983), the direct time-gradient terms (:827, 973-975, 984-985)
#pragma unroll
                for (int k = 0; k < 6; k++) {
                    cx[k] = kq.b0[k] * grad_p[0] + kq.b1[k] * grad_v[0] + kq.b2[k] * grad_a[0];
                    cx[6 + k] = kq.b0[k] * grad_p[1] + kq.b1[k] * grad_v[1] + kq.b2[k] * grad_a[1];
                }
                cx[12] = user_cost / (R)K +
                         ((grad_p[0] * kq.vel[0] + grad_p[1] * kq.vel[1]) + (grad_v[0] * kq.acc[0] + grad_v[1] * kq.acc[1]) + (grad_a[0] * kq.jer[0] + grad_a[1] * kq.jer[1])) * alpha +
                         ydot * (alpha + (R)i);
                {
                    const R y1 = kq.sy1;
                    R pw = 1, pw1 = 0;
#pragma unroll
                    for (int k = 0; k < 6; k++) { cw[k] = pw * grad_yaw + pw1 * grad_dyaw; pw1 = pw1 * y1 + pw; pw = pw * y1; }
                }
                cw[6] = -ydot * (R)kq.yaw_idx;
            }
            kp.mark(3);
            chunk_scatter<R>(P, on, pl, kq.yaw_idx - ybase, cx, cw, accY, accTy, ybase, M);
            cost_acc += (double)cost;
        }
        parity ^= 1u;
        __syncthreads();
        kp.mark(4);
        // fixed-order sums of this chunk's table; meanwhile the other table and the tile origins are reset for the next chunk
        chunk_gather<R>(P, p0, np, N, M, ybase, gdc, gdt, accY, accTy, tid);
        chunk_part_zero(Pbuf[(it + 1) & 1], tid);
        if (tid < TP_MAXPPC) { sh.org[tid][0] = sh.org[tid][1] = sh.org[tid][2] = 0x7fffffff; sh.org[tid][3] = 0; }
        kp.mark(5);
        __syncthreads();
    }
    // yaw accumulators and the cost out
    for (int q = tid; q < ny; q += TP_KB_THREADS) gdc[TP_CYAW + q] = accY[q];
    for (int q = tid; q < M; q += TP_KB_THREADS) gdt[TP_NMAX + q] = accTy[q];
    cost_acc = warp_sum(cost_acc);
    if ((tid & 31) == 0) s_cost[tid >> 5] = cost_acc;
    __syncthreads();
    if (tid == 0) {
        double c = 0.0;
        for (int w = 0; w < TP_KB_THREADS / 32; w++) c += s_cost[w];
        E.kb_cost[slot] = c;
    }
    kp.mark(6);
}

// ---------------------------------------------------------------------------------------------------------------------
// ks_kernel: initScaling (alm_traj_opt.cpp:349-661) for the trajectories admitted this round.  Per constraint (sample x 7) the
// gradient w.r.t. the decision vector is formed without a linear solve: waypoint part = (waypoint rows of A(1)^-T) . (C^-1 dc),
// time part = z . dc + the direct terms (see scaling_z); scale = 1 / max(1, ||grad||_inf).  scale_fx likewise from the gradient
// of f = jerk + rho_ter int sigma^2 + rho_T T.
// ---------------------------------------------------------------------------------------------------------------------
template <class R>
__global__ void __launch_bounds__(TP_KB_THREADS) ks_kernel(const __grid_constant__ TpPool E, const __grid_constant__ TpParams p, const __grid_constant__ TpMap map, int group)
{
    if ((int)blockIdx.x >= E.n_active[group]) return;
    const int slot = E.active[(size_t)group * E.capacity + blockIdx.x];
    TpState *st = E.st + slot;
    if (!st->need_scale || st->phase == PH_NEW || st->phase == PH_DONE || st->phase == PH_FREE) return;
    const int N = st->N, M = st->M, S = st->S, K = p.int_K, K1 = K + 1, nx = 6 * N, ny = 6 * M, tid = threadIdx.x;
    extern __shared__ __align__(128) unsigned char ks_smem[];
    // layout: ChunkPart | c_xy (12N) | c_yaw (6M) | gf_xy (12N) | gf_yaw (6M) | gT (N + M) | z_xy (12N) | z_yaw (6M)
    ChunkPart<R> &P = *(ChunkPart<R> *)ks_smem;
    R *cxy = (R *)(&P + 1);
    R *cyaw = cxy + 12 * N;
    R *gfx = cyaw + ny;
    R *gfy = gfx + 12 * N;
    R *gT = gfy + ny;
    R *zx = gT + N + M;
    R *zy = zx + 12 * N;
    __shared__ double s_red[TP_KB_THREADS / 32][3];
    const double *cd = E.cd + (size_t)slot * TP_CSTRIDE, *zd = E.gw + (size_t)slot * TP_CSTRIDE;
    for (int q = tid; q < 2 * nx; q += TP_KB_THREADS) { cxy[q] = (R)cd[q]; zx[q] = (R)zd[q]; }
    for (int q = tid; q < ny; q += TP_KB_THREADS) { cyaw[q] = (R)cd[TP_CYAW + q]; zy[q] = (R)zd[TP_CYAW + q]; gfy[q] = 0; }
    for (int q = tid; q < M; q += TP_KB_THREADS) gT[N + q] = 0;
    const int ppc = max(1, min(TP_MAXPPC, TP_KB_THREADS / K1));
    const R Tx = (R)st->Tx, Ty = (R)st->Ty, step = Tx / (R)K, gravity = (R)p.gravity, rho_ter = (R)st->pp[1];
    const R dtdtau = (R)dTdtau(st->tau);
    R ix[6], iy[6];
    ix[0] = iy[0] = 1;
#pragma unroll
    for (int k = 1; k < 6; k++) { ix[k] = ix[k - 1] / Tx; iy[k] = iy[k - 1] / Ty; }
    const R *Wn = (const R *)E.wway + E.wway_off[N], *Wm = (const R *)E.wway + E.wway_off[M];
    R *du = (R *)E.dual + (size_t)slot * TP_NDUAL * E.Smax;
    __syncthreads();
    for (int p0 = 0; p0 < N; p0 += ppc) {
        const int np = min(ppc, N - p0), ns = np * K1;
        chunk_part_zero(P, tid);
        const int ybase = max(0, min((int)((R)p0 * Tx / Ty), M - 1) - 1);
        __syncthreads();
        {
            const int q = tid;               // one pass: ns <= TP_KB_THREADS (int_K <= 127 on this path)
            const bool on = q < ns;
            R cx[13], cw[7];
#pragma unroll
            for (int e = 0; e < 13; e++) cx[e] = 0;
#pragma unroll
            for (int e = 0; e < 7; e++) cw[e] = 0;
            Kin<R> kq;
            kq.yaw_idx = 0;
            int pl = 0;
            if (on) {
            pl = q / K1;
            const int j = q - pl * K1, i = p0 + pl, s = i * K1 + j;
            R pos[2];
            kin_spline<R>(cxy + 6 * i, cxy + nx + 6 * i, cyaw, M, (R)j * step, (R)i * Tx, Ty, kq, pos);
            kin_terrain<R>(map, gravity, pos, norm_yaw(kq.yaw), nullptr, 0, 0, 0, false, kq);
            const R alpha = (R)j / (R)K;
            const int yi = kq.yaw_idx;
            const R icx = kq.tv[0], icy = kq.tv[2], inv_cos_xi = kq.tv[5];
            for (int ct = 0; ct < 7; ct++) {
                R gp[2] = {0, 0}, gv[2] = {0, 0}, ga[2] = {0, 0}, gse[3] = {0, 0, 0}, gyaw = 0, gdyaw = 0;
                if (ct == 0) {                      // non-holonomic (alm_traj_opt.cpp:521-529)
                    gv[0] = kq.syaw; gv[1] = -kq.cyaw;
                    gyaw = kq.vel[0] * kq.cyaw + kq.vel[1] * kq.syaw;
                } else if (ct == 1) {               // vx^2 (:531-544)
                    for (int d = 0; d < 2; d++) gv[d] = icx * icx * 2 * kq.vel[d];
                    for (int k = 0; k < 3; k++) gse[k] = kq.v_norm * kq.v_norm * 2 * icx * kq.tg[0][k];
                } else if (ct == 2) {               // ax^2 (:546-560)
                    const R g = 2 * kq.ax;
                    ga[0] = g * icx * kq.cyaw; ga[1] = g * icx * kq.syaw;
                    gyaw = g * icx * kq.lat_acc;
                    for (int k = 0; k < 3; k++) gse[k] = g * (gravity * kq.tg[1][k] + kq.tg[0][k] * kq.lon_acc);
                } else if (ct == 3) {               // ay^2 (:562-576)
                    const R g = 2 * kq.ay;
                    ga[0] = -g * icy * kq.syaw; ga[1] = g * icy * kq.cyaw;
                    gyaw = -g * icy * kq.lon_acc;
                    for (int k = 0; k < 3; k++) gse[k] = g * (gravity * kq.tg[3][k] + kq.tg[2][k] * kq.lat_acc);
                } else if (ct == 4) {               // curvature (:578-598)
                    const R den = (R)1 / (kq.vx * kq.vx + (R)TP_DELTA_SIGL);
                    const R gwz = den * 2 * kq.wz, gvx2 = -kq.curv_snorm * den;
                    gdyaw = gwz * inv_cos_xi;
                    for (int d = 0; d < 2; d++) gv[d] = gvx2 * icx * icx * 2 * kq.vel[d];
                    for (int k = 0; k < 3; k++) gse[k] = gwz * kq.dyaw * kq.tg[5][k] + gvx2 * kq.v_norm * kq.v_norm * 2 * icx * kq.tg[0][k];
                } else if (ct == 5) {               // attitude (:600-609)
                    for (int k = 0; k < 3; k++) gse[k] = -kq.tg[4][k];
                } else {                            // surface variation (:611-620)
                    for (int k = 0; k < 3; k++) gse[k] = kq.tg[6][k];
                }
                gp[0] = gse[0]; gp[1] = gse[1]; gyaw += gse[2];
                // this constraint's dc: block i of the xy system, block yi of the yaw system; C^-1 applied for the waypoint rows
                R vx[2][6], vw[6];
                R zdot = 0, zdoty = 0;
#pragma unroll
                for (int k = 0; k < 6; k++) {
                    vx[0][k] = kq.b0[k] * gp[0] + kq.b1[k] * gv[0] + kq.b2[k] * ga[0];
                    vx[1][k] = kq.b0[k] * gp[1] + kq.b1[k] * gv[1] + kq.b2[k] * ga[1];
                }
                {
                    const R y1 = kq.sy1;
                    R pw = 1, pw1 = 0;
#pragma unroll
                    for (int k = 0; k < 6; k++) {
                        vw[k] = pw * gyaw + pw1 * gdyaw;
                        pw1 = pw1 * y1 + pw; pw = pw * y1;           // (k+1) y^k , y^(k+1)
                    }
                }
#pragma unroll
                for (int k = 0; k < 6; k++) {
                    zdot += zx[6 * i + k] * vx[0][k] + zx[nx + 6 * i + k] * vx[1][k];
                    zdoty += zy[6 * yi + k] * vw[k];
                    vx[0][k] *= ix[k]; vx[1][k] *= ix[k]; vw[k] *= iy[k];
                }
                R m1 = 0;
                for (int r = 0; r < N - 1; r++) {
                    const R *wr = Wn + (size_t)r * nx + 6 * i;
                    R a = 0, b = 0;
#pragma unroll
                    for (int k = 0; k < 6; k++) { const R wv = wr[k]; a += wv * vx[0][k]; b += wv * vx[1][k]; }
                    m1 = max_(m1, max_(abs_(a), abs_(b)));
                }
                for (int r = 0; r < M - 1; r++) {
                    const R *wr = Wm + (size_t)r * ny + 6 * yi;
                    R a = 0;
#pragma unroll
                    for (int k = 0; k < 6; k++) a += wr[k] * vw[k];
                    m1 = max_(m1, abs_(a));
                }
                const R ydot = gyaw * kq.dyaw + gdyaw * kq.d2yaw;
                const R dTx = ((gp[0] * kq.vel[0] + gp[1] * kq.vel[1]) + (gv[0] * kq.acc[0] + gv[1] * kq.acc[1]) + (ga[0] * kq.jer[0] + ga[1] * kq.jer[1])) * alpha + ydot * (alpha + (R)i);
                const R dTy = -ydot * (R)yi;
                const R gtau = ((dTx + zdot) / (R)N + (dTy + zdoty) / (R)M) * dtdtau;
                du[(7 + ct) * S + s] = (R)1 / max_((R)1, max_(m1, abs_(gtau)));
            }
            // f's user-cost part (alm_traj_opt.cpp:507-519), without scale_fx
            const R omega = ((j == 0 || j == K) ? (R)0.5 : (R)1) * rho_ter * step;
            const R sigma = kq.tv[6];
            const R user_cost = omega * sigma * sigma;
            R gs[3];
            for (int k = 0; k < 3; k++) gs[k] = omega * kq.tg[6][k] * sigma * 2;
#pragma unroll
            for (int k = 0; k < 6; k++) { cx[k] = kq.b0[k] * gs[0]; cx[6 + k] = kq.b0[k] * gs[1]; }
            cx[12] = user_cost / (R)K + (gs[0] * kq.vel[0] + gs[1] * kq.vel[1]) * alpha + gs[2] * kq.dyaw * (alpha + (R)i);
            {
                const R y1 = kq.sy1;
                R pw = 1;
#pragma unroll
                for (int k = 0; k < 6; k++) { cw[k] = pw * gs[2]; pw *= y1; }
            }
            cw[6] = -(gs[2] * kq.dyaw) * (R)yi;
            }
            chunk_scatter<R>(P, on, pl, kq.yaw_idx - ybase, cx, cw, gfy, gT + N, ybase, M);
        }
        __syncthreads();
        chunk_gather<R>(P, p0, np, N, M, ybase, gfx, gT, gfy, gT + N, tid);
        __syncthreads();
    }
    // f gradient: + jerk part (no x1000 factor here: Q7), then waypoint rows / time part as above
    {
        const double X1 = st->Tx, X2 = X1 * X1, X3 = X2 * X1, X4 = X2 * X2, X5 = X4 * X1;
        const double Y1 = st->Ty, Y2 = Y1 * Y1, Y3 = Y2 * Y1, Y4 = Y2 * Y2, Y5 = Y4 * Y1;
        for (int q = tid; q < 2 * nx; q += TP_KB_THREADS) { const int r = q >= nx ? q - nx : q, k = r % 6; gfx[q] += (R)jerk_gc(cd + (q - k), k, X1, X2, X3, X4, X5); }
        for (int q = tid; q < ny; q += TP_KB_THREADS) { const int k = q % 6; gfy[q] += (R)jerk_gc(cd + TP_CYAW + (q - k), k, Y1, Y2, Y3, Y4, Y5); }
        for (int q = tid; q < N + M; q += TP_KB_THREADS) {
            double e, gt;
            if (q < N) jerk_piece(cd + 6 * q, cd + nx + 6 * q, X1, X2, X3, X4, X5, e, gt);
            else jerk_piece(cd + TP_CYAW + 6 * (q - N), nullptr, Y1, Y2, Y3, Y4, Y5, e, gt);
            gT[q] += (R)gt;
        }
    }
    __syncthreads();
    double mx = 0.0, sx = 0.0, sy = 0.0;
    for (int t = tid; t < 2 * (N - 1) + (M - 1); t += TP_KB_THREADS) {
        double a = 0.0;
        if (t < 2 * (N - 1)) {
            const int d = t / (N - 1), r = t - d * (N - 1);
            const R *wr = Wn + (size_t)r * nx;
            for (int c = 0; c < nx; c++) a += (double)wr[c] * (double)gfx[d * nx + c] * (double)ix[c % 6];
        } else {
            const int r = t - 2 * (N - 1);
            const R *wr = Wm + (size_t)r * ny;
            for (int c = 0; c < ny; c++) a += (double)wr[c] * (double)gfy[c] * (double)iy[c % 6];
        }
        mx = fmax(mx, fabs(a));
    }
    for (int q = tid; q < 2 * nx; q += TP_KB_THREADS) sx += (double)zx[q] * (double)gfx[q];
    for (int q = tid; q < ny; q += TP_KB_THREADS) sy += (double)zy[q] * (double)gfy[q];
    for (int q = tid; q < N + M; q += TP_KB_THREADS) { if (q < N) sx += (double)gT[q]; else sy += (double)gT[q]; }
    mx = warp_max(mx); sx = warp_sum(sx); sy = warp_sum(sy);
    if ((tid & 31) == 0) { s_red[tid >> 5][0] = mx; s_red[tid >> 5][1] = sx; s_red[tid >> 5][2] = sy; }
    __syncthreads();
    if (tid == 0) {
        double m = 0.0, a = 0.0, b = 0.0;
        for (int w = 0; w < TP_KB_THREADS / 32; w++) { m = fmax(m, s_red[w][0]); a += s_red[w][1]; b += s_red[w][2]; }
        const double gtau = (st->pp[0] + a / (double)N + b / (double)M) * dTdtau(st->tau);
        st->scale_fx = 1.0 / fmax(1.0, fmax(m, fabs(gtau)));
        st->need_scale = 0;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// results of a finished batch -> packed outputs (reference layouts of include/ualm.h)
// ---------------------------------------------------------------------------------------------------------------------
struct GatherDesc { int slot, N, M, pad; long long off_cxy, off_cyaw, off_x, off_s; };

// problem b (admitted, in slot g.slot) -> the outputs given (null = not wanted), by one CTA
template <class R>
__device__ void gather_one(const TpPool &E, const GatherDesc &g, int b, ualm_result_t *res, double *c_xy, double *c_yaw, double *x_out, double *f_out,
                           double *grad_out, double *hx_out, double *gx_out, double *sfx_out, double *scx_out)
{
    const TpState *st = E.st + g.slot;
    const int N = g.N, M = g.M, n = st->n, S = st->S;
    const double *cd = E.cd + (size_t)g.slot * TP_CSTRIDE;
    const double *vb = E.vec + (size_t)g.slot * 5 * TP_NVAR;
    if (c_xy) for (int q = threadIdx.x; q < 12 * N; q += blockDim.x) c_xy[g.off_cxy + q] = cd[q];
    if (c_yaw) for (int q = threadIdx.x; q < 6 * M; q += blockDim.x) c_yaw[g.off_cyaw + q] = cd[TP_CYAW + q];
    if (x_out) for (int q = threadIdx.x; q < n; q += blockDim.x) x_out[g.off_x + q] = vb[q];
    if (grad_out) for (int q = threadIdx.x; q < n; q += blockDim.x) grad_out[g.off_x + q] = vb[TP_NVAR + q];
    const R *du = (const R *)E.dual + (size_t)g.slot * TP_NDUAL * E.Smax;
    if (hx_out) for (int q = threadIdx.x; q < S; q += blockDim.x) hx_out[g.off_s + q] = (double)du[14 * S + q];
    if (gx_out) for (int q = threadIdx.x; q < S; q += blockDim.x) for (int t = 0; t < 6; t++) gx_out[6 * (g.off_s + q) + t] = (double)du[(15 + t) * S + q];
    if (scx_out) for (int q = threadIdx.x; q < S; q += blockDim.x) for (int t = 0; t < 7; t++) scx_out[7 * (g.off_s + q) + t] = (double)du[(7 + t) * S + q];
    if (threadIdx.x == 0) {
        if (res) {
            ualm_result_t r;
            r.ret_code = st->ret_code; r.outer_iters = st->outer_iter; r.n_evals = st->n_evals; r.n_lbfgs_iters = st->iters_total; r.last_lbfgs_ret = st->last_ret;
            r.max_bound = st->max_bound; r.sum_bound = st->sum_bound; r.reserved = 0; r.inner_cost = st->inner_cost; r.jerk_cost = st->jerk_raw;
            double tt = 0.0;
            for (int i = 0; i < N; i++) tt += st->Tx;
            r.total_T = tt; r.res_h = st->res_h; r.res_g = st->res_g; r.scale_fx = st->scale_fx; r.rho_final = st->rho;
            r.piece_T_xy = st->Tx; r.piece_T_yaw = st->Ty;
            res[b] = r;
        }
        if (f_out) f_out[b] = st->f_last;
        if (sfx_out) sfx_out[b] = st->scale_fx;
    }
}

template <class R>
__global__ void gather_kernel(const __grid_constant__ TpPool E, const GatherDesc *gd, int B, ualm_result_t *res, double *c_xy, double *c_yaw, double *x_out,
                              double *f_out, double *grad_out, double *hx_out, double *gx_out, double *sfx_out, double *scx_out)
{
    const int b = blockIdx.x;
    if (b >= B) return;
    const GatherDesc g = gd[b];
    if (g.slot < 0) return;        // over the compiled limits: its record (UALM_ELIMIT) and zero outputs were written at admission
    gather_one<R>(E, g, b, res, c_xy, c_yaw, x_out, f_out, grad_out, hx_out, gx_out, sfx_out, scx_out);
}

// finished problems of a batch in flight -> the lane's result mailbox (ualm_poll_batch, ualm_mailbox.h), one CTA per problem.  A slot
// is freed only when its batch is collected, so a slot in PH_DONE holds the final state gather_kernel will read: the mailbox gets
// the bits ualm_wait_batch returns.  pub[b] marks problem b published (device memory: the device never reads the mailbox).  Runs
// in the round loop of a group between its rounds, over descriptors that list only that group's problems (ualm_tp.cu)
template <class R>
__global__ void publish_kernel(const __grid_constant__ TpPool E, const GatherDesc *gd, int B, int *pub, const __grid_constant__ ualm_mbox::Ptrs mb)
{
    const int b = blockIdx.x;
    if (b >= B) return;
    const GatherDesc g = gd[b];
    if (g.slot < 0 || pub[b] || E.st[g.slot].phase != PH_DONE) return;     // the same for every thread of the CTA
    gather_one<R>(E, g, b, mb.res, mb.c_xy, mb.c_yaw, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        *(volatile int32_t *)(mb.flag + b) = 1;
        pub[b] = 1;
    }
}

// free the slots of a collected batch
__global__ void free_kernel(const __grid_constant__ TpPool E, const GatherDesc *gd, int B)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B && gd[b].slot >= 0) E.st[gd[b].slot].phase = PH_FREE;
}

} // namespace ualm_tp
