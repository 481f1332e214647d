/*
 * oracle.cpp -- CPU ORACLE (test infrastructure; see oracle.h for the scope statement).
 *
 * Plain C++ restatement of the reference's ALMTrajOpt back-end, same operation order as the
 * reference source wherever that order is visible in the source (explicit loops, `+=` chains).
 * Where the reference hands the order to Eigen (fixed-size products, dot/norm reductions) the
 * oracle uses plain ascending-index accumulation.  Every function cites the file:line it follows
 * (paths relative to /root/reference/src/uneven_planner/).
 *
 * PARITY UNPINNED (no golden vectors exist in the reference; see oracle.h).
 */
#include "oracle.h"
/* Deterministic sin/cos/atan2 shared with the CUDA path (bit-identical on host and device); build with
 * -DORC_LIBM=1 to use libm instead (liboracle_libm.so: shows the last-bit sensitivity, never the gate). */
#include "../include/ualm_detmath.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <vector>

namespace {

#ifndef ORC_LIBM
#define ORC_LIBM 0
#endif
template <class R> struct Mth {
    static R sin(R x) { return std::sin(x); }
    static R cos(R x) { return std::cos(x); }
    static R atan2(R y, R x) { return std::atan2(y, x); }
};
template <> struct Mth<double> {
    static double sin(double x) { return ORC_LIBM ? std::sin(x) : ualm_sin(x); }
    static double cos(double x) { return ORC_LIBM ? std::cos(x) : ualm_cos(x); }
    static double atan2(double y, double x) { return ORC_LIBM ? std::atan2(y, x) : ualm_atan2(y, x); }
};

using clk = std::chrono::steady_clock;
static inline double secs(clk::time_point a, clk::time_point b)
{
    return std::chrono::duration<double>(b - a).count();
}

/* ------------------------------------------------------------------------------------------
 * BandedSystem  (back_end/include/utils/banded_system.hpp:25-145)
 * storage ptrData[(i-j+upperBw)*N + j]; LU without pivoting; exact-zero multipliers skipped (Q10)
 * ---------------------------------------------------------------------------------------- */
template <class R>
struct Banded {
    int N = 0, lo = 0, up = 0;
    std::vector<R> d;
    void create(int n, int p, int q) { N = n; lo = p; up = q; d.assign((size_t)N * (lo + up + 1), R(0)); }
    void reset() { std::fill(d.begin(), d.end(), R(0)); }
    R &operator()(int i, int j) { return d[(size_t)(i - j + up) * N + j]; }
    const R &operator()(int i, int j) const { return d[(size_t)(i - j + up) * N + j]; }

    void factorizeLU() /* banded_system.hpp:66-91 */
    {
        for (int k = 0; k <= N - 2; k++) {
            int iM = std::min(k + lo, N - 1);
            R cVl = (*this)(k, k);
            for (int i = k + 1; i <= iM; i++)
                if ((*this)(i, k) != R(0)) (*this)(i, k) /= cVl;
            int jM = std::min(k + up, N - 1);
            for (int j = k + 1; j <= jM; j++) {
                cVl = (*this)(k, j);
                if (cVl != R(0))
                    for (int i = k + 1; i <= iM; i++)
                        if ((*this)(i, k) != R(0)) (*this)(i, j) -= (*this)(i, k) * cVl;
            }
        }
    }
    /* b: N x m, column-major with leading dimension N (b.row(i) = b[i + c*N], c<m) */
    void solve(R *b, int m) const /* banded_system.hpp:96-118 */
    {
        for (int j = 0; j <= N - 1; j++) {
            int iM = std::min(j + lo, N - 1);
            for (int i = j + 1; i <= iM; i++)
                if ((*this)(i, j) != R(0))
                    for (int c = 0; c < m; c++) b[i + c * N] -= (*this)(i, j) * b[j + c * N];
        }
        for (int j = N - 1; j >= 0; j--) {
            for (int c = 0; c < m; c++) b[j + c * N] /= (*this)(j, j);
            int iM = std::max(0, j - up);
            for (int i = iM; i <= j - 1; i++)
                if ((*this)(i, j) != R(0))
                    for (int c = 0; c < m; c++) b[i + c * N] -= (*this)(i, j) * b[j + c * N];
        }
    }
    void solveAdj(R *b, int m) const /* banded_system.hpp:123-145 */
    {
        for (int j = 0; j <= N - 1; j++) {
            for (int c = 0; c < m; c++) b[j + c * N] /= (*this)(j, j);
            int iM = std::min(j + up, N - 1);
            for (int i = j + 1; i <= iM; i++)
                if ((*this)(j, i) != R(0))
                    for (int c = 0; c < m; c++) b[i + c * N] -= (*this)(j, i) * b[j + c * N];
        }
        for (int j = N - 1; j >= 0; j--) {
            int iM = std::max(0, j - lo);
            for (int i = iM; i <= j - 1; i++)
                if ((*this)(j, i) != R(0))
                    for (int c = 0; c < m; c++) b[i + c * N] -= (*this)(j, i) * b[j + c * N];
        }
    }
};

/* ------------------------------------------------------------------------------------------
 * MinJerkOpt<Dim>  (back_end/include/utils/se2traj.hpp:564-817)
 * c is 6N x Dim, column-major (c(r, d) = c[r + d*6N]) like Eigen::MatrixXd.
 * ---------------------------------------------------------------------------------------- */
template <class R>
struct MinJerk {
    int N = 0, Dim = 1;
    Banded<R> A;
    std::vector<R> c, T1, T2, T3, T4, T5;
    std::vector<R> headPVA, tailPVA; /* Dim x 3 col-major */

    R &C(int r, int d) { return c[r + (size_t)d * 6 * N]; }
    const R &C(int r, int d) const { return c[r + (size_t)d * 6 * N]; }

    void reset(int pieceNum, int dim) /* se2traj.hpp:581-592 */
    {
        N = pieceNum; Dim = dim;
        A.create(6 * N, 6, 6);
        c.assign((size_t)6 * N * Dim, R(0));
        T1.assign(N, 0); T2.assign(N, 0); T3.assign(N, 0); T4.assign(N, 0); T5.assign(N, 0);
    }

    /* inPs Dim x (N-1) col-major; head/tail Dim x 3 col-major   (se2traj.hpp:595-680) */
    void generate(const R *inPs, const R *ts, const R *head, const R *tail)
    {
        headPVA.assign(head, head + 3 * Dim);
        tailPVA.assign(tail, tail + 3 * Dim);
        for (int i = 0; i < N; i++) {
            T1[i] = ts[i];
            T2[i] = T1[i] * T1[i];
            T3[i] = T2[i] * T1[i];
            T4[i] = T2[i] * T2[i];
            T5[i] = T4[i] * T1[i];
        }
        A.reset();
        std::fill(c.begin(), c.end(), R(0));

        A(0, 0) = 1.0; A(1, 1) = 1.0; A(2, 2) = 2.0;
        for (int d = 0; d < Dim; d++) {
            C(0, d) = headPVA[d + 0 * Dim];
            C(1, d) = headPVA[d + 1 * Dim];
            C(2, d) = headPVA[d + 2 * Dim];
        }
        for (int i = 0; i < N - 1; i++) {
            A(6 * i + 3, 6 * i + 3) = 6.0;
            A(6 * i + 3, 6 * i + 4) = R(24.0) * T1[i];
            A(6 * i + 3, 6 * i + 5) = R(60.0) * T2[i];
            A(6 * i + 3, 6 * i + 9) = -6.0;
            A(6 * i + 4, 6 * i + 4) = 24.0;
            A(6 * i + 4, 6 * i + 5) = R(120.0) * T1[i];
            A(6 * i + 4, 6 * i + 10) = -24.0;
            A(6 * i + 5, 6 * i) = 1.0;
            A(6 * i + 5, 6 * i + 1) = T1[i];
            A(6 * i + 5, 6 * i + 2) = T2[i];
            A(6 * i + 5, 6 * i + 3) = T3[i];
            A(6 * i + 5, 6 * i + 4) = T4[i];
            A(6 * i + 5, 6 * i + 5) = T5[i];
            A(6 * i + 6, 6 * i) = 1.0;
            A(6 * i + 6, 6 * i + 1) = T1[i];
            A(6 * i + 6, 6 * i + 2) = T2[i];
            A(6 * i + 6, 6 * i + 3) = T3[i];
            A(6 * i + 6, 6 * i + 4) = T4[i];
            A(6 * i + 6, 6 * i + 5) = T5[i];
            A(6 * i + 6, 6 * i + 6) = -1.0;
            A(6 * i + 7, 6 * i + 1) = 1.0;
            A(6 * i + 7, 6 * i + 2) = R(2) * T1[i];
            A(6 * i + 7, 6 * i + 3) = R(3) * T2[i];
            A(6 * i + 7, 6 * i + 4) = R(4) * T3[i];
            A(6 * i + 7, 6 * i + 5) = R(5) * T4[i];
            A(6 * i + 7, 6 * i + 7) = -1.0;
            A(6 * i + 8, 6 * i + 2) = 2.0;
            A(6 * i + 8, 6 * i + 3) = R(6) * T1[i];
            A(6 * i + 8, 6 * i + 4) = R(12) * T2[i];
            A(6 * i + 8, 6 * i + 5) = R(20) * T3[i];
            A(6 * i + 8, 6 * i + 8) = -2.0;
            for (int d = 0; d < Dim; d++) C(6 * i + 5, d) = inPs[d + (size_t)i * Dim];
        }
        A(6 * N - 3, 6 * N - 6) = 1.0;
        A(6 * N - 3, 6 * N - 5) = T1[N - 1];
        A(6 * N - 3, 6 * N - 4) = T2[N - 1];
        A(6 * N - 3, 6 * N - 3) = T3[N - 1];
        A(6 * N - 3, 6 * N - 2) = T4[N - 1];
        A(6 * N - 3, 6 * N - 1) = T5[N - 1];
        A(6 * N - 2, 6 * N - 5) = 1.0;
        A(6 * N - 2, 6 * N - 4) = R(2) * T1[N - 1];
        A(6 * N - 2, 6 * N - 3) = R(3) * T2[N - 1];
        A(6 * N - 2, 6 * N - 2) = R(4) * T3[N - 1];
        A(6 * N - 2, 6 * N - 1) = R(5) * T4[N - 1];
        A(6 * N - 1, 6 * N - 4) = 2;
        A(6 * N - 1, 6 * N - 3) = R(6) * T1[N - 1];
        A(6 * N - 1, 6 * N - 2) = R(12) * T2[N - 1];
        A(6 * N - 1, 6 * N - 1) = R(20) * T3[N - 1];
        for (int d = 0; d < Dim; d++) {
            C(6 * N - 3, d) = tailPVA[d + 0 * Dim];
            C(6 * N - 2, d) = tailPVA[d + 1 * Dim];
            C(6 * N - 1, d) = tailPVA[d + 2 * Dim];
        }
        A.factorizeLU();
        A.solve(c.data(), Dim);
    }

    R rowdot(int r1, int r2) const
    {
        R s = 0;
        for (int d = 0; d < Dim; d++) s += C(r1, d) * C(r2, d);
        return s;
    }

    R getTrajJerkCost() const /* se2traj.hpp:697-710 */
    {
        R energy = 0.0;
        for (int i = 0; i < N; i++) {
            energy += R(36.0) * rowdot(6 * i + 3, 6 * i + 3) * T1[i] +
                      R(144.0) * rowdot(6 * i + 4, 6 * i + 3) * T2[i] +
                      R(192.0) * rowdot(6 * i + 4, 6 * i + 4) * T3[i] +
                      R(240.0) * rowdot(6 * i + 5, 6 * i + 3) * T3[i] +
                      R(720.0) * rowdot(6 * i + 5, 6 * i + 4) * T4[i] +
                      R(720.0) * rowdot(6 * i + 5, 6 * i + 5) * T5[i];
        }
        return energy;
    }

    /* gdC 6N x Dim col-major, gdT[N]   (se2traj.hpp:719-747) */
    void calJerkGradCT(std::vector<R> &gdC, std::vector<R> &gdT) const
    {
        gdC.assign((size_t)6 * N * Dim, R(0));
        auto G = [&](int r, int d) -> R & { return gdC[r + (size_t)d * 6 * N]; };
        for (int i = 0; i < N; i++)
            for (int d = 0; d < Dim; d++) {
                G(6 * i + 5, d) = R(240.0) * C(6 * i + 3, d) * T3[i] + R(720.0) * C(6 * i + 4, d) * T4[i] +
                                  R(1440.0) * C(6 * i + 5, d) * T5[i];
                G(6 * i + 4, d) = R(144.0) * C(6 * i + 3, d) * T2[i] + R(384.0) * C(6 * i + 4, d) * T3[i] +
                                  R(720.0) * C(6 * i + 5, d) * T4[i];
                G(6 * i + 3, d) = R(72.0) * C(6 * i + 3, d) * T1[i] + R(144.0) * C(6 * i + 4, d) * T2[i] +
                                  R(240.0) * C(6 * i + 5, d) * T3[i];
                G(6 * i + 0, d) = 0; G(6 * i + 1, d) = 0; G(6 * i + 2, d) = 0;
            }
        gdT.assign(N, R(0));
        for (int i = 0; i < N; i++)
            gdT[i] = R(36.0) * rowdot(6 * i + 3, 6 * i + 3) + R(288.0) * rowdot(6 * i + 4, 6 * i + 3) * T1[i] +
                     R(576.0) * rowdot(6 * i + 4, 6 * i + 4) * T2[i] + R(720.0) * rowdot(6 * i + 5, 6 * i + 3) * T2[i] +
                     R(2880.0) * rowdot(6 * i + 5, 6 * i + 4) * T3[i] + R(3600.0) * rowdot(6 * i + 5, 6 * i + 5) * T4[i];
    }

    /* gdC 6N x Dim; gdT in/out; gdP Dim x (N-1) col-major    (se2traj.hpp:751-816) */
    void calGradCTtoQT(const std::vector<R> &gdC, std::vector<R> &gdT, std::vector<R> &gdP,
                       std::vector<R> &adj) const
    {
        gdP.assign((size_t)Dim * std::max(N - 1, 0), R(0));
        adj = gdC;
        A.solveAdj(adj.data(), Dim);
        auto AD = [&](int r, int d) -> R { return adj[r + (size_t)d * 6 * N]; };
        for (int i = 0; i < N - 1; i++)
            for (int d = 0; d < Dim; d++) gdP[d + (size_t)i * Dim] = AD(6 * i + 5, d);

        R B1[6][2];
        for (int i = 0; i < N - 1; i++) {
            for (int d = 0; d < Dim; d++) {
                /* negative velocity */
                B1[2][d] = -(C(i * 6 + 1, d) + R(2.0) * T1[i] * C(i * 6 + 2, d) + R(3.0) * T2[i] * C(i * 6 + 3, d) +
                             R(4.0) * T3[i] * C(i * 6 + 4, d) + R(5.0) * T4[i] * C(i * 6 + 5, d));
                B1[3][d] = B1[2][d];
                /* negative acceleration */
                B1[4][d] = -(R(2.0) * C(i * 6 + 2, d) + R(6.0) * T1[i] * C(i * 6 + 3, d) +
                             R(12.0) * T2[i] * C(i * 6 + 4, d) + R(20.0) * T3[i] * C(i * 6 + 5, d));
                /* negative jerk */
                B1[5][d] = -(R(6.0) * C(i * 6 + 3, d) + R(24.0) * T1[i] * C(i * 6 + 4, d) +
                             R(60.0) * T2[i] * C(i * 6 + 5, d));
                /* negative snap */
                B1[0][d] = -(R(24.0) * C(i * 6 + 4, d) + R(120.0) * T1[i] * C(i * 6 + 5, d));
                /* negative crackle */
                B1[1][d] = R(-120.0) * C(i * 6 + 5, d);
            }
            /* B1.cwiseProduct(adj.block<6,Dim>(6i+3,0)).sum(): column-major traversal */
            R s = 0;
            for (int d = 0; d < Dim; d++)
                for (int r = 0; r < 6; r++) s += B1[r][d] * AD(6 * i + 3 + r, d);
            gdT[i] += s;
        }
        R B2[3][2];
        for (int d = 0; d < Dim; d++) {
            B2[0][d] = -(C(6 * N - 5, d) + R(2.0) * T1[N - 1] * C(6 * N - 4, d) + R(3.0) * T2[N - 1] * C(6 * N - 3, d) +
                         R(4.0) * T3[N - 1] * C(6 * N - 2, d) + R(5.0) * T4[N - 1] * C(6 * N - 1, d));
            B2[1][d] = -(R(2.0) * C(6 * N - 4, d) + R(6.0) * T1[N - 1] * C(6 * N - 3, d) +
                         R(12.0) * T2[N - 1] * C(6 * N - 2, d) + R(20.0) * T3[N - 1] * C(6 * N - 1, d));
            B2[2][d] = -(R(6.0) * C(6 * N - 3, d) + R(24.0) * T1[N - 1] * C(6 * N - 2, d) +
                         R(60.0) * T2[N - 1] * C(6 * N - 1, d));
        }
        R s = 0;
        for (int d = 0; d < Dim; d++)
            for (int r = 0; r < 3; r++) s += B2[r][d] * AD(6 * N - 3 + r, d);
        gdT[N - 1] += s;
    }
};

/* ------------------------------------------------------------------------------------------
 * UnevenMap query half  (uneven_map/include/uneven_map/uneven_map.h:258-377, 398-454;
 *                        uneven_map/src/uneven_map.cpp:64-71)
 * ---------------------------------------------------------------------------------------- */
template <class R>
static inline void normSO2(R &yaw) /* uneven_map.cpp:64-71 */
{
    while (yaw < R(-M_PI)) yaw += R(2 * M_PI);
    while (yaw > R(M_PI)) yaw -= R(2 * M_PI);
}

template <class R>
struct MapQ {
    const double *cells;
    int vn[3];
    R origin[3], maxb[3], xy_res, yaw_res, xy_inv, yaw_inv;

    explicit MapQ(const orc_map_t &m)
    {
        cells = m.cells;
        for (int k = 0; k < 3; k++) { vn[k] = m.voxel_num[k]; origin[k] = (R)m.origin[k]; maxb[k] = (R)m.max_boundary[k]; }
        xy_res = (R)m.xy_resolution; yaw_res = (R)m.yaw_resolution;
        xy_inv = R(1.0) / xy_res; yaw_inv = R(1.0) / yaw_res; /* uneven_map.cpp:104-105 */
    }
    bool isInMap(const R pos[3]) const /* uneven_map.h:437-454 */
    {
        if (pos[0] < origin[0] + R(1e-4) || pos[1] < origin[1] + R(1e-4) || pos[2] < origin[2] + R(1e-4)) return false;
        if (pos[0] > maxb[0] - R(1e-4) || pos[1] > maxb[1] - R(1e-4) || pos[2] > maxb[2] - R(1e-4)) return false;
        return true;
    }
    /* value = {sigma, zbx, zby}; grad 4x3 rows {sigma, zbx, zby, c} cols {x, y, yaw}
     * (uneven_map.h:258-315); z is never interpolated on this path (toVector, uneven_map.h:60-63) */
    void getTerrainWithGradI(const R pos[3], R val[3], R grad[4][3]) const
    {
        if (!isInMap(pos)) {
            for (int r = 0; r < 4; r++) for (int k = 0; k < 3; k++) grad[r][k] = 0;
            val[0] = val[1] = val[2] = 0;
            return;
        }
        R pos_m[3] = {pos[0] - R(0.5) * xy_res, pos[1] - R(0.5) * xy_res, pos[2] - R(0.5) * yaw_res};
        normSO2(pos_m[2]);
        int idx[3];
        idx[0] = (int)std::floor((pos_m[0] - origin[0]) * xy_inv); /* posToIndex uneven_map.h:411-417 */
        idx[1] = (int)std::floor((pos_m[1] - origin[1]) * xy_inv);
        idx[2] = (int)std::floor((pos_m[2] - origin[2]) * yaw_inv);
        R idx_pos[3]; /* indexToPos uneven_map.h:419-425 */
        idx_pos[0] = (R(idx[0]) + R(0.5)) * xy_res + origin[0];
        idx_pos[1] = (R(idx[1]) + R(0.5)) * xy_res + origin[1];
        idx_pos[2] = (R(idx[2]) + R(0.5)) * yaw_res + origin[2];
        R diff[3];
        diff[0] = (pos[0] - idx_pos[0]) * xy_inv;
        diff[1] = (pos[1] - idx_pos[1]) * xy_inv;
        diff[2] = Mth<R>::atan2(Mth<R>::sin(pos[2] - idx_pos[2]), Mth<R>::cos(pos[2] - idx_pos[2])) * yaw_inv;

        R v[2][2][2][3];
        for (int x = 0; x < 2; x++)
            for (int y = 0; y < 2; y++)
                for (int w = 0; w < 2; w++) {
                    int ci[3] = {idx[0] + x, idx[1] + y, idx[2] + w};
                    /* boundIndex uneven_map.h:398-409 */
                    ci[0] = std::max(std::min(ci[0], vn[0] - 1), 0);
                    ci[1] = std::max(std::min(ci[1], vn[1] - 1), 0);
                    while (ci[2] > vn[2] - 1) ci[2] -= vn[2];
                    while (ci[2] < 0) ci[2] += vn[2];
                    size_t a = (size_t)ci[0] * vn[1] * vn[2] + (size_t)ci[1] * vn[2] + ci[2];
                    v[x][y][w][0] = (R)cells[4 * a + 1];
                    v[x][y][w][1] = (R)cells[4 * a + 2];
                    v[x][y][w][2] = (R)cells[4 * a + 3];
                }
        R v00[3], v01[3], v10[3], v11[3], v0[3], v1[3];
        for (int k = 0; k < 3; k++) {
            v00[k] = v[0][0][0][k] * (1 - diff[0]) + v[1][0][0][k] * diff[0];
            v01[k] = v[0][0][1][k] * (1 - diff[0]) + v[1][0][1][k] * diff[0];
            v10[k] = v[0][1][0][k] * (1 - diff[0]) + v[1][1][0][k] * diff[0];
            v11[k] = v[0][1][1][k] * (1 - diff[0]) + v[1][1][1][k] * diff[0];
            v0[k] = v00[k] * (1 - diff[1]) + v10[k] * diff[1];
            v1[k] = v01[k] * (1 - diff[1]) + v11[k] * diff[1];
            val[k] = v0[k] * (1 - diff[2]) + v1[k] * diff[2];
        }
        for (int k = 0; k < 3; k++) {
            grad[k][2] = (v1[k] - v0[k]) * yaw_inv;
            grad[k][1] = ((v10[k] - v00[k]) * (1 - diff[2]) + (v11[k] - v01[k]) * diff[2]) * xy_inv;
            R g0 = (1 - diff[2]) * (1 - diff[1]) * (v[1][0][0][k] - v[0][0][0][k]);
            g0 += (1 - diff[2]) * diff[1] * (v[1][1][0][k] - v[0][1][0][k]);
            g0 += diff[2] * (1 - diff[1]) * (v[1][0][1][k] - v[0][0][1][k]);
            g0 += diff[2] * diff[1] * (v[1][1][1][k] - v[0][1][1][k]);
            g0 *= xy_inv;
            grad[k][0] = g0;
        }
        R c = std::sqrt(R(1.0) - val[1] * val[1] - val[2] * val[2]); /* getC uneven_map.h:46 */
        for (int k = 0; k < 3; k++) grad[3][k] = -(grad[1][k] * val[1] + grad[2][k] * val[2]) / c;
    }

    /* values[7] / grads[7][3] = {inv_cos_vphix, sin_phix, inv_cos_vphiy, sin_phiy, cos_xi,
     * inv_cos_xi, sigma}  (uneven_map.h:318-377) */
    void getAllWithGrad(const R pos[3], R values[7], R grads[7][3]) const
    {
        R rs[3], rg[4][3];
        getTerrainWithGradI(pos, rs, rg);
        R c = std::sqrt(R(1.0) - rs[1] * rs[1] - rs[2] * rs[2]);
        R inv_c = R(1.0) / c;
        R cyaw = Mth<R>::cos(pos[2]);
        R syaw = Mth<R>::sin(pos[2]);
        R xyaw[2] = {cyaw, syaw};
        R yyaw[2] = {-syaw, cyaw};
        R t = xyaw[0] * rs[1] + xyaw[1] * rs[2];
        R s = -(yyaw[0] * rs[1] + yyaw[1] * rs[2]);
        R sqrt_1_t2 = std::sqrt(R(1.0) - t * t);
        R inv_sqrt_1_t2 = R(1.0) / sqrt_1_t2;
        R inv_sqrt_1_t2_3 = inv_sqrt_1_t2 * inv_sqrt_1_t2 * inv_sqrt_1_t2;
        R dt[3], ds[3];
        for (int k = 0; k < 3; k++) {
            dt[k] = rg[1][k] * xyaw[0] + rg[2][k] * xyaw[1];
            ds[k] = -(rg[1][k] * yyaw[0] + rg[2][k] * yyaw[1]);
        }
        dt[2] -= s;
        ds[2] += t;

        values[0] = inv_sqrt_1_t2;
        values[1] = -c * t * inv_sqrt_1_t2;
        values[2] = sqrt_1_t2 * inv_c;
        values[3] = s * inv_sqrt_1_t2;
        values[4] = c;
        values[5] = inv_c;
        values[6] = rs[0];
        for (int k = 0; k < 3; k++) {
            grads[0][k] = t * inv_sqrt_1_t2_3 * dt[k];
            grads[1][k] = -(t * inv_sqrt_1_t2 * rg[3][k] + inv_sqrt_1_t2_3 * c * dt[k]);
            grads[2][k] = -inv_c * (t * inv_sqrt_1_t2 * dt[k] + sqrt_1_t2 * inv_c * rg[3][k]);
            grads[3][k] = inv_sqrt_1_t2 * ds[k] + t * inv_sqrt_1_t2_3 * s * dt[k];
            grads[4][k] = rg[3][k];
            grads[5][k] = -inv_c * inv_c * rg[3][k];
            grads[6][k] = rg[0][k];
        }
    }
};

/* ------------------------------------------------------------------------------------------
 * lbfgs  (back_end/include/utils/lbfgs.hpp:15-129 parameters, 276-389 line search, 439-722 driver)
 * ---------------------------------------------------------------------------------------- */
enum {
    LBFGS_CONVERGENCE = 0, LBFGS_STOP, LBFGS_CANCELED,
    LBFGSERR_UNKNOWNERROR = -1024, LBFGSERR_INVALID_N, LBFGSERR_INVALID_MEMSIZE, LBFGSERR_INVALID_GEPSILON,
    LBFGSERR_INVALID_TESTPERIOD, LBFGSERR_INVALID_DELTA, LBFGSERR_INVALID_MINSTEP, LBFGSERR_INVALID_MAXSTEP,
    LBFGSERR_INVALID_FDECCOEFF, LBFGSERR_INVALID_SCURVCOEFF, LBFGSERR_INVALID_MACHINEPREC,
    LBFGSERR_INVALID_MAXLINESEARCH, LBFGSERR_INVALID_FUNCVAL, LBFGSERR_MINIMUMSTEP, LBFGSERR_MAXIMUMSTEP,
    LBFGSERR_MAXIMUMLINESEARCH, LBFGSERR_MAXIMUMITERATION, LBFGSERR_WIDTHTOOSMALL, LBFGSERR_INVALIDPARAMETERS,
    LBFGSERR_INCREASEGRADIENT,
};

template <class R>
struct LbfgsParam {
    int mem_size = 8;
    R g_epsilon = R(1.0e-5);
    int past = 3;
    R delta = R(1.0e-6);
    int max_iterations = 0;
    int max_linesearch = 64;
    R min_step = R(1.0e-20);
    R max_step = R(1.0e+20);
    R f_dec_coeff = R(1.0e-4);
    R s_curv_coeff = R(0.9);
    R cautious_factor = R(1.0e-6);
    R machine_prec = R(1.0e-16);
};

/* Dot product in the CANONICAL 32-LANE ORDER.  The reference leaves the order of dot()/norm() reductions to
 * Eigen's SIMD packet code (unspecified, version- and flag-dependent); the oracle fixes it to the order a GPU warp
 * produces so the CUDA path can reproduce it bit for bit: lane l accumulates elements l, l+32, l+64, ... in
 * ascending order, then the 32 partials are combined by the xor-butterfly 16, 8, 4, 2, 1. */
template <class R>
static R vdot(const R *a, const R *b, int n)
{
    R p[32], q[32];
    for (int l = 0; l < 32; l++) p[l] = 0;
    for (int i = 0; i < n; i++) p[i & 31] += a[i] * b[i];
    for (int off = 16; off >= 1; off >>= 1) {
        for (int l = 0; l < 32; l++) q[l] = p[l] + p[l ^ off];
        for (int l = 0; l < 32; l++) p[l] = q[l];
    }
    return p[0];
}
template <class R>
static R vabsmax(const R *a, int n) { R s = 0; for (int i = 0; i < n; i++) s = std::max(s, std::fabs(a[i])); return s; }

template <class R, class Eval>
static int line_search_lewisoverton(std::vector<R> &x, R &f, std::vector<R> &g, R &stp, const std::vector<R> &s,
                                    const std::vector<R> &xp, const std::vector<R> &gp, R stpmin, R stpmax,
                                    Eval &eval, const LbfgsParam<R> &param) /* lbfgs.hpp:276-389 */
{
    const int n = (int)x.size();
    int count = 0;
    bool brackt = false, touched = false;
    R finit, dginit, dgtest, dstest;
    R mu = 0.0, nu = stpmax;

    if (!(stp > R(0.0))) return LBFGSERR_INVALIDPARAMETERS;
    dginit = vdot(gp.data(), s.data(), n);
    if (R(0.0) < dginit) return LBFGSERR_INCREASEGRADIENT;
    finit = f;
    dgtest = param.f_dec_coeff * dginit;
    dstest = param.s_curv_coeff * dginit;

    while (true) {
        for (int i = 0; i < n; i++) x[i] = xp[i] + stp * s[i];
        f = eval(x, g);
        ++count;
        if (std::isinf(f) || std::isnan(f)) return LBFGSERR_INVALID_FUNCVAL;
        /* local modification of the reference (lbfgs.hpp:327-330) */
        if (param.past > 0 && std::fabs(finit - f) / (std::fabs(finit) + R(1.0)) < param.delta / R(param.past)) return count;
        if (f > finit + stp * dgtest) {
            nu = stp;
            brackt = true;
        } else {
            if (vdot(g.data(), s.data(), n) < dstest) mu = stp;
            else return count;
        }
        if (param.max_linesearch <= count) return LBFGSERR_MAXIMUMLINESEARCH;
        if (brackt && (nu - mu) < param.machine_prec * nu) return LBFGSERR_WIDTHTOOSMALL;
        if (brackt) stp = R(0.5) * (mu + nu);
        else stp *= R(2.0);
        if (stp < stpmin) return LBFGSERR_MINIMUMSTEP;
        if (stp > stpmax) {
            if (touched) return LBFGSERR_MAXIMUMSTEP;
            touched = true;
            stp = stpmax;
        }
    }
}

struct LbfgsStats { int iters = 0; int max_bound = 0; };

/* progress(k) returns non-zero to cancel   (lbfgs.hpp:439-722) */
template <class R, class Eval, class Progress>
static int lbfgs_optimize(std::vector<R> &x, R &f, Eval &eval, Progress &progress, const LbfgsParam<R> &param,
                          LbfgsStats &st)
{
    int ret, i, j, k, ls, end, bound;
    R step, step_min, step_max, fx, ys, yy;
    R gnorm_inf, xnorm_inf, beta, rate, cau;
    const int n = (int)x.size();
    const int m = param.mem_size;

    if (n <= 0) return LBFGSERR_INVALID_N;
    if (m <= 0) return LBFGSERR_INVALID_MEMSIZE;
    if (param.g_epsilon < R(0.0)) return LBFGSERR_INVALID_GEPSILON;
    if (param.past < 0) return LBFGSERR_INVALID_TESTPERIOD;
    if (param.delta < R(0.0)) return LBFGSERR_INVALID_DELTA;
    if (param.min_step < R(0.0)) return LBFGSERR_INVALID_MINSTEP;
    if (param.max_step < param.min_step) return LBFGSERR_INVALID_MAXSTEP;
    if (!(param.f_dec_coeff > R(0.0) && param.f_dec_coeff < R(1.0))) return LBFGSERR_INVALID_FDECCOEFF;
    if (!(param.s_curv_coeff < R(1.0) && param.s_curv_coeff > param.f_dec_coeff)) return LBFGSERR_INVALID_SCURVCOEFF;
    if (!(param.machine_prec > R(0.0))) return LBFGSERR_INVALID_MACHINEPREC;
    if (param.max_linesearch <= 0) return LBFGSERR_INVALID_MAXLINESEARCH;

    std::vector<R> xp(n), g(n), gp(n), d(n), pf(std::max(1, param.past));
    std::vector<R> lm_alpha(m, R(0)), lm_ys(m, R(0));
    std::vector<R> lm_s((size_t)n * m, R(0)), lm_y((size_t)n * m, R(0)); /* col-major n x m */

    fx = eval(x, g);
    pf[0] = fx;
    for (i = 0; i < n; i++) d[i] = -g[i];
    gnorm_inf = vabsmax(g.data(), n);
    xnorm_inf = vabsmax(x.data(), n);

    if (gnorm_inf / std::max(R(1.0), xnorm_inf) < param.g_epsilon) {
        ret = LBFGS_CONVERGENCE;
    } else {
        step = R(1.0) / std::sqrt(vdot(d.data(), d.data(), n));
        k = 1; end = 0; bound = 0;
        while (true) {
            xp = x; gp = g;
            step_min = param.min_step;
            step_max = param.max_step;
            ls = line_search_lewisoverton(x, fx, g, step, d, xp, gp, step_min, step_max, eval, param);
            if (ls < 0) { x = xp; g = gp; ret = ls; break; }
            st.iters++;
            if (progress(k)) { ret = LBFGS_CANCELED; break; }
            gnorm_inf = vabsmax(g.data(), n);
            xnorm_inf = vabsmax(x.data(), n);
            if (gnorm_inf / std::max(R(1.0), xnorm_inf) < param.g_epsilon) { ret = LBFGS_CONVERGENCE; break; }
            if (0 < param.past) {
                if (param.past <= k) {
                    rate = std::fabs(pf[k % param.past] - fx) / std::max(R(1.0), std::fabs(fx));
                    if (rate < param.delta) { ret = LBFGS_STOP; break; }
                }
                pf[k % param.past] = fx;
            }
            if (param.max_iterations != 0 && param.max_iterations <= k) { ret = LBFGSERR_MAXIMUMITERATION; break; }
            ++k;
            R *sE = &lm_s[(size_t)end * n], *yE = &lm_y[(size_t)end * n];
            for (i = 0; i < n; i++) { sE[i] = x[i] - xp[i]; yE[i] = g[i] - gp[i]; }
            ys = vdot(yE, sE, n);
            yy = vdot(yE, yE, n);
            lm_ys[end] = ys;
            for (i = 0; i < n; i++) d[i] = -g[i];
            cau = vdot(sE, sE, n) * std::sqrt(vdot(gp.data(), gp.data(), n)) * param.cautious_factor;
            if (ys > cau) {
                ++bound;
                bound = m < bound ? m : bound;
                st.max_bound = std::max(st.max_bound, bound);
                end = (end + 1) % m;
                j = end;
                for (i = 0; i < bound; ++i) {
                    j = (j + m - 1) % m;
                    lm_alpha[j] = vdot(&lm_s[(size_t)j * n], d.data(), n) / lm_ys[j];
                    const R na = -lm_alpha[j];
                    const R *yj = &lm_y[(size_t)j * n];
                    for (int q = 0; q < n; q++) d[q] += na * yj[q];
                }
                const R sc = ys / yy;
                for (int q = 0; q < n; q++) d[q] *= sc;
                for (i = 0; i < bound; ++i) {
                    beta = vdot(&lm_y[(size_t)j * n], d.data(), n) / lm_ys[j];
                    const R cf = lm_alpha[j] - beta;
                    const R *sj = &lm_s[(size_t)j * n];
                    for (int q = 0; q < n; q++) d[q] += cf * sj[q];
                    j = (j + 1) % m;
                }
            }
            step = 1.0;
        }
    }
    f = fx;
    return ret;
}

/* ------------------------------------------------------------------------------------------
 * ALMTrajOpt  (back_end/src/alm_traj_opt.cpp, back_end/include/back_end/alm_traj_opt.h)
 * ---------------------------------------------------------------------------------------- */
constexpr double delta_sigl = 0.01;        /* alm_traj_opt.h:16-19 */
constexpr double cur_scale = 10.0;
constexpr double sig_scale = 1000.0;
constexpr double scale_trick_jerk = 1000.0;

template <class R>
static inline R expC2(R tau) /* alm_traj_opt.h:232-235 */
{
    return tau > R(0.0) ? ((R(0.5) * tau + R(1.0)) * tau + R(1.0)) : R(1.0) / ((R(0.5) * tau - R(1.0)) * tau + R(1.0));
}
template <class R>
static inline R logC2(R T) /* alm_traj_opt.h:238-241 */
{
    return T > R(1.0) ? (std::sqrt(R(2.0) * T - R(1.0)) - R(1.0)) : (R(1.0) - std::sqrt(R(2.0) / T - R(1.0)));
}
template <class R>
static inline R getTtoTauGrad(R tau) /* alm_traj_opt.h:244-253 */
{
    if (tau > 0) return tau + R(1.0);
    R denSqrt = (R(0.5) * tau - R(1.0)) * tau + R(1.0);
    return (R(1.0) - tau) / (denSqrt * denSqrt);
}

template <class R>
struct ALM {
    /* params */
    R rho_T, rho_ter, max_vel, max_acc_lon, max_acc_lat, max_kap, min_cxi, max_sig;
    bool use_scaling;
    R rho, beta, gamma, epsilon_con;
    double max_iter;
    R g_epsilon, min_step, delta;
    double inner_max_iter;
    int mem_size, past, int_K;
    R gravity;
    /* data (alm_traj_opt.h:60-78) */
    int piece_xy = 0, piece_yaw = 0, dim_T = 1;
    int equal_num = 0, non_equal_num = 0;
    R scale_fx = 1;
    std::vector<R> lambda, mu, hx, gx, scale_cx;
    R init_xy[6], end_xy[6], init_yaw[3], end_yaw[3];
    MinJerk<R> pos_minco, yaw_minco;
    const MapQ<R> *map = nullptr;
    /* bookkeeping */
    int n_evals = 0;
    double t_minco = 0, t_penalty = 0, t_adjoint = 0, t_scaling = 0;
    /* last constraint-term (C,T) gradients, for kernel-level parity */
    std::vector<R> last_gdCxy, last_gdTxy, last_gdCyaw, last_gdTyaw;
    R last_parts[3];

    ALM(const orc_params_t &p, const MapQ<R> *m) : map(m)
    {
        rho_T = (R)p.rho_T; rho_ter = (R)p.rho_ter; max_vel = (R)p.max_vel; max_acc_lon = (R)p.max_acc_lon;
        max_acc_lat = (R)p.max_acc_lat; max_kap = (R)p.max_kap; min_cxi = (R)p.min_cxi; max_sig = (R)p.max_sig;
        use_scaling = p.use_scaling != 0; rho = (R)p.rho; beta = (R)p.beta; gamma = (R)p.gamma;
        epsilon_con = (R)p.epsilon_con; max_iter = p.max_iter; g_epsilon = (R)p.g_epsilon; min_step = (R)p.min_step;
        delta = (R)p.delta; inner_max_iter = p.inner_max_iter; mem_size = p.mem_size; past = p.past; int_K = p.int_K;
        gravity = (R)p.gravity;
    }

    R getAugmentedCost(R h_or_g, R lambda_or_mu) const { return h_or_g * (lambda_or_mu + R(0.5) * rho * h_or_g); } /* alm_traj_opt.h:154-157 */
    R getAugmentedGrad(R h_or_g, R lambda_or_mu) const { return rho * h_or_g + lambda_or_mu; }                     /* alm_traj_opt.h:160-163 */

    void setup(const orc_problem_t &pr) /* alm_traj_opt.cpp:180-203 */
    {
        piece_xy = pr.N; piece_yaw = pr.M;
        pos_minco.reset(piece_xy, 2);
        yaw_minco.reset(piece_yaw, 1);
        for (int i = 0; i < 6; i++) { init_xy[i] = (R)pr.init_xy[i]; end_xy[i] = (R)pr.end_xy[i]; }
        for (int i = 0; i < 3; i++) { init_yaw[i] = (R)pr.init_yaw[i]; end_yaw[i] = (R)pr.end_yaw[i]; }
        equal_num = piece_xy * (int_K + 1);
        non_equal_num = piece_xy * (int_K + 1) * 6;
        hx.assign(equal_num, R(0)); lambda.assign(equal_num, R(0));
        gx.assign(non_equal_num, R(0)); mu.assign(non_equal_num, R(0));
        scale_fx = 1.0;
        scale_cx.assign(equal_num + non_equal_num, R(1.0));
    }
    int nvar() const { return 2 * (piece_xy - 1) + (piece_yaw - 1) + 1; }

    void generate(const R *x) /* alm_traj_opt.cpp:293-299: uniform durations (alm_traj_opt.h:257-261) */
    {
        const R tau = x[0];
        std::vector<R> Txy(piece_xy), Tyaw(piece_yaw);
        const R Tx = expC2(tau) / R(piece_xy), Ty = expC2(tau) / R(piece_yaw);
        for (auto &t : Txy) t = Tx;
        for (auto &t : Tyaw) t = Ty;
        pos_minco.generate(x + dim_T, Txy.data(), init_xy, end_xy);
        yaw_minco.generate(x + dim_T + 2 * (piece_xy - 1), Tyaw.data(), init_yaw, end_yaw);
    }

    /* ----- per-sample kinematics shared by calConstrainCostGrad and initScaling ----- */
    struct Sample {
        R beta0_xy[6], beta1_xy[6], beta2_xy[6], beta3_xy[6];
        R beta0_yaw[6], beta1_yaw[6], beta2_yaw[6];
        R pos[2], vel[2], acc[2], jer[2];
        R yaw, dyaw, d2yaw, syaw, cyaw, v_norm, xb[2], yb[2], lon_acc, lat_acc;
        R tv[7], tg[7][3];
        R vx, wz, ax, ay, curv_snorm;
        int yaw_idx;
    };
    void sample(int i, R s1, R base_time, Sample &S) const /* alm_traj_opt.cpp:733-817 (== 439-505) */
    {
        const int NX = 6 * piece_xy;
        R s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2, s5 = s4 * s1;
        R b0[6] = {R(1.0), s1, s2, s3, s4, s5};
        R b1[6] = {R(0.0), R(1.0), R(2.0) * s1, R(3.0) * s2, R(4.0) * s3, R(5.0) * s4};
        R b2[6] = {R(0.0), R(0.0), R(2.0), R(6.0) * s1, R(12.0) * s2, R(20.0) * s3};
        R b3[6] = {R(0.0), R(0.0), R(0.0), R(6.0), R(24.0) * s1, R(60.0) * s2};
        for (int k = 0; k < 6; k++) { S.beta0_xy[k] = b0[k]; S.beta1_xy[k] = b1[k]; S.beta2_xy[k] = b2[k]; S.beta3_xy[k] = b3[k]; }
        for (int d = 0; d < 2; d++) {
            R p = 0, v = 0, a = 0, j = 0;
            for (int k = 0; k < 6; k++) {
                const R c = pos_minco.c[6 * i + k + (size_t)d * NX];
                p += c * b0[k]; v += c * b1[k]; a += c * b2[k]; j += c * b3[k];
            }
            S.pos[d] = p; S.vel[d] = v; S.acc[d] = a; S.jer[d] = j;
        }
        /* Q4: yaw duration vector indexed with the xy piece index i (alm_traj_opt.cpp:749,753) */
        R now_time = s1 + base_time;
        int yaw_idx = int((now_time) / yaw_minco.T1[std::min(i, piece_yaw - 1)]);
        if (yaw_idx >= piece_yaw) yaw_idx = piece_yaw - 1;
        S.yaw_idx = yaw_idx;
        R sy1 = now_time - R(yaw_idx) * yaw_minco.T1[std::min(i, piece_yaw - 1)];
        R sy2 = sy1 * sy1, sy3 = sy2 * sy1, sy4 = sy2 * sy2, sy5 = sy4 * sy1;
        R y0[6] = {R(1.0), sy1, sy2, sy3, sy4, sy5};
        R y1[6] = {R(0.0), R(1.0), R(2.0) * sy1, R(3.0) * sy2, R(4.0) * sy3, R(5.0) * sy4};
        R y2[6] = {R(0.0), R(0.0), R(2.0), R(6.0) * sy1, R(12.0) * sy2, R(20.0) * sy3};
        R yaw = 0, dyaw = 0, d2yaw = 0;
        for (int k = 0; k < 6; k++) {
            const R c = yaw_minco.c[6 * yaw_idx + k];
            yaw += c * y0[k]; dyaw += c * y1[k]; d2yaw += c * y2[k];
            S.beta0_yaw[k] = y0[k]; S.beta1_yaw[k] = y1[k]; S.beta2_yaw[k] = y2[k];
        }
        S.yaw = yaw; S.dyaw = dyaw; S.d2yaw = d2yaw;
        R se2_pos[3] = {S.pos[0], S.pos[1], yaw};
        normSO2(se2_pos[2]);
        S.syaw = Mth<R>::sin(yaw); S.cyaw = Mth<R>::cos(yaw);
        S.v_norm = std::sqrt(S.vel[0] * S.vel[0] + S.vel[1] * S.vel[1]);
        S.xb[0] = S.cyaw; S.xb[1] = S.syaw; S.yb[0] = -S.syaw; S.yb[1] = S.cyaw;
        S.lon_acc = S.acc[0] * S.xb[0] + S.acc[1] * S.xb[1];
        S.lat_acc = S.acc[0] * S.yb[0] + S.acc[1] * S.yb[1];
        map->getAllWithGrad(se2_pos, S.tv, S.tg);
        S.vx = S.v_norm * S.tv[0];
        S.wz = dyaw * S.tv[5];
        S.ax = S.lon_acc * S.tv[0] + gravity * S.tv[1];
        S.ay = S.lat_acc * S.tv[2] + gravity * S.tv[3];
        S.curv_snorm = S.wz * S.wz / (S.vx * S.vx + R(delta_sigl));
    }

    /* alm_traj_opt.cpp:663-991.  gdCxy 6N x 2 col-major, gdTxy[N], gdCyaw[6M], gdTyaw[M] */
    void calConstrainCostGrad(R &cost, std::vector<R> &gdCxy, std::vector<R> &gdTxy, std::vector<R> &gdCyaw,
                              std::vector<R> &gdTyaw)
    {
        const int NX = 6 * piece_xy;
        cost = 0.0;
        gdCxy.assign((size_t)NX * 2, R(0)); gdTxy.assign(piece_xy, R(0));
        gdCyaw.assign((size_t)6 * piece_yaw, R(0)); gdTyaw.assign(piece_yaw, R(0));
        Sample S;
        int equal_idx = 0, non_equal_idx = 0, constrain_idx = 0;
        R base_time = 0.0;
        for (int i = 0; i < piece_xy; i++) {
            R step = pos_minco.T1[i] / R(int_K);
            R s1 = 0.0;
            for (int j = 0; j <= int_K; j++) {
                R alpha = R(1.0) / R(int_K) * R(j);
                R grad_p[2] = {0, 0}, grad_v[2] = {0, 0}, grad_a[2] = {0, 0}, grad_se2[3] = {0, 0, 0};
                R grad_yaw = 0, grad_dyaw = 0, grad_d2yaw = 0, grad_vx2 = 0, grad_wz = 0, grad_ax = 0, grad_ay = 0;
                R aug_grad = 0;
                sample(i, s1, base_time, S);
                const R inv_cos_vphix = S.tv[0], inv_cos_vphiy = S.tv[2], cos_xi = S.tv[4], inv_cos_xi = S.tv[5], sigma = S.tv[6];
                const R *g_icvx = S.tg[0], *g_spx = S.tg[1], *g_icvy = S.tg[2], *g_spy = S.tg[3], *g_cxi = S.tg[4],
                        *g_icxi = S.tg[5], *g_sig = S.tg[6];
                const R vx = S.vx, wz = S.wz, ax = S.ax, ay = S.ay, curv_snorm = S.curv_snorm;

                /* user-defined cost: surface variation (819-827) */
                R omega;
                if (j == 0 || j == int_K) omega = R(0.5) * rho_ter * step * scale_fx;
                else omega = rho_ter * step * scale_fx;
                R user_cost = omega * sigma * sigma;
                cost += user_cost;
                for (int k = 0; k < 3; k++) grad_se2[k] += omega * g_sig[k] * sigma * R(2.0);
                gdTxy[i] += user_cost / R(int_K); /* Q3 */

                /* non-holonomic (829-838) */
                R nonh_lambda = lambda[equal_idx];
                R nhy[2] = {S.syaw, -S.cyaw};
                hx[equal_idx] = (S.vel[0] * nhy[0] + S.vel[1] * nhy[1]) * scale_cx[constrain_idx];
                cost += getAugmentedCost(hx[equal_idx], nonh_lambda);
                R nonh_grad = getAugmentedGrad(hx[equal_idx], nonh_lambda) * scale_cx[constrain_idx];
                grad_v[0] += nonh_grad * nhy[0]; grad_v[1] += nonh_grad * nhy[1];
                grad_yaw += nonh_grad * (S.vel[0] * S.xb[0] + S.vel[1] * S.xb[1]);
                equal_idx++; constrain_idx++;

                /* longitude velocity (840-854) */
                R v_mu = mu[non_equal_idx];
                gx[non_equal_idx] = (vx * vx - max_vel * max_vel) * scale_cx[constrain_idx];
                if (rho * gx[non_equal_idx] + v_mu > 0) {
                    cost += getAugmentedCost(gx[non_equal_idx], v_mu);
                    aug_grad = getAugmentedGrad(gx[non_equal_idx], v_mu) * scale_cx[constrain_idx];
                    grad_vx2 += aug_grad;
                } else cost += R(-0.5) * v_mu * v_mu / rho;
                non_equal_idx++; constrain_idx++;

                /* longitude acceleration (856-870) */
                R lona_mu = mu[non_equal_idx];
                gx[non_equal_idx] = (ax * ax - max_acc_lon * max_acc_lon) * scale_cx[constrain_idx];
                if (rho * gx[non_equal_idx] + lona_mu > 0) {
                    cost += getAugmentedCost(gx[non_equal_idx], lona_mu);
                    aug_grad = getAugmentedGrad(gx[non_equal_idx], lona_mu) * scale_cx[constrain_idx];
                    grad_ax += aug_grad * R(2.0) * ax;
                } else cost += R(-0.5) * lona_mu * lona_mu / rho;
                non_equal_idx++; constrain_idx++;

                /* latitude acceleration (872-886) */
                R lata_mu = mu[non_equal_idx];
                gx[non_equal_idx] = (ay * ay - max_acc_lat * max_acc_lat) * scale_cx[constrain_idx];
                if (rho * gx[non_equal_idx] + lata_mu > 0) {
                    cost += getAugmentedCost(gx[non_equal_idx], lata_mu);
                    aug_grad = getAugmentedGrad(gx[non_equal_idx], lata_mu) * scale_cx[constrain_idx];
                    grad_ay += aug_grad * R(2.0) * ay;
                } else cost += R(-0.5) * lata_mu * lata_mu / rho;
                non_equal_idx++; constrain_idx++;

                /* curvature (888-910), Q6 */
                R curv_mu = mu[non_equal_idx];
                if (use_scaling) gx[non_equal_idx] = (curv_snorm - max_kap * max_kap) * scale_cx[constrain_idx];
                else gx[non_equal_idx] = (curv_snorm - max_kap * max_kap) * R(cur_scale);
                if (rho * gx[non_equal_idx] + curv_mu > 0) {
                    R denominator = R(1.0) / (vx * vx + R(delta_sigl));
                    cost += getAugmentedCost(gx[non_equal_idx], curv_mu);
                    if (use_scaling) aug_grad = getAugmentedGrad(gx[non_equal_idx], curv_mu) * scale_cx[constrain_idx];
                    else aug_grad = getAugmentedGrad(gx[non_equal_idx], curv_mu) * R(cur_scale);
                    grad_wz += aug_grad * denominator * R(2.0) * wz;
                    grad_vx2 -= aug_grad * curv_snorm * denominator;
                } else cost += R(-0.5) * curv_mu * curv_mu / rho;
                non_equal_idx++; constrain_idx++;

                /* attitude (912-925) */
                R att_mu = mu[non_equal_idx];
                gx[non_equal_idx] = (min_cxi - cos_xi) * scale_cx[constrain_idx];
                if (rho * gx[non_equal_idx] + att_mu > 0) {
                    cost += getAugmentedCost(gx[non_equal_idx], att_mu);
                    R ag = getAugmentedGrad(gx[non_equal_idx], att_mu);
                    for (int k = 0; k < 3; k++) grad_se2[k] -= ag * g_cxi[k] * scale_cx[constrain_idx];
                } else cost += R(-0.5) * att_mu * att_mu / rho;
                non_equal_idx++; constrain_idx++;

                /* surface variation (927-946), Q6 */
                R sig_mu = mu[non_equal_idx];
                if (use_scaling) gx[non_equal_idx] = (sigma - max_sig) * scale_cx[constrain_idx];
                else gx[non_equal_idx] = (sigma - max_sig) * R(sig_scale);
                if (rho * gx[non_equal_idx] + sig_mu > 0) {
                    cost += getAugmentedCost(gx[non_equal_idx], sig_mu);
                    R ag = getAugmentedGrad(gx[non_equal_idx], sig_mu);
                    if (use_scaling) for (int k = 0; k < 3; k++) grad_se2[k] += ag * g_sig[k] * scale_cx[constrain_idx];
                    else for (int k = 0; k < 3; k++) grad_se2[k] += ag * g_sig[k] * R(sig_scale);
                } else cost += R(-0.5) * sig_mu * sig_mu / rho;
                non_equal_idx++; constrain_idx++;

                /* process with vx, wz, ax (948-964) */
                for (int d = 0; d < 2; d++) grad_v[d] += grad_vx2 * inv_cos_vphix * inv_cos_vphix * R(2.0) * S.vel[d];
                for (int k = 0; k < 3; k++) grad_se2[k] += grad_vx2 * S.v_norm * S.v_norm * R(2.0) * inv_cos_vphix * g_icvx[k];
                grad_dyaw += grad_wz * inv_cos_xi;
                for (int k = 0; k < 3; k++) grad_se2[k] += grad_wz * S.dyaw * g_icxi[k];
                for (int d = 0; d < 2; d++) grad_a[d] += grad_ax * inv_cos_vphix * S.xb[d];
                grad_yaw += grad_ax * inv_cos_vphix * S.lat_acc;
                for (int k = 0; k < 3; k++) grad_se2[k] += grad_ax * (gravity * g_spx[k] + g_icvx[k] * S.lon_acc);
                for (int d = 0; d < 2; d++) grad_a[d] += grad_ay * inv_cos_vphiy * S.yb[d];
                grad_yaw -= grad_ay * inv_cos_vphiy * S.lon_acc;
                for (int k = 0; k < 3; k++) grad_se2[k] += grad_ay * (gravity * g_spy[k] + g_icvy[k] * S.lat_acc);
                grad_p[0] += grad_se2[0]; grad_p[1] += grad_se2[1];
                grad_yaw += grad_se2[2];

                /* add all grad into C,T (966-985) */
                for (int d = 0; d < 2; d++)
                    for (int k = 0; k < 6; k++)
                        gdCxy[6 * i + k + (size_t)d * NX] +=
                            (S.beta0_xy[k] * grad_p[d] + S.beta1_xy[k] * grad_v[d] + S.beta2_xy[k] * grad_a[d]);
                gdTxy[i] += ((grad_p[0] * S.vel[0] + grad_p[1] * S.vel[1]) + (grad_v[0] * S.acc[0] + grad_v[1] * S.acc[1]) +
                             (grad_a[0] * S.jer[0] + grad_a[1] * S.jer[1])) * alpha;
                for (int k = 0; k < 6; k++)
                    gdCyaw[6 * S.yaw_idx + k] += (S.beta0_yaw[k] * grad_yaw + S.beta1_yaw[k] * grad_dyaw + S.beta2_yaw[k] * grad_d2yaw);
                gdTyaw[S.yaw_idx] += -(grad_yaw * S.dyaw + grad_dyaw * S.d2yaw) * R(S.yaw_idx);
                gdTxy[i] += (grad_yaw * S.dyaw + grad_dyaw * S.d2yaw) * (alpha + R(i));

                s1 += step;
            }
            base_time += pos_minco.T1[i];
        }
    }

    /* innerCallback  alm_traj_opt.cpp:280-347 */
    R evaluate(const std::vector<R> &x, std::vector<R> &grad)
    {
        n_evals++;
        auto t0 = clk::now();
        const R tau = x[0];
        generate(x.data());
        std::vector<R> gdCxy_jerk, gdTxy_jerk, gdCyaw_jerk, gdTyaw_jerk;
        pos_minco.calJerkGradCT(gdCxy_jerk, gdTxy_jerk);
        yaw_minco.calJerkGradCT(gdCyaw_jerk, gdTyaw_jerk);
        R jerk_cost = (pos_minco.getTrajJerkCost() + yaw_minco.getTrajJerkCost()) * scale_fx;
        if (use_scaling) jerk_cost *= R(scale_trick_jerk);
        auto t1 = clk::now();
        R constrain_cost = 0.0;
        std::vector<R> &gdCxy_c = last_gdCxy, &gdTxy_c = last_gdTxy, &gdCyaw_c = last_gdCyaw, &gdTyaw_c = last_gdTyaw;
        calConstrainCostGrad(constrain_cost, gdCxy_c, gdTxy_c, gdCyaw_c, gdTyaw_c);
        auto t2 = clk::now();
        if (use_scaling) {
            for (auto &v : gdCxy_jerk) v *= R(scale_trick_jerk);
            for (auto &v : gdTxy_jerk) v *= R(scale_trick_jerk);
            for (auto &v : gdCyaw_jerk) v *= R(scale_trick_jerk);
            for (auto &v : gdTyaw_jerk) v *= R(scale_trick_jerk);
        }
        std::vector<R> gdCxy(gdCxy_jerk.size()), gdTxy(gdTxy_jerk.size()), gdCyaw(gdCyaw_jerk.size()), gdTyaw(gdTyaw_jerk.size());
        for (size_t q = 0; q < gdCxy.size(); q++) gdCxy[q] = gdCxy_jerk[q] * scale_fx + gdCxy_c[q];
        for (size_t q = 0; q < gdTxy.size(); q++) gdTxy[q] = gdTxy_jerk[q] * scale_fx + gdTxy_c[q];
        for (size_t q = 0; q < gdCyaw.size(); q++) gdCyaw[q] = gdCyaw_jerk[q] * scale_fx + gdCyaw_c[q];
        for (size_t q = 0; q < gdTyaw.size(); q++) gdTyaw[q] = gdTyaw_jerk[q] * scale_fx + gdTyaw_c[q];
        std::vector<R> gradPxy, gradPyaw, adj;
        pos_minco.calGradCTtoQT(gdCxy, gdTxy, gradPxy, adj);
        yaw_minco.calGradCTtoQT(gdCyaw, gdTyaw, gradPyaw, adj);
        std::copy(gradPxy.begin(), gradPxy.end(), grad.begin() + dim_T);
        std::copy(gradPyaw.begin(), gradPyaw.end(), grad.begin() + dim_T + 2 * (piece_xy - 1));
        R tau_cost = rho_T * expC2(tau) * scale_fx;
        R sx = 0, sy = 0;
        for (auto v : gdTxy) sx += v;
        for (auto v : gdTyaw) sy += v;
        R grad_Tsum = rho_T * scale_fx + sx / R(piece_xy) + sy / R(piece_yaw);
        grad[0] = grad_Tsum * getTtoTauGrad(tau);
        auto t3 = clk::now();
        t_minco += secs(t0, t1); t_penalty += secs(t1, t2); t_adjoint += secs(t2, t3);
        last_parts[0] = jerk_cost; last_parts[1] = constrain_cost; last_parts[2] = tau_cost;
        return jerk_cost + constrain_cost + tau_cost;
    }

    /* initScaling  alm_traj_opt.cpp:349-661 */
    void initScaling(const std::vector<R> &x0)
    {
        auto t0 = clk::now();
        const int NX = 6 * piece_xy, NY = 6 * piece_yaw;
        const R tau = x0[0];
        generate(x0.data());
        std::vector<R> gdCxy_fx, gdTxy_fx, gdCyaw_fx, gdTyaw_fx;
        pos_minco.calJerkGradCT(gdCxy_fx, gdTxy_fx);
        yaw_minco.calJerkGradCT(gdCyaw_fx, gdTyaw_fx);
        const int nc = equal_num + non_equal_num;
        /* one (gdCxy,gdTxy,gdCyaw,gdTyaw) set per constraint; only one xy block and one yaw block of
         * each is non-zero, but the adjoint solve below is run on the full vectors as in the reference */
        std::vector<R> gdCxy((size_t)NX * 2), gdTxy(piece_xy), gdCyaw(NY), gdTyaw(piece_yaw), gdP, adj;
        Sample S;
        int constrain_idx = 0;
        R base_time = 0.0;
        const R dTdtau = getTtoTauGrad(tau);
        auto finish = [&](int ci) { /* alm_traj_opt.cpp:637-647, 654-660 */
            pos_minco.calGradCTtoQT(gdCxy, gdTxy, gdP, adj);
            R m1 = vabsmax(gdP.data(), (int)gdP.size());
            std::vector<R> gdPy;
            yaw_minco.calGradCTtoQT(gdCyaw, gdTyaw, gdPy, adj);
            R m2 = vabsmax(gdPy.data(), (int)gdPy.size());
            R sx = 0, sy = 0;
            for (auto v : gdTxy) sx += v;
            for (auto v : gdTyaw) sy += v;
            R gdTau = (sx / R(piece_xy) + sy / R(piece_yaw)) * dTdtau;
            scale_cx[ci] = R(1.0) / std::max(R(1.0), std::max(std::max(m1, m2), std::fabs(gdTau)));
        };
        auto clear = [&]() {
            std::fill(gdCxy.begin(), gdCxy.end(), R(0)); std::fill(gdTxy.begin(), gdTxy.end(), R(0));
            std::fill(gdCyaw.begin(), gdCyaw.end(), R(0)); std::fill(gdTyaw.begin(), gdTyaw.end(), R(0));
        };
        /* scatter helper: gdC += beta0*gp + beta1*gv + beta2*ga etc. */
        for (int i = 0; i < piece_xy; i++) {
            R step = pos_minco.T1[i] / R(int_K);
            R s1 = 0.0;
            for (int j = 0; j <= int_K; j++) {
                R alpha = R(1.0) / R(int_K) * R(j);
                sample(i, s1, base_time, S);
                const int yi = S.yaw_idx;
                const R inv_cos_vphix = S.tv[0], inv_cos_vphiy = S.tv[2], inv_cos_xi = S.tv[5], sigma = S.tv[6];
                const R *g_icvx = S.tg[0], *g_spx = S.tg[1], *g_icvy = S.tg[2], *g_spy = S.tg[3], *g_cxi = S.tg[4],
                        *g_icxi = S.tg[5], *g_sig = S.tg[6];
                R grad_p[2], grad_v[2], grad_a[2], grad_se2[3], grad_yaw, grad_dyaw;

                /* user-defined cost -> f gradient (507-519) */
                R omega = (j == 0 || j == int_K) ? R(0.5) * rho_ter * step : rho_ter * step;
                R user_cost = omega * sigma * sigma;
                for (int k = 0; k < 3; k++) grad_se2[k] = omega * g_sig[k] * sigma * R(2.0);
                gdTxy_fx[i] += user_cost / R(int_K);
                for (int d = 0; d < 2; d++)
                    for (int k = 0; k < 6; k++) gdCxy_fx[6 * i + k + (size_t)d * NX] += S.beta0_xy[k] * grad_se2[d];
                gdTxy_fx[i] += (grad_se2[0] * S.vel[0] + grad_se2[1] * S.vel[1]) * alpha;
                for (int k = 0; k < 6; k++) gdCyaw_fx[6 * yi + k] += (S.beta0_yaw[k] * grad_se2[2]);
                gdTyaw_fx[yi] += -(grad_se2[2] * S.dyaw) * R(yi);
                gdTxy_fx[i] += (grad_se2[2] * S.dyaw) * (alpha + R(i));

                auto yaw_part = [&](R gy, R gdy, bool with_dyaw) {
                    if (with_dyaw) {
                        for (int k = 0; k < 6; k++) gdCyaw[6 * yi + k] += (S.beta0_yaw[k] * gy + S.beta1_yaw[k] * gdy);
                        gdTyaw[yi] += -(gy * S.dyaw + gdy * S.d2yaw) * R(yi);
                        gdTxy[i] += (gy * S.dyaw + gdy * S.d2yaw) * (alpha + R(i));
                    } else {
                        for (int k = 0; k < 6; k++) gdCyaw[6 * yi + k] += S.beta0_yaw[k] * gy;
                        gdTyaw[yi] += -(gy * S.dyaw) * R(yi);
                        gdTxy[i] += (gy * S.dyaw) * (alpha + R(i));
                    }
                };

                /* non-holonomic (521-529) */
                clear();
                grad_v[0] = S.syaw; grad_v[1] = -S.cyaw;
                grad_yaw = S.vel[0] * S.xb[0] + S.vel[1] * S.xb[1];
                for (int d = 0; d < 2; d++)
                    for (int k = 0; k < 6; k++) gdCxy[6 * i + k + (size_t)d * NX] += S.beta1_xy[k] * grad_v[d];
                gdTxy[i] += (grad_v[0] * S.acc[0] + grad_v[1] * S.acc[1]) * alpha;
                yaw_part(grad_yaw, 0, false);
                finish(constrain_idx++);

                /* longitude velocity (531-544) */
                clear();
                R grad_vx2 = 1.0;
                for (int d = 0; d < 2; d++) grad_v[d] = grad_vx2 * inv_cos_vphix * inv_cos_vphix * R(2.0) * S.vel[d];
                for (int k = 0; k < 3; k++) grad_se2[k] = grad_vx2 * S.v_norm * S.v_norm * R(2.0) * inv_cos_vphix * g_icvx[k];
                grad_p[0] = grad_se2[0]; grad_p[1] = grad_se2[1]; grad_yaw = grad_se2[2];
                for (int d = 0; d < 2; d++)
                    for (int k = 0; k < 6; k++)
                        gdCxy[6 * i + k + (size_t)d * NX] += (S.beta0_xy[k] * grad_p[d] + S.beta1_xy[k] * grad_v[d]);
                gdTxy[i] += ((grad_p[0] * S.vel[0] + grad_p[1] * S.vel[1]) + (grad_v[0] * S.acc[0] + grad_v[1] * S.acc[1])) * alpha;
                yaw_part(grad_yaw, 0, false);
                finish(constrain_idx++);

                /* longitude acceleration (546-560) */
                clear();
                R grad_ax = R(2.0) * S.ax;
                for (int d = 0; d < 2; d++) grad_a[d] = grad_ax * inv_cos_vphix * S.xb[d];
                grad_yaw = grad_ax * inv_cos_vphix * S.lat_acc;
                for (int k = 0; k < 3; k++) grad_se2[k] = grad_ax * (gravity * g_spx[k] + g_icvx[k] * S.lon_acc);
                grad_p[0] = grad_se2[0]; grad_p[1] = grad_se2[1]; grad_yaw += grad_se2[2];
                for (int d = 0; d < 2; d++)
                    for (int k = 0; k < 6; k++)
                        gdCxy[6 * i + k + (size_t)d * NX] += (S.beta0_xy[k] * grad_p[d] + S.beta2_xy[k] * grad_a[d]);
                gdTxy[i] += ((grad_p[0] * S.vel[0] + grad_p[1] * S.vel[1]) + (grad_a[0] * S.jer[0] + grad_a[1] * S.jer[1])) * alpha;
                yaw_part(grad_yaw, 0, false);
                finish(constrain_idx++);

                /* latitude acceleration (562-576) */
                clear();
                R grad_ay = R(2.0) * S.ay;
                for (int d = 0; d < 2; d++) grad_a[d] = grad_ay * inv_cos_vphiy * S.yb[d];
                grad_yaw = -grad_ay * inv_cos_vphiy * S.lon_acc;
                for (int k = 0; k < 3; k++) grad_se2[k] = grad_ay * (gravity * g_spy[k] + g_icvy[k] * S.lat_acc);
                grad_p[0] = grad_se2[0]; grad_p[1] = grad_se2[1]; grad_yaw += grad_se2[2];
                for (int d = 0; d < 2; d++)
                    for (int k = 0; k < 6; k++)
                        gdCxy[6 * i + k + (size_t)d * NX] += (S.beta0_xy[k] * grad_p[d] + S.beta2_xy[k] * grad_a[d]);
                gdTxy[i] += ((grad_p[0] * S.vel[0] + grad_p[1] * S.vel[1]) + (grad_a[0] * S.jer[0] + grad_a[1] * S.jer[1])) * alpha;
                yaw_part(grad_yaw, 0, false);
                finish(constrain_idx++);

                /* curvature (578-598) */
                clear();
                R denominator = R(1.0) / (S.vx * S.vx + R(delta_sigl));
                R grad_wz = denominator * R(2.0) * S.wz;
                grad_vx2 = -S.curv_snorm * denominator;
                grad_dyaw = grad_wz * inv_cos_xi;
                for (int k = 0; k < 3; k++) grad_se2[k] = grad_wz * S.dyaw * g_icxi[k];
                for (int d = 0; d < 2; d++) grad_v[d] = grad_vx2 * inv_cos_vphix * inv_cos_vphix * R(2.0) * S.vel[d];
                for (int k = 0; k < 3; k++) grad_se2[k] += grad_vx2 * S.v_norm * S.v_norm * R(2.0) * inv_cos_vphix * g_icvx[k];
                grad_p[0] = grad_se2[0]; grad_p[1] = grad_se2[1]; grad_yaw = grad_se2[2];
                for (int d = 0; d < 2; d++)
                    for (int k = 0; k < 6; k++)
                        gdCxy[6 * i + k + (size_t)d * NX] += (S.beta0_xy[k] * grad_p[d] + S.beta1_xy[k] * grad_v[d]);
                gdTxy[i] += ((grad_p[0] * S.vel[0] + grad_p[1] * S.vel[1]) + (grad_v[0] * S.acc[0] + grad_v[1] * S.acc[1])) * alpha;
                yaw_part(grad_yaw, grad_dyaw, true);
                finish(constrain_idx++);

                /* attitude (600-609) */
                clear();
                for (int k = 0; k < 3; k++) grad_se2[k] = -g_cxi[k];
                grad_p[0] = grad_se2[0]; grad_p[1] = grad_se2[1]; grad_yaw = grad_se2[2];
                for (int d = 0; d < 2; d++)
                    for (int k = 0; k < 6; k++) gdCxy[6 * i + k + (size_t)d * NX] += (S.beta0_xy[k] * grad_p[d]);
                gdTxy[i] += (grad_p[0] * S.vel[0] + grad_p[1] * S.vel[1]) * alpha;
                yaw_part(grad_yaw, 0, false);
                finish(constrain_idx++);

                /* surface variation (611-620) */
                clear();
                for (int k = 0; k < 3; k++) grad_se2[k] = g_sig[k];
                grad_p[0] = grad_se2[0]; grad_p[1] = grad_se2[1]; grad_yaw = grad_se2[2];
                for (int d = 0; d < 2; d++)
                    for (int k = 0; k < 6; k++) gdCxy[6 * i + k + (size_t)d * NX] += (S.beta0_xy[k] * grad_p[d]);
                gdTxy[i] += (grad_p[0] * S.vel[0] + grad_p[1] * S.vel[1]) * alpha;
                yaw_part(grad_yaw, 0, false);
                finish(constrain_idx++);

                s1 += step;
            }
            base_time += pos_minco.T1[i];
        }
        (void)nc;
        /* f gradient (627-636, 649-652), Q7: no scale_trick_jerk here */
        std::vector<R> gdPxy_fx, gdPyaw_fx;
        pos_minco.calGradCTtoQT(gdCxy_fx, gdTxy_fx, gdPxy_fx, adj);
        yaw_minco.calGradCTtoQT(gdCyaw_fx, gdTyaw_fx, gdPyaw_fx, adj);
        R sx = 0, sy = 0;
        for (auto v : gdTxy_fx) sx += v;
        for (auto v : gdTyaw_fx) sy += v;
        R grad_Tsum_fx = rho_T + sx / R(piece_xy) + sy / R(piece_yaw);
        R gdTau_fx = grad_Tsum_fx * dTdtau;
        scale_fx = R(1.0) / std::max(R(1.0), std::max(std::max(vabsmax(gdPxy_fx.data(), (int)gdPxy_fx.size()),
                                                              vabsmax(gdPyaw_fx.data(), (int)gdPyaw_fx.size())),
                                                     std::fabs(gdTau_fx)));
        t_scaling += secs(t0, clk::now());
    }

    void updateDualVars() /* alm_traj_opt.h:132-138 */
    {
        for (int i = 0; i < equal_num; i++) lambda[i] += rho * hx[i];
        for (int i = 0; i < non_equal_num; i++) mu[i] = std::max(mu[i] + rho * gx[i], R(0.0));
        rho = std::min((1 + gamma) * rho, beta);
    }
    bool judgeConvergence(R &rh, R &rg) /* alm_traj_opt.h:140-151 (uses the UPDATED mu, rho) */
    {
        rh = vabsmax(hx.data(), equal_num);
        rg = 0;
        for (int i = 0; i < non_equal_num; i++) rg = std::max(rg, std::fabs(std::max(gx[i], -mu[i] / rho)));
        return std::max(rh, rg) < epsilon_con;
    }
};

constexpr int RET_STOPPED = 3;   /* UALM_RET_STOPPED (include/ualm.h) */

/* stop(n_evals, site) is the stop test of the CUDA paths (an evaluation budget, a cancel), called once per test in execution order:
 * site 0 where earlyExit tests k > 1000 (L-BFGS then returns CANCELED), site 1 after judgeConvergence when the inner solve was not
 * ended by a stop and the problem has not converged.  orc_solve / orc_solve_f32 pass a stop that never holds. */
template <class R, class Stop>
static int solve_impl(const orc_params_t *p, const orc_map_t *map, const orc_problem_t *prob, Stop stop, orc_result_t *res,
                      double *c_xy_out, double *c_yaw_out, double *x_out, double *lambda_out, double *mu_out,
                      double *scale_cx_out)
{
    auto T0 = clk::now();
    MapQ<R> mq(*map);
    ALM<R> alm(*p, &mq); /* Q2: fresh rho per problem */
    alm.setup(*prob);
    const int n = alm.nvar();
    std::vector<R> x(n);
    /* alm_traj_opt.cpp:205-216 */
    x[0] = logC2((R)prob->total_time);
    for (int i = 0; i < 2 * (alm.piece_xy - 1); i++) x[1 + i] = (R)prob->inner_xy[i];
    for (int i = 0; i < alm.piece_yaw - 1; i++) x[1 + 2 * (alm.piece_xy - 1) + i] = (R)prob->inner_yaw[i];

    LbfgsParam<R> lp;
    lp.mem_size = alm.mem_size; lp.past = alm.past; lp.g_epsilon = alm.g_epsilon; lp.min_step = alm.min_step;
    lp.delta = alm.delta; lp.max_iterations = (int)alm.inner_max_iter;
    R inner_cost = 0;
    int ret_code = 0, iter = 0, last = 0;
    LbfgsStats st;
    double t_lbfgs_all = 0;

    if (alm.use_scaling) alm.initScaling(x);

    auto eval = [&](const std::vector<R> &xx, std::vector<R> &gg) { return alm.evaluate(xx, gg); };
    bool fired = false;   /* the stop ended the inner solve that just returned */
    auto progress = [&](int k) { fired = stop(alm.n_evals, 0); return k > 1e3 || fired; }; /* earlyExit alm_traj_opt.cpp:1016 */
    R rh = 0, rg = 0;
    /* Exit order: a stop that ended the inner solve just finished -> RET_STOPPED even when judgeConvergence passes; else
     * converged -> 0; else the stop holds now -> RET_STOPPED; else ++iter > max_iter -> 2 */
    while (true) {
        fired = false;
        auto a = clk::now();
        int result = lbfgs_optimize(x, inner_cost, eval, progress, lp, st);
        t_lbfgs_all += secs(a, clk::now());
        last = result;
        if (result == LBFGS_CONVERGENCE || result == LBFGS_CANCELED || result == LBFGS_STOP ||
            result == LBFGSERR_MAXIMUMITERATION) {
        } else if (result == LBFGSERR_MAXIMUMLINESEARCH) {
        } else { ret_code = 1; break; }
        alm.updateDualVars();
        const bool converged = alm.judgeConvergence(rh, rg);
        if (fired) { ret_code = RET_STOPPED; break; }
        if (converged) break;
        if (stop(alm.n_evals, 1)) { ret_code = RET_STOPPED; break; }
        if (++iter > alm.max_iter) { ret_code = 2; break; }
    }
    res->ret_code = ret_code; res->outer_iters = iter; res->n_evals = alm.n_evals; res->n_lbfgs_iters = st.iters;
    res->last_lbfgs_ret = last; res->max_bound = st.max_bound; res->inner_cost = (double)inner_cost;
    res->jerk_cost = (double)(alm.pos_minco.getTrajJerkCost() + alm.yaw_minco.getTrajJerkCost());
    R tt = 0; for (auto t : alm.pos_minco.T1) tt += t;
    res->total_T = (double)tt;
    res->res_h = (double)rh; res->res_g = (double)rg; res->scale_fx = (double)alm.scale_fx; res->rho_final = (double)alm.rho;
    res->t_minco = alm.t_minco; res->t_penalty = alm.t_penalty; res->t_adjoint = alm.t_adjoint;
    res->t_scaling = alm.t_scaling;
    res->t_lbfgs = t_lbfgs_all - alm.t_minco - alm.t_penalty - alm.t_adjoint;
    if (c_xy_out) for (size_t i = 0; i < alm.pos_minco.c.size(); i++) c_xy_out[i] = (double)alm.pos_minco.c[i];
    if (c_yaw_out) for (size_t i = 0; i < alm.yaw_minco.c.size(); i++) c_yaw_out[i] = (double)alm.yaw_minco.c[i];
    if (x_out) for (int i = 0; i < n; i++) x_out[i] = (double)x[i];
    if (lambda_out) for (size_t i = 0; i < alm.lambda.size(); i++) lambda_out[i] = (double)alm.lambda[i];
    if (mu_out) for (size_t i = 0; i < alm.mu.size(); i++) mu_out[i] = (double)alm.mu[i];
    if (scale_cx_out) for (size_t i = 0; i < alm.scale_cx.size(); i++) scale_cx_out[i] = (double)alm.scale_cx[i];
    res->t_total = secs(T0, clk::now());
    return ret_code;
}

inline bool never_stop(int, int) { return false; }

} // namespace

extern "C" {

int orc_solve(const orc_params_t *p, const orc_map_t *map, const orc_problem_t *prob, orc_result_t *res,
              double *c_xy_out, double *c_yaw_out, double *x_out, double *lambda_out, double *mu_out,
              double *scale_cx_out)
{
    return solve_impl<double>(p, map, prob, never_stop, res, c_xy_out, c_yaw_out, x_out, lambda_out, mu_out, scale_cx_out);
}

int orc_solve_f32(const orc_params_t *p, const orc_map_t *map, const orc_problem_t *prob, orc_result_t *res,
                  double *c_xy_out, double *c_yaw_out, double *x_out)
{
    return solve_impl<float>(p, map, prob, never_stop, res, c_xy_out, c_yaw_out, x_out, nullptr, nullptr, nullptr);
}

int orc_eval(const orc_params_t *p, const orc_map_t *map, const orc_problem_t *prob, const double *x,
             const double *lambda, const double *mu, const double *scale_cx, double scale_fx, double rho, double *f,
             double *grad, double *hx, double *gx, double *parts, double *c_xy_out, double *c_yaw_out, double *gdCxy,
             double *gdTxy, double *gdCyaw, double *gdTyaw)
{
    MapQ<double> mq(*map);
    ALM<double> alm(*p, &mq);
    alm.setup(*prob);
    const int n = alm.nvar();
    if (lambda) alm.lambda.assign(lambda, lambda + alm.equal_num);
    if (mu) alm.mu.assign(mu, mu + alm.non_equal_num);
    if (scale_cx) alm.scale_cx.assign(scale_cx, scale_cx + alm.equal_num + alm.non_equal_num);
    alm.scale_fx = scale_fx;
    alm.rho = rho;
    std::vector<double> xx(x, x + n), gg(n);
    *f = alm.evaluate(xx, gg);
    std::copy(gg.begin(), gg.end(), grad);
    if (hx) std::copy(alm.hx.begin(), alm.hx.end(), hx);
    if (gx) std::copy(alm.gx.begin(), alm.gx.end(), gx);
    if (parts) for (int i = 0; i < 3; i++) parts[i] = alm.last_parts[i];
    if (c_xy_out) std::copy(alm.pos_minco.c.begin(), alm.pos_minco.c.end(), c_xy_out);
    if (c_yaw_out) std::copy(alm.yaw_minco.c.begin(), alm.yaw_minco.c.end(), c_yaw_out);
    if (gdCxy) std::copy(alm.last_gdCxy.begin(), alm.last_gdCxy.end(), gdCxy);
    if (gdTxy) std::copy(alm.last_gdTxy.begin(), alm.last_gdTxy.end(), gdTxy);
    if (gdCyaw) std::copy(alm.last_gdCyaw.begin(), alm.last_gdCyaw.end(), gdCyaw);
    if (gdTyaw) std::copy(alm.last_gdTyaw.begin(), alm.last_gdTyaw.end(), gdTyaw);
    return 0;
}

int orc_init_scaling(const orc_params_t *p, const orc_map_t *map, const orc_problem_t *prob, const double *x0,
                     double *scale_fx, double *scale_cx)
{
    MapQ<double> mq(*map);
    ALM<double> alm(*p, &mq);
    alm.setup(*prob);
    std::vector<double> xx(x0, x0 + alm.nvar());
    alm.initScaling(xx);
    *scale_fx = alm.scale_fx;
    std::copy(alm.scale_cx.begin(), alm.scale_cx.end(), scale_cx);
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * Post-solve scan: PolyTrajectory::locatePieceIdx / Piece::getValue, getDotValue, getDDotValue (se2traj.hpp:343-361, 106-150;
 * the reference stores the coefficients highest power first, so its loops i = order..0 walk this file's c[0], c[1], ...),
 * SE2Trajectory accessors (se2traj.hpp:420-481, 551-561), ALMTrajOpt::getMaxVxAxAyCurAttSig (alm_traj_opt.h:170-229).
 * getTerrainVariables (uneven_map.h:221-256) evaluates the same value expressions as getAllWithGrad (:318-348).
 * ---------------------------------------------------------------------------------------- */
namespace {
struct PieceRef { const double *c; int stride; };   /* c[k * 1 + d * stride]: coefficient k (low -> high) of dimension d */
inline int locate_piece(int P, double dur, double &t) /* se2traj.hpp:343-361, uniform durations */
{
    int idx;
    for (idx = 0; idx < P && t > dur; idx++) t -= dur;
    if (idx == P) { idx--; t += dur; }
    return idx;
}
inline double piece_value(const double *c, double t) /* se2traj.hpp:106-118 */
{
    double v = 0.0, tn = 1.0;
    for (int k = 0; k <= 5; k++) { v += tn * c[k]; tn *= t; }
    return v;
}
inline double piece_dot(const double *c, double t) /* se2traj.hpp:120-134 */
{
    double v = 0.0, tn = 1.0;
    int n = 1;
    for (int k = 1; k <= 5; k++) { v += n * tn * c[k]; tn *= t; n++; }
    return v;
}
inline double piece_ddot(const double *c, double t) /* se2traj.hpp:136-150 */
{
    double v = 0.0, tn = 1.0;
    int m = 1, n = 2;
    for (int k = 2; k <= 5; k++) { v += m * n * tn * c[k]; tn *= t; m++; n++; }
    return v;
}
/* PolyTrajectory::getTotalDuration (se2traj.hpp:291-300) of the xy and the yaw part, each summed piece by piece: an SE2 trajectory
 * lasts the smaller (se2traj.hpp:415-418) */
inline double traj_duration(int N, int M, double T_xy, double T_yaw)
{
    double tot_xy = 0.0, tot_yaw = 0.0;
    for (int i = 0; i < N; i++) tot_xy += T_xy;
    for (int i = 0; i < M; i++) tot_yaw += T_yaw;
    return std::min(tot_xy, tot_yaw);
}
/* The pieces at time t and the position, velocity and acceleration of the xy and the yaw part there (PolyTrajectory::getValue /
 * getVel / getAcc, se2traj.hpp:363-391) */
struct SE2State { int ip, iy; double x, y, yaw, vx, vy, dyaw, ax, ay, ddyaw; };
inline SE2State se2_eval(int N, int M, const double *c_xy, const double *c_yaw, double T_xy, double T_yaw, double t)
{
    double tl = t, ty = t;
    const int ip = locate_piece(N, T_xy, tl), iy = locate_piece(M, T_yaw, ty);
    const double *cx = c_xy + 6 * ip, *cy = c_xy + 6 * N + 6 * ip, *cw = c_yaw + 6 * iy;
    return {ip, iy, piece_value(cx, tl), piece_value(cy, tl), piece_value(cw, ty), piece_dot(cx, tl), piece_dot(cy, tl),
            piece_dot(cw, ty), piece_ddot(cx, tl), piece_ddot(cy, tl), piece_ddot(cw, ty)};
}
/* One sample of the post-solve scan at time t: vx, ax, ay, cur, att and sig of getMaxVxAxAyCurAttSig and the term getNonHolError
 * sums */
struct ScanSample { double vx, ax, ay, cur, att, sig, term; };
inline ScanSample scan_sample(const MapQ<double> &mq, double gravity, int N, int M, const double *c_xy, const double *c_yaw,
                              double T_xy, double T_yaw, double t)
{
    const SE2State e = se2_eval(N, M, c_xy, c_yaw, T_xy, T_yaw, t);
    double se2[3] = {e.x, e.y, e.yaw};
    while (se2[2] < -M_PI) se2[2] += 2 * M_PI; /* getNormSE2Pos, se2traj.hpp:433-443 */
    while (se2[2] > M_PI) se2[2] -= 2 * M_PI;
    double tv[7], tg[7][3];
    mq.getAllWithGrad(se2, tv, tg);
    const double cy_ = Mth<double>::cos(e.yaw), sy_ = Mth<double>::sin(e.yaw);
    const double vnorm = std::sqrt(e.vx * e.vx + e.vy * e.vy);   /* getVelNorm */
    const double lon = e.ax * cy_ + e.ay * sy_;                  /* getLonAcc */
    const double lat = -e.ax * sy_ + e.ay * cy_;                 /* getLatAcc */
    ScanSample s;
    s.vx = vnorm * tv[0];
    s.ax = lon * tv[0] + gravity * tv[1];
    s.ay = lat * tv[2] + gravity * tv[3];
    const double wz = e.dyaw * tv[5];
    s.cur = wz / std::sqrt(s.vx * s.vx + delta_sigl);
    s.att = -1.0 / tv[5];
    s.sig = tv[6];
    s.term = std::fabs(e.vx * sy_ + e.vy * (-cy_));              /* getNonHolError */
    return s;
}
} // namespace

void orc_feasibility(const orc_map_t *map, double gravity, int N, int M, const double *c_xy, const double *c_yaw, double T_xy,
                     double T_yaw, double dt, double *out)
{
    MapQ<double> mq(*map);
    const double total = traj_duration(N, M, T_xy, T_yaw);
    double max_ax = 0.0, max_ay = 0.0, max_vx = 0.0, max_cur = 0.0, max_att = -1.0, max_sig = 0.0, err = 0.0;
    long count = 0;
    for (double t = 0.0; t < total; t += dt) {
        const ScanSample s = scan_sample(mq, gravity, N, M, c_xy, c_yaw, T_xy, T_yaw, t);
        if (std::fabs(max_ax) < std::fabs(s.ax)) max_ax = s.ax;
        if (std::fabs(max_ay) < std::fabs(s.ay)) max_ay = s.ay;
        if (std::fabs(max_vx) < std::fabs(s.vx)) max_vx = s.vx;
        if (std::fabs(max_cur) < std::fabs(s.cur)) max_cur = s.cur;
        if (max_att < s.att) max_att = s.att;
        if (max_sig < s.sig) max_sig = s.sig;
        err += s.term;
        count++;
    }
    out[0] = max_vx; out[1] = max_ax; out[2] = max_ay; out[3] = max_cur; out[4] = max_att; out[5] = max_sig; out[6] = err;
    out[7] = (double)count;
}

void orc_map_query(const orc_map_t *map, const double pos[3], double *values, double *grads)
{
    MapQ<double> mq(*map);
    double g[7][3];
    mq.getAllWithGrad(pos, values, g);
    for (int i = 0; i < 7; i++) for (int k = 0; k < 3; k++) grads[3 * i + k] = g[i][k];
}

int orc_minco_generate(int Dim, int N, const double *inPs, const double *ts, const double *head, const double *tail,
                       double *c)
{
    MinJerk<double> mj;
    mj.reset(N, Dim);
    mj.generate(inPs, ts, head, tail);
    std::copy(mj.c.begin(), mj.c.end(), c);
    return 0;
}

double orc_minco_jerk(int Dim, int N, const double *c, const double *ts, double *gdC, double *gdT)
{
    MinJerk<double> mj;
    mj.reset(N, Dim);
    for (int i = 0; i < N; i++) {
        mj.T1[i] = ts[i]; mj.T2[i] = mj.T1[i] * mj.T1[i]; mj.T3[i] = mj.T2[i] * mj.T1[i];
        mj.T4[i] = mj.T2[i] * mj.T2[i]; mj.T5[i] = mj.T4[i] * mj.T1[i];
    }
    mj.c.assign(c, c + (size_t)6 * N * Dim);
    std::vector<double> a, b;
    mj.calJerkGradCT(a, b);
    if (gdC) std::copy(a.begin(), a.end(), gdC);
    if (gdT) std::copy(b.begin(), b.end(), gdT);
    return mj.getTrajJerkCost();
}

int orc_minco_grad_ct_to_qt(int Dim, int N, const double *inPs, const double *ts, const double *head,
                            const double *tail, const double *gdC, double *gdT, double *gdP)
{
    MinJerk<double> mj;
    mj.reset(N, Dim);
    mj.generate(inPs, ts, head, tail);
    std::vector<double> gC(gdC, gdC + (size_t)6 * N * Dim), gT(gdT, gdT + N), gP, adj;
    mj.calGradCTtoQT(gC, gT, gP, adj);
    std::copy(gT.begin(), gT.end(), gdT);
    std::copy(gP.begin(), gP.end(), gdP);
    return 0;
}

int orc_lbfgs_rosenbrock(int n, double *x, double *f, int mem_size, double g_epsilon, int past, double delta,
                         int *iters)
{
    std::vector<double> xx(x, x + n);
    auto eval = [&](const std::vector<double> &v, std::vector<double> &g) {
        double fx = 0.0;
        for (int i = 0; i < n; i += 2) {
            double t1 = 1.0 - v[i];
            double t2 = 10.0 * (v[i + 1] - v[i] * v[i]);
            g[i + 1] = 20.0 * t2;
            g[i] = -2.0 * (v[i] * g[i + 1] + t1);
            fx += t1 * t1 + t2 * t2;
        }
        return fx;
    };
    auto progress = [&](int) { return 0; };
    LbfgsParam<double> lp;
    lp.mem_size = mem_size; lp.g_epsilon = g_epsilon; lp.past = past; lp.delta = delta;
    LbfgsStats st;
    double fx = 0;
    int r = lbfgs_optimize(xx, fx, eval, progress, lp, st);
    std::copy(xx.begin(), xx.end(), x);
    *f = fx;
    if (iters) *iters = st.iters;
    return r;
}

double orc_expC2(double tau) { return expC2(tau); }
double orc_logC2(double T) { return logC2(T); }
double orc_dTdtau(double tau) { return getTtoTauGrad(tau); }
}
