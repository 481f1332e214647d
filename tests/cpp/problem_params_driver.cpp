// Drives the per-problem parameter overloads of the C++ ALMTrajOpt mirror (include/ualm_traj_opt.hpp): one environment with the
// run_hill.yaml parameters, every problem with its own row.  optimizeBatch(env, pp); then submitBatch(env, pp) and, while that ticket
// is in flight, checkTrajectories(env, pp) of the optimizeBatch trajectories; then waitBatch; then submitReplan(env, pp) of them from
// t = 0.5 and waitBatch.  Reads the map, the problems and the rows from a binary file written by the test and writes the outputs as raw
// bytes to a second file: records, c_xy, c_yaw of the solve and of the wait, the check's out16, then the replan's built N, M and its
// records, c_xy, c_yaw.
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "ualm_traj_opt.hpp"

template <class T>
static void put(FILE *f, const std::vector<T> &v) { fwrite(v.data(), sizeof(T), v.size(), f); }

int main(int argc, char **argv)
{
    if (argc < 3) return 2;
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 3;
    int32_t hdr[4];
    if (fread(hdr, 4, 4, f) != 4) return 4;   // X, Y, W, B
    const int B = hdr[3];
    const size_t ncell = (size_t)hdr[0] * hdr[1] * hdr[2];
    std::vector<float> cells(4 * ncell);
    if (fread(cells.data(), 4, cells.size(), f) != cells.size()) return 5;
    std::vector<int32_t> N(B), M(B), env(B, 0);
    std::vector<double> bnd(18 * (size_t)B), T(B), ixy, iyaw;
    std::vector<ualm_problem_params_t> pp(B);
    if (fread(N.data(), 4, B, f) != (size_t)B || fread(M.data(), 4, B, f) != (size_t)B) return 6;
    if (fread(bnd.data(), 8, bnd.size(), f) != bnd.size() || fread(T.data(), 8, B, f) != (size_t)B) return 7;
    if (fread(pp.data(), sizeof(ualm_problem_params_t), B, f) != (size_t)B) return 8;
    size_t nxy = 0, nyw = 0;
    for (int b = 0; b < B; b++) { nxy += 2 * (size_t)(N[b] - 1); nyw += (size_t)(M[b] - 1); }
    ixy.resize(nxy + 1); iyaw.resize(nyw + 1);
    if (fread(ixy.data(), 8, nxy, f) != nxy || fread(iyaw.data(), 8, nyw, f) != nyw) return 9;
    fclose(f);
    size_t ncx = 0, ncy = 0;
    for (int b = 0; b < B; b++) { ncx += 12 * (size_t)N[b]; ncy += 6 * (size_t)M[b]; }
    FILE *o = fopen(argv[2], "wb");
    if (!o) return 11;
    try {
        uneven_planner_b200::ALMTrajOpt opt(0, 64);
        ualm_map_geom_t g;
        ualm_map_geometry(10.0, 10.0, 0.05, 0.1, &g);
        ualm_params_t hill;
        ualm_default_params(&hill);
        opt.setEnvironment(0, hill, g, cells.data());
        std::vector<ualm_result_t> res(B), res2(B);
        std::vector<double> cxy(ncx), cyaw(ncy), cxy2(ncx), cyaw2(ncy);
        opt.optimizeBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), env.data(), pp.data(), res.data(), cxy.data(),
                          cyaw.data());
        std::vector<double> pt(2 * (size_t)B), tf(B, 0.5), out16(16 * (size_t)B);
        for (int b = 0; b < B; b++) { pt[2 * b] = res[b].piece_T_xy; pt[2 * b + 1] = res[b].piece_T_yaw; }
        const int t = opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), env.data(), pp.data(), 2);
        opt.checkTrajectories(B, N.data(), M.data(), pt.data(), cxy.data(), cyaw.data(), env.data(), pp.data(), tf.data(), 0.01, nullptr, out16.data());
        opt.waitBatch(t, res2.data(), cxy2.data(), cyaw2.data());
        put(o, res); put(o, cxy); put(o, cyaw); put(o, res2); put(o, cxy2); put(o, cyaw2); put(o, out16);
        std::vector<int32_t> No(B), Mo(B);
        std::vector<double> bo(18 * (size_t)B), To(B);
        const int r = opt.submitReplan(B, N.data(), M.data(), pt.data(), cxy.data(), cyaw.data(), bnd.data(), env.data(), pp.data(), tf.data(), 0.01,
                                       nullptr, 2, No.data(), Mo.data(), bo.data(), To.data());
        size_t rcx = 0, rcy = 0;
        for (int b = 0; b < B; b++) { rcx += 12 * (size_t)No[b]; rcy += 6 * (size_t)Mo[b]; }
        std::vector<ualm_result_t> res3(B);
        std::vector<double> cxy3(rcx), cyaw3(rcy);
        opt.waitBatch(r, res3.data(), cxy3.data(), cyaw3.data());
        put(o, No); put(o, Mo); put(o, res3); put(o, cxy3); put(o, cyaw3);
    } catch (const std::exception &e) {
        printf("EXCEPTION %s\n", e.what());
        fclose(o);
        return 10;
    }
    fclose(o);
    return 0;
}
