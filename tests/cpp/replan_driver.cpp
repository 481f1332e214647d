// Drives ALMTrajOpt::submitReplan of the C++ mirror (include/ualm_traj_opt.hpp): a batch solved on grid G0 and waited, the batch
// submitted again, the first batch's trajectories replanned from t_from while the second is in flight, then both tickets waited.  A
// replan with a t_from past the end must be refused.  Reads the grid, the problems and t_from from a binary file written by the test;
// prints per problem "b N' M' total_time bnd'(18) ret_code total_T" and then the replanned coefficients, c_xy then c_yaw, one per line.
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <vector>
#include "ualm_traj_opt.hpp"

int main(int argc, char **argv)
{
    if (argc < 2) return 2;
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 3;
    int32_t hdr[4];
    if (fread(hdr, 4, 4, f) != 4) return 4;   // X, Y, W, B
    const int B = hdr[3];
    const size_t ncell = (size_t)hdr[0] * hdr[1] * hdr[2];
    std::vector<float> g0(4 * ncell);
    if (fread(g0.data(), 4, g0.size(), f) != g0.size()) return 5;
    std::vector<int32_t> N(B), M(B);
    std::vector<double> bnd(18 * (size_t)B), T(B), tf(B), ixy, iyaw;
    if (fread(N.data(), 4, B, f) != (size_t)B || fread(M.data(), 4, B, f) != (size_t)B) return 6;
    if (fread(bnd.data(), 8, bnd.size(), f) != bnd.size() || fread(T.data(), 8, B, f) != (size_t)B) return 7;
    size_t nxy = 0, nyw = 0;
    for (int b = 0; b < B; b++) { nxy += 2 * (size_t)(N[b] - 1); nyw += (size_t)(M[b] - 1); }
    ixy.resize(nxy + 1); iyaw.resize(nyw + 1);
    if (fread(ixy.data(), 8, nxy, f) != nxy || fread(iyaw.data(), 8, nyw, f) != nyw || fread(tf.data(), 8, B, f) != (size_t)B) return 8;
    fclose(f);
    size_t ncx = 0, ncy = 0;
    for (int b = 0; b < B; b++) { ncx += 12 * (size_t)N[b]; ncy += 6 * (size_t)M[b]; }
    try {
        uneven_planner_b200::ALMTrajOpt opt(0, 64);
        ualm_map_geom_t g;
        ualm_map_geometry(10.0, 10.0, 0.05, 0.1, &g);
        opt.init();
        opt.setEnvironment(g, g0.data());
        std::vector<ualm_result_t> res(B);
        std::vector<double> cxy(ncx), cyaw(ncy), pt(2 * (size_t)B);
        opt.waitBatch(opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), 3), res.data(), cxy.data(), cyaw.data());
        for (int b = 0; b < B; b++) { pt[2 * b] = res[b].piece_T_xy; pt[2 * b + 1] = res[b].piece_T_yaw; }
        const int t2 = opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), 3);
        std::vector<int32_t> N2(B), M2(B);
        std::vector<double> bnd2(18 * (size_t)B), T2(B);
        std::vector<double> bad(tf);
        bad[0] = 1e9;
        try {
            opt.submitReplan(B, N.data(), M.data(), pt.data(), cxy.data(), cyaw.data(), bnd.data(), nullptr, bad.data(), 0.01, nullptr, 3, N2.data(),
                             M2.data(), bnd2.data(), T2.data());
            printf("NOT REFUSED\n");
            return 11;
        } catch (const std::runtime_error &) {
        }
        const int t3 = opt.submitReplan(B, N.data(), M.data(), pt.data(), cxy.data(), cyaw.data(), bnd.data(), nullptr, tf.data(), 0.01, nullptr, 3,
                                        N2.data(), M2.data(), bnd2.data(), T2.data());
        opt.waitBatch(t2, res.data(), cxy.data(), cyaw.data());
        size_t ncx2 = 0, ncy2 = 0;
        for (int b = 0; b < B; b++) { ncx2 += 12 * (size_t)N2[b]; ncy2 += 6 * (size_t)M2[b]; }
        std::vector<ualm_result_t> res2(B);
        std::vector<double> cxy2(ncx2), cyaw2(ncy2);
        opt.waitBatch(t3, res2.data(), cxy2.data(), cyaw2.data());
        for (int b = 0; b < B; b++) {
            printf("%d %d %d %.17g", b, N2[b], M2[b], T2[b]);
            for (int q = 0; q < 18; q++) printf(" %.17g", bnd2[18 * (size_t)b + q]);
            printf(" %d %.17g\n", res2[b].ret_code, res2[b].total_T);
        }
        for (double v : cxy2) printf("%.17g\n", v);
        for (double v : cyaw2) printf("%.17g\n", v);
    } catch (const std::exception &e) {
        printf("EXCEPTION %s\n", e.what());
        return 10;
    }
    return 0;
}
