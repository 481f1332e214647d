// Drives ALMTrajOpt::checkTrajectories of the C++ mirror (include/ualm_traj_opt.hpp): a batch solved on grid G0 and waited, the batch
// submitted again, the first batch's trajectories checked from t_from while the second is in flight, a box of G0 replaced by host cells,
// the same check again.  A check with a negative t_from must be refused.  Reads the grid, the box and its cells, the problems and
// t_from from a binary file written by the test; prints "pass problem" and the 16 values per problem and check.
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
    int32_t hdr[8];
    if (fread(hdr, 4, 8, f) != 8) return 4;   // X, Y, W, B, ix0, iy0, nx, ny
    const int W = hdr[2], B = hdr[3], ix0 = hdr[4], iy0 = hdr[5], nx = hdr[6], ny = hdr[7];
    const size_t ncell = (size_t)hdr[0] * hdr[1] * W, nbox = (size_t)nx * ny * W;
    std::vector<float> g0(4 * ncell), win(4 * nbox);
    if (fread(g0.data(), 4, g0.size(), f) != g0.size() || fread(win.data(), 4, win.size(), f) != win.size()) return 5;
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
        std::vector<double> cxy(ncx), cyaw(ncy), pt(2 * (size_t)B), out(16 * (size_t)B);
        opt.waitBatch(opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), 3), res.data(), cxy.data(), cyaw.data());
        for (int b = 0; b < B; b++) { pt[2 * b] = res[b].piece_T_xy; pt[2 * b + 1] = res[b].piece_T_yaw; }
        const int t2 = opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), 3);
        for (int pass = 0; pass < 2; pass++) {
            if (pass == 1) opt.updateEnvironmentWindow(0, ix0, iy0, nx, ny, win.data());
            opt.checkTrajectories(B, N.data(), M.data(), pt.data(), cxy.data(), cyaw.data(), nullptr, tf.data(), 0.01, nullptr, out.data());
            for (int b = 0; b < B; b++) {
                printf("%d %d", pass, b);
                for (int q = 0; q < 16; q++) printf(" %.17g", out[16 * (size_t)b + q]);
                printf("\n");
            }
        }
        std::vector<double> bad(tf);
        bad[0] = -1.0;
        try {
            opt.checkTrajectories(B, N.data(), M.data(), pt.data(), cxy.data(), cyaw.data(), nullptr, bad.data(), 0.01, nullptr, out.data());
            printf("NOT REFUSED\n");
            return 11;
        } catch (const std::runtime_error &) {
        }
        opt.waitBatch(t2, res.data(), cxy.data(), cyaw.data());
    } catch (const std::exception &e) {
        printf("EXCEPTION %s\n", e.what());
        return 10;
    }
    return 0;
}
