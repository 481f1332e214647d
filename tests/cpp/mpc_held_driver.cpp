// Drives ALMTrajOpt::exportToMpc of the C++ mirror (include/ualm_traj_opt.hpp): a batch solved and waited, the batch submitted again,
// the first batch's records handed over with each row's own boundary derivatives while the second is in flight.  Reads the grid, the
// problems and init_v / init_a (3 per row each) from a binary file written by the test; prints one line per output array: its name
// and its values.
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <vector>
#include "ualm_traj_opt.hpp"

static void print(const char *name, const std::vector<double> &v)
{
    printf("%s", name);
    for (double x : v) printf(" %.17g", x);
    printf("\n");
}

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
    std::vector<double> bnd(18 * (size_t)B), T(B), ixy, iyaw, iv(3 * (size_t)B), ia(3 * (size_t)B);
    if (fread(N.data(), 4, B, f) != (size_t)B || fread(M.data(), 4, B, f) != (size_t)B) return 6;
    if (fread(bnd.data(), 8, bnd.size(), f) != bnd.size() || fread(T.data(), 8, B, f) != (size_t)B) return 7;
    size_t nxy = 0, nyw = 0, sN = 0, sM = 0;
    for (int b = 0; b < B; b++) { nxy += 2 * (size_t)(N[b] - 1); nyw += (size_t)(M[b] - 1); sN += N[b]; sM += M[b]; }
    ixy.resize(nxy + 1); iyaw.resize(nyw + 1);
    if (fread(ixy.data(), 8, nxy, f) != nxy || fread(iyaw.data(), 8, nyw, f) != nyw) return 8;
    if (fread(iv.data(), 8, iv.size(), f) != iv.size() || fread(ia.data(), 8, ia.size(), f) != ia.size()) return 9;
    fclose(f);
    try {
        uneven_planner_b200::ALMTrajOpt opt(0, 64);
        ualm_map_geom_t g;
        ualm_map_geometry(10.0, 10.0, 0.05, 0.1, &g);
        opt.init();
        opt.setEnvironment(g, g0.data());
        std::vector<ualm_result_t> res(B);
        std::vector<double> cxy(12 * sN), cyaw(6 * sM), pt(2 * (size_t)B);
        opt.waitBatch(opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), 3), res.data(), cxy.data(), cyaw.data());
        for (int b = 0; b < B; b++) { pt[2 * b] = res[b].piece_T_xy; pt[2 * b + 1] = res[b].piece_T_yaw; }
        const int t2 = opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), 3);
        std::vector<double> pos(2 * (sN + B)), posT(sN), ang(sM + B), angT(sM), mxy(12 * sN), myaw(6 * sM), dev(4 * (size_t)B);
        opt.exportToMpc(B, N.data(), M.data(), pt.data(), cxy.data(), cyaw.data(), iv.data(), ia.data(), 0.01, pos.data(), posT.data(), ang.data(),
                        angT.data(), mxy.data(), myaw.data(), dev.data());
        opt.waitBatch(t2, res.data(), cxy.data(), cyaw.data());
        print("pos_pts", pos); print("posT_pts", posT); print("angle_pts", ang); print("angleT_pts", angT);
        print("c_mpc_xy", mxy); print("c_mpc_yaw", myaw); print("dev", dev);
    } catch (const std::exception &e) {
        printf("EXCEPTION %s\n", e.what());
        return 10;
    }
    return 0;
}
