// Drives ALMTrajOpt::updateEnvironment of the C++ mirror (include/ualm_traj_opt.hpp): one batch submitted on grid G0, the grid of
// environment 0 replaced by G1 while it is in flight, the same batch submitted again, then both waited.  Reads both grids and the
// problems from a binary file written by the test; prints one line per problem and submit.
#include <cstdio>
#include <cstdlib>
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
    std::vector<float> g0(4 * ncell), g1(4 * ncell);
    if (fread(g0.data(), 4, g0.size(), f) != g0.size() || fread(g1.data(), 4, g1.size(), f) != g1.size()) return 5;
    std::vector<int32_t> N(B), M(B);
    std::vector<double> bnd(18 * (size_t)B), T(B), ixy, iyaw;
    if (fread(N.data(), 4, B, f) != (size_t)B || fread(M.data(), 4, B, f) != (size_t)B) return 6;
    if (fread(bnd.data(), 8, bnd.size(), f) != bnd.size() || fread(T.data(), 8, B, f) != (size_t)B) return 7;
    size_t nxy = 0, nyw = 0;
    for (int b = 0; b < B; b++) { nxy += 2 * (size_t)(N[b] - 1); nyw += (size_t)(M[b] - 1); }
    ixy.resize(nxy + 1); iyaw.resize(nyw + 1);
    if (fread(ixy.data(), 8, nxy, f) != nxy || fread(iyaw.data(), 8, nyw, f) != nyw) return 8;
    fclose(f);
    size_t ncx = 0, ncy = 0;
    for (int b = 0; b < B; b++) { ncx += 12 * (size_t)N[b]; ncy += 6 * (size_t)M[b]; }
    try {
        uneven_planner_b200::ALMTrajOpt opt(0, 64);
        ualm_map_geom_t g;
        ualm_map_geometry(10.0, 10.0, 0.05, 0.1, &g);
        opt.init();
        opt.setEnvironment(g, g0.data());
        const int t0 = opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), 2);
        opt.updateEnvironment(0, g, g1.data());
        const int t1 = opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), 2);
        std::vector<ualm_result_t> res(B);
        std::vector<double> cxy(ncx), cyaw(ncy);
        for (int pass = 0; pass < 2; pass++) {
            opt.waitBatch(pass == 0 ? t0 : t1, res.data(), cxy.data(), cyaw.data());
            size_t ox = 0;
            for (int b = 0; b < B; b++) {
                printf("%d %d %d %d %.17g %.17g\n", pass, b, res[b].ret_code, res[b].n_evals, res[b].inner_cost, cxy[ox + 1]);
                ox += 12 * (size_t)N[b];
            }
        }
    } catch (const std::exception &e) {
        printf("EXCEPTION %s\n", e.what());
        return 10;
    }
    return 0;
}
