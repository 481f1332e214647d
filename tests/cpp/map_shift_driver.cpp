// Drives ALMTrajOpt::shiftEnvironment / shiftEnvironmentFromCloud of the C++ mirror (include/ualm_traj_opt.hpp): one batch submitted
// on grid G0, the grid moved by (dx, dy) cells with host cells for the uncovered strips while it is in flight, the batch submitted again,
// the grid moved once more by (dx2, dy2) with the strips built from a point cloud, the batch submitted a third time, then all three
// waited.  A zero shift must be refused.  Reads the grid, the shifts, the strip cells, the cloud and the problems from a binary file
// written by the test; prints one line per problem and submit, and writes the cloud shift's strip cells to the file named by the second
// argument.
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <vector>
#include "ualm_traj_opt.hpp"

int main(int argc, char **argv)
{
    if (argc < 3) return 2;
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 3;
    int32_t hdr[11];
    if (fread(hdr, 4, 11, f) != 11) return 4;   // X, Y, W, B, dx, dy, n strip floats, dx2, dy2, n cloud strip floats, npts
    const int B = hdr[3], dx = hdr[4], dy = hdr[5], dx2 = hdr[7], dy2 = hdr[8], npts = hdr[10];
    const size_t ncell = (size_t)hdr[0] * hdr[1] * hdr[2];
    std::vector<float> g0(4 * ncell), strips((size_t)hdr[6]), pts(3 * (size_t)npts + 1), out((size_t)hdr[9]);
    if (fread(g0.data(), 4, g0.size(), f) != g0.size() || fread(strips.data(), 4, strips.size(), f) != strips.size()) return 5;
    if (fread(pts.data(), 4, 3 * (size_t)npts, f) != 3 * (size_t)npts) return 5;
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
        int t[3];
        t[0] = opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), 3);
        opt.shiftEnvironment(0, dx, dy, strips.data());
        t[1] = opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), 3);
        float ms = 0.f;
        opt.shiftEnvironmentFromCloud(0, pts.data(), npts, dx2, dy2, 0.2, 0.1, 0.1, 2, out.data(), &ms);
        t[2] = opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), 3);
        try {
            opt.shiftEnvironment(0, 0, 0, strips.data());
            printf("NOT REFUSED\n");
            return 11;
        } catch (const std::runtime_error &) {
        }
        std::vector<ualm_result_t> res(B);
        std::vector<double> cxy(ncx), cyaw(ncy);
        for (int pass = 0; pass < 3; pass++) {
            opt.waitBatch(t[pass], res.data(), cxy.data(), cyaw.data());
            size_t ox = 0;
            for (int b = 0; b < B; b++) {
                printf("%d %d %d %d %.17g %.17g\n", pass, b, res[b].ret_code, res[b].n_evals, res[b].inner_cost, cxy[ox + 1]);
                ox += 12 * (size_t)N[b];
            }
        }
        if (!(ms > 0.f)) return 12;
    } catch (const std::exception &e) {
        printf("EXCEPTION %s\n", e.what());
        return 10;
    }
    FILE *o = fopen(argv[2], "wb");
    if (!o || fwrite(out.data(), 4, out.size(), o) != out.size()) return 13;
    fclose(o);
    return 0;
}
