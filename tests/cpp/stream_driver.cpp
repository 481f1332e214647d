// Drives pollBatch of the C++ ALMTrajOpt mirror (include/ualm_traj_opt.hpp): one batch through submitBatch, polled with a short
// wait until nothing is pending, then waitBatch on the same ticket into separate buffers.  Every problem must come back from the
// polls exactly once, and the union of the polled records and coefficients must equal waitBatch's byte for byte.  Reads the map
// and the problems from a binary file written by the test; argv[2] = precision.  Prints "OK <polls> <polls that returned problems>".
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "ualm_traj_opt.hpp"

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
        uneven_planner_b200::ALMTrajOpt opt(0, atoi(argv[2]));
        ualm_map_geom_t g;
        ualm_map_geometry(10.0, 10.0, 0.05, 0.1, &g);
        opt.setEnvironment(g, cells.data());
        opt.init();
        std::vector<ualm_result_t> pres(B), wres(B);
        std::vector<double> pcxy(ncx), pcyaw(ncy), wcxy(ncx), wcyaw(ncy);
        std::vector<int32_t> idx(B);
        std::vector<int> seen(B, 0);
        const int t = opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), 1);
        int pending = B, polls = 0, fruitful = 0;
        while (pending > 0) {
            const int n = opt.pollBatch(t, 5.0, idx.data(), &pending, pres.data(), pcxy.data(), pcyaw.data());
            polls++;
            if (n > 0) fruitful++;
            for (int k = 0; k < n; k++) {
                if (idx[k] < 0 || idx[k] >= B || seen[idx[k]]++) { printf("BAD index %d\n", idx[k]); return 11; }
            }
            if (polls > 1000000) { printf("BAD too many polls\n"); return 12; }
        }
        opt.waitBatch(t, wres.data(), wcxy.data(), wcyaw.data());
        for (int b = 0; b < B; b++)
            if (!seen[b]) { printf("BAD problem %d never returned\n", b); return 13; }
        if (memcmp(pres.data(), wres.data(), sizeof(ualm_result_t) * B) != 0 || memcmp(pcxy.data(), wcxy.data(), sizeof(double) * ncx) != 0 ||
            memcmp(pcyaw.data(), wcyaw.data(), sizeof(double) * ncy) != 0) {
            printf("BAD polled outputs differ from waitBatch\n");
            return 14;
        }
        printf("OK %d %d\n", polls, fruitful);
    } catch (const std::exception &e) {
        printf("EXCEPTION %s\n", e.what());
        return 10;
    }
    return 0;
}
