// Drives cancelProblems of the C++ ALMTrajOpt mirror (include/ualm_traj_opt.hpp): the batch is solved once through optimizeBatch,
// then submitted again, every even problem is cancelled right after submitBatch, and the batch is polled until nothing is pending
// and waited.  Every problem must come back from the polls exactly once, the polled outputs must equal waitBatch's byte for byte,
// every odd problem must equal its optimizeBatch result, and every even one too unless it ends with UALM_RET_STOPPED.  A refused
// call (an index out of range) must throw.  Reads the map and the problems from a binary file written by the test; argv[2] =
// precision.  Prints "OK <stopped problems>".
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
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
    std::vector<size_t> ocx(B + 1, 0), ocy(B + 1, 0);
    for (int b = 0; b < B; b++) { ocx[b + 1] = ocx[b] + 12 * (size_t)N[b]; ocy[b + 1] = ocy[b] + 6 * (size_t)M[b]; }
    const size_t ncx = ocx[B], ncy = ocy[B];
    try {
        uneven_planner_b200::ALMTrajOpt opt(0, atoi(argv[2]));
        ualm_map_geom_t g;
        ualm_map_geometry(10.0, 10.0, 0.05, 0.1, &g);
        opt.setEnvironment(g, cells.data());
        opt.init();
        std::vector<ualm_result_t> fres(B), pres(B), wres(B);
        std::vector<double> fcxy(ncx), fcyaw(ncy), pcxy(ncx), pcyaw(ncy), wcxy(ncx), wcyaw(ncy);
        opt.optimizeBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), fres.data(), fcxy.data(), fcyaw.data());
        const int t = opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), 1);
        std::vector<int32_t> even;
        for (int b = 0; b < B; b += 2) even.push_back(b);
        opt.cancelProblems(t, (int)even.size(), even.data());
        const int32_t bad[2] = {1, B};
        bool threw = false;
        try { opt.cancelProblems(t, 2, bad); } catch (const std::runtime_error &) { threw = true; }
        if (!threw) { printf("BAD an index out of range was accepted\n"); return 15; }
        std::vector<int32_t> idx(B);
        std::vector<int> seen(B, 0);
        int pending = B, polls = 0;
        while (pending > 0) {
            const int n = opt.pollBatch(t, 5.0, idx.data(), &pending, pres.data(), pcxy.data(), pcyaw.data());
            for (int k = 0; k < n; k++)
                if (idx[k] < 0 || idx[k] >= B || seen[idx[k]]++) { printf("BAD index %d\n", idx[k]); return 11; }
            if (++polls > 1000000) { printf("BAD too many polls\n"); return 12; }
        }
        opt.waitBatch(t, wres.data(), wcxy.data(), wcyaw.data());
        for (int b = 0; b < B; b++)
            if (!seen[b]) { printf("BAD problem %d never returned\n", b); return 13; }
        if (memcmp(pres.data(), wres.data(), sizeof(ualm_result_t) * B) != 0 || memcmp(pcxy.data(), wcxy.data(), sizeof(double) * ncx) != 0 ||
            memcmp(pcyaw.data(), wcyaw.data(), sizeof(double) * ncy) != 0) {
            printf("BAD polled outputs differ from waitBatch\n");
            return 14;
        }
        int stopped = 0;
        for (int b = 0; b < B; b++) {
            if (b % 2 == 0 && wres[b].ret_code == UALM_RET_STOPPED) { stopped++; continue; }
            if (memcmp(&wres[b], &fres[b], sizeof(ualm_result_t)) != 0 || memcmp(&wcxy[ocx[b]], &fcxy[ocx[b]], sizeof(double) * (ocx[b + 1] - ocx[b])) != 0 ||
                memcmp(&wcyaw[ocy[b]], &fcyaw[ocy[b]], sizeof(double) * (ocy[b + 1] - ocy[b])) != 0) {
                printf("BAD problem %d differs from its uncancelled solve\n", b);
                return 16;
            }
        }
        if (stopped == 0) { printf("BAD no cancelled problem stopped\n"); return 17; }
        printf("OK %d\n", stopped);
    } catch (const std::exception &e) {
        printf("EXCEPTION %s\n", e.what());
        return 10;
    }
    return 0;
}
