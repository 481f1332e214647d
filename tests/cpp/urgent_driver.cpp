// Drives ALMTrajOpt::setUrgent of the C++ mirror (include/ualm_traj_opt.hpp) at a given precision: a batch solved, checked and
// replanned idle; then two background tickets of a larger batch in flight and, with setUrgent(true), the same batch submitted, checked
// and replanned again, then setUrgent(false).  Every record and coefficient of every ticket, every check row and every built replan row
// must be byte-identical to the idle calls (the background tickets to the larger batch solved idle).  Reads the grid, the small batch,
// its t_from and the number of copies of it in the background batch from a binary file written by the test; prints "OK ..." or the
// first difference.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <vector>
#include "ualm_traj_opt.hpp"

template <class T>
static bool same(const std::vector<T> &a, const std::vector<T> &b)
{
    return a.size() == b.size() && (a.empty() || memcmp(a.data(), b.data(), sizeof(T) * a.size()) == 0);
}

int main(int argc, char **argv)
{
    if (argc < 3) return 2;
    const int precision = atoi(argv[2]);
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 3;
    int32_t hdr[5];
    if (fread(hdr, 4, 5, f) != 5) return 4;   // X, Y, W, B, copies
    const int B = hdr[3], copies = hdr[4];
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
    // the background batch: `copies` copies of the small one
    const int BB = B * copies;
    std::vector<int32_t> NB, MB;
    std::vector<double> bndB, TB, ixyB, iyawB;
    for (int k = 0; k < copies; k++) {
        NB.insert(NB.end(), N.begin(), N.end()); MB.insert(MB.end(), M.begin(), M.end());
        bndB.insert(bndB.end(), bnd.begin(), bnd.end()); TB.insert(TB.end(), T.begin(), T.end());
        ixyB.insert(ixyB.end(), ixy.begin(), ixy.begin() + nxy); iyawB.insert(iyawB.end(), iyaw.begin(), iyaw.begin() + nyw);
    }
    ixyB.push_back(0.0); iyawB.push_back(0.0);
    try {
        uneven_planner_b200::ALMTrajOpt opt(0, precision);
        ualm_map_geom_t g;
        ualm_map_geometry(10.0, 10.0, 0.05, 0.1, &g);
        opt.init();
        opt.setEnvironment(g, g0.data());
        const int depth = 4;
        // idle: the small batch, its check, its replan; the background batch
        std::vector<ualm_result_t> res(B), resB(BB);
        std::vector<double> cxy(ncx), cyaw(ncy), pt(2 * (size_t)B), chk(16 * (size_t)B), cxyB(ncx * copies), cyawB(ncy * copies);
        opt.waitBatch(opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), depth), res.data(), cxy.data(), cyaw.data());
        opt.waitBatch(opt.submitBatch(BB, NB.data(), MB.data(), bndB.data(), TB.data(), ixyB.data(), iyawB.data(), depth), resB.data(), cxyB.data(),
                      cyawB.data());
        for (int b = 0; b < B; b++) { pt[2 * b] = res[b].piece_T_xy; pt[2 * b + 1] = res[b].piece_T_yaw; }
        opt.checkTrajectories(B, N.data(), M.data(), pt.data(), cxy.data(), cyaw.data(), nullptr, nullptr, 0.01, nullptr, chk.data());
        std::vector<int32_t> N2(B), M2(B), N2u(B), M2u(B);
        std::vector<double> bnd2(18 * (size_t)B), T2(B), bnd2u(18 * (size_t)B), T2u(B);
        const int tr = opt.submitReplan(B, N.data(), M.data(), pt.data(), cxy.data(), cyaw.data(), bnd.data(), nullptr, tf.data(), 0.01, nullptr, depth,
                                        N2.data(), M2.data(), bnd2.data(), T2.data());
        size_t ncx2 = 0, ncy2 = 0;
        for (int b = 0; b < B; b++) { ncx2 += 12 * (size_t)N2[b]; ncy2 += 6 * (size_t)M2[b]; }
        std::vector<ualm_result_t> rr(B);
        std::vector<double> rcx(ncx2), rcy(ncy2);
        opt.waitBatch(tr, rr.data(), rcx.data(), rcy.data());
        // in flight: two background tickets, then the urgent calls
        const int b0 = opt.submitBatch(BB, NB.data(), MB.data(), bndB.data(), TB.data(), ixyB.data(), iyawB.data(), depth);
        const int b1 = opt.submitBatch(BB, NB.data(), MB.data(), bndB.data(), TB.data(), ixyB.data(), iyawB.data(), depth);
        opt.setUrgent(true);
        const int tu = opt.submitBatch(B, N.data(), M.data(), bnd.data(), T.data(), ixy.data(), iyaw.data(), depth);
        std::vector<double> chku(16 * (size_t)B);
        opt.checkTrajectories(B, N.data(), M.data(), pt.data(), cxy.data(), cyaw.data(), nullptr, nullptr, 0.01, nullptr, chku.data());
        const int tru = opt.submitReplan(B, N.data(), M.data(), pt.data(), cxy.data(), cyaw.data(), bnd.data(), nullptr, tf.data(), 0.01, nullptr, depth,
                                         N2u.data(), M2u.data(), bnd2u.data(), T2u.data());
        opt.setUrgent(false);
        std::vector<ualm_result_t> resu(B), rru(B), r0(BB), r1(BB);
        std::vector<double> cxyu(ncx), cyawu(ncy), rcxu(ncx2), rcyu(ncy2), c0(ncx * copies), y0(ncy * copies), c1(ncx * copies), y1(ncy * copies);
        opt.waitBatch(tu, resu.data(), cxyu.data(), cyawu.data());
        opt.waitBatch(tru, rru.data(), rcxu.data(), rcyu.data());
        opt.waitBatch(b0, r0.data(), c0.data(), y0.data());
        opt.waitBatch(b1, r1.data(), c1.data(), y1.data());
        const char *bad = nullptr;
        if (!same(res, resu) || !same(cxy, cxyu) || !same(cyaw, cyawu)) bad = "urgent ticket";
        else if (!same(chk, chku)) bad = "urgent check";
        else if (!same(N2, N2u) || !same(M2, M2u) || !same(bnd2, bnd2u) || !same(T2, T2u)) bad = "urgent replan build";
        else if (!same(rr, rru) || !same(rcx, rcxu) || !same(rcy, rcyu)) bad = "urgent replan ticket";
        else if (!same(resB, r0) || !same(cxyB, c0) || !same(cyawB, y0) || !same(resB, r1) || !same(cxyB, c1) || !same(cyawB, y1)) bad = "background ticket";
        if (bad) { printf("DIFFERS %s\n", bad); return 12; }
        printf("OK precision %d: %d urgent problems, check and replan rows byte-identical with %d background problems in flight\n", precision, B, 2 * BB);
    } catch (const std::exception &e) {
        printf("EXCEPTION %s\n", e.what());
        return 10;
    }
    return 0;
}
