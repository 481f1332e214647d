// cancel_oracle.cpp -- the CPU reference of a cancelled problem (include/ualm.h, ualm_cancel_problems): the oracle's optimizeSE2Traj
// restatement (oracle/oracle.cpp, included unmodified so every evaluation, line search and dual update is its code) with a stop
// predicate where the CUDA paths test it.  TEST INFRASTRUCTURE ONLY, built by tests/cancel_oracle.py.
//
// The GPU stops a cancelled problem at the first stop test that sees its stop word raised, and every later test sees it too.  So a
// cancelled solve is the solve with a predicate that holds from its s-th stop test on, counting both test sites in execution order:
// the earlyExit point (after every accepted line search, where earlyExit tests k > 1000; L-BFGS then returns CANCELED) and the ALM
// loop after judgeConvergence.  The exit order is the one of tests/budget_oracle.cpp: a stop that ended the inner solve just finished
// -> 3 even when judgeConvergence passes; else converged -> 0; else stop holds now -> 3; else ++iter > max_iter -> 2.
//   orc_solve_cancel(s)  the solve stopped from its s-th test on (s past the last test: orc_solve)
//   orc_stop_tests       n_evals and site of every test of the solve without a stop (the candidates for s)
#include "../oracle/oracle.cpp"

#define CANCEL_RET_STOPPED 3

namespace {

// stop_at(n_evals, site) is called once per stop test in execution order; site 0 = earlyExit point, 1 = after judgeConvergence
template <class Stop>
int solve_stop_impl(const orc_params_t *p, const orc_map_t *map, const orc_problem_t *prob, Stop stop_at, orc_result_t *res,
                    double *c_xy_out, double *c_yaw_out, double *x_out)
{
    using R = double;
    MapQ<R> mq(*map);
    ALM<R> alm(*p, &mq);
    alm.setup(*prob);
    const int n = alm.nvar();
    std::vector<R> x(n);
    x[0] = logC2((R)prob->total_time);
    for (int i = 0; i < 2 * (alm.piece_xy - 1); i++) x[1 + i] = (R)prob->inner_xy[i];
    for (int i = 0; i < alm.piece_yaw - 1; i++) x[1 + 2 * (alm.piece_xy - 1) + i] = (R)prob->inner_yaw[i];

    LbfgsParam<R> lp;
    lp.mem_size = alm.mem_size; lp.past = alm.past; lp.g_epsilon = alm.g_epsilon; lp.min_step = alm.min_step;
    lp.delta = alm.delta; lp.max_iterations = (int)alm.inner_max_iter;
    R inner_cost = 0;
    int ret_code = 0, iter = 0, last = 0;
    LbfgsStats st;

    if (alm.use_scaling) alm.initScaling(x);

    auto eval = [&](const std::vector<R> &xx, std::vector<R> &gg) { return alm.evaluate(xx, gg); };
    bool fired = false;   // the stop ended the inner solve that just returned
    auto progress = [&](int k) { fired = stop_at((int)alm.n_evals, 0); return k > 1e3 || fired; };   // earlyExit alm_traj_opt.cpp:1016
    R rh = 0, rg = 0;
    while (true) {
        fired = false;
        int result = lbfgs_optimize(x, inner_cost, eval, progress, lp, st);
        last = result;
        if (result == LBFGS_CONVERGENCE || result == LBFGS_CANCELED || result == LBFGS_STOP ||
            result == LBFGSERR_MAXIMUMITERATION) {
        } else if (result == LBFGSERR_MAXIMUMLINESEARCH) {
        } else { ret_code = 1; break; }
        alm.updateDualVars();
        const bool converged = alm.judgeConvergence(rh, rg);
        if (fired) { ret_code = CANCEL_RET_STOPPED; break; }
        if (converged) break;
        if (stop_at((int)alm.n_evals, 1)) { ret_code = CANCEL_RET_STOPPED; break; }
        if (++iter > alm.max_iter) { ret_code = 2; break; }
    }
    memset(res, 0, sizeof(*res));
    res->ret_code = ret_code; res->outer_iters = iter; res->n_evals = alm.n_evals; res->n_lbfgs_iters = st.iters;
    res->last_lbfgs_ret = last; res->max_bound = st.max_bound; res->inner_cost = inner_cost;
    res->jerk_cost = alm.pos_minco.getTrajJerkCost() + alm.yaw_minco.getTrajJerkCost();
    R tt = 0; for (auto t : alm.pos_minco.T1) tt += t;
    res->total_T = tt;
    res->res_h = rh; res->res_g = rg; res->scale_fx = alm.scale_fx; res->rho_final = alm.rho;
    if (c_xy_out) for (size_t i = 0; i < alm.pos_minco.c.size(); i++) c_xy_out[i] = alm.pos_minco.c[i];
    if (c_yaw_out) for (size_t i = 0; i < alm.yaw_minco.c.size(); i++) c_yaw_out[i] = alm.yaw_minco.c[i];
    if (x_out) for (int i = 0; i < n; i++) x_out[i] = x[i];
    return ret_code;
}

} // namespace

// the solve of a problem cancelled so that its s-th stop test (1-based, both sites counted in execution order) is the first to see
// its stop word: the predicate holds from that test on.  s past the last test is the solve without a stop (orc_solve)
extern "C" int orc_solve_cancel(const orc_params_t *p, const orc_map_t *map, const orc_problem_t *prob, int s, orc_result_t *res,
                                double *c_xy_out, double *c_yaw_out, double *x_out)
{
    int count = 0;
    return solve_stop_impl(p, map, prob, [&](int, int) { return ++count >= s; }, res, c_xy_out, c_yaw_out, x_out);
}

// the stop tests of the solve without a stop: n_evals and site (0 = earlyExit point, 1 = after judgeConvergence) of the first `cap`
// tests in execution order; returns how many tests the solve made
extern "C" int orc_stop_tests(const orc_params_t *p, const orc_map_t *map, const orc_problem_t *prob, int cap, int *n_evals_out, int *site_out)
{
    int count = 0;
    orc_result_t res;
    solve_stop_impl(p, map, prob, [&](int n_evals, int site) {
        if (count < cap) { n_evals_out[count] = n_evals; site_out[count] = site; }
        count++;
        return false;
    }, &res, nullptr, nullptr, nullptr);
    return count;
}
