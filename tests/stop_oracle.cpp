// stop_oracle.cpp -- the CPU references of a stopped solve (include/ualm.h, UALM_RET_STOPPED): the oracle's optimizeSE2Traj restatement
// (oracle/oracle.cpp, included unmodified, so the loop, every evaluation, line search and dual update is its solve_impl) with the stop
// predicate of an evaluation budget or of a cancel.  solve_impl calls the predicate at every stop test the CUDA paths make, in execution
// order, and documents the exit order.  TEST INFRASTRUCTURE ONLY, built by tests/stop_oracle.py.
//   orc_solve_budget(max_evals)  stop = max_evals > 0 && n_evals >= max_evals (max_evals = 0: orc_solve)
//   orc_solve_cancel(s)          the GPU stops a cancelled problem at the first stop test that sees its stop word raised, and every later
//                                test sees it too: the predicate holds from the s-th test on (s past the last test: orc_solve)
//   orc_stop_tests               n_evals and site of every test of the solve without a stop (the candidates for s)
#include "../oracle/oracle.cpp"

extern "C" int orc_solve_budget(const orc_params_t *p, const orc_map_t *map, const orc_problem_t *prob, int max_evals, orc_result_t *res,
                                double *c_xy_out, double *c_yaw_out, double *x_out)
{
    return solve_impl<double>(p, map, prob, [&](int n_evals, int) { return max_evals > 0 && n_evals >= max_evals; }, res, c_xy_out,
                              c_yaw_out, x_out, nullptr, nullptr, nullptr);
}

// the solve of a problem cancelled so that its s-th stop test (1-based, both sites counted in execution order) is the first to see
// its stop word
extern "C" int orc_solve_cancel(const orc_params_t *p, const orc_map_t *map, const orc_problem_t *prob, int s, orc_result_t *res,
                                double *c_xy_out, double *c_yaw_out, double *x_out)
{
    int count = 0;
    return solve_impl<double>(p, map, prob, [&](int, int) { return ++count >= s; }, res, c_xy_out, c_yaw_out, x_out, nullptr, nullptr,
                              nullptr);
}

// the stop tests of the solve without a stop: n_evals and site (0 = earlyExit point, 1 = after judgeConvergence) of the first `cap`
// tests in execution order; returns how many tests the solve made
extern "C" int orc_stop_tests(const orc_params_t *p, const orc_map_t *map, const orc_problem_t *prob, int cap, int *n_evals_out, int *site_out)
{
    int count = 0;
    orc_result_t res;
    solve_impl<double>(p, map, prob, [&](int n_evals, int site) {
        if (count < cap) { n_evals_out[count] = n_evals; site_out[count] = site; }
        count++;
        return false;
    }, &res, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    return count;
}
