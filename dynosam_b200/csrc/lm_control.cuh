// lm_control.cuh -- the decisions of GTSAM 4.2.0's LevenbergMarquardtOptimizer (NonlinearOptimizer::defaultOptimize,
// LevenbergMarquardtOptimizer::tryLambda, checkConvergence), stated once for the two loops that take them: the host loop
// of dynoba_optimize (api.cu) and the per-problem device loop run_lm of the batch kernels (kernels_star.cu).
// tests/capi/lm_control_host.cu compiles it for the host.
#pragma once
#include <cfloat>
#include <cmath>
#include <algorithm>
#include "../../include/dynoba.h"

namespace dynoba {

// The LM parameters every tryLambda loop is run with.  That loop ends on a run of failed steps only once lambda reaches
// lambda_upper_bound, so it refuses (false) what could keep it from getting there: lambda_initial not finite and > 0,
// lambda_factor not finite and > 1, a NaN upper bound.  It raises the lower bound to DBL_MIN so that a long run of
// accepted steps cannot divide lambda down to 0; below DBL_MIN, lambda I changes H + lambda I only where H has a diagonal
// entry below about 1e-290.  A factor so close to 1 that lambda needs more than LM_MAX_CLIMB failed steps to climb from
// the lowest value it can take to the upper bound is refused as well: that loop would end, but only after up to ~1e16
// damped solves.
//
// The outer loop ends after a give-up (lambda at its upper bound without a step) or a stop without a step only if
// lm_converged holds for a decrease of exactly 0, since neither adds an iteration and the next outer iteration would
// repeat it.  With currentError == newError = e finite: the absolute test holds for every e iff absolute_error_tol >= 0;
// the relative test, 0/e <= relative_error_tol, holds for every e != 0 iff relative_error_tol > 0 and never for e == 0
// (0/0 is NaN); e == 0 ends the loop through newError <= error_tol iff error_tol >= 0.  So the loop is certain to end
// iff absolute_error_tol >= 0 or (relative_error_tol > 0 and error_tol >= 0), or error_tol is +inf (no finite error
// starts the loop, and it ends after one pass at a non-finite one); NaN fails each comparison.
constexpr double LM_MAX_CLIMB = 1e4;
inline bool lm_params_usable(dynoba_lm_params& P) {
  if (!(std::isfinite(P.lambda_initial) && P.lambda_initial > 0.0) || !(std::isfinite(P.lambda_factor) && P.lambda_factor > 1.0) ||
      std::isnan(P.lambda_upper_bound)) return false;
  if (!(P.absolute_error_tol >= 0.0 || (P.relative_error_tol > 0.0 && P.error_tol >= 0.0) || P.error_tol == INFINITY)) return false;
  if (!(P.lambda_lower_bound >= DBL_MIN)) P.lambda_lower_bound = DBL_MIN;
  const double lo = std::min(P.lambda_initial, P.lambda_lower_bound), hi = std::min(P.lambda_upper_bound, DBL_MAX);
  return !(hi > lo && std::log(hi) - std::log(lo) > LM_MAX_CLIMB*std::log(P.lambda_factor));
}

// defaultOptimize: whether the loop runs at all (errorTol, then maxIterations; a NaN error runs)
__host__ __device__ inline bool lm_starts(double err, const dynoba_lm_params& P) {
  return !(err <= P.error_tol) && P.max_iterations > 0;
}

// checkConvergence (NonlinearOptimizer.cpp), relativeErrorTol tested as a bool as GTSAM does (NaN counts as set)
__host__ __device__ inline bool lm_converged(double currentError, double newError, const dynoba_lm_params& P) {
  if (newError <= P.error_tol) return true;
  return ((P.relative_error_tol != 0.0) && ((currentError - newError)/currentError <= P.relative_error_tol)) ||
         ((currentError - newError) <= P.absolute_error_tol);
}

// the do ... while condition of defaultOptimize after an outer iteration
__host__ __device__ inline bool lm_continues(int iterations, double currentError, double newError, const dynoba_lm_params& P) {
  return iterations < P.max_iterations && !lm_converged(currentError, newError, P) && isfinite(currentError);
}

// tryLambda on one trial.  solved: the damped system was positive definite; oldLin = linear.error(0); lin = the
// linearised cost decrease; err = the current error; nerr = the error at the candidate (read only for a valid step:
// solved, lin finite and >= 0).  A non-finite lin counts as a failed solve.
struct LmDecision { bool success, stop; };
__host__ __device__ inline LmDecision lm_decide(bool solved, double oldLin, double lin, double err, double nerr, const dynoba_lm_params& P) {
  LmDecision d{false, false};
  if (solved && isfinite(lin) && lin >= 0) {
    const double cost = err - nerr;
    if (lin > DBL_EPSILON*oldLin) { const double fid = cost/lin; d.success = fid > P.min_model_fidelity; }
    if (fabs(cost) < P.relative_error_tol*err) d.stop = true;
  }
  return d;
}

// The state change that follows a decision (decreaseLambda / increaseLambda); true when tryLambda returns: a step was
// accepted, the search stopped, or lambda reached its upper bound.  The caller moves to the candidate on d.success.
__host__ __device__ inline bool lm_update(LmDecision d, double nerr, const dynoba_lm_params& P, double& lambda, double& err,
                                          int& iterations, int& inner) {
  if (d.success) { lambda = fmax(P.lambda_lower_bound, lambda/P.lambda_factor); err = nerr; iterations++; inner++; return true; }
  if (!d.stop) { lambda *= P.lambda_factor; inner++; return lambda >= P.lambda_upper_bound; }
  return true;
}

}  // namespace dynoba
