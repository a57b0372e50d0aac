// lm_control_host.cu -- the LM decisions of dynosam_b200/csrc/lm_control.cuh compiled for the host, so that
// tests/test_lm_control.py can drive them with scripted trial scalars on a machine without a GPU.
#include <cstdint>
#include "lm_control.cuh"

using namespace dynoba;

extern "C" {
// lm_params_usable on a copy of *P; the copy (lower bound raised) is written to *out
int host_lm_params_usable(const dynoba_lm_params* P, dynoba_lm_params* out) {
  dynoba_lm_params Q = *P;
  const int ok = lm_params_usable(Q) ? 1 : 0;
  *out = Q;
  return ok;
}
int host_lm_converged(double currentError, double newError, const dynoba_lm_params* P) { return lm_converged(currentError, newError, *P) ? 1 : 0; }
// one decision: out = {success, stop}
void host_lm_decide(int solved, double oldLin, double lin, double err, double nerr, const dynoba_lm_params* P, int* out) {
  const LmDecision d = lm_decide(solved != 0, oldLin, lin, err, nerr, *P);
  out[0] = d.success; out[1] = d.stop;
}
// The loop of run_lm (kernels_star.cu) and dynoba_optimize (api.cu) with the trial scalars taken from script[n][4] =
// (solved, oldLin, lin, nerr), the last row repeated once the script is used up, and at most cap trials.  rows[cap][10]
// receives one dynoba_get_lm_trace row per trial.  out = {iterations, inner, trials, ended (0: stopped by the cap)},
// outd = {lambda_final, error_final}.
void host_lm_run(const dynoba_lm_params* Pp, double err0, const double* script, int n, int64_t cap, double* rows,
                 int64_t* out, double* outd) {
  const dynoba_lm_params P = *Pp;
  double err = err0, lambda = P.lambda_initial;
  int its = 0, inner = 0; int64_t t = 0; int ended = 1;
  if (lm_starts(err, P)) {
    double newError = err, currentError;
    do {
      currentError = newError;
      for (;;) {
        if (t >= cap) { ended = 0; break; }
        const double* s = script + 4*(t < n ? t : n - 1);
        const bool solved = s[0] != 0.0;
        const LmDecision d = lm_decide(solved, s[1], s[2], err, s[3], P);
        double* r = rows + 10*t;
        r[0] = its; r[1] = inner; r[2] = lambda; r[3] = s[1]; r[4] = s[2]; r[5] = err; r[6] = s[3]; r[7] = solved; r[8] = d.success; r[9] = d.stop;
        t++;
        if (lm_update(d, s[3], P, lambda, err, its, inner)) break;
      }
      if (!ended) break;
      newError = err;
    } while (lm_continues(its, currentError, newError, P));
  }
  out[0] = its; out[1] = inner; out[2] = t; out[3] = ended;
  outd[0] = lambda; outd[1] = err;
}
}
