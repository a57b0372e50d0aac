"""GTSAM 4.2.0's Levenberg-Marquardt control restated in Python, and the two scalars each of its decisions is made from,
computed exactly from the device's own linear system.

replay(trials, error0, P)
    A literal restatement of NonlinearOptimizer::defaultOptimize, LevenbergMarquardtOptimizer::iterate / tryLambda and
    checkConvergence (NonlinearOptimizer.cpp), with useFixedLambdaFactor (the project's only mode).  It is fed, per
    trial, what the linear solve and the error evaluation returned (solved, oldLin, lin, nerr) and re-derives every
    decision from them: success and stopSearchingLambda, the lambda of every trial, (iterations, inner), lambda_final,
    the final error and why the loop ended.  It is written from GTSAM, not from csrc/lm_control.cuh.  Two points are the
    project's own and are stated here as such: a non-finite lin counts as a failed solve (GTSAM's
    IndeterminantLinearSystemException), and lambda_lower_bound is raised to DBL_MIN (``effective``).

Exact model scalars (``ExactModel``)
    From the whitened J, b of every factor block (``Solver.linearization``), the step delta (``Solver.solve``) and the
    dense priors' G, g, f:
        oldLin = linear.error(0) = 1/2 |b|^2 + sum over priors of error(0) of the relinearised HessianFactor
        C(delta) = 1/2 g^T delta + 1/2 lambda |delta|^2,  g = J^T b (+ the priors' g - G d)     (what the device sums)
        L(delta) = linear.error(0) - linear.error(delta)                                      (what GTSAM evaluates)
    Every product is split error-free (Dekker's TwoProduct, vectorised) and the parts are summed by math.fsum, so each
    value is the correctly rounded exact value of its expression in the fp64 inputs.  ``terms`` is the sum of the
    absolute values of the summed products, the a-priori scale of a summation's rounding: a sum of those terms in any
    order is within (n - 1) u terms of the exact value.  C - L = 1/2 delta^T ((H + lambda I) delta - g) exactly
    (difference (i) in DESIGN.md section 4): zero for the exact solution of the damped system.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from fractions import Fraction

import numpy as np
import scipy.sparse as sp

from dynosam_b200.problem import CLASS_DIM, DIM, SLOT_CLASS

DBL_EPSILON = 2.0**-52
DBL_MIN = 2.2250738585072014e-308
U = 2.0**-53
TRACE_COLS = ("iterations", "inner", "lambda", "oldLin", "lin", "err", "nerr", "solved", "success", "stop")
PARAM_NAMES = ("lambda_initial", "lambda_factor", "lambda_upper_bound", "lambda_lower_bound", "min_model_fidelity",
               "relative_error_tol", "absolute_error_tol", "error_tol", "max_iterations")


def params(P=None, **kw):
    """a plain dict of LM parameters from a binding.LmParams, a dict, or GTSAM 4.2.0's defaults, with overrides"""
    d = dict(lambda_initial=1e-5, lambda_factor=10.0, lambda_upper_bound=1e5, lambda_lower_bound=0.0,
             min_model_fidelity=1e-3, relative_error_tol=1e-5, absolute_error_tol=1e-5, error_tol=0.0, max_iterations=100)
    if P is not None:
        d.update({k: (P[k] if isinstance(P, dict) else getattr(P, k)) for k in PARAM_NAMES})
    d.update(kw)
    return d


def effective(P):
    """the parameters as the library runs them: lambda_lower_bound raised to DBL_MIN (include/dynoba.h)"""
    P = dict(P)
    if not (P["lambda_lower_bound"] >= DBL_MIN):
        P["lambda_lower_bound"] = DBL_MIN
    return P


# ------------------------------------------------------------------------------------------------ GTSAM 4.2.0, restated
def check_convergence(relativeErrorTreshold, absoluteErrorTreshold, errorThreshold, currentError, newError):
    """NonlinearOptimizer.cpp checkConvergence; returns (converged, which test)"""
    if newError <= errorThreshold:
        return True, "error_tol"
    absoluteDecrease = currentError - newError
    with np.errstate(all="ignore"):
        relativeDecrease = float(np.float64(absoluteDecrease)/np.float64(currentError))
    if bool(relativeErrorTreshold) and relativeDecrease <= relativeErrorTreshold:   # `relativeErrorTreshold &&`: NaN is true
        return True, "relative"
    if absoluteDecrease <= absoluteErrorTreshold:
        return True, "absolute"
    return False, None


@dataclass
class Replay:
    rows: list            # per trial: (iterations, inner, lambda, err, success, stop)
    iterations: int
    inner: int
    lambda_final: float
    error_final: float
    reason: str           # "error_tol", "max_iterations", "relative", "absolute", "nonfinite", "cap"
    exits: list           # how each tryLambda loop ended: "accepted", "stop", "giveup"


def replay(trials, error0, P, cap=None):
    """trials: sequence of (solved, oldLin, lin, nerr), consumed in order (or a callable t -> that tuple).  cap: the
    largest number of trials to run; past it the result has reason "cap" (the loop had not ended)."""
    get = trials if callable(trials) else (lambda t: trials[t])
    lam, err, iterations, inner = P["lambda_initial"], error0, 0, 0
    rows, exits = [], []

    def result(reason):
        return Replay(rows, iterations, inner, lam, err, reason, exits)

    # defaultOptimize
    currentError = err
    if currentError <= P["error_tol"]:
        return result("error_tol")
    if iterations >= P["max_iterations"]:
        return result("max_iterations")
    newError = currentError
    while True:
        currentError = newError
        # iterate(): while (!tryLambda(...))
        while True:
            if cap is not None and len(rows) >= cap:
                return result("cap")
            solved, oldLin, lin, nerr = get(len(rows))
            # tryLambda
            systemSolvedSuccessfully = bool(solved) and math.isfinite(lin)
            step_is_successful = stopSearchingLambda = False
            if systemSolvedSuccessfully:
                oldLinearizedError, linearizedCostChange = oldLin, lin
                if linearizedCostChange >= 0:
                    newError_t = nerr
                    costChange = err - newError_t
                    if linearizedCostChange > DBL_EPSILON*oldLinearizedError:
                        with np.errstate(all="ignore"):
                            modelFidelity = float(np.float64(costChange)/np.float64(linearizedCostChange))
                        step_is_successful = modelFidelity > P["min_model_fidelity"]
                    minAbsoluteTolerance = P["relative_error_tol"]*err
                    if abs(costChange) < minAbsoluteTolerance:
                        stopSearchingLambda = True
            rows.append((iterations, inner, lam, err, step_is_successful, stopSearchingLambda))
            if step_is_successful:
                # decreaseLambda, then State(newValues, newError, lambda, iterations + 1, totalNumberInnerIterations + 1)
                lam = max(P["lambda_lower_bound"], float(np.float64(lam)/np.float64(P["lambda_factor"])))
                err = nerr
                iterations += 1
                inner += 1
                exits.append("accepted")
                break
            elif not stopSearchingLambda:
                lam *= P["lambda_factor"]          # increaseLambda
                inner += 1
                if lam >= P["lambda_upper_bound"]:
                    exits.append("giveup")
                    break
            else:
                exits.append("stop")
                break
        newError = err
        if not iterations < P["max_iterations"]:
            return result("max_iterations")
        conv, which = check_convergence(P["relative_error_tol"], P["absolute_error_tol"], P["error_tol"], currentError, newError)
        if conv:
            return result(which)
        if not math.isfinite(currentError):
            return result("nonfinite")


# ------------------------------------------------------------------------------------------------ error-free arithmetic
_SPLIT = 134217729.0      # 2^27 + 1


def _split(a):
    c = _SPLIT*a
    hi = c - (c - a)
    return hi, a - hi


def two_product(a, b):
    """Dekker's TwoProduct, elementwise: p + e == a*b exactly (no overflow, no underflow below 2^-969)"""
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    p = a*b
    ah, al = _split(a); bh, bl = _split(b)
    e = ((ah*bh - p) + ah*bl + al*bh) + al*bl
    return p, e


def exact_parts(*factors):
    """the products of the factor arrays (broadcast), as a flat array of doubles whose exact sum is the exact sum of the
    products, and the array of |products| (rounded) for the scale"""
    parts = [np.asarray(factors[0], np.float64)]
    for f in factors[1:]:
        nxt = []
        for q in parts:
            p, e = two_product(q, f)
            nxt += [p, e]
        parts = nxt
    mag = np.abs(parts[0])
    return np.concatenate([np.ravel(q) for q in parts]), np.ravel(mag)


def fsum_parts(groups):
    """(exact sum rounded once, sum of |terms|) of several (coefficient, factors...) groups"""
    vals, scale = [], 0.0
    for coef, *fs in groups:
        v, m = exact_parts(*fs)
        vals.append(v*coef)                 # coef is a power of two: exact
        scale += abs(coef)*math.fsum(m)
    return math.fsum(np.concatenate(vals) if vals else []), scale


# ------------------------------------------------------------------------------------------------ the device's linear system
def offsets(p):
    """first column of each variable class in the dynoba_solve layout [poses 6 | points 3 | flows 2 | vel 3 | bias 6]"""
    n = [p.n_pose, p.n_point, p.n_flow, p.n_vel, p.n_bias]
    off = np.concatenate([[0], np.cumsum([n[c]*CLASS_DIM[c] for c in range(5)])])
    return off[:5], int(off[5])


def jacobian(p, jac):
    """stacked whitened J (sparse, dynoba_solve column layout) and b from jac(bi) -> (A[n][dim][jcols], b[n][dim])"""
    off, n = offsets(p)
    rows, cols, vals, rhs = [], [], [], []
    r0 = 0
    for bi, b in enumerate(p.blocks):
        A, bv = jac(bi)
        d = DIM[b.type]
        r = r0 + np.arange(b.n)[:, None]*d + np.arange(d)[None, :]
        c0 = 0
        for k, cls in enumerate(SLOT_CLASS[b.type]):
            w = CLASS_DIM[cls]
            var = off[cls] + w*b.idx[:, k].astype(np.int64)
            for c in range(w):
                rows.append(r.reshape(-1)); cols.append(np.repeat(var + c, d)); vals.append(A[:, :, c0 + c].reshape(-1))
            c0 += w
        rhs.append(bv.reshape(-1))
        r0 += b.n*d
    cat = lambda xs, t: np.concatenate(xs).astype(t) if xs else np.zeros(0, t)
    J = sp.coo_matrix((cat(vals, np.float64), (cat(rows, np.int64), cat(cols, np.int64))), shape=(r0, n))
    return J, cat(rhs, np.float64)


@dataclass
class Prior:
    """a dense prior relinearised with local coordinates d at the current values: HessianFactor(G, g - G d, ...),
    error(0) = 1/2 d^T G d - g^T d + 1/2 f.  cols: its columns in the dynoba_solve layout."""
    cols: np.ndarray
    G: np.ndarray
    g: np.ndarray
    f: float
    d: np.ndarray


def priors_at_lin(p):
    """the problem's dense priors relinearised at their own linearisation point (d = 0)"""
    out = []
    for pr in getattr(p, "linear_priors", []):
        idx = np.asarray(pr["idx"], np.int64)
        cols = (6*idx[:, None] + np.arange(6)[None, :]).reshape(-1)
        out.append(Prior(cols, np.asarray(pr["G"], np.float64).reshape(cols.size, cols.size), np.asarray(pr["g"], np.float64),
                         float(pr.get("f", 0.0)), np.zeros(cols.size)))
    return out


class ExactModel:
    def __init__(self, J, b, priors=()):
        self.J = J.tocoo()
        self.b = b
        self.priors = list(priors)

    def old_lin(self):
        """(linear.error(0) exactly, sum of |terms|)"""
        groups = [(0.5, self.b, self.b)]
        for q in self.priors:
            gi, gj = np.meshgrid(np.arange(q.d.size), np.arange(q.d.size), indexing="ij")
            groups += [(0.5, q.d[gi], q.G, q.d[gj]), (-1.0, q.g, q.d), (0.5, np.array([q.f]))]
        return fsum_parts(groups)

    def model(self, delta, lam):
        """(C(delta) = 1/2 g^T delta + 1/2 lambda |delta|^2 exactly, sum of |terms|)"""
        Jc = self.J
        groups = [(0.5, self.b[Jc.row], Jc.data, delta[Jc.col]), (0.5, np.full(delta.size, lam), delta, delta)]
        for q in self.priors:
            dq = delta[q.cols]
            groups += [(0.5, q.g, dq), (-0.5, dq[:, None], q.G, q.d[None, :])]
        return fsum_parts(groups)

    def _exact(self, delta, lam):
        """(L(delta), 1/2 delta^T ((H + lambda I) delta - g)) in exact rational arithmetic (small systems)"""
        F = Fraction
        Jc = self.J.tocsr()
        x = [F(float(v)) for v in delta]
        Jd = [sum((F(float(Jc.data[k]))*x[Jc.indices[k]] for k in range(Jc.indptr[i], Jc.indptr[i + 1])), F(0))
              for i in range(Jc.shape[0])]
        bb = [F(float(v)) for v in self.b]
        # linear.error(0) - linear.error(delta): 1/2|b|^2 - 1/2|J delta - b|^2 - sum over priors (1/2 x^T G x - gcur^T x)
        L = sum((bi*bi - (ji - bi)**2 for ji, bi in zip(Jd, bb)), F(0))/2
        # H delta - g = J^T (J delta - b) + sum over priors (G x - gcur)
        Hd_g = [F(0)]*len(x)
        for i in range(Jc.shape[0]):
            ri = Jd[i] - bb[i]
            for k in range(Jc.indptr[i], Jc.indptr[i + 1]):
                Hd_g[Jc.indices[k]] += F(float(Jc.data[k]))*ri
        for q in self.priors:
            xq = [x[c] for c in q.cols]
            G = [[F(float(v)) for v in row] for row in q.G]
            gcur = [F(float(q.g[r])) - sum((G[r][c]*F(float(q.d[c])) for c in range(len(xq))), F(0)) for r in range(len(xq))]
            Gx = [sum((G[r][c]*xq[c] for c in range(len(xq))), F(0)) for r in range(len(xq))]
            L -= sum((xq[r]*Gx[r]/2 - gcur[r]*xq[r] for r in range(len(xq))), F(0))
            for r, c in enumerate(q.cols):
                Hd_g[c] += Gx[r] - gcur[r]
        R = sum((x[j]*(Hd_g[j] + F(lam)*x[j]) for j in range(len(x))), F(0))/2
        return L, R

    def literal_decrease(self, delta, lam):
        """GTSAM's L(delta) = linear.error(0) - linear.error(delta), correctly rounded"""
        return float(self._exact(delta, lam)[0])

    def identity_holds(self, delta, lam):
        """C(delta) - L(delta) == 1/2 delta^T ((H + lambda I) delta - g), both sides exact"""
        L, R = self._exact(delta, lam)
        C = self.model_exact(delta, lam)
        return C - L == R

    def model_exact(self, delta, lam):
        """C(delta) as an exact rational"""
        F = Fraction
        Jc = self.J
        C = sum((F(float(self.b[i]))*F(float(v))*F(float(delta[j])) for i, j, v in zip(Jc.row, Jc.col, Jc.data)), F(0))
        C += F(lam)*sum((F(float(v))**2 for v in delta), F(0))
        for q in self.priors:
            for r, c in enumerate(q.cols):
                gcur = F(float(q.g[r])) - sum((F(float(q.G[r, k]))*F(float(q.d[k])) for k in range(q.d.size)), F(0))
                C += gcur*F(float(delta[c]))
        return C/2
