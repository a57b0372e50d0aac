"""CPU restatement of cv::findFundamentalMat(p1, p2, FM_RANSAC, thr, conf, maxIters) (TEST INFRASTRUCTURE, NOT PRODUCT).

FeatureTracker::stereoTrack (dynosam/src/frontend/vision/FeatureTracker.cc:279-281) calls
cv::findFundamentalMat(left, right, cv::FM_RANSAC, 1.0, 0.99, mask), so maxIters is 1000.  OpenCV's sources are not vendored by
the reference, so what follows is a restatement, pinned against cv2 4.13 by tests/test_fundamental.py:

1. draws: homography_oracle's cv::RNG((uint64)-1) stream, groups of 7 distinct indices with duplicates re-drawn at once.  The
   subset test is haveCollinearPoints on either set (triples (j, k, 6), k < j < 6), as the homography's first half (on the parity
   set the masks are the same with and without it, so cv2 does not yet tell the two apart); 10 000
   rejected groups in a row end a RANSAC loop, 1000 an LMedS loop (and fail it in its first iteration).
2. model (run7Point): centroids with sequential double sums times 1/7, mean distance (sqrt(dx^2 + dy^2), times 1/7), no model
   when a mean distance is below FLT_EPSILON, scale = sqrt(2) / mean; the 7x9 system solved by SVDecomp(MODIFY_A | FULL_UV),
   which is OpenCV's one-sided Jacobi SVD (JacobiSVDImpl_: sequential dot products, OpenCV's hypot, 30 sweeps at most, eps
   10 DBL_EPSILON) on the transposed problem.  The two rows of Vt beyond the rank are completed from cv::RNG(0x12345678): a
   +-1/9 vector, twice Gram-Schmidt against the earlier rows with L1 renormalisation, then L2 normalisation.  f1 = Vt[7] - Vt[8],
   f2 = Vt[8], the determinant cubic, cv::solveCubic (below); per root in its order: lambda / mu scaling where
   |f1[8] r + f2[8]| > DBL_EPSILON, F = (T2^T F) T1 with Matx products, then F * (1 / F22) where |F22| > FLT_EPSILON.
3. solveCubic as cv2 4.13 computes it (solve_cubic below, equal to cv2.solveCubic bit for bit): the coefficients count as all
   zero (-1 roots) when max|a_i| < DBL_EPSILON, and leading coefficients below DBL_EPSILON of the largest count as zero.  A
   7-point cubic with -1 roots is what makes cv2 raise (-215, rowRange(0, -3) in FMEstimatorCallback::runKernel) inside
   findFundamentalMat, e.g. on raising_problem(), whose collinear points under a pure shift give coefficients near 1e-16.
   The restatement and the device treat such a draw as one without a model, which is defined where the reference is not.
4. error (computeError): the larger of the two squared point-to-epipolar-line distances in double (std::max(a, b) = a < b ? b :
   a), stored as float; an inlier when err <= (float)(thr * thr).
5. RANSAC (n >= 15): each draw gives 0-3 models, evaluated in root order; a model becomes the best when count > max(best, 6),
   then niters = RANSACUpdateNumIters(conf, (n - count) / n, 7, niters).  A draw without a model still counts as an iteration.
6. LMedS (8 <= n < 15): niters = max(RANSACUpdateNumIters(conf, 0.45, 7, maxIters), 3); a model's score is the (n/2)-th
   smallest float error (nth_element over the floats' bit patterns); a strictly smaller median replaces the best.  After the
   loop sigma = max(2.5 * 1.4826 * (1 + 5 / (n - 7)) * sqrt(median), 0.001), the mask is err <= (float)(sigma^2) and success
   needs at least 7 inliers.  thr is ignored on this path.
7. exactly 7 points: run7Point only, all-ones mask, up to 3 models; fewer than 7: no model.  A failed RANSAC / LMedS leaves
   cv2's mask unwritten (uninitialised memory); the restatement defines it as all zeros.

Every floating-point operation is a plain IEEE operation in the order written, which is the order frontend.cu's
fund_ransac_kernel evaluates with contraction off.  acos / cos / pow of solveCubic and pow / log of the stopping rule come from
different libraries on the two sides; the per-iteration margins returned here and explain_F (which replays a model with those
results moved by up to 2 ulp) let tests prove a difference is one of those last bits.
Only tests/ may import this module.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

from homography_oracle import RNG, update_num_iters

OK, LMEDS, SEVEN_POINT, TOO_FEW, FAILED = 0, 1, 2, 3, 4      # dynofront_fundamental_status
M32 = 0xFFFFFFFF
FLT_EPS = float(np.finfo(np.float32).eps)
DBL_EPS = float(np.finfo(np.float64).eps)
DBL_MIN = float(np.finfo(np.float64).tiny)
RANSAC_ATTEMPTS, LMEDS_ATTEMPTS = 10000, 1000
CHUNK = 128


# ---- step 1: draws and the subset test ------------------------------------------------------------------------------------
def draw_groups(rng: RNG, n: int, count: int, k: int = 7) -> np.ndarray:
    out = np.empty((count, k), np.int64)
    for g in range(count):
        i = 0
        while i < k:
            v = rng.next() % n
            if v in out[g, :i]:
                continue
            out[g, i] = v; i += 1
    return out


def collinear(p):
    """haveCollinearPoints(ms, K) on p[G, K, 2] float32: triples (j, k, K-1), k < j"""
    K = p.shape[1]
    bad = np.zeros(p.shape[0], bool)
    for j in range(K - 1):
        dx1 = (p[:, j, 0] - p[:, K - 1, 0]).astype(np.float64); dy1 = (p[:, j, 1] - p[:, K - 1, 1]).astype(np.float64)
        for k in range(j):
            dx2 = (p[:, k, 0] - p[:, K - 1, 0]).astype(np.float64); dy2 = (p[:, k, 1] - p[:, K - 1, 1]).astype(np.float64)
            bad |= np.abs(dx2*dy1 - dy2*dx1) <= FLT_EPS*(((np.abs(dx1) + np.abs(dy1)) + np.abs(dx2)) + np.abs(dy2))
    return bad


# ---- step 2: OpenCV's one-sided Jacobi SVD of a 7x9 system, vectorised over a batch ----------------------------------------
def cv_hypot(a, b):
    a = np.abs(a); b = np.abs(b)
    with np.errstate(all="ignore"):
        ga = a*np.sqrt(1 + (b/a)*(b/a)); gb = b*np.sqrt(1 + (a/b)*(a/b))
    return np.where(a > b, ga, np.where(b > 0, gb, 0.0))


def _dot(a, b):
    s = np.zeros(a.shape[:-1])
    for k in range(a.shape[-1]):
        s = s + a[..., k]*b[..., k]
    return s


def _complete_row(U, i, rng_state, m=9):
    """JacobiSVDImpl_'s completion of row i of U (float list of lists): returns the new RNG state"""
    eps = DBL_EPS*10
    s = rng_state
    sd = 0.0
    for _ in range(100):
        val0 = 1./m
        for k in range(m):
            s = ((s & M32)*4164903690 + (s >> 32)) & ((1 << 64) - 1)
            U[i][k] = val0 if (s & M32) & 256 else -val0
        for _ in range(2):
            for j in range(i):
                sd = 0.0
                for k in range(m):
                    sd += U[i][k]*U[j][k]
                asum = 0.0
                for k in range(m):
                    t = U[i][k] - sd*U[j][k]; U[i][k] = t; asum += abs(t)
                asum = 1/asum if asum > eps*100 else 0.0
                for k in range(m):
                    U[i][k] *= asum
        sd = 0.0
        for k in range(m):
            sd += U[i][k]*U[i][k]
        sd = math.sqrt(sd)
        if sd > DBL_MIN:
            break
    sc = 1/sd if sd > DBL_MIN else 0.0
    for k in range(m):
        U[i][k] *= sc
    return s


def svd_vt(A):
    """cv::SVDecomp(A, W, U, Vt, FULL_UV) of A [B, 7, 9] (or [7, 9]): Vt [B, 9, 9]"""
    A = np.asarray(A, np.float64)
    single = A.ndim == 2
    if single:
        A = A[None]
    B = A.shape[0]
    m, n = 9, 7
    At = np.array(A, copy=True)
    eps = DBL_EPS*10
    W = np.stack([_dot(At[:, i], At[:, i]) for i in range(n)], 1)
    for _ in range(max(m, 30)):
        changed = False
        for i in range(n - 1):
            for j in range(i + 1, n):
                a = W[:, i]; b = W[:, j]
                p = _dot(At[:, i], At[:, j])
                go = ~(np.abs(p) <= eps*np.sqrt(a*b))
                if not go.any():
                    continue
                changed = True
                p = p*2
                beta = a - b; gamma = cv_hypot(p, beta)
                with np.errstate(all="ignore"):
                    delta = (gamma - beta)*0.5
                    sn = np.sqrt(delta/gamma); cn = p/((gamma*sn)*2)
                    cp = np.sqrt((gamma + beta)/(gamma*2)); sp = p/((gamma*cp)*2)
                c = np.where(beta < 0, cn, cp)[:, None]; s = np.where(beta < 0, sn, sp)[:, None]
                Ai = At[:, i]; Aj = At[:, j]
                t0 = c*Ai + s*Aj
                t1 = -s*Ai + c*Aj
                g = go[:, None]
                At[:, i] = np.where(g, t0, Ai); At[:, j] = np.where(g, t1, Aj)
                W[:, i] = np.where(go, _dot(t0, t0), W[:, i]); W[:, j] = np.where(go, _dot(t1, t1), W[:, j])
        if not changed:
            break
    W = np.sqrt(np.stack([_dot(At[:, i], At[:, i]) for i in range(n)], 1))
    bi = np.arange(B)
    for i in range(n - 1):               # selection sort, descending, first maximum wins
        jj = np.full(B, i)
        for k in range(i + 1, n):
            jj = np.where(W[bi, jj] < W[:, k], k, jj)
        sw = jj != i
        if sw.any():
            b = bi[sw]; j2 = jj[sw]
            wi = W[b, i].copy(); W[b, i] = W[b, j2]; W[b, j2] = wi
            ai = At[b, i].copy(); At[b, i] = At[b, j2]; At[b, j2] = ai
    out = np.empty((B, 9, 9))
    for b in range(B):
        U = [list(map(float, At[b, i])) for i in range(n)] + [[0.0]*m for _ in range(m - n)]
        st = 0x12345678
        for i in range(m):
            sd = float(W[b, i]) if i < n else 0.0
            if sd <= DBL_MIN:
                st = _complete_row(U, i, st)
            else:
                sc = 1/sd
                U[i] = [u*sc for u in U[i]]
        out[b] = U
    return out[0] if single else out


# ---- step 3: cv::solveCubic -----------------------------------------------------------------------------------------------
def _acos(x):
    return math.acos(x) if -1. <= x <= 1. else math.nan           # C acos: NaN outside [-1, 1]


_ULPS = [0, 0]            # explain_F: steps of the acos result and of the cos / pow results (0: the C library's values)


def _shift(v, k):
    for _ in range(abs(k)):
        v = float(np.nextafter(v, math.inf if k > 0 else -math.inf))
    return v


def _div(a, b):
    with np.errstate(all="ignore"):
        return float(np.float64(a)/np.float64(b))                  # IEEE: x / 0 is +-inf or NaN


def _sqrt(x):
    return math.sqrt(x) if x >= 0 or math.isnan(x) else math.nan


def solve_cubic(c):
    """cv::solveCubic (OpenCV 4.13) of c = (a0, a1, a2, a3): (n, [x0, x1, x2], margin).  Every coefficient is 0 (n = -1) when
    max|a_i| < DBL_EPSILON; a coefficient with |a_i * (1 / max|a_j|)| < DBL_EPSILON counts as 0.  Then the classic branches:
    a0 == 0 falls to the quadratic, the linear or the constant case on the unscaled coefficients; otherwise the cubic branch
    works on the coefficients times 1 / max|a_j|, and the monic cubic's discriminant d picks three trigonometric roots (d > 0), the
    repeated-root form (d == 0) or one real root.  margin: |d| of the monic cubic, the distance from the branch boundary (inf on
    the a0 == 0 branches, which need no libm)."""
    a0, a1, a2, a3 = (float(v) for v in c)
    x0 = x1 = x2 = 0.0
    margin = math.inf
    m = max(abs(a0), abs(a1), abs(a2), abs(a3))
    if not m >= DBL_EPS:
        return -1, [x0, x1, x2], margin
    inv = 1./m
    small = lambda v: abs(v*inv) < DBL_EPS                          # noqa: E731
    if not small(a0):                                               # the cubic branch works on the scaled coefficients
        a0, a1, a2, a3 = (v*inv for v in (a0, a1, a2, a3))
    else:                                                           # the zero test cascades down the leading coefficients only
        a0 = 0.0
        if small(a1):
            a1 = 0.0
            if small(a2):
                a2 = 0.0
                if small(a3):
                    a3 = 0.0
    if a0 == 0:
        if a1 == 0:
            if a2 == 0:
                n = -1 if a3 == 0 else 0
            else:
                x0 = _div(-a3, a2); n = 1
        else:
            d = a2*a2 - 4*a1*a3
            n = 0
            if d >= 0:
                d = math.sqrt(d)
                q1 = (-a2 + d)*0.5
                q2 = (a2 + d)*-0.5
                if abs(q1) > abs(q2):
                    x0 = _div(q1, a1); x1 = _div(a3, q1)
                else:
                    x0 = _div(q2, a1); x1 = _div(a3, q2)
                n = 2 if d > 0 else 1
    else:
        a0 = 1./a0
        a1 *= a0; a2 *= a0; a3 *= a0
        Q = (a1*a1 - 3*a2)*(1./9)
        R = (a1*(2*a1*a1 - 9*a2) + 27*a3)*(1./54)
        Qcubed = Q*Q*Q
        d = (a1*a1*(a2*a2 - 4*a1*a3) + 2*a2*(9*a1*a3 - 2*a2*a2) - 27*a3*a3)*(1./108)
        margin = abs(d)
        if d > 0:
            theta = _shift(_acos(_div(R, _sqrt(Qcubed))), _ULPS[0])
            sqrtQ = _sqrt(Q)
            t0 = -2*sqrtQ
            t1 = theta*(1./3)
            t2 = a1*(1./3)
            x0 = t0*_shift(math.cos(t1), _ULPS[1]) - t2
            x1 = t0*_shift(math.cos(t1 + (2.*math.pi/3)), _ULPS[1]) - t2
            x2 = t0*_shift(math.cos(t1 + (4.*math.pi/3)), _ULPS[1]) - t2
            n = 3
        elif d == 0:
            if R >= 0:
                x0 = -2*_shift(math.pow(R, 1./3), _ULPS[1]) - a1/3
                x1 = _shift(math.pow(R, 1./3), _ULPS[1]) - a1/3
            else:
                x0 = 2*_shift(math.pow(-R, 1./3), _ULPS[1]) - a1/3
                x1 = -_shift(math.pow(-R, 1./3), _ULPS[1]) - a1/3
            x2 = 0
            n = 1 if x0 == x1 else 2
            x1 = 0 if x0 == x1 else x1
        else:
            d = math.sqrt(-d)
            e = _shift(math.pow(d + abs(R), 1./3), _ULPS[1])
            if R > 0:
                e = -e
            x0 = (e + _div(Q, e)) - a1*(1./3)
            n = 1
    return n, [x0, x1, x2], margin


# ---- step 2: run7Point ----------------------------------------------------------------------------------------------------
def _mm3(a, b):
    out = [[0.0]*3 for _ in range(3)]
    for i in range(3):
        for j in range(3):
            s = 0.0
            for k in range(3):
                s += a[i][k]*b[k][j]
            out[i][j] = s
    return out


def normalise(M, m):
    """run7Point's centroids and scales of M, m [G, 7, 2] float32 -> rows A [G, 7, 9], (c1, s1, c2, s2), ok [G]"""
    P1 = M.astype(np.float64); P2 = m.astype(np.float64)
    K = P1.shape[1]
    t = 1./K
    c1 = np.zeros((P1.shape[0], 2)); c2 = np.zeros_like(c1)
    for i in range(K):
        c1 = c1 + P1[:, i]; c2 = c2 + P2[:, i]
    c1 = c1*t; c2 = c2*t
    s1 = np.zeros(P1.shape[0]); s2 = np.zeros_like(s1)
    for i in range(K):
        d = P1[:, i] - c1; s1 = s1 + np.sqrt(d[:, 0]*d[:, 0] + d[:, 1]*d[:, 1])
        d = P2[:, i] - c2; s2 = s2 + np.sqrt(d[:, 0]*d[:, 0] + d[:, 1]*d[:, 1])
    s1 = s1*t; s2 = s2*t
    ok = ~((s1 < FLT_EPS) | (s2 < FLT_EPS))
    with np.errstate(divide="ignore"):
        s1 = np.where(ok, math.sqrt(2.)/s1, 1.0); s2 = np.where(ok, math.sqrt(2.)/s2, 1.0)
    x0 = (P1[..., 0] - c1[:, None, 0])*s1[:, None]; y0 = (P1[..., 1] - c1[:, None, 1])*s1[:, None]
    x1 = (P2[..., 0] - c2[:, None, 0])*s2[:, None]; y1 = (P2[..., 1] - c2[:, None, 1])*s2[:, None]
    A = np.stack([x1*x0, x1*y0, x1, y1*x0, y1*y0, y1, x0, y0, np.ones_like(x0)], -1)
    return A, (c1, s1, c2, s2), ok


def _cubic_coeffs(f1, f2):
    t0 = f2[4]*f2[8] - f2[5]*f2[7]
    t1 = f2[3]*f2[8] - f2[5]*f2[6]
    t2 = f2[3]*f2[7] - f2[4]*f2[6]
    c3 = f2[0]*t0 - f2[1]*t1 + f2[2]*t2
    c2 = (f1[0]*t0 - f1[1]*t1 + f1[2]*t2 - f1[3]*(f2[1]*f2[8] - f2[2]*f2[7]) + f1[4]*(f2[0]*f2[8] - f2[2]*f2[6])
          - f1[5]*(f2[0]*f2[7] - f2[1]*f2[6]) + f1[6]*(f2[1]*f2[5] - f2[2]*f2[4]) - f1[7]*(f2[0]*f2[5] - f2[2]*f2[3])
          + f1[8]*(f2[0]*f2[4] - f2[1]*f2[3]))
    t0 = f1[4]*f1[8] - f1[5]*f1[7]
    t1 = f1[3]*f1[8] - f1[5]*f1[6]
    t2 = f1[3]*f1[7] - f1[4]*f1[6]
    c1 = (f2[0]*t0 - f2[1]*t1 + f2[2]*t2 - f2[3]*(f1[1]*f1[8] - f1[2]*f1[7]) + f2[4]*(f1[0]*f1[8] - f1[2]*f1[6])
          - f2[5]*(f1[0]*f1[7] - f1[1]*f1[6]) + f2[6]*(f1[1]*f1[5] - f1[2]*f1[4]) - f2[7]*(f1[0]*f1[5] - f1[2]*f1[3])
          + f2[8]*(f1[0]*f1[4] - f1[1]*f1[3]))
    c0 = f1[0]*t0 - f1[1]*t1 + f1[2]*t2
    return (c0, c1, c2, c3)


def run7(M, m):
    """run7Point on draws M, m [G, 7, 2] float32: per draw (n, [F 3x3 ...], cubic margin).  n = -1: all-zero cubic (cv2 raises);
    n = 0: no model."""
    G = M.shape[0]
    A, (c1, s1, c2, s2), ok = normalise(M, m)
    Vt = svd_vt(np.where(ok[:, None, None], A, 0.0)) if G else np.zeros((0, 9, 9))
    out = []
    for g in range(G):
        if not ok[g]:
            out.append((0, [], math.inf)); continue
        f2 = [float(v) for v in Vt[g, 8]]
        f1 = [float(Vt[g, 7, i]) - f2[i] for i in range(9)]
        n, r, mg = solve_cubic(_cubic_coeffs(f1, f2))
        if n < 1 or n > 3:
            out.append((n, [], mg)); continue
        sc1 = float(s1[g]); sc2 = float(s2[g])
        T1 = [[sc1, 0., -sc1*float(c1[g, 0])], [0., sc1, -sc1*float(c1[g, 1])], [0., 0., 1.]]
        T2t = [[sc2, 0., 0.], [0., sc2, 0.], [-sc2*float(c2[g, 0]), -sc2*float(c2[g, 1]), 1.]]
        Fs = []
        for k in range(n):
            lam = r[k]; mu = 1.
            s = f1[8]*r[k] + f2[8]
            fm = [0.0]*9
            if abs(s) > DBL_EPS:
                mu = 1./s; lam *= mu; fm[8] = 1.
            else:
                fm[8] = 0.
            for i in range(8):
                fm[i] = f1[i]*lam + f2[i]*mu
            F = _mm3(_mm3(T2t, [fm[0:3], fm[3:6], fm[6:9]]), T1)
            if abs(F[2][2]) > FLT_EPS:
                inv = 1./F[2][2]
                F = [[v*inv for v in row] for row in F]
            Fs.append(np.array(F))
        out.append((n, Fs, mg))
    return out


# ---- step 4: computeError -------------------------------------------------------------------------------------------------
def errors(F, M, m):
    """float errors of F [3, 3] over all points [n]"""
    F = np.asarray(F, np.float64).reshape(9)
    x1 = M[:, 0].astype(np.float64); y1 = M[:, 1].astype(np.float64)
    x2 = m[:, 0].astype(np.float64); y2 = m[:, 1].astype(np.float64)
    with np.errstate(all="ignore"):
        a = (F[0]*x1 + F[1]*y1) + F[2]; b = (F[3]*x1 + F[4]*y1) + F[5]; c = (F[6]*x1 + F[7]*y1) + F[8]
        s2 = 1./(a*a + b*b); d2 = (x2*a + y2*b) + c
        a = (F[0]*x2 + F[3]*y2) + F[6]; b = (F[1]*x2 + F[4]*y2) + F[7]; c = (F[2]*x2 + F[5]*y2) + F[8]
        s1 = 1./(a*a + b*b); d1 = (x1*a + y1*b) + c
        e1 = (d1*d1)*s1; e2 = (d2*d2)*s2
        e = np.where(e1 < e2, e2, e1)
    return e.astype(np.float32)


def median_of(e):
    """nth_element over the int32 bit patterns: the (n/2)-th smallest"""
    bits = np.sort(e.view(np.int32))
    return float(bits[len(e)//2:len(e)//2 + 1].view(np.float32)[0])


# ---- the whole call -------------------------------------------------------------------------------------------------------
@dataclass
class Result:
    status: int
    F: list = field(default_factory=list)           # returned models (1 except SEVEN_POINT)
    mask: np.ndarray | None = None
    groups: int = 0                                 # groups of 7 drawn
    rejected: int = 0                               # groups the subset test rejected
    iterations: int = 0
    models: list = field(default_factory=list)      # models per iteration (-1: an all-zero cubic)
    scores: list = field(default_factory=list)      # every model's inlier count (RANSAC) or median (LMedS), in (draw, root) order
    best: tuple = (-1, -1)                          # (iteration, root) of the best model
    success: bool = False                           # LMedS: at least 7 final inliers
    niters_margin: float = math.inf
    score_margin: float = math.inf                  # smallest |err - thr^2| over every counted error (RANSAC)
    cubic_margin: float = math.inf                  # smallest |discriminant| of the drawn cubics
    raised: int = -1                                # first iteration whose cubic is all zeros (cv2 raises there)
    draws: list = field(default_factory=list)       # the 7 indices of each iteration's group
    draw_margins: list = field(default_factory=list)   # |discriminant| of each iteration's cubic (inf: no libm branch)
    model_margins: list = field(default_factory=list)  # per model in (draw, root) order: min |err - thr^2| (RANSAC)

    @property
    def n_inliers(self):
        return int(self.mask.sum()) if self.mask is not None else 0


def find_fundamental(src, dst, thr=1.0, confidence=0.99, max_iters=1000, chunk=CHUNK):
    """cv2.findFundamentalMat(src, dst, cv2.FM_RANSAC, thr, confidence, max_iters) with its trace"""
    M = np.ascontiguousarray(src, np.float32).reshape(-1, 2); m = np.ascontiguousarray(dst, np.float32).reshape(-1, 2)
    n = len(M)
    if n < 7:
        return Result(TOO_FEW, mask=np.zeros(n, np.uint8))
    if n == 7:
        (k, Fs, mg), = run7(M[None], m[None])
        res = Result(SEVEN_POINT, F=Fs, mask=np.ones(n, np.uint8) if Fs else np.zeros(n, np.uint8), cubic_margin=mg)
        res.models = [k]; res.raised = 0 if k == -1 else -1
        return res
    lmeds = n < 15
    res = Result(LMEDS if lmeds else OK)
    rng = RNG()
    t = np.float32(thr*thr)
    if lmeds:
        niters = max(update_num_iters(confidence, 0.45, 7, max_iters)[0], 3)
        attempts = LMEDS_ATTEMPTS
    else:
        niters = max(max_iters, 1)
        attempts = RANSAC_ATTEMPTS
    it = 0; best = 0; best_med = math.inf; best_F = None; best_mask = None
    run = 0; fail = False; done = False
    while not done:
        g = draw_groups(rng, n, chunk)
        passed = ~(collinear(M[g]) | collinear(m[g]))
        pi = np.nonzero(passed)[0]
        models = dict(zip(pi.tolist(), run7(M[g[pi]], m[g[pi]]))) if len(pi) else {}
        for q in range(chunk):
            res.groups += 1
            if not passed[q]:
                res.rejected += 1; run += 1
                if run >= attempts:
                    done = True; fail = it == 0
                    break
                continue
            run = 0
            k, Fs, mg = models[q]
            res.models.append(k); res.cubic_margin = min(res.cubic_margin, mg)
            res.draws.append(g[q].copy()); res.draw_margins.append(mg)
            if k == -1 and res.raised < 0:
                res.raised = it
            for r, F in enumerate(Fs):
                e = errors(F, M, m)
                if lmeds:
                    med = median_of(e)
                    res.scores.append(med)
                    if med < best_med:
                        best_med = med; best_F = F; res.best = (it, r)
                else:
                    inl = e <= t
                    cnt = int(inl.sum())
                    res.scores.append(cnt)
                    mm = float(np.abs(e.astype(np.float64) - float(t)).min())
                    res.score_margin = min(res.score_margin, mm); res.model_margins.append(mm)
                    if cnt > max(best, 6):
                        best = cnt; best_F = F; best_mask = inl.astype(np.uint8); res.best = (it, r)
                        niters, mg2 = update_num_iters(confidence, (n - cnt)/n, 7, niters)
                        res.niters_margin = min(res.niters_margin, mg2)
            it += 1
            if it >= niters:
                done = True
                break
    res.iterations = 0 if fail else it
    if fail or best_F is None:
        res.status = FAILED
        res.mask = np.zeros(n, np.uint8)
        return res
    res.F = [best_F]
    if lmeds:
        sigma = 2.5*1.4826*(1 + 5./(n - 7))*math.sqrt(best_med)
        sigma = max(sigma, 0.001)
        ts = np.float32(sigma*sigma)
        e = errors(best_F, M, m)
        res.mask = (e <= ts).astype(np.uint8)
        res.score_margin = float(np.abs(e.astype(np.float64) - float(ts)).min())
        res.success = int(res.mask.sum()) >= 7
    else:
        res.mask = best_mask
        res.success = True
    return res


def explain_F(src, dst, group, root, F_dev, max_ulps=2):
    """True when run7Point on the 7 points `group`, with its acos result and its cos / pow results each moved by at most
    max_ulps units in the last place (CUDA's libm bounds for acos, cos and pow are 2 ulp), gives F_dev bit for bit as model
    `root`: the proof that a device F differs from this restatement only through the C library's transcendental functions."""
    M = np.ascontiguousarray(src, np.float32).reshape(-1, 2)[group][None]
    m = np.ascontiguousarray(dst, np.float32).reshape(-1, 2)[group][None]
    try:
        for ka in range(-max_ulps, max_ulps + 1):
            for kc in range(-max_ulps, max_ulps + 1):
                _ULPS[:] = [ka, kc]
                n, Fs, _ = run7(M, m)[0]
                if root < len(Fs) and np.array_equal(Fs[root], np.asarray(F_dev).reshape(3, 3)):
                    return True
    finally:
        _ULPS[:] = [0, 0]
    return False


# ---- the parity set -------------------------------------------------------------------------------------------------------
def _project(X, R, tvec, f=700., cx=620., cy=187.):
    Y = X @ R.T + tvec
    return np.stack([f*Y[:, 0]/Y[:, 2] + cx, f*Y[:, 1]/Y[:, 2] + cy], 1)


def make_problem(seed, n, outlier_frac, kind="general", noise=0.3):
    """a two-view correspondence set in a 1242 x 375 image.  kind: "general" (a rotated and translated second camera), "stereo"
    (a rectified pair: a pure 0.5 m x shift), "planar" (every point on one plane), "duplicate" (a few points repeated many times),
    "identical" (every point the same).  The first outlier_frac of the points move by tens of pixels."""
    r = np.random.default_rng(seed)
    X = np.stack([r.uniform(-8, 8, n), r.uniform(-2, 2, n), r.uniform(4, 40, n)], 1)
    if kind == "planar":
        X[:, 2] = 12 + 0.3*X[:, 0] + 0.5*X[:, 1]
    if kind == "stereo":
        R = np.eye(3); tv = np.array([-0.5, 0., 0.])
    else:
        w = r.normal(0, 0.03, 3); th = np.linalg.norm(w); kx = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
        R = np.eye(3) + math.sin(th)/th*kx + (1 - math.cos(th))/th**2*(kx @ kx)
        tv = np.array([r.normal(0, .5), r.normal(0, .1), r.normal(0, .5)])
    a = _project(X, np.eye(3), np.zeros(3)); b = _project(X, R, tv)
    if kind == "duplicate":
        i = r.integers(0, max(n//8, 2), n); a = a[i]; b = b[i]
    if kind == "identical":
        a[:] = a[0]; b[:] = b[0]
    else:
        a += r.normal(0, noise, a.shape); b += r.normal(0, noise, b.shape)
    k = int(n*outlier_frac)
    b[:k] += r.normal(0, 30, (k, 2))
    return a.astype(np.float32), b.astype(np.float32)


def parity_set(size="full"):
    """[(name, src, dst, max_iters)]: n in {8, 9, 14, 15, 16, 31-33, 255-257, 800, 2700, 20000}, 0-70 % outliers, max_iters in
    {1, 2, 3, 5, 1000}, general two-view, rectified stereo and planar scenes, duplicated and identical points.  size="small"
    keeps a quick subset."""
    out = []
    seed = 0
    sizes = [8, 9, 14, 15, 16, 31, 32, 33, 255, 256, 257, 800, 2700]
    kinds = ["general", "stereo", "planar"]
    for n in sizes:
        for mi in (1, 2, 3, 5, 1000):
            for frac in (0.0, 0.3, 0.7):
                kind = kinds[seed % 3]
                if size == "small" and seed % 5:
                    seed += 1; continue
                a, b = make_problem(seed, n, frac, kind)
                out.append((f"{kind}_n{n}_it{mi}_out{int(frac*100)}_s{seed}", a, b, mi)); seed += 1
    for kind, n in (("duplicate", 9), ("duplicate", 30), ("duplicate", 300)):
        for mi in (3, 1000):
            a, b = make_problem(seed, n, 0.2, kind)
            out.append((f"{kind}_n{n}_it{mi}_s{seed}", a, b, mi)); seed += 1
    for n in (10, 50):
        a, b = make_problem(seed, n, 0.0, "identical"); out.append((f"identical_n{n}_s{seed}", a, b, 1000)); seed += 1
    if size != "small":
        for frac in (0.05, 0.3, 0.6):
            a, b = make_problem(seed, 20000, frac, "general"); out.append((f"general_n20000_out{int(frac*100)}_s{seed}", a, b, 1000))
            seed += 1
    return out


def raising_problem():
    """20 points, 16 of them on one horizontal line, under a pure 9 px shift: cv2.findFundamentalMat raises (-215) at the first
    draw whose 7-point cubic is all zeros"""
    r = np.random.default_rng(7)
    a = np.zeros((20, 2), np.float32)
    a[:16, 0] = np.round(r.uniform(50, 1200, 16)); a[:16, 1] = 200
    a[16:] = np.round(r.uniform([50, 20], [1200, 360], (4, 2)))
    b = a.copy(); b[:, 0] -= 9
    return a, b
