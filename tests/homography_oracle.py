"""CPU restatement of cv::findHomography(src, dst, RANSAC, thr) (TEST INFRASTRUCTURE, NOT PRODUCT).

KltFeatureTracker::geometricVerification (dynosam/src/frontend/vision/StaticFeatureTracker.cc:627-639) calls
cv::findHomography(good_old, good_new, cv::RANSAC, 5.0, mask).  OpenCV's sources are not vendored by the reference, so what
follows is a restatement, pinned operation by operation against cv2 by tests/test_homography.py:

1. draws: cv::RNG((uint64)-1), multiply-with-carry state = (uint32)state * 4164903690 + (state >> 32), next() = (uint32)state,
   uniform(0, n) = next() % n.  A group is 4 distinct indices; a duplicate is re-drawn at once.  The split of the stream into
   groups does not depend on the subset test.  An iteration takes groups until one passes the subset test; 10 000 rejected
   groups in a row end the loop (and fail the run in its first iteration).
2. subset test: haveCollinearPoints on either set (triples with the last point; float differences, double products, against
   FLT_EPSILON * (|dx1| + |dy1| + |dx2| + |dy2|)) rejects, and the four triples {012, 123, 023, 013} must have
   det(A) det(B) < 0 all or none (3x3 determinants by cofactors of the first row, in double).
3. model (HomographyEstimatorCallback::runKernel): centroid and mean absolute deviation with sequential double sums, LtL over
   the upper triangle summed in point order, cv::eigen (OpenCV's Jacobi, below), the eigenvector of the smallest eigenvalue,
   invHnorm * H0 * Hnorm2 (3x3 products, sums left to right), times 1 / H22.  No model when a deviation is below DBL_EPSILON.
4. error: H cast to float, ww = 1 / (H6 x + H7 y + 1), dx = (H0 x + H1 y + H2) ww - x', dy likewise, err = dx dx + dy dy in
   float; an inlier when err <= (float)(thr * thr).
5. loop: a model becomes the best when its count > max(best, 3); then niters = RANSACUpdateNumIters(conf, (n - count) / n, 4,
   niters) (pow, log, cvRound); the loop runs while iter < niters, and an iteration without a model still counts.
6. after RANSAC: the inliers are compressed in order, runKernel runs over all of them, an 8-parameter Levenberg-Marquardt
   (OpenCV 4's LMSolver: lambda = 10^lg, lg from -3, down one on success and up one on failure, within [-16, 16];
   (A + lambda diag A) d = J^T r; at most 10 successful steps; stop when |d|_inf < FLT_EPSILON or S < FLT_EPSILON^2) refines
   H, which is scaled by 1 / H22, and the returned mask is err(H_final) <= thr^2 over all points.  OpenCV's own 8x8 solve is
   not restated: the normal equations are summed in the kernel's fixed block order and solved by its Cholesky (refine below),
   so the device must equal this restatement bit for bit, and it agrees with cv2 to 1e-6 relative where the LM converges.
7. exactly 4 points: runKernel only, mask all ones (all zeros without a model); RANSAC failed: no H, mask all zeros.

Every floating-point operation is a plain IEEE operation in the order written, which is the order frontend.cu's
hom_ransac_kernel evaluates with contraction off.  Only pow / log of step 5 come from different libraries on the two sides
(the LM's lambdas are computed by the C library on both: the kernel receives them from the host); the margins returned here
let tests prove a difference is one of those last bits.
Only tests/ may import this module.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

TOO_FEW, FOUR_POINT, RANSAC_FAILED, OK = 1, 2, 3, 0      # dynofront_homography_status
M32 = 0xFFFFFFFF
FLT_EPS = float(np.finfo(np.float32).eps)
DBL_EPS = float(np.finfo(np.float64).eps)
DBL_MIN = float(np.finfo(np.float64).tiny)
MAX_ATTEMPTS = 10000
CHUNK = 256


# ---- step 1: cv::RNG ------------------------------------------------------------------------------------------------------
class RNG:
    def __init__(self, state=(1 << 64) - 1):
        self.s = state

    def next(self) -> int:
        self.s = ((self.s & M32)*4164903690 + (self.s >> 32)) & ((1 << 64) - 1)
        return self.s & M32


def draw_groups(rng: RNG, n: int, count: int) -> np.ndarray:
    """the next `count` groups of 4 distinct indices in [0, n), duplicates re-drawn at once (RANSACPointSetRegistrator::getSubset)"""
    out = np.empty((count, 4), np.int64)
    for g in range(count):
        i = 0
        while i < 4:
            k = rng.next() % n
            if k in out[g, :i]:
                continue
            out[g, i] = k; i += 1
    return out


# ---- step 2: checkSubset --------------------------------------------------------------------------------------------------
def _collinear(p):
    """haveCollinearPoints(ms, 4) on p[G, 4, 2] float32: triples (j, k, 3), k < j"""
    bad = np.zeros(p.shape[0], bool)
    for j in range(3):
        dx1 = (p[:, j, 0] - p[:, 3, 0]).astype(np.float64); dy1 = (p[:, j, 1] - p[:, 3, 1]).astype(np.float64)
        for k in range(j):
            dx2 = (p[:, k, 0] - p[:, 3, 0]).astype(np.float64); dy2 = (p[:, k, 1] - p[:, 3, 1]).astype(np.float64)
            bad |= np.abs(dx2*dy1 - dy2*dx1) <= FLT_EPS*(((np.abs(dx1) + np.abs(dy1)) + np.abs(dx2)) + np.abs(dy2))
    return bad


def _det3(a0, a1, a2):
    """cv::determinant(Matx33d) of rows (x, y, 1)"""
    return (a0[:, 0]*(a1[:, 1]*1.0 - a2[:, 1]*1.0) - a0[:, 1]*(a1[:, 0]*1.0 - a2[:, 0]*1.0)
            + 1.0*(a1[:, 0]*a2[:, 1] - a2[:, 0]*a1[:, 1]))


def check_subset(S, D):
    """S, D [G, 4, 2] float32 -> bool[G]"""
    ok = ~(_collinear(S) | _collinear(D))
    s = S.astype(np.float64); d = D.astype(np.float64)
    neg = np.zeros(S.shape[0], np.int64)
    for t in ((0, 1, 2), (1, 2, 3), (0, 2, 3), (0, 1, 3)):
        neg += (_det3(s[:, t[0]], s[:, t[1]], s[:, t[2]])*_det3(d[:, t[0]], d[:, t[1]], d[:, t[2]]) < 0)
    return ok & ((neg == 0) | (neg == 4))


# ---- step 3: OpenCV's Jacobi eigen solver, vectorised over a batch of symmetric matrices -----------------------------------
def _hypot(a, b):
    a = np.abs(a); b = np.abs(b)
    out = np.zeros_like(a)
    g = a > b
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(g, b/a, a/b)
        v = np.where(g, a*np.sqrt(1 + r*r), b*np.sqrt(1 + r*r))
    out = np.where(g, v, np.where(b > 0, v, 0.0))
    return out


def jacobi(A):
    """cv::eigen(A, W, V) on A[B, n, n] (double, symmetric; the upper triangle is read): W[B, n] descending, V[B, n, n] rows =
    eigenvectors.  JacobiImpl_: pivot by row / column maxima indices, its own hypot, rotations without FMA."""
    A = np.array(A, np.float64, copy=True)
    single = A.ndim == 2
    if single:
        A = A[None]
    B, n, _ = A.shape
    bi = np.arange(B)
    V = np.broadcast_to(np.eye(n), (B, n, n)).copy()
    W = np.array([A[:, k, k] for k in range(n)]).T.copy()
    indR = np.zeros((B, n), np.int64); indC = np.zeros((B, n), np.int64)

    def row_max(idx):            # indR[idx]: argmax |A[idx, m]| over m > idx, first wins
        m = np.full(B, idx + 1); mv = np.abs(A[bi, idx, idx + 1])
        for i in range(idx + 2, n):
            v = np.abs(A[bi, idx, i]); g = mv < v; mv = np.where(g, v, mv); m = np.where(g, i, m)
        return m

    def col_max(idx):            # indC[idx]: argmax |A[m, idx]| over m < idx
        m = np.zeros(B, np.int64); mv = np.abs(A[bi, 0, idx])
        for i in range(1, idx):
            v = np.abs(A[bi, i, idx]); g = mv < v; mv = np.where(g, v, mv); m = np.where(g, i, m)
        return m

    def row_max_b(idx):          # per-batch idx
        m = idx + 1; mv = np.abs(A[bi, idx, np.minimum(idx + 1, n - 1)])
        for i in range(2, n):
            c = idx + i; valid = c < n; cc = np.minimum(c, n - 1)
            v = np.abs(A[bi, idx, cc]); g = valid & (mv < v); mv = np.where(g, v, mv); m = np.where(g, c, m)
        return m

    def col_max_b(idx):
        m = np.zeros(B, np.int64); mv = np.abs(A[bi, 0, idx])
        for i in range(1, n):
            valid = i < idx
            v = np.abs(A[bi, i, idx]); g = valid & (mv < v); mv = np.where(g, v, mv); m = np.where(g, i, m)
        return m

    for k in range(n):
        if k < n - 1:
            indR[:, k] = row_max(k)
        if k > 0:
            indC[:, k] = col_max(k)
    live = np.ones(B, bool) if n > 1 else np.zeros(B, bool)
    for _ in range(n*n*30):
        if not live.any():
            break
        k = np.zeros(B, np.int64); mv = np.abs(A[bi, 0, indR[:, 0]])
        for i in range(1, n - 1):
            v = np.abs(A[bi, i, indR[:, i]]); g = mv < v; mv = np.where(g, v, mv); k = np.where(g, i, k)
        l = indR[bi, k]
        for i in range(1, n):
            v = np.abs(A[bi, indC[:, i], i]); g = mv < v; mv = np.where(g, v, mv); k = np.where(g, indC[:, i], k); l = np.where(g, i, l)
        p = A[bi, k, l]
        live &= ~(np.abs(p) <= DBL_EPS)
        if not live.any():
            break
        y = (W[bi, l] - W[bi, k])*0.5
        t = np.abs(y) + _hypot(p, y)
        s = _hypot(p, t)
        with np.errstate(divide="ignore", invalid="ignore"):
            c = t/s
            s = p/s; t = (p/t)*p
        s = np.where(y < 0, -s, s); t = np.where(y < 0, -t, t)
        L = live
        A[bi[L], k[L], l[L]] = 0
        W[bi[L], k[L]] -= t[L]
        W[bi[L], l[L]] += t[L]

        def rot(r0, c0, r1, c1, sel):
            b = bi[sel]
            a0 = A[b, r0[sel], c0[sel]]; b0 = A[b, r1[sel], c1[sel]]
            cs = c[sel]; ss = s[sel]
            A[b, r0[sel], c0[sel]] = a0*cs - b0*ss
            A[b, r1[sel], c1[sel]] = a0*ss + b0*cs
        for i in range(n):
            ii = np.full(B, i)
            rot(ii, k, ii, l, L & (i < k))
            rot(k, ii, ii, l, L & (i > k) & (i < l))
            rot(k, ii, l, ii, L & (i > l))
            b = bi[L]
            a0 = V[b, k[L], i]; b0 = V[b, l[L], i]
            V[b, k[L], i] = a0*c[L] - b0*s[L]
            V[b, l[L], i] = a0*s[L] + b0*c[L]
        for idx in (k, l):
            upd = L & (idx < n - 1)
            if upd.any():
                r = row_max_b(np.minimum(idx, n - 2))
                indR[bi[upd], idx[upd]] = r[upd]
            upd = L & (idx > 0)
            if upd.any():
                cmx = col_max_b(idx)
                indC[bi[upd], idx[upd]] = cmx[upd]
    for k in range(n - 1):           # selection sort, descending, first maximum wins, swaps rows of V
        m = np.full(B, k); wm = W[bi, k].copy()
        for i in range(k + 1, n):
            g = wm < W[:, i]; m = np.where(g, i, m); wm = np.where(g, W[:, i], wm)
        sw = m != k
        if sw.any():
            b = bi[sw]; mm = m[sw]
            wk = W[b, k].copy(); W[b, k] = W[b, mm]; W[b, mm] = wk
            vk = V[b, k, :].copy(); V[b, k, :] = V[b, mm, :]; V[b, mm, :] = vk
    return (W[0], V[0]) if single else (W, V)


# ---- step 3: runKernel ----------------------------------------------------------------------------------------------------
def _mm3(a, b):
    """3x3 products, each entry (a0 b0 + a1 b1) + a2 b2"""
    out = np.empty(np.broadcast_shapes(a.shape, b.shape))
    for i in range(3):
        for j in range(3):
            out[..., i, j] = (a[..., i, 0]*b[..., 0, j] + a[..., i, 1]*b[..., 1, j]) + a[..., i, 2]*b[..., 2, j]
    return out


def ltl(M, m):
    """centroids, deviations and LtL of runKernel for point sets M, m [G, k, 2] float32 (sums sequential in point order).
    Returns (LtL [G, 9, 9] symmetric, cM, cm, sM, sm [G, 2], ok [G])."""
    M = M.astype(np.float64); m = m.astype(np.float64)
    cnt = M.shape[1]
    cm = np.cumsum(m, axis=1)[:, -1]/cnt; cM = np.cumsum(M, axis=1)[:, -1]/cnt
    sm = np.cumsum(np.abs(m - cm[:, None]), axis=1)[:, -1]; sM = np.cumsum(np.abs(M - cM[:, None]), axis=1)[:, -1]
    ok = ~((np.abs(sm) < DBL_EPS).any(1) | (np.abs(sM) < DBL_EPS).any(1))
    with np.errstate(divide="ignore"):
        sm = cnt/sm; sM = cnt/sM
    x = (m[..., 0] - cm[:, None, 0])*sm[:, None, 0]; y = (m[..., 1] - cm[:, None, 1])*sm[:, None, 1]
    X = (M[..., 0] - cM[:, None, 0])*sM[:, None, 0]; Y = (M[..., 1] - cM[:, None, 1])*sM[:, None, 1]
    one = np.ones_like(X); zero = np.zeros_like(X)
    Lx = [X, Y, one, zero, zero, zero, -x*X, -x*Y, -x]
    Ly = [zero, zero, zero, X, Y, one, -y*X, -y*Y, -y]
    L = np.zeros((M.shape[0], 9, 9))
    for j in range(9):
        for k in range(j, 9):
            L[:, j, k] = np.cumsum(Lx[j]*Lx[k] + Ly[j]*Ly[k], axis=1)[:, -1]
            L[:, k, j] = L[:, j, k]
    return L, cM, cm, sM, sm, ok


def run_kernel(M, m):
    """HomographyEstimatorCallback::runKernel on point sets M, m [G, k, 2] float32: (H [G, 3, 3], ok [G], LtL)"""
    L, cM, cm, sM, sm, ok = ltl(M, m)
    G = M.shape[0]
    Ls = np.where(ok[:, None, None], L, np.eye(9))
    _, V = jacobi(Ls)
    H0 = V[:, 8, :].reshape(G, 3, 3)
    inv = np.zeros((G, 3, 3)); inv[:, 0, 0] = 1./sm[:, 0]; inv[:, 0, 2] = cm[:, 0]; inv[:, 1, 1] = 1./sm[:, 1]; inv[:, 1, 2] = cm[:, 1]; inv[:, 2, 2] = 1
    h2 = np.zeros((G, 3, 3)); h2[:, 0, 0] = sM[:, 0]; h2[:, 0, 2] = -cM[:, 0]*sM[:, 0]; h2[:, 1, 1] = sM[:, 1]; h2[:, 1, 2] = -cM[:, 1]*sM[:, 1]; h2[:, 2, 2] = 1
    H = _mm3(_mm3(inv, H0), h2)
    H = H*(1./H[:, 2, 2])[:, None, None]
    return H, ok, L


# ---- step 4: computeError -------------------------------------------------------------------------------------------------
def errors(H, M, m):
    """float errors of H [G, 3, 3] (or [3, 3]) over all points: [G, n]"""
    H = np.asarray(H, np.float64)
    single = H.ndim == 2
    Hf = H.reshape(-1, 9).astype(np.float32)[:, :, None]
    x = M[None, :, 0].astype(np.float32); y = M[None, :, 1].astype(np.float32)
    one = np.float32(1)
    with np.errstate(all="ignore"):
        ww = one/((Hf[:, 6]*x + Hf[:, 7]*y) + one)
        dx = ((Hf[:, 0]*x + Hf[:, 1]*y) + Hf[:, 2])*ww - m[None, :, 0]
        dy = ((Hf[:, 3]*x + Hf[:, 4]*y) + Hf[:, 5])*ww - m[None, :, 1]
        e = dx*dx + dy*dy
    return e[0] if single else e


# ---- step 5: RANSACUpdateNumIters -----------------------------------------------------------------------------------------
def update_num_iters(p, ep, model_points, max_iters):
    """returns (niters, margin): margin = distance of num/denom from a cvRound tie (inf where no rounding is involved)"""
    p = min(max(p, 0.), 1.); ep = min(max(ep, 0.), 1.)
    num = max(1. - p, DBL_MIN)
    denom = 1. - math.pow(1. - ep, model_points)
    if denom < DBL_MIN:
        return 0, math.inf
    num = math.log(num); denom = math.log(denom)
    if denom >= 0 or -num >= max_iters*(-denom):
        return max_iters, abs(-num - max_iters*(-denom))/max(abs(num), 1e-300)
    q = num/denom
    return int(np.rint(q)), abs(abs(q - math.floor(q)) - 0.5)


# ---- step 6: Levenberg-Marquardt refinement -------------------------------------------------------------------------------
THREADS, WARPS = 256, 8                           # hom_ransac_kernel's block


def lm_lambdas():
    """lambda = exp(lg * log(10.)) for lg in [-16, 16] from the C library, as OpenCV's LMSolver computes it; the kernel receives
    the same table from the host"""
    return {lg: math.exp(lg*math.log(10.)) for lg in range(-16, 17)}


def block_sum(contrib):
    """hom_block_sum over per-point contributions contrib[m, rows, NV]: thread t adds the rows of points t, t + 256, ... in order,
    each warp reduces by xor butterflies (16, 8, 4, 2, 1) and thread 0 adds the warps' lane-0 values in warp order"""
    m, rows, nv = contrib.shape
    acc = np.zeros((THREADS, nv))
    for r0 in range(0, m, THREADS):
        k = min(THREADS, m - r0)
        for row in range(rows):
            acc[:k] = acc[:k] + contrib[r0:r0 + k, row]
    x = acc.reshape(WARPS, 32, nv)
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        x = x + x[:, lane ^ o]
    tot = x[0, 0].copy()
    for w in range(1, WARPS):
        tot = tot + x[w, 0]
    return tot


def _lm_rows(h, M, m):
    """HomographyRefineCallback::compute per correspondence: residual rows and Jacobian rows, [m, 2] and [m, 2, 8]"""
    Mx = M[:, 0].astype(np.float64); My = M[:, 1].astype(np.float64)
    ww = (h[6]*Mx + h[7]*My) + 1.
    with np.errstate(divide="ignore"):
        ww = np.where(np.abs(ww) > DBL_EPS, 1./ww, 0.)
    xi = ((h[0]*Mx + h[1]*My) + h[2])*ww
    yi = ((h[3]*Mx + h[4]*My) + h[5])*ww
    r = np.stack([xi - m[:, 0].astype(np.float64), yi - m[:, 1].astype(np.float64)], 1)
    J = np.zeros((len(Mx), 2, 8))
    J[:, 0, 0] = Mx*ww; J[:, 0, 1] = My*ww; J[:, 0, 2] = ww; J[:, 0, 6] = -Mx*ww*xi; J[:, 0, 7] = -My*ww*xi
    J[:, 1, 3] = Mx*ww; J[:, 1, 4] = My*ww; J[:, 1, 5] = ww; J[:, 1, 6] = -Mx*ww*yi; J[:, 1, 7] = -My*ww*yi
    return r, J


_UPPER = [(a, b) for a in range(8) for b in range(a, 8)]


def _normal_eq(h, M, m):
    """J^T J (upper triangle, row-major), J^T r and S summed as the kernel sums them"""
    r, J = _lm_rows(h, M, m)
    c = np.empty((len(r), 2, 45))
    for e, (a, b) in enumerate(_UPPER):
        c[:, :, e] = J[:, :, a]*J[:, :, b]
    for a in range(8):
        c[:, :, 36 + a] = J[:, :, a]*r
    c[:, :, 44] = r*r
    tot = block_sum(c)
    A = np.zeros((8, 8))
    for e, (a, b) in enumerate(_UPPER):
        A[a, b] = A[b, a] = tot[e]
    return A, tot[36:44].copy(), float(tot[44])


def _cholesky_solve(A, v, lam):
    """(A + lambda diag A) d = v by the kernel's Cholesky: sequential sums, an unusable pivot gives 0"""
    L = [[float(A[i, j]) for j in range(8)] for i in range(8)]
    for a in range(8):
        L[a][a] *= 1 + lam
    for j in range(8):
        s = L[j][j]
        for k in range(j):
            s -= L[j][k]*L[j][k]
        lj = math.sqrt(max(s, 0.0)); L[j][j] = lj
        for i in range(j + 1, 8):
            q = L[i][j]
            for k in range(j):
                q -= L[i][k]*L[j][k]
            L[i][j] = q/lj if lj > 0 else 0.
    d = [0.]*8
    for i in range(8):
        q = float(v[i])
        for k in range(i):
            q -= L[i][k]*d[k]
        d[i] = q/L[i][i] if L[i][i] > 0 else 0.
    for i in range(7, -1, -1):
        q = d[i]
        for k in range(i + 1, 8):
            q -= L[k][i]*d[k]
        d[i] = q/L[i][i] if L[i][i] > 0 else 0.
    return np.array(d)


def refine(H, M, m, max_iters=10):
    """The 8-parameter Levenberg-Marquardt of cv::findHomography's refinement with OpenCV 4's LMSolver control (lambda = 10^lg,
    lg from -3, down one on success, up one on failure, within [-16, 16]; at most max_iters successful steps; stop when
    |d|_inf < FLT_EPSILON or S < FLT_EPSILON^2), then H / H22.  The normal equations are summed in the kernel's block order and
    solved by its Cholesky, so this is the device's arithmetic bit for bit (OpenCV's own solve is not restated: the refined H
    agrees with cv2 to 1e-6 relative where the LM converges).  Returns (H, steps, evaluations)."""
    lam_of = lm_lambdas()
    x = np.asarray(H, np.float64).reshape(9).copy()
    A, v, S = _normal_eq(x, M, m)
    lg = -3; it = 0; evals = 0
    while True:
        d = _cholesky_solve(A, v, lam_of[lg])
        xd = x.copy(); xd[:8] = x[:8] - d
        rd, _ = _lm_rows(xd, M, m)
        Sd = float(block_sum((rd*rd)[:, :, None])[0]); evals += 1
        if Sd < S:
            lg = max(lg - 1, -16); it += 1
            x = xd; A, v, S = _normal_eq(x, M, m)
        else:
            it += lg == 16
            lg = min(lg + 1, 16)
        if not (it < max_iters and np.abs(d).max() >= FLT_EPS and S >= FLT_EPS*FLT_EPS):
            break
    s = 1./x[8] if abs(x[8]) > FLT_EPS else 1.
    return (x*s).reshape(3, 3), it, evals


# ---- the whole call -------------------------------------------------------------------------------------------------------
@dataclass
class Result:
    status: int
    H: np.ndarray | None = None
    mask: np.ndarray | None = None                 # the returned mask (u8)
    ransac_mask: np.ndarray | None = None
    H_ransac: np.ndarray | None = None
    groups: int = 0                                 # groups of 4 drawn
    rejected: int = 0                               # groups the subset test rejected
    iterations: int = 0
    counts: list = field(default_factory=list)      # inlier count of each model, in iteration order (-1: no model)
    best: int = -1                                  # iteration of the best model
    niters_margin: float = np.inf                   # smallest cvRound / cap margin of the niters updates
    margin: np.ndarray | None = None                # |err(H_final) - thr^2| per point
    ransac_margin: float = np.inf                   # smallest |err - thr^2| over every model's counted errors

    @property
    def n_inliers(self):
        return int(self.mask.sum()) if self.mask is not None else 0


def find_homography(src, dst, thr=5.0, confidence=0.995, max_iters=2000, refine_model=True):
    """cv2.findHomography(src, dst, cv2.RANSAC, thr, maxIters=max_iters, confidence=confidence) with its trace.  With fewer than 4
    points: KltFeatureTracker::geometricVerification's all-ones mask (status TOO_FEW).  refine_model=False returns the RANSAC
    model and mask."""
    M = np.ascontiguousarray(src, np.float32).reshape(-1, 2); m = np.ascontiguousarray(dst, np.float32).reshape(-1, 2)
    n = len(M)
    t = np.float32(thr*thr)
    if n < 4:
        return Result(TOO_FEW, None, np.ones(n, np.uint8))
    if n == 4:
        H, ok, _ = run_kernel(M[None], m[None])
        if not ok[0]:
            return Result(FOUR_POINT, None, np.zeros(n, np.uint8))
        mk = np.ones(n, np.uint8)
        return Result(FOUR_POINT, H[0], mk, mk.copy(), H[0])
    res = Result(RANSAC_FAILED)
    rng = RNG()
    niters = max(max_iters, 1); it = 0; best_count = 0; best_mask = None; best_H = None
    run = 0                                    # rejected groups in a row
    fail = False
    chunk = 0
    while it < niters and not fail:
        nch = min(CHUNK, 32 << min(chunk, 3)); chunk += 1          # the device's chunk sizes (the result does not depend on them)
        g = draw_groups(rng, n, nch)
        passed = check_subset(M[g], m[g])
        # models of the passing groups of this chunk
        pi = np.nonzero(passed)[0]
        Hs, oks, _ = run_kernel(M[g[pi]], m[g[pi]]) if len(pi) else (None, None, None)
        errs = errors(Hs, M, m) if len(pi) else None
        j = 0
        for q in range(nch):
            res.groups += 1
            if not passed[q]:
                res.rejected += 1; run += 1
                if run >= MAX_ATTEMPTS:
                    if it == 0:
                        fail = True
                    else:
                        niters = it             # break
                    break
                continue
            run = 0
            if oks[j]:
                e = errs[j]
                cnt = int((e <= t).sum())
                res.ransac_margin = min(res.ransac_margin, float(np.abs(e.astype(np.float64) - float(t)).min()))
                res.counts.append(cnt)
                if cnt > max(best_count, 3):
                    best_count = cnt; best_mask = (e <= t).astype(np.uint8); best_H = Hs[j]; res.best = it
                    niters, mg = update_num_iters(confidence, (n - cnt)/n, 4, niters)
                    res.niters_margin = min(res.niters_margin, mg)
            else:
                res.counts.append(-1)
            j += 1
            it += 1
            if it >= niters:
                break
    res.iterations = it
    if fail or best_count == 0:
        res.iterations = 0 if fail else it
        res.mask = np.zeros(n, np.uint8)
        return res
    res.status = OK; res.ransac_mask = best_mask; res.H_ransac = best_H
    if not refine_model:
        res.H = best_H; res.mask = best_mask
        return res
    sel = best_mask.astype(bool)
    H, _, _ = run_kernel(M[sel][None], m[sel][None])
    H, _, _ = refine(H[0], M[sel], m[sel])
    res.H = H
    e = errors(H, M, m)
    res.mask = (e <= t).astype(np.uint8)
    res.margin = np.abs(e.astype(np.float64) - float(t))
    return res


# ---- the parity set -------------------------------------------------------------------------------------------------------
def make_problem(seed, n, outlier_frac, noise=1.0, kind="plain"):
    """a KLT-like correspondence set: src in a 1242 x 375 image, dst = a near-identity homography of src plus noise, the first
    outlier_frac of the points moved by tens of pixels.  kind: "collinear" puts most points on three lines (subset rejections),
    "duplicate" repeats a few points many times, "identical" makes every point the same (RANSAC fails)."""
    r = np.random.default_rng(seed)
    a = (r.random((n, 2))*[1242, 375]).astype(np.float64)
    if kind == "collinear":
        k = int(n*0.8); t = r.random(k); line = r.integers(0, 3, k)
        a[:k, 0] = 100 + 1000*t; a[:k, 1] = np.choose(line, [50 + 0*t, 150 + 0.1*(1000*t), 300 - 0.2*(1000*t)])
    if kind == "duplicate":
        a = a[r.integers(0, max(n//8, 2), n)]
    if kind == "identical":
        a[:] = a[0]
    H0 = np.array([[1 + r.normal(0, .01), r.normal(0, .01), r.normal(0, 5)], [r.normal(0, .01), 1 + r.normal(0, .01), r.normal(0, 5)],
                   [r.normal(0, 1e-5), r.normal(0, 1e-5), 1]])
    w = a @ H0[2, :2] + H0[2, 2]
    b = np.stack([(a @ H0[0, :2] + H0[0, 2])/w, (a @ H0[1, :2] + H0[1, 2])/w], 1)
    if kind != "identical":
        b += r.normal(0, noise, b.shape)
    k = int(n*outlier_frac)
    b[:k] += r.normal(0, 40, (k, 2))
    return a.astype(np.float32), b.astype(np.float32)


def parity_set(size="full"):
    """[(name, src, dst, max_iters)]: n from 5 to 20 000, 0-70 % outliers, max_iters in {1, 2, 3, 5, 2000}, collinear and
    duplicated points, and all points identical.  size="small" keeps a quick subset."""
    out = []
    r = np.random.default_rng(2024)
    sizes = [5, 6, 7, 9, 12, 20, 40, 100, 300, 800, 2000, 1200, 5000]
    iters = [1, 2, 3, 5, 2000]
    seed = 0
    for n in sizes:
        for mi in iters:
            for frac in (0.0, 0.3, 0.7):
                if size == "small" and (seed % 4):
                    seed += 1; continue
                a, b = make_problem(seed, n, frac if n > 6 else 0.0)
                out.append((f"n{n}_it{mi}_out{int(frac*100)}_s{seed}", a, b, mi)); seed += 1
    for kind, n in (("collinear", 60), ("collinear", 400), ("duplicate", 7), ("duplicate", 30), ("duplicate", 200)):
        for mi in (3, 2000):
            a, b = make_problem(seed, n, 0.2, kind=kind)
            out.append((f"{kind}_n{n}_it{mi}_s{seed}", a, b, mi)); seed += 1
    a, b = make_problem(seed, 50, 0.0, kind="identical"); out.append((f"identical_n50_s{seed}", a, b, 2000)); seed += 1
    if size != "small":
        for frac in (0.05, 0.3, 0.6):
            a, b = make_problem(seed, 20000, frac); out.append((f"n20000_out{int(frac*100)}_s{seed}", a, b, 2000)); seed += 1
    del r
    return out


# problems of parity_set("full") on which cv2's returned mask differs from this restatement's, named by tests/test_homography.py
CV2_LM_DIFFERENCES = ("n800_it3_out70_s143", "collinear_n400_it3_s197", "duplicate_n200_it3_s203")
