"""A 50-digit reference of the first stage of the solver: the SO(3) / SE(3) maps, every non-IMU factor's residual and
Jacobian, whitening, the Huber weight and chi^2.  Plain mpmath on Python lists, written from the mathematics; it imports
neither the CUDA library nor the CPU oracle.

Two sets of maps:

* the TRUE maps (`exp_so3`, `log_so3`, `exp_se3`, `log_se3`): Rodrigues' formula and its inverse, the closed forms of
  V(omega) and V^-1, each evaluated in 50 digits with a series below theta = 1e-10, where the closed form would cancel;
* the GTSAM 4.2.0 FORMULA maps (`g_exp_so3`, `g_log_so3`, `g_exp_se3`, `g_log_se3`): GTSAM's branch structure (the
  thresholds are the named constants below) with each branch's formula evaluated in 50 digits on the fp64 inputs as
  given -- "what GTSAM computes, without rounding".  This is what the device must equal to rounding.

Error of GTSAM's formulas in exact arithmetic against the true maps (test_factor_cases.py asserts each row):

    branch                               condition                          |formula - true|
    Expmap first order                   theta^2 <= DBL_EPSILON             R: theta^2/2 <= 1.2e-16;  t: theta |v|/2
    Logmap Taylor                        tr - 3 >= -1e-7                    theta^5/30 <= 1.1e-19   
    Logmap acos                          otherwise                          0
    Logmap pi (three sub-branches)       tr + 1 < 1e-10                     ~ (pi - theta)/min(1, 2 |a_k|): the angle is pi exactly,
                                                                            the axis misses the sin(theta) terms; a_k the
                                                                            axis component of the sub-branch
    Pose3 Logmap small angle             |omega| < 1e-10                    |omega| |t|/2

In fp64 the acos branch is ill conditioned towards pi: acos returns theta with an absolute error of about
eps/(pi - theta) and theta/(2 sin theta) divides by sin theta ~ pi - theta, so a faithful evaluation carries
pi eps/(pi - theta)^2, 1e-7 where the pi branch begins.  `log_rot_bound` is that bound.

Jacobians: `jacobian_exact` differentiates a residual through the true retraction by central differences in 50 digits
with step 1e-20 (truncation 1e-40, i.e. the analytic derivative to ~30 digits; it shares nothing with a closed form);
`jacobian_gtsam` is the Jacobian GTSAM 4.2.0 itself uses: I for PriorFactor, (-Ad(hx^-1), I) for BetweenFactor (both
omit the derivative of Logmap), gtsam::numericalDerivative with delta = 1e-5 for the three numerically differentiated
factors (evaluated in 50 digits: the number a fp64 implementation approximates), the exact derivative without the skew
terms for Pose3FlowProjectionFactor (its Jacobian is written for a skew-free camera), and the exact derivative otherwise.
"""
from mpmath import mp, mpf

mp.dps = 50

# GTSAM 4.2.0's branch constants
EPS = mpf(2)**-52                # DBL_EPSILON
EXP_NEAR_ZERO = EPS              # SO3 ExpmapFunctor: theta^2 <= DBL_EPSILON
LOG_PI_TRACE = mpf("1e-10")      # SO3::Logmap: tr + 1 < 1e-10
LOG_PI_DIAG = mpf("1e-5")        # ... |R_kk + 1| > 1e-5 picks the sub-branch
LOG_TAYLOR = mpf("-1e-7")        # ... tr - 3 < -1e-7 -> acos, else Taylor
POSE_LOG_SMALL = mpf("1e-10")    # Pose3::Logmap: |omega| < 1e-10
NUMERIC_DELTA = mpf("1e-5")      # gtsam::numericalDerivative

(PRIOR6, BETWEEN6, POSE2POINT3, STEREO3, TERNARY3, HYBRID3, HYBRID_STEREO3, MOTIONPOSE3, SMOOTH_HYBRID6, SMOOTH_POSE6,
 FLOWPROJ2) = range(11)
NUMERIC_TYPES = (MOTIONPOSE3, SMOOTH_HYBRID6, SMOOTH_POSE6)
# variable class per key slot: 'T' pose, 'p' point, 'f' flow
SLOTS = ["T", "TT", "Tp", "Tp", "ppT", "TTp", "TTp", "ppTT", "TTT", "TTT", "fT"]
SLOT_DIM = {"T": 6, "p": 3, "f": 2}
I3 = [mpf(1), mpf(0), mpf(0), mpf(0), mpf(1), mpf(0), mpf(0), mpf(0), mpf(1)]

# branch recorder: the names of the branches the formula maps took since `trace_start()`, and "close:<map>" for a
# threshold quantity within a factor 2 of its threshold
TRACE = None


def trace_start():
    global TRACE
    TRACE = set()


def trace_stop():
    global TRACE
    t, TRACE = TRACE, None
    return t


def _note(name, q=None, thr=None):
    if TRACE is None:
        return
    TRACE.add(name)
    if q is not None and thr / 2 < abs(q) < 2 * thr:
        TRACE.add("close:" + name.split(":")[0])


def vec(x):
    return [mpf(float(v)) for v in x]


def to_float(x):
    """the one conversion back to float64 (nested lists keep their shape)"""
    if isinstance(x, (list, tuple)):
        return [to_float(v) for v in x]
    return float(x)


# ---- 3x3 algebra on row-major lists
def mul3(A, B):
    return [A[3*i]*B[j] + A[3*i+1]*B[3+j] + A[3*i+2]*B[6+j] for i in range(3) for j in range(3)]


def tr3(A):
    return [A[0], A[3], A[6], A[1], A[4], A[7], A[2], A[5], A[8]]


def mv3(A, v):
    return [A[3*i]*v[0] + A[3*i+1]*v[1] + A[3*i+2]*v[2] for i in range(3)]


def skew(w):
    z = mpf(0)
    return [z, -w[2], w[1], w[2], z, -w[0], -w[1], w[0], z]


def cross(a, b):
    return [a[1]*b[2] - a[2]*b[1], a[2]*b[0] - a[0]*b[2], a[0]*b[1] - a[1]*b[0]]


def dot(a, b):
    return sum(x*y for x, y in zip(a, b))


def norm(a):
    return mp.sqrt(dot(a, a))


def lin3(a, A, b, B, c, C):
    return [a*x + b*y + c*z for x, y, z in zip(A, B, C)]


# ---- true maps
def _abc(th):
    """sin(th)/th, (1 - cos th)/th^2, (th - sin th)/th^3"""
    if th < mpf("1e-10"):
        t2 = th*th
        return 1 - t2/6, mpf(1)/2 - t2/24, mpf(1)/6 - t2/120
    s = mp.sin(th/2)
    return mp.sin(th)/th, 2*s*s/(th*th), (th - mp.sin(th))/th**3


def exp_so3(w):
    th = norm(w); A, B, _ = _abc(th); W = skew(w)
    return lin3(mpf(1), I3, A, W, B, mul3(W, W))


def log_so3(R):
    """principal logarithm of a rotation matrix (theta in [0, pi]); well conditioned at every angle: the angle from atan2,
    the axis from the antisymmetric part below 2 rad and from the symmetric part above"""
    a = [(R[7] - R[5])/2, (R[2] - R[6])/2, (R[3] - R[1])/2]        # sin(theta) axis
    s = norm(a); c = (R[0] + R[4] + R[8] - 1)/2
    th = mp.atan2(s, c)
    if th < 2:
        A, _, _ = _abc(th)
        return [x/A for x in a]
    S = [(R[3*i+j] + R[3*j+i])/2 - (c if i == j else 0) for i in range(3) for j in range(3)]    # (1 - cos) a a^T
    k = max(range(3), key=lambda i: S[4*i])
    ax = [S[3*i+k] for i in range(3)]; n = norm(ax); ax = [x/n for x in ax]
    if dot(ax, a) < 0:
        ax = [-x for x in ax]
    return [th*x for x in ax]


def exp_se3(xi):
    w, v = xi[:3], xi[3:]
    th = norm(w); A, B, C = _abc(th); W = skew(w); WW = mul3(W, W)
    R = lin3(mpf(1), I3, A, W, B, WW)
    V = lin3(mpf(1), I3, B, W, C, WW)
    return (R, mv3(V, v))


def log_se3(P):
    R, t = P
    w = log_so3(R); th = norm(w)
    if th < mpf("1e-10"):
        D = mpf(1)/12 + th*th/720
    else:
        D = (1 - th/(2*mp.tan(th/2)))/(th*th)
    W = skew(w)
    Vi = lin3(mpf(1), I3, -mpf(1)/2, W, D, mul3(W, W))
    return w + mv3(Vi, t)


# ---- group operations on (R, t)
def compose(a, b):
    return (mul3(a[0], b[0]), [x + y for x, y in zip(mv3(a[0], b[1]), a[1])])


def inverse(a):
    Rt = tr3(a[0])
    return (Rt, [-x for x in mv3(Rt, a[1])])


def between(a, b):
    return compose(inverse(a), b)


def retract(T, xi):
    return compose(T, exp_se3(xi))


def act(T, p):
    return [x + y for x, y in zip(mv3(T[0], p), T[1])]


def act_inv(T, p):
    return mv3(tr3(T[0]), [x - y for x, y in zip(p, T[1])])


def adjoint(T):
    """Ad(T) = [[R, 0], [[t]x R, R]] in the [omega; v] order, 6 x 6 as a list of rows"""
    R = T[0]; tR = mul3(skew(T[1]), R); z = mpf(0)
    return [[R[3*i+j] for j in range(3)] + [z]*3 for i in range(3)] + \
           [[tR[3*i+j] for j in range(3)] + [R[3*i+j] for j in range(3)] for i in range(3)]


def pose(x12):
    x = vec(x12)
    return (x[:9], x[9:])


def pose_flat(T):
    return list(T[0]) + list(T[1])


# ---- GTSAM 4.2.0 formula maps, each branch evaluated in 50 digits
def g_exp_so3(w):
    th2 = dot(w, w); W = skew(w)
    if th2 <= EXP_NEAR_ZERO:
        _note("exp:first_order", th2, EXP_NEAR_ZERO)
        return [a + b for a, b in zip(I3, W)]
    _note("exp:full", th2, EXP_NEAR_ZERO)
    th = mp.sqrt(th2); K = [x/th for x in W]; s2 = mp.sin(th/2)
    return lin3(mpf(1), I3, mp.sin(th), K, 2*s2*s2, mul3(K, K))


def g_exp_se3(xi):
    w, v = xi[:3], xi[3:]
    R = g_exp_so3(w); th2 = dot(w, w)
    if th2 > EXP_NEAR_ZERO:
        c = cross(w, v); Rc = mv3(R, c); wv = dot(w, v)
        return (R, [(c[i] - Rc[i] + w[i]*wv)/th2 for i in range(3)])
    return (R, list(v))


def g_log_so3(R, pi_sub=None, force=None):
    """SO3::Logmap.  `force` ('pi' / 'acos' / 'taylor') and `pi_sub` (0 z, 1 y, 2 x) override the branch choice: the
    straddle cases evaluate both neighbours of a threshold."""
    tr = R[0] + R[4] + R[8]
    if force == "pi" or (force is None and tr + 1 < LOG_PI_TRACE):
        _note("log:pi", tr + 1, LOG_PI_TRACE)
        if pi_sub == 0 or (pi_sub is None and abs(R[8] + 1) > LOG_PI_DIAG):
            _note("logpi:z", R[8] + 1, LOG_PI_DIAG)
            f = mp.pi/mp.sqrt(2 + 2*R[8])
            return [f*R[2], f*R[5], f*(1 + R[8])]
        if pi_sub == 1 or (pi_sub is None and abs(R[4] + 1) > LOG_PI_DIAG):
            _note("logpi:y", R[4] + 1, LOG_PI_DIAG)
            f = mp.pi/mp.sqrt(2 + 2*R[4])
            return [f*R[1], f*(1 + R[4]), f*R[7]]
        _note("logpi:x")
        f = mp.pi/mp.sqrt(2 + 2*R[0])
        return [f*(1 + R[0]), f*R[3], f*R[6]]
    t3 = tr - 3
    if force == "acos" or (force is None and t3 < LOG_TAYLOR):
        _note("log:acos", tr + 1, LOG_PI_TRACE); _note("log:acos", t3, -LOG_TAYLOR)
        th = mp.acos((tr - 1)/2); mag = th/(2*mp.sin(th))
    else:
        _note("log:taylor", t3, -LOG_TAYLOR)
        mag = mpf(1)/2 - t3/12
    return [mag*(R[7] - R[5]), mag*(R[2] - R[6]), mag*(R[3] - R[1])]


def g_log_se3(P, **kw):
    R, T = P
    w = g_log_so3(R, **kw); t = norm(w)
    if t < POSE_LOG_SMALL:
        _note("selog:small", t, POSE_LOG_SMALL)
        return w + list(T)
    _note("selog:full", t, POSE_LOG_SMALL)
    W = skew([x/t for x in w]); WT = mv3(W, T); WWT = mv3(W, WT)
    k = 1 - t/(2*mp.tan(t/2))
    return w + [T[i] - (t/2)*WT[i] + k*WWT[i] for i in range(3)]


def g_retract(T, xi):
    return compose(T, g_exp_se3(xi))


def g_local(a, b):
    return g_log_se3(between(a, b))


def log_rot_bound(R):
    """a-priori bound, in units of eps, of the absolute error a faithful fp64 SO3::Logmap makes on R"""
    c = (R[0] + R[4] + R[8] - 1)/2
    th = mp.acos(max(min(c, 1), -1))
    if R[0] + R[4] + R[8] + 1 < LOG_PI_TRACE or R[0] + R[4] + R[8] - 3 >= LOG_TAYLOR:
        return mpf(8)*max(th, mpf(1))
    return 8 + 4*mp.pi/(mp.pi - th)**2


# ---- factors
def project_stereo(K, q):
    """gtsam::StereoCamera::project2 at the camera-frame point q; None on cheirality (z <= 0)"""
    if q[2] <= 0:
        return None
    fx, fy, u0, v0, b = K[0], K[1], K[3], K[4], K[5]
    return [u0 + fx*q[0]/q[2], u0 + fx*(q[0] - b)/q[2], v0 + fy*q[1]/q[2]]


def camera_point(t, v, z, aux, K):
    """the camera-frame point whose depth decides cheirality (STEREO3, HYBRID_STEREO3, FLOWPROJ2)"""
    if t == STEREO3:
        return act_inv(v[0], v[1])
    if t == HYBRID_STEREO3:
        return act_inv(v[0], act(v[1], act(aux, v[2])))
    fx, fy, s, u0, v0 = K[:5]
    yn = (z[1] - v0)/fy; xn = (z[0] - u0 - s*yn)/fx; d = z[2]
    return act_inv(v[1], act((z[3:12], z[12:15]), [xn*d, yn*d, d]))


def log_argument(t, v, z, aux):
    """the pose whose Logmap is the residual of a pose-valued factor (negated for PRIOR6)"""
    if t == PRIOR6:                       # -Local(x, prior)
        return between(v[0], (z[:9], z[9:]))
    if t == BETWEEN6:                     # Local(measured, x1^-1 x2)
        return between((z[:9], z[9:]), between(v[0], v[1]))
    if t == SMOOTH_HYBRID6:               # Local(L_{k-2}^-1 L_{k-1}, L_{k-1}^-1 L_k), L = E L_e
        L2, L1, L0 = (compose(e, aux) for e in v)
        return between(between(L2, L1), between(L1, L0))
    if t == SMOOTH_POSE6:                 # Local(P_{k-1} P_{k-2}^-1, P_k P_{k-1}^-1)
        return between(compose(v[1], inverse(v[0])), compose(v[2], inverse(v[1])))
    return None


def residual(t, v, z, aux, K, log=g_log_se3):
    """unwhitened residual of factor type t.  v: variables in key-slot order (poses as (R, t), points and flows as lists),
    z: the measurement record, aux: the auxiliary pose (HYBRID3, HYBRID_STEREO3, SMOOTH_HYBRID6), K: fx fy s u0 v0 b"""
    if t in (PRIOR6, BETWEEN6, SMOOTH_HYBRID6, SMOOTH_POSE6):
        r = log(log_argument(t, v, z, aux))
        return [-x for x in r] if t == PRIOR6 else r
    if t == POSE2POINT3:
        return [a - b for a, b in zip(act_inv(v[0], v[1]), z)]
    if t == TERNARY3:                     # m_{k-1} - H^-1 m_k
        return [a - b for a, b in zip(v[0], act_inv(v[2], v[1]))]
    if t == HYBRID3:                      # X^-1 H L_e m - z
        return [a - b for a, b in zip(act_inv(v[0], act(v[1], act(aux, v[2]))), z)]
    if t in (STEREO3, HYBRID_STEREO3):
        uv = project_stereo(K, camera_point(t, v, z, aux, K))
        if uv is None:
            return [2*K[0]]*3
        return [a - b for a, b in zip(uv, z)]
    if t == MOTIONPOSE3:                  # m_k - L_k L_{k-1}^-1 m_{k-1}
        return [a - b for a, b in zip(v[1], act(v[3], act_inv(v[2], v[0])))]
    if t == FLOWPROJ2:                    # kp + flow - project(X^-1 X_prev backproject(kp, depth))
        q = camera_point(t, v, z, aux, K)
        fx, fy, s, u0, v0 = K[:5]
        if q[2] <= 0:
            return [2*fx]*2
        un, vn = q[0]/q[2], q[1]/q[2]
        return [z[0] + v[0][0] - (fx*un + s*vn + u0), z[1] + v[0][1] - (fy*vn + v0)]
    raise ValueError(t)


def _perturbed(t, v, slot, j, d, retr):
    w = list(v)
    if SLOTS[t][slot] == "T":
        xi = [mpf(0)]*6; xi[j] = d
        w[slot] = retr(v[slot], xi)
    else:
        x = list(v[slot]); x[j] = x[j] + d; w[slot] = x
    return w


def _difference_jacobian(t, v, z, aux, K, d, log, retr, gtsam_form):
    hx = residual(t, v, z, aux, K, log)
    cols = []
    for slot, c in enumerate(SLOTS[t]):
        for j in range(SLOT_DIM[c]):
            h1 = residual(t, _perturbed(t, v, slot, j, d, retr), z, aux, K, log)
            h2 = residual(t, _perturbed(t, v, slot, j, -d, retr), z, aux, K, log)
            if gtsam_form:
                cols.append([((a - h) - (b - h))/(2*d) for a, b, h in zip(h1, h2, hx)])
            else:
                cols.append([(a - b)/(2*d) for a, b in zip(h1, h2)])
    return [[col[i] for col in cols] for i in range(len(hx))]


def jacobian_exact(t, v, z, aux, K):
    """the derivative of the residual through the true retraction (true Logmap inside the residual)"""
    return _difference_jacobian(t, v, z, aux, K, mpf("1e-20"), log_se3, retract, False)


def jacobian_gtsam(t, v, z, aux, K):
    """the Jacobian GTSAM 4.2.0 uses for the factor (module docstring)"""
    if t == PRIOR6:
        return [[mpf(int(i == j)) for j in range(6)] for i in range(6)]
    if t == BETWEEN6:
        Ad = adjoint(inverse(between(v[0], v[1])))
        return [[-Ad[i][j] for j in range(6)] + [mpf(int(i == j)) for j in range(6)] for i in range(6)]
    if t in NUMERIC_TYPES:
        return _difference_jacobian(t, v, z, aux, K, NUMERIC_DELTA, g_log_se3, g_retract, True)
    if t in (STEREO3, HYBRID_STEREO3, FLOWPROJ2) and camera_point(t, v, z, aux, K)[2] <= 0:
        n = 2 if t == FLOWPROJ2 else 3
        return [[mpf(0)]*sum(SLOT_DIM[c] for c in SLOTS[t]) for _ in range(n)]
    if t == FLOWPROJ2 and K[2] != 0:
        # Pose3FlowProjectionFactor's Jacobian has no skew term: it is the derivative of the skew-free projection of the
        # same camera-frame point (the key-point moved so that the skew-free back-projection gives that point)
        yn = (z[1] - K[4])/K[1]
        return jacobian_exact(t, v, [z[0] - K[2]*yn] + list(z[1:]), aux, [K[0], K[1], mpf(0)] + list(K[3:]))
    return jacobian_exact(t, v, z, aux, K)


def whiten(r, sigma, k):
    """(whitened residual, sqrt(weight), factor error): noiseModel::Isotropic / Diagonal whitening, then
    noiseModel::Robust(Huber, k) for k > 0 -- weight 1 at |r| <= k, sqrt(k/|r|) above; the comparison in 50 digits"""
    rw = [x/(sigma[0] if len(sigma) == 1 else sigma[i]) for i, x in enumerate(r)]
    n2 = dot(rw, rw)
    if k > 0:
        n = mp.sqrt(n2)
        if n <= k:
            _note("huber:inside")
            return rw, mpf(1), n2/2
        _note("huber:outside")
        return rw, mp.sqrt(k/n), k*(n - k/2)
    return rw, mpf(1), n2/2


def linearized(t, v, z, aux, K, sigma, k, with_jacobian=True):
    """(A, b, error): the whitened, weighted Jacobian, the negated whitened weighted residual, the factor's error"""
    rw, sw, e = whiten(residual(t, v, z, aux, K), sigma, k)
    b = [-x*sw for x in rw]
    if not with_jacobian:
        return None, b, e
    J = jacobian_gtsam(t, v, z, aux, K)
    A = [[x*sw/(sigma[0] if len(sigma) == 1 else sigma[i]) for x in row] for i, row in enumerate(J)]
    return A, b, e
