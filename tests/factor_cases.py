"""The case list of the factor kernels and the SE(3) maps: small `Problem`s, each naming the branch boundaries and
block-size edges it reaches (`hits`), the 50-digit reference of a case (`reference`) and the comparator both halves of
the test use (`compare`).  tests/test_factor_cases.py checks on the CPU that every name of `REQUIRED` is reached and
that every claim is true; tests/test_factors_gpu.py runs the cases on the device.

Rotations are built in 50 digits (`lie_reference.exp_so3`) and rounded once to fp64, so the 12 doubles of a pose are a
case's exact input.  Values of a block may be tiled with a period (7 distinct factors, or 257 for the two 131 k-factor
blocks): the reference evaluates each distinct factor once.

Comparator.  Every number is compared in units of its a-priori bound, so one tolerance serves a family:

    b:  |db_i| / (eps * B * (|r|_inf + S_i))      A:  |dA_ij| / (eps * B * max_j |A_ij|)      (whitening applied to both)

S_i is the magnitude of the terms that cancel in row i (1 for a rotation row; 1 + the largest |t|, |p| involved for a
translation row; the projected magnitudes for a pixel row), so an exactly-zero residual is held to a few eps * S and
not to a meaningless relative error.  B is 1 for a closed form, `lie_reference.log_rot_bound` / 8 for a residual that
goes through Logmap (pi eps/(pi - theta)^2 towards pi), and for the numerically differentiated Jacobians the rounding
of GTSAM's difference quotient, (|h|_inf + S)/delta per unit of the row.
"""
from dataclasses import dataclass, field

import numpy as np
from mpmath import mp, mpf

import lie_reference as LR
from dynosam_b200.problem import (ARITY, BETWEEN6, DIM, FLOWPROJ2, HYBRID3, HYBRID_STEREO3, JCOLS, MEAS_DIM, MOTIONPOSE3,
                                  NEEDS_AUX, POSE2POINT3, PRIOR6, SLOT_CLASS, SMOOTH_HYBRID6, SMOOTH_POSE6, STEREO3, TERNARY3,
                                  TYPE_NAMES, FactorBlock, Problem)

EPS = 2.0**-52
THETAS = ["0", "1e-12", "1e-9", "0.7e-8", "2.2e-8", "1e-5", "2e-4", "5e-4", "0.3", "2.5", "pi-1e-3", "pi-3e-5", "pi-5e-6",
          "pi-1e-8", "pi"]
AXES = {"z": (0, 0, 1), "y": (0, 1, 0), "x": (1, 0, 0), "xy": (0.6, 0.8, 0), "diag": (1, 1, 1), "-xz": (-0.6, 0, -0.8),
        "smallz": (0.6, 0.8, 0.005)}
BLOCK_SIZES = [1, 31, 32, 33, 127, 128, 129, 257]
LOG_TYPES = (PRIOR6, BETWEEN6, SMOOTH_HYBRID6, SMOOTH_POSE6)
CAMERA_TYPES = (STEREO3, HYBRID_STEREO3, FLOWPROJ2)
CHEIRALITY_Z = {"z<0": -1.0, "z=-tiny": -1e-300, "z=-0": -0.0, "z=+0": 0.0, "z=denormal": 5e-324, "z=1e-12": 1e-12,
                "z=1e-3": 1e-3, "z=1": 1.0}

REQUIRED = (
    ["log:pi", "logpi:z", "logpi:y", "logpi:x", "log:acos", "log:taylor", "log:acos_near_pi", "log:acos_near_taylor",
     "log:taylor_near_acos", "log:identity", "selog:small", "selog:full", "exp:first_order", "exp:full", "exp:beyond_pi",
     "straddle:exp", "straddle:log_taylor", "straddle:log_pi", "straddle:selog"]
    + [f"zero_residual:{TYPE_NAMES[t]}" for t in LOG_TYPES] + [f"near_pi:{TYPE_NAMES[t]}" for t in LOG_TYPES]
    + [f"cheirality:{TYPE_NAMES[t]}:{z}" for t in CAMERA_TYPES for z in CHEIRALITY_Z] + ["skew:0", "skew:3.7"]
    + [f"huber:{w}:{m}" for w in ("n==k", "n=k+ulp", "n=k-ulp", "n=0", "n=10k") for m in ("isotropic", "diagonal")]
    + ["huber:k=1e-4", "huber:k=1.345", "huber:k=1e3", "huber:dim6", "huber:dim2", "sigma:1e-6..1e6"]
    + [f"F={f}:{TYPE_NAMES[t]}" for f in BLOCK_SIZES for t in range(11)]
    + ["partials:1024", "partials:1025", "gather:aux_reversed", "gather:last_pose", "gather:last_point",
       "gather:between_same_pose", "gather:smooth_same_pose", "gather:blocks_of_one_type",
       "retract:t=1e3", "retract:v=0", "retract:v=1e3", "retract:point", "retract:flow"])


@dataclass
class Case:
    name: str
    problem: Problem
    hits: tuple
    period: dict = field(default_factory=dict)        # block index -> number of distinct factors (values tiled)
    check_A: dict = field(default_factory=dict)       # block index -> False: the Jacobian is not compared (says why in `note`)
    delta: np.ndarray = None                          # a retraction step (poses, points, flows)
    straddle: bool = False                            # a threshold lies within a factor 2: both branches must agree
    bit_exact: bool = False                           # inputs chosen so that the residual is exact: b compared bit for bit
    note: str = ""


def theta(s):
    return mp.pi - mpf(s[3:]) if s.startswith("pi-") else (mp.pi if s == "pi" else mpf(s))


def rotation(th, axis):
    """fp64(Exp(theta a)) built in 50 digits, a = axis/|axis|"""
    a = LR.vec(axis) if not isinstance(axis[0], mpf) else axis
    n = LR.norm(a)
    return np.array(LR.to_float(LR.exp_so3([theta(th)*x/n for x in a]))) if isinstance(th, str) else \
        np.array(LR.to_float(LR.exp_so3([th*x/n for x in a])))


def pose12(R, t):
    return np.concatenate([np.asarray(R, float).reshape(9), np.asarray(t, float).reshape(3)])


def compose12(a, b):
    """fp64(a b) from the 50-digit product (one rounding)"""
    return np.array(LR.to_float(LR.pose_flat(LR.compose(LR.pose(a), LR.pose(b)))))


def random_pose(rng, rot=0.2, trans=0.5):
    return pose12(rotation(mpf(float(rng.uniform(0.3, 1.0)*rot)), tuple(rng.normal(size=3))), rng.normal(0, trans, 3))


IDENT = pose12(np.eye(3), np.zeros(3))
K_DEFAULT = np.array([721.5377, 721.5377, 0.0, 609.5593, 172.854, 0.5372])
TRANSLATIONS = [0.0, 1e-3, 1.0, 1e3]


# ---------------------------------------------------------------------------------------------- rotation cases
def _relative_rotations(thetas, axes, rng):
    """(name, relative pose) for every theta x axis; the translation cycles through 0, 1e-3, 1, 1e3"""
    out = []
    for i, th in enumerate(thetas):
        for j, ax in enumerate(axes):
            tm = TRANSLATIONS[(i + j) % 4]
            out.append((f"{th}@{ax}", pose12(rotation(th, AXES[ax]), tm*np.array([0.48, -0.6, 0.64]))))
    return out


def _pose_block_case(t, rels, name, general, seed, hits, **kw):
    """one block of pose-valued factors of type t whose Logmap argument is (up to rounding of the products, when
    `general`) each of `rels`; exact when the other poses are pure translations"""
    rng = np.random.default_rng(seed)
    poses, idx, meas, aux, aux_idx = [], [], [], [], []
    for k, (_, rel) in enumerate(rels):
        G = random_pose(rng, 1.0, 2.0) if general else pose12(np.eye(3), [4.0, -2.0, 0.5])
        if t == PRIOR6:                       # x^-1 prior = rel
            poses += [G]; idx.append([len(poses) - 1]); meas.append(compose12(G, rel))
        elif t == BETWEEN6:                   # m^-1 (x1^-1 x2) = rel, m a pure translation
            m = pose12(np.eye(3), [0.25, 0.5, -1.0]) if not general else random_pose(rng, 1.0, 1.0)
            poses += [G, compose12(G, compose12(m, rel))]; idx.append([len(poses) - 2, len(poses) - 1]); meas.append(m)
        elif t == SMOOTH_POSE6:               # a = P1 P2^-1 = I, b = P0 P1^-1 = rel  (world-frame motions)
            poses += [G, G, compose12(rel, G)]; idx.append([len(poses) - 3, len(poses) - 2, len(poses) - 1])
        else:                                 # SMOOTH_HYBRID6: L = E L_e; E2 = E1 = G, E0 L_e = G L_e rel
            Le = random_pose(rng, 0.7, 1.0) if general else pose12(np.eye(3), [1.0, 2.0, -0.5])
            aux.append(Le); aux_idx.append(len(aux) - 1)
            E0 = compose12(compose12(G, compose12(Le, rel)), np.array(LR.to_float(LR.pose_flat(LR.inverse(LR.pose(Le))))))
            poses += [G, G, E0]; idx.append([len(poses) - 3, len(poses) - 2, len(poses) - 1])
    sig = np.array([0.01, 0.02, 0.03, 0.1, 0.2, 0.3])
    blk = FactorBlock(t, np.array(idx), np.array(meas) if meas else None, sig, 0.0, np.array(aux_idx) if aux else None)
    p = Problem(np.array(poses), np.zeros((0, 3)), aux_pose=np.array(aux) if aux else np.zeros((0, 12)), blocks=[blk])
    return Case(name, p, tuple(hits), **kw)


def rotation_cases():
    rng = np.random.default_rng(0)
    cases = []
    all_axes = ["z", "y", "x", "xy", "diag", "-xz", "smallz"]
    rot_hits = ["log:pi", "logpi:z", "logpi:y", "logpi:x", "log:acos", "log:taylor", "log:acos_near_pi", "log:acos_near_taylor",
                "log:taylor_near_acos", "log:identity", "selog:small", "selog:full"]
    for t in (PRIOR6, BETWEEN6):
        n = TYPE_NAMES[t]
        cases.append(_pose_block_case(t, _relative_rotations(THETAS, all_axes, rng), f"rot_exact_{n}", False, 1,
                                      rot_hits + [f"near_pi:{n}"]))
        cases.append(_pose_block_case(t, _relative_rotations(THETAS[5:12], all_axes[:6], rng), f"rot_general_{n}", True, 2,
                                      ["log:acos", "log:taylor", "log:acos_near_pi"]))
    # the numerically differentiated factors: the Jacobian is GTSAM's difference quotient with delta = 1e-5, which is only
    # meaningful where Logmap is smooth over +-delta -- up to pi - 1e-3; nearer to pi the quotient straddles the
    # discontinuity of the formula (and its 1e-7 conditioning), so only the residual is compared there
    for t in (SMOOTH_HYBRID6, SMOOTH_POSE6):
        n = TYPE_NAMES[t]
        cases.append(_pose_block_case(t, _relative_rotations(THETAS[:11], ["z", "diag"], rng), f"rot_exact_{n}", False, 3,
                                      ["log:acos", "log:taylor", "log:identity", "selog:small", "selog:full"]))
        cases.append(_pose_block_case(t, _relative_rotations(THETAS[11:], ["y", "xy", "-xz"], rng), f"rot_pi_{n}", False, 4,
                                      ["log:pi", "logpi:y", "logpi:z", f"near_pi:{n}"], check_A={0: False},
                                      note="difference quotient across the pi discontinuity: residual only"))
    # every residual exactly zero: noise-free constant motion (pure translations and rotations about z by a dyadic-exact
    # angle would still round; the poses are built so that the products are exact: translations only, dyadic)
    for t in LOG_TYPES:
        rels = [(f"zero{k}", IDENT) for k in range(5)]
        c = _pose_block_case(t, rels, f"zero_residual_{TYPE_NAMES[t]}", False, 5, [f"zero_residual:{TYPE_NAMES[t]}", "log:identity"],
                             bit_exact=True)
        cases.append(c)
    return cases


def straddle_cases():
    """a threshold within rounding of the input: whichever side fp64 picks, the two neighbouring branches agree to the
    bound of the module docstring of lie_reference, which is what `compare` allows these cases"""
    out = []
    for name, th, hit in (("exp", None, "straddle:exp"), ("log_taylor", "3.1622776e-4", "straddle:log_taylor"),
                          ("log_pi", "pi-1e-5", "straddle:log_pi"), ("selog", "1e-10", "straddle:selog")):
        if th is None:
            continue
        rels = [(f"{th}@{ax}", pose12(rotation(th, AXES[ax]), [0.3, -0.2, 0.1])) for ax in ("z", "xy", "diag")]
        out.append(_pose_block_case(PRIOR6, rels, f"straddle_{name}", False, 6, [hit], straddle=True))
    return out


# ---------------------------------------------------------------------------------------------- cheirality
def cheirality_cases():
    """camera-frame depth z at and around 0, exactly representable after transform_to: identity rotations and dyadic
    translations (the camera sits at (0, 0, -2) ... so that p_z - t_z is exact)"""
    cases = []
    zs = list(CHEIRALITY_Z.items())
    for skew in (0.0, 3.7):
        K = K_DEFAULT.copy(); K[2] = skew
        n = len(zs)
        X = IDENT.copy()                                      # camera at the origin: q = p exactly
        pts = np.array([[0.25, -0.5, z] for _, z in zs])
        blocks = [FactorBlock(STEREO3, np.stack([np.zeros(n, int), np.arange(n)], 1), np.tile([600.0, 590.0, 170.0], (n, 1)),
                              np.array([0.5]))]
        # HYBRID_STEREO3: X = H = L_e = identity -> q = m exactly
        blocks.append(FactorBlock(HYBRID_STEREO3, np.stack([np.zeros(n, int), np.ones(n, int), np.arange(n)], 1),
                                  np.tile([600.0, 590.0, 170.0], (n, 1)), np.array([0.5, 0.25, 2.0]), 0.0, np.zeros(n, int)))
        # FLOWPROJ2: X_prev = X = identity, the key-point at the principal point when skew = 0 -> q = (0, 0, depth)
        meas = np.array([np.concatenate([[K[3], K[4], z], IDENT]) for _, z in zs])
        flow = np.tile([1.5, -0.75], (n, 1))
        blocks.append(FactorBlock(FLOWPROJ2, np.stack([np.arange(n), np.zeros(n, int)], 1), meas, np.array([0.5])))
        p = Problem(np.stack([X, IDENT]), pts, flow=flow, aux_pose=IDENT[None], calib=K, blocks=blocks)
        hits = [f"cheirality:{TYPE_NAMES[t]}:{z}" for t in CAMERA_TYPES for z, _ in zs] + [f"skew:{skew:g}"]
        cases.append(Case(f"cheirality_skew{skew:g}", p, tuple(hits)))
    # FLOWPROJ2 in general position with skew: key-points off the principal point, a moving camera
    rng = np.random.default_rng(7)
    K = K_DEFAULT.copy(); K[2] = 3.7
    n = 9
    Xp, X = random_pose(rng), random_pose(rng)
    kp = np.stack([rng.uniform(100, 1100, n), rng.uniform(40, 330, n)], 1); depth = rng.uniform(4, 30, n)
    meas = np.concatenate([kp, depth[:, None], np.tile(Xp, (n, 1))], 1)
    blk = FactorBlock(FLOWPROJ2, np.stack([np.arange(n), np.zeros(n, int)], 1), meas, np.array([0.5, 0.8]))
    cases.append(Case("flowproj_skew_general", Problem(X[None], np.zeros((0, 3)), flow=rng.normal(0, 3, (n, 2)), calib=K, blocks=[blk]),
                      ("skew:3.7",)))
    return cases


# ---------------------------------------------------------------------------------------------- Huber and whitening
def huber_cases():
    cases = []
    up = lambda x: np.nextafter(x, np.inf); dn = lambda x: np.nextafter(x, -np.inf)
    for mode, sig in (("isotropic", np.array([0.125])), ("diagonal", np.array([0.125, 1.0, 4.0]))):
        for k in (1e-4, 1.345, 1e3):
            # POSE2POINT3 at the identity pose with z = 0: r = p exactly; sigma_0 = 2^-3, so r_w = 8 p_x exactly
            norms = {"n==k": k, "n=k+ulp": up(k), "n=k-ulp": dn(k), "n=0": 0.0, "n=10k": 10*k}
            pts = np.array([[v*0.125, 0.0, 0.0] for v in norms.values()])
            n = len(pts)
            blk = FactorBlock(POSE2POINT3, np.stack([np.zeros(n, int), np.arange(n)], 1), np.zeros((n, 3)), sig, k)
            hits = [f"huber:{w}:{mode}" for w in norms] + [f"huber:k={k:g}".replace("0.0001", "1e-4").replace("1000", "1e3")]
            cases.append(Case(f"huber_{mode}_k{k:g}", Problem(IDENT[None], pts, blocks=[blk]), tuple(hits), bit_exact=True))
    # the 3-4-0 triple over a dyadic sigma: n = 5/4 / 0.25 = 5 exactly = k
    pts = np.array([[0.75, 1.0, 0.0], [0.0, 0.75, 1.0], [0.75, 1.0, 2.0**-50]])
    blk = FactorBlock(POSE2POINT3, np.stack([np.zeros(3, int), np.arange(3)], 1), np.zeros((3, 3)), np.array([0.25]), 5.0)
    cases.append(Case("huber_345", Problem(IDENT[None], pts, blocks=[blk]), ("huber:n==k:isotropic",), bit_exact=True))
    # 6-dim: PRIOR6 on pure translations (Logmap of a translation is the translation, exactly); 2-dim: FLOWPROJ2 with the
    # principal point at 0 and the key-point on it, so r = flow exactly
    k = 1.345
    tr = [k, up(k), dn(k), 0.0, 10*k]
    poses = np.array([pose12(np.eye(3), [-v, 0, 0]) for v in tr])
    blk6 = FactorBlock(PRIOR6, np.arange(5)[:, None], np.tile(IDENT, (5, 1)), np.array([1.0]), k)
    K0 = np.array([512.0, 512.0, 0.0, 0.0, 0.0, 0.5])
    meas = np.tile(np.concatenate([[0.0, 0.0, 1.0], IDENT]), (5, 1))
    blk2 = FactorBlock(FLOWPROJ2, np.stack([np.arange(5), np.full(5, 5)], 1), meas, np.array([1.0, 4.0]), k)
    p = Problem(np.concatenate([poses, IDENT[None]]), np.zeros((0, 3)), flow=np.array([[v, 0.0] for v in tr]), calib=K0, blocks=[blk6, blk2])
    cases.append(Case("huber_dim6_dim2", p, ("huber:dim6", "huber:dim2"), bit_exact=True))
    # sigma spanning 1e-6 .. 1e6 inside one block, on every dim
    rng = np.random.default_rng(8)
    X = random_pose(rng); pts = rng.normal(0, 1, (6, 3)) + [0, 0, 8.0]
    sig3 = np.array([1e-6, 1.0, 1e6]); sig6 = np.array([1e-6, 1e-3, 1.0, 1e2, 1e4, 1e6]); sig2 = np.array([1e-6, 1e6])
    blocks = [FactorBlock(POSE2POINT3, np.stack([np.zeros(6, int), np.arange(6)], 1), rng.normal(0, 1, (6, 3)) + [0, 0, 8.0], sig3, 1.345),
              FactorBlock(PRIOR6, np.array([[0]]), random_pose(rng)[None], sig6, 0.0),
              FactorBlock(FLOWPROJ2, np.array([[0, 0]]), np.concatenate([[400.0, 200.0, 9.0], IDENT])[None], sig2, 0.0)]
    cases.append(Case("sigma_span", Problem(X[None], pts, flow=np.array([[2.0, -1.0]]), blocks=blocks), ("sigma:1e-6..1e6",)))
    return cases


# ---------------------------------------------------------------------------------------------- block sizes, gather
class Pool:
    """a small seeded set of variables in general position -- cameras near the origin looking down +z, object motions
    near the identity, points 5 to 12 m ahead -- and 7 distinct factors of every type over it"""

    def __init__(self, seed=11, n_pose=9, n_point=8, n_flow=5, n_aux=3):
        rng = np.random.default_rng(seed); self.rng = rng
        self.pose = np.array([random_pose(rng) for _ in range(n_pose)])
        self.aux = np.array([random_pose(rng, 0.2, 0.3) for _ in range(n_aux)])
        self.point = np.stack([rng.uniform(-2, 2, n_point), rng.uniform(-2, 2, n_point), rng.uniform(5, 12, n_point)], 1)
        self.flow = rng.normal(0, 2, (n_flow, 2))

    def factors(self, t, count, period=7, reverse_aux=False, last=False):
        rng = np.random.default_rng(100 + t)
        P, Q, A = len(self.pose), len(self.point), len(self.aux)
        idx, meas, aux = [], [], []
        for j in range(period):
            slots = []
            for s, c in enumerate(SLOT_CLASS[t]):
                nvar = {0: P, 1: Q, 2: len(self.flow)}[c]
                slots.append(nvar - 1 - (j + 2*s) % nvar if last else (j + 2*s + s*s) % nvar)
            idx.append(slots)
            aux.append((A - 1 - j % A) if reverse_aux else (j + 1) % A)
            m = np.zeros(MEAS_DIM[t])
            if t in (PRIOR6, BETWEEN6):
                m = random_pose(rng, 0.3, 0.8)
            elif t in (POSE2POINT3, HYBRID3):
                m = self.point[slots[-1]] + rng.normal(0, 0.3, 3)
            elif t in (STEREO3, HYBRID_STEREO3):
                m = np.array([640.0, 600.0, 180.0]) + rng.normal(0, 30, 3)
            elif t == FLOWPROJ2:
                m = np.concatenate([[rng.uniform(100, 1100), rng.uniform(40, 330), rng.uniform(4, 30)], self.pose[(j + 3) % P]])
            meas.append(m)
        rep = lambda a: np.array([a[f % period] for f in range(count)])
        sig = {6: np.array([0.02, 0.03, 0.05, 0.1, 0.2, 0.3]), 3: np.array([0.2]), 2: np.array([0.7, 0.9])}[DIM[t]]
        return FactorBlock(t, rep(idx), rep(meas) if MEAS_DIM[t] else None, sig, 1.345 if DIM[t] == 3 else 0.0,
                           rep(aux) if NEEDS_AUX[t] else None)

    def problem(self, blocks):
        return Problem(self.pose, self.point, flow=self.flow, aux_pose=self.aux, blocks=blocks)


def block_size_cases():
    pool = Pool()
    cases = []
    for F in BLOCK_SIZES:
        blocks = [pool.factors(t, F) for t in range(11)]
        cases.append(Case(f"blocks_F{F}", pool.problem(blocks), tuple(f"F={F}:{TYPE_NAMES[t]}" for t in range(11)),
                          period={bi: min(7, F) for bi in range(11)}))
    return cases


def gather_case():
    pool = Pool(seed=12)
    P = len(pool.pose)
    blocks = [pool.factors(t, 9, reverse_aux=True, last=True) for t in (HYBRID3, HYBRID_STEREO3, SMOOTH_HYBRID6, POSE2POINT3, TERNARY3)]
    blocks.append(pool.factors(POSE2POINT3, 5))                                     # a second block of the same type
    blocks.append(FactorBlock(BETWEEN6, np.array([[3, 3], [P - 1, P - 1]]), np.stack([random_pose(pool.rng), IDENT]), np.array([0.1])))
    blocks.append(FactorBlock(SMOOTH_POSE6, np.array([[2, 5, 2], [P - 1, 0, P - 1]]), None, np.array([0.1])))
    return Case("gather", pool.problem(blocks),
                ("gather:aux_reversed", "gather:last_pose", "gather:last_point", "gather:between_same_pose", "gather:smooth_same_pose",
                 "gather:blocks_of_one_type"), period={bi: 7 for bi in range(6)})


def big_block_case(n_factors):
    """one POSE2POINT3 block of n_factors (n_factors / 128 partial sums reach the final reduction), values tiled from 257"""
    rng = np.random.default_rng(13)
    poses = np.array([random_pose(rng) for _ in range(257)])
    pts = np.stack([rng.uniform(-2, 2, 257), rng.uniform(-2, 2, 257), rng.uniform(5, 12, 257)], 1)
    m = pts + rng.normal(0, 0.3, (257, 3))
    f = np.arange(n_factors) % 257
    blk = FactorBlock(POSE2POINT3, np.stack([f, f], 1), m[f], np.array([0.2]), 1.345)
    return Case(f"big_{n_factors}", Problem(poses, pts, blocks=[blk]), (f"partials:{(n_factors + 127)//128}",), period={0: 257})


# ---------------------------------------------------------------------------------------------- retraction
def retract_case():
    """steps with |omega| over THETAS (0 and beyond pi included) times |v| in {0, 1e-9, 1, 1e3}, on poses 1e3 from the
    origin, plus point and flow steps"""
    rng = np.random.default_rng(14)
    thetas = THETAS + ["3.5", "6.0", "1.5e-8"]
    steps, poses = [], []
    axes = list(AXES.values())
    for i, th in enumerate(thetas):
        for j, vm in enumerate((0.0, 1e-9, 1.0, 1e3)):
            a = np.array(axes[(i + j) % len(axes)], float); a /= np.linalg.norm(a)
            w = float(theta(th))*a
            v = vm*np.array([0.64, 0.48, -0.6])
            steps.append(np.concatenate([w, v]))
            poses.append(pose12(random_pose(rng, 2.0)[:9], 1e3*np.array([0.6, -0.64, 0.48])))
    n = len(poses)
    pts = rng.normal(0, 1, (3, 3)) + [600, -640, 488]
    flow = rng.normal(0, 2, (2, 2))
    blocks = [FactorBlock(PRIOR6, np.arange(n)[:, None], np.array(poses), np.array([1.0])),
              FactorBlock(POSE2POINT3, np.stack([np.zeros(3, int), np.arange(3)], 1), np.zeros((3, 3)), np.array([1.0])),
              FactorBlock(FLOWPROJ2, np.stack([np.arange(2), np.zeros(2, int)], 1),
                          np.tile(np.concatenate([[400.0, 200.0, 9.0], poses[0]]), (2, 1)), np.array([1.0]))]
    delta = np.concatenate([np.concatenate(steps), rng.normal(0, 1, 9), rng.normal(0, 1, 4)])
    return Case("retract", Problem(np.array(poses), pts, flow=flow, blocks=blocks),
                ("exp:first_order", "exp:full", "exp:beyond_pi", "straddle:exp", "retract:t=1e3", "retract:v=0", "retract:v=1e3",
                 "retract:point", "retract:flow"), delta=delta, straddle=True)


def _build():
    cases = rotation_cases() + straddle_cases() + cheirality_cases() + huber_cases() + block_size_cases()
    cases += [gather_case(), big_block_case(131072), big_block_case(131073), retract_case()]
    assert len({c.name for c in cases}) == len(cases)
    return {c.name: c for c in cases}


_CASES = None


def cases():
    global _CASES
    if _CASES is None:
        _CASES = _build()
    return _CASES


# ---------------------------------------------------------------------------------------------- reference of a case
@dataclass
class BlockRef:
    A: np.ndarray          # [n, dim, jcols] fp64 of the 50-digit value
    b: np.ndarray          # [n, dim]
    e: np.ndarray          # [n]
    unit_b: np.ndarray     # [n, dim]  a-priori bound of |db| per unit of tolerance
    unit_A: np.ndarray     # [n, dim]  ... of |dA| along the row
    behind: np.ndarray     # [n] cheirality
    inside: np.ndarray     # [n] Huber weight exactly 1 (or no Huber)
    trace: set
    e_mp: object           # the block's error summed in 50 digits


_FACTOR_CACHE = {}


def _factor(p, b, f, with_A):
    """reference of factor f of block b: evaluated once per distinct input"""
    t = b.type
    v, S = [], 1.0
    for s, c in enumerate(SLOT_CLASS[t]):
        x = (p.pose, p.point, p.flow)[c][b.idx[f, s]]
        v.append(LR.pose(x) if c == 0 else LR.vec(x))
        if c != 2:
            S = max(S, 1.0 + np.abs(x[-3:]).max())
    z = LR.vec(b.meas[f]) if b.meas is not None else []
    if t in (PRIOR6, BETWEEN6):
        S = max(S, 1.0 + np.abs(b.meas[f][9:]).max())
    if t in (POSE2POINT3, HYBRID3):
        S = max(S, 1.0 + np.abs(b.meas[f]).max())
    aux = LR.pose(p.aux_pose[b.aux_idx[f]]) if NEEDS_AUX[t] else None
    if aux is not None:
        S = 2*S + np.abs(p.aux_pose[b.aux_idx[f]][9:]).max()
    sigma = LR.vec(b.sigma if b.sigma_bcast else b.sigma[f])
    flat = [(p.pose, p.point, p.flow)[c][b.idx[f, s]] for s, c in enumerate(SLOT_CLASS[t])] + \
        [b.meas[f] if b.meas is not None else np.zeros(0), p.aux_pose[b.aux_idx[f]] if aux else np.zeros(0),
         b.sigma if b.sigma_bcast else b.sigma[f], p.calib]
    key = (t, with_A, float(b.robust_k), np.concatenate(flat).tobytes())          # (bytes: -0.0 and 0.0 are different inputs)
    if key in _FACTOR_CACHE:
        return _FACTOR_CACHE[key]
    K = LR.vec(p.calib); k = mpf(float(b.robust_k))
    LR.trace_start()
    r = LR.residual(t, v, z, aux, K)
    rw, sw, e = LR.whiten(r, sigma, k)
    trace = LR.trace_stop()
    A, bb, _ = LR.linearized(t, v, z, aux, K, sigma, k, with_A)
    D = DIM[t]
    sg = [float(sigma[0] if len(sigma) == 1 else sigma[i]) for i in range(D)]
    rinf = float(max(abs(x) for x in r))
    B = np.ones(D); Srow = np.full(D, S); behind = False
    if t in LOG_TYPES:
        arg = LR.log_argument(t, v, z, aux)
        B[:] = float(LR.log_rot_bound(arg[0]))/8
        Srow[:3] = 1.0; Srow[3:] = S*(3 if t in (SMOOTH_HYBRID6, SMOOTH_POSE6) else 1)
        w = LR.to_float(r[:3])
        if all(x == 0 for x in w):
            trace.add("log:identity")
        th = np.linalg.norm(w)
        if "log:acos" in trace and np.pi - th < 1e-4: trace.add("log:acos_near_pi")
        if "log:acos" in trace and th < 1e-3: trace.add("log:acos_near_taylor")
        if "log:taylor" in trace and th > 1e-4: trace.add("log:taylor_near_acos")
        if th > np.pi - 1e-4: trace.add(f"near_pi:{TYPE_NAMES[t]}")
        if rinf == 0: trace.add(f"zero_residual:{TYPE_NAMES[t]}")
    if t in CAMERA_TYPES:
        q = LR.camera_point(t, v, z, aux, K); zc = q[2]; behind = bool(zc <= 0)
        qf = np.array(LR.to_float(q))
        exact = all(mpf(float(x)) == x for x in q)
        zin = b.meas[f][2] if t == FLOWPROJ2 else p.point[b.idx[f, -1], 2]      # (mpmath has no -0: the sign is the input's)
        for name, zv in CHEIRALITY_Z.items():
            if exact and qf[2] == zv and np.signbit(zin) == np.signbit(zv):
                trace.add(f"cheirality:{TYPE_NAMES[t]}:{name}")
        if not behind and float(zc) < 1e-300:       # 1/z overflows in fp64, as it does in GTSAM: only the branch is compared
            Srow[:] = np.inf
        elif not behind:
            cz = 1.0 if exact else 1.0 + S/float(zc)
            fx = float(K[0])
            Srow[:] = cz*fx*(1 + np.abs(qf).max()/float(zc)) + 2*np.abs(p.calib[3:5]).max() + (np.abs(b.meas[f][:3]).max())
            B[:] = cz
        if t == FLOWPROJ2:
            trace.add(f"skew:{float(K[2]):g}")
    unit_b = np.array([EPS*B[i]*(rinf + Srow[i])*float(sw)/sg[i] for i in range(D)])
    if with_A:
        Af = np.array(LR.to_float(A)); unit_A = EPS*B*np.abs(Af).max(1)
        if t in LR.NUMERIC_TYPES:          # rounding of the difference quotient: eps * max|h| / delta, whitened
            unit_A = np.array([EPS*B[i]*(rinf + Srow[i])/1e-5*float(sw)/sg[i] for i in range(D)])
    else:
        Af = np.zeros((D, JCOLS[t])); unit_A = np.zeros(D)
    out = (Af, np.array(LR.to_float(bb)), float(e), unit_b, np.maximum(unit_A, 1e-300), behind, "huber:outside" not in trace, trace, e)
    _FACTOR_CACHE[key] = out
    return out


def reference(case):
    """[BlockRef] of the case's problem, and its chi^2 summed in 50 digits (as a float)"""
    p = case.problem
    refs, total = [], mpf(0)
    for bi, b in enumerate(p.blocks):
        per = min(case.period.get(bi, b.n), b.n)
        with_A = case.check_A.get(bi, True)
        rows = [_factor(p, b, f, with_A) for f in range(per)]
        pick = np.arange(b.n) % per
        st = lambda k: np.array([rows[i][k] for i in range(per)])[pick]
        trace = set().union(*(r[7] for r in rows))
        mult = np.bincount(pick, minlength=per)
        e_mp = sum(rows[i][8]*int(mult[i]) for i in range(per))
        refs.append(BlockRef(st(0), st(1), st(2), st(3), st(4), st(5), st(6), trace, e_mp))
        total += e_mp
    return refs, float(total)


def reference_retract(case):
    """(pose, point, flow) after values.retract(delta): T g_exp_se3(xi) in 50 digits, and the trace of the Expmap branches"""
    p = case.problem; n = p.n_pose
    LR.trace_start()
    pose = np.array([LR.to_float(LR.pose_flat(LR.g_retract(LR.pose(p.pose[i]), LR.vec(case.delta[6*i:6*i + 6])))) for i in range(n)])
    trace = LR.trace_stop()
    d = case.delta[6*n:]
    point = np.array(LR.to_float([[mpf(float(a)) + mpf(float(b)) for a, b in zip(r, dr)] for r, dr in zip(p.point, d[:3*p.n_point].reshape(-1, 3))]))
    flow = np.array(LR.to_float([[mpf(float(a)) + mpf(float(b)) for a, b in zip(r, dr)] for r, dr in zip(p.flow, d[3*p.n_point:].reshape(-1, 2))]))
    return pose, point, flow, trace


def boundaries(case):
    """what the case really reaches, by the 50-digit branch classifier and the shape of its blocks"""
    p = case.problem
    if case.delta is not None:
        _, _, _, tr = reference_retract(case)
        w = np.linalg.norm(case.delta[:6*p.n_pose].reshape(-1, 6)[:, :3], axis=1); v = np.linalg.norm(case.delta[:6*p.n_pose].reshape(-1, 6)[:, 3:], axis=1)
        out = {x for x in tr if not x.startswith("close:")}
        if "close:exp" in tr: out.add("straddle:exp")
        if (w > np.pi).any(): out.add("exp:beyond_pi")
        if (np.abs(np.linalg.norm(p.pose[:, 9:], axis=1) - 1e3) < 1).all(): out.add("retract:t=1e3")
        if (v == 0).any(): out.add("retract:v=0")
        if (v >= 999).any(): out.add("retract:v=1e3")
        if p.n_point and np.any(case.delta[6*p.n_pose:6*p.n_pose + 3*p.n_point]): out.add("retract:point")
        if p.n_flow and np.any(case.delta[6*p.n_pose + 3*p.n_point:]): out.add("retract:flow")
        return out
    refs, _ = reference(case)
    out = set()
    types = [b.type for b in p.blocks]
    for bi, (b, r) in enumerate(zip(p.blocks, refs)):
        tr = r.trace
        near = {x for x in tr if x.startswith("close:")}
        if case.straddle:
            assert near, (case.name, "claims a straddle but no threshold is within a factor 2")
            out |= {"straddle:" + {"close:log": "log", "close:logpi": "logpi", "close:selog": "selog", "close:exp": "exp"}[x] for x in near}
            rot = [np.linalg.norm(r.b[f, :3]*b.sigma[:3]) for f in range(b.n)] if b.sigma.size >= 3 else []
            if "straddle:log" in out:
                out.discard("straddle:log")
                out.add("straddle:log_pi" if max(rot) > 3 else "straddle:log_taylor")
        else:
            assert not near, (case.name, TYPE_NAMES[b.type], near)
        out |= {x for x in tr if not x.startswith("close:") and not x.startswith("huber:")}
        out.add(f"F={b.n}:{TYPE_NAMES[b.type]}")
        if b.n > 1000: out.add(f"partials:{(b.n + 127)//128}")
        if b.robust_k > 0:
            k = b.robust_k; mode = "isotropic" if b.sigma_dim == 1 else "diagonal"
            n = np.linalg.norm(r.b, axis=1)                     # inside: |b| = |r_w|
            for f in range(b.n):
                if r.inside[f]:
                    for w, val in (("n==k", k), ("n=k-ulp", np.nextafter(k, -np.inf)), ("n=0", 0.0)):
                        if n[f] == val: out.add(f"huber:{w}:{mode}")
                else:
                    rw = n[f]**2/k                              # |b| = sqrt(k |r_w|)
                    if abs(rw - np.nextafter(k, np.inf)) <= 4*EPS*k: out.add(f"huber:n=k+ulp:{mode}")
                    if abs(rw - 10*k) <= 1e-12*k: out.add(f"huber:n=10k:{mode}")
            out.add(f"huber:k={k:g}".replace("0.0001", "1e-4").replace("1000", "1e3"))
            if DIM[b.type] == 6: out.add("huber:dim6")
            if DIM[b.type] == 2: out.add("huber:dim2")
        s = b.sigma.reshape(-1)
        if s.max()/s.min() >= 1e12: out.add("sigma:1e-6..1e6")
        if b.aux_idx is not None and b.n > 1 and (np.diff(b.aux_idx[:len(set(b.aux_idx))]) < 0).all(): out.add("gather:aux_reversed")
        for s_, c in enumerate(SLOT_CLASS[b.type]):
            if c == 0 and (b.idx[:, s_] == p.n_pose - 1).any(): out.add("gather:last_pose")
            if c == 1 and (b.idx[:, s_] == p.n_point - 1).any(): out.add("gather:last_point")
        if b.type == BETWEEN6 and (b.idx[:, 0] == b.idx[:, 1]).any(): out.add("gather:between_same_pose")
        if b.type == SMOOTH_POSE6 and (b.idx[:, 0] == b.idx[:, 2]).any(): out.add("gather:smooth_same_pose")
        if types.count(b.type) > 1: out.add("gather:blocks_of_one_type")
    return out


# ---------------------------------------------------------------------------------------------- comparator
def compare(case, bi, ref, A, b, e):
    """(err_b, err_A, err_e) of one block in units of the a-priori bound (module docstring); err_e relative"""
    ok = np.isfinite(ref.unit_b).all(1)             # (a depth of one denormal overflows 1/z: the branch taken is all there is)
    assert not (A[~ok] == 0).all((1, 2)).any(), "a factor in front of the camera took the cheirality branch"
    A, b, e, ref = A[ok], b[ok], e[ok], BlockRef(ref.A[ok], ref.b[ok], ref.e[ok], ref.unit_b[ok], ref.unit_A[ok], None, None, None, None)
    err_b = float((np.abs(b - ref.b)/ref.unit_b).max())
    err_A = float((np.abs(A - ref.A)/ref.unit_A[:, :, None]).max()) if case.check_A.get(bi, True) else 0.0
    err_e = float((np.abs(e - ref.e)/(((2*np.abs(ref.b) + ref.unit_b)*ref.unit_b).sum(1) + EPS*np.abs(ref.e))).max())
    return err_b, err_A, err_e


# tolerances in units of the a-priori bound (the metric of `compare`): worst measured per family in the docstring of
# tests/test_factors_gpu.py; `family` of a case is the prefix of its name
TOL = {"b": 16.0, "A": 64.0, "A_numeric": 16.0, "e": 8.0, "chi2": EPS}


def family(case):
    return case.name.split("_")[0]


def check_problem(case, linearization, factor_errors, chi2, label):
    """one implementation (`linearization(bi) -> (A, b)`, `factor_errors(bi) -> e`, `chi2`: its total error) against the
    50-digit reference of the case; prints one line per case and returns the worst errors"""
    p = case.problem
    refs, total = reference(case)
    worst = dict(b=0.0, A=0.0, A_numeric=0.0, e=0.0, e_rel=0.0)
    n_partials = 0
    for bi, (blk, ref) in enumerate(zip(p.blocks, refs)):
        A, b = linearization(bi); e = factor_errors(bi)
        fin = np.isfinite(ref.unit_b).all(1)
        # the discontinuous decisions, bit for bit: cheirality gives zero rows and 2 fx exactly, a Huber weight of
        # exactly 1 leaves the whitened residual untouched
        beh = ref.behind
        assert (A[beh] == 0).all() and np.array_equal(b[beh], ref.b[beh]), (case.name, TYPE_NAMES[blk.type], "cheirality")
        assert (np.abs(A[~beh & fin]).max((1, 2)) > 0).all() if (~beh & fin).any() else True, (case.name, "zero Jacobian in front of the camera")
        if case.bit_exact:
            assert np.array_equal(b[fin], ref.b[fin]), (case.name, TYPE_NAMES[blk.type], np.abs(b[fin] - ref.b[fin]).max())
            assert np.array_equal(e[fin], ref.e[fin]), (case.name, TYPE_NAMES[blk.type], "factor error")
        eb, eA, ee = compare(case, bi, ref, A, b, e)
        kA = "A_numeric" if blk.type in LR.NUMERIC_TYPES else "A"
        worst["b"] = max(worst["b"], eb); worst[kA] = max(worst[kA], eA); worst["e"] = max(worst["e"], ee)
        assert eb <= TOL["b"] and eA <= TOL[kA] and ee <= TOL["e"], (case.name, TYPE_NAMES[blk.type], eb, eA, ee)
        n_partials += (blk.n + 127)//128
        fe = np.isfinite(ref.e)
        worst["e_rel"] += float(np.abs(e[fe] - ref.e[fe]).sum())/max(total, 1e-300) if np.isfinite(total) else 0.0
    if np.isfinite(total):
        worst["chi2"] = abs(chi2 - total)/max(total, 1e-300) if total > 0 else abs(chi2)
        assert worst["chi2"] <= max(n_partials, 8)*TOL["chi2"] + worst["e_rel"], (case.name, chi2, total)
    print(f"FACTOR {label} {case.name}: b {worst['b']:.2g} A {worst['A']:.2g} A_numeric {worst['A_numeric']:.2g} "
          f"e {worst['e']:.2g} chi2 {worst.get('chi2', float('nan')):.2g}")
    return worst


def expmap_translation_bound(th):
    """Pose3::Expmap forms (omega x v - R (omega x v) + omega omega^T v)/theta^2: the first two terms, of size theta |v|,
    cancel to theta^2 |v|, so a faithful fp64 evaluation carries eps |v| (1 + 1/theta) above the first-order branch"""
    th = np.asarray(th, float)
    return np.where(th*th > EPS, 1 + 1/np.maximum(th, 1e-300), 1.0)


def retract_errors(case, pose, point, flow):
    """(|dR| / eps, |dt| / (eps (1 + |t| + |v| expmap_translation_bound)), |R^T R - I| / eps, |d point, flow|) after
    values.retract(delta)"""
    rp, rpt, rfl, _ = reference_retract(case)
    n = case.problem.n_pose
    xi = case.delta[:6*n].reshape(n, 6); th = np.linalg.norm(xi[:, :3], axis=1)
    S = 1 + np.abs(case.problem.pose[:, 9:]).max(1) + np.abs(xi[:, 3:]).max(1)*expmap_translation_bound(th)
    R = pose[:, :9].reshape(n, 3, 3)
    orth = np.abs(np.einsum("nij,nik->njk", R, R) - np.eye(3)).max()
    vec = max(np.abs(point - rpt).max() if point.size else 0.0, np.abs(flow - rfl).max() if flow.size else 0.0)
    return np.abs(pose[:, :9] - rp[:, :9]).max()/EPS, (np.abs(pose[:, 9:] - rp[:, 9:]).max(1)/(EPS*S)).max(), orth/EPS, vec
