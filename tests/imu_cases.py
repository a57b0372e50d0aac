"""The case list of the visual-inertial factors: small `Problem`s of COMBINED_IMU15 / PRIOR_VEL3 / PRIOR_BIAS6 blocks, each
naming the branch boundaries and block-size edges it reaches (`hits`), their 50-digit reference (tests/imu_lie_reference.py)
and the one comparator both the host build (tests/test_imu_cases.py) and the device (tests/test_imu_cases_gpu.py) are
held to.  A CPU test checks that every name of `REQUIRED` is reached.

Construction.  Each IMU factor is built from the quantities that pick the branches: the bias-correction angle
theta = |delRdelBiasOmega dbw| (delRdelBiasOmega a rotation times -1, so |JRw| = 1), the angle of
phi = Log(dR Exp(theta)) (dR = Exp(phi) Exp(theta)^-1 in 50 digits), and the residual rotation r = Log(R_p^T R_j)
(R_j = R_p Exp(r)); positions and velocities of frame j sit a chosen small offset from the prediction.  Every input is
rounded once to fp64, and that fp64 record is the case's exact input.  Values of a block may be tiled: `pick[bi][f]` is
the distinct factor that slot f copies, and the reference evaluates each distinct factor once.

Comparator, in units of an a-priori bound, as tests/factor_cases.py:

    b:  |db_i| / (eps B sum_k |R_ik| (|r|_inf + S_k))          A:  |dA_ij| / (eps B sum_k |R_ik| (max_j |J_kj| + S_k))

S_k is the size of the terms that cancel in row k of the unwhitened residual:
    rotation rows  1;
    position rows  1 + |t_i| + |t_j| + |dPc| + dt |v_i| + dt^2 |g| / 2;
    velocity rows  1 + |v_i| + |v_j| + |dVc| + dt |g|;
    bias rows      1 + |b_i| + |b_j|;
and the whitening goes through |R|.  B is 1 for closed forms and, where a Logmap is involved, the largest of
`lie_reference.log_rot_bound / 8` of the two Logmaps (phi and r: pi eps/(pi - theta)^2 towards pi) and, for the
Jacobian, `imu_lie_reference.jr_inv_bound` of |r|: GTSAM's (1 + cos)/(2 theta sin) carries eps pi/(2 (pi - theta)) near
pi.  Where phi or r takes Logmap's pi branch, the formula misses the true Logmap by ~(pi - theta), so the closed-form
Jacobian (a function of the formula's phi and r) is not the true derivative to any eps bound: those blocks compare the
residual and the error only (`check_A`, with the reason in `note`).
"""
from dataclasses import dataclass, field

import numpy as np
from mpmath import mp, mpf

import imu_lie_reference as IL
import lie_reference as LR
from dynosam_b200.problem import COMBINED_IMU15, PRIOR_BIAS6, PRIOR_VEL3, FactorBlock, Problem

EPS = 2.0**-52
G_DOWN = np.array([0.0, 0.0, -9.81])
G_TILT = np.array([0.6, -0.8, -9.75])
THETAS = ["0", "1e-9", "0.999e-5", "1.001e-5", "2e-5", "1e-4", "3e-4", "1e-3", "0.3", "2.5", "pi-1e-3"]
IMU_SIZES = [1, 3, 4, 5, 8, 9, 127, 128, 129]
PRIOR_SIZES = [1, 127, 128, 129, 257]
PHI_HITS = ["log:pi", "logpi:z", "logpi:y", "logpi:x", "log:acos", "log:taylor", "log:acos_near_pi", "log:acos_near_taylor",
            "log:taylor_near_acos", "log:identity", "straddle:log_taylor", "straddle:log_pi"]
RES_HITS = ["zero", "0.999e-5", "1.001e-5", "straddle:log_taylor", "pi-1e-3", "pi-5e-6"]

REQUIRED = (
    [f"theta:{t}" for t in THETAS] + [f"phi:{h}" for h in PHI_HITS] + [f"res:{h}" for h in RES_HITS]
    + [f"dt:{d:g}" for d in (0.0, 1e-3, 0.1, 5.0)] + ["g:0", "g:down", "g:tilted", "t:1e3", "dba:0", "bias:equal"]
    + ["R:cholesky", "R:diagonal", "R:dense", "R:scale1e-3", "R:scale1e6", "R:bcast", "R:per_factor"]
    + [f"prior:{k}:{w}" for k in ("VEL3", "BIAS6") for w in ("sigma_dim1", "sigma_dimD", "bcast", "per_factor", "zero")]
    + ["prior:sigma:1e-6..1e6"]
    + [f"imu:F={n}" for n in IMU_SIZES] + [f"prior:{k}:F={n}" for k in ("VEL3", "BIAS6") for n in PRIOR_SIZES]
    + ["partials:1024", "partials:1025", "shuffled"])


@dataclass
class Case:
    name: str
    problem: Problem
    hits: tuple
    pick: dict = field(default_factory=dict)          # block index -> [n] distinct factor of each slot (values tiled)
    check_A: dict = field(default_factory=dict)       # block index -> False: the Jacobian is not compared (see `note`)
    note: str = ""


def theta_of(s):
    return mp.pi - mpf(s[3:]) if s.startswith("pi-") else (mp.pi if s == "pi" else mpf(s))


def unit(v):
    v = LR.vec(v); n = LR.norm(v)
    return [x/n for x in v]


def f64(x):
    return np.array(LR.to_float(x))


# ---------------------------------------------------------------------------------------------- one factor
JR_AXIS = (0.48, 0.6, -0.64)
JRW_ROT = LR.exp_so3([mpf("0.9")*x for x in unit((0.2, -1.0, 0.5))])       # delRdelBiasOmega = -this (|JRw| = 1)


def build_factor(rng, Xi, vi, bi_acc, bh, theta="1e-3", phi="0.3", phi_axis=(0.3, -0.5, 0.8), res="1e-3", res_axis=(0.6, 0.0, 0.8),
                 offset=1e-2, dt=0.1, g=G_DOWN, dba_zero=False, bias_equal=False):
    """(z[70], X_j[12], v_j[3], b_i[6], b_j[6]) of one factor from frame i = (X_i[12], v_i[3]); `theta`, `phi`, `res`:
    the three angles (strings: 'pi-1e-3' ...); `offset`: size of R_p^T (p_j - p_p) and R_p^T (v_j - v_p)"""
    JRw = f64([-x for x in JRW_ROT])
    th_t = [theta_of(theta)*x for x in unit(JR_AXIS)]
    # dbw = JRw^-1 theta = -JRW_ROT^T theta; b_i.gyro = biasHat.gyro + dbw
    dbw = LR.mv3(LR.tr3([-x for x in LR.vec(JRw)]), th_t) if theta != "0" else [mpf(0)]*3
    bg = bh[3:] + f64(dbw) if theta != "0" else bh[3:].copy()
    ba = bh[:3].copy() if dba_zero else bi_acc
    bi = np.concatenate([ba, bg])
    bj = bi.copy() if bias_equal else bi + rng.normal(0, 0.01, 6)
    th = LR.mv3(LR.vec(JRw), [mpf(float(a)) - mpf(float(b)) for a, b in zip(bg, bh[3:])])
    Rc = LR.exp_so3([theta_of(phi)*x for x in unit(phi_axis)]) if phi != "0" else list(LR.I3)
    dR = f64(LR.mul3(Rc, LR.tr3(LR.exp_so3(th)))) if not (phi == "0" and theta == "0") else np.eye(3).ravel()
    z = np.concatenate([dR, rng.normal(0, 0.3, 3)*dt, rng.normal(0, 0.5, 3)*dt, [dt], bh, JRw,
                        rng.normal(0, 0.05, 36)*max(dt, 1e-2), g])
    # frame j from the 50-digit prediction of the rounded record
    Xm = LR.pose(Xi); P = IL.parts(Xm, LR.vec(vi), Xm, LR.vec(vi), LR.vec(bi), LR.vec(bj), z)
    Rp = P["Rp"]
    Rr = LR.exp_so3([theta_of(res)*x for x in unit(res_axis)]) if res != "0" else list(LR.I3)
    Rj = LR.mul3(Rp, Rr)
    ep = LR.vec(rng.normal(0, 1, 3)*offset); ev = LR.vec(rng.normal(0, 1, 3)*offset)
    tj = [a + b for a, b in zip(P["pp"], LR.mv3(Rp, ep))]
    vj = [a + b for a, b in zip(P["vp"], LR.mv3(Rp, ev))]
    return z, f64(Rj + tj), f64(vj), bi, bj


def sqrt_info(kind, rng, scale=1.0):
    """15 x 15 square-root information: 'cholesky' (upper triangular, what GTSAM passes), 'diagonal', 'dense' (full,
    not triangular: used as given)"""
    d = scale*np.exp(rng.uniform(-1, 1, 15))
    if kind == "diagonal":
        return np.diag(d)
    M = rng.normal(0, 0.3, (15, 15))
    if kind == "cholesky":
        return np.triu(M, 1)*d[None, :] + np.diag(d)
    return (M + np.eye(15))*d[:, None]


class Chain:
    """frames (pose, velocity, bias) and IMU factors between them"""

    def __init__(self, seed, tmag=1.0):
        self.rng = np.random.default_rng(seed)
        self.tmag = tmag
        self.pose, self.vel, self.bias, self.fac = [], [], [], []

    def frame(self):
        rng = self.rng
        R = f64(LR.exp_so3([mpf(float(rng.uniform(0.3, 1.2)))*x for x in unit(rng.normal(size=3))]))
        t = rng.normal(size=3); t *= self.tmag/np.linalg.norm(t)
        self.pose.append(np.concatenate([R, t])); self.vel.append(rng.normal(0, 1, 3))
        self.bias.append(np.concatenate([rng.normal(0, 0.05, 3), rng.normal(0, 0.01, 3)]))
        return len(self.pose) - 1

    def factor(self, i=None, **kw):
        """one factor from frame i (a new frame when None) to a new frame j"""
        rng = self.rng
        i = self.frame() if i is None else i
        bh = np.concatenate([rng.normal(0, 0.05, 3), [0.0078125, -0.00390625, 0.001953125]])
        z, Xj, vj, bi, bj = build_factor(rng, self.pose[i], self.vel[i], self.bias[i][:3], bh, **kw)
        self.bias[i] = bi
        self.pose.append(Xj); self.vel.append(vj); self.bias.append(bj)
        j = len(self.pose) - 1
        self.fac.append(([i, i, j, j, i, j], z))
        return j

    def block(self, R, facs=None, order=None):
        facs = self.fac if facs is None else facs
        order = np.arange(len(facs)) if order is None else order
        idx = np.array([facs[k][0] for k in order]); z = np.array([facs[k][1] for k in order])
        sig = R.reshape(-1) if R.ndim == 2 else R[order].reshape(len(order), 225)
        return FactorBlock(COMBINED_IMU15, idx, z, sig)

    def problem(self, blocks):
        return Problem(np.array(self.pose), np.zeros((0, 3)), blocks=blocks, vel=np.array(self.vel), bias=np.array(self.bias))


def _single(name, specs, hits, R="diagonal", scale=1.0, seed=1, tmag=1.0, per_factor=False, **kw):
    """one IMU block of independent factors, one per spec"""
    ch = Chain(seed, tmag)
    for s in specs:
        ch.factor(**s)
    rng = np.random.default_rng(seed + 1000)
    Rm = np.array([sqrt_info(R, rng, scale) for _ in specs]) if per_factor else sqrt_info(R, rng, scale)
    return Case(name, ch.problem([ch.block(Rm)]), tuple(hits), **kw)


# ---------------------------------------------------------------------------------------------- cases
def angle_cases():
    out = []
    # theta: the gyro-bias Jacobian through Jr(theta).  |JRw| = 1, a small residual and a diagonal R, so that the rotation
    # rows' gyro columns carry Jr(theta)'s rounding unmixed
    out.append(_single("theta", [dict(theta=t, res="1e-7", offset=1e-7, bias_equal=True) for t in THETAS],
                       [f"theta:{t}" for t in THETAS] + ["bias:equal", "R:diagonal", "R:bcast"]))
    # phi = Log(dR Exp(theta)): every so3_logmap branch; phi near pi is a fast spin over a long interval
    spec = [("0", (0, 0, 1)), ("1e-9", (0.6, 0.8, 0)), ("2e-4", (1, 1, 1)), ("5e-4", (1, 1, 1)), ("0.3", (0.6, 0.8, 0)),
            ("2.5", (1, 1, 1)), ("pi-1e-3", (0, 1, 0)), ("pi-3e-5", (0.6, 0.8, 0.005))]
    out.append(_single("phi", [dict(phi=p, phi_axis=a, theta="0" if p == "0" else "1e-3") for p, a in spec],
                       ["phi:log:identity", "phi:log:taylor", "phi:log:acos", "phi:log:acos_near_pi", "phi:log:acos_near_taylor",
                        "phi:log:taylor_near_acos"], seed=2))
    out.append(_single("phi_straddle", [dict(phi=p, phi_axis=(0.6, 0.48, 0.64)) for p in ("3.1622776e-4", "pi-1e-5")],
                       ["phi:straddle:log_taylor", "phi:straddle:log_pi"], seed=3, check_A={0: False},
                       note="phi within rounding of tr + 1 = 1e-10: the pi-branch side misses the true Logmap by (pi - theta)"))
    pis = [("pi-5e-6", (0.6, 0.0, 0.8)), ("pi-5e-6", (0.6, 0.8, 0.0)), ("pi-5e-6", (1, 0, 0)), ("pi-1e-8", (1, 0, 0)), ("pi", (0, 1, 0))]
    out.append(_single("phi_pi", [dict(phi=p, phi_axis=a) for p, a in pis], ["phi:log:pi", "phi:logpi:z", "phi:logpi:y", "phi:logpi:x"],
                       seed=4, check_A={0: False},
                       note="phi in Logmap's pi branch: Exp(phi) misses dR Exp(theta) by (pi - theta), residual only"))
    # the residual rotation: zero, |r|^2 straddling so3_jr_inv's 1e-10, the Taylor / acos boundary, near pi
    out.append(_single("res", [dict(res=r, bias_equal=True, offset=o) for r, o in
                               (("0", 0.0), ("0.999e-5", 1e-6), ("1.001e-5", 1e-6), ("3.1622776e-4", 1e-3), ("pi-1e-3", 1e-2))],
                       ["res:zero", "res:0.999e-5", "res:1.001e-5", "res:straddle:log_taylor", "res:pi-1e-3"], seed=5))
    out.append(_single("res_pi", [dict(res="pi-5e-6", res_axis=a) for a in ((0.6, 0.0, 0.8), (0.6, 0.8, 0.0), (1, 0, 0))],
                       ["res:pi-5e-6"], seed=6, check_A={0: False},
                       note="r in Logmap's pi branch: the formula's r misses the true one by (pi - theta), so does Jr^-1(r)"))
    return out


def input_cases():
    out = []
    specs = [dict(dt=d, g=g) for d in (0.0, 1e-3, 0.1, 5.0) for g in (np.zeros(3), G_DOWN, G_TILT)]
    out.append(_single("dt_g", specs, [f"dt:{d:g}" for d in (0.0, 1e-3, 0.1, 5.0)] + ["g:0", "g:down", "g:tilted"], seed=7))
    out.append(_single("far", [dict(dba_zero=True), dict(theta="0.3", dt=5.0)], ["t:1e3", "dba:0"], seed=8, tmag=1e3))
    # square-root information: upper-triangular Cholesky, diagonal, dense non-triangular; scales 1e-3 .. 1e6
    for R in ("cholesky", "dense"):
        out.append(_single(f"R_{R}", [dict() for _ in range(3)], [f"R:{R}", "R:per_factor"], R=R, seed=9, per_factor=True))
    for s, h in ((1e-3, "R:scale1e-3"), (1e6, "R:scale1e6")):
        out.append(_single(f"R_scale{s:g}", [dict() for _ in range(2)], [h, "R:cholesky", "R:bcast"], R="cholesky", scale=s, seed=10))
    return out


def _prior_block(kind, n, rng, sig_dim, bcast, span=False, zero=False, x=None):
    D = 3 if kind == PRIOR_VEL3 else 6
    m = x[np.arange(n) % len(x)].copy() if zero else rng.normal(0, 1, (n, D))
    if span:
        s = np.geomspace(1e-6, 1e6, D if sig_dim != 1 else n)
        sig = s if sig_dim != 1 else s[:, None]
    else:
        sig = np.exp(rng.uniform(-2, 2, sig_dim if bcast else (n, sig_dim)))
    if not bcast and sig.ndim == 1:
        sig = np.tile(sig, (n, 1))
    return FactorBlock(kind, np.arange(n)[:, None] % len(x), m, sig)


def prior_cases():
    out = []
    rng = np.random.default_rng(11)
    ch = Chain(12); ch.factor()
    for k in range(3):
        ch.frame()
    x = {PRIOR_VEL3: np.array(ch.vel), PRIOR_BIAS6: np.array(ch.bias)}
    for kind, nm in ((PRIOR_VEL3, "VEL3"), (PRIOR_BIAS6, "BIAS6")):
        D = 3 if kind == PRIOR_VEL3 else 6
        blocks = [_prior_block(kind, 5, rng, 1, True, x=x[kind]), _prior_block(kind, 5, rng, D, True, x=x[kind]),
                  _prior_block(kind, 5, rng, 1, False, x=x[kind]), _prior_block(kind, 5, rng, D, False, span=True, x=x[kind]),
                  _prior_block(kind, 5, rng, 1, False, span=True, x=x[kind]), _prior_block(kind, 5, rng, D, True, zero=True, x=x[kind])]
        out.append(Case(f"prior_{nm}", ch.problem(blocks),
                        tuple(f"prior:{nm}:{w}" for w in ("sigma_dim1", "sigma_dimD", "bcast", "per_factor", "zero")) + ("prior:sigma:1e-6..1e6",)))
    return out


def block_cases():
    """block-size edges: values tiled with period 7 over a chain, so every copy of a distinct factor must come back
    bit-identical to it (the device checks that against the factor alone at n = 1)"""
    out = []
    ch = Chain(13)
    j = None
    for k in range(7):
        j = ch.factor(j, theta=["1e-4", "2e-5", "0.3", "0", "1e-3", "2.5", "3e-4"][k], phi=["0.3", "1e-3", "2.5", "0.7", "1.0", "0.1", "2.0"][k])
    R = sqrt_info("cholesky", np.random.default_rng(14))
    x = {PRIOR_VEL3: np.array(ch.vel), PRIOR_BIAS6: np.array(ch.bias)}
    rng = np.random.default_rng(15)
    for n in IMU_SIZES:
        order = np.arange(n) % 7
        out.append(Case(f"blocks_imu{n}", ch.problem([ch.block(R, order=order)]), (f"imu:F={n}",), pick={0: order}))
    for n in PRIOR_SIZES:
        blocks = [_prior_block(PRIOR_VEL3, n, rng, 1, True, x=x[PRIOR_VEL3]), _prior_block(PRIOR_BIAS6, n, rng, 6, False, x=x[PRIOR_BIAS6])]
        out.append(Case(f"blocks_prior{n}", ch.problem(blocks), (f"prior:VEL3:F={n}", f"prior:BIAS6:F={n}"), pick={}))
    # 1024 and 1025 partial sums of 0.5 |r_w|^2 reach the final reduction (4 IMU factors per CTA)
    for n, h in ((4096, "partials:1024"), (4097, "partials:1025")):
        order = np.arange(n) % 7
        out.append(Case(f"big_imu{n}", ch.problem([ch.block(R, order=order)]), (h,), pick={0: order}))
    # one block in shuffled order: linearization() and factor_errors() come back in the caller's order
    order = np.random.default_rng(16).permutation(np.arange(21) % 7)
    out.append(Case("blocks_shuffled", ch.problem([ch.block(R, order=order)]), ("shuffled",), pick={0: order}))
    return out


def _build():
    cases = angle_cases() + input_cases() + prior_cases() + block_cases()
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
    unit_b: np.ndarray     # [n, dim]
    unit_A: np.ndarray     # [n, dim]
    trace: set
    e_mp: object           # the block's error summed in 50 digits
    b_alt: np.ndarray      # [n, dim] b through the other branch of a straddled phi (else b)


_FACTOR_CACHE = {}


def _R(blk, f):
    return blk.sigma.reshape(15, 15) if blk.sigma_bcast else blk.sigma[f].reshape(15, 15)


def imu_factor(p, blk, f, with_A=True):
    """reference of IMU factor f of block blk: (A, b, e, unit_b, unit_A, hits, e_mp)"""
    i0, v0, i1, v1, b0, b1 = blk.idx[f]
    xs = [p.pose[i0], p.vel[v0], p.pose[i1], p.vel[v1], p.bias[b0], p.bias[b1]]
    R = _R(blk, f); z = blk.meas[f]
    key = (with_A, np.concatenate(xs + [z, R.ravel()]).tobytes())
    if key in _FACTOR_CACHE:
        return _FACTOR_CACHE[key]
    Xi, Xj = LR.pose(xs[0]), LR.pose(xs[2])
    a = [Xi, LR.vec(xs[1]), Xj, LR.vec(xs[3]), LR.vec(xs[4]), LR.vec(xs[5])]
    tr = {}
    P = IL.parts(*a, z, maps="gtsam", trace=tr)
    Rm = [LR.vec(row) for row in R]
    A, bb, e = IL.linearized(*a, z, Rm, with_A)
    r = np.array(LR.to_float(P["r"]))
    hits = set()
    # bounds
    B_phi = float(LR.log_rot_bound(P["Rc"]))/8; B_res = float(LR.log_rot_bound(P["E"]))/8
    th_r = float(LR.norm(P["r"][:3]))
    B = max(1.0, B_phi, B_res)
    BA = max(B, float(IL.jr_inv_bound(th_r))/8)
    dt = abs(z[15]); g = np.abs(z[67:70]).max(); nrm = lambda v: np.abs(np.asarray(v, float)).max()
    S = np.ones(15)
    S[3:6] = 1 + nrm(xs[0][9:]) + nrm(xs[2][9:]) + nrm(LR.to_float(P["dPc"])) + dt*nrm(xs[1]) + dt*dt*g/2
    S[6:9] = 1 + nrm(xs[1]) + nrm(xs[3]) + nrm(LR.to_float(P["dVc"])) + dt*g
    S[9:15] = 1 + nrm(xs[4]) + nrm(xs[5])
    aR = np.abs(R)
    b_alt = None
    if "close:log" in tr["phi"]:
        # phi within rounding of a threshold: either neighbouring branch, to the bound of the acos side (both straddles
        # of lie_reference: theta^5/30 at the Taylor side, 3e-5 at the pi side)
        ph = float(LR.norm(P["phi"]))
        other = ("acos" if "log:pi" in tr["phi"] else "pi") if ph > 3 else ("acos" if "log:taylor" in tr["phi"] else "taylor")
        ra = IL.parts(*a, z, maps="gtsam", phi_force=other)["r"]
        b_alt = np.array(LR.to_float([-x for x in IL.whiten(ra, Rm)[0]]))
        c = (P["Rc"][0] + P["Rc"][4] + P["Rc"][8] - 1)/2
        B = max(B, float(8 + 4*mp.pi/(mp.pi - mp.acos(max(min(c, 1), -1)))**2)/8)
    unit_b = EPS*B*(aR@(np.abs(r).max() + S))
    if with_A:
        Af = np.array(LR.to_float(A))
        Jmax = np.abs(np.linalg.solve(R, Af)).max(1)                    # max_j |J_kj| of the unwhitened rows
        unit_A = EPS*BA*(aR@(Jmax + S))
    else:
        Af = np.zeros((15, 30)); unit_A = np.full(15, np.inf)
    # hits
    thf = np.linalg.norm(np.array(z[22:31]).reshape(3, 3)@(xs[4][3:] - z[19:22]))
    for t in THETAS:
        want = float(theta_of(t))
        if (thf == 0 and want == 0) or (want > 0 and abs(thf - want) <= 1e-6*want):
            hits.add(f"theta:{t}")
    phi = np.array(LR.to_float(P["phi"])); ph = np.linalg.norm(phi)
    tp = tr["phi"]; trr = tr["res"]
    hits |= {"phi:" + x for x in tp if not x.startswith("close:") and x in PHI_HITS}
    if "log:acos" in tp and np.pi - ph < 1e-4: hits.add("phi:log:acos_near_pi")
    if "log:acos" in tp and ph < 1e-3: hits.add("phi:log:acos_near_taylor")
    if "log:taylor" in tp and ph > 1e-4: hits.add("phi:log:taylor_near_acos")
    if (phi == 0).all(): hits.add("phi:log:identity")
    if "close:log" in tp: hits.add("phi:straddle:" + ("log_pi" if ph > 3 else "log_taylor"))
    if np.abs(r[:3]).max() <= 1e-14: hits.add("res:zero")
    for nm, v in (("0.999e-5", 0.999e-5), ("1.001e-5", 1.001e-5), ("pi-1e-3", np.pi - 1e-3)):
        if abs(th_r - v) <= 1e-3*min(v, np.pi - v): hits.add("res:" + nm)
    if "log:pi" in trr and "close:log" not in trr: hits.add("res:pi-5e-6")       # (the pi branch's angle is pi itself)
    if "close:log" in trr and th_r < 1: hits.add("res:straddle:log_taylor")
    hits.add(f"dt:{z[15]:g}")
    gz = z[67:70]
    hits.add("g:0" if not gz.any() else ("g:down" if gz[0] == 0 and gz[1] == 0 else "g:tilted"))
    if min(np.linalg.norm(xs[0][9:]), np.linalg.norm(xs[2][9:])) >= 999: hits.add("t:1e3")
    if np.array_equal(xs[4][:3], z[16:19]): hits.add("dba:0")
    if np.array_equal(xs[4], xs[5]): hits.add("bias:equal")
    if np.count_nonzero(R - np.diag(np.diag(R))) == 0: hits.add("R:diagonal")
    elif np.count_nonzero(np.tril(R, -1)) == 0: hits.add("R:cholesky")
    elif np.count_nonzero(np.triu(R, 1)) and np.count_nonzero(np.tril(R, -1)): hits.add("R:dense")
    dmed = np.median(np.abs(np.diag(R)))
    if dmed < 1e-2: hits.add("R:scale1e-3")
    if dmed > 1e5: hits.add("R:scale1e6")
    bf = np.array(LR.to_float(bb))
    out = (Af, bf, float(e), unit_b, np.maximum(unit_A, 1e-300), hits, e, r, bf if b_alt is None else b_alt)
    _FACTOR_CACHE[key] = out
    return out


def prior_factor(p, blk, f):
    """(A, b, e, unit_b, unit_A, hits, e_mp): r = x - m, whitened by 1/sigma"""
    D = 3 if blk.type == PRIOR_VEL3 else 6
    x = (p.vel if blk.type == PRIOR_VEL3 else p.bias)[blk.idx[f, 0]]
    s = np.ones(D)*(blk.sigma if blk.sigma_bcast else blk.sigma[f])
    r = [mpf(float(a)) - mpf(float(b)) for a, b in zip(x, blk.meas[f])]
    rw = [v/mpf(float(sg)) for v, sg in zip(r, s)]
    e = LR.dot(rw, rw)/2
    isg = 1.0/s
    A = np.diag(isg); b = np.array(LR.to_float([-v for v in rw]))
    unit_b = EPS*(np.abs(b) + EPS*isg*(np.abs(x) + np.abs(blk.meas[f])))*2
    return A, b, float(e), unit_b, np.full(D, EPS), set(), e, None, b


def reference(case):
    """[BlockRef] of the case's problem and its chi^2 summed in 50 digits (as a float)"""
    p = case.problem
    refs, total = [], mpf(0)
    for bi, blk in enumerate(p.blocks):
        pick = case.pick.get(bi, np.arange(blk.n))
        first = {}
        for f, d in enumerate(pick):
            first.setdefault(int(d), f)
        with_A = case.check_A.get(bi, True)
        rows = {d: (imu_factor(p, blk, f, with_A) if blk.type == COMBINED_IMU15 else prior_factor(p, blk, f)) for d, f in first.items()}
        st = lambda k: np.array([rows[int(d)][k] for d in pick])
        trace = set().union(*(r[5] for r in rows.values()))
        e_mp = sum((rows[int(d)][6] for d in pick), mpf(0))
        refs.append(BlockRef(st(0), st(1), st(2), st(3), st(4), trace, e_mp, st(8)))
        total += e_mp
    return refs, float(total)


def boundaries(case):
    """what the case really reaches, by the 50-digit classifier and the shape of its blocks"""
    p = case.problem
    refs, _ = reference(case)
    out = set()
    for bi, (blk, ref) in enumerate(zip(p.blocks, refs)):
        out |= ref.trace
        if blk.type == COMBINED_IMU15:
            out.add("R:bcast" if blk.sigma_bcast else "R:per_factor")
            out.add(f"imu:F={blk.n}")
            if blk.n > 4000: out.add(f"partials:{(blk.n + 3)//4}")
            pick = case.pick.get(bi)
            if pick is not None and (np.diff(pick) < 0).any() and len(set(pick.tolist())) == 7 and blk.n == 21: out.add("shuffled")
        else:
            nm = "VEL3" if blk.type == PRIOR_VEL3 else "BIAS6"
            D = 3 if blk.type == PRIOR_VEL3 else 6
            out.add(f"prior:{nm}:F={blk.n}")
            out.add(f"prior:{nm}:" + ("sigma_dim1" if blk.sigma_dim == 1 else "sigma_dimD" if blk.sigma_dim == D else "?"))
            out.add(f"prior:{nm}:" + ("bcast" if blk.sigma_bcast else "per_factor"))
            if (ref.b == 0).all(): out.add(f"prior:{nm}:zero")
            if blk.sigma.max()/blk.sigma.min() >= 1e12: out.add("prior:sigma:1e-6..1e6")
    return out


# ---------------------------------------------------------------------------------------------- comparator
TOL = {"b": 16.0, "A": 16.0, "e": 8.0}


def n_partials(blk):
    return (blk.n + 3)//4 if blk.type == COMBINED_IMU15 else (blk.n + 127)//128


def check_problem(case, linearization, factor_errors, chi2, label, tol=TOL):
    """one implementation (`linearization(bi) -> (A, b)`, `factor_errors(bi) -> e`, `chi2`) against the 50-digit
    reference; the priors bit for bit (b, A) and the IMU bias rows bit for bit where b_i == b_j.  Returns the worst errors."""
    p = case.problem
    refs, total = reference(case)
    worst = dict(b=0.0, A=0.0, e=0.0, chi2=0.0)
    npart, e_rel = 0, 0.0
    for bi, (blk, ref) in enumerate(zip(p.blocks, refs)):
        A, b = linearization(bi); e = factor_errors(bi)
        if blk.type != COMBINED_IMU15:
            D = b.shape[1]
            x = (p.vel if blk.type == PRIOR_VEL3 else p.bias)[blk.idx[:, 0]]
            sg = np.broadcast_to(blk.sigma, (blk.n, blk.sigma.shape[-1])) if blk.sigma_bcast else blk.sigma
            isg = np.broadcast_to(1.0/sg, (blk.n, D))
            assert np.array_equal(b, -(x - blk.meas)*isg), (case.name, bi, "prior b")
            assert np.array_equal(A, np.einsum("ni,ij->nij", isg, np.eye(D))), (case.name, bi, "prior A")
            if (ref.b == 0).all():
                assert (e == 0).all() and not np.signbit(e).any()
        else:
            eq = np.array([np.array_equal(p.bias[blk.idx[f, 4]], p.bias[blk.idx[f, 5]]) for f in range(blk.n)])
            # b_i == b_j: the bias rows of r are exact zeros, and so are those of R r where R[9:, :9] = 0 (diagonal or
            # upper-triangular R), bit for bit
            Rs = np.broadcast_to(blk.sigma.reshape(-1, 15, 15), (blk.n, 15, 15))
            m = np.array([np.array_equal(p.bias[blk.idx[f, 4]], p.bias[blk.idx[f, 5]]) and not Rs[f][9:, :9].any()
                          for f in range(blk.n)])
            assert (b[m][:, 9:] == 0).all(), (case.name, "bias rows with b_i == b_j")
            err_b = np.minimum(np.abs(b - ref.b), np.abs(b - ref.b_alt))/ref.unit_b
            worst["b"] = max(worst["b"], float(err_b.max()))
            if case.check_A.get(bi, True):
                err_A = np.abs(A - ref.A)/ref.unit_A[:, :, None]
                worst["A"] = max(worst["A"], float(err_A.max()))
        e_alt = 0.5*(ref.b_alt*ref.b_alt).sum(1)
        err_e = np.minimum(np.abs(e - ref.e), np.abs(e - e_alt))/(((2*np.abs(ref.b) + ref.unit_b)*ref.unit_b).sum(1) + EPS*np.abs(ref.e))
        worst["e"] = max(worst["e"], float(err_e.max()))
        npart += n_partials(blk)
        e_rel += float(np.abs(e - ref.e).sum())/max(total, 1e-300)
    worst["chi2"] = abs(chi2 - total)/max(total, 1e-300)
    print(f"IMU {label} {case.name}: b {worst['b']:.2g} A {worst['A']:.2g} e {worst['e']:.2g} chi2 {worst['chi2']:.2g}")
    assert worst["b"] <= tol["b"] and worst["A"] <= tol["A"] and worst["e"] <= tol["e"], (case.name, worst)
    assert worst["chi2"] <= npart*EPS + e_rel, (case.name, chi2, total)
    return worst
