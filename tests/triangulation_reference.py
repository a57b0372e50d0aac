"""A 50-digit statement of the triangulation of dynosam_b200/csrc/triangulate.cuh (gtsam::triangulateSafe with default
TriangulationParameters, then the stereo formulation's reprojection test), and an independent numpy statement of the
builder's STEREO_PROJECTION rules (Formulation-impl.hpp:258-411, 552-582).

DLT: A (2m x 4) has rows x_c P_c[2] - P_c[0] and y_c P_c[2] - P_c[1], P_c = K [R_c^T | -R_c^T t_c], formed exactly from
the double inputs; its singular values and right singular vectors come from mpmath's SVD at 50 digits."""
import mpmath as mp
import numpy as np

OK, DEGENERATE, BEHIND_CAMERA, OUTLIER = 0, 1, 2, 3
DPS = 50


def _mpf(x):
    return mp.mpf(float(x))


def dlt_matrix(poses, kp, K5):
    """A at 50 digits from double inputs (exact conversions)"""
    fx, fy, s, u0, v0 = (_mpf(k) for k in K5)
    Kmat = mp.matrix([[fx, s, u0], [0, fy, v0], [0, 0, 1]])
    rows = []
    for X, z in zip(np.asarray(poses).reshape(-1, 12), np.asarray(kp).reshape(-1, 2)):
        R = mp.matrix([[_mpf(X[3*i + j]) for j in range(3)] for i in range(3)])
        t = mp.matrix([_mpf(X[9 + i]) for i in range(3)])
        Rt = R.T
        M = mp.matrix(3, 4)
        mt = -(Rt*t)
        for i in range(3):
            for j in range(3):
                M[i, j] = Rt[i, j]
            M[i, 3] = mt[i]
        P = Kmat*M
        x, y = _mpf(z[0]), _mpf(z[1])
        rows.append([x*P[2, j] - P[0, j] for j in range(4)])
        rows.append([y*P[2, j] - P[1, j] for j in range(4)])
    return mp.matrix(rows)


def triangulate(poses, kp, K5, rank_tol=1.0, thr=3.0):
    """dict(status, point [3], reproj, sv [4] descending, kappa = sigma_1 / (sigma_3 - sigma_4), depths [m])"""
    with mp.workdps(DPS):
        m = np.asarray(kp).reshape(-1, 2).shape[0]
        out = dict(status=DEGENERATE, point=np.full(3, np.nan), reproj=np.nan, sv=np.full(4, np.nan), kappa=np.inf, depths=None)
        if m < 2:
            return out
        A = dlt_matrix(poses, kp, K5)
        _, S, Vt = mp.svd_r(A, compute_uv=True)
        order = sorted(range(4), key=lambda i: -S[i])
        sv = [S[i] for i in order]
        out["sv"] = np.array([float(x) for x in sv])
        out["kappa"] = float(sv[0]/(sv[2] - sv[3])) if sv[2] > sv[3] else np.inf
        rank = sum(1 for x in sv if x > rank_tol)
        if rank < 3:
            return out
        j = order[3]
        v = [Vt[j, i] for i in range(4)]
        if v[3] == 0:
            return out
        p = [v[i]/v[3] for i in range(3)]
        out["point"] = np.array([float(x) for x in p])
        fx, fy, s, u0, v0 = (_mpf(k) for k in K5)
        e2 = mp.mpf(0); depths = []
        for X, z in zip(np.asarray(poses).reshape(-1, 12), np.asarray(kp).reshape(-1, 2)):
            d = [p[i] - _mpf(X[9 + i]) for i in range(3)]
            q = [sum(_mpf(X[3*k + i])*d[k] for k in range(3)) for i in range(3)]      # R^T (p - t)
            depths.append(q[2])
            if q[2] > 0:
                x, y = q[0]/q[2], q[1]/q[2]
                e2 += (fx*x + s*y + u0 - _mpf(z[0]))**2 + (fy*y + v0 - _mpf(z[1]))**2
        out["depths"] = np.array([float(x) for x in depths])
        if min(depths) <= 0:
            out["status"] = BEHIND_CAMERA
            return out
        out["reproj"] = float(mp.sqrt(e2))
        out["status"] = OUTLIER if mp.sqrt(e2) > thr else OK
        return out


def point_bound(ref, c=64.0):
    """a-priori bound on |point - exact point| of a double DLT: c kappa eps |dv| propagated through v[0:3] / v[3]"""
    p = np.linalg.norm(ref["point"])
    return c*ref["kappa"]*np.finfo(np.float64).eps*(1.0 + p)*np.sqrt(1.0 + p*p)


# ----------------------------------------------------------------------------------------------- the builder's rules
def right_pose(X, b):
    """X * Pose3(I, (b, 0, 0)) as 12 doubles"""
    Y = np.array(X, np.float64).copy()
    Y[9:] = Y[9:] + b*Y[[0, 3, 6]]
    return Y


def stereo_graph(frames, obs, K6, tri):
    """The STEREO_PROJECTION static graph by the rules of Formulation-impl.hpp:258-411 applied frame by frame:
    frames {frame: X[12]}, obs list of (frame, tracklet, (uL, uR, v)), tri(poses, kp, K5) -> (status, point).  Returns
    dict(landmarks [tracklet in first-appearance order], points {tracklet: point}, factors {tracklet: [frames]},
    cameras {tracklet: (poses, kp) of the attempt that added it}, failed {status: attempts; OK: a valid point with fewer
    than two factors}, never [tracklets])."""
    tracks = {}
    for f, t, z in sorted(obs, key=lambda o: o[0]):                 # stable: insertion order inside a frame
        tracks.setdefault(t, []).append((f, np.asarray(z, np.float64)))
    added, points, factors, cameras, failed = {}, {}, {}, {}, {OK: 0, DEGENERATE: 0, BEHIND_CAMERA: 0, OUTLIER: 0}
    for k in sorted({f for f, _, _ in obs}):                        # frame k: every tracklet seen at k, not yet added
        for t, tr in tracks.items():
            seen = [o for o in tr if o[0] <= k]
            if t in added or not seen or seen[-1][0] != k:
                continue
            poses, kp = [], []
            for f, z in seen:
                poses.append(frames[f]); kp.append((z[0], z[2]))
                if not np.isnan(z[1]):
                    poses.append(right_pose(frames[f], K6[5])); kp.append((z[1], z[2]))
            st, pt = tri(np.array(poses), np.array(kp), K6[:5])
            if st != OK:
                failed[st] += 1
                continue
            good = [f for f, z in seen if z[0] - z[1] > 0.5]
            if len(good) < 2:
                failed[OK] += 1
                continue
            added[t] = k; points[t] = pt; factors[t] = list(good); cameras[t] = (np.array(poses), np.array(kp))
        for t, tr in tracks.items():                                # later observations of landmarks already in the graph
            if t in added and added[t] < k:
                factors[t] += [f for f, z in tr if f == k and not np.isnan(z[1])]
    land = [t for t in tracks if t in added]
    return dict(landmarks=land, points=points, factors=factors, cameras=cameras, failed=failed, never=[t for t in tracks if t not in added])
