"""numpy statement of the band selected inversion (csrc/kernels_cov.cu) and the dense covariance references of
dynoba_marginal_covariance.

Selected inversion.  S = L L^T in band_reference's plain layout: 32x32 tiles, tile (K, t) = block (K + t, K) for
t = 0..WB, NT tile columns, the bandwidth clamp of band_plan_layout, padding rows with a unit diagonal.  Sigma = S^-1 on
the same tiles, backward over the tile columns K = NT-1 ... 0 with B = K+1 .. min(K+WB, NT-1):

    Sigma(B,K) = -Sigma(B,B) L(B,K) L_KK^-1
    Sigma(K,K) = L_KK^-T (L_KK^-1 - L(B,K)^T Sigma(B,K))

Sigma(I,J) for I < J is the transpose of the stored tile (J, I).  The kernel forms the second line as the sum of the
per-tile products P = L(K+dd,K)^T Sigma(K+dd,K) and keeps the lower triangle of Sigma(K,K), mirrored.

Dense references.  ``marginal_blocks`` cuts the diagonal blocks of H^-1 for every variable kind out of an information
matrix in the column order [poses 6 | points 3 | flows 2 | velocities 3 | biases 6] (oracle.dense_normal and
Reference use the first three), inverted equilibrated so that a 1e-6-sigma prior keeps the other rows' digits.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla
import scipy.sparse as sp

import band_reference as BR

TILE = BR.TILE


def band_tiles(S, WB):
    """lower band tiles [NT][WB+1][32][32] of the dense symmetric S, padded to NT*32 with a unit diagonal"""
    n = S.shape[0]
    NT = max(-(-n//TILE), 1)
    P = np.eye(NT*TILE)
    P[:n, :n] = S
    T = np.zeros((NT, WB + 1, TILE, TILE))
    for K in range(NT):
        for t in range(min(WB, NT - 1 - K) + 1):
            T[K, t] = P[(K + t)*TILE:(K + t + 1)*TILE, K*TILE:(K + 1)*TILE]
    return T


def selinv(L):
    """Sigma tiles from the Cholesky factor's tiles L [NT][WB+1][32][32] (the recurrence above)"""
    NT, W1 = L.shape[:2]
    WB = W1 - 1
    Sg = np.zeros_like(L)

    def sig(I, J):
        return Sg[J, I - J] if I >= J else Sg[I, J - I].T
    for K in range(NT - 1, -1, -1):
        m = min(WB, NT - 1 - K)
        Li = sla.solve_triangular(np.tril(L[K, 0]), np.eye(TILE), lower=True)
        X = [-sum(sig(K + dd, J) @ L[K, J - K] for J in range(K + 1, K + m + 1)) @ Li for dd in range(1, m + 1)]
        M = Li - sum((L[K, dd].T @ X[dd - 1] for dd in range(1, m + 1)), np.zeros((TILE, TILE)))
        D = Li.T @ M
        Sg[K, 0] = np.tril(D) + np.tril(D, -1).T
        for dd in range(1, m + 1):
            Sg[K, dd] = X[dd - 1]
    return Sg


def factor_tiles(S, WB):
    """the Cholesky factor of S (padded) cut into the same tiles: the band layout holds L's whole envelope"""
    n = S.shape[0]
    NT = max(-(-n//TILE), 1)
    P = np.eye(NT*TILE)
    P[:n, :n] = S
    return band_tiles(np.linalg.cholesky(P), WB)


def tiles_entry(T, i, j):
    """entry (i, j) of the symmetric matrix whose lower band is stored in T"""
    if i < j:
        i, j = j, i
    return T[j//TILE, i//TILE - j//TILE, i % TILE, j % TILE]


def equilibrated_inverse(H):
    d = np.sqrt(np.abs(np.diag(H)))
    d[d == 0] = 1.0
    return np.linalg.inv(H/d[:, None]/d[None, :])/d[:, None]/d[None, :]


def marginal_blocks(Hinv, counts, kind, idx=None):
    """(n, d, d) diagonal blocks of Hinv for variables of `kind`, columns [poses | points | flows | vel | bias] with
    counts (n_pose, n_point, n_flow, n_vel, n_bias)"""
    dims = (6, 3, 2, 3, 6)
    base = np.concatenate([[0], np.cumsum([c*d for c, d in zip(counts, dims)])])
    d = dims[kind]
    idx = np.arange(counts[kind]) if idx is None else np.asarray(idx)
    cols = base[kind] + d*idx[:, None] + np.arange(d)[None, :]
    return Hinv[cols[:, :, None], cols[:, None, :]]


def schur_inverse_blocks(H, pcols, blocks):
    """diagonal blocks of H^-1 (sparse H) for the column lists `blocks`, through the Schur complement on the pose-like
    columns pcols: Sigma_pp = (Hpp - Hpl Hll^-1 Hlp)^-1 and Sigma_ll = Hll^-1 + Z Sigma_pp Z^T, Z = Hll^-1 Hlp -- for
    graphs too large for a dense inverse of H.  Column lists either lie in pcols or outside it.  Also returns
    kappa(D^-1/2 S D^-1/2), D = diag S, which the error of any backward-stable inverse scales with."""
    from schur_reference import _block_inverse
    H = sp.csr_matrix(H)
    n = H.shape[0]
    lcols = np.setdiff1d(np.arange(n), pcols)
    Hpp = H[pcols][:, pcols].toarray()
    Hpl = H[pcols][:, lcols].tocsr()
    Hll_inv = _block_inverse(H[lcols][:, lcols]).tocsr()
    Z = (Hll_inv @ Hpl.T).toarray()
    S = Hpp - Hpl @ Z
    S = 0.5*(S + S.T)
    Spp = equilibrated_inverse(S)
    d = np.sqrt(np.diag(S))
    ev = np.linalg.eigvalsh(S/d[:, None]/d[None, :])
    Y = Z @ Spp
    ploc = np.full(n, -1); ploc[pcols] = np.arange(len(pcols))
    lloc = np.full(n, -1); lloc[lcols] = np.arange(len(lcols))
    out = []
    for c in blocks:
        c = np.asarray(c)
        if ploc[c[0]] >= 0:
            q = ploc[c]; out.append(Spp[np.ix_(q, q)])
        else:
            q = lloc[c]; out.append(Hll_inv[q][:, q].toarray() + Y[q] @ Z[q].T)
    return np.array(out), float(ev.max()/ev.min())


def _all_pose_priors(p, sigma=1.0):
    import dataclasses
    from dynosam_b200.problem import PRIOR6, FactorBlock
    prior = FactorBlock(PRIOR6, np.arange(p.n_pose, dtype=np.int32)[:, None], p.pose.copy(), np.array([sigma]))
    return dataclasses.replace(p, blocks=list(p.blocks) + [prior])


def cov_graphs():
    """name -> builder of the full graphs test_covariance_gpu.py checks: together they reach every route of
    schur_reference.routes (test_covariance.py checks that)"""
    from dynosam_b200 import synth
    import schur_reference as SR
    return {
        # static (window NP = 1) and hybrid (window NP = 2) landmarks, Huber k = 1e-4: nearly every factor re-weighted
        "hybrid": lambda: SR._weak_priors(synth.make_problem(n_frames=30, n_objects=2, n_static=300, n_dynamic=120, seed=7,
                                                             object_span=(30, 30))),
        # T > WIN_TMAX, repeated poses, staged and unstaged groups, a flow star
        "simple": SR.simple_graph,
        "wcme": lambda: SR._weak_priors(synth.make_problem(n_frames=30, n_objects=1, n_static=100, n_dynamic=40,
                                                           formulation="wcme", seed=4, object_span=(30, 30),
                                                           max_dynamic_age=SR.GG_MAXL)),
        # schur_reference's WCPE graph is singular at lambda = 0 (LM only solves it damped): a unit prior on every pose
        # fixes its gauge
        "wcpe": lambda: _all_pose_priors(SR.general_wcpe_graph()),
        "imu": lambda: synth.make_problem(n_frames=12, n_objects=1, n_static=120, n_dynamic=60, seed=11, imu=True),
    }


def cov_error(C, Cref):
    """max over blocks and entries of |C_ab - Cref_ab| / sqrt(Cref_aa Cref_bb)"""
    d = np.sqrt(np.abs(np.diagonal(Cref, axis1=-2, axis2=-1)))
    return float((np.abs(C - Cref)/d[..., :, None]/d[..., None, :]).max(initial=0.0))
