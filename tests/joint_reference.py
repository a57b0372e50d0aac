"""numpy statement of dynoba_joint_marginal_covariance (csrc/kernels_cov.cu: the band sweeps; csrc/kernels_chain.cu: the
landmark strips; csrc/api.cu: the assembly).

Sweeps.  S = L L^T in band_reference's plain layout (selinv_reference.factor_tiles: tile (K, t) = block (K + t, K),
t = 0..WB).  E_C holds the unit columns of the requested scalars C (ascending).  L^-1 E_C is zero above min(C), so both
sweeps run over the tile columns [J0, NT), J0 = min(C) // 32:

    forward   Y_J = L_JJ^-1 (E_J - sum_{t=1..WB} L(J, J-t) Y_{J-t})          J = J0 .. NT-1
    backward  X_J = L_JJ^-T (Y_J - sum_{t=1..WB} L(J+t, J)^T X_{J+t})      J = NT-1 .. J0

and X[C, C] is read off.

Landmark strips.  H = [[U, W], [W^T, V]] over pose-like variables P and landmarks, V block diagonal per landmark group g
(a point alone, a WCME / WCPE chain, a flow), S = U - W V^-1 W^T.  C = the requested pose-like variables and every pose
a requested landmark's group touches.  For a requested landmark l of group g:

    M_l = (W V_g^-1)[C, l]            Z_l = Sigma(l, C) = -M_l^T X[C, C]
    Sigma(l1, l2) = delta_{g1 g2} (V_g^-1)(l1, l2) - Z_l1 M_l2

The assembly writes the lower triangle of the D x D result in caller order and mirrors it.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

TILE = 32


def sweeps(L, cs):
    """(X[C, C], X) for the factor tiles L [NT][WB+1][32][32] and the ascending scalar list cs: X = S^-1 E_C on rows
    >= 32 J0 (rows above the span are left 0: they are never computed)"""
    NT, W1 = L.shape[:2]
    WB = W1 - 1
    cs = np.asarray(cs)
    nc = cs.size
    J0 = int(cs[0])//TILE
    Y = np.zeros((NT, TILE, nc))
    for J in range(J0, NT):
        Z = np.zeros((TILE, nc))
        hit = cs//TILE == J
        Z[cs[hit] % TILE, np.flatnonzero(hit)] = 1.0
        for t in range(1, min(WB, J - J0) + 1):
            Z -= L[J - t, t] @ Y[J - t]
        Y[J] = sla.solve_triangular(np.tril(L[J, 0]), Z, lower=True)
    for J in range(NT - 1, J0 - 1, -1):
        Z = Y[J].copy()
        for t in range(1, min(WB, NT - 1 - J) + 1):
            Z -= L[J, t].T @ Y[J + t]
        Y[J] = sla.solve_triangular(np.tril(L[J, 0]).T, Z, lower=False)
    X = Y.reshape(NT*TILE, nc)
    return X[cs], X


def landmark_groups(H, lcols):
    """the landmark groups of H: connected components of V = H[lcols, lcols]; returns the group of every column of lcols"""
    V = sp.csr_matrix(H)[lcols][:, lcols]
    return connected_components(V != 0, directed=False)[1]


def joint_covariance(H, pcols, lcols, request, factor=None):
    """the D x D joint covariance of the variables `request` (a list of column lists of H, caller order; each lies in
    pcols or in lcols) by the route above.  factor(S) -> (L tiles, WB) defaults to selinv_reference.factor_tiles over
    the whole envelope."""
    import selinv_reference as SI
    H = sp.csr_matrix(H)
    pcols, lcols = np.asarray(pcols), np.asarray(lcols)
    n = H.shape[0]
    ploc = np.full(n, -1); ploc[pcols] = np.arange(pcols.size)
    lloc = np.full(n, -1); lloc[lcols] = np.arange(lcols.size)
    U = H[pcols][:, pcols].toarray()
    W = H[pcols][:, lcols].toarray()
    V = H[lcols][:, lcols].toarray()
    grp = landmark_groups(H, lcols)
    ginv = {}
    for g in np.unique(grp):
        m = np.flatnonzero(grp == g)
        ginv[g] = (m, np.linalg.inv(V[np.ix_(m, m)]))
    Vinv = np.zeros_like(V)
    for m, vi in ginv.values():
        Vinv[np.ix_(m, m)] = vi
    S = U - W @ Vinv @ W.T
    S = 0.5*(S + S.T)
    # C: requested pose-like scalars and every pose scalar the requested groups' factors touch
    inC = np.zeros(pcols.size, bool)
    req_groups = set()
    for c in request:
        c = np.asarray(c)
        if ploc[c[0]] >= 0:
            inC[ploc[c]] = True
        else:
            req_groups.add(int(grp[lloc[c[0]]]))
    for g in req_groups:
        m = ginv[g][0]
        inC |= np.abs(W[:, m]).sum(axis=1) != 0
    cs = np.flatnonzero(inC)
    if factor is None:
        NT = max(-(-S.shape[0]//TILE), 1)
        L = SI.factor_tiles(S, NT - 1)
    else:
        L = factor(S)
    Xcc, _ = sweeps(L, cs)
    cpos = np.full(pcols.size, -1); cpos[cs] = np.arange(cs.size)
    M, Z = {}, {}
    for c in request:
        c = np.asarray(c)
        if lloc[c[0]] < 0:
            continue
        q = lloc[c]
        Ml = (W @ Vinv[:, q])[cs]                  # (W V_g^-1)[C, l]: W's rows outside C are zero for the group
        M[c[0]] = Ml
        Z[c[0]] = -Ml.T @ Xcc
    dims = [len(c) for c in request]
    off = np.concatenate([[0], np.cumsum(dims)])
    out = np.zeros((off[-1], off[-1]))
    for a, ca in enumerate(request):
        ca = np.asarray(ca)
        for b, cb in enumerate(request[:a + 1]):
            cb = np.asarray(cb)
            pa, pb = ploc[ca[0]] >= 0, ploc[cb[0]] >= 0
            if pa and pb:
                blk = Xcc[np.ix_(cpos[ploc[ca]], cpos[ploc[cb]])]
            elif not pa and pb:
                blk = Z[ca[0]][:, cpos[ploc[cb]]]
            elif pa and not pb:
                blk = Z[cb[0]][:, cpos[ploc[ca]]].T
            else:
                ga, gb = grp[lloc[ca[0]]], grp[lloc[cb[0]]]
                blk = (Vinv[np.ix_(lloc[ca], lloc[cb])] if ga == gb else 0.0) - Z[ca[0]] @ M[cb[0]]
            out[off[a]:off[a + 1], off[b]:off[b + 1]] = blk
    i, j = np.tril_indices(off[-1], -1)
    out[j, i] = out[i, j]
    return out
