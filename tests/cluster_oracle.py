"""Restatement of the Gaussian Vecchia GP with independent realizations (cluster_ids) on top of the oracle (oracle/vecchia.py): Ψ is
block diagonal, so every cluster is searched and factored on its own (the reference calls find_nearest_neighbors_Vecchia_fast and
CalcCovFactorGradientVecchia once per cluster) and the likelihood sums and gradient sums add up over the clusters."""
import numpy as np

from oracle import vecchia as ov


def cluster_rows(lab, perm=None):
    """rows (original indices) of every cluster, clusters in order of first appearance; within a cluster the data order, or the order of
    `perm` (an engine's ordered position -> original index) when given"""
    labels = list(dict.fromkeys(np.asarray(lab).tolist()))
    if perm is None:
        return [np.flatnonzero(lab == l) for l in labels]
    perm = np.asarray(perm)
    return [perm[lab[perm] == l] for l in labels]


def cluster_knn(coords_c, m):
    """neighbour sets of one cluster (local indices, -1 padded to the reference's cap min(m, |c| - 1), width at least 1)"""
    nc = coords_c.shape[0]
    if nc == 1:
        return np.full((1, 1), -1, dtype=np.int32)
    return np.ascontiguousarray(ov.knn_range(coords_c, m, 0, nc - 2), dtype=np.int32)


def clustered(coords, lab, y, m, cov_function, shape, cov_pars, perm=None, calc_grad=False):
    """per cluster (rows, nn, A, Dinv) and the totals: negll, y^T Psi^-1 y, log|Psi| and, with calc_grad, the gradient w.r.t.
    log(sigma_1^2 / sigma^2) and log(range) at sigma^2 = cov_pars[0] (the formula of the Vecchia gradient, sums over the clusters)"""
    s2, pt = ov.transform_cov_pars(cov_pars, cov_function, shape)
    cid = ov.cov_id(cov_function, shape)
    parts, ypy, ld, grad = [], 0., 0., np.zeros(2)
    for rows in cluster_rows(lab, perm):
        cs = np.ascontiguousarray(coords[rows])
        yc = np.ascontiguousarray(y[rows], dtype=np.float64)
        nn = cluster_knn(cs, m)
        A, Dinv, Ag, Dg, _ = ov.factor(cs, nn, cid, pt, calc_grad=calc_grad)
        _, q, l = ov.nll_from_factor(nn, A, Dinv, yc, 1.0)
        ypy += q
        ld += l
        if calc_grad:
            grad += ov.grad_from_factor(nn, A, Dinv, Ag, Dg, yc, s2)
        parts.append((rows, nn, A, Dinv))
    n = len(y)
    negll = ypy / 2. / s2 + ld / 2. + n / 2. * (np.log(s2) + np.log(2. * np.pi))
    return dict(parts=parts, negll=negll, ypy=ypy, logdet=ld, grad=grad if calc_grad else None)
