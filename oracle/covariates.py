"""TEST INFRASTRUCTURE ONLY (oracle). Linear regression coefficients of the Gaussian Vecchia model, profiled out by GLS: a numpy
restatement on top of `vecchia.factor(...)` of what one objective evaluation of the reference computes with covariates
(ProfileOutCoef, include/GPBoost/re_model_template.h:2665-2683; UpdateCoefGLS :10012-10019; EvalLLforLBFGSpp, optim_utils.h:244-365):
    w_i = (B X)_i,  b_i = (B y0)_i,  y0 = y - offset (Vecchia order)
    G = sum D^-1_i w_i w_i^T = X^T Psi^-1 X,  r = sum D^-1_i w_i b_i = X^T Psi^-1 y0,  beta = G^-1 r
    NLL at the residual y0 - X beta with sigma^2 profiled (ProfileOutSigma2, :2640).
Also the closed-form initial coefficients of the iid model (InitCoefAuxParsFromIidModel, src/GPBoost/re_model.cpp:380-481: one
group, variances fixed at 1, Psi = I + 1 1^T) and the prediction mean with covariates (:11141-11160, :3576-3582).
"""
import numpy as np

from . import predict as op
from . import vecchia as ov


def b_apply(nn, A, Z):
    """(B Z) for Z (n,) or (n, p) in Vecchia order: Z_i - sum_k A_ik Z_nn(i,k), -1 padding skipped."""
    Z = np.asarray(Z, dtype=np.float64)
    out = Z.copy()
    for k in range(nn.shape[1]):
        j = nn[:, k]
        ok = j >= 0
        a = np.where(ok, A[:, k], 0.)
        zj = Z[np.where(ok, j, 0)]
        out -= (a[:, None] * zj) if Z.ndim == 2 else a * zj
    return out


def gram(nn, A, Dinv, Xo, y0o):
    """G = X^T Psi^-1 X and r = X^T Psi^-1 y0 for covariates Xo (n, p) and y0o (n,), both in Vecchia order."""
    W = b_apply(nn, A, Xo)
    b = b_apply(nn, A, y0o)
    Wd = W * Dinv[:, None]
    return Wd.T @ W, Wd.T @ b


def profiled(vo, pars_trans, y, X, offset=None):
    """One profiled evaluation at transformed (sigma1^2/sigma^2, range_t) for a VecchiaOracle `vo`; y, X, offset in the original
    order. Returns dict(G, r, beta, negll, sigma2)."""
    y0 = np.asarray(y, dtype=np.float64) - (0. if offset is None else np.asarray(offset, dtype=np.float64))
    X = np.asarray(X, dtype=np.float64).reshape(len(y0), -1)
    A, Dinv, _, _, _ = ov.factor(vo.coords, vo.nn, vo.cid, np.asarray(pars_trans, dtype=np.float64))
    Xo, y0o = X[vo.perm], y0[vo.perm]
    G, r = gram(vo.nn, A, Dinv, Xo, y0o)
    beta = np.linalg.solve(G, r)
    _, ypy, ld = ov.nll_from_factor(vo.nn, A, Dinv, y0o - Xo @ beta, 1.0)
    n = len(y0)
    s2 = ypy / n
    negll = ypy / 2. / s2 + ld / 2. + n / 2. * (np.log(s2) + np.log(2 * np.pi))
    return dict(G=G, r=r, beta=beta, negll=negll, sigma2=s2)


def profiled_at_cov_pars(vo, cov_pars, y, X, offset=None):
    """`profiled` at covariance parameters on the original scale (sigma2, sigma1^2, rho); sigma2 only fixes the ratio."""
    _, pt = ov.transform_cov_pars(cov_pars, vo.cov_function, vo.shape)
    return profiled(vo, pt, y, X, offset)


def iid_init_coef(y, X, offset=None):
    """Closed-form GLS with Psi = I + 1 1^T: Psi^-1 = I - 1 1^T / (n + 1)."""
    y0 = np.asarray(y, dtype=np.float64) - (0. if offset is None else np.asarray(offset, dtype=np.float64))
    X = np.asarray(X, dtype=np.float64).reshape(len(y0), -1)
    n = len(y0)
    s = X.sum(0)
    G = X.T @ X - np.outer(s, s) / (n + 1.)
    r = X.T @ y0 - s * y0.sum() / (n + 1.)
    return np.linalg.solve(G, r)


def predict_mean(coords_obs_ordered, y, X, beta, coords_pred, X_pred, cov_pars, cov_function, shape, num_neighbors, perm):
    """Predictive mean with covariates: GP part from the residual y - X beta, plus X_pred beta. coords_obs_ordered / perm: the
    model's Vecchia order (ties of the neighbour search are broken in that order)."""
    resid = np.asarray(y, dtype=np.float64) - np.asarray(X, dtype=np.float64).reshape(len(y), -1) @ beta
    mu, var = op.predict_gaussian(coords_obs_ordered, resid[perm], coords_pred, cov_pars, cov_function, shape, num_neighbors)
    return mu + np.asarray(X_pred, dtype=np.float64).reshape(len(mu), -1) @ beta, var
