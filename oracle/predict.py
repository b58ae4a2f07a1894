"""TEST INFRASTRUCTURE ONLY (oracle). Vecchia prediction for a Gaussian likelihood, observed data ordered first and the
prediction points conditioning on observed points only (the reference's default `vecchia_pred_type`
"order_obs_first_cond_obs_only"): numpy restatement of
  CalcPredVecchiaObservedFirstOrder(CondObsOnly = true)   src/GPBoost/Vecchia_utils.cpp:1701-2100
    neighbours of a prediction point = its m nearest OBSERVED points (:1784-1800, search restricted to indices < n),
    covariance blocks on the transformed scale with the nugget 1 on the neighbour block (:1940-1952),
    A_p = Sigma_NN^-1 Sigma_pN (:1960), D_p = v - A_p . Sigma_pN (:1925-1931, :1969), pred_mean = -B_po y = A_p y_N (:2061),
    pred_var = D_p (:2074);
  REModelTemplate::Predict back-transformation: variances times sigma^2, plus sigma^2 when the response is predicted
    (include/GPBoost/re_model_template.h:3427 ff.).
SURVEY §8 row f1 ("next"): the product does not export GPB_PredictREModel yet; this module and tests/golden/predict_golden.json
(reference outputs) are the target it will be built against. Pinned by tests/test_predict_oracle_pinned.py.
"""
import numpy as np

from . import vecchia as ov


def _cov(cid, dist, var, rt):
    if cid == 0:
        return var * np.exp(-rt * dist)
    if cid == 1:
        rd = rt * dist
        return var * (1. + rd) * np.exp(-rd)
    if cid == 2:
        rd = rt * dist
        return var * (1. + rd + rd * rd / 3.) * np.exp(-rd)
    return var * np.exp(-rt * dist * dist)


def predict_gaussian(coords_obs, y_obs, coords_pred, cov_pars, cov_function="matern", shape=1.5, num_neighbors=20,
                     predict_response=True, num_neighbors_pred=None):
    """Returns (mean, variance) at coords_pred. cov_pars = (sigma2, sigma1^2, rho) on the original scale. The neighbour sets
    come from the reference's walk over the observed points followed by the prediction points (find_nearest_neighbors_Vecchia_fast
    with start_at = end_search_at + 1 = n, Vecchia_utils.cpp:1784-1800), so distance ties are broken as the reference breaks them
    when coords_obs is in the model's Vecchia order (the order only matters for ties). The number of neighbours used for
    prediction defaults to TWICE the model's num_neighbors (re_model_template.h:299)."""
    if num_neighbors_pred is None:
        num_neighbors_pred = 2 * int(num_neighbors)
    num_neighbors = num_neighbors_pred
    coords_obs = np.asarray(coords_obs, dtype=np.float64)
    coords_pred = np.asarray(coords_pred, dtype=np.float64)
    n = coords_obs.shape[0]
    nbs = ov.knn_range(np.concatenate([coords_obs, coords_pred]), int(num_neighbors), n, n - 1)
    s2, pt = ov.transform_cov_pars(cov_pars, cov_function, shape)
    v, rt = float(pt[0]), float(pt[1])
    cid = ov.cov_id(cov_function, shape)
    mu = np.empty(coords_pred.shape[0]); var = np.empty(coords_pred.shape[0])
    for p in range(coords_pred.shape[0]):
        d = np.sqrt(((coords_obs - coords_pred[p]) ** 2).sum(1))
        nb = nbs[p]
        cn = coords_obs[nb]
        S = _cov(cid, np.sqrt(((cn[:, None, :] - cn[None, :, :]) ** 2).sum(-1)), v, rt)
        np.fill_diagonal(S, v + 1.)  # marginal variance + nugget (transformed scale)
        s = _cov(cid, d[nb], v, rt)
        A = np.linalg.solve(S, s)
        mu[p] = A @ y_obs[nb]
        Dp = v - A @ s
        var[p] = s2 * (Dp + (1. if predict_response else 0.))
    return mu, var
