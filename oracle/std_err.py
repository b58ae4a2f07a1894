"""TEST INFRASTRUCTURE ONLY (oracle). Standard errors of the Gaussian Vecchia model's covariance parameters.

numpy/scipy restatement of the reference's
  REModel::GetCovPar (calc_std_dev)        src/GPBoost/re_model.cpp:921-965
  CalcStdDevCovPar                         include/GPBoost/re_model_template.h:10788-10815
  CalcFisherInformation_Vecchia            include/GPBoost/re_model_template.h:10145-10230  (stochastic trace, no weights,
                                           transf_scale = false, include_error_var = true)
  GenRandVecNormalParallel                 src/GPBoost/CG_utils.cpp:978-994 (oracle.laplace.gen_rand_normal)
on top of the factor of the C restatement (oracle.vecchia.factor with calc_grad=True), which gives B, D^-1 and their derivatives
on the transformed scale (Psi = Sigma~ / sigma2, s = sigma1^2 / sigma2, derivatives w.r.t. log s and log rho_t).
Pinned against the reference library by tests/golden/make_std_err_golden.py -> tests/golden/std_err_golden.json.
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl

from . import laplace as ol
from . import vecchia as ov


def original_scale_factor(coords_ordered, nn, cid, cov_pars):
    """B, D and (B_grad_k, D_grad_k) for k = sigma1^2, rho on the ORIGINAL scale: CalcCovFactor(false, sigma2) and
    CalcGradientVecchia(false, sigma2, true) (Vecchia_utils.cpp:1386-1699, the !transf_scale branches at :1412, :1556, :1574,
    :1604), from the transformed-scale factor by B(Sigma~) = B(Psi), D_Sigma~ = sigma2 D_Psi:
      dB/dsigma1^2 = (dB/dlog s) / sigma1^2,   dD/dsigma1^2 = (dD_Psi/dlog s) / s,
      dB/drho = (dB/dlog rho_t) dlog rho_t/drho,  dD/drho = sigma2 (dD_Psi/dlog rho_t) dlog rho_t/drho,
    with rho_t = c / rho (Matern family, exponential) or 1 / rho^2 (Gaussian kernel), cov_fcts.h:485-623."""
    s2, s1, rho = [float(v) for v in cov_pars]
    _, pt = ov.transform_cov_pars(cov_pars, {0: "exponential", 1: "matern", 2: "matern", 3: "gaussian"}[cid],
                                  {0: 0.5, 1: 1.5, 2: 2.5, 3: 0.}[cid])
    A, Dinv, Ag, Dg, bad = ov.factor(coords_ordered, nn, cid, pt, calc_grad=True)
    n, m = nn.shape
    rows = np.repeat(np.arange(n), m)
    mask = nn.ravel() >= 0

    def pattern(vals):
        return sp.csr_matrix((vals.ravel()[mask], (rows[mask], nn.ravel()[mask])), shape=(n, n))

    B = ol.build_B(nn, A)
    D = s2 / Dinv
    dlog_rt = (-2. if cid == 3 else -1.) / rho
    dB = [pattern(-Ag[0] / s1), pattern(-Ag[1] * dlog_rt)]
    dD = [Dg[0] / pt[0], s2 * Dg[1] * dlog_rt]
    return B, D, dB, dD, bad


def fisher_info(coords_ordered, nn, cid, cov_pars, Z):
    """3 x 3 Fisher information (sigma2, sigma1^2, rho) of CalcFisherInformation_Vecchia (re_model_template.h:10145-10230) at the
    probe block Z (n x t, Vecchia order): W1 = B^-T Z, W2 = B^-1 D W1, S_k = B^T D^-1 (-dB_k W2 + dD_k W1) - dB_k^T W1,
    S_0 = B^T D^-1 B Z (the derivative w.r.t. the nugget is taken as the identity, :10172-10175), FI(a, b) = mean over the columns of
    sum_rows S_a .* S_b / 2."""
    B, D, dB, dD, _ = original_scale_factor(coords_ordered, nn, cid, cov_pars)
    Bt = B.T.tocsr()
    Dinv = 1. / D
    W1 = spl.spsolve_triangular(Bt, Z, lower=False, unit_diagonal=True)
    W2 = spl.spsolve_triangular(B, D[:, None] * W1, lower=True, unit_diagonal=True)
    S = [Bt @ (Dinv[:, None] * (B @ Z))]
    for k in range(2):
        S.append(Bt @ (Dinv[:, None] * (-(dB[k] @ W2) + dD[k][:, None] * W1)) - dB[k].T @ W1)
    FI = np.empty((3, 3))
    for a in range(3):
        for b in range(a, 3):
            FI[a, b] = FI[b, a] = (S[a] * S[b]).sum(0).mean() / 2.
    return FI


def std_dev_from_fi(FI):
    """sqrt(diag(FI^-1)) through a Cholesky factor (CalcStdDevCovPar, re_model_template.h:10800-10814): all NaN when the factorisation
    fails, NaN for a non-finite or negative diagonal entry."""
    out = np.full(FI.shape[0], np.nan)
    try:
        L = np.linalg.cholesky(FI)
    except np.linalg.LinAlgError:
        return out
    Linv = np.linalg.solve(L, np.eye(FI.shape[0]))
    d = (Linv * Linv).sum(0)
    ok = np.isfinite(d) & (d >= 0)
    out[ok] = np.sqrt(d[ok])
    return out


def probes(n, t, seed_rand_vec_trace=1, run_id=0):
    """rand_vec_fisher_info_: n x t, GenRandVecNormalParallel(seed_rand_vec_trace_, cg_generator_counter_) (:10151-10156)."""
    return ol.gen_rand_normal(seed_rand_vec_trace, run_id, n, t)


def std_err(coords, cov_pars, cov_function="matern", cov_fct_shape=1.5, num_neighbors=20, vecchia_ordering="random", seed=0,
            num_rand_vec_trace=50, seed_rand_vec_trace=1, run_id=0):
    """What GPModel.get_cov_pars(std_err=True) reports as the standard errors for a Gaussian Vecchia model with parameters
    cov_pars (original scale): returns (std_dev, FI)."""
    vo = ov.VecchiaOracle(coords, num_neighbors=num_neighbors, cov_function=cov_function, cov_fct_shape=cov_fct_shape,
                          vecchia_ordering=vecchia_ordering, seed=seed)
    Z = probes(vo.n, num_rand_vec_trace, seed_rand_vec_trace, run_id)
    FI = fisher_info(vo.coords, vo.nn, vo.cid, cov_pars, Z)
    return std_dev_from_fi(FI), FI
