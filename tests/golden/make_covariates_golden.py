"""Generates tests/golden/covariates_golden.json with the UNMODIFIED reference library (oracle/_ref) through the shared frontend:
Gaussian Vecchia GP with linear regression covariates, GPB_OptimLinRegrCoefCovPar ("wls": coefficients profiled out by GLS),
GPB_GetCoef, and prediction with X_pred. Every case records the fitted covariance parameters, coefficients, negative
log-likelihood and iteration count; the prediction (mean and response variance, 100 points) is made by a second model that holds
the fitted coefficients (init_coef, maxit = 0) at the fitted covariance parameters, so that it depends on them only; it is
given y - offset as its response.
Run from the repository root after building oracle/_ref:  python tests/golden/make_covariates_golden.py"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import datagen  # noqa: E402
from gpboost_b200 import GPModel  # noqa: E402
from gpboost_b200.libpath import load_lib  # noqa: E402
from oracle import ref_lib_path  # noqa: E402

# kernels x neighbour counts x number of covariates (p = 1: intercept only); one case each with an offset, init_coef,
# init_cov_pars, maxit = 0, and a mean large against the noise
CASES = [
    dict(n=2000, dseed=11, cov_function="matern", shape=1.5, m=10, seed=1, p=1),
    dict(n=3000, dseed=12, cov_function="exponential", shape=0.5, m=30, seed=2, p=2, offset=True),
    dict(n=2500, dseed=13, cov_function="matern", shape=2.5, m=45, seed=3, p=5),
    dict(n=1500, dseed=14, cov_function="gaussian", shape=0., m=10, seed=4, p=2, init_cov_pars=[0.3, 0.8, 0.2]),
    dict(n=4000, dseed=15, cov_function="matern", shape=1.5, m=30, seed=5, p=40),
    dict(n=1500, dseed=16, cov_function="exponential", shape=0.5, m=10, seed=6, p=3, init_coef=[0.5, -1.0, 2.0]),
    dict(n=1500, dseed=17, cov_function="matern", shape=1.5, m=10, seed=7, p=2, maxit=0),
    dict(n=2000, dseed=18, cov_function="matern", shape=2.5, m=30, seed=8, p=2, big_mean=True),
]


def case_data(c):
    """coords, y, X (n x p, first column 1), offset or None, prediction coords and X_pred (100 points)"""
    coords, y = datagen.synth(c["n"], 2, c["dseed"])
    rng = np.random.default_rng(c["dseed"] + 100)
    p = c["p"]
    X = np.ones((c["n"], p))
    X[:, 1:] = rng.standard_normal((c["n"], p - 1))
    beta = np.concatenate([[1e5 if c.get("big_mean") else 1.5], rng.uniform(-2., 2., p - 1)])
    y = y + X @ beta
    offset = 0.3 * np.cos(5 * coords[:, 1]) if c.get("offset") else None
    if offset is not None:
        y = y + offset
    cp = rng.random((100, 2))
    Xp = np.ones((100, p))
    Xp[:, 1:] = rng.standard_normal((100, p - 1))
    return coords, y, X, offset, cp, Xp


def model(c, coords, lib=None):
    kw = {} if lib is None else dict(_lib=lib)
    return GPModel(gp_coords=coords, cov_function=c["cov_function"], cov_fct_shape=c["shape"], gp_approx="vecchia",
                   num_neighbors=c["m"], vecchia_ordering="random", seed=c["seed"], **kw)


def fit_params(c):
    params = {}
    if "init_cov_pars" in c:
        params["init_cov_pars"] = np.array(c["init_cov_pars"])
    if "init_coef" in c:
        params["init_coef"] = np.array(c["init_coef"])
    if "maxit" in c:
        params["maxit"] = c["maxit"]
    return params


if __name__ == "__main__":
    ref = load_lib(ref_lib_path())
    out = {"generator": "tests/golden/make_covariates_golden.py", "cases": []}
    for c in CASES:
        coords, y, X, offset, cp, Xp = case_data(c)
        m = model(c, coords, ref)
        m.fit(y, X=X, params=fit_params(c), offset=offset)
        rec = dict(c)
        rec["cov_pars"] = m.get_cov_pars().tolist()
        rec["coef"] = m.get_coef().tolist()
        try:
            rec["negll"] = m.get_current_neg_log_likelihood()
        except Exception:  # maxit = 0: the reference has no estimate
            rec["negll"] = None
        rec["num_it"] = m._get_num_optim_iter()
        mp = model(c, coords, ref)
        yo = y - (0. if offset is None else offset)
        mp.fit(yo, X=X, params=dict(init_coef=np.array(rec["coef"]), maxit=0))
        r = mp.predict(yo, cp, np.array(rec["cov_pars"]), predict_var=True, predict_response=True, X_pred=Xp)
        rec["mu_head"] = r["mu"][:32].tolist(); rec["mu_sum"] = float(r["mu"].sum())
        rec["var_head"] = r["var"][:32].tolist(); rec["var_sum"] = float(r["var"].sum())
        print(c["cov_function"], c["m"], c["p"], rec["num_it"], rec["negll"], rec["cov_pars"], rec["coef"][:3])
        out["cases"].append(rec)
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "covariates_golden.json"), "w") as f:
        json.dump(out, f, indent=1)
