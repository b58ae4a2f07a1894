"""The oracle's restatement of the profiled objective with covariates (oracle/covariates.py) against the reference's own fits
(tests/golden/covariates_golden.json, made by tests/golden/make_covariates_golden.py): at each golden case's fitted covariance
parameters the GLS coefficients and the profiled negative log-likelihood reproduce the reference's, and at maxit = 0 the reference's
initial coefficients are the closed-form GLS of the iid model (Psi = I + 1 1^T). CPU only."""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_covariates_golden as mk  # noqa: E402
from oracle import covariates as oc  # noqa: E402
from oracle import vecchia as ov  # noqa: E402

with open(os.path.join(HERE, "golden", "covariates_golden.json")) as f:
    GOLD = json.load(f)["cases"]
FITTED = [i for i, c in enumerate(GOLD) if c.get("maxit", 1) > 0]


def oracle_of(c, coords):
    return ov.VecchiaOracle(coords, c["m"], c["cov_function"], c["shape"], "random", c["seed"])


def test_golden_covers_the_issue_grid():
    assert {c["cov_function"] + str(c["shape"]) for c in GOLD} >= {"matern1.5", "matern2.5", "exponential0.5", "gaussian0.0"}
    assert {c["m"] for c in GOLD} >= {10, 30, 45}
    assert {c["p"] for c in GOLD} >= {1, 2, 5, 40}
    assert any(c.get("offset") for c in GOLD) and any("init_coef" in c for c in GOLD)
    assert any("init_cov_pars" in c for c in GOLD) and any(c.get("maxit") == 0 for c in GOLD)


@pytest.mark.parametrize("idx", FITTED)
def test_profiled_coefficients_and_negll_at_the_reference_fit(idx):
    c = GOLD[idx]
    coords, y, X, offset, _, _ = mk.case_data(c)
    res = oc.profiled_at_cov_pars(oracle_of(c, coords), c["cov_pars"], y, X, offset)
    coef = np.array(c["coef"])
    assert np.abs(res["beta"] - coef).max() <= 1e-8 * np.abs(coef).max(), (res["beta"], coef)
    assert abs(res["negll"] - c["negll"]) <= 1e-8 * abs(c["negll"]), (res["negll"], c["negll"])
    assert abs(res["sigma2"] - c["cov_pars"][0]) <= 1e-8 * c["cov_pars"][0]


def test_initial_coefficients_are_the_iid_gls():
    for c in GOLD:
        if c.get("maxit") != 0:
            continue
        coords, y, X, offset, _, _ = mk.case_data(c)
        want = oc.iid_init_coef(y, X, offset)
        assert np.abs(np.array(c["coef"]) - want).max() <= 1e-10 * np.abs(want).max(), (c["coef"], want)


def test_gram_matches_dense_gls():
    """G, r of the sparse restatement equal X^T Psi^-1 X, X^T Psi^-1 y with Psi^-1 = B^T D^-1 B formed densely"""
    coords, y = np.random.default_rng(3).random((300, 2)), np.random.default_rng(4).standard_normal(300)
    X = np.random.default_rng(5).standard_normal((300, 4))
    vo = ov.VecchiaOracle(coords, 12, "matern", 1.5, "random", 2)
    A, Dinv, _, _, _ = ov.factor(vo.coords, vo.nn, vo.cid, np.array([1.7, np.sqrt(3.) / 0.2]))
    G, r = oc.gram(vo.nn, A, Dinv, X[vo.perm], y[vo.perm])
    B = np.eye(300)
    for i in range(300):
        for k in range(vo.nn.shape[1]):
            if vo.nn[i, k] >= 0:
                B[i, vo.nn[i, k]] -= A[i, k]
    P = B.T @ np.diag(Dinv) @ B
    Xo, yo = X[vo.perm], y[vo.perm]
    assert np.allclose(G, Xo.T @ P @ Xo, rtol=1e-12, atol=1e-12 * np.abs(G).max())
    assert np.allclose(r, Xo.T @ P @ yo, rtol=1e-12, atol=1e-12 * np.abs(r).max())
