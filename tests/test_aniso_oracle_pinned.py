"""CPU tests pinning the restatement of the anisotropic Vecchia GP (tests/aniso_oracle.py) to the reference's goldens
(tests/golden/aniso_golden.json), and the coordinate-share identity the device gradient uses to the kernels' element formulas."""
import json
import os

import numpy as np
import pytest

import aniso_oracle as ao

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "aniso_golden.json")


@pytest.fixture(scope="module")
def gold():
    return {c["name"]: c for c in json.load(open(GOLDEN))["cases"]}


def test_golden_grid_covers_the_cases(gold):
    assert set(gold) == {c["name"] for c in ao.CASES}
    parsed = [ao.parse(c["cov"], c["shape"]) for c in ao.CASES]
    assert {s for f, s in parsed if f == "matern_ard"} >= {0.5, 1.5, 2.5}
    assert {f for f, _ in parsed} == {"matern_ard", "gaussian_ard", "matern_space_time"}
    assert {c["m"] for c in ao.CASES} >= {10, 20, 30, 45, 60}
    assert {c["ordering"] for c in ao.CASES} >= {"time", "time_random_space"}
    # the reference searches the sets at the parameters of each evaluation: theta2 gives the same value after theta1 as on a fresh model
    assert all(g["nll_t2_same"] == g["nll_t2_fresh"] for g in gold.values())


@pytest.mark.parametrize("case", [c["name"] for c in ao.CASES])
def test_oracle_reproduces_golden_likelihoods(gold, case):
    c = next(x for x in ao.CASES if x["name"] == case)
    X, y, _ = ao.case_data(c)
    t1, t2 = ao.thetas(c)
    o = ao.AnisoOracle(X, c["m"], c["cov"], c["shape"], c["ordering"], c["seed"])
    g = gold[case]
    assert abs(o.neg_log_likelihood(t1, y) - g["nll_t1"]) <= 1e-8 * abs(g["nll_t1"])
    assert abs(o.neg_log_likelihood(t2, y) - g["nll_t2_same"]) <= 1e-8 * abs(g["nll_t2_same"])  # sets frozen at theta1
    o2 = ao.AnisoOracle(X, c["m"], c["cov"], c["shape"], c["ordering"], c["seed"])
    assert abs(o2.neg_log_likelihood(t2, y) - g["nll_t2_fresh"]) <= 1e-8 * abs(g["nll_t2_fresh"])


def test_initial_values_equal_the_maxit0_golden(gold):
    c = next(x for x in ao.CASES if x.get("maxit") == 0)
    X, y, _ = ao.case_data(c)
    o = ao.AnisoOracle(X, c["m"], c["cov"], c["shape"], c["ordering"], c["seed"])
    want = ao.init_cov_pars(o.coords, y, o.cov_function, o.shape)
    np.testing.assert_allclose(want, gold[c["name"]]["cov_pars"], rtol=1e-10)


@pytest.mark.parametrize("cov,shape,d", [("matern_ard", 0.5, 3), ("matern_ard", 1.5, 2), ("matern_ard", 2.5, 5), ("gaussian_ard", 0., 3),
                                         ("matern_space_time", 1.5, 3)])
def test_share_identity_equals_element_formulas(cov, shape, d):
    """dk/dlog(lambda_c) = (dk/dlog(lambda))_iso(r) S_c / r^2 on scaled coordinates, 0 at r = 0"""
    rng = np.random.default_rng(d)
    dx = rng.standard_normal((500, d))
    dx[:5] = 0.
    C = 2 if cov == "matern_space_time" else d
    lam = rng.uniform(0.5, 5., C)
    k, dk = ao.kernel_and_grads(dx, cov, shape, lam)
    dxs = dx * ao.scale_factors(lam, cov, d)
    r2 = (dxs ** 2).sum(-1)
    r = np.sqrt(r2)
    e = np.exp(-r)
    if cov == "gaussian_ard":
        giso = -r2 * np.exp(-r2)
    elif shape == 0.5:
        giso = -r * e
    elif shape == 1.5:
        giso = -r2 * e
    else:
        giso = -r2 / 3. * (1. + r) * e
    g = ao.groups(cov, d)
    share = np.stack([(dxs ** 2)[:, g == c].sum(-1) for c in range(C)], -1)
    with np.errstate(invalid="ignore", divide="ignore"):
        ident = np.where(r2[:, None] > 0, giso[:, None] * share / r2[:, None], 0.)
    np.testing.assert_allclose(ident, dk, rtol=0, atol=1e-13)


@pytest.mark.parametrize("cov,shape,d,m", [("matern_ard", 1.5, 2, 10), ("gaussian_ard", 0., 3, 8), ("matern_space_time", 0.5, 3, 12)])
def test_oracle_gradient_equals_central_differences(cov, shape, d, m):
    rng = np.random.default_rng(m)
    n = 150
    X = rng.uniform(0., 1., (n, d))
    y = rng.standard_normal(n)
    cf, sh = ao.parse(cov, shape)
    C = 2 if cf == "matern_space_time" else d
    cp = np.concatenate([[0.2, 1.0], rng.uniform(0.1, 0.5, C)])
    o = ao.AnisoOracle(X, m, cov, shape, "random", 1)
    o.search(cp)
    _, g = o.grad_profiled(cp, y)
    s2, var, lam = ao.transform(cp, cf, sh)
    x0 = np.log(np.concatenate([[var], lam]))

    def f(x):  # profiled likelihood at fixed sets, as a function of log(var ratio), log(lambda)
        lam_ = np.exp(x[1:])
        rho = 1. / np.sqrt(lam_) if cf == "gaussian_ard" else ao.MULT[sh] / lam_
        return o.grad_profiled(np.concatenate([[1., np.exp(x[0])], rho]), y)[0]
    h = 1e-5
    num = np.array([(f(x0 + h * np.eye(len(x0))[k]) - f(x0 - h * np.eye(len(x0))[k])) / (2 * h) for k in range(len(x0))])
    np.testing.assert_allclose(g, num, rtol=1e-5, atol=1e-5)
