"""Pins tests/laplace_poisson_oracle.py (poisson likelihood, log link, latent Vecchia GP) against the golden vectors of the unmodified
reference library (tests/golden/make_laplace_poisson_golden.py): the iterative Laplace likelihood (same probe vectors), the
reference's Newton iteration count, its gradient and its L-BFGS fit. Bars are those of tests/test_laplace_oracle_pinned.py."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import poisson_data
import laplace_poisson_oracle as olp
from oracle import vecchia as ov

HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(HERE, "golden", "laplace_poisson_golden.json")) as f:
    GOLD = json.load(f)["cases"]


def oracle(c, grad=False, cov_pars=None, **kw):
    X, y, off = poisson_data.case_data(c)
    vo = ov.VecchiaOracle(X, c["m"], c["cov_function"], c["shape"], c["ordering"], c["seed"])
    th = c["cov_pars"] if cov_pars is None else cov_pars
    _, pt = ov.transform_cov_pars([1.0] + list(th), c["cov_function"], c["shape"])
    f = olp.grad_negll if grad else olp.negll
    return f(vo.coords, vo.nn, vo.cid, th[0], pt[1], y[vo.perm], fixed_effects=None if off is None else off[vo.perm],
             method="iterative", num_rand_vec_trace=c["t"], **kw)


def test_golden_cases_cover_the_intended_data():
    names = {c["name"]: c for c in GOLD}
    assert {(c["cov_function"], c["shape"]) for c in GOLD} >= {("exponential", 0.5), ("matern", 1.5), ("matern", 2.5)}
    assert {c["m"] for c in GOLD} >= {10, 20, 30} and {c["ordering"] for c in GOLD} == {"random", "none"}
    assert any(c.get("offset") or c.get("offset_is_mean") for c in GOLD) and any(not c.get("offset") for c in GOLD)
    assert names["many_zeros"]["y_zeros"] >= 0.8 * names["many_zeros"]["n"]
    big = names["large_counts"]
    assert 500. <= big["y_sum"] / big["n"] <= 2000.
    assert any(c["t"] != 50 for c in GOLD)


def test_log_normalising_constant_is_minus_log_factorial():
    from scipy.special import gammaln
    y = np.array([0., 1., 2., 3., 17., 1000., 123456.])
    assert abs(olp.log_norm_const(y) + gammaln(y + 1).sum()) <= 1e-12 * gammaln(y + 1).sum()


@pytest.mark.parametrize("idx", range(len(GOLD)))
def test_golden_negll_and_iterations(idx):
    c = GOLD[idx]
    r = oracle(c)
    assert abs(r["negll"] - c["negll"]) <= 1e-9 * abs(c["negll"]), (r["negll"], c["negll"])
    assert r["newton_it"] == c["newton_it"], (r["newton_it"], c["newton_it"])


@pytest.mark.parametrize("idx", range(len(GOLD)))
def test_golden_gradient(idx):
    c = GOLD[idx]
    r = oracle(c, grad=True)
    g = np.array(c["grad"])
    assert np.all(np.abs(r["grad"] - g) <= 1e-6 * np.abs(g).max()), (r["grad"], g)


@pytest.mark.parametrize("cov,shape", [("matern", 1.5), ("exponential", 0.5)])
def test_gradient_is_the_derivative_of_the_likelihood(cov, shape):
    """Central differences of the oracle's poisson likelihood (Cholesky branch: exact traces) against grad_consistent."""
    X, y, off = poisson_data.count_synth(400, 12, True)
    vo = ov.VecchiaOracle(X, 10, cov, shape, "random", 1)
    th = np.array([0.9, 0.15])

    def f(t):
        _, pt = ov.transform_cov_pars([1.0] + list(t), cov, shape)
        return olp.negll(vo.coords, vo.nn, vo.cid, t[0], pt[1], y[vo.perm], fixed_effects=off[vo.perm], method="cholesky",
                        delta_conv_mode_finding=1e-13)["negll"]
    _, pt = ov.transform_cov_pars([1.0] + list(th), cov, shape)
    g = olp.grad_negll(vo.coords, vo.nn, vo.cid, th[0], pt[1], y[vo.perm], fixed_effects=off[vo.perm], method="cholesky",
                      delta_conv_mode_finding=1e-13)["grad_consistent"]
    for j in range(2):
        e = np.zeros(2); e[j] = 1e-5
        fd = (f(th * np.exp(e)) - f(th * np.exp(-e))) / 2e-5
        # the reference's shortcut dSigma^-1/dlog(var) = -Sigma^-1 ignores the jitter on the neighbour blocks' diagonal
        # (Vecchia_utils.cpp:1607): with the exponential kernel and W up to e^loc that shows at ~2e-6 of the variance derivative
        tol = 1e-5 if (cov == "exponential" and j == 0) else 1e-6
        assert abs(fd - g[j]) <= tol * max(1., abs(g[j])), (cov, j, fd, g[j])


@pytest.mark.parametrize("idx", [i for i, c in enumerate(GOLD) if "fit" in c and c["n"] <= 2000])
def test_fit_glue_reproduces_reference_fit(idx):
    """The library's L-BFGS driver (GPB200_LbfgsMinimize, what REModel::OptimCovParLaplace runs) with the pinned oracle as objective,
    from the reference's initial values: the reference's optimum and iteration count."""
    from gpboost_b200.libpath import load_lib
    lib = load_lib()
    c = GOLD[idx]

    def obj(xp, n, gp, ctx):
        th = np.exp(np.array([xp[0], xp[1]]))
        r = oracle(c, grad=bool(gp), cov_pars=list(th))
        if bool(gp):
            gp[0], gp[1] = r["grad"][0], r["grad"][1]
        return float(r["negll"])
    cb = C.CFUNCTYPE(C.c_double, C.POINTER(C.c_double), C.c_int, C.POINTER(C.c_double), C.c_void_p)(obj)
    fit = c["fit"]
    assert fit["init_cov_pars"][0] == 1.0  # marginal variance 1 for every non-Gaussian likelihood (re_model_template.h:4865-4911)
    x = np.log(np.array(fit["init_cov_pars"]))
    fx = C.c_double(0.); it = C.c_int(0)
    rc = lib.GPB200_LbfgsMinimize(cb, None, 2, x.ctypes.data_as(C.POINTER(C.c_double)), C.byref(fx), 1000, C.c_double(1e-6), 6,
                                  C.c_double(1.0), C.byref(it))
    assert rc == 0, lib.LGBM_GetLastError().decode()
    assert abs(it.value - fit["num_it"]) <= 3, (it.value, fit["num_it"])
    assert np.all(np.abs(np.exp(x) - np.array(fit["cov_pars"])) <= 5e-3 * np.array(fit["cov_pars"])), (np.exp(x), fit["cov_pars"])
    assert abs(fx.value - fit["negll"]) <= 1e-5 * abs(fit["negll"])
