"""GPU parity tests for the Laplace-Vecchia path (SURVEY §8 a12; bernoulli_logit likelihood, latent Vecchia GP),
through the reference's C API (GPB_CreateREModel / GPB_EvalNegLogLikelihood) of lib_gpboost_b200.so.

The reference's default for this model is matrix_inversion_method = "iterative" (VADU-preconditioned CG + stochastic
Lanczos quadrature with 50 probe vectors). The product draws the *same* probe vectors (same standard-library generator
calls), so the comparison with the reference's iterative value is deterministic: tolerance 1e-6 relative (CG stopping
rules are evaluated on sums with a different association order; in practice ~1e-12). Against the sparse-Cholesky variant
the difference is the reference's own stochastic error: 2e-3 relative."""
import json
import os

import numpy as np
import pytest

import datagen
from gpboost_b200 import GPModel
from oracle import laplace as ol
from oracle import vecchia as ov

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(HERE, "golden", "laplace_golden.json")) as f:
    GOLD = json.load(f)["cases"]


def data_of(c):
    if c["name"] == "r_binary":
        X, y = datagen.r_binary_test_data()
        return X, y, None
    return datagen.binary_synth(c["n"], c["dseed"], c["offset"])


def product_model(c, X):
    return GPModel(likelihood="bernoulli_logit", gp_coords=X, cov_function=c["cov_function"], cov_fct_shape=c["shape"],
                   gp_approx="vecchia", num_neighbors=c["m"], vecchia_ordering=c["ordering"], seed=c["seed"],
                   matrix_inversion_method="iterative")


@pytest.mark.parametrize("idx", range(len(GOLD)))
def test_negll_matches_reference_golden(idx):
    c = GOLD[idx]
    X, y, off = data_of(c)
    gm = product_model(c, X)
    v = gm.neg_log_likelihood(np.array(c["cov_pars"]), y, fixed_effects=off)
    assert abs(v - c["negll_iterative"]) <= 1e-6 * abs(c["negll_iterative"])
    assert abs(v - c["negll_cholesky"]) <= 2e-3 * abs(c["negll_cholesky"])


@pytest.mark.parametrize("idx", [1, 2])
def test_mode_and_iterations_match_oracle(idx):
    c = GOLD[idx]
    X, y, off = data_of(c)
    gm = product_model(c, X)
    v = gm.neg_log_likelihood(np.array(c["cov_pars"]), y, fixed_effects=off)
    info = gm.laplace_info()
    vo = ov.VecchiaOracle(X, c["m"], c["cov_function"], c["shape"], c["ordering"], c["seed"])
    _, pt = ov.transform_cov_pars([1.0] + list(c["cov_pars"]), c["cov_function"], c["shape"])
    r = ol.negll(vo.coords, vo.nn, vo.cid, c["cov_pars"][0], pt[1], y[vo.perm], fixed_effects=None if off is None else off[vo.perm],
                 method="iterative")
    assert int(info[1]) == r["newton_it"]
    assert int(info[2]) == r["cg_it"]
    assert int(info[3]) == r["slq_it"]
    assert abs(info[4] - r["logdet"]) <= 1e-8 * abs(r["logdet"])
    mode = gm.laplace_mode()
    mode_oracle = np.empty_like(mode)
    mode_oracle[vo.perm] = r["mode"]
    # the Newton systems are solved to the reference's CG tolerance (||r|| < 1e-2), so the mode is only defined to that
    # accuracy; CG iterates of two implementations drift apart by rounding amplification well below it
    assert np.max(np.abs(mode - mode_oracle)) <= 1e-5 * (1. + np.max(np.abs(mode_oracle)))
    assert abs(v - r["negll"]) <= 1e-9 * abs(r["negll"])


def test_repeatable_and_label_check():
    X, y, _ = datagen.binary_synth(4000, 11, False)
    gm = GPModel(likelihood="bernoulli_logit", gp_coords=X, gp_approx="vecchia", num_neighbors=15, seed=3)
    a = gm.neg_log_likelihood(np.array([1.0, 0.1]), y)
    b = gm.neg_log_likelihood(np.array([1.0, 0.1]), y)
    assert a == b  # deterministic kernels, mode re-initialised to zero
    with pytest.raises(Exception, match="needs to be 0 or 1"):
        gm.neg_log_likelihood(np.array([1.0, 0.1]), y + 0.5)
    with pytest.raises(Exception, match="not supported"):
        GPModel(likelihood="bernoulli_logit", gp_coords=X, gp_approx="vecchia", num_neighbors=15, matrix_inversion_method="cholesky")


def test_large_n_self_consistency():
    """n = 200k: the Laplace objective at the mode must dominate the objective at zero and the Newton system must be
    solved (residual of the stationarity condition Sigma^-1 b = y - p(b))."""
    n = 200000
    X, y, _ = datagen.binary_synth(n, 21, False)
    gm = GPModel(likelihood="bernoulli_logit", gp_coords=X, gp_approx="vecchia", num_neighbors=30, seed=1)
    v = gm.neg_log_likelihood(np.array([1.0, 0.05]), y)
    info = gm.laplace_info()
    assert np.isfinite(v)
    assert info[5] > -n * np.log(2.)  # objective at b = 0 is -n log 2
    assert 1 <= info[1] <= 20 and info[3] >= 2


@pytest.mark.parametrize("idx", range(len(GOLD)))
def test_latent_factor_range_derivative_matches_oracle(idx):
    """MODE_STORE_GRAD of the factor kernel: A, D^-1 and their derivatives w.r.t. log(range) of the latent factor
    (B_grad[1], D_grad[1] of CalcCovFactorGradientVecchia) against the oracle's restatement, <= 1e-8 of the largest entry (the
    north_star's fp64 tolerance; the latent blocks carry no nugget, so two fp64 evaluation orders differ by ~2e-9 there)."""
    import ctypes as C
    c = GOLD[idx]
    X, y, off = data_of(c)
    mdl = product_model(c, X)
    eng = C.c_void_p()
    assert mdl._LIB.GPB200_GetDeviceEngine(mdl.handle, C.byref(eng)) == 0
    vo = ov.VecchiaOracle(X, c["m"], c["cov_function"], c["shape"], c["ordering"], c["seed"])
    _, pt = ov.transform_cov_pars([1.0] + list(c["cov_pars"]), c["cov_function"], c["shape"])
    n, m = vo.nn.shape
    A = np.empty((n, m)); Dinv = np.empty(n); dA = np.empty((n, m)); dD = np.empty(n)
    P = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    mdl._LIB.gpbdev_last_error.restype = C.c_char_p
    rc = mdl._LIB.gpbdev_vecchia_latent_factor_grad(eng, C.c_int(vo.cid), C.c_double(c["cov_pars"][0]), C.c_double(pt[1]), P(A), P(Dinv), P(dA), P(dD))
    assert rc == 0, mdl._LIB.gpbdev_last_error().decode()
    A0, Dinv0, dA0, dD0, bad = ol.factor_latent_grad(vo.coords, vo.nn, vo.cid, c["cov_pars"][0], pt[1])
    assert bad == 0
    # The smooth kernels (Matern-2.5, Gaussian) give neighbour blocks with condition numbers ~1e8-1e10 on the latent scale (jitter 1e-10,
    # no nugget): two correct fp64 evaluation orders of dA = S^-1 r then differ by ~1e-8 relative — the oracle (LAPACK order) is no more
    # exact than the kernel. The bar is the north_star's 1e-8 where the blocks are well conditioned and 1e-6 for those two kernels, the
    # same split the prediction goldens use (tests/test_predict_oracle_pinned.py).
    tol = 1e-6 if (c["cov_function"] == "gaussian" or c["shape"] == 2.5) else 1e-8
    # D_i = v - A_i . s_i is a difference of O(v) terms and reaches 3e-8 v for the smooth kernels (no nugget on the latent scale), so the
    # conditional variance is compared as D = 1 / D^-1 on the scale it is computed on: both sides carry an absolute error of ~1e-16 v
    for got, want, name in ((A, A0, "A"), (1. / Dinv, 1. / Dinv0, "D"), (dA, dA0, "dA"), (dD, dD0, "dD")):
        assert np.max(np.abs(got - want)) <= tol * np.max(np.abs(want)), name


@pytest.mark.parametrize("idx", range(len(GOLD)))
def test_laplace_gradient_matches_reference_golden(idx):
    """Gradient of the Laplace-approximated likelihood w.r.t. (log variance, log range), iterative branch with the reference's
    probe vectors, against the reference's own gradient (recovered from one gradient-descent step; tests/golden)."""
    import ctypes as C
    c = GOLD[idx]
    X, y, off = data_of(c)
    mdl = product_model(c, X)
    P = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    yy = np.ascontiguousarray(y, dtype=np.float64); cp = np.array(c["cov_pars"], dtype=np.float64)
    offc = None if off is None else np.ascontiguousarray(off, dtype=np.float64)
    negll = C.c_double(0.); g = np.zeros(2)
    rc = mdl._LIB.GPB200_EvalLaplaceGradient(mdl.handle, P(yy), P(cp), None if offc is None else P(offc), C.byref(negll), P(g))
    assert rc == 0, mdl._LIB.LGBM_GetLastError().decode()
    assert abs(negll.value - c["negll_iterative"]) <= 1e-6 * abs(c["negll_iterative"])
    want = np.array(c["grad_iterative"])
    assert np.all(np.abs(g - want) <= 1e-5 * np.abs(want).max()), (g, want)


@pytest.mark.parametrize("idx", [i for i, c in enumerate(GOLD) if "fit_iterative" in c])
def test_laplace_fit_matches_reference_golden(idx):
    """GPB_OptimCovPar for the bernoulli_logit Vecchia model on the device against the reference's fit (defaults: L-BFGS,
    iterative method, 50 probes)."""
    c = GOLD[idx]
    X, y, off = data_of(c)
    mdl = product_model(c, X)
    mdl.fit(y, offset=off)
    fit = c["fit_iterative"]
    cp = mdl.get_cov_pars()
    assert np.all(np.abs(cp - np.array(fit["cov_pars"])) <= 5e-3 * np.array(fit["cov_pars"])), (cp, fit["cov_pars"])
    assert abs(mdl._get_num_optim_iter() - fit["num_it"]) <= 3
    assert abs(mdl.get_current_neg_log_likelihood() - fit["negll"]) <= 1e-5 * abs(fit["negll"])
