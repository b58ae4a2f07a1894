"""GPU tests of the Laplace-Vecchia path with the poisson likelihood (log link, latent Vecchia GP), through the reference's C API
(GPB_CreateREModel / GPB_EvalNegLogLikelihood / GPB_OptimCovPar) of lib_gpboost_b200.so, against the goldens of the unmodified
reference library (tests/golden/make_laplace_poisson_golden.py) and the pinned oracle (tests/laplace_poisson_oracle.py).

Bars (those of the bernoulli_logit tests, DESIGN §5): likelihood 1e-6 relative, gradient 1e-5 of max|g|, fits 5e-3 relative on the
covariance parameters and +-3 L-BFGS iterations; Newton iteration counts equal to the reference's and the oracle's, CG and SLQ counts
equal to the oracle's up to one iteration per stopping test (see test_mode_and_iterations_match_oracle). The per-row kernels are checked one by one against an np.longdouble restatement with bars derived from
the rounding of each operation (see test_row_kernels_against_longdouble)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import dropin
import poisson_data
from gpboost_b200 import GPModel
from gpboost_b200.basic import GPBoostError
import laplace_poisson_oracle as olp
from oracle import vecchia as ov

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(HERE, "golden", "laplace_poisson_golden.json")) as f:
    _G = json.load(f)
GOLD = _G["cases"]
P = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))


def product_model(c, **kw):
    X = poisson_data.case_data(c)[0]
    mdl = GPModel(likelihood="poisson", gp_coords=X, cov_function=c["cov_function"], cov_fct_shape=c["shape"], gp_approx="vecchia",
                  num_neighbors=c["m"], vecchia_ordering=c["ordering"], seed=c["seed"], matrix_inversion_method="iterative", **kw)
    mdl.set_optim_params(dict(num_rand_vec_trace=c["t"]))
    return mdl


def oracle_eval(c, grad=False):
    X, y, off = poisson_data.case_data(c)
    vo = ov.VecchiaOracle(X, c["m"], c["cov_function"], c["shape"], c["ordering"], c["seed"])
    _, pt = ov.transform_cov_pars([1.0] + list(c["cov_pars"]), c["cov_function"], c["shape"])
    f = olp.grad_negll if grad else olp.negll
    r = f(vo.coords, vo.nn, vo.cid, c["cov_pars"][0], pt[1], y[vo.perm], fixed_effects=None if off is None else off[vo.perm],
          method="iterative", num_rand_vec_trace=c["t"])
    return vo, r


@pytest.mark.parametrize("idx", range(len(GOLD)))
def test_negll_matches_reference_golden(idx):
    c = GOLD[idx]
    _, y, off = poisson_data.case_data(c)
    gm = product_model(c)
    v = gm.neg_log_likelihood(np.array(c["cov_pars"]), y, fixed_effects=off)
    assert abs(v - c["negll"]) <= 1e-6 * abs(c["negll"]), (v, c["negll"])
    info = gm.laplace_info()
    assert int(info[1]) == c["newton_it"], (info, c["newton_it"])
    print("poisson %s: Newton %d, CG %d, SLQ %d" % (c["name"], info[1], info[2], info[3]))


@pytest.mark.parametrize("idx", range(len(GOLD)))
def test_mode_and_iterations_match_oracle(idx):
    c = GOLD[idx]
    X, y, off = poisson_data.case_data(c)
    gm = product_model(c)
    v = gm.neg_log_likelihood(np.array(c["cov_pars"]), y, fixed_effects=off)
    info = gm.laplace_info()
    vo, r = oracle_eval(c)
    # Newton counts are equal. The PCG stops when ||r|| < 1e-2 and the SLQ when the mean column residual norm does; with W = e^loc
    # (up to ~3e3 here) those norms fall slowly near the threshold, and two summation orders can put one iteration's norm on either
    # side of it: one CG iteration per Newton step and one SLQ iteration may differ (measured on the H100: 79 vs 80 CG, 99 vs 100 SLQ)
    assert int(info[1]) == r["newton_it"], (info, r["newton_it"])
    assert abs(int(info[2]) - r["cg_it"]) <= r["newton_it"] + 1 and abs(int(info[3]) - r["slq_it"]) <= 1, (info, r["cg_it"], r["slq_it"])
    same = int(info[2]) == r["cg_it"] and int(info[3]) == r["slq_it"]
    assert abs(info[4] - r["logdet"]) <= (1e-8 if same else 1e-5) * abs(r["logdet"]), (info[4], r["logdet"])
    mode = gm.laplace_mode()
    mode_oracle = np.empty_like(mode)
    mode_oracle[vo.perm] = r["mode"]
    # the Newton systems are solved to the reference's CG tolerance (||r|| < 1e-2): the mode is defined to that accuracy only
    assert np.max(np.abs(mode - mode_oracle)) <= 1e-5 * (1. + np.max(np.abs(mode_oracle)))
    assert abs(v - r["negll"]) <= (1e-9 if same else 1e-6) * abs(r["negll"]), (v, r["negll"])


def _device_gradient(c):
    _, y, off = poisson_data.case_data(c)
    mdl = product_model(c)
    yy = np.ascontiguousarray(y); cp = np.array(c["cov_pars"], dtype=np.float64)
    offc = None if off is None else np.ascontiguousarray(off)
    negll = C.c_double(0.); g = np.zeros(2)
    rc = mdl._LIB.GPB200_EvalLaplaceGradient(mdl.handle, P(yy), P(cp), None if offc is None else P(offc), C.byref(negll), P(g))
    assert rc == 0, mdl._LIB.LGBM_GetLastError().decode()
    return negll.value, g


@pytest.mark.parametrize("idx", range(len(GOLD)))
def test_gradient_matches_reference_golden(idx):
    c = GOLD[idx]
    v, g = _device_gradient(c)
    assert abs(v - c["negll"]) <= 1e-6 * abs(c["negll"])
    want = np.array(c["grad"])
    assert np.all(np.abs(g - want) <= 1e-5 * np.abs(want).max()), (g, want)


@pytest.mark.parametrize("idx", [i for i, c in enumerate(GOLD) if "fit" in c])
def test_fit_matches_reference_golden(idx):
    c = GOLD[idx]
    _, y, off = poisson_data.case_data(c)
    mdl = product_model(c)
    mdl.fit(y, offset=off, params=dict(num_rand_vec_trace=c["t"]))
    fit = c["fit"]
    cp = mdl.get_cov_pars()
    assert np.all(np.abs(cp - np.array(fit["cov_pars"])) <= 5e-3 * np.array(fit["cov_pars"])), (cp, fit["cov_pars"])
    assert abs(mdl._get_num_optim_iter() - fit["num_it"]) <= 3, (mdl._get_num_optim_iter(), fit["num_it"])
    assert abs(mdl.get_current_neg_log_likelihood() - fit["negll"]) <= 1e-5 * abs(fit["negll"])
    assert mdl._get_likelihood_name() == "poisson"


def test_two_runs_repeat_bit_for_bit():
    c = GOLD[4]  # large counts: W ~ 1e3
    _, y, off = poisson_data.case_data(c)
    a = product_model(c).neg_log_likelihood(np.array(c["cov_pars"]), y, fixed_effects=off)
    mdl = product_model(c)
    b = mdl.neg_log_likelihood(np.array(c["cov_pars"]), y, fixed_effects=off)
    b2 = mdl.neg_log_likelihood(np.array(c["cov_pars"]), y, fixed_effects=off)
    assert a == b == b2
    (va, ga), (vb, gb) = _device_gradient(c), _device_gradient(c)
    assert va == vb and np.array_equal(ga, gb)


def test_row_kernels_against_longdouble():
    """prep_kernel, row_stats_kernel and grad_coef_kernel of the poisson instance (gpbdev_laplace_rows) against np.longdouble at
    locations 0, +-1, +-20, +-700 (split between mode and fixed effect) and y in {0, 1, 1e6}. loc = mode + fe is rounded in fp64 on
    both sides; from there on the restatement is exact to ~1e-19. Device errors, with u = 2^-53 and CUDA's exp within 1 ulp (2u):
      W = dW = exp(loc): 2u relative;  dw = D^-1 + W: |D^-1 + W| u + 2u W;
      rhs = W mode + (y - W): (3u W + u (y + W)) |mode|-weighted terms -> 4u (W |mode| + y + W);
      log-lik y loc - exp(loc): u |y loc| + 2u W + u |y loc - W| -> 3u (|y loc| + W).
    A factor 2 on each bar covers the restatement's own rounding to fp64 of its inputs."""
    import itertools
    from gpboost_b200 import load_lib
    lib = load_lib()
    lib.gpbdev_last_error.restype = C.c_char_p
    locs = [0., 1., -1., 20., -20., 700., -700.]
    ys = [0., 1., 1e6]
    rows = list(itertools.product(locs, ys, [0., 0.25, -3.]))  # (loc, y, fe share): mode = loc - fe
    n = len(rows)
    loc_t = np.array([r[0] for r in rows]); y = np.array([r[1] for r in rows]); fe = np.array([r[2] for r in rows])
    mode = loc_t - fe
    Dinv = np.linspace(0.3, 40., n)
    out = np.zeros(5 * n)
    for with_fe in (True, False):
        f = fe if with_fe else np.zeros(n)
        md = mode if with_fe else loc_t
        rc = lib.gpbdev_laplace_rows(C.c_int(0), C.c_int(1), C.c_int64(n), P(y), P(md), P(f) if with_fe else None, P(Dinv), P(out))
        assert rc == 0, lib.gpbdev_last_error().decode()
        W, rhs, dw, ll, dW = out.reshape(5, n)
        loc = (md + f).astype(np.longdouble)  # fp64 sum, as on the device
        mu = np.exp(loc)
        u = 2. ** -53
        mdl = md.astype(np.longdouble); yl = y.astype(np.longdouble)
        want = dict(W=mu, dW=mu, dw=Dinv + mu, rhs=mu * mdl + (yl - mu), ll=yl * loc - mu)
        bar = dict(W=4 * u * mu, dW=4 * u * mu, dw=2 * (u * np.abs(Dinv + mu) + 2 * u * mu),
                   rhs=8 * u * (mu * np.abs(mdl) + yl + mu), ll=6 * u * (np.abs(yl * loc) + mu))
        for name, got in (("W", W), ("dW", dW), ("dw", dw), ("rhs", rhs), ("ll", ll)):
            err = np.abs(got.astype(np.longdouble) - want[name])
            assert np.all(np.isfinite(got)), name
            assert np.all(err <= bar[name]), (name, with_fe, [(rows[i], float(err[i]), float(bar[name][i])) for i in np.nonzero(err > bar[name])[0]])
    # bernoulli_logit instance of the same kernels is finite and p(1 - p) <= 1/4 on the same rows
    rc = lib.gpbdev_laplace_rows(C.c_int(0), C.c_int(0), C.c_int64(n), P((y > 0).astype(np.float64)), P(mode), P(fe), P(Dinv), P(out))
    assert rc == 0, lib.gpbdev_last_error().decode()
    W = out[:n]
    assert np.all((W >= 0) & (W <= 0.25))
    assert lib.gpbdev_laplace_rows(C.c_int(0), C.c_int(2), C.c_int64(n), P(y), P(mode), None, P(Dinv), P(out)) != 0


def test_refusals():
    X, y, _ = poisson_data.count_synth(1500, 41)
    cp = np.array([1.0, 0.1])
    gm = GPModel(likelihood="poisson", gp_coords=X, gp_approx="vecchia", num_neighbors=15, seed=3)
    assert gm._get_likelihood_name() == "poisson"
    with pytest.raises(GPBoostError, match="Must have y >= 0"):
        gm.neg_log_likelihood(cp, np.where(np.arange(len(y)) == 7, -1., y))
    with pytest.raises(GPBoostError, match="non-integer"):
        gm.neg_log_likelihood(cp, y + 0.5)
    with pytest.raises(GPBoostError, match="non-integer"):
        gm.neg_log_likelihood(cp, np.where(np.arange(len(y)) == 3, np.nan, y))
    with pytest.raises(GPBoostError, match="at most 2\\^31 - 1"):
        gm.neg_log_likelihood(cp, np.where(np.arange(len(y)) == 3, np.inf, y))
    with pytest.raises(GPBoostError, match="non-integer"):
        gm.fit(y + 0.25)
    with pytest.raises(GPBoostError, match="matrix_inversion_method"):
        GPModel(likelihood="poisson", gp_coords=X, gp_approx="vecchia", num_neighbors=15, matrix_inversion_method="cholesky")
    with pytest.raises(GPBoostError, match="single GP and gp_approx = 'vecchia'"):
        GPModel(likelihood="poisson", gp_coords=X, gp_approx="none")
    with pytest.raises(GPBoostError, match="num_neighbors must be <= 30"):
        GPModel(likelihood="poisson", gp_coords=X, gp_approx="vecchia", num_neighbors=31).neg_log_likelihood(cp, y)
    for lik in ("gamma", "negative_binomial", "hurdle_poisson", "zero_inflated_poisson"):
        with pytest.raises(GPBoostError, match="supported: 'gaussian', 'bernoulli_logit', 'poisson'"):
            GPModel(likelihood=lik, gp_coords=X, gp_approx="vecchia", num_neighbors=15)
    fitted = GPModel(likelihood="poisson", gp_coords=X, gp_approx="vecchia", num_neighbors=15, seed=3)
    with pytest.raises(GPBoostError, match="covariates are only supported for the Gaussian"):
        fitted.fit(y, X=np.ones((len(y), 1)))
    fitted.set_optim_params(dict(maxit=2))
    fitted.fit(y)
    with pytest.raises(GPBoostError, match="Prediction is not supported for likelihood 'poisson'"):
        fitted.predict(y, X[:5], fitted.get_cov_pars())
    with pytest.raises(GPBoostError, match="CalcGradient for likelihood 'poisson'"):
        fitted.response_gradient(y)


@pytest.mark.skipif(dropin.ref_package_dir() is None, reason="reference Python package not present")
def test_unmodified_package_on_the_device_matches_the_reference_library():
    want = _G["dropin"]
    got = dropin.run_with(os.path.join(os.path.dirname(HERE), "gpboost_b200", "lib_gpboost_b200.so"), poisson_data.DROPIN_SCRIPT)
    assert np.allclose(got["cov_pars"], want["cov_pars"], rtol=5e-3), (got["cov_pars"], want["cov_pars"])
    assert abs(got["negll_opt"] - want["negll_opt"]) <= 1e-5 * abs(want["negll_opt"])
    assert abs(got["negll_at"] - want["negll_at"]) <= 1e-6 * abs(want["negll_at"])
