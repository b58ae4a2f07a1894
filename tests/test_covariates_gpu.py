"""Linear regression covariates of the Gaussian Vecchia model on the device (gpboost_b200/csrc/dev/covariates.cuh, REModel::
OptimLinRegrCoefCovPar): the GLS Gram kernel at fixed covariance parameters against the oracle (oracle/covariates.py) for every
kernel, neighbour-count band and register-tile width; fits, coefficients, initial values and predictions with X_pred against the
reference's goldens (tests/golden/covariates_golden.json); and the refusals."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

import datagen
from oracle import covariates as oc
from oracle import vecchia as ov

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_covariates_golden as mk  # noqa: E402

pytestmark = pytest.mark.gpu

with open(os.path.join(HERE, "golden", "covariates_golden.json")) as f:
    GOLD = json.load(f)["cases"]
FITTED = [i for i, c in enumerate(GOLD) if c.get("maxit", 1) > 0]
COVS = [("exponential", 0.5), ("matern", 1.5), ("matern", 2.5), ("gaussian", 0.)]
MODE_STORE = 1


def P(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


@pytest.fixture(scope="module")
def lib(product_lib):
    assert product_lib.gpbdev_device_count() > 0, "no CUDA device visible — GPU tests need an H100"
    return product_lib


def chk(lib, rc):
    assert rc == 0, lib.gpbdev_last_error().decode()


def engine_with_factor(lib, coords, y, m, cid, var, range_t, seed=1, nn_in=None):
    """engine on coords (original order) with y installed and the factor stored at (var, range_t); returns h, perm, nn, A, Dinv.
    nn_in: neighbour sets to supply (n x m, -1 padded) instead of the device search"""
    n, d = coords.shape
    perm = ov.random_order(n, seed)
    co = np.ascontiguousarray(coords[perm])
    h = C.c_void_p()
    nn_c = None if nn_in is None else P(np.ascontiguousarray(nn_in, dtype=np.int32), C.c_int32)
    chk(lib, lib.gpbdev_vecchia_create(C.byref(h), 0, C.c_int64(n), d, m, P(co), P(perm, C.c_int32), nn_c, C.c_int64(0), C.c_int64(n)))
    yy = np.ascontiguousarray(y, dtype=np.float64)
    chk(lib, lib.gpbdev_vecchia_set_y(h, P(yy)))
    sums = np.zeros(9)
    chk(lib, lib.gpbdev_vecchia_eval(h, cid, C.c_double(var), C.c_double(range_t), MODE_STORE, P(sums)))
    nn = np.empty((n, m), dtype=np.int32)
    chk(lib, lib.gpbdev_vecchia_get_nn(h, P(nn, C.c_int32)))
    A = np.empty((n, m)); Dinv = np.empty(n)
    chk(lib, lib.gpbdev_vecchia_get_factor(h, P(A), P(Dinv)))
    return h, perm, nn, A, Dinv


def device_gram(lib, h, X):
    n, p = X.shape
    Xc = np.ascontiguousarray(X.flatten(order="F"))
    chk(lib, lib.gpbdev_vecchia_set_covariates(h, P(Xc), p))
    G = np.empty((p, p)); r = np.empty(p)
    chk(lib, lib.gpbdev_vecchia_gls_gram(h, P(G), P(r)))
    return G, r


def rel(a, b):
    return np.linalg.norm(a - b) / np.linalg.norm(b)


@pytest.mark.parametrize("cov", COVS, ids=["exponential", "matern1.5", "matern2.5", "gaussian"])
@pytest.mark.parametrize("m", [1, 10, 30, 31, 45, 60])
@pytest.mark.parametrize("n_kind", ["below_m", "m+1", "4000"])
def test_gram_kernel_matches_oracle(lib, cov, m, n_kind):
    """every register-tile width (p = 1, 2: T = 1; 31, 32: T = 2; 33: T = 3; 64: T = 4) and every lane layout (p <= 32: lanes split
    over neighbour slices; p > 32: two columns per lane), -1 padded rows; and a second call is bitwise identical.
    below_m: n <= m, an engine whose every row is padded (neighbours = all earlier rows, supplied), batches and chunks mostly empty"""
    n = {"below_m": max(1, m // 2), "m+1": m + 1, "4000": 4000}[n_kind]
    nn_in = None
    if n_kind == "below_m":
        nn_in = np.full((n, m), -1, dtype=np.int32)
        for i in range(n):
            nn_in[i, :i] = np.arange(i)[::-1]
    coords, y = datagen.synth(n, 2, 7 + m)
    cid = ov.cov_id(*cov)
    rho = 2. * n ** -0.5  # about the neighbour spacing
    h, perm, nn, A, Dinv = engine_with_factor(lib, coords, y, m, cid, 1.3, 1. / rho if cid != 3 else 1. / rho ** 2, seed=m,
                                              nn_in=nn_in)
    try:
        rng = np.random.default_rng(m)
        if nn_in is not None:
            assert np.array_equal(nn, nn_in)
        for p in (1, 2, 31, 32, 33, 64):
            X = rng.standard_normal((n, p))
            X[:, 0] = 1.
            G, r = device_gram(lib, h, X)
            Gw, rw = oc.gram(nn, A, Dinv, X[perm], y[perm])
            assert rel(G, Gw) <= 1e-10 and rel(r, rw) <= 1e-10, (p, rel(G, Gw), rel(r, rw))
            assert np.array_equal(G, G.T)
            G2 = np.empty((p, p)); r2 = np.empty(p)
            chk(lib, lib.gpbdev_vecchia_gls_gram(h, P(G2), P(r2)))
            assert np.array_equal(G, G2) and np.array_equal(r, r2)
    finally:
        lib.gpbdev_vecchia_free(h)


def test_gram_kernel_at_one_million_rows(lib):
    n, m, p = 1_000_000, 30, 8
    coords, y = datagen.synth(n, 2, 99)
    h, perm, nn, A, Dinv = engine_with_factor(lib, coords, y, m, 1, 0.9, np.sqrt(3.) / 0.05)
    try:
        X = np.random.default_rng(5).standard_normal((n, p))
        X[:, 0] = 1.
        G, r = device_gram(lib, h, X)
        Gw, rw = oc.gram(nn, A, Dinv, X[perm], y[perm])
        assert rel(G, Gw) <= 1e-10 and rel(r, rw) <= 1e-10, (rel(G, Gw), rel(r, rw))
    finally:
        lib.gpbdev_vecchia_free(h)


def test_residual_pass_matches_oracle(lib):
    """y - X beta becomes the response: its quadratic form and log-determinant from the resident factor, for a mean that is large
    against the noise (no cancellation), and Psi^-1 y_r read back through the store path equals the oracle's"""
    n, m, p = 3000, 20, 3
    coords, y = datagen.synth(n, 2, 5)
    X = np.random.default_rng(1).standard_normal((n, p)); X[:, 0] = 1.
    beta = np.array([1e5, 2., -3.])
    y = y + X @ beta
    h, perm, nn, A, Dinv = engine_with_factor(lib, coords, y, m, 1, 1.1, np.sqrt(3.) / 0.1)
    try:
        device_gram(lib, h, X)
        b = beta + np.array([0.1, -0.05, 0.02])
        out = np.zeros(3)
        chk(lib, lib.gpbdev_vecchia_gls_residual(h, P(b), P(out)))
        _, ypy, ld = ov.nll_from_factor(nn, A, Dinv, (y - X @ b)[perm], 1.0)
        assert abs(out[0] - ypy) <= 1e-10 * ypy and abs(out[1] - ld) <= 1e-10 * abs(ld) and out[2] == 0.
        ya = np.empty(n)
        chk(lib, lib.gpbdev_vecchia_yaux(h, P(ya)))
        want = np.empty(n); want[perm] = ov.yaux(nn, A, Dinv, (y - X @ b)[perm])
        assert np.abs(ya - want).max() <= 1e-9 * np.abs(want).max()
    finally:
        lib.gpbdev_vecchia_free(h)


def fit_device(c, params=None):
    coords, y, X, offset, cp, Xp = mk.case_data(c)
    mdl = mk.model(c, coords)
    mdl.fit(y, X=X, params=mk.fit_params(c) if params is None else params, offset=offset)
    return mdl, coords, y, X, offset


@pytest.mark.parametrize("idx", FITTED)
def test_fit_matches_reference_golden(idx):
    c = GOLD[idx]
    mdl, coords, y, X, offset = fit_device(c)
    cp, coef, negll = mdl.get_cov_pars(), mdl.get_coef(), mdl.get_current_neg_log_likelihood()
    assert abs(negll - c["negll"]) <= 1e-6 * abs(c["negll"]), (negll, c["negll"])
    assert np.all(np.abs(cp - c["cov_pars"]) <= 2e-3 * np.abs(c["cov_pars"])), (cp, c["cov_pars"])
    assert abs(mdl._get_num_optim_iter() - c["num_it"]) <= 3, (mdl._get_num_optim_iter(), c["num_it"])
    gc = np.array(c["coef"])
    assert np.abs(coef - gc).max() <= 2e-3 * np.abs(gc).max(), (coef, gc)
    # self-consistency: the oracle's GLS and profiled NLL at the device's own fitted parameters
    vo = ov.VecchiaOracle(coords, c["m"], c["cov_function"], c["shape"], "random", c["seed"])
    res = oc.profiled_at_cov_pars(vo, cp, y, X, offset)
    assert np.abs(coef - res["beta"]).max() <= 1e-9 * np.abs(res["beta"]).max(), (coef, res["beta"])
    assert abs(negll - res["negll"]) <= 1e-9 * abs(res["negll"]), (negll, res["negll"])


def test_initial_coefficients_at_maxit_zero():
    for c in GOLD:
        if c.get("maxit") != 0:
            continue
        mdl, *_ = fit_device(c)
        want = np.array(c["coef"])
        assert np.abs(mdl.get_coef() - want).max() <= 1e-10 * np.abs(want).max(), (mdl.get_coef(), want)
    c = dict(GOLD[0])
    init = np.array([0.123])
    mdl, *_ = fit_device(c, params=dict(init_coef=init, maxit=0))
    assert np.array_equal(mdl.get_coef(), init)


def test_initial_coefficients_without_the_iid_model():
    """init_coef_aux_pars_from_iid_model = False: zero, the constant column at the mean of y - offset (FindInitialIntercept); the
    coefficients of an earlier fit with as many covariates are the starting point instead. At maxit = 0 the current negative
    log-likelihood is the one at the initial parameters and coefficients."""
    c = next(g for g in GOLD if g.get("offset"))
    coords, y, X, offset, _, _ = mk.case_data(c)
    X3 = X.copy(); X3[:, 0] = 2.  # a constant column that is not 1
    mdl = mk.model(c, coords).fit(y, X=X3, offset=offset, params=dict(init_coef_aux_pars_from_iid_model=False, maxit=0))
    want = np.zeros(X.shape[1]); want[0] = (y - offset).mean()
    assert np.abs(mdl.get_coef() - want).max() <= 1e-12 * np.abs(want).max()
    vo = ov.VecchiaOracle(coords, c["m"], c["cov_function"], c["shape"], "random", c["seed"])
    cp = mdl.get_cov_pars()
    s2, pt = ov.transform_cov_pars(cp, c["cov_function"], c["shape"])
    A, Dinv, _, _, _ = ov.factor(vo.coords, vo.nn, vo.cid, pt)
    nll = ov.nll_from_factor(vo.nn, A, Dinv, (y - offset - X3 @ want)[vo.perm], s2)[0]
    assert abs(mdl.get_current_neg_log_likelihood() - nll) <= 1e-9 * abs(nll)
    fitted = mk.model(c, coords).fit(y, X=X, offset=offset)
    beta = fitted.get_coef()
    fitted.fit(y, X=X, offset=offset, params=dict(init_coef_aux_pars_from_iid_model=False, maxit=0))
    assert np.array_equal(fitted.get_coef(), beta)


def test_optimizer_coef_is_checked_only_by_fits_with_covariates():
    """the reference's package passes back what GPB_GetOptimizerCoef reports ("lbfgs" for bernoulli_logit, "wls" for Gaussian data)
    through set_optim_params: models without covariates accept any value, as before"""
    from gpboost_b200 import GPModel
    from gpboost_b200.basic import GPBoostError
    coords, yb, _ = datagen.binary_synth(400, 2, False)
    logit = GPModel(likelihood="bernoulli_logit", gp_coords=coords, cov_function="exponential", gp_approx="vecchia", num_neighbors=10)
    logit.set_optim_params(dict(optimizer_coef="lbfgs"))
    assert np.isfinite(logit.neg_log_likelihood(np.array([1.0, 0.2]), yb))
    c = GOLD[0]
    coords, y, X, offset, _, _ = mk.case_data(c)
    plain = mk.model(c, coords)
    plain.set_optim_params(dict(optimizer_coef="gradient_descent"))
    plain.fit(y, params=dict(optimizer_coef="gradient_descent"))
    ref = mk.model(c, coords).fit(y)
    assert abs(plain.get_current_neg_log_likelihood() - ref.get_current_neg_log_likelihood()) <= 1e-12 * abs(ref.get_current_neg_log_likelihood())
    with pytest.raises(GPBoostError):
        plain.fit(y, X=X)
    plain.fit(y, X=X, params=dict(optimizer_coef="wls"))
    assert np.all(np.isfinite(plain.get_coef()))


def test_offset_enters_the_residual():
    c = next(g for g in GOLD if g.get("offset"))
    coords, y, X, offset, _, _ = mk.case_data(c)
    a = mk.model(c, coords).fit(y, X=X, offset=offset)
    b = mk.model(c, coords).fit(y - offset, X=X)
    assert np.abs(a.get_coef() - b.get_coef()).max() <= 1e-10 * np.abs(b.get_coef()).max()
    assert abs(a.get_current_neg_log_likelihood() - b.get_current_neg_log_likelihood()) <= 1e-12 * abs(b.get_current_neg_log_likelihood())
    d = mk.model(c, coords).fit(y, X=X)  # the offset changes the fit
    assert np.abs(d.get_coef() - b.get_coef()).max() > 1e-6


# the device predicts with at most 60 neighbours (2 x num_neighbors by default)
@pytest.mark.parametrize("idx", [i for i, c in enumerate(GOLD) if 2 * c["m"] <= 60])
def test_prediction_with_X_pred_matches_golden_and_oracle(idx):
    c = GOLD[idx]
    coords, y, X, offset, cpred, Xp = mk.case_data(c)
    coef = np.array(c["coef"])
    yo = y - (0. if offset is None else offset)
    mdl = mk.model(c, coords)
    mdl.fit(yo, X=X, params=dict(init_coef=coef, maxit=0))
    r = mdl.predict(yo, cpred, np.array(c["cov_pars"]), predict_var=True, predict_response=True, X_pred=Xp)
    tol = 1e-6 if c["cov_function"] == "gaussian" else 1e-8
    assert np.abs(r["mu"][:32] - np.array(c["mu_head"])).max() <= tol * np.abs(c["mu_head"]).max()
    assert abs(r["mu"].sum() - c["mu_sum"]) <= tol * np.abs(r["mu"]).sum()
    assert np.abs(r["var"][:32] - np.array(c["var_head"])).max() <= tol * np.abs(c["var_head"]).max()
    assert abs(r["var"].sum() - c["var_sum"]) <= tol * abs(c["var_sum"])
    vo = ov.VecchiaOracle(coords, c["m"], c["cov_function"], c["shape"], "random", c["seed"])
    mu, var = oc.predict_mean(vo.coords, yo, X, coef, cpred, Xp, c["cov_pars"], c["cov_function"], c["shape"], c["m"], vo.perm)
    assert np.abs(r["mu"] - mu).max() <= tol * np.abs(mu).max() and np.abs(r["var"] - var).max() <= tol * np.abs(var).max()


def test_prediction_after_fit_uses_the_fitted_coefficients():
    c = GOLD[1]
    mdl, coords, y, X, offset = fit_device(c)
    _, _, _, _, cpred, Xp = mk.case_data(c)
    r = mdl.predict(None, cpred, None, X_pred=Xp)  # the fitted residual stays installed
    r2 = mdl.predict(y - offset, cpred, mdl.get_cov_pars(), X_pred=Xp)
    assert np.abs(r["mu"] - r2["mu"]).max() <= 1e-10 * np.abs(r2["mu"]).max()


def test_refusals_are_clean():
    from gpboost_b200 import GPModel
    from gpboost_b200.basic import GPBoostError
    c = GOLD[0]
    coords, y, X, offset, cpred, Xp = mk.case_data(c)
    n = len(y)
    X2 = np.column_stack([np.ones(n), coords[:, 0]])
    bad = [np.column_stack([X2, X2[:, 1]]),                       # rank-deficient
           np.where(np.arange(n)[:, None] == 5, np.nan, X2),        # NaN
           np.random.default_rng(0).standard_normal((n, 65)),       # p = 65
           X2[:-1]]                                                 # wrong row count
    for Xb in bad:
        with pytest.raises(GPBoostError):
            mk.model(c, coords).fit(y, X=Xb)
    # rank-deficient X refused inside the optimiser's first evaluation (device Gram pass + host Cholesky), not by the iid start;
    # the failed fit leaves no covariates behind
    Xr = np.column_stack([X2, 2. * X2[:, 1]])
    for params in (dict(init_coef=np.zeros(3)), dict(init_coef_aux_pars_from_iid_model=False)):
        m_rd = mk.model(c, coords)
        with pytest.raises(GPBoostError, match="not positive definite"):
            m_rd.fit(y, X=Xr, params=params)
        with pytest.raises(GPBoostError):
            m_rd.get_coef()
        r_plain = m_rd.predict(y, cpred, np.array([0.3, 1.0, 0.2]))  # no X_pred needed: the model has no covariates
        assert np.all(np.isfinite(r_plain["mu"]))
    with pytest.raises(GPBoostError):
        mk.model(c, coords).fit(y, X=X2, params=dict(optimizer_coef="gradient_descent"))
    mdl = mk.model(c, coords).fit(y, X=X2)
    assert np.all(np.isfinite(mdl.get_coef()))
    with pytest.raises(GPBoostError):
        mdl.get_coef(std_err=True)
    with pytest.raises(GPBoostError):
        mdl.predict(y, cpred, mdl.get_cov_pars())  # X_pred missing
    plain = mk.model(c, coords).fit(y)
    with pytest.raises(GPBoostError):
        plain.predict(y, cpred, plain.get_cov_pars(), X_pred=np.ones((len(cpred), 1)))  # X_pred unexpected
    with pytest.raises(GPBoostError):
        plain.get_coef()
    grp = GPModel(group_data=np.arange(n) % 20)
    dense = GPModel(gp_coords=coords[:300], cov_function="exponential", gp_approx="none")
    logit = GPModel(likelihood="bernoulli_logit", gp_coords=coords, cov_function="exponential", gp_approx="vecchia", num_neighbors=10)
    for mdl_other, yy, XX in ((grp, y, X2), (dense, y[:300], X2[:300]), (logit, (y > np.median(y)).astype(float), X2)):
        with pytest.raises(GPBoostError):
            mdl_other.fit(yy, X=XX)
