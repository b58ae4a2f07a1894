"""GPU tests of the anisotropic covariance functions (matern_ard, gaussian_ard, matern_space_time) of the Gaussian Vecchia GP, through
the C ABI: neighbour sets searched on scaled coordinates, likelihood and store sums against the isotropic kernels on host-scaled
coordinates (bitwise), the per-group gradient pass against the restatement of the kernels' element formulas (tests/aniso_oracle.py)
at every kernel path, and the model (neighbour sets searched per evaluation and on the fit's schedule, fits, prediction,
refusals) against the reference's goldens."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import aniso_oracle as ao

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "aniso_golden.json")


def P(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


@pytest.fixture(scope="module")
def lib(product_lib):
    assert product_lib.gpbdev_device_count() > 0, "no CUDA device visible — GPU tests need an H100"
    return product_lib


def chk(lib, rc):
    assert rc == 0, lib.gpbdev_last_error().decode()


def rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


class Engine:
    """unsearched engine on ordered coordinates, scaled on the device"""

    def __init__(self, lib, co, m):
        self.lib, self.n, self.d, self.m = lib, co.shape[0], co.shape[1], m
        self.h = C.c_void_p()
        perm = np.arange(self.n, dtype=np.int32)
        chk(lib, lib.gpbdev_vecchia_create_unsearched(C.byref(self.h), 0, C.c_int64(self.n), self.d, m, P(np.ascontiguousarray(co)),
                                                       P(perm, C.c_int32), C.c_int64(0), C.c_int64(self.n)))

    def set_y(self, y):
        chk(self.lib, self.lib.gpbdev_vecchia_set_y(self.h, P(np.ascontiguousarray(y, dtype=np.float64))))

    def scale(self, s):
        chk(self.lib, self.lib.gpbdev_vecchia_set_coord_scale(self.h, P(np.ascontiguousarray(s, dtype=np.float64))))

    def search(self):
        chk(self.lib, self.lib.gpbdev_vecchia_search_neighbors(self.h))

    def nn(self):
        out = np.empty((self.n, self.m), dtype=np.int32)
        chk(self.lib, self.lib.gpbdev_vecchia_get_nn(self.h, P(out, C.c_int32)))
        return out

    def eval(self, cid, var, range_, mode):
        out = np.empty(9)
        chk(self.lib, self.lib.gpbdev_vecchia_eval(self.h, cid, C.c_double(var), C.c_double(range_), mode, P(out)))
        return out

    def grad_aniso(self, cid, var, groups):
        C_ = int(groups.max()) + 1
        out = np.empty(3 + 3 * (1 + C_))
        g = np.ascontiguousarray(groups, dtype=np.int32)
        chk(self.lib, self.lib.gpbdev_vecchia_eval_grad_aniso(self.h, cid, C.c_double(var), P(g, C.c_int32), C_, P(out)))
        return out

    def free(self):
        self.lib.gpbdev_vecchia_free(self.h)


def grad_from_sums(out, n):
    s2 = out[0] / n
    negll = out[0] / 2. / s2 + out[1] / 2. + n / 2. * (np.log(s2) + np.log(2 * np.pi))
    k = (len(out) - 3) // 3
    g = np.array([(out[3 + 3 * j] - 0.5 * out[4 + 3 * j]) / s2 + 0.5 * out[5 + 3 * j] for j in range(k)])
    return negll, g


def small_case(n, d, cov, shape, seed, dup=False):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0., 1., (n, d))
    if dup:  # duplicate coordinates: r = 0 pairs
        X[n // 2: n // 2 + 20] = X[:20]
    y = rng.standard_normal(n)
    C_ = 2 if ao.parse(cov, shape)[0] == "matern_space_time" else d
    ranges = rng.uniform(0.1, 0.6, C_)
    return X, y, np.concatenate([[0.3, 1.1], ranges])


# ---------------------------------------------------------------------------------------- kernel level
@pytest.mark.parametrize("m,d", [(5, 1), (10, 2), (15, 3), (20, 2), (25, 5), (30, 2), (30, 3), (45, 2), (60, 3), (30, 16), (10, 16),
                                 (20, 5)])
@pytest.mark.parametrize("cov,shape", [("matern_ard", 0.5), ("matern_ard", 1.5), ("matern_ard", 2.5), ("gaussian_ard", 0.)])
def test_grad_aniso_against_element_formulas(lib, m, d, cov, shape):
    n = 240
    X, y, cp = small_case(n, d, cov, shape, 100 * m + d, dup=(m == 20))
    o = ao.AnisoOracle(X, m, cov, shape, "none", 0)
    o.search(cp)
    e = Engine(lib, o.coords, o.m)
    _, var, lam = ao.transform(cp, o.cov_function, o.shape)
    e.scale(ao.scale_factors(lam, o.cov_function, d))
    e.search()
    assert np.array_equal(e.nn(), o.nn)
    e.set_y(y[o.perm])
    out = e.grad_aniso(o.cid, var, ao.groups(o.cov_function, d))
    negll, g = grad_from_sums(out, n)
    want_f, want_g = o.grad_profiled(cp, y)
    tol = 1e-6 if (cov == "gaussian_ard" or shape == 2.5) else 1e-8
    assert rel(negll, want_f) <= 1e-10
    np.testing.assert_allclose(g, want_g, rtol=tol, atol=tol * np.abs(want_g).max())
    again = e.grad_aniso(o.cid, var, ao.groups(o.cov_function, d))
    assert np.array_equal(out, again)  # fixed-order reductions
    e.free()


@pytest.mark.parametrize("m,d,shape,ordering", [(20, 3, 1.5, "time"), (30, 2, 0.5, "time_random_space"), (45, 3, 2.5, "time")])
def test_grad_space_time_layouts(lib, m, d, shape, ordering):
    n = 240
    X, y, cp = small_case(n, d, "matern_space_time", shape, 7 * m + d)
    o = ao.AnisoOracle(X, m, "matern_space_time", shape, ordering, 3)
    o.search(cp)
    e = Engine(lib, o.coords, o.m)
    _, var, lam = ao.transform(cp, o.cov_function, o.shape)
    e.scale(ao.scale_factors(lam, o.cov_function, d))
    e.search()
    assert np.array_equal(e.nn(), o.nn)
    e.set_y(y[o.perm])
    _, g = grad_from_sums(e.grad_aniso(o.cid, var, ao.groups(o.cov_function, d)), n)
    _, want_g = o.grad_profiled(cp, y)
    tol = 1e-6 if shape == 2.5 else 1e-8
    np.testing.assert_allclose(g, want_g, rtol=tol, atol=tol * np.abs(want_g).max())
    e.free()


@pytest.mark.parametrize("n,d,m,cid", [(5000, 2, 30, 1), (4000, 2, 10, 0), (3000, 3, 20, 2), (2000, 2, 45, 3)])
def test_sums_bitwise_equal_to_isotropic_on_host_scaled_coordinates(lib, n, d, m, cid):
    rng = np.random.default_rng(n + m)
    X = rng.uniform(0., 1., (n, d))
    y = rng.standard_normal(n)
    s = rng.uniform(2., 9., d)
    e = Engine(lib, X, m)
    e.scale(s)
    e.search()
    e.set_y(y)
    Xs = np.ascontiguousarray(X * s)
    iso = C.c_void_p()
    perm = np.arange(n, dtype=np.int32)
    chk(lib, lib.gpbdev_vecchia_create(C.byref(iso), 0, C.c_int64(n), d, m, P(Xs), P(perm, C.c_int32), None, C.c_int64(0), C.c_int64(n)))
    chk(lib, lib.gpbdev_vecchia_set_y(iso, P(y)))
    nn_iso = np.empty((n, m), dtype=np.int32)
    chk(lib, lib.gpbdev_vecchia_get_nn(iso, P(nn_iso, C.c_int32)))
    assert np.array_equal(e.nn(), nn_iso)
    for mode in (0, 1):
        a = e.eval(cid, 1.3, 1., mode)
        b = np.empty(9)
        chk(lib, lib.gpbdev_vecchia_eval(iso, cid, C.c_double(1.3), C.c_double(1.), mode, P(b)))
        assert np.array_equal(a[:3], b[:3])
    # equal ARD ranges: the per-coordinate range derivatives add up to the isotropic one
    e.scale(np.full(d, s[0]))
    e.search()
    chk(lib, lib.gpbdev_vecchia_free(iso))
    Xs = np.ascontiguousarray(X * s[0])
    chk(lib, lib.gpbdev_vecchia_create(C.byref(iso), 0, C.c_int64(n), d, m, P(Xs), P(perm, C.c_int32), None, C.c_int64(0), C.c_int64(n)))
    chk(lib, lib.gpbdev_vecchia_set_y(iso, P(y)))
    b = np.empty(9)
    chk(lib, lib.gpbdev_vecchia_eval(iso, cid, C.c_double(1.3), C.c_double(1.), 2, P(b)))
    a = e.grad_aniso(cid, 1.3, np.arange(d, dtype=np.int32))
    # sum u_k u, sum u^2 dD_k, sum dD_k / D of the range (isotropic sums 4, 6, 8) and of the variance (3, 5, 7)
    iso_rng = np.array([b[4], b[6], b[8]])
    ani_rng = np.array([sum(a[3 + 3 * k + j] for k in range(1, d + 1)) for j in range(3)])
    np.testing.assert_allclose(ani_rng, iso_rng, rtol=1e-11, atol=1e-11 * np.abs(iso_rng).max())
    np.testing.assert_allclose(a[3:6], [b[3], b[5], b[7]], rtol=1e-11, atol=1e-11 * max(abs(b[3]), abs(b[5]), abs(b[7])))
    chk(lib, lib.gpbdev_vecchia_free(iso))
    e.free()


# ---------------------------------------------------------------------------------------- model
def golden_cases():
    if not os.path.exists(GOLDEN):
        return []
    return json.load(open(GOLDEN))["cases"]


def spec(name):
    return next(c for c in ao.CASES if c["name"] == name)


def search_schedule(num_it):
    """least number of searches of a fit on a fresh model: one at the initial parameters, then after iteration k when k - 1 is 0 or
    2^j - 1, and after the last one. A convergence that the search after it revokes adds one more."""
    ks = [k for k in range(1, num_it + 1) if ((k - 1) & k) == 0]
    return 1 + len(ks) + (0 if num_it in ks else 1)


@pytest.mark.parametrize("case", [c["name"] for c in ao.CASES])
def test_model_against_reference_goldens(lib, case):
    from gpboost_b200 import GPModel
    c = spec(case)
    got, mdl = ao.run_case(GPModel, c)
    gold = {g["name"]: g for g in golden_cases()}.get(case)
    # the frozen-set likelihoods against the restatement
    X, y, _ = ao.case_data(c)
    t1, t2 = ao.thetas(c)
    o = ao.AnisoOracle(X, c["m"], c["cov"], c["shape"], c["ordering"], c["seed"])
    assert rel(got["nll_t1"], o.neg_log_likelihood(t1, y)) <= 1e-8
    assert rel(got["nll_t2_same"], o.neg_log_likelihood(t2, y)) <= 1e-8
    assert got["nll_t2_same"] == got["nll_t2_fresh"]
    assert got["names"][2:] == (["GP_range_time", "GP_range_space"] if "space_time" in c["cov"] else
                                ["GP_range_%d" % (k + 1) for k in range(c["d"])])
    if c.get("maxit", 1000) > 0:
        assert search_schedule(got["num_it"]) <= mdl._get_num_neighbor_searches() <= 1 + got["num_it"]
    assert gold is not None, "no golden for " + case
    for k in ("nll_t1", "nll_t2_same", "nll_t2_fresh"):
        assert rel(got[k], gold[k]) <= 1e-8, (k, got[k], gold[k])
    if c.get("maxit", 1000) == 0:
        np.testing.assert_allclose(got["cov_pars"], gold["cov_pars"], rtol=1e-10)
        return
    assert abs(got["num_it"] - gold["num_it"]) <= 3
    assert rel(got["nll_fit"], gold["nll_fit"]) <= 1e-6
    np.testing.assert_allclose(got["cov_pars"], gold["cov_pars"], rtol=2e-2)
    tol = 1e-6 if (c["cov"] == "gaussian_ard" or c["shape"] == 2.5) else 1e-8
    if got["cov_pars"] == gold["cov_pars"] and "pred_mu" in gold:
        np.testing.assert_allclose(got["pred_mu"], gold["pred_mu"], rtol=tol, atol=tol)
        np.testing.assert_allclose(got["pred_var"], gold["pred_var"], rtol=tol, atol=tol)


def test_prediction_at_golden_parameters(lib):
    """prediction at the reference's fitted parameters: neighbours searched in the space scaled by them"""
    from gpboost_b200 import GPModel
    for gold in golden_cases():
        c = spec(gold["name"])
        if c.get("maxit", 1000) == 0 or 2 * c["m"] > 60:
            continue
        X, y, Xp = ao.case_data(c)
        m = ao.make_model(GPModel, c, X)
        p = m.predict(y, Xp, np.array(gold["cov_pars"]), predict_var=True, predict_response=True)
        tol = 1e-6 if (c["cov"] == "gaussian_ard" or c["shape"] == 2.5) else 1e-8
        np.testing.assert_allclose(p["mu"], gold["pred_mu"], rtol=tol, atol=tol * np.abs(gold["pred_mu"]).max())
        np.testing.assert_allclose(p["var"], gold["pred_var"], rtol=tol)


def test_refusals(lib):
    from gpboost_b200 import GPModel, GPBoostError
    from gpboost_b200.booster import Booster, Dataset
    rng = np.random.default_rng(0)
    X = rng.uniform(0., 1., (300, 2))
    y = rng.standard_normal(300)
    with pytest.raises(GPBoostError, match="only supported for likelihood 'gaussian'"):
        GPModel(likelihood="bernoulli_logit", gp_coords=X, cov_function="matern_ard", gp_approx="vecchia")
    with pytest.raises(GPBoostError, match="only supported with gp_approx = 'vecchia'"):
        GPModel(gp_coords=X, cov_function="matern_ard", gp_approx="none")
    with pytest.raises(GPBoostError, match="not supported by the CUDA engine"):
        GPModel(gp_coords=X, cov_function="matern_ard_estimate_shape", gp_approx="vecchia")
    with pytest.raises(GPBoostError, match="not supported by the CUDA engine"):
        GPModel(gp_coords=X, cov_function="space_time_gneiting", gp_approx="vecchia")
    with pytest.raises(GPBoostError, match="Matern smoothness"):
        GPModel(gp_coords=X, cov_function="matern_ard", cov_fct_shape=0.8, gp_approx="vecchia")
    with pytest.raises(GPBoostError, match="not a space-time covariance function"):
        GPModel(gp_coords=X, cov_function="matern_ard", gp_approx="vecchia", vecchia_ordering="time")
    with pytest.raises(GPBoostError, match="at most 16 coordinates"):
        GPModel(gp_coords=rng.uniform(0., 1., (300, 17)), cov_function="matern_ard", gp_approx="vecchia")
    with pytest.raises(GPBoostError, match="num_neighbors"):
        GPModel(gp_coords=X, cov_function="matern_ard", gp_approx="vecchia", num_neighbors=61)
    m = GPModel(gp_coords=X, cov_function="matern_ard", gp_approx="vecchia", num_neighbors=10)
    with pytest.raises(GPBoostError, match="covariates are not supported"):
        m.fit(y, X=np.ones((300, 1)))
    m.fit(y, params=dict(maxit=5))
    assert not m._can_calculate_standard_errors_cov_pars()
    with pytest.raises(GPBoostError, match="Standard errors"):
        out = np.zeros(8)
        m._safe_call(m._LIB.GPB_GetCovPar(m.handle, P(out), C.c_bool(True)))
    with pytest.raises(GPBoostError, match="GPBoost algorithm"):
        params = dict(objective="regression", num_leaves=4, verbose=-1)
        Booster(params, Dataset(rng.standard_normal((300, 3)), y, params=params), gp_model=m)
