"""Standard errors of the Gaussian Vecchia model's covariance parameters on the device (gpboost_b200/csrc/dev/fisher.cuh,
REModel::GetCovPar with calc_std_dev): the device Fisher information against the oracle's (oracle/std_err.py) at every probe-column
grouping; get_cov_pars(std_err=True) against the reference's goldens (tests/golden/std_err_golden.json); which models can compute
them; the per-fit cache and the probe draws; and that computing them changes nothing that follows."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

import datagen
from oracle import std_err as ose
from oracle import vecchia as ov

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_std_err_golden as mk  # noqa: E402

pytestmark = pytest.mark.gpu

with open(os.path.join(HERE, "golden", "std_err_golden.json")) as f:
    GOLD = json.load(f)["cases"]
BY_NAME = {c["name"]: c for c in GOLD}


def P(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


@pytest.fixture(scope="module")
def lib(product_lib):
    assert product_lib.gpbdev_device_count() > 0, "no CUDA device visible — GPU tests need an H100"
    return product_lib


def chk(lib, rc):
    assert rc == 0, lib.gpbdev_last_error().decode()


def gp_model(coords, cov_function="matern", shape=1.5, m=20, seed=1, **kw):
    from gpboost_b200 import GPModel
    return GPModel(gp_coords=coords, cov_function=cov_function, cov_fct_shape=shape, gp_approx="vecchia", num_neighbors=m,
                   vecchia_ordering="random", seed=seed, **kw)


def engine_of(model):
    eng = C.c_void_p()
    model._safe_call(model._LIB.GPB200_GetDeviceEngine(model.handle, C.byref(eng)))
    return eng


# (n, d, kernel, shape, m, t): t = 1, a partial column group, the default 50, exactly one block of 128, one column past it, three
# blocks; n = 60 with m = 30 puts half the rows in the chain-like start of the order (row i conditions on all i predecessors)
FI_CASES = [(2000, 2, "matern", 1.5, 20, 1), (2000, 2, "matern", 1.5, 20, 32), (3000, 2, "exponential", 0.5, 30, 50),
            (1500, 3, "matern", 1.5, 10, 128), (1500, 1, "exponential", 0.5, 20, 129), (1000, 2, "matern", 1.5, 30, 300),
            (60, 1, "exponential", 0.5, 30, 129)]


@pytest.mark.parametrize("case", FI_CASES, ids=lambda c: "n%d_d%d_%s%.1f_m%d_t%d" % c)
def test_device_fisher_information_matches_oracle(lib, case):
    """gpbdev_vecchia_fisher_info at the oracle's order and neighbour sets and the same probe block: every entry within 1e-9 of the
    scale sqrt(FI_aa FI_bb) (fp64 sums over n t products in another order), finite, symmetric, and bitwise equal over two calls."""
    n, d, cf, shape, m, t = case
    coords, _ = datagen.synth(n, d, 40 + t)
    vo = ov.VecchiaOracle(coords, m, cf, shape, "random", 3)
    cov_pars = [0.3, 1.2, 0.15]
    s2, pt = ov.transform_cov_pars(cov_pars, cf, shape)
    Z = ose.probes(n, t, 1, 0)
    FI0 = ose.fisher_info(vo.coords, vo.nn, vo.cid, cov_pars, Z)
    h = C.c_void_p()
    chk(lib, lib.gpbdev_vecchia_create(C.byref(h), 0, C.c_int64(n), d, vo.m, P(vo.coords), P(vo.perm, C.c_int32),
                                       P(np.ascontiguousarray(vo.nn), C.c_int32), C.c_int64(0), C.c_int64(n)))
    try:
        Zc = np.asfortranarray(Z)
        out = [np.zeros(9), np.zeros(9)]
        for o in out:
            chk(lib, lib.gpbdev_vecchia_fisher_info(h, vo.cid, C.c_double(s2), C.c_double(pt[0]), C.c_double(pt[1]), P(Zc), t, P(o)))
    finally:
        lib.gpbdev_vecchia_free(h)
    FI = out[0].reshape(3, 3)
    assert np.array_equal(out[0], out[1])
    assert np.all(np.isfinite(FI)) and np.array_equal(FI, FI.T)
    scale = np.sqrt(np.outer(np.diag(FI0), np.diag(FI0)))
    assert np.max(np.abs(FI - FI0) / scale) <= 1e-9, (FI, FI0)


@pytest.mark.parametrize("name", [c["name"] for c in GOLD])
def test_get_cov_pars_std_err_matches_reference(lib, name):
    """get_cov_pars(std_err=True) through the same fits as the reference's script: the parameters and their standard errors within
    1e-8 (1e-6 for the Gaussian and Matern-2.5 kernels); after a real fit within 1e-3, the fits agreeing to the optimiser's
    tolerance only."""
    c = BY_NAME[name]
    fits = mk.run(c, None)
    assert len(fits) == len(c["fits"])
    tol = 1e-3 if c.get("fit") else (1e-6 if c["cov_function"] == "gaussian" or c["shape"] == 2.5 else 1e-8)
    for got, ref in zip(fits, c["fits"]):
        np.testing.assert_allclose(got["params"], ref["params"], rtol=tol if c.get("fit") else 1e-14, atol=0)
        np.testing.assert_allclose(got["std_err"], ref["std_err"], rtol=tol, atol=0)


def _can(model):
    out = C.c_int(-1)
    model._safe_call(model._LIB.GPB_CanCalculateStandardErrorsCovPars(model.handle, C.byref(out)))
    return out.value


def _refused(model, word):
    buf = np.zeros(2 * model.num_cov_pars)
    rc = model._LIB.GPB_GetCovPar(model.handle, P(buf), C.c_bool(True))
    msg = model._LIB.LGBM_GetLastError().decode()
    assert rc == -1 and "Standard errors" in msg and word in msg, msg
    # the table without the standard errors is what the frontend returns for such a model
    assert model.get_cov_pars(std_err=True).shape == (model.num_cov_pars,)


def test_which_models_can_calculate_standard_errors(lib):
    from gpboost_b200 import GPModel
    from gpboost_b200.booster import Booster, Dataset
    rng = np.random.default_rng(5)
    n = 400
    coords = rng.random((n, 2))
    y = np.sin(4 * coords[:, 0]) + 0.3 * rng.standard_normal(n)
    fixed = dict(init_cov_pars=np.array([0.3, 1.0, 0.1]), maxit=0)
    for m in (1, 30):
        g = gp_model(coords, m=m)
        g.fit(y, params=fixed)
        assert _can(g) == 1
        assert g.get_cov_pars(std_err=True).shape == (2, 3)
    gx = gp_model(coords, m=20)
    gx.fit(y, X=np.column_stack([np.ones(n), rng.standard_normal(n)]), params=fixed)
    assert _can(gx) == 1 and np.all(np.isfinite(gx.get_cov_pars(std_err=True)))
    # the GP model behind a booster (the Fisher information does not depend on the response)
    gb = gp_model(coords, m=15)
    X = rng.random((n, 3))
    bst = Booster({"objective": "regression", "num_leaves": 8, "min_data_in_leaf": 20, "learning_rate": 0.1, "verbose": -1},
                  Dataset(X, y + X[:, 0]), gp_model=gb)
    for _ in range(2):
        bst.update()
    assert _can(gb) == 1 and np.all(np.isfinite(gb.get_cov_pars(std_err=True)))
    # refused: m > 30, grouped, exact dense GP, non-Gaussian likelihoods
    g40 = gp_model(coords, m=40)
    g40.fit(y, params=fixed)
    assert _can(g40) == 0
    _refused(g40, "num_neighbors")
    grp = GPModel(group_data=rng.integers(0, 20, n))
    grp.fit(y, params=dict(init_cov_pars=np.array([0.3, 1.0]), maxit=0))
    assert _can(grp) == 0
    _refused(grp, "vecchia")
    dense = GPModel(gp_coords=coords[:200], cov_function="matern", cov_fct_shape=1.5, gp_approx="none")
    dense.fit(y[:200], params=fixed)
    assert _can(dense) == 0
    _refused(dense, "vecchia")
    for lik, yy in (("bernoulli_logit", (y > 0).astype(float)), ("poisson", rng.poisson(2., n).astype(float))):
        gl = gp_model(coords, m=10, likelihood=lik)
        gl.fit(yy, params=dict(init_cov_pars=np.array([1.0, 0.1]), maxit=0))
        assert _can(gl) == 0
        _refused(gl, lik)


def test_cache_refit_and_probe_draws(lib):
    """Computed once per fit: a second call launches no kernel and returns the same numbers; a refit recomputes. Without
    reuse_rand_vec_trace every computation draws new probes (the generator counter advances): recomputing at the same parameters
    after a refit changes the estimate, with it the estimate is reproduced bit for bit."""
    coords, y = datagen.synth(1500, 2, 61)
    fixed = dict(init_cov_pars=np.array([0.3, 1.0, 0.1]), maxit=0)
    for reuse in (True, False):
        g = gp_model(coords, m=20)
        g.fit(y, params=dict(fixed, reuse_rand_vec_trace=reuse))
        eng = engine_of(g)
        a = g.get_cov_pars(std_err=True)
        k = lib.gpbdev_vecchia_launch_count(eng)
        b = g.get_cov_pars(std_err=True)
        assert lib.gpbdev_vecchia_launch_count(eng) == k and np.array_equal(a, b)
        g.fit(y, params=fixed)
        c = g.get_cov_pars(std_err=True)
        assert lib.gpbdev_vecchia_launch_count(eng) > k
        assert np.array_equal(a, c) == reuse
        g.fit(y, params=dict(init_cov_pars=np.array([0.5, 0.7, 0.3]), maxit=0))
        d = g.get_cov_pars(std_err=True)
        assert not np.array_equal(d[1], c[1])


def test_later_results_are_unchanged(lib):
    """A likelihood, a response gradient, a prediction and three boosting iterations with a GP model give bit-identical results with
    and without get_cov_pars(std_err=True) in between (the Fisher pass forms its factor in buffers of its own and leaves the engine's
    stored factor and its shortcut state alone)."""
    from gpboost_b200.booster import Booster, Dataset
    coords, y = datagen.synth(3000, 2, 62)
    rng = np.random.default_rng(62)
    cp = rng.random((50, 2))

    def run(with_se):
        g = gp_model(coords, m=25)
        g.fit(y, params=dict(maxit=5))
        res = []
        if with_se:
            g.get_cov_pars(std_err=True)
        res.append(g.get_cov_pars())
        res.append(np.array([g.neg_log_likelihood(g.get_cov_pars(), y)]))
        if with_se:
            g.get_cov_pars(std_err=True)
        res.append(g.response_gradient(y))
        r = g.predict(y, cp, g.get_cov_pars(), predict_var=True)
        res += [r["mu"], r["var"]]
        gb = gp_model(coords, m=15)
        X = np.random.default_rng(7).random((3000, 3))
        bst = Booster({"objective": "regression", "num_leaves": 8, "min_data_in_leaf": 20, "learning_rate": 0.1, "verbose": -1},
                      Dataset(X, y + X[:, 0]), gp_model=gb)
        for _ in range(3):
            bst.update()
            if with_se:
                gb.get_cov_pars(std_err=True)
        res += [bst.inner_predict_train(), gb.get_cov_pars()]
        return res, bst.model_to_string()

    (a, ta), (b, tb) = run(False), run(True)
    assert ta == tb
    for x, z in zip(a, b):
        assert np.array_equal(x, z)


def test_large_n_runs(lib):
    """n = 1e5, m = 30: the large-n path (many column blocks of rows per warp, long dependency chains of the solves) gives finite,
    positive standard errors."""
    coords, y = datagen.synth(100000, 2, 63)
    g = gp_model(coords, m=30)
    g.fit(y, params=dict(init_cov_pars=np.array([0.25, 1.0, 0.1]), maxit=0))
    tab = g.get_cov_pars(std_err=True)
    assert tab.shape == (2, 3) and np.all(np.isfinite(tab)) and np.all(tab[1] > 0)


DROPIN = """
rng = np.random.default_rng(8)
n = 800
coords = rng.random((n, 2))
y = np.sin(4 * coords[:, 0]) + np.cos(3 * coords[:, 1]) + 0.3 * rng.standard_normal(n)
m = gpb.GPModel(gp_coords=coords, cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia", num_neighbors=10,
                vecchia_ordering="random", seed=1)
m.fit(y=y, params={"init_cov_pars": np.array([0.3, 1.0, 0.1]), "maxit": 0})
out["table"] = np.asarray(m.get_cov_pars(std_err=True, format_pandas=False)).tolist()
df = m.get_cov_pars(std_err=True)
out["index"] = list(df.index)
m.summary()
"""


def test_reference_package_std_err_matches_reference_library(lib):
    """The unmodified reference package: get_cov_pars(std_err=True) and summary() on this library give the reference library's
    table (rows Param. and Std. err.). Runs where the upstream checkout and the reference build are present."""
    import dropin
    from oracle import ref_lib_path
    if dropin.ref_package_dir() is None or not os.path.exists(ref_lib_path()):
        pytest.skip("upstream GPBoost checkout / reference build not present")
    prod = dropin.run_with(os.path.join(os.path.dirname(HERE), "gpboost_b200", "lib_gpboost_b200.so"), DROPIN)
    ref = dropin.run_with(ref_lib_path(), DROPIN)
    assert prod["index"] == ref["index"] == ["Param.", "Std. err."]
    np.testing.assert_allclose(prod["table"], ref["table"], rtol=1e-8, atol=0)
