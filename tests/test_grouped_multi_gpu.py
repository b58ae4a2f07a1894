"""Several grouped random effects (crossed, nested, K = 3), Gaussian likelihood, on the device: the iterative method with the SSOR
preconditioner against the reference's goldens (tests/golden/grouped_multi_golden.json) and the numpy restatement (oracle/grouped_multi.py).

Tolerances and why:
- NLL against the reference's iterative value 1e-6 relative (the Laplace bar): same probe vectors, iterations and stopping rules, so
  only summation order and fused multiply-adds differ, and the SLQ estimate passes them through eigenvalue logs;
- NLL against the reference's Cholesky value 2e-3 relative: the iterative value carries the stochastic error of 50 probe vectors;
- CG / Lanczos iteration counts equal to the reference's and the oracle's; log-det and quadratic form against the oracle 1e-9 relative;
- single operators (M X, P^-1 X, L D^-1/2 X, D^-1 upper(M) X) against the oracle 1e-12 relative to the largest entry: one sparse row
  product and at most K diagonal scalings per entry;
- gradient against the oracle 1e-7 relative to its largest entry: a difference of means of 50 probe columns, each a sum over G rows;
- fits: parameters within 2e-3 and iteration count within 2 of the golden, as for the single-level model;
- GPBoost with fixed covariance parameters: every tree's structure equal, leaf values within 1e-6 relative (the gradient is a CG
  solution to an absolute residual of 1e-2, reached in the same iterations); with trained parameters 5e-3 on the covariance parameters
  and 2e-3 on the scores (optimiser tolerance);
- repeated calls bitwise equal (every reduction has a fixed order)."""
import ctypes
import json
import os

import numpy as np
import pytest

import grouped_multi_data as gmd
from oracle import grouped_multi as gm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DP = ctypes.POINTER(ctypes.c_double)


@pytest.fixture(scope="module")
def gold():
    with open(os.path.join(ROOT, "tests", "golden", "grouped_multi_golden.json")) as f:
        return json.load(f)


def _p(a):
    return a.ctypes.data_as(DP)


class Engine:
    """The device engine driven directly (gpbdev_grouped_multi_*), with the oracle's structure."""

    def __init__(self, lib, group, y, probes):
        self.lib, self.st = lib, gm.Structure(group)
        lib.gpbdev_grouped_last_error.restype = ctypes.c_char_p
        idx = np.ascontiguousarray(np.concatenate(self.st.idx).astype(np.int32))
        lv = np.array(self.st.levels, dtype=np.int32)
        self.h = ctypes.c_void_p()
        self._ok(lib.gpbdev_grouped_multi_create(ctypes.byref(self.h), 0, ctypes.c_int64(len(y)), len(lv),
                                                 idx.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), lv.ctypes.data_as(ctypes.POINTER(ctypes.c_int))))
        self._ok(lib.gpbdev_grouped_multi_set_y(self.h, _p(np.ascontiguousarray(y, dtype=np.float64))))
        pr = np.asfortranarray(probes)
        self._ok(lib.gpbdev_grouped_multi_set_probes(self.h, _p(pr.reshape(-1, order="F")), probes.shape[1]))

    def _ok(self, rc):
        assert rc == 0, self.lib.gpbdev_grouped_last_error().decode()

    def eval(self, v, cfg=(1000, 1000, 1e-2, 0)):
        out = np.zeros(5)
        self._ok(self.lib.gpbdev_grouped_multi_eval(self.h, _p(np.asarray(v, dtype=np.float64)), _p(np.asarray(cfg, dtype=np.float64)), _p(out)))
        return out

    def grad(self, sigma2):
        g = np.zeros(self.st.K)
        self._ok(self.lib.gpbdev_grouped_multi_grad(self.h, ctypes.c_double(sigma2), _p(g)))
        return g

    def apply(self, v, which, X):
        X = np.ascontiguousarray(X, dtype=np.float64)
        Y = np.zeros_like(X)
        self._ok(self.lib.gpbdev_grouped_multi_apply(self.h, _p(np.asarray(v, dtype=np.float64)), which, _p(X), X.shape[1], _p(Y)))
        return Y

    def __del__(self):
        self.lib.gpbdev_grouped_multi_free(self.h)


def _cov(name, j=0):
    group, y, it = gmd.case(name)
    return group, y, it, np.array(gmd.COV_PARS[group.shape[1]][j])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["crossed", "nested", "three", "strings"])
def test_operators_against_oracle(product_lib, name):
    group, y, _, cp = _cov(name)
    st = gm.Structure(group)
    v = cp[1:] / cp[0]
    e = Engine(product_lib, group, y, gm.probes(st, 7))
    M = st.M(v)
    pc = gm.SSOR(M)
    X = np.random.default_rng(5).standard_normal((st.G, 7))
    import scipy.sparse as sp
    want = [M @ X, pc.solve(X), pc.LD @ X, pc.Dinv[:, None] * (sp.triu(M, format="csr") @ X)]
    for which, w in enumerate(want):
        got = e.apply(v, which, X)
        assert np.abs(got - w).max() <= 1e-12 * np.abs(w).max(), (name, which, np.abs(got - w).max())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(gmd.CASES))
def test_engine_eval_and_gradient_against_oracle(product_lib, name):
    group, y, it, cp = _cov(name)
    st = gm.Structure(group)
    cfg = dict(gm.DEFAULTS, **it)
    r = gm.probes(st, cfg["num_rand_vec_trace"], cfg["seed_rand_vec_trace"])
    v = cp[1:] / cp[0]
    want = gm.evaluate(st, y, v, sigma2=cp[0], r=r, with_grad=True, **it)
    e = Engine(product_lib, group, y, r)
    out = e.eval(v, (cfg["cg_max_num_it"], cfg["cg_max_num_it_tridiag"], cfg["cg_delta_conv"], 0))
    assert out[2] == want["its"] and out[3] == want["its_tridiag"], (out, want["its"], want["its_tridiag"])
    assert abs(out[0] - want["quad"]) <= 1e-9 * abs(want["quad"])
    assert abs(out[1] - want["logdet"]) <= 1e-9 * abs(want["logdet"])
    x = np.zeros(st.G)
    product_lib.gpbdev_grouped_multi_apply(e.h, _p(v), 4, None, 1, _p(x))
    assert np.abs(x - want["x"]).max() <= 1e-10 * np.abs(want["x"]).max()
    g = e.grad(cp[0])
    assert np.abs(g - want["grad"]).max() <= 1e-7 * np.abs(want["grad"]).max(), (g, want["grad"])
    # repeat: bitwise
    out2 = e.eval(v, (cfg["cg_max_num_it"], cfg["cg_max_num_it_tridiag"], cfg["cg_delta_conv"], 0))
    assert np.array_equal(out, out2)
    assert np.array_equal(g, e.grad(cp[0]))


@pytest.mark.gpu
def test_negll_against_reference(gold, product_lib):
    from gpboost_b200 import GPModel
    for rec in gold["nll"]:
        group, y, it = gmd.case(rec["case"])
        m = GPModel(group_data=group)
        if it:
            m.set_optim_params(dict(it))
        v = m.neg_log_likelihood(np.array(rec["cov_pars"]), y)
        assert abs(v - rec["negll"]) <= 1e-6 * abs(rec["negll"]), (rec, v)
        assert abs(v - rec["negll_cholesky"]) <= 2e-3 * abs(rec["negll_cholesky"]), (rec, v)
        info = m.laplace_info()
        assert (info[2], info[3]) == (rec["cg_its"], rec["cg_its_tridiag"]), (rec, info)
        assert m.neg_log_likelihood(np.array(rec["cov_pars"]), y) == v  # repeat: bitwise


@pytest.mark.gpu
def test_fit_against_reference(gold, product_lib):
    from gpboost_b200 import GPModel
    for rec in gold["fit"]:
        group, y, _ = gmd.case(rec["case"])
        m = GPModel(group_data=group)
        m.fit(y)
        cp = m.get_cov_pars()
        print(rec["case"], "iters", m._get_num_optim_iter(), "ref", rec["num_it"], cp, rec["cov_pars"])
        assert np.all(np.abs(cp - np.array(rec["cov_pars"])) <= 2e-3 * np.abs(rec["cov_pars"])), (rec, cp)
        assert abs(m._get_num_optim_iter() - rec["num_it"]) <= 2
        assert abs(m.get_current_neg_log_likelihood() - rec["negll"]) <= 1e-5 * abs(rec["negll"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["crossed", "three"])
def test_response_gradient_against_oracle(product_lib, name):
    from gpboost_b200 import GPModel
    group, y, _, cp = _cov(name)
    m = GPModel(group_data=group)
    m.set_optim_params({"init_cov_pars": cp})
    g = m.response_gradient(y)
    st = gm.Structure(group)
    M = st.M(cp[1:] / cp[0])
    x, _ = gm.cg_vec(M, gm.SSOR(M), st.Z.T @ y, None, 1000, 1e-2)
    want = (y - st.Z @ x) / cp[0]
    assert np.abs(g - want).max() <= 1e-10 * np.abs(want).max()
    assert np.array_equal(g, m.response_gradient(y))


@pytest.mark.gpu
def test_gpboost_against_reference(gold, product_lib):
    from gpboost_b200 import GPModel
    from gpboost_b200.booster import Booster, Dataset, parse_model_string
    X, y, group = gmd.boost_case()
    for rec in gold["boost"]:
        params = dict(gmd.BOOST_PARAMS)
        gp = GPModel(group_data=group)
        if not rec["train_cov"]:
            params["train_gp_model_cov_pars"] = False
            gp.set_optim_params({"init_cov_pars": gmd.BOOST_FIXED_COV_PARS})
        b = Booster(params, Dataset(X, y, params=params), gp_model=gp)
        for _ in range(4):
            b.update()
        trees = parse_model_string(b.model_to_string())
        score = b.inner_predict_train()[:64]
        cp = gp.get_cov_pars()
        if not rec["train_cov"]:
            for t, g in zip(trees, rec["trees"]):
                assert np.array_equal(t["split_feature"], np.array(g["split_feature"]))
                assert np.array_equal(t["threshold"], np.array(g["threshold"]))
                assert np.max(np.abs(t["leaf_value"] - np.array(g["leaf_value"]))) <= 1e-6 * np.max(np.abs(g["leaf_value"]))
            assert np.abs(score - np.array(rec["score_head"])).max() <= 1e-6 * np.abs(rec["score_head"]).max()
        else:
            assert np.array_equal(trees[0]["split_feature"], np.array(rec["trees"][0]["split_feature"]))
            assert np.all(np.abs(cp - np.array(rec["cov_pars"])) <= 5e-3 * np.abs(rec["cov_pars"])), (cp, rec["cov_pars"])
            assert np.abs(score - np.array(rec["score_head"])).max() <= 2e-3 * np.abs(rec["score_head"]).max()
    # line_search_step_length runs on the device path
    params = dict(gmd.BOOST_PARAMS, line_search_step_length=True)
    b = Booster(params, Dataset(X, y, params=params), gp_model=GPModel(group_data=group))
    b.update()
    b.update()
    assert np.all(np.isfinite(b.inner_predict_train()))


@pytest.mark.gpu
def test_refusals(product_lib):
    from gpboost_b200 import GPModel
    from gpboost_b200.basic import GPBoostError
    from gpboost_b200.booster import Booster, Dataset
    group, y, _, cp = _cov("crossed")
    with pytest.raises(GPBoostError, match="use 'iterative', the reference's default"):
        GPModel(group_data=group, matrix_inversion_method="cholesky")
    m = GPModel(group_data=group)
    with pytest.raises(GPBoostError, match="supported: 'ssor'"):
        m.set_optim_params({"cg_preconditioner_type": "incomplete_cholesky"})
    m = GPModel(group_data=group)
    m.set_optim_params({"cg_preconditioner_type": "SSOR"})  # the reference's alias
    m.fit(y)
    out = np.zeros(6)
    with pytest.raises(GPBoostError, match="Standard errors"):
        m._safe_call(m._LIB.GPB_GetCovPar(m.handle, _p(out), ctypes.c_bool(True)))
    with pytest.raises(GPBoostError):
        m.predict(y, np.zeros((3, 1)), None)
    with pytest.raises(GPBoostError, match="covariates"):
        GPModel(group_data=group).fit(y, X=np.c_[np.ones(len(y)), np.arange(len(y)) / len(y)])
    X, yb, gb = gmd.boost_case()
    params = dict(gmd.BOOST_PARAMS, leaves_newton_update=True)
    b = Booster(params, Dataset(X, yb, params=params), gp_model=GPModel(group_data=gb))
    with pytest.raises(GPBoostError, match="Newton"):
        b.update()
