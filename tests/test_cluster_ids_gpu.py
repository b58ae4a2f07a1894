"""Gaussian Vecchia GP with several independent realizations (cluster_ids) on the device, against the reference library's outputs
(tests/golden/cluster_golden.json, tests/golden/make_cluster_golden.py) and the oracle's per-cluster neighbour search and factor."""
import ctypes
import json
import os

import numpy as np
import pytest

import cluster_cases as cc
import cluster_oracle as co
from gpboost_b200 import GPModel
from gpboost_b200.booster import Booster, Dataset, parse_model_string
from oracle import vecchia as ov

pytestmark = pytest.mark.gpu

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "cluster_golden.json")))
GCASES = {r["name"]: r for r in GOLDEN["cases"]}


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-300)))


@pytest.mark.parametrize("c", cc.CASES, ids=[c["name"] for c in cc.CASES])
def test_against_reference(c):
    g = GCASES[c["name"]]
    r = cc.run_case(c)
    assert rel(r["nll"], g["nll"]) <= 1e-8, (r["nll"], g["nll"])
    assert r["num_it"] == g["num_it"]
    assert rel(r["cov_pars"], g["cov_pars"]) <= 1e-6, (r["cov_pars"], g["cov_pars"])
    assert rel(r["nll_fit"], g["nll_fit"]) <= 1e-8
    # means: relative to the scale of the means (a mean near 0 has no relative precision)
    scale = np.max(np.abs(g["pred_mu_fixed"]))
    assert np.max(np.abs(np.subtract(r["pred_mu_fixed"], g["pred_mu_fixed"]))) <= 1e-8 * scale
    assert rel(r["pred_var_latent_fixed"], g["pred_var_latent_fixed"]) <= 1e-8
    scale = np.max(np.abs(g["pred_mu"]))
    assert np.max(np.abs(np.subtract(r["pred_mu"], g["pred_mu"]))) <= 1e-6 * scale
    assert rel(r["pred_var"], g["pred_var"]) <= 1e-6
    # a label without training data: the prior, mean 0 and variance sigma_1^2 + sigma^2 (the reference keeps the nugget in the latent
    # variance of such a point)
    lab_p = cc.case_data(c)[4]
    new = lab_p == cc.NEW_LABEL
    assert np.all(np.asarray(r["pred_mu_fixed"])[new] == 0.)
    assert np.allclose(np.asarray(r["pred_var_latent_fixed"])[new], cc.COV_PARS[0] + cc.COV_PARS[1], rtol=1e-14, atol=0.)


def _device_state(gp, n, m, cov_pars, y, c):
    """the engine's ordering and neighbour table, its stored factor and its gradient sums at cov_pars"""
    lib = gp._LIB
    eng = gp.device_engine()
    ip = ctypes.POINTER(ctypes.c_int32)
    dp = ctypes.POINTER(ctypes.c_double)
    nn = np.empty((n, m), dtype=np.int32)
    perm = np.empty(n, dtype=np.int32)
    assert lib.gpbdev_vecchia_get_nn(eng, nn.ctypes.data_as(ip)) == 0
    assert lib.gpbdev_vecchia_get_perm(eng, perm.ctypes.data_as(ip)) == 0
    gp.neg_log_likelihood(np.array(cov_pars), y)  # installs y
    _, pt = ov.transform_cov_pars(cov_pars, c["cov"], c["shape"])
    cid = ov.cov_id(c["cov"], c["shape"])
    gsums = np.empty(9)
    assert lib.gpbdev_vecchia_eval(eng, cid, ctypes.c_double(pt[0]), ctypes.c_double(pt[1]), 2, gsums.ctypes.data_as(dp)) == 0
    sums = np.empty(9)
    assert lib.gpbdev_vecchia_eval(eng, cid, ctypes.c_double(pt[0]), ctypes.c_double(pt[1]), 1, sums.ctypes.data_as(dp)) == 0
    A = np.empty((n, m)); Dinv = np.empty(n)
    assert lib.gpbdev_vecchia_get_factor(eng, A.ctypes.data_as(dp), Dinv.ctypes.data_as(dp)) == 0
    s2 = cov_pars[0]
    grad = np.array([(gsums[3 + k] - 0.5 * gsums[5 + k]) / s2 + 0.5 * gsums[7 + k] for k in range(2)])  # re_model.cpp gradient assembly
    return perm, nn, A, Dinv, grad


# a cluster of more than 4096 points searches its own cell grid from its 4097th point on
BIG_GRID_CASE = dict(name="grid_cluster_none", labels=[8, 3, 5], sizes=[5000, 300, 4], m=10, cov="matern", shape=1.5, ordering="none", seed=9)
BIG_GRID_RANDOM = dict(BIG_GRID_CASE, name="grid_cluster_random", ordering="random")


@pytest.mark.parametrize("c", cc.CASES + [BIG_GRID_CASE, BIG_GRID_RANDOM], ids=lambda c: c["name"])
def test_neighbours_factor_and_gradient_per_cluster(c):
    """The engine's rows are cluster-major (clusters in order of first appearance). Within every cluster, in the engine's own order
    ('none': data order; 'random': the per-cluster shuffle), every row's neighbours are the oracle's search of that cluster alone,
    bit-exact, head rows and the head/body boundary included; the factor matches the oracle's factor of the cluster, with the padded
    coefficients of short rows exactly 0; and the gradient at given parameters is the sum of the clusters' gradients"""
    coords, y, lab, _, _ = cc.case_data(c)
    gp = cc.model_of(c, coords, lab)
    n = len(lab)
    sizes = [int(np.sum(lab == l)) for l in dict.fromkeys(lab.tolist())]
    m = min(c["m"], max(sizes) - 1)
    perm, nn, A, Dinv, grad = _device_state(gp, n, m, cc.COV_PARS, y, c)
    want = co.clustered(coords, lab, y, c["m"], c["cov"], c["shape"], cc.COV_PARS, perm=perm, calc_grad=True)
    start = 0
    for rows, wn, Ao, Do in want["parts"]:
        nc = len(rows)
        assert np.array_equal(perm[start:start + nc], rows)  # cluster-major, the cluster's own order
        k = wn.shape[1] if nc > 1 else 0
        w = np.full((nc, m), -1, dtype=np.int32)
        w[:, :k] = np.where(wn[:, :k] >= 0, wn[:, :k] + start, -1)
        got = nn[start:start + nc]
        assert np.array_equal(got, w), (nc, np.argwhere(got != w)[:5])
        assert np.max(np.abs(Dinv[start:start + nc] - Do) / np.abs(Do)) <= 1e-10
        if k:
            assert np.max(np.abs(A[start:start + nc, :k] - Ao[:, :k])) <= 1e-10
        assert np.all(A[start:start + nc][got == -1] == 0.)  # padding and dummy slots carry no coefficient
        start += nc
    assert start == n
    assert np.max(np.abs(grad - want["grad"]) / np.abs(want["grad"])) <= 1e-8, (grad, want["grad"])


@pytest.mark.parametrize("c", [cc.CASES[1], cc.CASES[2]], ids=lambda c: c["name"])
def test_all_equal_cluster_ids_bitwise(c):
    """one label for every point: the model is the model without cluster_ids, to the bit"""
    coords, y, _, coords_p, _ = cc.case_data(c)
    lab = np.full(len(y), 3, dtype=np.int32)
    a = cc.model_of(c, coords, lab)
    b = cc.model_of(c, coords, lab, cluster_ids=False)
    assert a.neg_log_likelihood(np.array(cc.COV_PARS), y) == b.neg_log_likelihood(np.array(cc.COV_PARS), y)
    a.fit(y); b.fit(y)
    assert np.array_equal(a.get_cov_pars(), b.get_cov_pars()) and a._get_num_optim_iter() == b._get_num_optim_iter()
    mp = c.get("mp", -1)
    pa = a.predict(y=y, gp_coords_pred=coords_p, cov_pars=None, predict_var=True, cluster_ids_pred=np.full(len(coords_p), 3),
                   num_neighbors_pred=mp)
    pb = b.predict(y=y, gp_coords_pred=coords_p, cov_pars=None, predict_var=True, num_neighbors_pred=mp)
    assert np.array_equal(pa["mu"], pb["mu"]) and np.array_equal(pa["var"], pb["var"])
    # the same label as the training data's, and a label of no training data (the prior)
    pc = a.predict(y=y, gp_coords_pred=coords_p, cov_pars=None, predict_var=True, predict_response=False,
                   cluster_ids_pred=np.full(len(coords_p), 4), num_neighbors_pred=mp)
    cp = np.asarray(a.get_cov_pars()).reshape(-1)
    assert np.all(pc["mu"] == 0.) and np.allclose(pc["var"], cp[0] + cp[1], rtol=1e-14)


def _trees(model):
    return parse_model_string(model)


def test_gpboost_fixed_cov_pars_every_tree():
    g = GOLDEN["boost_fixed"]
    r, _ = cc.run_boost(cc.BOOST_CASE, train_cov_pars=False)
    tg, tr = _trees(g["model"]), _trees(r["model"])
    assert len(tg) == len(tr)
    for a, b in zip(tr, tg):
        assert a["num_leaves"] == b["num_leaves"]
        for k in ("split_feature", "left_child", "right_child", "threshold"):
            assert np.array_equal(a[k], b[k]), k
        assert np.allclose(a["leaf_value"], b["leaf_value"], rtol=1e-9, atol=1e-12)
    for er, eg in zip(r["evals"], g["evals"]):
        assert [e[1] for e in er] == [e[1] for e in eg]
        assert rel([e[2] for e in er], [e[2] for e in eg]) <= 1e-8


@pytest.mark.parametrize("key", sorted(cc.BOOST_VARIANTS))
def test_gpboost_newton_leaf_updates(key):
    """Newton leaf updates read the resident factor of the clustered model (its -1 padded head rows included): every tree and validation
    metric against the reference"""
    g = GOLDEN[key]
    r, _ = cc.run_boost(cc.BOOST_CASE, train_cov_pars=False, extra=cc.BOOST_VARIANTS[key])
    tg, tr = _trees(g["model"]), _trees(r["model"])
    assert len(tg) == len(tr)
    for a, b in zip(tr, tg):
        assert a["num_leaves"] == b["num_leaves"]
        for k in ("split_feature", "left_child", "right_child", "threshold"):
            assert np.array_equal(a[k], b[k]), k
        assert np.allclose(a["leaf_value"], b["leaf_value"], rtol=1e-8, atol=1e-12)
    for er, eg in zip(r["evals"], g["evals"]):
        assert rel([e[2] for e in er], [e[2] for e in eg]) <= 1e-8


def test_gpboost_trained_cov_pars_first_tree():
    g = GOLDEN["boost_trained"]
    r, _ = cc.run_boost(cc.BOOST_CASE, train_cov_pars=True, num_it=1)
    assert rel(r["cov_pars"], g["cov_pars"]) <= 1e-5
    a, b = _trees(r["model"])[0], _trees(g["model"])[0]
    assert a["num_leaves"] == b["num_leaves"] and np.array_equal(a["split_feature"], b["split_feature"])
    assert np.allclose(a["leaf_value"], b["leaf_value"], rtol=1e-5, atol=1e-8)


def test_refusals():
    c = cc.CASES[0]
    coords, y, lab, _, _ = cc.case_data(c)
    with pytest.raises(Exception, match="cluster_ids"):
        GPModel(gp_coords=coords, cov_function="matern_ard", gp_approx="vecchia", num_neighbors=10, cluster_ids=lab)
    with pytest.raises(Exception, match="cluster_ids"):
        GPModel(gp_coords=coords, cov_function="exponential", gp_approx="none", cluster_ids=lab)
    with pytest.raises(Exception, match="cluster_ids"):
        GPModel(gp_coords=coords, likelihood="bernoulli_logit", cov_function="exponential", gp_approx="vecchia", cluster_ids=lab)
    with pytest.raises(Exception, match="cluster_ids"):
        GPModel(group_data=lab % 3, cluster_ids=lab)
    gp = cc.model_of(c, coords, lab)
    with pytest.raises(Exception, match="cluster_ids"):
        gp.fit(y, X=np.ones((len(y), 1)))
    gp.fit(y)
    # standard errors: the frontend asks first and returns the parameters alone, as the reference package does
    assert not gp._can_calculate_standard_errors_cov_pars()
    assert np.asarray(gp.get_cov_pars(std_err=True)).shape == (3,)
    out = np.zeros(6)
    assert gp._LIB.GPB_GetCovPar(gp.handle, out.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), ctypes.c_bool(True)) != 0
    assert "cluster_ids" in gp._LIB.LGBM_GetLastError().decode()


def test_line_search_is_refused():
    """the reference library fails an index assertion in the line search of the step length with cluster_ids, so there is nothing to
    match: refused with a message"""
    with pytest.raises(Exception, match="cluster_ids"):
        cc.run_boost(cc.BOOST_CASE, num_it=1, extra=dict(line_search_step_length=True))


def test_prediction_without_labels_is_refused():
    """a model of several clusters needs the prediction points' labels (re_model_template.h:3522): GPModel.predict, Booster.predict and
    the validation data of the boosting loop refuse to predict without them"""
    c = cc.CASES[0]
    coords, y, lab, coords_p, lab_p = cc.case_data(c)
    gp = cc.model_of(c, coords, lab)
    gp.fit(y)
    with pytest.raises(Exception, match="Missing cluster_id data"):
        gp.predict(y=y, gp_coords_pred=coords_p, cov_pars=None, predict_var=True)
    _, bst = cc.run_boost(cc.BOOST_CASE, num_it=1)
    X, yb, coords_b, lab_b, Xv, yv, coords_v, lab_v = cc.boost_data(cc.BOOST_CASE)
    with pytest.raises(Exception, match="Missing cluster_id data"):
        bst.predict(Xv, gp_coords_pred=coords_v)
    out = bst.predict(Xv, gp_coords_pred=coords_v, cluster_ids_pred=lab_v, predict_var=True)
    assert np.all(np.isfinite(out["response_mean"])) and np.all(out["response_var"] > 0.)
    # validation data set without labels
    params = dict(objective="regression", num_leaves=8, min_data_in_leaf=20, verbose=-1, use_gp_model_for_validation=True,
                  train_gp_model_cov_pars=False)
    gpv = cc.model_of(cc.BOOST_CASE, coords_b, lab_b)
    gpv.set_optim_params(dict(init_cov_pars=np.array(cc.COV_PARS)))
    gpv.set_prediction_data(gp_coords_pred=coords_v)
    dtrain = Dataset(X, yb, params=params, free_raw_data=False)
    b2 = Booster(params, dtrain, gp_model=gpv)
    b2.add_valid(Dataset(Xv, yv, params=params, reference=dtrain), "valid")
    with pytest.raises(Exception, match="Missing cluster_id data"):
        b2.update()
        b2.eval_valid()


def test_one_label_without_prediction_labels():
    """cluster_ids all equal to 5: prediction without labels reads every point as label 0, as the reference does (SetUpClusterIds), so
    the points belong to no training cluster and get the prior; with label 5 they are the model without cluster_ids, to the bit"""
    c = cc.CASES[0]
    coords, y, _, coords_p, _ = cc.case_data(c)
    a = cc.model_of(c, coords, np.full(len(y), 5, dtype=np.int32))
    b = cc.model_of(c, coords, None, cluster_ids=False)
    pa = a.predict(y=y, gp_coords_pred=coords_p, cov_pars=np.array(cc.COV_PARS), predict_var=True, predict_response=False)
    assert np.all(pa["mu"] == 0.) and np.allclose(pa["var"], cc.COV_PARS[0] + cc.COV_PARS[1], rtol=1e-14)
    p5 = a.predict(y=y, gp_coords_pred=coords_p, cov_pars=np.array(cc.COV_PARS), predict_var=True, predict_response=False,
                   cluster_ids_pred=np.full(len(coords_p), 5))
    pb = b.predict(y=y, gp_coords_pred=coords_p, cov_pars=np.array(cc.COV_PARS), predict_var=True, predict_response=False)
    assert np.array_equal(p5["mu"], pb["mu"]) and np.array_equal(p5["var"], pb["var"])
