"""Validation data of the boosting loop on the device: reference-binned Datasets, validation scores (one tree walk per row and tree),
the fused metric kernel, the Vecchia GP's cached prediction at the validation points and gpboost_b200.train's early stopping.
Goldens: tests/golden/validation_golden.json (the unmodified reference library through the same frontend)."""
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import validation_cases as vc  # noqa: E402
from gpboost_b200 import GPModel, GPBoostError, train  # noqa: E402
from gpboost_b200.booster import Booster, Dataset, parse_model_string  # noqa: E402

pytestmark = pytest.mark.gpu

with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "validation_golden.json")) as _f:
    GOLD = json.load(_f)
GOLD_CASES = {c["name"]: c for c in GOLD["cases"]}
LOG2PI = np.log(2. * np.pi)


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


def _check_evals(got, want, tol):
    assert len(got) == len(want)
    for g_it, w_it in zip(got, want):
        assert [r[:2] for r in g_it] == [r[:2] for r in w_it]
        for g, w in zip(g_it, w_it):
            assert _rel(g[2], w[2]) <= tol, (g, w)


def _check_scores(got, want):
    """raw scores against the reference's GetPredict(data_idx): equal up to the last bits (the initial score BoostFromAverage adds
    to every score is a mean the reference sums in another order); this build's own Booster.predict is matched bitwise below"""
    for g, w in zip(got, want):
        g = np.array([float.fromhex(x) for x in g])
        w = np.array([float.fromhex(x) for x in w])
        np.testing.assert_allclose(g, w, rtol=1e-13, atol=1e-13)


@pytest.mark.parametrize("name", ["plain_two_valid", "train_as_valid", "late_add_replay", "plain_test_nll", "vecchia_default_nogpval",
                                  "grouped_nogpval"])
def test_tree_score_metrics_match_reference(name):
    """tree-only metrics within 1e-12 of the reference; final validation raw scores bitwise equal to its GetPredict(data_idx)"""
    c = GOLD_CASES[name]
    got, _, _, _ = vc.run_case(c)
    assert got["eval_names"] == c["eval_names"]
    _check_evals(got["evals"], c["evals"], 1e-12)
    _check_scores(got["valid_scores"], c["valid_scores"])
    if "train_scores" in c:
        _check_scores([got["train_scores"]], [c["train_scores"]])


@pytest.mark.parametrize("name", ["vecchia_default_gpval", "vecchia_l2_gpval"])
def test_gp_metrics_match_reference(name):
    """GP-augmented metrics at fixed covariance parameters within the prediction tolerance (1e-8)"""
    c = GOLD_CASES[name]
    got, _, _, _ = vc.run_case(c)
    assert got["eval_names"] == c["eval_names"]
    _check_evals(got["evals"], c["evals"], 1e-8)
    _check_scores(got["valid_scores"], c["valid_scores"])


@pytest.mark.parametrize("num_leaves", [31, 1024])
def test_valid_scores_equal_host_predict_every_iteration(num_leaves):
    c = dict(name="leaves", n=6000, nv=[1500], F=8, seed=11, num_leaves=num_leaves, metric="l2", gp=None)
    data = vc.case_data(c)
    params = vc.params_of(c)
    params["min_data_in_leaf"] = 2
    dtrain = Dataset(data[0][0], data[0][1], params=params)
    dvalid = Dataset(data[1][0], data[1][1], params=params, reference=dtrain)
    bst = Booster(params, dtrain)
    bst.add_valid(dvalid, "v")
    for _ in range(6):
        bst.update()
        got = bst.inner_predict(1)
        want = bst.predict(data[1][0], raw_score=True)
        assert np.array_equal(got, want)
        l2 = bst.eval_valid()[0][2]
        assert _rel(l2, np.mean((got - data[1][1].astype(np.float32)) ** 2)) <= 1e-12
    assert max(t["num_leaves"] for t in parse_model_string(bst.model_to_string())) > 256 or num_leaves == 31


def _direct_gp_metrics(bst, gp, data, cov_pars, num_neighbors_pred=20):
    """GPModel.predict(y = F - y) plus Booster.predict, restated in numpy"""
    (X, y, coords, _), (Xv, yv, coords_v, _) = data[0], data[1]
    F = bst.inner_predict(0)
    resid = F - y.astype(np.float32).astype(np.float64)
    pred = gp.predict(y=resid, gp_coords_pred=coords_v, cov_pars=cov_pars, predict_var=True, predict_response=True,
                      num_neighbors_pred=num_neighbors_pred)
    p = bst.predict(Xv, raw_score=True) - pred["mu"]
    lab = yv.astype(np.float32).astype(np.float64)
    l2 = np.mean((p - lab) ** 2)
    nll = 0.5 * np.mean((p - lab) ** 2 / pred["var"] + np.log(pred["var"]) + LOG2PI)
    return l2, nll


def _gp_booster(train_cov_pars, metric="l2,test_neg_log_likelihood", seed=5):
    c = dict(name="gp", n=1500, nv=[400], F=4, seed=seed, num_leaves=10, metric=metric, gp="vecchia", use_gp=True)
    data = vc.case_data(c)
    params = vc.params_of(c)
    params["train_gp_model_cov_pars"] = train_cov_pars
    dtrain = Dataset(data[0][0], data[0][1], params=params)
    dvalid = Dataset(data[1][0], data[1][1], params=params, reference=dtrain)
    gp = vc.gp_model_of(c, data)
    bst = Booster(params, dtrain, gp_model=gp)
    bst.add_valid(dvalid, "v")
    return bst, gp, data


@pytest.mark.parametrize("train_cov_pars", [False, True])
def test_gp_metrics_equal_direct_computation(train_cov_pars):
    """fixed parameters: within 1e-8; refitted parameters: the same computation at the fitted parameters within 1e-12"""
    bst, gp, data = _gp_booster(train_cov_pars)
    for _ in range(4):
        bst.update()
        ev = bst.eval_valid()
        ev2 = bst.eval_valid()
        assert [e[2] for e in ev] == [e[2] for e in ev2]  # repeated GetEval: bitwise equal
        cov_pars = gp.get_cov_pars() if train_cov_pars else np.array(vc.COV_PARS)
        l2, nll = _direct_gp_metrics(bst, gp, data, cov_pars)
        tol = 1e-12 if train_cov_pars else 1e-8
        assert _rel(ev[0][2], l2) <= tol, (ev, l2)
        assert _rel(ev[1][2], nll) <= tol, (ev, nll)
        gp.set_prediction_data(gp_coords_pred=data[1][2], num_neighbors_pred=20)  # predict() replaced the saved prediction data


def test_validation_does_not_perturb_training():
    """models and covariance parameters bitwise identical with and without validation data"""
    outs = []
    for with_valid in (False, True):
        c = dict(name="gp", n=1500, nv=[400], F=4, seed=9, num_leaves=10, metric="l2", gp="vecchia", use_gp=True)
        data = vc.case_data(c)
        params = vc.params_of(c)
        params["train_gp_model_cov_pars"] = True
        dtrain = Dataset(data[0][0], data[0][1], params=params)
        gp = vc.gp_model_of(c, data)
        bst = Booster(params, dtrain, gp_model=gp)
        if with_valid:
            bst.add_valid(Dataset(data[1][0], data[1][1], params=params, reference=dtrain), "v")
        for _ in range(5):
            bst.update()
            if with_valid:
                bst.eval_valid()
        outs.append((bst.model_to_string(), gp.get_cov_pars().tobytes()))
    assert outs[0] == outs[1]


def test_early_stopping_matches_reference():
    es = GOLD["early_stopping"]
    got = vc.run_es_case(vc.ES_CASE)
    want = es["frontend"]
    assert got["best_iteration"] == want["best_iteration"]
    assert got["best_iteration"] < vc.ES_CASE["num_boost_round"]
    assert got["num_trees"] == want["num_trees"]
    for m, vals in want["evals_result"]["valid"].items():
        assert len(got["evals_result"]["valid"][m]) == len(vals)
        assert all(_rel(a, b) <= 1e-12 for a, b in zip(got["evals_result"]["valid"][m], vals))
    if "package" in es:
        assert got["best_iteration"] == es["package"]["best_iteration"]
        for m, vals in es["package"]["evals_result"]["valid"].items():
            assert all(_rel(a, b) <= 1e-12 for a, b in zip(got["evals_result"]["valid"][m], vals))


# ---- refusals ---------------------------------------------------------------------------------------------------------------
def _plain(metric="l2", seed=12):
    c = dict(name="r", n=800, nv=[200], F=4, seed=seed, num_leaves=8, metric=metric, gp=None)
    data = vc.case_data(c)
    params = vc.params_of(c)
    dtrain = Dataset(data[0][0], data[0][1], params=params)
    return c, data, params, dtrain


def test_grouped_model_with_gp_validation_is_refused():
    c = dict(GOLD_CASES["grouped_nogpval"], use_gp=True)
    data = vc.case_data(c)
    params = vc.params_of(c)
    dtrain = Dataset(data[0][0], data[0][1], params=params)
    bst = Booster(params, dtrain, gp_model=vc.gp_model_of(c, data))
    with pytest.raises(GPBoostError, match="use_gp_model_for_validation=False"):
        bst.add_valid(Dataset(data[1][0], data[1][1], params=params, reference=dtrain), "v")


def test_dense_model_with_gp_validation_is_refused():
    c, data, params, dtrain = _plain()
    params = dict(params, use_gp_model_for_validation=True, train_gp_model_cov_pars=False)
    gp = GPModel(gp_coords=data[0][2], cov_function="exponential")
    gp.set_optim_params(dict(init_cov_pars=np.array(vc.COV_PARS)))
    bst = Booster(params, dtrain, gp_model=gp)
    with pytest.raises(GPBoostError, match="use_gp_model_for_validation=False"):
        bst.add_valid(Dataset(data[1][0], data[1][1], params=params, reference=dtrain), "v")


def test_unsupported_metric_refused_only_when_evaluated():
    c, data, params, dtrain = _plain(metric="auc")
    bst = Booster(params, dtrain)
    for _ in range(3):
        bst.update()  # a booster with an unsupported metric and no validation data trains
    assert bst.current_iteration() == 3
    assert bst._eval_names() == ["auc"]
    with pytest.raises(GPBoostError, match="Metric 'auc' is not supported"):
        bst.add_valid(Dataset(data[1][0], data[1][1], params=params, reference=dtrain), "v")
    with pytest.raises(GPBoostError, match="Metric 'auc' is not supported"):
        bst.eval_train()


def test_misaligned_dataset_refused():
    c, data, params, dtrain = _plain()
    bst = Booster(params, dtrain)
    own_bins = Dataset(data[1][0], data[1][1], params=params)  # binned on its own: other bin mappers
    with pytest.raises(GPBoostError, match="different bin mappers"):
        bst._safe_call(bst._LIB.LGBM_BoosterAddValidData(bst.handle, own_bins.handle))
    with pytest.raises(GPBoostError, match="number of features"):
        Dataset(data[1][0][:, :3], data[1][1], params=params, reference=dtrain)


def test_missing_prediction_data_refused():
    c = dict(GOLD_CASES["vecchia_l2_gpval"])
    data = vc.case_data(c)
    params = vc.params_of(c)
    dtrain = Dataset(data[0][0], data[0][1], params=params)
    gp = GPModel(gp_coords=data[0][2], cov_function="exponential", gp_approx="vecchia", num_neighbors=10, seed=5)
    gp.set_optim_params(dict(init_cov_pars=np.array(vc.COV_PARS)))
    bst = Booster(params, dtrain, gp_model=gp)
    bst.add_valid(Dataset(data[1][0], data[1][1], params=params, reference=dtrain), "v")
    bst.update()
    with pytest.raises(GPBoostError, match="set_prediction_data"):
        bst.eval_valid()
    dv = Dataset(data[1][0], data[1][1], params=params, reference=dtrain)
    with pytest.raises(ValueError, match="set_prediction_data"):
        train(params, dtrain, num_boost_round=2, valid_sets=[dv], gp_model=gp)


def test_training_metric_with_gp_validation_refused():
    bst, gp, data = _gp_booster(False, metric="l2")
    bst.update()
    with pytest.raises(GPBoostError, match="use_gp_model_for_validation = true"):
        bst.eval_train()
    bst2, _, _ = _gp_booster(False, metric="test_neg_log_likelihood")
    bst2.update()
    with pytest.raises(GPBoostError, match="Cannot use the metric 'test_neg_log_likelihood' on the training data"):
        bst2.eval_train()


def test_train_refuses_two_validation_sets_with_gp():
    bst, gp, data = _gp_booster(False)
    params = vc.params_of(dict(GOLD_CASES["vecchia_l2_gpval"]))
    dtrain = bst.train_set
    dv = [Dataset(data[1][0], data[1][1], params=params, reference=dtrain) for _ in range(2)]
    with pytest.raises(ValueError, match="only one validation set"):
        train(params, dtrain, num_boost_round=2, valid_sets=dv, gp_model=gp)
