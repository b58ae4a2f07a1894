"""GPU parity tests of the device tree learner and the boosting driver (run with -m gpu). Through the C ABI only.
Split features, threshold bins, tree topology and leaf counts: bit-exact. Leaf values / scores: <= 1e-10 relative (the device
merges chunk partial sums, the reference adds row by row)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import treedata
from oracle import tree as ot

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class DevCfg(C.Structure):
    _fields_ = [("num_leaves", C.c_int), ("min_data_in_leaf", C.c_int), ("min_sum_hessian_in_leaf", C.c_double),
                ("lambda_l2", C.c_double), ("min_gain_to_split", C.c_double), ("max_depth", C.c_int)]


@pytest.fixture(scope="module")
def lib(product_lib):
    assert product_lib.gpbdev_device_count() > 0
    product_lib.gpbdev_tree_last_error.restype = C.c_char_p
    return product_lib


@pytest.fixture(scope="module")
def tree_golden():
    with open(os.path.join(ROOT, "tests", "golden", "tree_golden.json")) as f:
        return json.load(f)


def P(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def dev_train(lib, bins_fm, num_bin, grad, cfg, on_device=False):
    """on_device: the gradient goes through a device buffer (the only way into the graph-replayed leaf loop)"""
    F, n = bins_fm.shape
    h = C.c_void_p()
    dc = DevCfg(cfg.num_leaves, cfg.min_data_in_leaf, cfg.min_sum_hessian_in_leaf, cfg.lambda_l2, cfg.min_gain_to_split, cfg.max_depth)
    nb = np.ascontiguousarray(num_bin, dtype=np.int32)
    rc = lib.gpbdev_tree_create(C.byref(h), 0, C.c_int64(n), F, P(np.ascontiguousarray(bins_fm), C.c_uint8), P(nb, C.c_int32), C.byref(dc))
    assert rc == 0, lib.gpbdev_tree_last_error().decode()
    L = cfg.num_leaves
    nl = C.c_int(0)
    sf = np.zeros(L, np.int32); tb = np.zeros(L, np.int32); lc = np.zeros(L, np.int32); rcd = np.zeros(L, np.int32)
    sg = np.zeros(L, np.float32); lv = np.zeros(L, np.float64); cnt = np.zeros(L, np.int32)
    g = np.ascontiguousarray(grad, dtype=np.float64)
    gp = P(g, C.c_double)
    if on_device:
        gp = C.c_void_p()
        assert lib.gpbdev_vec_alloc(h, C.byref(gp), C.c_int64(n)) == 0
        assert lib.gpbdev_vec_upload(h, gp, P(g, C.c_double), C.c_int64(n)) == 0
    rc = lib.gpbdev_tree_train(h, gp, 1 if on_device else 0, C.c_double(1.0), C.byref(nl), P(sf, C.c_int), P(tb, C.c_int), P(lc, C.c_int), P(rcd, C.c_int),
                               P(sg, C.c_float), P(lv, C.c_double), P(cnt, C.c_int))
    if on_device:
        lib.gpbdev_vec_free(h, gp)
    assert rc == 0, lib.gpbdev_tree_last_error().decode()
    k = nl.value
    lib.gpbdev_tree_free(h)
    return {"num_leaves": k, "split_feature": sf[:k - 1], "threshold_bin": tb[:k - 1], "left_child": lc[:k - 1], "right_child": rcd[:k - 1],
            "split_gain": sg[:k - 1], "leaf_value": lv[:k], "leaf_count": cnt[:k]}


@pytest.mark.parametrize("n,F,levels,L,mdl", [(4000, 5, 30, 8, 20), (30000, 40, 255, 31, 20), (10000, 70, 16, 63, 3), (500, 3, 5, 31, 1), (50, 2, 4, 4, 30)])
def test_device_tree_matches_oracle(lib, n, F, levels, L, mdl):
    rng = np.random.default_rng(n + F)
    bins = rng.integers(0, levels, size=(F, n)).astype(np.uint8)
    grad = rng.standard_normal(n) + (bins[0] > levels // 2) * 0.8 - (bins[min(1, F - 1)] % 3 == 0) * 0.5
    cfg = ot.make_config(num_leaves=L, min_data_in_leaf=mdl)
    a = ot.train_tree(bins, np.full(F, levels), grad, cfg)
    d = dev_train(lib, bins, np.full(F, levels), grad, cfg)
    assert d["num_leaves"] == a["num_leaves"]
    for k in ("split_feature", "threshold_bin", "left_child", "right_child", "leaf_count"):
        assert np.array_equal(d[k], a[k]), k
    if a["num_leaves"] > 1:
        assert np.max(np.abs(d["leaf_value"] - a["leaf_value"])) <= 1e-10 * np.max(np.abs(a["leaf_value"]))
        assert np.allclose(d["split_gain"], a["split_gain"], rtol=1e-5)


# the two ways the leaf loop is enqueued on one GPU: a replayed graph (device gradients) and eagerly (host gradients); the Booster
# always passes device gradients (test_booster_matches_reference_golden)
VARIANTS = {"graph": True, "eager": False}
VARIANT_CASES = [(30000, 40, 255, 31, 20), (10000, 70, 16, 63, 3), (500, 3, 5, 31, 1), (20000, 9, 2, 16, 50), (50, 2, 4, 4, 30)]


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("n,F,levels,L,mdl", VARIANT_CASES)
def test_tree_kernel_variants_match_oracle(lib, variant, n, F, levels, L, mdl):
    """Same parity bar on both ways of enqueuing the leaf loop: oracle trees (incl. binary and constant-heavy features, F > 64, a
    leaf budget the data cannot fill) through gpbdev_tree_train. tests/test_tree_kernels_gpu.py covers every path."""
    rng = np.random.default_rng(n + F)
    bins = rng.integers(0, levels, size=(F, n)).astype(np.uint8)
    grad = rng.standard_normal(n) + (bins[0] > levels // 2) * 0.8 - (bins[min(1, F - 1)] % 3 == 0) * 0.5
    cfg = ot.make_config(num_leaves=L, min_data_in_leaf=mdl)
    a = ot.train_tree(bins, np.full(F, levels), grad, cfg)
    d = dev_train(lib, bins, np.full(F, levels), grad, cfg, on_device=VARIANTS[variant])
    assert d["num_leaves"] == a["num_leaves"], (variant, n, F)
    for k in ("split_feature", "threshold_bin", "left_child", "right_child", "leaf_count"):
        assert np.array_equal(d[k], a[k]), (variant, n, F, k)
    if a["num_leaves"] > 1:
        assert np.max(np.abs(d["leaf_value"] - a["leaf_value"])) <= 1e-10 * np.max(np.abs(a["leaf_value"])), (variant, n, F)


def _run_product(spec):
    from gpboost_b200 import GPModel
    from gpboost_b200.booster import Booster, Dataset, parse_model_string
    X, y, coords = treedata.make_case(spec)
    params = treedata.booster_params(spec, reference=False)
    ds = Dataset(X, y, params=params)
    gp = None
    if coords is not None:
        gp = GPModel(gp_coords=coords, cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia", num_neighbors=spec["num_neighbors"],
                     vecchia_ordering="random", seed=1)
        if spec.get("init_cov_pars"):
            gp.set_optim_params({"init_cov_pars": np.array(spec["init_cov_pars"])})
    b = Booster(params, ds, gp_model=gp)
    for _ in range(spec["num_iter"]):
        b.update()
    return parse_model_string(b.model_to_string()), b.inner_predict_train(), gp, b, X


def test_booster_matches_reference_golden(lib, tree_golden):
    """LGBM_DatasetCreateFromMat -> LGBM_BoosterCreate -> LGBM_BoosterUpdateOneIter against the reference's trees:
    integer and real-valued features (bin finding incl. the sampled path for n > 200000, zeros, negative values, a constant column)."""
    for rec in tree_golden["cases"]:
        spec = rec["spec"]
        if spec.get("gp"):
            continue
        trees, score, _, b, X = _run_product(spec)
        assert len(trees) == len(rec["trees"]), spec["name"]
        for t, g in zip(trees, rec["trees"]):
            assert t["num_leaves"] == g["num_leaves"], spec["name"]
            assert np.array_equal(t["split_feature"], np.array(g["split_feature"])), spec["name"]
            assert np.array_equal(t["threshold"], np.array(g["threshold"])), spec["name"]  # same bin upper bounds, bit for bit
            assert np.array_equal(t["left_child"], np.array(g["left_child"])) and np.array_equal(t["right_child"], np.array(g["right_child"]))
            assert np.array_equal(t["leaf_count"], np.array(g["leaf_count"]))
            assert np.max(np.abs(t["leaf_value"] - np.array(g["leaf_value"]))) <= 1e-10 * np.max(np.abs(g["leaf_value"]))
        assert np.abs(score[:64] - np.array(rec["score_head"])).max() <= 1e-10 * np.abs(rec["score_head"]).max()
        assert abs(score.sum() - rec["score_sum"]) <= 1e-9 * abs(rec["score_sum"])
        # host traversal of the stored model reproduces the device-maintained training score
        assert np.abs(b.predict(X[:2000]) - score[:2000]).max() <= 1e-12 * np.abs(score).max()


def test_gpboost_iteration_matches_reference_golden(lib, tree_golden):
    """GPBoost algorithm (LGBM_GPBoosterCreate): every iteration re-fits the covariance parameters (L-BFGS on the device
    likelihood) and boosts on Psi^-1 (F - y). The optimiser path is decision dependent, so trees are compared on structure
    of the FIRST tree (same init parameters) and the final state within optimiser tolerance."""
    rec = [r for r in tree_golden["cases"] if r["spec"]["name"] == "gpboost_vecchia"][0]
    trees, score, gp, _, _ = _run_product(rec["spec"])
    g0 = rec["trees"][0]
    assert np.array_equal(trees[0]["split_feature"], np.array(g0["split_feature"]))
    assert np.array_equal(trees[0]["threshold"], np.array(g0["threshold"]))
    assert np.max(np.abs(trees[0]["leaf_value"] - np.array(g0["leaf_value"]))) <= 1e-4 * np.max(np.abs(g0["leaf_value"]))
    cp = gp.get_cov_pars()
    assert np.all(np.abs(cp - np.array(rec["cov_pars"])) <= 5e-3 * np.abs(rec["cov_pars"])), (cp, rec["cov_pars"])
    assert np.abs(score[:64] - np.array(rec["score_head"])).max() <= 2e-3 * np.abs(rec["score_head"]).max()


@pytest.mark.parametrize("name", ["gpboost_vecchia_line_search", "gpboost_vecchia_newton_line_search"])
def test_gpboost_line_search_step_length_matches_reference_golden(lib, tree_golden, name):
    """line_search_step_length (SURVEY §8 f2, gbdt.cpp:480-492, re_model_template.h:1163-1181): every tree is scaled by
    -(F - y)' Psi^-1 f / f' Psi^-1 f before the learning rate, two inner products against the device-resident factor. The reference only
    supports it with trained covariance parameters (it reads F - y from its last OptimCovPar call), so the comparison carries the
    optimiser tolerance of test_gpboost_iteration_matches_reference_golden: first tree's structure bit-exact, its values (which contain
    the first step length) to 1e-3, the later step lengths (the stored shrinkage) to 2 %. After a Newton leaf update the step is 1."""
    rec = [r for r in tree_golden["cases"] if r["spec"]["name"] == name][0]
    trees, score, gp, _, _ = _run_product(rec["spec"])
    assert len(trees) == len(rec["trees"])
    g0 = rec["trees"][0]
    assert np.array_equal(trees[0]["split_feature"], np.array(g0["split_feature"])) and np.array_equal(trees[0]["threshold"], np.array(g0["threshold"]))
    assert np.array_equal(trees[0]["leaf_count"], np.array(g0["leaf_count"]))
    assert np.max(np.abs(trees[0]["leaf_value"] - np.array(g0["leaf_value"]))) <= 1e-3 * np.max(np.abs(g0["leaf_value"]))
    for t, g in zip(trees[1:], rec["trees"][1:]):
        assert abs(t["shrinkage"] - g["shrinkage"]) <= 2e-2 * abs(g["shrinkage"]), (t["shrinkage"], g["shrinkage"])
    if rec["spec"].get("newton"):
        assert all(abs(t["shrinkage"] - 0.1) <= 1e-6 for t in trees[1:])
    else:
        assert all(abs(t["shrinkage"] - 0.1) > 1e-3 for t in trees[1:])  # the step length is not a no-op
    cp = gp.get_cov_pars()
    assert np.all(np.abs(cp - np.array(rec["cov_pars"])) <= 1e-2 * np.abs(rec["cov_pars"])), (cp, rec["cov_pars"])
    assert np.abs(score[:64] - np.array(rec["score_head"])).max() <= 5e-3 * np.abs(rec["score_head"]).max()


@pytest.mark.parametrize("name", ["gpboost_vecchia_fixed_pars", "gpboost_vecchia_newton", "gpboost_vecchia_newton_many_leaves"])
def test_gpboost_fixed_parameters_all_trees_match_reference(lib, tree_golden, name):
    """GPBoost iterations at fixed covariance parameters (train_gp_model_cov_pars = false): gradient Psi^-1 (F - y) / sigma^2 from the
    device factor, trees on it, optionally Newton leaf values (H^T Psi^-1 H)^-1 H^T Psi^-1 (y - F) (leaves_newton_update, SURVEY §8 f2).
    Nothing is decided by an optimiser, so EVERY tree is compared: split features / thresholds / counts bit-exact, leaf values and the
    training scores to 1e-8 — the reference's own GPU-vs-CPU bar (SURVEY §4)."""
    rec = [r for r in tree_golden["cases"] if r["spec"]["name"] == name][0]
    trees, score, gp, _, _ = _run_product(rec["spec"])
    assert len(trees) == len(rec["trees"])
    for t, g in zip(trees, rec["trees"]):
        assert t["num_leaves"] == g["num_leaves"]
        assert np.array_equal(t["split_feature"], np.array(g["split_feature"])) and np.array_equal(t["threshold"], np.array(g["threshold"]))
        assert np.array_equal(t["left_child"], np.array(g["left_child"])) and np.array_equal(t["right_child"], np.array(g["right_child"]))
        assert np.array_equal(t["leaf_count"], np.array(g["leaf_count"]))
        assert np.max(np.abs(t["leaf_value"] - np.array(g["leaf_value"]))) <= 1e-8 * np.max(np.abs(g["leaf_value"]))
    assert np.abs(score[:64] - np.array(rec["score_head"])).max() <= 1e-8 * np.abs(rec["score_head"]).max()
    assert abs(score.sum() - rec["score_sum"]) <= 1e-8 * max(abs(rec["score_sum"]), np.abs(score).sum() * 1e-3)
    assert np.allclose(gp.get_cov_pars(), rec["spec"]["init_cov_pars"], rtol=1e-12)


def test_full_size_histogram_properties(lib):
    """n = 1e6 x 50 features x 255 bins (BASELINE config 3 shape): a 2-leaf tree's counts and sums are checked against
    numpy reductions of the same bins (size-independent properties: count conservation, exact child counts, leaf outputs)."""
    n, F, levels = 1000000, 50, 255
    rng = np.random.default_rng(1)
    bins = rng.integers(0, levels, size=(F, n), dtype=np.uint8)
    grad = rng.standard_normal(n) + (bins[7] > 100) * 0.5
    cfg = ot.make_config(num_leaves=2, min_data_in_leaf=20)
    d = dev_train(lib, bins, np.full(F, levels), grad, cfg)
    assert d["num_leaves"] == 2 and d["split_feature"][0] == 7 and d["threshold_bin"][0] == 100
    left = bins[7] <= 100
    assert d["leaf_count"][0] == left.sum() and d["leaf_count"][1] == n - left.sum()
    assert abs(d["leaf_value"][0] + grad[left].sum() / left.sum()) <= 1e-9
    assert abs(d["leaf_value"][1] + grad[~left].sum() / (~left).sum()) <= 1e-9
