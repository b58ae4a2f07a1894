"""Device ensemble prediction (gpbdev_ensemble_predict behind LGBM_BoosterPredictForMat) and Booster.predict with a GP model.
Every device result is compared bitwise with the host walk (GPB200_BoosterPredictForMatHost), with the numpy restatement
(tests/ensemble_walk.py) and, for the reference-trained models, with the reference library's predictions
(tests/golden/ensemble_predict_golden.json): every tile / staging-chunk / shared-memory edge, both element types and layouts, iteration
ranges, one-leaf and chain-shaped trees, ensembles larger than one shared-memory stage and the missing-value rules on special values."""
import ctypes as C
import gc
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ensemble_walk as ew  # noqa: E402
import treedata  # noqa: E402
import validation_cases as vc  # noqa: E402
from gpboost_b200 import GPModel, GPBoostError, train  # noqa: E402
from gpboost_b200.booster import Booster, Dataset, parse_model_string  # noqa: E402
from test_model_text_io import RANGES, missing_cases, text_io_case  # noqa: E402

pytestmark = pytest.mark.gpu

with open(os.path.join(HERE, "golden", "ensemble_predict_golden.json")) as _f:
    GOLD = json.load(_f)

RAW, LEAF = 1, 2
ALL_DECISION_TYPES = (0, 2, 4, 6, 8, 10)  # missing None / Zero / NaN x default right / left
ODD_RANGES = ((-5, 3), (100, 2), (0, 1000), (7, 0), (39, 1))


def _hex(v):
    return np.array([float.fromhex(x) for x in v])


def c_predict(lib, bst, X, ptype=RAW, start=0, num=-1, dtype=np.float64, row_major=True, host=False):
    """LGBM_BoosterPredictForMat (or the host-walk hook) through ctypes: any element type and layout"""
    A = np.ascontiguousarray(X, dtype=dtype) if row_major else np.asfortranarray(X, dtype=dtype)
    nrow, ncol = A.shape
    n = C.c_int64(-1)
    assert lib.LGBM_BoosterCalcNumPredict(bst.handle, C.c_int(nrow), C.c_int(ptype), C.c_int(start), C.c_int(num), C.byref(n)) == 0
    out = np.full(n.value, np.nan)
    fn = lib.GPB200_BoosterPredictForMatHost if host else lib.LGBM_BoosterPredictForMat
    got = C.c_int64(-1)
    rc = fn(bst.handle, A.ctypes.data_as(C.c_void_p), C.c_int(0 if dtype == np.float32 else 1), C.c_int32(nrow), C.c_int32(ncol),
            C.c_int(1 if row_major else 0), C.c_int(ptype), C.c_int(start), C.c_int(num), b"", C.byref(got), out.ctypes.data_as(C.POINTER(C.c_double)))
    assert rc == 0, lib.LGBM_GetLastError().decode()
    assert got.value == n.value
    return out


def plan(lib, bst, ncol, dtype=np.float64, ptype=RAW, start=0, num=-1):
    """(tile rows, staging-chunk rows, features in shared memory, tree stages)"""
    out = (C.c_int64 * 4)()
    assert lib.GPB200_BoosterPredictPlan(bst.handle, C.c_int(0 if dtype == np.float32 else 1), C.c_int32(ncol), C.c_int(ptype), C.c_int(start),
                                         C.c_int(num), out) == 0, lib.LGBM_GetLastError().decode()
    return tuple(int(v) for v in out)


def features(rng, nrow, ncol):
    X = rng.standard_normal((nrow, ncol))
    X[rng.random(X.shape) < 0.05] = np.nan
    X[rng.random(X.shape) < 0.05] = 0.
    return X


def synthetic(seed, ncol, num_trees, num_leaves, decision_types=ALL_DECISION_TYPES):
    rng = np.random.default_rng(seed)
    return ew.model_text(ncol, [ew.random_tree(rng, k, ncol, num_leaves, decision_types) for k in range(num_trees)])


def check_all(lib, bst, trees, X, dtype=np.float64, row_major=True, start=0, num=-1, leaf=True, walk=True):
    with np.errstate(over="ignore"):  # 1e300 -> inf in float32
        Xd = np.asarray(X, dtype=dtype)
    got = c_predict(lib, bst, Xd, RAW, start, num, dtype, row_major)
    assert np.array_equal(got, c_predict(lib, bst, Xd, RAW, start, num, dtype, row_major, host=True))
    if walk:
        assert np.array_equal(got, ew.predict(trees, Xd, start, num))
    if leaf:
        gl = c_predict(lib, bst, Xd, LEAF, start, num, dtype, row_major)
        assert np.array_equal(gl, c_predict(lib, bst, Xd, LEAF, start, num, dtype, row_major, host=True))
        if walk:
            want = ew.predict(trees, Xd, start, num, pred_leaf=True)
            assert np.array_equal(gl.reshape(want.shape), want)
    return got


@pytest.fixture(scope="module")
def lib(product_lib):
    assert product_lib.gpbdev_device_count() > 0
    return product_lib


@pytest.fixture(scope="module")
def ens50(lib):
    text = synthetic(1, 50, 40, 31)
    return Booster(model_str=text, _lib=lib), parse_model_string(text)


def test_reference_models_match_the_reference_bitwise(lib, ref_golden):
    models = [("text_io", ref_golden["text_io"]["model"], text_io_case()[2])]
    for i, ((_, _, Xt, _), rec) in enumerate(zip(missing_cases(), ref_golden["missing"])):
        models.append(("missing_%d" % i, rec["model"], Xt))
    for (name, text, Xt), rec in zip(models, GOLD["leaf"]):
        b = Booster(model_str=text, _lib=lib)
        trees = parse_model_string(text)
        for r in rec["ranges"]:
            st, nit = r["start"], r["num"]
            got = check_all(lib, b, trees, Xt, start=st, num=nit)
            assert ew.digest(got, np.float64) == r["raw_sha256"], (name, st, nit)
            leaf = b.predict(Xt, start_iteration=st, num_iteration=nit, pred_leaf=True)
            assert leaf.dtype == np.int32 and list(leaf.shape) == r["shape"] and ew.digest(leaf, np.int32) == r["leaf_sha256"], (name, st, nit)


def test_row_counts_around_every_tile_and_chunk_edge(lib, ens50):
    bst, trees = ens50
    tile, chunk, in_smem, stages = plan(lib, bst, 50)
    assert tile in (32, 64, 128, 256) and in_smem == 1 and stages == 1 and chunk > 4 * tile
    rng = np.random.default_rng(2)
    small = sorted({1, 31, 32, 33, tile - 1, tile, tile + 1})
    for nrow in small:
        X = features(rng, nrow, 50)
        for dtype in (np.float64, np.float32):
            for row_major in (True, False):
                check_all(lib, bst, trees, X, dtype, row_major)
    for nrow in (chunk - 1, chunk, chunk + 1, 3 * chunk + 5):
        X = features(rng, nrow, 50)
        for row_major in (True, False):
            check_all(lib, bst, trees, X, np.float64, row_major, leaf=row_major, walk=False)
        assert np.array_equal(c_predict(lib, bst, X[:2000]), ew.predict(trees, X[:2000]))
    chunk32 = plan(lib, bst, 50, np.float32)[1]  # float32 chunks hold twice the rows
    assert chunk32 == 2 * chunk
    for nrow, layouts in ((chunk32 - 1, (True,)), (chunk32 + 1, (True, False)), (3 * chunk32 + 5, (True,))):
        X = features(rng, nrow, 50).astype(np.float32)
        for row_major in layouts:
            check_all(lib, bst, trees, X, np.float32, row_major, leaf=False, walk=False)
    # leaf indices have their own chunk length (the output is the larger side): one more than it
    lchunk = plan(lib, bst, 50, ptype=LEAF)[1]
    if lchunk + 1 != chunk + 1:
        check_all(lib, bst, trees, features(rng, lchunk + 1, 50), walk=False)


def test_column_counts_around_the_widest_tile(lib):
    rng = np.random.default_rng(3)
    # the plan depends on the ensemble's size only, which is the same for every ncol below
    probe = Booster(model_str=synthetic(4, 1, 10, 15), _lib=lib)
    assert plan(lib, probe, 1)[2] == 1
    widest = max(ncol for ncol in range(1, 3000) if plan(lib, probe, ncol)[2] == 1)
    assert 300 <= widest < 2998 and plan(lib, probe, widest)[0] == 32
    for ncol in (1, 50, widest, widest + 1, 2 * widest):
        text = synthetic(5, ncol, 10, 15)
        b, trees = Booster(model_str=text, _lib=lib), parse_model_string(text)
        tile, _, in_smem, _ = plan(lib, b, ncol)
        assert in_smem == (1 if ncol <= widest else 0)
        X = features(rng, 3 * 256 + 7, ncol)
        for dtype in (np.float64, np.float32):
            for row_major in (True, False):
                check_all(lib, b, trees, X, dtype, row_major)


def test_iteration_ranges(lib, ens50):
    bst, trees = ens50
    X = features(np.random.default_rng(6), 777, 50)
    for st, nit in RANGES + ODD_RANGES:
        check_all(lib, bst, trees, X, start=st, num=nit)
        first, count = ew.iteration_range(40, st, nit)
        assert c_predict(lib, bst, X, LEAF, st, nit).shape[0] == 777 * count
    assert np.array_equal(c_predict(lib, bst, X, RAW, 40, -1), np.zeros(777))  # an empty range: the empty sum


def test_one_leaf_trees_in_the_middle(lib):
    rng = np.random.default_rng(7)
    sizes = [31, 1, 1, 8, 1, 2, 31, 1]
    text = ew.model_text(6, [ew.random_tree(rng, k, 6, nl, ALL_DECISION_TYPES) for k, nl in enumerate(sizes)])
    b, trees = Booster(model_str=text, _lib=lib), parse_model_string(text)
    X = features(rng, 1000, 6)
    for st, nit in ((0, -1), (1, 2), (1, 1), (4, 4), (7, 1)):
        check_all(lib, b, trees, X, start=st, num=nit)


def test_ensemble_larger_than_one_shared_memory_stage(lib):
    rng = np.random.default_rng(8)
    ncol, num_trees = 20, 400
    tt = []
    for k in range(num_trees):
        if k in (0, 57, 399):
            tt.append(ew.chain_tree(rng, k, ncol, 255, ALL_DECISION_TYPES))
        else:
            tt.append(ew.random_tree(rng, k, ncol, 255 if k % 3 else int(rng.integers(2, 255)), ALL_DECISION_TYPES))
    text = ew.model_text(ncol, tt)
    b, trees = Booster(model_str=text, _lib=lib), parse_model_string(text)
    assert plan(lib, b, ncol)[3] > 4  # several stages
    X = features(rng, 3000, ncol)
    X[:, :] = np.where(np.isnan(X), np.nan, X * 1.5)
    for st, nit in ((0, -1), (3, 200), (57, 1), (390, -1)):
        check_all(lib, b, trees, X, start=st, num=nit)
    check_all(lib, b, trees, X[:300], np.float32, False)
    # the depth-254 chain is walked to its end
    leaf = b.predict(X, start_iteration=57, num_iteration=1, pred_leaf=True)
    assert leaf.max() == 254 and leaf.min() == 0


def test_special_values_against_every_missing_type(lib):
    rng = np.random.default_rng(9)
    special = np.array([np.nan, 0., -0., 1e-36, -1e-36, 1e-35, -1e-35, 2e-35, -2e-35, np.inf, -np.inf, 0.5, -0.5, 1e300, -1e300])
    thresholds = np.array([0., -0., 1e-36, -1e-36, 1e-35, -1e-35, 1., -1., 1e300, -1e300])
    ncol = 4
    X = special[rng.integers(0, len(special), size=(5000, ncol))]
    X[:len(special), 0] = special
    for dts in ((0,), (2,), (4,), (6,), (8,), (10,), ALL_DECISION_TYPES):
        text = ew.model_text(ncol, [ew.random_tree(rng, k, ncol, 31, dts, thresholds) for k in range(12)])
        b, trees = Booster(model_str=text, _lib=lib), parse_model_string(text)
        check_all(lib, b, trees, X)
        check_all(lib, b, trees, X, np.float32, False)  # 1e-36, 1e300 round to 0 / inf in float32 before the walk


def test_training_booster_predicts_on_the_device_and_sees_new_trees(lib):
    spec = dict(n=20000, F=10, kind="real", num_leaves=31, min_data_in_leaf=20, seed=5)
    X, y, _ = treedata.make_case(spec)
    params = treedata.booster_params(spec, reference=False)
    b = Booster(params, Dataset(X, y, params=params))
    for _ in range(5):
        b.update()
    score = b.inner_predict_train()
    p5 = b.predict(X)
    assert np.abs(p5 - score).max() <= 1e-12 * np.abs(score).max()
    assert np.array_equal(p5, c_predict(lib, b, X, host=True))
    b.update()  # one more tree: the packed ensemble is rebuilt
    score6 = b.inner_predict_train()
    p6 = b.predict(X)
    assert not np.array_equal(p6, p5)
    assert np.abs(p6 - score6).max() <= 1e-12 * np.abs(score6).max()
    assert np.array_equal(p6, c_predict(lib, b, X, host=True))
    assert b.predict(X, pred_leaf=True).shape == (20000, 6)
    assert np.array_equal(b.predict(X, num_iteration=5), p5)


# ---- Booster.predict with a GP model ----------------------------------------------------------------------------------------------
def _gp_case(c):
    X, y, coords = treedata.make_case(c)
    Xt, _, coords_t = treedata.make_case(dict(c, n=c["n_test"], seed=c["seed"] + 100))
    gp = GPModel(gp_coords=coords, cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia", num_neighbors=c["num_neighbors"],
                 vecchia_ordering="random", seed=c["seed"])
    return X, y, coords, Xt, coords_t, gp


def _check_dict(got, want, tol):
    assert set(got) == {"fixed_effect", "random_effect_mean", "random_effect_cov", "response_mean", "response_var"}
    for k, w in want.items():
        if w is None:
            assert got[k] is None, k
        else:
            w = _hex(w)
            assert got[k] is not None and got[k].shape == w.shape, k
            assert np.abs(got[k] - w).max() <= tol * np.abs(w).max(), (k, np.abs(got[k] - w).max(), np.abs(w).max())


@pytest.mark.parametrize("case", GOLD["gpboost"], ids=lambda c: c["name"])
def test_gpboost_prediction_of_the_reference_model_matches_the_reference(case):
    """the reference's trees (model text) and covariance parameters: fixed effects bitwise, the GP part within the prediction tolerance"""
    X, y, coords, Xt, coords_t, gp = _gp_case(case)
    params = treedata.booster_params(case, reference=False)
    dtrain = Dataset(X, y, params=params, free_raw_data=False)
    bst = Booster(model_str=case["model"], train_set=dtrain, gp_model=gp)
    cov_pars = _hex(case["cov_pars"])
    for latent in (False, True):
        got = bst.predict(Xt, gp_coords_pred=coords_t, predict_var=True, pred_latent=latent, cov_pars=cov_pars)
        _check_dict(got, case["pred_latent_%s" % latent], 1e-8)
    assert np.array_equal(got["fixed_effect"], _hex(case["pred_latent_True"]["fixed_effect"]))
    no_var = bst.predict(Xt, gp_coords_pred=coords_t, pred_latent=True, cov_pars=cov_pars)
    assert no_var["random_effect_cov"] is None and np.array_equal(no_var["random_effect_mean"], got["random_effect_mean"])
    off = np.linspace(-1., 1., Xt.shape[0])
    with_off = bst.predict(Xt, gp_coords_pred=coords_t, pred_latent=False, cov_pars=cov_pars, offset_pred=off)
    assert np.allclose(with_off["response_mean"], got["fixed_effect"] + got["random_effect_mean"] + off, rtol=1e-13, atol=1e-13)
    # ignore_gp_model, or the explicit raw_score of earlier versions: the tree ensemble alone
    assert np.array_equal(bst.predict(Xt, ignore_gp_model=True), got["fixed_effect"])
    assert np.array_equal(bst.predict(Xt, raw_score=True), got["fixed_effect"])


def test_gpboost_trained_here_at_fixed_parameters_matches_the_reference():
    case = GOLD["gpboost"][0]
    assert case["name"] == "fixed_cov_pars"
    X, y, coords, Xt, coords_t, gp = _gp_case(case)
    gp.set_optim_params(dict(init_cov_pars=np.array(case["init_cov_pars"])))
    params = treedata.booster_params(case, reference=False)
    dtrain = Dataset(X, y, params=params, free_raw_data=False)
    bst = train(params, dtrain, num_boost_round=case["num_boost_round"], gp_model=gp, train_gp_model_cov_pars=False)
    assert bst.current_iteration() == case["num_boost_round"]
    for latent in (False, True):
        got = bst.predict(Xt, gp_coords_pred=coords_t, predict_var=True, pred_latent=latent, cov_pars=np.array(case["init_cov_pars"]))
        _check_dict(got, case["pred_latent_%s" % latent], 1e-8)


def test_num_iteration_none_uses_best_iteration():
    c = vc.ES_CASE
    data = vc.case_data(c)
    params = vc.params_of(c)
    dtrain = Dataset(data[0][0], data[0][1], params=params)
    dvalid = Dataset(data[1][0], data[1][1], params=params, reference=dtrain)
    bst = train(params, dtrain, num_boost_round=c["num_boost_round"], valid_sets=[dvalid], valid_names=["valid"],
                early_stopping_rounds=c["early_stopping_rounds"])
    assert 0 < bst.best_iteration < bst.current_iteration()
    Xv = data[1][0]
    best = bst.predict(Xv)
    assert np.array_equal(best, bst.predict(Xv, num_iteration=bst.best_iteration))
    assert not np.array_equal(best, bst.predict(Xv, num_iteration=-1))
    assert np.array_equal(bst.predict(Xv, start_iteration=2), bst.predict(Xv, start_iteration=2, num_iteration=-1))


def test_gpboost_prediction_error_cases(lib):
    case = GOLD["gpboost"][0]
    X, y, coords, Xt, coords_t, gp = _gp_case(case)
    params = treedata.booster_params(case, reference=False)
    cov_pars = _hex(case["cov_pars"])
    freed = Booster(model_str=case["model"], train_set=Dataset(X, y, params=params), gp_model=gp)
    with pytest.raises(GPBoostError, match="Set free_raw_data = False when you construct the Dataset"):
        freed.predict(Xt, gp_coords_pred=coords_t, cov_pars=cov_pars)
    dtrain = Dataset(X, y, params=params, free_raw_data=False)
    assert dtrain.data is not None and Dataset(X, y, params=params).data is None
    bst = Booster(model_str=case["model"], train_set=dtrain, gp_model=gp)
    for kw in (dict(pred_contrib=True), dict(predict_cov_mat=True), dict(sample_posterior=True)):
        with pytest.raises(GPBoostError, match="not supported by this build"):
            bst.predict(Xt, gp_coords_pred=coords_t, cov_pars=cov_pars, **kw)
    with pytest.raises(GPBoostError, match="gp_coords_pred"):
        bst.predict(Xt, cov_pars=cov_pars)
    counts = GPModel(likelihood="poisson", gp_coords=coords, cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia",
                     num_neighbors=10, vecchia_ordering="random", seed=1)
    with pytest.raises(GPBoostError, match="only supported for the gaussian likelihood"):
        Booster(model_str=case["model"], train_set=dtrain, gp_model=counts).predict(Xt, gp_coords_pred=coords_t)
    n = C.c_int64(0)
    out = np.zeros(Xt.shape[0] * (Xt.shape[1] + 1))
    A = np.ascontiguousarray(Xt)
    assert lib.LGBM_BoosterPredictForMat(bst.handle, A.ctypes.data_as(C.c_void_p), 1, C.c_int32(A.shape[0]), C.c_int32(A.shape[1]), 1, 3, 0, -1, b"",
                                         C.byref(n), out.ctypes.data_as(C.POINTER(C.c_double))) != 0
    assert "not supported by this build" in lib.LGBM_GetLastError().decode()
    with pytest.raises(GPBoostError, match="number of features"):
        bst.predict(Xt[:, :3], ignore_gp_model=True)


def test_repeated_predictions_are_bitwise_equal_and_allocate_nothing(lib, ens50):
    """The staging buffers are allocated by the first prediction of a shape and reused: free device memory does not move over 50 more
    predictions, and freeing the booster returns it. Free memory is device-wide (the driver's lazily created state and other
    processes move it by some MB; in a process of its own the three readings are exactly equal), so the bound is a fraction of ONE staging
    buffer of this shape (64 MiB): a buffer leaked per call would show 50 times that."""
    import torch
    slack = 32 << 20
    _, trees = ens50
    text = synthetic(1, 50, 40, 31)
    X = features(np.random.default_rng(10), 200000, 50)  # two staging chunks
    warm = Booster(model_str=text, _lib=lib)
    warm.predict(X[:1000])
    del warm
    gc.collect()
    torch.cuda.synchronize()
    free_before = torch.cuda.mem_get_info()[0]
    b = Booster(model_str=text, _lib=lib)
    first = b.predict(X)
    free_first = torch.cuda.mem_get_info()[0]
    assert free_before - free_first >= 2 * 64 << 20  # two input buffers of 64 MiB and the two small output buffers
    for _ in range(50):
        assert np.array_equal(b.predict(X), first)
    assert abs(torch.cuda.mem_get_info()[0] - free_first) <= slack
    assert np.array_equal(first[:3000], ew.predict(trees, X[:3000]))
    del b
    gc.collect()
    assert abs(torch.cuda.mem_get_info()[0] - free_before) <= slack
