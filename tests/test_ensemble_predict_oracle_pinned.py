"""Pins the prediction goldens (tests/golden/ensemble_predict_golden.json, tests/golden/make_ensemble_predict_golden.py) and the numpy
restatement of the ensemble walk (tests/ensemble_walk.py) to the reference library: the golden file regenerates where the reference
is built (tree walks identically, the GPBoost cases within training tolerance); the numpy walk reproduces the reference's raw scores
and leaf indices bitwise; and a booster loaded from a model string predicts leaf indices equal to the golden through
LGBM_BoosterPredictForMat (the host walk where there is no CUDA device),
with LGBM_BoosterCalcNumPredict returning the length that call writes. The device kernel is checked against the same goldens in
tests/test_ensemble_predict_gpu.py."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import dropin  # noqa: E402
import ensemble_walk as ew  # noqa: E402
from gpboost_b200.booster import Booster, parse_model_string  # noqa: E402
from test_model_text_io import RANGES, missing_cases, text_io_case  # noqa: E402

with open(os.path.join(HERE, "golden", "ensemble_predict_golden.json")) as _f:
    GOLD = json.load(_f)


def _hex(v):
    return np.array([float.fromhex(x) for x in v])


def leaf_models(ref_golden):
    """(name, model text, prediction inputs) in the order of GOLD["leaf"]"""
    out = [("text_io", ref_golden["text_io"]["model"], text_io_case()[2])]
    for i, ((_, _, Xt, _), rec) in enumerate(zip(missing_cases(), ref_golden["missing"])):
        out.append(("missing_%d" % i, rec["model"], Xt))
    return out


def test_golden_regenerates(ref_lib):
    """The tree walks of the stored models are pure functions of the model text: identical. The GPBoost cases train with the reference
    (threaded sums, and for the second case its optimiser), so another CPU may move last bits: same shape and None pattern, values
    within 1e-6 at fixed covariance parameters and within the fit tolerance where they are fitted."""
    if ref_lib is None:
        pytest.skip("reference library not built")
    import make_ensemble_predict_golden as gen
    assert gen.leaf_records(ref_lib) == GOLD["leaf"]
    if dropin.ref_package_dir() is None:
        pytest.skip("reference Python package not present")
    for got, want in zip(gen.gp_records(), GOLD["gpboost"]):
        tol = 1e-6 if want.get("train_cov") is False else 5e-3
        assert got["name"] == want["name"] and got["model"].count("Tree=") == want["model"].count("Tree=") == want["num_boost_round"]
        np.testing.assert_allclose(_hex(got["cov_pars"]), _hex(want["cov_pars"]), rtol=tol)
        for key in ("pred_latent_False", "pred_latent_True"):
            for k, w in want[key].items():
                if w is None:
                    assert got[key][k] is None, (key, k)
                else:
                    assert np.abs(_hex(got[key][k]) - _hex(w)).max() <= tol * np.abs(_hex(w)).max(), (want["name"], key, k)


def test_golden_covers_the_ranges_and_both_latent_modes():
    assert [r["name"] for r in GOLD["leaf"]] == ["text_io", "missing_0", "missing_1"]
    for rec in GOLD["leaf"]:
        assert [(r["start"], r["num"]) for r in rec["ranges"]] == list(RANGES)
    assert [c["name"] for c in GOLD["gpboost"]] == ["fixed_cov_pars", "fitted_cov_pars"]
    for c in GOLD["gpboost"]:
        lat, resp = c["pred_latent_True"], c["pred_latent_False"]
        assert lat["response_mean"] is None and lat["response_var"] is None and resp["fixed_effect"] is None
        assert resp["random_effect_mean"] is None and resp["random_effect_cov"] is None
        for v in (lat["fixed_effect"], lat["random_effect_mean"], lat["random_effect_cov"], resp["response_mean"], resp["response_var"]):
            assert len(v) == c["n_test"]
        # response = latent + fixed effect, response variance = latent variance + error variance (the golden is self-consistent)
        np.testing.assert_allclose(_hex(resp["response_mean"]), _hex(lat["fixed_effect"]) + _hex(lat["random_effect_mean"]), rtol=1e-12)
        np.testing.assert_allclose(_hex(resp["response_var"]), _hex(lat["random_effect_cov"]) + _hex(c["cov_pars"])[0], rtol=1e-10)


def test_numpy_walk_matches_reference_bitwise(ref_golden):
    for (name, text, Xt), rec in zip(leaf_models(ref_golden), GOLD["leaf"]):
        trees = parse_model_string(text)
        for r in rec["ranges"]:
            st, nit = r["start"], r["num"]
            assert ew.digest(ew.predict(trees, Xt, st, nit), np.float64) == r["raw_sha256"], (name, st, nit)
            leaf = ew.predict(trees, Xt, st, nit, pred_leaf=True)
            assert list(leaf.shape) == r["shape"] and ew.digest(leaf, np.int32) == r["leaf_sha256"], (name, st, nit)
    # the digests are of the arrays test_model_text_io.py compares with value by value
    for got, want in zip(GOLD["leaf"][0]["ranges"], ref_golden["text_io"]["ranges"]):
        assert got["raw_sha256"] == ew.digest(np.array(want["pred"]), np.float64)
    # the GPBoost models' tree part
    for c in GOLD["gpboost"]:
        import treedata
        Xt = treedata.make_case(dict(c, n=c["n_test"], seed=c["seed"] + 100))[0]
        assert np.array_equal(ew.predict(parse_model_string(c["model"]), Xt), _hex(c["pred_latent_True"]["fixed_effect"])), c["name"]


def test_model_string_booster_predicts_leaf_indices(ref_golden, product_lib):
    for (name, text, Xt), rec in zip(leaf_models(ref_golden), GOLD["leaf"]):
        b = Booster(model_str=text, _lib=product_lib)
        for r in rec["ranges"]:
            st, nit = r["start"], r["num"]
            got = b.predict(Xt, start_iteration=st, num_iteration=nit, pred_leaf=True)
            assert list(got.shape) == r["shape"] and ew.digest(got, np.int32) == r["leaf_sha256"], (name, st, nit)
            assert ew.digest(b.predict(Xt, start_iteration=st, num_iteration=nit), np.float64) == r["raw_sha256"], (name, st, nit)
            for ptype, per_row in ((0, 1), (1, 1), (2, r["shape"][1])):
                n = C.c_int64(-1)
                assert product_lib.LGBM_BoosterCalcNumPredict(b.handle, C.c_int(Xt.shape[0]), C.c_int(ptype), C.c_int(st), C.c_int(nit),
                                                              C.byref(n)) == 0
                assert n.value == Xt.shape[0] * per_row, (name, st, nit, ptype)


def test_contributions_stay_refused(ref_golden, product_lib):
    from gpboost_b200.basic import GPBoostError
    b = Booster(model_str=ref_golden["text_io"]["model"], _lib=product_lib)
    n = C.c_int64(0)
    assert product_lib.LGBM_BoosterCalcNumPredict(b.handle, C.c_int(10), C.c_int(3), C.c_int(0), C.c_int(-1), C.byref(n)) != 0
    assert "not supported by this build" in product_lib.LGBM_GetLastError().decode()
    with pytest.raises(GPBoostError, match="not supported by this build"):
        b.predict(text_io_case()[2], pred_contrib=True)
