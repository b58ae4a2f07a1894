"""Pins a numpy restatement of the validation metrics (l2, rmse, l1, test_neg_log_likelihood without the GP: regression_metric.hpp
:28-190, :401-479, the residual variance of gbdt.cpp:525-542) to the reference library's values in tests/golden/validation_golden.json,
from the raw scores the goldens store. The device metric kernel is checked against the same goldens in tests/test_validation_gpu.py."""
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import validation_cases as vc  # noqa: E402

with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "validation_golden.json")) as _f:
    GOLD = json.load(_f)


def metrics(names, score, label, train_score=None, train_label=None):
    e = score - label
    out = []
    for m in names:
        if m == "l2":
            out.append(np.mean(e ** 2))
        elif m == "rmse":
            out.append(np.sqrt(np.mean(e ** 2)))
        elif m == "l1":
            out.append(np.mean(np.abs(e)))
        elif m == "test_neg_log_likelihood":
            r = train_label - train_score
            rv = np.sum((r - np.mean(r)) ** 2) / (r.shape[0] - 1)
            out.append(0.5 * np.mean(e ** 2 / rv + np.log(rv) + np.log(2. * np.pi)))
    return out


def _hex(v):
    return np.array([float.fromhex(x) for x in v])


@pytest.mark.parametrize("case", [c for c in GOLD["cases"] if not (c.get("gp") and c.get("use_gp"))], ids=lambda c: c["name"])
def test_numpy_metrics_match_reference(case):
    data = vc.case_data(case)
    lab = [d[1].astype(np.float32).astype(np.float64) for d in data]  # label_t = float
    final = case["evals"][-1]
    names = case["eval_names"]
    assert len(names) == len(vc.metric_names(case))  # aliases resolved by the library (mse -> l2, l2_root -> rmse, mae -> l1)
    ts = _hex(case["train_scores"]) if "train_scores" in case else None
    rows = [r for r in final if not r[0].startswith("valid_")]
    for k, scores in enumerate(case["valid_scores"]):
        want = [r[2] for r in final if r[0] == "valid_%d" % k]
        got = metrics(names, _hex(scores), lab[k + 1], ts, lab[0])
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
    if rows:  # the training data as a validation set: its metrics need the training scores, which the goldens do not store
        assert [r[1] for r in rows] == names


def test_early_stopping_golden_stops_early():
    es = GOLD["early_stopping"]
    assert es["frontend"]["best_iteration"] < es["num_boost_round"]
    n_rounds = len(es["frontend"]["evals_result"]["valid"]["l2"])
    assert n_rounds == es["frontend"]["best_iteration"] + es["early_stopping_rounds"]
    if "package" in es:
        assert es["package"]["best_iteration"] == es["frontend"]["best_iteration"]
        for m, v in es["package"]["evals_result"]["valid"].items():
            np.testing.assert_allclose(es["frontend"]["evals_result"]["valid"][m], v, rtol=1e-12, atol=0)
