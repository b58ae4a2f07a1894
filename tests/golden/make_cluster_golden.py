"""Generates tests/golden/cluster_golden.json with the UNMODIFIED reference library (oracle/_ref) through the shared frontend: Gaussian
Vecchia GPs with several independent realizations (cluster_ids). Every case of tests/cluster_cases.py:CASES records the likelihood at
fixed parameters, a fit and the predictions (tests/cluster_cases.py:run_case); BOOST_CASE records the trees and validation metrics of
GPBoost at fixed covariance parameters (also with Newton leaf updates) and the first tree with trained ones. Run from the repository root after building oracle/_ref:
    python tests/golden/make_cluster_golden.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cluster_cases as cc  # noqa: E402
from gpboost_b200.libpath import load_lib  # noqa: E402
from oracle import ref_lib_path  # noqa: E402

if __name__ == "__main__":
    ref = load_lib(ref_lib_path())
    out = {"generator": "tests/golden/make_cluster_golden.py", "reference": "fabsig/GPBoost c93fa49 (v1.7.3), CPU build", "cases": []}
    for c in cc.CASES:
        r = cc.run_case(c, ref)
        print(c["name"], r["nll"], r["num_it"], r["cov_pars"], flush=True)
        out["cases"].append(r)
    fixed, _ = cc.run_boost(cc.BOOST_CASE, ref, train_cov_pars=False)
    trained, _ = cc.run_boost(cc.BOOST_CASE, ref, train_cov_pars=True, num_it=1)
    out["boost_fixed"] = fixed
    out["boost_trained"] = trained
    for key, extra in cc.BOOST_VARIANTS.items():
        out[key], _ = cc.run_boost(cc.BOOST_CASE, ref, train_cov_pars=False, extra=extra)
        print(key, out[key]["evals"][-1], flush=True)
    print("boost", fixed["evals"][-1], trained["cov_pars"], flush=True)
    with open(os.path.join(ROOT, "tests", "golden", "cluster_golden.json"), "w") as f:
        json.dump(out, f)
