"""Generates tests/golden/validation_golden.json with the UNMODIFIED reference library (oracle/_ref) through the shared frontend:
validation data of the boosting loop (LGBM_DatasetCreateFromMat with a reference, LGBM_BoosterAddValidData, LGBM_BoosterGetEval,
LGBM_BoosterGetPredict(data_idx >= 1)). Every case of tests/validation_cases.py records the evaluation list after every iteration and
the final raw validation scores (hex floats, compared bitwise). The early-stopping case records gpboost_b200.train on the reference
library and, where the reference's Python package is present, the package's gpb.train (best_iteration, evals_result).
Run from the repository root after building oracle/_ref:  python tests/golden/make_validation_golden.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import validation_cases as vc  # noqa: E402
from gpboost_b200.libpath import load_lib  # noqa: E402
from oracle import ref_lib_path  # noqa: E402

ES_BODY = """
import sys
sys.path.insert(1, %r)
sys.path.insert(2, %r)
import validation_cases as vc
c = vc.ES_CASE
data = vc.case_data(c)
params = vc.params_of(c)
dtrain = gpb.Dataset(data[0][0], data[0][1], params=params, free_raw_data=False)
dvalid = gpb.Dataset(data[1][0], data[1][1], params=params, reference=dtrain)
ev = {}
bst = gpb.train(params, dtrain, num_boost_round=c["num_boost_round"], valid_sets=[dvalid], valid_names=["valid"],
                early_stopping_rounds=c["early_stopping_rounds"], evals_result=ev, verbose_eval=False)
out["best_iteration"] = bst.best_iteration
out["evals_result"] = {k: {m: list(map(float, v)) for m, v in d.items()} for k, d in ev.items()}
"""

if __name__ == "__main__":
    ref = load_lib(ref_lib_path())
    out = {"generator": "tests/golden/make_validation_golden.py", "num_it": vc.NUM_IT, "cases": []}
    for c in vc.CASES:
        rec = dict(c)
        res, _, _, _ = vc.run_case(c, lib=ref)
        rec.update(res)
        print(c["name"], res["eval_names"], res["evals"][-1])
        out["cases"].append(rec)
    es = dict(vc.ES_CASE)
    es["frontend"] = vc.run_es_case(vc.ES_CASE, lib=ref)
    print("early stopping (frontend on the reference library):", es["frontend"]["best_iteration"])
    import dropin
    if dropin.ref_package_dir() is not None:
        es["package"] = dropin.run_with(ref_lib_path(), ES_BODY % (os.path.join(ROOT, "tests"), ROOT))
        print("early stopping (reference package):", es["package"]["best_iteration"])
    out["early_stopping"] = es
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "validation_golden.json"), "w") as f:
        json.dump(out, f, indent=0)
