"""Generates tests/golden/grouped_multi_golden.json with the UNMODIFIED reference library (oracle/_ref) through the shared frontend:
K >= 2 grouped random effects, Gaussian likelihood. Negative log-likelihoods with the reference's default method ("iterative",
SSOR preconditioner) together with its CG iteration counts, the same with matrix_inversion_method = "cholesky", fits and GPBoost runs.
Run from the repository root after building oracle/_ref:  python tests/golden/make_grouped_multi_golden.py"""
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import grouped_multi_data as gmd  # noqa: E402
from gpboost_b200 import GPModel  # noqa: E402
from gpboost_b200.booster import Booster, Dataset, parse_model_string  # noqa: E402
from gpboost_b200.libpath import load_lib  # noqa: E402
from oracle import ref_lib_path  # noqa: E402

ref = load_lib(ref_lib_path())


def cg_counts(m):
    a, b = ctypes.c_int(0), ctypes.c_int(0)
    m._safe_call(ref.GPB_GetNumCGSteps(m.handle, ctypes.byref(a)))
    m._safe_call(ref.GPB_GetNumCGStepsTridiag(m.handle, ctypes.byref(b)))
    return a.value, b.value


out = {"generator": "tests/golden/make_grouped_multi_golden.py", "nll": [], "fit": [], "boost": []}
for name in gmd.CASES:
    group, y, it = gmd.case(name)
    K = group.shape[1]
    for cp in gmd.COV_PARS[K]:
        rec = {"case": name, "cov_pars": cp}
        m = GPModel(group_data=group, _lib=ref)
        if it:
            m.set_optim_params(dict(it))
        rec["negll"] = m.neg_log_likelihood(np.array(cp), y)
        rec["cg_its"], rec["cg_its_tridiag"] = cg_counts(m)
        mc = GPModel(group_data=group, matrix_inversion_method="cholesky", _lib=ref)
        rec["negll_cholesky"] = mc.neg_log_likelihood(np.array(cp), y)
        out["nll"].append(rec)
        print(rec)
    if it:
        continue
    m = GPModel(group_data=group, _lib=ref)
    m.fit(y)
    rec = {"case": name, "cov_pars": m.get_cov_pars().tolist(), "negll": m.get_current_neg_log_likelihood(),
           "num_it": m._get_num_optim_iter()}
    out["fit"].append(rec)
    print(rec)

X, y, group = gmd.boost_case()
for train_cov in (False, True):
    params = dict(gmd.BOOST_PARAMS, force_col_wise=True, deterministic=True, num_threads=4)
    gp = GPModel(group_data=group, _lib=ref)
    if not train_cov:
        params["train_gp_model_cov_pars"] = False
        gp.set_optim_params({"init_cov_pars": gmd.BOOST_FIXED_COV_PARS})
    b = Booster(params, Dataset(X, y, params=params, _lib=ref), gp_model=gp, _lib=ref)
    for _ in range(4):
        b.update()
    trees = parse_model_string(b.model_to_string())
    out["boost"].append({"train_cov": train_cov, "cov_pars": gp.get_cov_pars().tolist(), "score_head": b.inner_predict_train()[:64].tolist(),
                         "trees": [{k: (v.tolist() if hasattr(v, "tolist") else v) for k, v in t.items()
                                    if k in ("num_leaves", "split_feature", "threshold", "leaf_value")} for t in trees]})
    print("boost", train_cov, out["boost"][-1]["cov_pars"])
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "grouped_multi_golden.json"), "w") as f:
    json.dump(out, f)
