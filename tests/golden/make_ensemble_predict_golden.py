"""Generates tests/golden/ensemble_predict_golden.json with the UNMODIFIED reference library (oracle/_ref) and its unmodified Python
package: what a trained model predicts at new data.
  * "leaf": for the reference-trained models of tests/golden/reference_golden.json (the text-IO model and the two missing-value models)
    the leaf indices (pred_leaf, int32) and raw scores (float64) over the iteration ranges of test_model_text_io.RANGES, through the
    shared frontend on the reference library — stored as sha256 digests of the arrays' bytes (ensemble_walk.digest), which is all a
    bitwise comparison needs;
  * "gpboost": two GPBoost models (Gaussian Vecchia GP, m = 15, Matern-1.5, 20 rounds on 2000 x 5 training data) trained by the package's
    gpb.train — one at fixed covariance parameters (train_gp_model_cov_pars=False), one with the parameters fitted — with the package's
    bst.predict(Xtest, gp_coords_pred=..., predict_var=True, pred_latent=False / True) dicts at 100 test rows (hex floats), the
    covariance parameters the prediction used and the model text reduced to the fields a tree walk reads.
Run from the repository root after building oracle/_ref:  python tests/golden/make_ensemble_predict_golden.py"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import dropin  # noqa: E402
import ensemble_walk as ew  # noqa: E402
from gpboost_b200.booster import Booster  # noqa: E402
from gpboost_b200.libpath import load_lib  # noqa: E402
from oracle import ref_lib_path  # noqa: E402
from test_model_text_io import RANGES, missing_cases, text_io_case  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ensemble_predict_golden.json")

# the GPBoost cases: data of treedata.make_case(spec); test rows from the same generator at n_test rows and seed + 100
GP_CASES = [
    dict(name="fixed_cov_pars", n=2000, F=5, kind="real", num_leaves=15, min_data_in_leaf=20, seed=31, gp=True, num_neighbors=15,
         train_cov=False, init_cov_pars=[0.1, 0.4, 0.15], num_boost_round=20, n_test=100),
    dict(name="fitted_cov_pars", n=2000, F=5, kind="real", num_leaves=15, min_data_in_leaf=20, seed=32, gp=True, num_neighbors=15,
         num_boost_round=20, n_test=100),
]

GP_BODY = """
import sys
sys.path.insert(1, %r)
import treedata
spec = %r
X, y, coords = treedata.make_case(spec)
Xt, _, coords_t = treedata.make_case(dict(spec, n=spec["n_test"], seed=spec["seed"] + 100))
params = treedata.booster_params(spec, reference=True)
fixed = spec.get("train_cov") is False
params.pop("train_gp_model_cov_pars", None)
gp = gpb.GPModel(gp_coords=coords, cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia", num_neighbors=spec["num_neighbors"],
                 vecchia_ordering="random", seed=spec["seed"])
if fixed:
    gp.set_optim_params({"init_cov_pars": np.array(spec["init_cov_pars"])})
ds = gpb.Dataset(X, y, free_raw_data=False)
bst = gpb.train(params=params, train_set=ds, gp_model=gp, num_boost_round=spec["num_boost_round"], train_gp_model_cov_pars=not fixed)
cov_pars = np.array(spec["init_cov_pars"]) if fixed else np.asarray(gp.get_cov_pars()).reshape(-1)[:3]
txt = bst.model_to_string()
if txt.lstrip().startswith("{"):
    txt = json.loads(txt)["booster_str"]
out["model"] = txt
out["cov_pars"] = [float(v).hex() for v in cov_pars]
hexes = lambda a: None if a is None else [float(v).hex() for v in np.asarray(a).reshape(-1)]
for latent in (False, True):
    r = bst.predict(Xt, gp_coords_pred=coords_t, predict_var=True, pred_latent=latent, cov_pars=cov_pars)
    out["pred_latent_%%s" %% latent] = {k: hexes(r[k]) for k in ("fixed_effect", "random_effect_mean", "random_effect_cov", "response_mean",
                                                              "response_var")}
"""


def leaf_records(lib):
    with open(os.path.join(ROOT, "tests", "golden", "reference_golden.json")) as f:
        ref_golden = json.load(f)
    models = [("text_io", ref_golden["text_io"]["model"], text_io_case()[2])]
    for i, ((_, _, Xt, _), rec) in enumerate(zip(missing_cases(), ref_golden["missing"])):
        models.append(("missing_%d" % i, rec["model"], Xt))
    out = []
    for name, text, Xt in models:
        b = Booster(model_str=text, _lib=lib)
        rec = {"name": name, "ranges": []}
        for st, nit in RANGES:
            leaf = b.predict(Xt, start_iteration=st, num_iteration=nit, pred_leaf=True)
            raw = b.predict(Xt, start_iteration=st, num_iteration=nit)
            rec["ranges"].append({"start": st, "num": nit, "shape": list(leaf.shape), "leaf_sha256": ew.digest(leaf, np.int32),
                                  "raw_sha256": ew.digest(raw, np.float64)})
        out.append(rec)
    return out


HEAD_KEYS = ("version", "num_class", "num_tree_per_iteration", "label_index", "max_feature_idx", "objective", "feature_names", "feature_infos")
TREE_KEYS = ("num_leaves", "num_cat", "split_feature", "threshold", "decision_type", "left_child", "right_child", "leaf_value", "shrinkage")


def walk_fields(text):
    """the model text without what no prediction reads (gains, counts, internal values, the parameter dump)"""
    out, in_trees = ["tree"], False
    for ln in text.split("\n"):
        if ln.startswith("end of trees"):
            break
        if ln.startswith("Tree="):
            in_trees = True
            out += ["", ln]
        elif ln.split("=")[0] in (TREE_KEYS if in_trees else HEAD_KEYS):
            out.append(ln)
    return "\n".join(out) + "\n\nend of trees\n"


def gp_records():
    out = []
    for spec in GP_CASES:
        rec = dict(spec)
        rec.update(dropin.run_with(ref_lib_path(), GP_BODY % (os.path.join(ROOT, "tests"), spec)))
        rec["model"] = walk_fields(rec["model"])
        out.append(rec)
    return out


def generate():
    out = {"generator": "tests/golden/make_ensemble_predict_golden.py", "leaf": leaf_records(load_lib(ref_lib_path()))}
    assert dropin.ref_package_dir() is not None, "no reference checkout at oracle.reference_dir()"
    out["gpboost"] = gp_records()
    return out


if __name__ == "__main__":
    g = generate()
    with open(GOLDEN, "w") as f:  # one record per line
        f.write('{"generator": %s,\n"leaf": [\n%s],\n"gpboost": [\n%s]}\n' % (
            json.dumps(g["generator"]), ",\n".join(json.dumps(r) for r in g["leaf"]), ",\n".join(json.dumps(r) for r in g["gpboost"])))
