"""Generates tests/golden/std_err_golden.json with the UNMODIFIED reference library (oracle/_ref) through the shared frontend:
standard errors of the covariance parameters of the Gaussian Vecchia GP, GPModel.get_cov_pars(std_err=True) -> GPB_GetCovPar with
calc_std_dev (CalcStdDevCovPar: stochastic Fisher information, re_model_template.h:10788-10815, :10145-10230).

Most cases hold the parameters fixed (init_cov_pars, maxit = 0), so that the standard errors depend on the parameters and the probe
vectors only. Every case records the parameters and standard errors the reference reports (the 2 x 3 table). The Fisher information
itself is not exported by the reference's C API; tests/test_std_err_oracle_pinned.py pins the oracle's (oracle/std_err.py) through
the standard errors it implies.
Run from the repository root after building oracle/_ref:  python tests/golden/make_std_err_golden.py"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import datagen  # noqa: E402
from gpboost_b200 import GPModel  # noqa: E402
from gpboost_b200.libpath import load_lib  # noqa: E402
from oracle import ref_lib_path  # noqa: E402

# kernels x neighbour counts x dimensions x probe counts; a non-default probe seed; two fits with reuse_rand_vec_trace = False
# (and the default True for contrast); a model with covariates; two cases after a real fit
CASES = [
    dict(name="exp_m10_d2", n=500, d=2, dseed=21, cov_function="exponential", shape=0.5, m=10, seed=1, t=50,
         cov_pars=[0.3, 1.2, 0.15]),
    dict(name="m15_m20_d2", n=2000, d=2, dseed=22, cov_function="matern", shape=1.5, m=20, seed=2, t=50,
         cov_pars=[0.25, 1.0, 0.1]),
    dict(name="m25_m30_d2_t1", n=1000, d=2, dseed=23, cov_function="matern", shape=2.5, m=30, seed=3, t=1,
         cov_pars=[0.2, 0.8, 0.12]),
    dict(name="gauss_m10_d2_t128", n=800, d=2, dseed=24, cov_function="gaussian", shape=0., m=10, seed=4, t=128,
         cov_pars=[0.3, 1.0, 0.2]),
    dict(name="m15_m30_d3_t129", n=3000, d=3, dseed=25, cov_function="matern", shape=1.5, m=30, seed=5, t=129,
         cov_pars=[0.4, 1.5, 0.2]),
    dict(name="exp_m1_d1", n=300, d=1, dseed=26, cov_function="exponential", shape=0.5, m=1, seed=6, t=50,
         cov_pars=[0.1, 1.0, 0.1]),
    dict(name="m25_m20_d1_t300", n=1500, d=1, dseed=27, cov_function="matern", shape=2.5, m=20, seed=7, t=300,
         cov_pars=[0.3, 0.9, 0.05]),
    dict(name="gauss_m30_d3_n2e4", n=20000, d=3, dseed=28, cov_function="gaussian", shape=0., m=30, seed=8, t=50,
         cov_pars=[0.25, 1.1, 0.25]),
    dict(name="m15_m10_seed7", n=1000, d=2, dseed=29, cov_function="matern", shape=1.5, m=10, seed=9, t=50,
         seed_rand_vec_trace=7, cov_pars=[0.3, 1.0, 0.1]),
    dict(name="exp_m20_noreuse", n=1200, d=2, dseed=30, cov_function="exponential", shape=0.5, m=20, seed=10, t=50,
         reuse=False, cov_pars=[0.3, 1.2, 0.15], cov_pars2=[0.5, 0.7, 0.3]),
    dict(name="exp_m20_reuse", n=1200, d=2, dseed=30, cov_function="exponential", shape=0.5, m=20, seed=10, t=50,
         reuse=True, cov_pars=[0.3, 1.2, 0.15], cov_pars2=[0.5, 0.7, 0.3]),
    dict(name="m15_m20_covariates", n=1500, d=2, dseed=31, cov_function="matern", shape=1.5, m=20, seed=11, t=50, p=3,
         cov_pars=[0.3, 1.0, 0.1]),
    dict(name="m15_m20_fit", n=1000, d=2, dseed=32, cov_function="matern", shape=1.5, m=20, seed=12, t=50, fit=True),
    dict(name="exp_m10_fit", n=800, d=2, dseed=33, cov_function="exponential", shape=0.5, m=10, seed=13, t=50, fit=True),
]


def case_data(c):
    """coords, y and (with p) X: n x p, first column 1"""
    coords, y = datagen.synth(c["n"], c["d"], c["dseed"])
    X = None
    if c.get("p"):
        rng = np.random.default_rng(c["dseed"] + 100)
        X = np.ones((c["n"], c["p"]))
        X[:, 1:] = rng.standard_normal((c["n"], c["p"] - 1))
        y = y + X @ np.concatenate([[1.5], rng.uniform(-2., 2., c["p"] - 1)])
    return coords, y, X


def model(c, coords, lib=None):
    kw = {} if lib is None else dict(_lib=lib)
    return GPModel(gp_coords=coords, cov_function=c["cov_function"], cov_fct_shape=c["shape"], gp_approx="vecchia",
                   num_neighbors=c["m"], vecchia_ordering="random", seed=c["seed"], **kw)


def fit_params(c, cov_pars=None):
    params = dict(num_rand_vec_trace=c["t"], reuse_rand_vec_trace=c.get("reuse", True),
                  seed_rand_vec_trace=c.get("seed_rand_vec_trace", 1))
    if cov_pars is not None:
        params.update(init_cov_pars=np.array(cov_pars), maxit=0)
    return params


def run(c, lib):
    """[(parameters, standard errors)] of the case's fits on `lib`, one entry per fit"""
    coords, y, X = case_data(c)
    mod = model(c, coords, lib)
    out = []
    for key in ("cov_pars", "cov_pars2"):
        if key not in c and not (key == "cov_pars" and c.get("fit")):
            continue
        mod.fit(y, X=X, params=fit_params(c, c.get(key)))
        tab = mod.get_cov_pars(std_err=True)
        out.append(dict(params=tab[0].tolist(), std_err=tab[1].tolist()))
    return out


if __name__ == "__main__":
    ref = load_lib(ref_lib_path())
    out = {"generator": "tests/golden/make_std_err_golden.py", "cases": []}
    for c in CASES:
        rec = dict(c)
        rec["fits"] = run(c, ref)
        print(c["name"], rec["fits"])
        out["cases"].append(rec)
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "std_err_golden.json"), "w") as f:
        json.dump(out, f, indent=1)
