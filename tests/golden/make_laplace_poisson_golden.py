"""Generates tests/golden/laplace_poisson_golden.json with the UNMODIFIED reference library (oracle/_ref) through the shared
frontend: latent Vecchia GP + poisson likelihood (log link), Laplace-approximated negative log-likelihood with
matrix_inversion_method = "iterative" (VADU preconditioner, seed 1, num_rand_vec_trace probes), the reference's Newton iteration
count of that evaluation (its SLQ count is not exported for this model), the gradient w.r.t. the log covariance parameters
(recovered from one gradient-descent step of the reference's optimiser, as in make_laplace_golden.py), a fit with the reference's
defaults (L-BFGS), and the result of the unmodified reference Python package fitting counts (poisson_data.DROPIN_SCRIPT).
Run from the repository root after building oracle/_ref:  python tests/golden/make_laplace_poisson_golden.py"""
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import poisson_data  # noqa: E402
from gpboost_b200 import GPModel  # noqa: E402
from gpboost_b200.libpath import load_lib  # noqa: E402
from oracle import ref_lib_path  # noqa: E402

# log_mean -2.5: ~90% zeros; log(1000) as an offset: counts around 1e3, W = exp(loc) ~ 1e3
CASES = [
    dict(name="exp_m10", n=2000, dseed=31, cov_function="exponential", shape=0.5, m=10, ordering="random", seed=1,
         cov_pars=[0.8, 0.12], t=50),
    dict(name="m15_m20_offset", n=2500, dseed=32, offset=True, cov_function="matern", shape=1.5, m=20, ordering="random", seed=2,
         cov_pars=[0.5, 0.1], t=30),
    dict(name="m25_m30_none", n=2000, dseed=33, cov_function="matern", shape=2.5, m=30, ordering="none", seed=3,
         cov_pars=[0.6, 0.08], t=50),
    dict(name="many_zeros", n=2000, dseed=34, log_mean=-2.5, cov_function="matern", shape=1.5, m=20, ordering="random", seed=4,
         cov_pars=[1.0, 0.1], t=50),
    dict(name="large_counts", n=1500, dseed=35, log_mean=float(np.log(1000.)), offset_is_mean=True, cov_function="exponential",
         shape=0.5, m=30, ordering="random", seed=5, cov_pars=[0.7, 0.15], t=64),
    dict(name="m15_m10_none_offset", n=3000, dseed=36, offset=True, cov_function="matern", shape=1.5, m=10, ordering="none", seed=6,
         cov_pars=[1.2, 0.07], t=50),
]


def model(c, lib=None):
    return GPModel(likelihood="poisson", gp_coords=poisson_data.case_data(c)[0], cov_function=c["cov_function"], cov_fct_shape=c["shape"],
                   gp_approx="vecchia", num_neighbors=c["m"], vecchia_ordering=c["ordering"], seed=c["seed"],
                   matrix_inversion_method="iterative", _lib=lib)


def reference_gradient(ref, c, y, off):
    th0 = np.array(c["cov_pars"], dtype=np.float64)
    got = []
    for lr in (1e-4, 5e-5):
        g = model(c, ref)
        g.params["use_nesterov_acc"] = False
        g.fit(y, params=dict(optimizer_cov="gradient_descent", lr_cov=lr, maxit=1, init_cov_pars=th0, delta_rel_conv=1e-30,
                             num_rand_vec_trace=c["t"]), offset=off)
        got.append(-np.log(g.get_cov_pars() / th0) / lr)
    assert np.all(np.abs(got[0] - got[1]) <= 1e-7 * np.abs(got[0])), got
    return got[0].tolist()


def count(g, name):
    v = ctypes.c_int(0)
    g._safe_call(getattr(g._LIB, name)(g.handle, ctypes.byref(v)))
    return int(v.value)


if __name__ == "__main__":
    ref = load_lib(ref_lib_path())
    out = {"generator": "tests/golden/make_laplace_poisson_golden.py", "cases": []}
    for c in CASES:
        X, y, off = poisson_data.case_data(c)
        rec = dict(c)
        rec["y_sum"], rec["y_zeros"], rec["y_max"] = float(y.sum()), int((y == 0).sum()), float(y.max())
        m = model(c, ref)
        m.set_optim_params(dict(num_rand_vec_trace=c["t"]))
        rec["negll"] = m.neg_log_likelihood(np.array(c["cov_pars"]), y, fixed_effects=off)
        rec["newton_it"] = count(m, "GPB_GetNumModeFindingSteps")
        rec["grad"] = reference_gradient(ref, c, y, off)
        if c["n"] <= 2500:
            g = model(c, ref)
            g.fit(y, params=dict(num_rand_vec_trace=c["t"]), offset=off)
            init = np.zeros(2)
            g._safe_call(g._LIB.GPB_GetInitCovPar(g.handle, init.ctypes.data_as(ctypes.POINTER(ctypes.c_double))))
            rec["fit"] = dict(init_cov_pars=init.tolist(), cov_pars=g.get_cov_pars().tolist(), num_it=int(g._get_num_optim_iter()),
                              negll=float(g.get_current_neg_log_likelihood()))
        print(rec, flush=True)
        out["cases"].append(rec)
    # the unmodified reference Python package on the reference library (tests/test_laplace_poisson_gpu.py runs it on the product)
    import dropin
    out["dropin"] = dropin.run_with(ref_lib_path(), poisson_data.DROPIN_SCRIPT)
    print(out["dropin"], flush=True)
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "laplace_poisson_golden.json"), "w") as f:
        json.dump(out, f, indent=1)
