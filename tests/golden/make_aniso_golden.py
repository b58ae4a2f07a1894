"""Generates tests/golden/aniso_golden.json with the UNMODIFIED reference library (oracle/_ref) through the shared frontend: the
anisotropic covariance functions matern_ard, gaussian_ard and matern_space_time with the Gaussian Vecchia GP. Every case of
tests/aniso_oracle.py:CASES runs tests/aniso_oracle.py:run_case: the likelihood at theta1 and then theta2 on one model (the second
reuses the neighbour sets the first searched), at theta2 on a fresh model, a fit (parameters, likelihood, iterations) and the
prediction at 100 points at the fitted parameters. Run from the repository root after building oracle/_ref:
    python tests/golden/make_aniso_golden.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import aniso_oracle as ao  # noqa: E402
from gpboost_b200 import GPModel  # noqa: E402
from gpboost_b200.libpath import load_lib  # noqa: E402
from oracle import ref_lib_path  # noqa: E402

if __name__ == "__main__":
    ref = load_lib(ref_lib_path())
    out = {"generator": "tests/golden/make_aniso_golden.py", "reference": "fabsig/GPBoost c93fa49 (v1.7.3), CPU build", "cases": []}
    for c in ao.CASES:
        r, _ = ao.run_case(GPModel, c, ref)
        print(c["name"], r["nll_t1"], r["nll_t2_same"], r["nll_t2_fresh"], r["num_it"], r["cov_pars"], flush=True)
        out["cases"].append(r)
    with open(os.path.join(ROOT, "tests", "golden", "aniso_golden.json"), "w") as f:
        json.dump(out, f)
