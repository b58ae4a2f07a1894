"""CPU: the oracle's standard errors of the Gaussian Vecchia covariance parameters (oracle/std_err.py) reproduce the reference
library's (tests/golden/std_err_golden.json, tests/golden/make_std_err_golden.py), and the golden grid covers what it has to."""
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from golden.make_std_err_golden import case_data  # noqa: E402
from oracle import std_err as ose  # noqa: E402

with open(os.path.join(ROOT, "tests", "golden", "std_err_golden.json")) as f:
    GOLD = json.load(f)["cases"]
BY_NAME = {c["name"]: c for c in GOLD}


def rtol_of(c):
    """1e-8; 1e-6 for the ill-conditioned Gaussian and Matern-2.5 kernels (DESIGN.md §5)"""
    return 1e-6 if c["cov_function"] == "gaussian" or c["shape"] == 2.5 else 1e-8


def oracle_fits(c):
    """the oracle's standard errors for every fit of a golden case, with the probe draws the reference makes: one draw per model
    with reuse_rand_vec_trace, a new draw (the generator counter advanced) for every computation without it"""
    coords, _, _ = case_data(c)
    out = []
    for k, fit in enumerate(c["fits"]):
        run_id = 0 if c.get("reuse", True) else k
        sd, FI = ose.std_err(coords, fit["params"], cov_function=c["cov_function"], cov_fct_shape=c["shape"],
                             num_neighbors=c["m"], seed=c["seed"], num_rand_vec_trace=c["t"],
                             seed_rand_vec_trace=c.get("seed_rand_vec_trace", 1), run_id=run_id)
        out.append((sd, FI))
    return out


@pytest.mark.parametrize("name", [c["name"] for c in GOLD])
def test_oracle_reproduces_reference_std_err(name):
    c = BY_NAME[name]
    for fit, (sd, FI) in zip(c["fits"], oracle_fits(c)):
        assert np.all(np.isfinite(FI)) and np.allclose(FI, FI.T, rtol=0, atol=0)
        np.testing.assert_allclose(sd, fit["std_err"], rtol=rtol_of(c), atol=0)


def test_golden_grid_covers_the_contract():
    kernels = {(c["cov_function"], c["shape"]) for c in GOLD}
    assert kernels >= {("exponential", 0.5), ("matern", 1.5), ("matern", 2.5), ("gaussian", 0.)}
    assert {1, 10, 20, 30} <= {c["m"] for c in GOLD}
    assert {1, 2, 3} <= {c["d"] for c in GOLD}
    ns = [c["n"] for c in GOLD]
    assert min(ns) <= 500 and max(ns) >= 20000
    assert {1, 50, 128, 129, 300} <= {c["t"] for c in GOLD}
    assert any(c.get("seed_rand_vec_trace", 1) != 1 for c in GOLD)
    noreuse = [c for c in GOLD if c.get("reuse") is False]
    assert noreuse and all(len(c["fits"]) == 2 for c in noreuse)
    assert any(c.get("p") for c in GOLD)
    assert sum(1 for c in GOLD if c.get("fit")) >= 2
    # the probe draw of the second fit differs exactly when the probes are not reused
    a, b = BY_NAME["exp_m20_noreuse"]["fits"][1], BY_NAME["exp_m20_reuse"]["fits"][1]
    assert a["params"] == b["params"] and a["std_err"] != b["std_err"]
