"""Several grouped random effects (crossed, nested, K = 3), Gaussian likelihood: the numpy restatement of the reference's iterative
path (oracle/grouped_multi.py) pinned to the reference's values in tests/golden/grouped_multi_golden.json, on the CPU.

Tolerances:
- iterative negative log-likelihood 1e-8 relative, CG and Lanczos iteration counts equal: the restatement draws the same probe vectors
  and runs the same iterations and stopping rules, so only the summation order differs;
- the exact dense log|Psi| and y^T Psi^-1 y against the reference's Cholesky value 1e-10 relative: both are exact up to rounding."""
import json
import os

import numpy as np
import pytest

import grouped_multi_data as gmd
from oracle import grouped_multi as gm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold():
    with open(os.path.join(ROOT, "tests", "golden", "grouped_multi_golden.json")) as f:
        return json.load(f)


def oracle_eval(name, cp, **extra):
    group, y, it = gmd.case(name)
    st = gm.Structure(group)
    cfg = dict(gm.DEFAULTS, **it)
    r = gm.probes(st, cfg["num_rand_vec_trace"], cfg["seed_rand_vec_trace"])
    cp = np.asarray(cp, dtype=np.float64)
    return gm.evaluate(st, y, cp[1:] / cp[0], sigma2=cp[0], r=r, **dict(it, **extra))


def test_golden_covers_the_cases(gold):
    names = {r["case"] for r in gold["nll"]}
    assert names == set(gmd.CASES)
    assert {r["case"] for r in gold["fit"]} == {"crossed", "nested", "three", "strings"}
    assert any(r["case"] == "tridiag_cap" and r["cg_its_tridiag"] == 4 for r in gold["nll"])  # stops on cg_max_num_it_tridiag


def test_iterative_negll_and_iterations_match_reference(gold):
    for rec in gold["nll"]:
        o = oracle_eval(rec["case"], rec["cov_pars"])
        assert abs(o["negll"] - rec["negll"]) <= 1e-8 * abs(rec["negll"]), (rec, o["negll"])
        assert o["its"] == rec["cg_its"], rec
        assert o["its_tridiag"] == rec["cg_its_tridiag"], rec


def test_exact_negll_matches_reference_cholesky(gold):
    for rec in gold["nll"]:
        group, y, _ = gmd.case(rec["case"])
        d = gm.dense_negll(group, y, rec["cov_pars"])
        assert abs(d["negll"] - rec["negll_cholesky"]) <= 1e-10 * abs(rec["negll_cholesky"]), rec


def test_level_map_is_first_appearance_per_factor():
    group = np.array([["b", "x"], ["a", "x"], ["b", "y"], ["c", "x"]])
    st = gm.Structure(group)
    assert [list(i) for i in st.idx] == [[0, 1, 0, 2], [0, 0, 1, 0]]
    assert st.levels == [3, 2] and st.G == 5
    # off-diagonal block of Z^T Z: co-occurrence counts
    assert st.ZtZ[0, 3] == 1 and st.ZtZ[0, 4] == 1 and st.ZtZ[1, 3] == 1 and st.ZtZ[2, 3] == 1
