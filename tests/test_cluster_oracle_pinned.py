"""The per-cluster restatement (tests/cluster_oracle.py) reproduces the unmodified reference library's likelihood of models with
cluster_ids (tests/golden/cluster_golden.json) for the cases with ordering 'none', whose rows stay in data order within every cluster:
its neighbour sets (the oracle's search of each cluster alone, head rows included) and factors are the reference's. The GPU tests then
compare the device's neighbour sets, factor and gradient against this restatement."""
import json
import os

import numpy as np
import pytest

import cluster_cases as cc
import cluster_oracle as co

GOLDEN = {r["name"]: r for r in json.load(open(os.path.join(os.path.dirname(__file__), "golden", "cluster_golden.json")))["cases"]}


@pytest.mark.parametrize("c", [c for c in cc.CASES if c["ordering"] == "none"], ids=lambda c: c["name"])
def test_restatement_matches_reference_likelihood(c):
    coords, y, lab, _, _ = cc.case_data(c)
    r = co.clustered(coords, lab, y, c["m"], c["cov"], c["shape"], cc.COV_PARS)
    g = GOLDEN[c["name"]]["nll"]
    assert abs(r["negll"] - g) <= 1e-8 * abs(g), (r["negll"], g)
    # the caps: a cluster of c points keeps at most c - 1 neighbours, its first min(c, m + 1) rows take all their predecessors
    for rows, nn, _, _ in r["parts"]:
        nc = len(rows)
        assert nn.shape[1] == max(1, min(c["m"], nc - 1))
        for i in range(min(nc, c["m"] + 1)):
            assert list(nn[i, :i]) == list(range(i)) and np.all(nn[i, i:] == -1)


def test_restatement_distinguishes_clusters():
    """the same data as one realization gives another likelihood: the golden pins the block structure, not only the data"""
    c = cc.CASES[0]
    coords, y, lab, _, _ = cc.case_data(c)
    one = co.clustered(coords, np.zeros_like(lab), y, c["m"], c["cov"], c["shape"], cc.COV_PARS)["negll"]
    assert abs(one - GOLDEN[c["name"]]["nll"]) > 1e-3 * abs(one)
