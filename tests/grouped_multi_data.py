"""Seeded data for the multi-level grouped random-effects tests and their golden file (tests/golden/make_grouped_multi_golden.py)."""
import numpy as np

# name -> (kind, kwargs, iterative settings passed through set_optim_params)
CASES = {
    "crossed": ("crossed", dict(n=3000, G1=300, G2=40, seed=1), {}),
    "nested": ("nested", dict(n=2400, schools=30, classes=6, seed=2), {}),
    "three": ("three", dict(n=2500, G=(80, 25, 7), seed=3), {}),
    "strings": ("strings", dict(n=1500, G1=90, G2=15, seed=4), {}),
    "tridiag_cap": ("crossed", dict(n=3000, G1=300, G2=40, seed=1), {"cg_max_num_it_tridiag": 4}),
    "probes": ("crossed", dict(n=3000, G1=300, G2=40, seed=1), {"num_rand_vec_trace": 20, "seed_rand_vec_trace": 7}),
}
COV_PARS = {2: ([0.6, 1.1, 0.4], [1.3, 0.2, 0.9]), 3: ([0.5, 1.0, 0.3, 0.7], [1.1, 0.4, 1.6, 0.2])}


def make(kind, kw):
    """(group n x K, y). Crossed levels are unbalanced (a Zipf-like draw) and include singleton levels."""
    rng = np.random.default_rng(kw["seed"])
    n = kw["n"]
    if kind in ("crossed", "strings"):
        G1, G2 = kw["G1"], kw["G2"]
        w = 1. / np.arange(1, G1 + 1) ** 0.8
        g1 = rng.choice(G1 - 10, size=n - 10, p=w[:G1 - 10] / w[:G1 - 10].sum())
        g1 = np.concatenate([g1, np.arange(G1 - 10, G1)])  # ten singleton levels
        g2 = rng.integers(0, G2, size=n)
        group = np.c_[g1, g2]
    elif kind == "nested":
        school = rng.integers(0, kw["schools"], size=n)
        cls = school * kw["classes"] + rng.integers(0, kw["classes"], size=n)
        group = np.c_[school, cls]
    else:
        group = np.c_[tuple(rng.integers(0, g, size=n) for g in kw["G"])]
    K = group.shape[1]
    sd = [1.0, 0.6, 0.8][:K]
    y = 0.7 * rng.standard_normal(n)
    for k in range(K):
        y += sd[k] * rng.standard_normal(group[:, k].max() + 1)[group[:, k]]
    if kind == "strings":
        group = np.array([["lvl%d_%s" % (k, chr(97 + v % 26) * (1 + v // 26)) for k, v in enumerate(row)] for row in group])
    return group, y


def case(name):
    kind, kw, it = CASES[name]
    group, y = make(kind, kw)
    return group, y, it


def boost_case():
    """GPBoost data: tree signal plus two crossed random effects."""
    rng = np.random.default_rng(21)
    n, F = 4000, 5
    X = rng.random((n, F))
    f = 2 * np.sin(3 * X[:, 0]) + X[:, 1] ** 2 + 0.5 * (X[:, 2] > 0.6)
    g1 = rng.integers(0, 150, size=n)
    g2 = rng.integers(0, 30, size=n)
    y = f + 0.3 * rng.standard_normal(n) + rng.standard_normal(150)[g1] + 0.5 * rng.standard_normal(30)[g2]
    return X, y, np.c_[g1, g2]


BOOST_PARAMS = {"objective": "regression", "num_leaves": 8, "min_data_in_leaf": 20, "learning_rate": 0.1, "max_bin": 255, "verbose": -1}
BOOST_FIXED_COV_PARS = [0.1, 0.9, 0.2]
