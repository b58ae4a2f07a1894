"""The factor-derivative passes and the Fisher-information contraction row by row against a long-double reference with per-row
error bounds.

vecchia_factor_kernel has two modes that store the derivative of the factor for other kernels to consume:
  * MODE_STORE_GRAD (read back with gpbdev_vecchia_latent_factor_grad): the latent factor of the Laplace-Vecchia likelihoods (no
    nugget, jitter var 1e-10 on the neighbour diagonal) with dA, dD w.r.t. log range;
  * MODE_STORE_GRAD2 (read back with gpbdev_vecchia_gaussian_factor_grad, launched by the routine of gpbdev_vecchia_fisher_info):
    the Gaussian factor with dA_k, dD_k w.r.t. log var (k = 0, by the device's identities S^-1 A and D - 1 - A.A) and log range
    (k = 1).

Reference: oracle.vecchia.rows_dfactor_ld (oracle/vecchia_oracle.c: orc_vecchia_rows_dfactor_ld) evaluates every row in long double
from the fp64 inputs by the generic formula dA_k = S^-1 (g_k - G_k A), dD_k = b^T G_k b (b = [-A, 1]) for both parameters, with
first-order bounds of an fp64 evaluation: entrywise for dA_k, |S^-1| applied to the perturbation of S (E of oracle.vecchia.rows_ld),
the bound of A propagated through |G_k|, the evaluation errors of the derivative entries (closed form, distance and coordinate
rounding through |dG_k/dr|), the rounding of G_k b and the backward error of the two substitutions; per row for dD_k,
kappa (eps + rho_k) times its magnitude. Where a pair's exponent exceeds 700 the evaluation errors also take exp(-700) times the
factor in front of the exp: the kernels' exp(-x) saturates there (exp_neg), an absolute error near 1e-300 that only entries far
below the fp64 range can see (rows of far neighbours at d = 1, and the Gaussian kernel). A and D^-1 are checked against oracle.vecchia.rows_ld. Every comparison is
|device - reference| <= C_BOUND * bound with the C_BOUND = 4 of tests/test_vecchia_rows_gpu.py.

The Fisher contraction (fi_contract_kernel after the solves and products of fisher.cuh) is checked against a long-double restatement
built from the device's own A, D^-1, dA_k, dD_k and the same probe block Z:
  V1 = B^-T Z,  V2 = B^-1 D V1,  U0 = D^-1 B Z,  Y_k = -dA_k V2,  H_k = D^-1 (Y_k - dD_k V1),
  T_0 = B^T U0,  T_k = B^T H_k - dA_k^T V1,  FI_ab = fac_a fac_b sum T_a .* T_b / (2 t)
with the original-scale factors fac of fisher.cuh. The bar of every entry propagates the solve and product bars of
tests/test_laplace_kernels_gpu.py into T_a and adds the n t summation (per-warp partials, the column reduction and the host sum over
column blocks: 2 gamma(n + t) sum |T_a T_b|) and the final scaling; every entry is compared against its own bar.

CPU tests (no gpu mark): the reference against 50-digit mpmath (coincident and near points, q < m, -1 tails, latent rows); the fp64
oracle (ov.factor with calc_grad, oracle.laplace.factor_latent_grad) inside the bounds at every row; four deliberate faults down to a
relative 1e-10 rejected; the bounds tight; the cases reaching every (kernel, DIM, cap) bucket of the derivative modes. GPU tests run
at n = 13001 (at least three rows per warp at grid_cap), and the Fisher contraction on the engine's own neighbour sets and on the
chain, star, column-count and comb patterns of the Laplace suite, at t around the 32-column groups and the 128-column blocks."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import laplace as ol
from oracle import std_err as ose
from oracle import vecchia as ov
from test_laplace_kernels_gpu import COL_COUNTS, LD, Ref, chain_nn, col_counts, colcount_nn, comb_nn, gamma, star_nn
from test_laplace_kernels_gpu import case_coords as pattern_coords
from test_vecchia_kernels_gpu import MODE_STORE, MODE_STORE_GRAD, STORE_GRAD_BUCKETS, kernel_bucket, spread_range
from test_vecchia_rows_gpu import C_BOUND, N_ROWS, P, U, case_data, chk, create, eval_pass, get_factor, mp_rows, pars, ratio

if np.finfo(np.longdouble).eps > 1e-18:
    pytest.skip("long double has no extended precision on this host", allow_module_level=True)

MODE_STORE_GRAD2 = 4
LATENT_VAR = 0.7
# MODE_STORE_GRAD2 at every (DIM, cap) and every covariance at d = 2, cap 30 (an instantiation of the derivative modes only)
GRAD2_CASES = [(2, 10, "matern1.5"), (2, 20, "matern2.5")] + [(2, 30, c) for c in ("exponential", "matern1.5", "matern2.5", "gaussian")]
GRAD2_CASES += [(1, 15, "exponential"), (5, 8, "gaussian"), (3, 30, "matern1.5")]
# MODE_STORE_GRAD at every (DIM, cap)
LATENT_CASES = [(2, 10, "matern1.5"), (2, 20, "exponential"), (2, 30, "matern1.5"), (2, 30, "matern2.5"), (1, 15, "matern1.5"),
                (5, 8, "exponential"), (3, 30, "gaussian")]
# Fisher contraction: (pattern, n, d, m, cov id, t); "knn" = the engine's own neighbour search
FISHER_CASES = [("knn", N_ROWS, 2, 20, 1, t) for t in (1, 50, 129)]
FISHER_CASES += [(p, n, 2, m, cid, t) for (p, n, m, cid) in (("chain", 3000, 1, 0), ("star", 3000, 5, 1), ("cols", 800, 2, 1),
                                                              ("comb", 3000, 30, 2))
                 for t in (32, 33, 128, 129, 300)]


def family_of(d, m):
    kern, dim, cap = kernel_bucket(d, m, MODE_STORE_GRAD2)
    return "%s-%s-cap%d" % (kern, "d2" if dim == 2 else "gen", cap)


def spaced_coords(n, d, seed):
    """n points of a jittered grid in [0, 1]^d: one per chosen cell of width 1/k, at most half a cell from its corner, so that two
    points are at least 1/(2k) apart. Without a nugget the latent neighbour blocks of arbitrarily close points are singular to
    fp64 (see test_vecchia_kernels_gpu.latent_coords), and their bounds would say nothing."""
    rng = np.random.default_rng(seed)
    k = int(math.ceil(n ** (1. / d)))
    cells = rng.choice(k ** d, size=n, replace=False)
    idx = np.stack(np.unravel_index(cells, (k,) * d), axis=1)
    return (idx + 0.5 * rng.random((n, d))) / k


def latent_data(n, d, m, variant, seed):
    """Vecchia-ordered spaced points, the ordering, and supplied sets with the -1 tails of case_data for 'tails' (None: searched)"""
    rng = np.random.default_rng(seed)
    perm = ov.random_order(n, seed)
    co = np.ascontiguousarray(spaced_coords(n, d, seed)[perm])
    nn = None
    if variant == "tails":
        nn = ov.knn(co, m)
        for i in rng.choice(np.arange(m, n), size=n // 10, replace=False):
            nn[i, rng.integers(1, m):] = -1
        c0 = n // 2
        for i in range(c0, c0 + m):
            nn[i, i - c0:] = -1
    return co, perm, nn


def latent_pars(cov, n, d):
    cf, shape = {"exponential": ("exponential", 0.5), "matern1.5": ("matern", 1.5), "matern2.5": ("matern", 2.5),
                 "gaussian": ("gaussian", 0.)}[cov]
    _, pt = ov.transform_cov_pars([1.0, LATENT_VAR, spread_range(n, d)], cf, shape)
    return ov.cov_id(cf, shape), LATENT_VAR, pt[1]


def gauss_ref(co, nn, cid, var, rg, **faults):
    r, dA, bdA, bad = ov.rows_dfactor_ld(co, nn, cid, var, rg, var + 1., var + 1., **faults)
    assert bad == 0
    return r, dA, bdA


def latent_ref(co, nn, cid, var, rg, **faults):
    r, dA, bdA, bad = ov.rows_dfactor_ld(co, nn, cid, var, rg, var * (1. + 1e-10), var, **faults)
    assert bad == 0
    return r, dA, bdA


def deriv_ratios(dev, r, dA, bdA, ks):
    """largest ratio per derivative quantity; dev holds dA<k> (n, m) and dD<k> (n) for k in ks"""
    out = {}
    for k in ks:
        if "dA%d" % k in dev:
            out["dA%d" % k] = ratio(dev["dA%d" % k], dA[k], bdA[k])
        if "dD%d" % k in dev:
            out["dD%d" % k] = ratio(dev["dD%d" % k], r["dD%d" % k], r["bdD%d" % k])
    return out


# ---------------------------------------------------------------------------------------------------------- CPU-only
@pytest.mark.parametrize("cov", ["exponential", "matern1.5", "matern2.5", "gaussian"])
def test_long_double_derivatives_match_mpmath(cov):
    """Gaussian rows (q < m, a neighbour coinciding with the row's point, a neighbour 1e-9 away, a row truncated to 4 neighbours)
    and latent rows on spaced points (q < m, a -1 tail): dA_k and dD_k of both parameters agree with 50-digit mpmath to a
    hundredth of the fp64 bound"""
    tol = 1e-2 / C_BOUND
    n, d, m = 80, 2, 10
    cid, _, pt = pars(cov, n, d)
    rng = np.random.default_rng(5)
    co = rng.random((n, d))
    co[41] = co[17]  # coincident
    co[52] = co[23] + 1e-9  # near
    nn = ov.knn(co, m)
    nn[60, 4:] = -1
    assert 17 in nn[41] and 23 in nn[52]
    lco, _, lnn = latent_data(n, d, m, "tails", 6)
    lnn[70, 3:] = -1
    lcid, lvar, lrg = latent_pars(cov, n, d)
    cases = [(co, nn, cid, pt[0], pt[1], pt[0] + 1., pt[0] + 1., [0, 1, 2, 5, 9, 10, 20, 41, 52, 60, 75, 79]),
             (lco, lnn, lcid, lvar, lrg, lvar * (1. + 1e-10), lvar, [1, 3, 9, 10, 40, 70, 79])]
    for co_, nn_, cid_, var, rg, dn, do, rows in cases:
        for i in rows:
            r, dA, bdA, bad = ov.rows_dfactor_ld(co_, nn_[i:i + 1], cid_, var, rg, dn, do, i)
            assert bad == 0
            want = mp_rows(co_, nn_[i:i + 1], cid_, var, rg, dn, do, np.zeros(n), [i])[0]
            for k in range(2):
                a_mp = np.zeros(m)
                a_mp[nn_[i] >= 0] = [float(v) for v in want["dA"][k]]
                assert ratio(dA[k, 0], a_mp, tol * bdA[k, 0]) <= 1., (i, k, dA[k, 0], a_mp)
                assert ratio(r["dD%d" % k], float(want["dD"][k]), tol * r["bdD%d" % k]) <= 1., (i, k)


CPU_CASES = [(1500, d, m, cov, v) for (d, m) in ((2, 25), (3, 30), (1, 15)) for cov in ("exponential", "matern1.5", "matern2.5",
                                                                                         "gaussian") for v in ("unif", "tails", "near")]


@pytest.mark.parametrize("case", CPU_CASES, ids=["n%d-d%d-m%d-%s-%s" % c for c in CPU_CASES])
def test_fp64_oracle_within_bounds(case):
    """ov.factor(calc_grad=True) (libm exp, differences before scaling, the generic formula in fp64) for the Gaussian pair, and
    oracle.laplace.factor_latent_grad on spaced points for the latent range pair, at every row"""
    n, d, m, cov, variant = case
    co, perm, y, nn = case_data(n, d, m, variant, 7 + d)
    nn = ov.knn(co, m) if nn is None else nn
    cid, _, pt = pars(cov, n, d)
    r, dA, bdA = gauss_ref(co, nn, cid, pt[0], pt[1])
    _, _, Ag, Dg, bad = ov.factor(co, nn, cid, pt, calc_grad=True)
    assert bad == 0
    worst = deriv_ratios({"dA0": Ag[0], "dA1": Ag[1], "dD0": Dg[0], "dD1": Dg[1]}, r, dA, bdA, (0, 1))
    assert max(worst.values()) <= 1., worst
    if variant == "near":
        return
    lco, _, lnn = latent_data(n, d, m, variant, 8 + d)
    lnn = ov.knn(lco, m) if lnn is None else lnn
    lcid, lvar, lrg = latent_pars(cov, n, d)
    r, dA, bdA = latent_ref(lco, lnn, lcid, lvar, lrg)
    _, _, Ag, Dg, bad = ol.factor_latent_grad(lco, lnn, lcid, lvar, lrg)
    assert bad == 0
    worst = deriv_ratios({"dA1": Ag, "dD1": Dg}, r, dA, bdA, (1,))
    assert max(worst.values()) <= 1., worst


FAULT_CASES = [(1500, 2, 25, cov) for cov in ("exponential", "matern1.5", "matern2.5", "gaussian")] + [(1500, 3, 30, "matern1.5")]
FAULTS = [("range_mult", 1e-8), ("range_mult", 1e-10), ("drop_pair", None), ("jitter_leak", None), ("nugget", 1e-8),
          ("nugget", 1e-10)]


def rejected_by(fault, delta, case):
    """largest ratio of the faulted reference (standing in for a device) over the clean one's bounds, over all rows"""
    n, d, m, cov = case
    if fault == "jitter_leak":  # the latent factor, where the jitter exists
        co, _, nn = latent_data(n, d, m, "unif", 30 + d)
        nn = ov.knn(co, m)
        cid, var, rg = latent_pars(cov, n, d)
        ref = lambda **kw: latent_ref(co, nn, cid, var, rg, **kw)
        kw, ks = {"g1_diag": var * 1e-10}, (1,)
    else:
        co, _, _, _ = case_data(n, d, m, "unif", 30 + d)
        nn = ov.knn(co, m)
        cid, _, pt = pars(cov, n, d)
        ref = lambda **kw: gauss_ref(co, nn, cid, pt[0], pt[1], **kw)
        i = n // 3
        kw = {"range_mult": {"range_mult": 1. + (delta or 0.)}, "drop_pair": {"drop": (i, 0, int(np.sum(nn[i] >= 0)))},
              "nugget": {"g0_shift": delta}}[fault]
        ks = (0,) if fault == "nugget" else (1,)
    r, dA, bdA = ref()
    rf, dAf, _ = ref(**kw)
    dev = {}
    for k in ks:
        dev["dA%d" % k], dev["dD%d" % k] = dAf[k], rf["dD%d" % k]
    return max(deriv_ratios(dev, r, dA, bdA, ks).values())


@pytest.mark.parametrize("fault,delta", FAULTS, ids=["%s-%s" % (f, d) for f, d in FAULTS])
def test_bounds_reject_deliberate_faults(fault, delta):
    """every range derivative entry off by a relative delta; one pair (nearest neighbour, own point) missing from one row's range
    derivative; the latent jitter var 1e-10 on the range derivative's neighbour diagonal; the variance derivative taken as
    Sigma~ - (1 - delta) I: each is rejected on at least one case"""
    worst = [rejected_by(fault, delta, c) for c in FAULT_CASES]
    assert max(worst) > 1., worst


def test_bounds_are_tight():
    """Matern 1.5 and exponential, d = 2, m = 30, n = 3001 (median kappa 51 and 31): the median C_BOUND bound / |value| stays within
    1e4 u kappa^2 for dA_k (entries above 1e-3 of the row's largest; the bound applies |S^-1| twice) and within 1e5 u kappa for
    dD_k, kappa the median of the rows; a later change cannot quietly loosen the bounds"""
    n, d, m = 3001, 2, 30
    co, perm, y, _ = case_data(n, d, m, "unif", 3)
    nn = ov.knn(co, m)
    for cov in ("matern1.5", "exponential"):
        cid, _, pt = pars(cov, n, d)
        r, dA, bdA = gauss_ref(co, nn, cid, pt[0], pt[1])
        kap = float(np.median(r["kappa"][1:]))
        med = {}
        for k in range(2):
            a, b = dA[k, 1:], bdA[k, 1:]
            big = np.abs(a) >= 1e-3 * np.abs(a).max(axis=1, keepdims=True)
            med["dA%d" % k] = float(np.median((C_BOUND * b / np.abs(np.where(big, a, 1.)))[big])) / (U * kap ** 2)
            med["dD%d" % k] = float(np.median(C_BOUND * r["bdD%d" % k][1:] / np.abs(r["dD%d" % k][1:]))) / (U * kap)
        print(cov, "median kappa %.3g, median C bound / |value| in units of u kappa^2 (dA) and u kappa (dD):" % kap, med)
        assert max(med["dA0"], med["dA1"]) <= 1e4 and max(med["dD0"], med["dD1"]) <= 1e5, med


def test_cases_reach_every_derivative_bucket():
    """the MODE_STORE_GRAD2 and MODE_STORE_GRAD cases run every (kernel, DIM, cap) of the derivative modes, including the d = 2 cap
    30 instantiation; n gives three rows per warp at grid_cap up to 135 SMs; the column-count pattern has columns of 7, 8, 9 and 64
    entries around fi_contract_kernel's 8-row batches and 32-entry chunks; t crosses the 32-column groups and the 128-column blocks"""
    assert {kernel_bucket(d, m, MODE_STORE_GRAD2) for d, m, _ in GRAD2_CASES} == STORE_GRAD_BUCKETS
    assert {kernel_bucket(d, m, MODE_STORE_GRAD) for d, m, _ in LATENT_CASES} == STORE_GRAD_BUCKETS
    assert ("one_obs", 2, 30) in STORE_GRAD_BUCKETS
    assert N_ROWS >= 3 * 32 * 135 + 1
    cc = set(col_counts(colcount_nn(800)))
    assert {7, 8, 9, 31, 32, 33, 64, 127, 128, 129} <= cc and {7, 8, 9, 64} <= set(COL_COUNTS)
    assert {t for c in FISHER_CASES for t in [c[5]]} >= {1, 32, 33, 128, 129, 300}
    assert {c[0] for c in FISHER_CASES} == {"knn", "chain", "star", "cols", "comb"}


# ---------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def lib(product_lib):
    assert product_lib.gpbdev_device_count() > 0, "no CUDA device visible — GPU tests need an H100"
    return product_lib


REPORT = {}


def record(family, what, value):
    key = (family, what)
    REPORT[key] = max(REPORT.get(key, 0.), value)


@pytest.fixture(scope="module", autouse=True)
def report_ratios():
    yield
    if REPORT:
        print("\nlargest |device - reference| / (C bound), C = %g" % C_BOUND)
        for (fam, what), v in sorted(REPORT.items()):
            print("  %-26s %-8s %.3g" % (fam, what, v))


def gaussian_factor_grad(lib, h, n, m, cid, var, rg):
    A, dA0, dA1 = np.empty((n, m)), np.empty((n, m)), np.empty((n, m))
    Dinv, dD0, dD1 = np.empty(n), np.empty(n), np.empty(n)
    chk(lib, lib.gpbdev_vecchia_gaussian_factor_grad(h, C.c_int(cid), C.c_double(var), C.c_double(rg), P(A), P(Dinv), P(dA0), P(dD0),
                                                     P(dA1), P(dD1)))
    return {"A": A, "Dinv": Dinv, "dA0": dA0, "dD0": dD0, "dA1": dA1, "dD1": dD1}


def latent_factor_grad(lib, h, n, m, cid, var, rg):
    A, dA1, Dinv, dD1 = np.empty((n, m)), np.empty((n, m)), np.empty(n), np.empty(n)
    chk(lib, lib.gpbdev_vecchia_latent_factor_grad(h, C.c_int(cid), C.c_double(var), C.c_double(rg), P(A), P(Dinv), P(dA1), P(dD1)))
    return {"A": A, "Dinv": Dinv, "dA1": dA1, "dD1": dD1}


def same_bits(a, b):
    return all(a[k].tobytes() == b[k].tobytes() for k in a)


def check_factor_rows(dev, co, nn, cid, var, rg, diag_nb, diag_obs, family, ks):
    """A and D^-1 against rows_ld, dA_k and dD_k against rows_dfactor_ld, at every row"""
    r0, A, bA, bad = ov.rows_ld(co, nn, cid, var, rg, diag_nb, diag_obs, None)
    assert bad == 0
    r, dA, bdA, bad = ov.rows_dfactor_ld(co, nn, cid, var, rg, diag_nb, diag_obs)
    assert bad == 0
    w = {"A": ratio(dev["A"], A, bA), "Dinv": ratio(dev["Dinv"], 1. / r0["D"], r0["bD"] / r0["D"] ** 2)}
    w.update(deriv_ratios(dev, r, dA, bdA, ks))
    for k, v in w.items():
        record(family, k, v)
    assert max(w.values()) <= 1., w


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["unif", "tails", "near"])
@pytest.mark.parametrize("case", GRAD2_CASES, ids=["d%d-m%d-%s" % c for c in GRAD2_CASES])
def test_gaussian_factor_derivatives_match_long_double(lib, case, variant):
    """MODE_STORE_GRAD2 through gpbdev_vecchia_gaussian_factor_grad at n = 13001: A, D^-1, dA_0, dD_0, dA_1, dD_1 at every row; a
    second call is bitwise the same; after a STORE pass the entry leaves the engine's factor, its sums and its STORE shortcut as
    they were"""
    d, m, cov = case
    n = N_ROWS
    co, perm, y, nn = case_data(n, d, m, variant, 400 + d * 61 + m)
    cid, _, pt = pars(cov, n, d)
    var, rg = pt
    h = create(lib, co, perm, m, nn)
    try:
        nn_d = np.empty((n, m), dtype=np.int32)
        chk(lib, lib.gpbdev_vecchia_get_nn(h, P(nn_d, C.c_int32)))
        if nn is not None:
            assert np.array_equal(nn_d, nn)
        chk(lib, lib.gpbdev_vecchia_set_y(h, P(np.ascontiguousarray(y))))
        sums = eval_pass(lib, h, cid, var, 1.3 * rg, MODE_STORE)
        stored = get_factor(lib, h, n, m)
        dev = gaussian_factor_grad(lib, h, n, m, cid, var, rg)
        assert same_bits(dev, gaussian_factor_grad(lib, h, n, m, cid, var, rg))
        k = lib.gpbdev_vecchia_launch_count(h)
        assert np.array_equal(eval_pass(lib, h, cid, var, 1.3 * rg, MODE_STORE), sums)
        assert lib.gpbdev_vecchia_launch_count(h) == k
        assert all(a.tobytes() == b.tobytes() for a, b in zip(get_factor(lib, h, n, m), stored))
        check_factor_rows(dev, co, nn_d, cid, var, rg, var + 1., var + 1., "grad2 " + family_of(d, m), (0, 1))
    finally:
        lib.gpbdev_vecchia_free(h)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["unif", "tails"])
@pytest.mark.parametrize("case", LATENT_CASES, ids=["d%d-m%d-%s" % c for c in LATENT_CASES])
def test_latent_factor_derivative_matches_long_double(lib, case, variant):
    """MODE_STORE_GRAD through gpbdev_vecchia_latent_factor_grad at n = 13001 on spaced points: A, D^-1, dA_1, dD_1 at every row;
    a second call is bitwise the same"""
    d, m, cov = case
    n = N_ROWS
    co, perm, nn = latent_data(n, d, m, variant, 600 + d * 61 + m)
    cid, var, rg = latent_pars(cov, n, d)
    h = create(lib, co, perm, m, nn)
    try:
        nn_d = np.empty((n, m), dtype=np.int32)
        chk(lib, lib.gpbdev_vecchia_get_nn(h, P(nn_d, C.c_int32)))
        if nn is not None:
            assert np.array_equal(nn_d, nn)
        dev = latent_factor_grad(lib, h, n, m, cid, var, rg)
        assert same_bits(dev, latent_factor_grad(lib, h, n, m, cid, var, rg))
        check_factor_rows(dev, co, nn_d, cid, var, rg, var * (1. + 1e-10), var, "latent " + family_of(d, m), (1,))
    finally:
        lib.gpbdev_vecchia_free(h)


@pytest.mark.gpu
def test_gaussian_factor_grad_refuses_what_fisher_info_refuses(lib):
    """null buffers, an unknown covariance id, non-positive parameters, a row-sharded engine and m > 30, with the message of
    gpbdev_vecchia_fisher_info"""
    n, d = 300, 2
    co, perm, _, _ = case_data(n, d, 10, "unif", 1)
    h, hs, hb = create(lib, co, perm, 10, None), create(lib, co, perm, 10, ov.knn(co, 10), 0, 150), create(lib, co, perm, 31, None)
    try:
        buf = np.empty(n * 31)
        Z = np.asfortranarray(np.ones((n, 2)))
        FI = np.empty(9)
        f, g = lib.gpbdev_vecchia_gaussian_factor_grad, lib.gpbdev_vecchia_fisher_info
        cases = [(h, 1, 1., 5., "null argument", True), (h, 4, 1., 5., "unknown covariance id", False),
                 (h, -1, 1., 5., "unknown covariance id", False), (h, 1, 0., 5., "covariance parameters must be positive", False),
                 (h, 1, 1., -5., "covariance parameters must be positive", False),
                 (hs, 1, 1., 5., "row-sharded engines are not supported", False), (hb, 1, 1., 5., "num_neighbors must be <= 30", False)]
        for hh, cid, var, rg, msg, null in cases:
            bufs = [P(buf)] * 6
            if null:
                bufs[3] = None
            assert f(hh, cid, C.c_double(var), C.c_double(rg), *bufs) != 0
            assert lib.gpbdev_last_error().decode() == "gpbdev_vecchia_gaussian_factor_grad: " + msg
            if not null:
                assert g(hh, cid, C.c_double(0.5), C.c_double(var), C.c_double(rg), P(Z), 2, P(FI)) != 0
                assert lib.gpbdev_last_error().decode() == "gpbdev_vecchia_fisher_info: " + msg
    finally:
        for hh in (h, hs, hb):
            lib.gpbdev_vecchia_free(hh)


def fisher_nn(pattern, n, m):
    return {"chain": lambda: chain_nn(n), "star": lambda: star_nn(n, m), "cols": lambda: colcount_nn(n),
            "comb": lambda: comb_nn(n, m)}[pattern]()


def fisher_pars(pattern, n, d, cid):
    """(sigma2, var, transformed range, original-scale range rho): the range of the Laplace suite's case_pars"""
    rho = {"knn": 2. * n ** (-1. / d), "chain": 50. / n}.get(pattern, 0.5)
    rt = 1. / rho ** 2 if cid == 3 else {0: 1., 1: np.sqrt(3.), 2: np.sqrt(5.)}[cid] / rho
    return 0.3, 0.7 / 0.3, rt, rho


def fisher_reference(nn, dev, Z, fac):
    """FI (3 x 3) and the bar of every entry, in long double from the device's factor and derivatives (module docstring)"""
    n, t = Z.shape
    R = Ref(nn, dev["A"], dev["Dinv"], dev["dA0"], np.zeros(n), scipy_solves=n > 20000)
    c2 = 4. if R.scipy else 2.
    gr, gc = gamma(R.krow + 3)[:, None], gamma(R.kcol + 3)[:, None]
    ZL, Dv = Z.astype(LD), R.Dinv[:, None]
    V1 = R.bwd(ZL)
    b_V1 = c2 * R.bwd(gc * R.absBt(V1), absA=True)
    V2 = R.fwd(V1 / Dv)
    b_V2 = c2 * R.fwd(gr * R.absB(V2) + (U * np.abs(V1) + b_V1) / Dv, absA=True)
    U0 = Dv * (ZL - R.gather(R.A, ZL))
    b_U0 = 2. * gr * Dv * R.absB(ZL)
    T = [U0 - R.scatter(R.a_e(R.A), U0)]
    bT = [R.absBt(b_U0) + 2. * gc * R.absBt(U0)]
    for k in range(2):
        dAk = np.where(R.mask, dev["dA%d" % k], 0.).astype(LD)
        adA = np.abs(dAk)
        dDk = dev["dD%d" % k].astype(LD)[:, None]
        Y = -R.gather(dAk, V2)
        b_Y = 2. * gr * R.gather(adA, np.abs(V2)) + R.gather(adA, b_V2)
        H = Dv * (Y - dDk * V1)
        b_H = Dv * (b_Y + np.abs(dDk) * b_V1) + 2. * gamma(4) * Dv * (np.abs(Y) + np.abs(dDk * V1))
        T.append(H - R.scatter(R.a_e(R.A), H) - R.scatter(R.a_e(dAk), V1))
        bT.append(R.absBt(b_H) + R.scatter(R.a_e(adA), b_V1) + 2. * gc * (R.absBt(H) + R.scatter(R.a_e(adA), np.abs(V1))))
    FI, bar = np.zeros((3, 3), dtype=LD), np.zeros((3, 3), dtype=LD)
    for a in range(3):
        for b in range(a, 3):
            f = LD(fac[a]) * LD(fac[b]) / LD(2 * t)
            v = (T[a] * T[b]).sum() * f
            mag = (np.abs(T[a] * T[b])).sum()
            bb = ((np.abs(T[a]) * bT[b]).sum() + (bT[a] * np.abs(T[b])).sum() + 2. * gamma(n + t) * mag) * abs(f) + 8. * U * abs(v)
            FI[a, b] = FI[b, a] = v
            bar[a, b] = bar[b, a] = bb
    return FI, bar


@pytest.mark.gpu
@pytest.mark.parametrize("case", FISHER_CASES, ids=["%s-n%d-d%d-m%d-cov%d-t%d" % c for c in FISHER_CASES])
def test_fisher_contraction_matches_long_double(lib, case):
    """gpbdev_vecchia_fisher_info against the long-double restatement from the device's own factor and derivatives (read back
    with gpbdev_vecchia_gaussian_factor_grad) and the same probe block: every one of the 9 entries within its own bar"""
    pattern, n, d, m, cid, t = case
    if pattern == "knn":
        co, perm, _, _ = case_data(n, d, m, "unif", 800 + t)
        nn = None
    else:
        co = pattern_coords(pattern + "-fisher", n, d, pattern)
        perm = np.arange(n, dtype=np.int32)
        nn = np.ascontiguousarray(fisher_nn(pattern, n, m), dtype=np.int32)
        m = nn.shape[1]
    s2, var, rt, rho = fisher_pars(pattern, n, d, cid)
    fac = [1. / s2, -1. / (s2 * var), (2. if cid == 3 else 1.) / rho]
    Z = ose.probes(n, t, 1, 0)
    h = create(lib, co, perm, m, nn)
    try:
        nn_d = np.empty((n, m), dtype=np.int32)
        chk(lib, lib.gpbdev_vecchia_get_nn(h, P(nn_d, C.c_int32)))
        dev = gaussian_factor_grad(lib, h, n, m, cid, var, rt)
        FI = np.empty(9)
        chk(lib, lib.gpbdev_vecchia_fisher_info(h, cid, C.c_double(s2), C.c_double(var), C.c_double(rt), P(np.asfortranarray(Z)), t,
                                                P(FI)))
    finally:
        lib.gpbdev_vecchia_free(h)
    want, bar = fisher_reference(nn_d, dev, Z, fac)
    family = "fisher " + pattern
    for a in range(3):
        for b in range(a, 3):
            rr = ratio(FI[3 * a + b], float(want[a, b]), float(bar[a, b]))
            record(family, "FI%d%d" % (a, b), rr)
            assert rr <= 1., (a, b, FI[3 * a + b], float(want[a, b]), float(bar[a, b]))
