"""The Vecchia factor passes row by row against a long-double reference with per-row error bounds.

Reference: oracle.vecchia.rows_ld (oracle/vecchia_oracle.c: orc_vecchia_rows_ld) evaluates every row's distances, covariances and
augmented Cholesky in long double from the fp64 inputs and returns, per row, D_i, A_i, (By)_i, u_i = (By)_i / D_i, the six GRAD
accumulator terms (kNumAcc slots 3..8) and first-order bounds of what an fp64 evaluation of the row may differ by:

  * E, an entrywise perturbation of the augmented matrix: covariance evaluation (c_v u |Sigma_ab|), distance rounding
    (c_r u r_ab |dSigma/dr|), rounding of the coordinates themselves (sqrt(d) u (|x_a|_inf + |x_b|_inf) |dSigma/dr|: the
    two-observation kernel pre-scales the points by the range before it takes differences, the others take differences first;
    both lose this much), and the Cholesky backward error gam(q + 2) sqrt(St_aa St_bb);
  * beta_D = |b|^T E |b| (b = [-A_i, 1]), beta_By = |b|^T E |w~| (w~ = [S^-1 y_N, 0]) plus the rounding of the y column,
    beta_A = |S^-1| (E_N. |b|); log D, 1/D, u and (By)^2 / D take the first-order bounds that follow from these;
  * the GRAD terms take kappa_i (eps_i + rho_i) times the term with every factor in absolute value (kappa_i: 1-norm condition
    number of the row's neighbour block, an upper bound of the 2-norm one; eps_i = max_ab E_ab / sqrt(St_aa St_bb); rho_i the
    largest relative evaluation error of one of the row's covariances, which eps_i does not see when a covariance is tiny).

A sum's bound is the sum of its rows' bounds plus (ceil(rows / accumulators) + 16) u sum |terms| for the fp64 summation
(accumulators: a lower bound of the per-warp partial rows of any family, min(2 SMs, rows / 8)). Every comparison is
|device - reference| <= C_BOUND * bound with one constant C_BOUND = 4.

CPU tests (no gpu mark) check the reference against mpmath, that the fp64 oracle (libm exp, no pre-scaling: a different route
from the kernels) stays inside the bounds, that three subtle faults are rejected, and that the bounds stay tight. GPU tests run
the kernels in the multi-row regime (n >= 3 * 32 * SMs + 1: at least three rows or pairs per warp for every family), on row
shards (0..5, 31..33 and 4097 rows, odd row_begin) and for prediction (BIG_PRED)."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import vecchia as ov
from test_vecchia_kernels_gpu import ALL_BUCKETS, MODE_GRAD, MODE_NLL, MODE_STORE, P, chk, kernel_bucket, spread_range

if np.finfo(np.longdouble).eps > 1e-18:
    pytest.skip("long double has no extended precision on this host", allow_module_level=True)

C_BOUND = 4.
U = 2. ** -53
CP = [0.4, 1.3]  # error variance, marginal variance; the range is spread_range(n, d)
COVS = {"exponential": ("exponential", 0.5), "matern1.5": ("matern", 1.5), "matern2.5": ("matern", 2.5), "gaussian": ("gaussian", 0.)}
VARIANTS = ["unif", "tails", "near"]
N_ROWS = 13001

# multi-row cases (d, m, cov): the two-observation kernel at every m of its band for Matern-1.5 and at three for the others, the
# one-observation kernel at each (DIM, cap) and the big kernel at d = 2 and 3
MULTI_CASES = [(2, m, "matern1.5") for m in range(21, 31)]
MULTI_CASES += [(2, m, c) for c in ("exponential", "matern2.5", "gaussian") for m in (21, 25, 30)]
MULTI_CASES += [(2, 10, "matern1.5"), (2, 20, "matern1.5"), (3, 30, "matern1.5"), (1, 15, "matern1.5"), (5, 8, "matern1.5")]
MULTI_CASES += [(2, 45, "matern1.5"), (3, 60, "matern1.5")]

SHARD_LENGTHS = [1, 0, 2, 3, 4, 5, 31, 32, 33, 4097]  # a 1-row shard first: the following ones begin at odd rows
SHARD_CASES = [(2, 30, "matern1.5"), (2, 30, "gaussian"), (3, 20, "matern1.5"), (2, 45, "matern1.5")]


def pars(cov, n, d):
    cf, shape = COVS[cov]
    s2, pt = ov.transform_cov_pars(CP + [spread_range(n, d)], cf, shape)
    return ov.cov_id(cf, shape), s2, pt


def case_data(n, d, m, variant, seed):
    """Vecchia-ordered coordinates, the ordering, y (original order) and supplied neighbour sets (None: searched by the engine).
    unif: U[0,1]^d. tails: supplied sets with -1 tails at scattered rows >= m and, in the middle of the table, a block of rows
    with 0..m-1 neighbours (the first rows of a cluster of cluster_ids). near: a quarter of the points repeat others 1e-9 apart,
    where the coordinate-rounding term of E dominates."""
    rng = np.random.default_rng(seed)
    if variant == "near":
        base = rng.random((n - n // 4, d))
        coords = np.concatenate([base, base[:n // 4] + 1e-9 * rng.random((n // 4, d))])
    else:
        coords = rng.random((n, d))
    y = rng.standard_normal(n) * 0.5 + np.sin(4 * coords[:, 0])
    perm = ov.random_order(n, seed)
    co = np.ascontiguousarray(coords[perm])
    nn = None
    if variant == "tails":
        nn = ov.knn(co, m)
        rows = rng.choice(np.arange(m, n), size=n // 10, replace=False)
        for i in rows:
            nn[i, rng.integers(1, m):] = -1
        c0 = n // 2
        for i in range(c0, c0 + m):
            nn[i, i - c0:] = -1
    return co, perm, y, nn


def ratio(got, want, bound):
    """largest |got - want| / (C_BOUND bound); 0 where both the difference and the bound are 0"""
    diff = np.abs(np.asarray(got, dtype=np.float64) - np.asarray(want, dtype=np.float64))
    b = C_BOUND * np.asarray(bound, dtype=np.float64)
    r = np.where(diff == 0, 0., diff / np.where(b > 0, b, 1e-300))
    return float(r.max()) if r.size else 0.


def accumulators(rows, sms):
    return max(1, min(2 * sms, rows // 8))


def sum_bound(terms, bterms, sms):
    rows = len(terms)
    return float(np.sum(bterms) + (math.ceil(rows / accumulators(rows, sms)) + 16) * U * np.sum(np.abs(terms)))


def yaux_ref(n, nn_rows, row_begin, A, bA, r):
    """B_rows^T u_rows (ordered index) and its bound, from the reference rows [row_begin, row_begin + len(nn_rows))"""
    nr, m = nn_rows.shape
    u, bu = r["u"], r["bu"]
    ya = np.zeros(n); bnd = np.zeros(n); mag = np.zeros(n); cnt = np.zeros(n)
    idx = np.arange(row_begin, row_begin + nr)
    ya[idx] += u; mag[idx] += np.abs(u); bnd[idx] += bu; cnt[idx] += 1
    rr, kk = np.nonzero(nn_rows >= 0)
    j = nn_rows[rr, kk]
    np.add.at(ya, j, -A[rr, kk] * u[rr])
    np.add.at(mag, j, np.abs(A[rr, kk] * u[rr]))
    np.add.at(bnd, j, bA[rr, kk] * np.abs(u[rr]) + np.abs(A[rr, kk]) * bu[rr])
    np.add.at(cnt, j, 1)
    return ya, bnd + 2 * (cnt + 2) * U * mag  # the summation of the kernel and of this reference


def reference(co, nn, cid, pt, y_ord, row_begin=0, row_end=None, **faults):
    row_end = co.shape[0] if row_end is None else row_end
    r, A, bA, bad = ov.rows_ld(co, nn[row_begin:row_end], cid, pt[0], pt[1], pt[0] + 1., pt[0] + 1., y_ord, row_begin, **faults)
    assert bad == 0
    return r, A, bA


# ---------------------------------------------------------------------------------------------------------- CPU-only
def mp_rows(co, nn, cid, var, rng_, diag_nb, diag_obs, y, rows, qcoords=None):
    """the same row quantities with mpmath at 50 digits; "dA" and "dD" hold the factor derivatives w.r.t. log var (k = 0,
    dSigma~ = Sigma~ - I) and log range (k = 1): dA_k = S^-1 (g_k - G_k A), dD_k = G_k,qq - 2 A.g_k + A^T G_k A"""
    mp = pytest.importorskip("mpmath")
    mp.mp.dps = 50
    var, rng_ = mp.mpf(var), mp.mpf(rng_)

    def cov(dist):
        rd = rng_ * dist
        if cid == 0: return var * mp.exp(-rd)
        if cid == 1: return var * (1 + rd) * mp.exp(-rd)
        if cid == 2: return var * (1 + rd + rd * rd / 3) * mp.exp(-rd)
        return var * mp.exp(-rng_ * dist * dist)

    def grad_range(dist):
        rd = rng_ * dist
        if cid == 0: return -rd * cov(dist)
        if cid == 1: return -var * rd * rd * mp.exp(-rd)
        if cid == 2: return -var * rd * rd * (1 + rd) / 3 * mp.exp(-rd)
        return -rng_ * dist * dist * cov(dist)

    res = []
    for t, i in enumerate(rows):
        nb = [int(j) for j in nn[t] if j >= 0]
        pts = [[mp.mpf(float(v)) for v in co[j]] for j in nb]
        own = [mp.mpf(float(v)) for v in (qcoords[t] if qcoords is not None else co[i])]
        yi = mp.mpf(0) if qcoords is not None else mp.mpf(float(y[i]))
        q = len(nb)
        dist = lambda a, b: mp.sqrt(sum((a[k] - b[k]) ** 2 for k in range(len(a))))
        D = mp.mpf(diag_obs)
        By = yi
        out = {"A": [], "t": [mp.mpf(0)] * 6, "dA": [[], []], "dD": [var, mp.mpf(0)]}
        if q == 0:
            u = By / D
            out.update(D=D, By=By)
            out["t"] = [0, 0, u * u * var, 0, var / D, 0]
            res.append(out)
            continue
        S = mp.matrix(q, q); G = [mp.matrix(q, q), mp.matrix(q, q)]
        s = mp.matrix(q, 1); g = [mp.matrix(q, 1), mp.matrix(q, 1)]
        yn = mp.matrix(q, 1)
        for a in range(q):
            yn[a] = mp.mpf(float(y[nb[a]]))
            dd = dist(pts[a], own)
            s[a] = cov(dd); g[0][a] = s[a]; g[1][a] = grad_range(dd)
            for b in range(q):
                if a == b:
                    S[a, a] = mp.mpf(diag_nb); G[0][a, a] = var; G[1][a, a] = 0
                else:
                    dab = dist(pts[a], pts[b])
                    S[a, b] = cov(dab); G[0][a, b] = S[a, b]; G[1][a, b] = grad_range(dab)
        A = mp.lu_solve(S, s)
        w = mp.lu_solve(S, yn)
        D = D - sum(A[k] * s[k] for k in range(q))
        By = By - sum(A[k] * yn[k] for k in range(q))
        u = By / D
        t = []
        for k in range(2):
            GA = G[k] * A
            uk = -sum((g[k][a] - GA[a]) * w[a] for a in range(q))
            dD = (var if k == 0 else 0) - 2 * sum(A[a] * g[k][a] for a in range(q)) + sum(A[a] * GA[a] for a in range(q))
            t.append((uk * u, u * u * dD, dD / D))
            dAk = mp.lu_solve(S, g[k] - GA)
            out["dA"][k] = [dAk[a] for a in range(q)]
            out["dD"][k] = dD
        out.update(D=D, By=By, A=[A[k] for k in range(q)], t=[t[0][0], t[1][0], t[0][1], t[1][1], t[0][2], t[1][2]])
        res.append(out)
    return res


@pytest.mark.parametrize("cov", list(COVS))
def test_long_double_reference_matches_mpmath(cov):
    """20 rows per covariance: rows with q < m, a row whose neighbour coincides with its point, a row truncated to 4
    neighbours, and two prediction rows (one at an observed point). The long-double values agree with 50-digit mpmath to a
    hundredth of the fp64 bound."""
    n, d, m = 80, 2, 10
    cid, _, pt = pars(cov, n, d)
    rng = np.random.default_rng(5)
    co = rng.random((n, d))
    co[41] = co[17]  # coincident points
    y = rng.standard_normal(n)
    nn = ov.knn(co, m)
    nn[60, 4:] = -1
    assert 17 in nn[41]
    rows = [0, 1, 2, 5, 9, 10, 11, 20, 33, 41, 47, 50, 60, 64, 70, 75, 78, 79]
    sel = np.array(rows)
    for i in rows:
        r, A, bA, bad = ov.rows_ld(co, nn[i:i + 1], cid, pt[0], pt[1], pt[0] + 1., pt[0] + 1., y, i)
        assert bad == 0
        want = mp_rows(co, nn[i:i + 1], cid, pt[0], pt[1], pt[0] + 1., pt[0] + 1., y, [i])[0]
        check_against_mp(r, A, bA, want, nn[i])
    qc = np.stack([co[33], rng.random(d)])
    nnq = ov.knn_range(np.concatenate([co, qc]), m, n, n - 1)
    r, A, bA, bad = ov.rows_ld(co, nnq, cid, pt[0], pt[1], pt[0] + 1., pt[0], y, 0, qcoords=qc)
    assert bad == 0 and len(sel) + 2 == 20
    for t, want in enumerate(mp_rows(co, nnq, cid, pt[0], pt[1], pt[0] + 1., pt[0], y, [0, 1], qcoords=qc)):
        check_against_mp({k: v[t:t + 1] for k, v in r.items()}, A[t:t + 1], bA[t:t + 1], want, nnq[t])


def check_against_mp(r, A, bA, want, nb_row):
    tol = 1e-2 / C_BOUND
    assert ratio(r["D"], float(want["D"]), tol * r["bD"]) <= 1.
    assert ratio(r["By"], float(want["By"]), tol * r["bBy"]) <= 1.
    a_mp = np.zeros(A.shape[1]); a_mp[nb_row >= 0] = [float(v) for v in want["A"]]
    assert ratio(A[0], a_mp, tol * bA[0]) <= 1.
    for k in range(6):
        assert ratio(r["t%d" % (3 + k)], float(want["t"][k]), tol * r["bt%d" % (3 + k)]) <= 1., k


CPU_CASES = [(1500, d, m, cov, v) for (d, m) in ((2, 25), (3, 45), (1, 15)) for cov in COVS for v in VARIANTS]


def fp64_oracle_rows(co, nn, cid, pt, yo):
    """the fp64 oracle's (ov.factor: libm exp, differences before scaling) row quantities"""
    n, m = nn.shape
    A, Dinv, Ag, Dg, bad = ov.factor(co, nn, cid, pt, calc_grad=True)
    assert bad == 0
    yN = np.where(nn >= 0, yo[np.maximum(nn, 0)], 0.)
    By = yo - (A * yN).sum(1)
    u = By * Dinv
    out = {"A": A, "Dinv": Dinv, "D": 1. / Dinv, "By": By, "u": u, "quad": By * By * Dinv, "logD": -np.log(Dinv)}
    for k in range(2):
        out["t%d" % (3 + k)] = -(Ag[k] * yN).sum(1) * u
        out["t%d" % (5 + k)] = u * u * Dg[k]
        out["t%d" % (7 + k)] = Dg[k] * Dinv
    return out


ROW_CHECKS = [("D", "bD"), ("By", "bBy"), ("u", "bu"), ("quad", "bquad"), ("logD", "blogD")] + \
             [("t%d" % k, "bt%d" % k) for k in range(3, 9)]


def row_ratios(dev, r, A, bA):
    """largest ratio per quantity: dev holds A, Dinv and any of the row columns"""
    out = {"A": ratio(dev["A"], A, bA), "Dinv": ratio(dev["Dinv"], 1. / r["D"], r["bD"] / r["D"] ** 2)}
    for k, b in ROW_CHECKS:
        if k in dev:
            out[k] = ratio(dev[k], r[k], r[b])
    return out


@pytest.mark.parametrize("case", CPU_CASES, ids=["n%d-d%d-m%d-%s-%s" % c for c in CPU_CASES])
def test_fp64_oracle_within_bounds(case):
    n, d, m, cov, variant = case
    co, perm, y, nn = case_data(n, d, m, variant, 7 + d)
    nn = ov.knn(co, m) if nn is None else nn
    cid, _, pt = pars(cov, n, d)
    yo = y[perm]
    r, A, bA = reference(co, nn, cid, pt, yo)
    worst = row_ratios(fp64_oracle_rows(co, nn, cid, pt, yo), r, A, bA)
    assert max(worst.values()) <= 1., worst


FAULTS = {"jitter": {"diag": lambda v: (v + 1.) * (1. + 1e-10)}, "cov_mult": {"cov_mult": 1. + 1e-11}, "drop_pair": {}}
FAULT_CASES = [(1500, d, m, cov, v) for (d, m) in ((2, 25), (3, 45)) for cov in COVS for v in VARIANTS]


def close_pairs(co, nn, i):
    """the row's neighbour pairs, closest points (largest covariances) first"""
    nb = nn[i][nn[i] >= 0]
    pairs = [(np.sum((co[nb[a]] - co[nb[b]]) ** 2), a, b) for a in range(len(nb)) for b in range(a + 1, len(nb))]
    return [(a, b) for _, a, b in sorted(pairs)]


@pytest.mark.parametrize("fault", list(FAULTS))
@pytest.mark.parametrize("case", FAULT_CASES, ids=["n%d-d%d-m%d-%s-%s" % c for c in FAULT_CASES])
def test_bounds_reject_subtle_faults(fault, case):
    """the reference itself, run with a fault, stands in for a device: a 1e-10 jitter on the neighbour diagonal, every
    covariance off by 1e-11 relative, or one pair of one row's neighbour block dropped, must each be rejected"""
    n, d, m, cov, variant = case
    co, perm, y, nn = case_data(n, d, m, variant, 7 + d)
    nn = ov.knn(co, m) if nn is None else nn
    cid, _, pt = pars(cov, n, d)
    yo = y[perm]
    r, A, bA = reference(co, nn, cid, pt, yo)
    dn = do = pt[0] + 1.
    kw = {}
    if fault == "jitter":
        dn = FAULTS[fault]["diag"](pt[0])
    elif fault == "cov_mult":
        kw["cov_mult"] = FAULTS[fault]["cov_mult"]
    else:
        # the closest pair whose removal leaves the block positive definite (a device would flag the others through acc[2])
        i = next(i for i in range(n // 3, n) if np.sum(nn[i] >= 0) >= 2)
        for a, b in close_pairs(co, nn, i):
            if ov.rows_ld(co, nn[i:i + 1], cid, pt[0], pt[1], dn, do, yo, i, drop=(0, a, b))[3] == 0:
                break
        kw["drop"] = (i, a, b)
    rf, Af, _, bad = ov.rows_ld(co, nn, cid, pt[0], pt[1], dn, do, yo, 0, **kw)
    assert bad == 0
    dev = {"A": Af, "Dinv": 1. / rf["D"], "D": rf["D"], "By": rf["By"]}
    worst = row_ratios(dev, r, A, bA)
    assert max(worst.values()) > 1., worst


@pytest.mark.parametrize("cov", ["exponential", "matern1.5", "matern2.5"])
def test_bounds_are_tight(cov):
    """the median relative bound of D stays near fp64 resolution: a later change cannot quietly loosen it"""
    n, d, m = 3001, 2, 30
    co, perm, y, _ = case_data(n, d, m, "unif", 3)
    cid, _, pt = pars(cov, n, d)
    r, _, _ = reference(co, ov.knn(co, m), cid, pt, y[perm])
    assert np.median(C_BOUND * r["bD"] / r["D"]) <= 1e-11


def test_cases_reach_every_kernel_bucket():
    """the multi-row and shard cases run every (kernel, DIM, cap) bucket of launch_eval; every family serves the shards; the
    multi-row size keeps three rows (pairs) per warp up to 135 SMs"""
    reached = {kernel_bucket(d, m, mode) for d, m, _ in MULTI_CASES for mode in (MODE_NLL, MODE_STORE, MODE_GRAD)}
    assert reached == ALL_BUCKETS
    assert {kernel_bucket(d, m, MODE_STORE)[0] for d, m, _ in SHARD_CASES} == {"two_obs", "one_obs", "big"}
    assert N_ROWS % 2 == 1 and N_ROWS >= 3 * 32 * 132 + 1
    assert set(SHARD_LENGTHS) >= {0, 1, 2, 3, 4, 5, 31, 32, 33, 4097}
    assert any(b % 2 == 1 for b in np.cumsum([0] + SHARD_LENGTHS)[:-1])


# ---------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def lib(product_lib):
    assert product_lib.gpbdev_device_count() > 0, "no CUDA device visible — GPU tests need an H100"
    return product_lib


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


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
            print("  %-8s %-12s %.3g" % (fam, what, v))


def create(lib, co, perm, m, nn, row_begin=0, row_end=None):
    n, d = co.shape
    row_end = n if row_end is None else row_end
    h = C.c_void_p()
    chk(lib, lib.gpbdev_vecchia_create(C.byref(h), 0, C.c_int64(n), d, m, P(co), P(perm, C.c_int32),
                                       None if nn is None else P(nn, C.c_int32), C.c_int64(row_begin), C.c_int64(row_end)))
    return h


def get_factor(lib, h, n, m):
    A = np.empty((n, m)); Dinv = np.empty(n)
    chk(lib, lib.gpbdev_vecchia_get_factor(h, P(A), P(Dinv)))
    return A, Dinv


def eval_pass(lib, h, cid, var, rng_, mode):
    out = np.zeros(9)
    chk(lib, lib.gpbdev_vecchia_eval(h, cid, C.c_double(var), C.c_double(rng_), mode, P(out)))
    return out


def check_sums(out, r, idx, sms, family, mode):
    """the 3 likelihood sums (and with mode GRAD the 6 gradient sums) against the reference rows idx"""
    terms = [("quad", "bquad"), ("logD", "blogD")] + ([("t%d" % k, "bt%d" % k) for k in range(3, 9)] if mode == MODE_GRAD else [])
    slot = [0, 1] + ([3, 4, 5, 6, 7, 8] if mode == MODE_GRAD else [])
    assert out[2] == 0
    for s, (k, b) in zip(slot, terms):
        rr = ratio(out[s], np.sum(r[k][idx]), sum_bound(r[k][idx], r[b][idx], sms))
        record(family, "sum%d/%s" % (s, "grad" if mode == MODE_GRAD else ("store" if mode == MODE_STORE else "nll")), rr)
        assert rr <= 1., (s, out[s], np.sum(r[k][idx]))


def check_rows(lib, h, n, m, r, A, bA, lo, hi, family, what):
    Ad, Did = get_factor(lib, h, n, m)
    w = row_ratios({"A": Ad[lo:hi], "Dinv": Did[lo:hi]}, r, A, bA)
    for k, v in w.items():
        record(family, "%s/%s" % (k, what), v)
    assert max(w.values()) <= 1., (what, w)


def check_yaux(lib, h, perm, n, nn, lo, A, bA, r, family):
    ya_d = np.empty(n)
    chk(lib, lib.gpbdev_vecchia_yaux(h, P(ya_d)))
    ya, bnd = yaux_ref(n, nn[lo:lo + len(A)], lo, A, bA, r)
    rr = ratio(ya_d[perm], ya, bnd)
    record(family, "yaux", rr)
    assert rr <= 1.


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("case", MULTI_CASES, ids=["d%d-m%d-%s" % c for c in MULTI_CASES])
def test_multi_row_passes_match_long_double(lib, sms, case, variant):
    """STORE (A, D^-1 at every row, yaux), GRAD (9 sums) and NLL (3 sums) with several rows or pairs per warp; for the
    two-observation kernel also the factor its GRAD pass writes (STORE at other parameters first, then GRAD, then get_factor)"""
    d, m, cov = case
    n = N_ROWS
    assert n >= 3 * 32 * sms + 1
    family = kernel_bucket(d, m, MODE_STORE)[0]
    co, perm, y, nn = case_data(n, d, m, variant, 100 + d * 61 + m)
    cid, _, pt = pars(cov, n, d)
    h = create(lib, co, perm, m, nn)
    try:
        nn_d = np.empty((n, m), dtype=np.int32)
        chk(lib, lib.gpbdev_vecchia_get_nn(h, P(nn_d, C.c_int32)))
        if nn is not None:
            assert np.array_equal(nn_d, nn)
        chk(lib, lib.gpbdev_vecchia_set_y(h, P(np.ascontiguousarray(y))))
        r, A, bA = reference(co, nn_d, cid, pt, y[perm])
        idx = np.arange(n)
        out = eval_pass(lib, h, cid, pt[0], pt[1], MODE_STORE)
        check_sums(out, r, idx, sms, family, MODE_STORE)
        check_rows(lib, h, n, m, r, A, bA, 0, n, family, "store")
        check_yaux(lib, h, perm, n, nn_d, 0, A, bA, r, family)
        eval_pass(lib, h, cid, pt[0], 1.5 * pt[1], MODE_STORE)
        out = eval_pass(lib, h, cid, pt[0], pt[1], MODE_GRAD)
        check_sums(out, r, idx, sms, family, MODE_GRAD)
        if family == "two_obs":
            check_rows(lib, h, n, m, r, A, bA, 0, n, family, "grad")
        out = eval_pass(lib, h, cid, pt[0], pt[1], MODE_NLL)
        check_sums(out, r, idx, sms, family, MODE_NLL)
    finally:
        lib.gpbdev_vecchia_free(h)


@pytest.mark.gpu
@pytest.mark.parametrize("case", SHARD_CASES, ids=["d%d-m%d-%s" % c for c in SHARD_CASES])
def test_row_shards_match_long_double(lib, sms, case):
    """one engine per row shard (supplied neighbour sets, no all-reduce): its NLL and GRAD sums, the A and D^-1 of its rows and
    its partial yaux = B_shard^T u_shard against the reference over the shard's rows; a 0-row shard gives sums of exactly 0; the
    shard sums add up to the whole engine's"""
    d, m, cov = case
    n = 6001
    co, perm, y, nn = case_data(n, d, m, "tails", 300 + d * 7 + m)
    family = kernel_bucket(d, m, MODE_STORE)[0]
    cid, _, pt = pars(cov, n, d)
    r, A, bA = reference(co, nn, cid, pt, y[perm])
    bounds = np.cumsum([0] + SHARD_LENGTHS + [n - sum(SHARD_LENGTHS)])
    totals = {MODE_NLL: np.zeros(9), MODE_GRAD: np.zeros(9)}
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        h = create(lib, co, perm, m, nn, lo, hi)
        try:
            chk(lib, lib.gpbdev_vecchia_set_y(h, P(np.ascontiguousarray(y))))
            idx = np.arange(lo, hi)
            rs = {k: v[lo:hi] for k, v in r.items()}
            out = eval_pass(lib, h, cid, pt[0], pt[1], MODE_STORE)
            if hi == lo:
                assert np.all(out == 0.)
            check_sums(out, r, idx, sms, family + "-shard", MODE_STORE)
            check_rows(lib, h, n, m, rs, A[lo:hi], bA[lo:hi], lo, hi, family + "-shard", "store")
            check_yaux(lib, h, perm, n, nn, lo, A[lo:hi], bA[lo:hi], rs, family + "-shard")
            for mode in (MODE_GRAD, MODE_NLL):
                out = eval_pass(lib, h, cid, pt[0], pt[1], mode)
                if hi == lo:
                    assert np.all(out == 0.)
                check_sums(out, r, idx, sms, family + "-shard", mode)
                totals[mode] += out
        finally:
            lib.gpbdev_vecchia_free(h)
    h = create(lib, co, perm, m, nn)
    try:
        chk(lib, lib.gpbdev_vecchia_set_y(h, P(np.ascontiguousarray(y))))
        idx = np.arange(n)
        for mode in (MODE_GRAD, MODE_NLL):
            whole = eval_pass(lib, h, cid, pt[0], pt[1], mode)
            terms = [("quad", "bquad"), ("logD", "blogD")] + [("t%d" % k, "bt%d" % k) for k in range(3, 9)]
            for s, (k, b) in zip([0, 1, 3, 4, 5, 6, 7, 8] if mode == MODE_GRAD else [0, 1], terms):
                # both sides carry their own summation error: twice the bound of the whole sum
                assert ratio(totals[mode][s], whole[s], 2 * sum_bound(r[k][idx], r[b][idx], sms)) <= 1., (mode, s)
    finally:
        lib.gpbdev_vecchia_free(h)


def device_to_host(ptr, count):
    """copy count doubles from a device pointer (unified addressing: any context of the process)"""
    cuda = C.CDLL("libcuda.so.1")
    out = np.empty(count)
    rc = cuda.cuMemcpyDtoH_v2(P(out, C.c_double), C.c_uint64(ptr.value), C.c_size_t(8 * count))
    assert rc == 0, rc
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("cov", list(COVS))
def test_prediction_rows_match_long_double(lib, sms, cov):
    """BIG_PRED through one prediction set evaluated at two parameter values: the mean A_p y_N(p) and D_p at every point, for
    nnp in {7, 31, 33, 60}, with query points that coincide with observed ones; more than three points per warp"""
    n, d = 4001, 2
    co, perm, y, _ = case_data(n, d, 20, "unif", 77)
    npred = 3 * 4 * sms + 1 + 200
    rng = np.random.default_rng(11)
    Xp = np.concatenate([rng.random((npred - 200, d)), co[rng.choice(n, 200, replace=False)]])
    h = create(lib, co, perm, 20, None)
    try:
        chk(lib, lib.gpbdev_vecchia_set_y(h, P(np.ascontiguousarray(y))))
        yo = y[perm]
        for nnp in (7, 31, 33, 60):
            ps = C.c_void_p()
            chk(lib, lib.gpbdev_vecchia_predset_create(h, P(Xp), C.c_int64(npred), nnp, C.byref(ps)))
            try:
                nnq = ov.knn_range(np.concatenate([co, Xp]), nnp, n, n - 1)
                for scale in (1., 0.6):
                    cid, _, pt = pars(cov, n, d)
                    var, rg = pt[0] * scale, pt[1] / scale
                    mean_p, var_p = C.c_void_p(), C.c_void_p()
                    chk(lib, lib.gpbdev_vecchia_predset_eval(ps, cid, C.c_double(var), C.c_double(rg), C.byref(mean_p), C.byref(var_p)))
                    mu_d, dp_d = device_to_host(mean_p, npred), device_to_host(var_p, npred)
                    r, _, _, bad = ov.rows_ld(co, nnq, cid, var, rg, var + 1., var, yo, 0, qcoords=Xp)
                    assert bad == 0
                    rm = ratio(mu_d, -r["By"], r["bBy"])
                    rd = ratio(dp_d, r["D"], r["bD"])
                    record("big-pred", "mean", rm)
                    record("big-pred", "D", rd)
                    assert rm <= 1. and rd <= 1., (nnp, scale, rm, rd)
            finally:
                lib.gpbdev_vecchia_predset_free(ps)
    finally:
        lib.gpbdev_vecchia_free(h)
