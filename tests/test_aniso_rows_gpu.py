"""The anisotropic gradient pass row by row against a long-double reference with per-group error bounds.

`gpbdev_vecchia_eval_grad_aniso` runs MODE_GRAD_ANISO of vecchia_factor_kernel (m <= 30; DIM = 2 at d = 2, generic otherwise; caps
10 / 20 / 30, the d = 2 cap 30 existing only for the derivative modes and this one) or BIG_GRAD_ANISO of vecchia_big_kernel
(30 < m <= 60). It returns 3 + 3 (1 + C) sums: sum (By)^2 / D, sum log D, the count of bad rows, then for the variance (k = 0) and
each coordinate group (k = 1..C) sum u_k u, sum u^2 dD_k and sum dD_k / D. The device splits each pair's isotropic derivative g by
coordinate share, g S_c / r^2.

Reference: oracle.vecchia.rows_aniso_ld (oracle/vecchia_oracle.c: orc_vecchia_rows_aniso_ld) evaluates every row in long double
from the fp64 scaled coordinates at range 1. The group derivative entries come from the kernels' element formulas on the scaled
differences (exponential -var e^-r S_c / r, Matern 1.5 -var e^-r S_c, Matern 2.5 -var (1 + r) / 3 e^-r S_c, Gaussian
-var e^-r^2 S_c), not from the device's g / r^2. Bounds:

  * D, By, u, (By)^2 / D, log D and the three variance terms: as oracle.vecchia.rows_ld (tests/test_vecchia_rows_gpu.py) at range
    1: an entrywise perturbation E of the augmented matrix (covariance evaluation c_v = 8 u, distance rounding c_r = (d + 4) u,
    rounding of the coordinates, Cholesky backward error gam(q + 2)) propagated through b = [-A_i, 1] and w~ = [S^-1 y_N, 0];
    the terms take kappa_i (eps_i + rho_i) times the term with every factor in absolute value;
  * the terms of group c: kappa_i (eps_i + rho_i + (d + d_c + 6) u) times the same magnitude, the extra ulps covering the
    device's roundings of one group entry: the division g / r^2 (1), S_c over the d_c coordinates of group c (d_c + 2), the r^2
    it divides by (d + 2) and the final multiply (1) (oracle.vecchia.share_ulps).

A sum's bound is the sum of its rows' bounds plus (ceil(rows / accumulators) + 16) u sum |terms| (sum_bound of
test_vecchia_rows_gpu). Every comparison is |device - reference| <= C_BOUND * bound, C_BOUND = 4.

CPU tests (no gpu mark) check the reference against 50-digit mpmath written in the original coordinates, that one group
reproduces the isotropic range terms and that ARD groups add up to them, that the fp64 restatement (tests/aniso_oracle.py)
stays inside the bounds, that four plausible kernel faults are rejected, that the bounds stay tight, and that the cases reach
every kernel instantiation. GPU tests run the pass with at least three rows per warp (n = 13001), on row shards (0..5, 31..33 and
4097 rows from odd rows, and single chosen rows) and through the product route (unsearched engine, device scaling, device
search, twice)."""
import ctypes as C

import numpy as np
import pytest

import aniso_oracle as ao
from oracle import vecchia as ov
from test_vecchia_rows_gpu import C_BOUND, P, case_data, chk, ratio, sum_bound
from test_vecchia_kernels_gpu import spread_range

if np.finfo(np.longdouble).eps > 1e-18:
    pytest.skip("long double has no extended precision on this host", allow_module_level=True)

VAR = 3.25  # sigma_1^2 / sigma^2 on the transformed scale
KERNELS = {"exponential": 0, "matern1.5": 1, "matern2.5": 2, "gaussian": 3}
VARIANTS = ["unif", "tails", "near"]
N_ROWS = 13001
FACTORS = np.array([0.7, 1.6, 1.1, 0.85, 1.3, 0.6, 1.9, 1.0])  # anisotropy: coordinate j is scaled by FACTORS[j % 8] / spread


def groups_of(kind, d):
    if kind == "ard":
        return np.arange(d, dtype=np.int32)
    if kind == "st":
        return np.array([0] + [1] * (d - 1), dtype=np.int32)
    if kind == "mix":
        return np.array([0, 1, 0, 2, 1], dtype=np.int32)
    return np.zeros(d, dtype=np.int32)


def scales(n, d, mult=1.):
    return mult * FACTORS[np.arange(d) % len(FACTORS)] / spread_range(n, d)


def aniso_bucket(d, m):
    """(kernel, DIM, cap) that gpbdev_vecchia_eval_grad_aniso runs: its big-kernel branch (m > 30) or pick_cap / pick_dim"""
    if m > 30:
        return ("big", 0, 60)
    return ("one_obs", 2 if d == 2 else 0, 10 if m <= 10 else (20 if m <= 20 else 30))


# (d, m, kernel, groups): every (DIM, cap) of MODE_GRAD_ANISO and BIG_GRAD_ANISO; one, two, d and 16 groups
MULTI_CASES = [(1, 15, "matern1.5", "ard")]
MULTI_CASES += [(2, m, k, "ard") for m in (10, 20, 25, 30) for k in KERNELS]
MULTI_CASES += [(3, 30, "matern1.5", "st"), (5, 8, "matern1.5", "mix"), (16, 10, "exponential", "ard"),
                (2, 45, "matern1.5", "ard"), (3, 60, "gaussian", "ard")]

SHARD_LENGTHS = [1, 0, 2, 3, 4, 5, 31, 32, 33, 4097]  # a 1-row shard first: the following ones begin at odd rows
SHARD_CASES = [(2, 30, "matern1.5", "ard"), (3, 20, "matern1.5", "ard"), (2, 45, "matern1.5", "ard")]
PRODUCT_CASES = [(2, 30, "matern1.5", "ard"), (3, 45, "gaussian", "st")]


def reference(Xs, nn, cid, grp, y_ord, row_begin=0, row_end=None, **faults):
    row_end = Xs.shape[0] if row_end is None else row_end
    r, bad = ov.rows_aniso_ld(Xs, nn[row_begin:row_end], cid, VAR, grp, y_ord, row_begin, **faults)
    assert bad == 0
    return r


def sum_slots(r):
    """(slot of the device's output, row terms, row bounds) for every sum but the bad-row count"""
    out = [(0, r["quad"], r["bquad"]), (1, r["logD"], r["blogD"])]
    return out + [(3 + s, r["terms"][:, s], r["bterms"][:, s]) for s in range(r["terms"].shape[1])]


def slot_name(s):
    if s < 3:
        return ["quad", "logD", "bad"][s]
    k, j = divmod(s - 3, 3)
    return "%s/%s" % ("var" if k == 0 else "group", ["u_k u", "u^2 dD", "dD/D"][j])


# ---------------------------------------------------------------------------------------------------------- CPU-only
def mp_aniso_rows(X, lam, cid, var, grp, y, nn, rows):
    """the same row quantities with mpmath at 50 digits from the original coordinates X: Matern / exponential ARD on
    r^2 = sum_j (lambda_j dx_j)^2, Gaussian ARD on r^2 = sum_j lambda_j dx_j^2; returns per row (D, By, quad, logD, terms)"""
    mp = pytest.importorskip("mpmath")
    mp.mp.dps = 50
    var = mp.mpf(var)
    ng = int(grp.max()) + 1
    lam = [mp.mpf(float(v)) for v in lam]

    def pair(a, b):
        parts = [lam[j] * (a[j] - b[j]) ** 2 if cid == 3 else (lam[j] * (a[j] - b[j])) ** 2 for j in range(len(a))]
        Sc = [sum((parts[j] for j in range(len(a)) if grp[j] == c), mp.mpf(0)) for c in range(ng)]
        r2 = sum(parts, mp.mpf(0))
        r = mp.sqrt(r2)
        e = mp.exp(-r)
        if cid == 0:
            k, dk = e, [(-e * s / r if r > 0 else mp.mpf(0)) for s in Sc]
        elif cid == 1:
            k, dk = (1 + r) * e, [-e * s for s in Sc]
        elif cid == 2:
            k, dk = (1 + r + r * r / 3) * e, [-(1 + r) / 3 * e * s for s in Sc]
        else:
            k = mp.exp(-r2)
            dk = [-k * s for s in Sc]
        return var * k, [var * v for v in dk]

    res = []
    for t, i in enumerate(rows):
        nb = [int(j) for j in nn[t] if j >= 0]
        pts = [[mp.mpf(float(v)) for v in X[j]] for j in nb] + [[mp.mpf(float(v)) for v in X[i]]]
        q = len(nb)
        Sig = mp.matrix(q + 1, q + 1)
        Gs = [mp.matrix(q + 1, q + 1) for _ in range(1 + ng)]
        for a in range(q + 1):
            Sig[a, a] = var + 1
            Gs[0][a, a] = var
            for b in range(a + 1, q + 1):
                c, dk = pair(pts[a], pts[b])
                Sig[a, b] = Sig[b, a] = c
                Gs[0][a, b] = Gs[0][b, a] = c
                for g in range(ng):
                    Gs[1 + g][a, b] = Gs[1 + g][b, a] = dk[g]
        yn = [mp.mpf(float(y[j])) for j in nb]
        if q:
            S = Sig[:q, :q]
            s = Sig[:q, q]
            A = mp.lu_solve(S, s)
            w = mp.lu_solve(S, mp.matrix(yn))
        D = Sig[q, q] - sum((A[k] * Sig[k, q] for k in range(q)), mp.mpf(0))
        By = mp.mpf(float(y[i])) - sum((A[k] * yn[k] for k in range(q)), mp.mpf(0))
        u = By / D
        terms = []
        for G in Gs:
            b = [-A[k] for k in range(q)] + [mp.mpf(1)]
            wt = [w[k] for k in range(q)] + [mp.mpf(0)]
            dD = sum((b[a] * G[a, c] * b[c] for a in range(q + 1) for c in range(q + 1)), mp.mpf(0))
            uk = -sum((b[a] * G[a, c] * wt[c] for a in range(q + 1) for c in range(q + 1)), mp.mpf(0))
            terms += [uk * u, u * u * dD, dD / D]
        res.append((D, By, By * By / D, mp.log(D), terms))
    return res


def dyadic_case(n, d, cid, seed, s):
    """original coordinates on a 2^-20 grid and scale factors s on a 2^-10 grid below 2^10 (s = lambda; s = sqrt(lambda) for the
    Gaussian kernel): every product X * s has at most 40 significant bits, so the host's scaling is exact and mpmath in the
    original coordinates sees the points the reference sees"""
    rng = np.random.default_rng(seed)
    X = rng.integers(0, 2 ** 20, (n, d)) / 2. ** 20
    assert np.all(s * 2. ** 10 == np.round(s * 2. ** 10)) and np.all(s < 2. ** 10)
    lam = s * s if cid == 3 else s
    return X, lam, np.ascontiguousarray(X * s), rng.standard_normal(n)


@pytest.mark.parametrize("kernel", list(KERNELS))
def test_long_double_reference_matches_mpmath(kernel):
    """20 rows per kernel: row 0, rows with q < m, a row whose neighbour coincides with its point, a row truncated to 4 neighbours
    (d = 3, ARD), and two d = 16 rows with 16 groups. The long-double values agree with 50-digit mpmath to a hundredth of the
    fp64 bound."""
    cid = KERNELS[kernel]
    tol = 1e-2 / C_BOUND
    X, lam, Xs, y = dyadic_case(80, 3, cid, 5, np.array([3.25, 5.5, 2.375]) if cid != 3 else np.array([1.75, 2.5, 1.25]))
    X[41] = X[17]
    Xs[41] = Xs[17]
    m = 10
    nn = ov.knn(Xs, m)
    assert 17 in nn[41]
    nn[60, 4:] = -1
    rows = [0, 1, 2, 5, 9, 10, 11, 20, 33, 41, 47, 50, 60, 64, 70, 75, 78, 79]
    X16, lam16, Xs16, y16 = dyadic_case(60, 16, cid, 6, 0.5 + np.arange(16) / 16.)
    nn16 = ov.knn(Xs16, 8)
    cases = [(X, lam, Xs, y, nn, groups_of("ard", 3), rows), (X16, lam16, Xs16, y16, nn16, groups_of("ard", 16), [30, 59])]
    assert sum(len(c[-1]) for c in cases) == 20
    for X_, lam_, Xs_, y_, nn_, grp, rows_ in cases:
        for i in rows_:
            r = reference(Xs_, nn_, cid, grp, y_, i, i + 1)
            D, By, quad, logD, terms = mp_aniso_rows(X_, lam_, cid, VAR, grp, y_, nn_[i:i + 1], [i])[0]
            for k, want in (("D", D), ("By", By), ("quad", quad), ("logD", logD)):
                assert ratio(r[k], float(want), tol * r["b" + k]) <= 1., (i, k)
            got = r["terms"][0]
            assert ratio(got, np.array([float(v) for v in terms]), tol * r["bterms"][0]) <= 1., (i, got, terms)


def iso_terms(ri):
    """rows_ld's variance (t3, t5, t7) and range (t4, t6, t8) terms in the aniso layout and their bounds"""
    t = np.column_stack([ri[k] for k in ("t3", "t5", "t7", "t4", "t6", "t8")])
    b = np.column_stack([ri["b" + k] for k in ("t3", "t5", "t7", "t4", "t6", "t8")])
    return t, b


IDENTITY_CASES = [(1500, d, m, k, v) for (d, m) in ((2, 25), (3, 45)) for k in KERNELS for v in ("unif", "near")]


@pytest.mark.parametrize("case", IDENTITY_CASES, ids=["n%d-d%d-m%d-%s-%s" % c for c in IDENTITY_CASES])
def test_one_group_and_ard_groups_reproduce_isotropic_terms(case):
    """With one group covering every coordinate, the group terms are rows_ld's range terms at range 1 (and the variance terms its
    variance terms); with one group per coordinate, the group terms add up to them: each within the sum of both bounds"""
    n, d, m, kernel, variant = case
    cid = KERNELS[kernel]
    co, perm, y, _ = case_data(n, d, m, variant, 11 + d)
    Xs = np.ascontiguousarray(co * scales(n, d))
    nn = ov.knn(Xs, m)
    yo = y[perm]
    ri, _, _, bad = ov.rows_ld(Xs, nn, cid, VAR, 1., VAR + 1., VAR + 1., yo)
    assert bad == 0
    it, ib = iso_terms(ri)
    r1 = reference(Xs, nn, cid, groups_of("one", d), yo)
    assert np.array_equal(r1["D"], ri["D"]) and np.array_equal(r1["bD"], ri["bD"]) and np.array_equal(r1["By"], ri["By"])
    assert np.all(np.abs(r1["terms"] - it) <= r1["bterms"] + ib)
    ra = reference(Xs, nn, cid, groups_of("ard", d), yo)
    assert np.array_equal(ra["terms"][:, :3], r1["terms"][:, :3])
    for j in range(3):
        gsum = sum(ra["terms"][:, 3 + 3 * c + j] for c in range(d))
        gb = sum(ra["bterms"][:, 3 + 3 * c + j] for c in range(d))
        assert np.all(np.abs(gsum - it[:, 3 + j]) <= gb + ib[:, 3 + j]), j


FP64_CASES = [(d, m, cov, shape, v) for (d, m, cov) in ((2, 10, "matern_ard"), (3, 20, "matern_space_time"))
              for shape in (0.5, 1.5, 2.5) for v in ("unif", "near")]
FP64_CASES += [(d, m, "gaussian_ard", 0., v) for (d, m) in ((2, 10), (3, 20)) for v in ("unif", "near")]


@pytest.mark.parametrize("case", FP64_CASES, ids=["d%d-m%d-%s-%s-%s" % c for c in FP64_CASES])
def test_fp64_restatement_within_bounds(case):
    """tests/aniso_oracle.py (numpy LU solves, the element formulas in the original coordinates: a different route from the
    kernels) at n = 240: every per-parameter sum and the profiled gradient inside the reference's bounds"""
    d, m, cov, shape, variant = case
    n = 240
    rng = np.random.default_rng(17 * d + m)
    X = rng.uniform(0., 1., (n, d))
    if variant == "near":
        X[n - n // 4:] = X[:n // 4] + 1e-9 * rng.random((n // 4, d))
    y = rng.standard_normal(n)
    C_ = 2 if cov == "matern_space_time" else d
    cp = np.concatenate([[0.4, 1.3], rng.uniform(0.1, 0.4, C_)])
    o = ao.AnisoOracle(X, m, cov, shape, "random", 3)
    o.search(cp)
    _, var, lam = ao.transform(cp, o.cov_function, o.shape)
    Xs = o.scaled(cp)
    r, bad = ov.rows_aniso_ld(Xs, o.nn, o.cid, var, ao.groups(o.cov_function, d), y[o.perm], 0)
    assert bad == 0
    quad, logdet, uk, udu, tr = o.grad_sums(cp, y)
    got = np.concatenate([[quad, logdet], np.column_stack([uk, udu, tr]).ravel()])
    bnd = {}
    for (s, t, b), g in zip(sum_slots(r), got):
        bnd[s] = sum_bound(t, b, 0)  # sms = 0: one accumulator, the restatement sums sequentially
        assert ratio(g, np.sum(t), bnd[s]) <= 1., (slot_name(s), g, np.sum(t))
    # the profiled gradient (uk - udu / 2) / s2 + tr / 2, s2 = quad / n
    S = {s: np.sum(t) for s, t, _ in sum_slots(r)}
    s2 = S[0] / n
    _, g = o.grad_profiled(cp, y)
    for k in range(1 + C_):
        a, b, c = (3 + 3 * k + j for j in range(3))
        want = (S[a] - 0.5 * S[b]) / s2 + 0.5 * S[c]
        bg = (bnd[a] + 0.5 * bnd[b]) / s2 + abs(S[a] - 0.5 * S[b]) / s2 * bnd[0] / S[0] + 0.5 * bnd[c]
        assert ratio(g[k], want, bg) <= 1., (k, g[k], want)


FAULT_CASES = [(1500, 2, 25, "matern1.5", "ard"), (1500, 3, 45, "gaussian", "ard"), (1500, 5, 8, "exponential", "mix"),
               (1500, 3, 20, "matern2.5", "st")]
FAULTS = ["group_mult", "swap", "drop", "unmasked"]


def rejected(rf, r, sms=132):
    """largest ratio of a faulted reference (standing in for a device) over the clean one's bounds, per row and per sum"""
    worst = ratio(rf["terms"], r["terms"], r["bterms"])
    for (s, t, b), (_, tf, _) in zip(sum_slots(r), sum_slots(rf)):
        worst = max(worst, ratio(np.sum(tf), np.sum(t), sum_bound(t, b, sms)))
    return worst


@pytest.mark.parametrize("fault", FAULTS)
@pytest.mark.parametrize("case", FAULT_CASES, ids=["n%d-d%d-m%d-%s-%s" % c for c in FAULT_CASES])
def test_bounds_reject_plausible_kernel_faults(fault, case):
    """the reference run with a fault stands in for a device: group 1's entries off by a relative 1e-10; one row attributing
    group 0's share to group 1 and back; the pair (nearest neighbour, own point) missing from group 1's contraction in one row;
    group 0 using the whole r^2. Each must be rejected by some row or sum."""
    n, d, m, kernel, gk = case
    cid = KERNELS[kernel]
    grp = groups_of(gk, d)
    co, perm, y, _ = case_data(n, d, m, "unif", 21 + d)
    Xs = np.ascontiguousarray(co * scales(n, d))
    nn = ov.knn(Xs, m)
    yo = y[perm]
    r = reference(Xs, nn, cid, grp, yo)
    i = n // 3
    q = int(np.sum(nn[i] >= 0))
    kw = {"group_mult": {"group_mult": (1, 1. + 1e-10)}, "swap": {"swap": (i, 0, 1)}, "drop": {"drop": (i, 1, 0, q)},
          "unmasked": {"unmasked": 0}}[fault]
    rf = reference(Xs, nn, cid, grp, yo, **kw)
    assert not np.array_equal(rf["terms"], r["terms"])
    assert rejected(rf, r) > 1.


def test_bounds_are_tight():
    """Matern 1.5, d = 2, m = 30: the median 4 bound / |term| of the group dD_k / D terms stays below 1e-11 where neighbours are
    weakly correlated (scales x 4, median kappa ~ 14), and 4 bound / (kappa |term|) below 1e-12 at the scales of the GPU cases
    (median kappa ~ 90): a later change cannot quietly loosen the bounds"""
    n, d, m = 3001, 2, 30
    co, perm, y, _ = case_data(n, d, m, "unif", 3)
    for mult, lim, by_kappa in ((4., 1e-11, False), (1., 1e-12, True)):
        Xs = np.ascontiguousarray(co * scales(n, d, mult))
        r = reference(Xs, ov.knn(Xs, m), 1, groups_of("ard", d), y[perm])
        t, b = r["terms"][1:, [5, 8]], r["bterms"][1:, [5, 8]]  # row 0 has no neighbours: its group terms are 0
        rel = C_BOUND * b / np.abs(t)
        if by_kappa:
            rel = rel / r["kappa"][1:, None]
        assert np.median(rel) <= lim, (mult, np.median(rel))


def test_cases_reach_every_kernel_instantiation():
    """the multi-row cases run every (DIM, cap) instantiation of MODE_GRAD_ANISO and BIG_GRAD_ANISO with one, two, d (> 2) and
    16 groups; the shard and product cases reach every family; the multi-row size keeps three rows per warp up to 135 SMs"""
    reached = {aniso_bucket(d, m) for d, m, _, _ in MULTI_CASES}
    assert reached == {("one_obs", dim, cap) for dim in (2, 0) for cap in (10, 20, 30)} | {("big", 0, 60)}
    ngroups = {(d, int(groups_of(g, d).max()) + 1) for d, _, _, g in MULTI_CASES}
    assert {c for _, c in ngroups} >= {1, 2, 16} and any(c == d > 2 for d, c in ngroups)
    assert {aniso_bucket(d, m)[0] for d, m, _, _ in SHARD_CASES} == {"one_obs", "big"}
    assert ("one_obs", 2, 30) in {aniso_bucket(d, m) for d, m, _, _ in SHARD_CASES}
    assert {aniso_bucket(d, m)[0] for d, m, _, _ in PRODUCT_CASES} == {"one_obs", "big"}
    assert N_ROWS % 2 == 1 and N_ROWS >= 3 * 32 * 135 + 1
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
            print("  %-26s %-13s %.3g" % (fam, what, v))


def create(lib, Xs, perm, m, nn, row_begin=0, row_end=None):
    n, d = Xs.shape
    row_end = n if row_end is None else row_end
    h = C.c_void_p()
    chk(lib, lib.gpbdev_vecchia_create(C.byref(h), 0, C.c_int64(n), d, m, P(np.ascontiguousarray(Xs)), P(perm, C.c_int32),
                                       None if nn is None else P(nn, C.c_int32), C.c_int64(row_begin), C.c_int64(row_end)))
    return h


def grad_aniso(lib, h, cid, grp):
    ng = int(grp.max()) + 1
    out = np.full(3 + 3 * (1 + ng), np.nan)
    chk(lib, lib.gpbdev_vecchia_eval_grad_aniso(h, cid, C.c_double(VAR), P(np.ascontiguousarray(grp, dtype=np.int32), C.c_int32),
                                                ng, P(out)))
    return out


def check_sums(out, r, idx, sms, family):
    """every sum of the pass against the reference rows idx; no bad rows"""
    assert out[2] == 0
    for s, t, b in sum_slots(r):
        rr = ratio(out[s], np.sum(t[idx]), sum_bound(t[idx], b[idx], sms))
        record(family, slot_name(s), rr)
        assert rr <= 1., (slot_name(s), s, out[s], np.sum(t[idx]))


def family_of(d, m):
    kern, dim, cap = aniso_bucket(d, m)
    return "big" if kern == "big" else "%s-%s-cap%d" % (kern, "d2" if dim == 2 else "gen", cap)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("case", MULTI_CASES, ids=["d%d-m%d-%s-%s" % c for c in MULTI_CASES])
def test_multi_row_pass_matches_long_double(lib, sms, case, variant):
    """all 3 + 3 (1 + C) sums with at least three rows per warp (about 49 for the big kernel), on pre-scaled coordinates with
    searched (unif, near) or supplied sets with -1 tails (tails); a second pass is bitwise the same"""
    d, m, kernel, gk = case
    n = N_ROWS
    assert n >= 3 * 32 * sms + 1
    cid, grp = KERNELS[kernel], groups_of(gk, d)
    co, perm, y, nn = case_data(n, d, m, variant, 500 + d * 61 + m)
    Xs = np.ascontiguousarray(co * scales(n, d))
    h = create(lib, Xs, perm, m, nn)
    try:
        nn_d = np.empty((n, m), dtype=np.int32)
        chk(lib, lib.gpbdev_vecchia_get_nn(h, P(nn_d, C.c_int32)))
        if nn is not None:
            assert np.array_equal(nn_d, nn)
        chk(lib, lib.gpbdev_vecchia_set_y(h, P(np.ascontiguousarray(y))))
        r = reference(Xs, nn_d, cid, grp, y[perm])
        out = grad_aniso(lib, h, cid, grp)
        check_sums(out, r, np.arange(n), sms, family_of(d, m))
        assert np.array_equal(grad_aniso(lib, h, cid, grp), out)  # fixed-order reductions
    finally:
        lib.gpbdev_vecchia_free(h)


def chosen_rows(nn, r, m, i_coinc):
    """single rows checked on their own: row 0, rows 1 and m - 1 (q < m), a row with a -1 tail, the row with a coincident
    neighbour and the row with the largest kappa"""
    tail = next(i for i in range(m, nn.shape[0]) if np.any(nn[i] < 0) and nn[i, 0] >= 0)
    return {"row0": 0, "row1": 1, "row m-1": m - 1, "tail": tail, "coincident": i_coinc, "max-kappa": int(np.argmax(r["kappa"]))}


@pytest.mark.gpu
@pytest.mark.parametrize("case", SHARD_CASES, ids=["d%d-m%d-%s-%s" % c for c in SHARD_CASES])
def test_row_shards_match_long_double(lib, sms, case):
    """one engine per row shard (supplied sets): its sums against the reference over the shard's rows, exact zeros for a 0-row
    shard, the shard sums adding up to the whole engine's within twice its bound; then 1-row engines at chosen rows"""
    d, m, kernel, gk = case
    n = 6001
    cid, grp = KERNELS[kernel], groups_of(gk, d)
    co, perm, y, nn = case_data(n, d, m, "tails", 700 + d * 7 + m)
    i_coinc = next(i for i in range(n // 3, n) if np.all(nn[i] >= 0))
    co[i_coinc] = co[nn[i_coinc, 0]]  # the row's point coincides with its first neighbour
    Xs = np.ascontiguousarray(co * scales(n, d))
    yo = y[perm]
    r = reference(Xs, nn, cid, grp, yo)
    family = family_of(d, m)
    ng = int(grp.max()) + 1
    bounds = np.cumsum([0] + SHARD_LENGTHS + [n - sum(SHARD_LENGTHS)])
    total = np.zeros(3 + 3 * (1 + ng))
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        h = create(lib, Xs, perm, m, nn, lo, hi)
        try:
            chk(lib, lib.gpbdev_vecchia_set_y(h, P(np.ascontiguousarray(y))))
            out = grad_aniso(lib, h, cid, grp)
            if hi == lo:
                assert np.all(out == 0.)
            check_sums(out, r, np.arange(lo, hi), sms, family + " shard")
            total += out
        finally:
            lib.gpbdev_vecchia_free(h)
    h = create(lib, Xs, perm, m, nn)
    try:
        chk(lib, lib.gpbdev_vecchia_set_y(h, P(np.ascontiguousarray(y))))
        whole = grad_aniso(lib, h, cid, grp)
        check_sums(whole, r, np.arange(n), sms, family)
        for s, t, b in sum_slots(r):  # both sides carry their own summation error
            assert ratio(total[s], whole[s], 2 * sum_bound(t, b, sms)) <= 1., slot_name(s)
    finally:
        lib.gpbdev_vecchia_free(h)
    for what, i in chosen_rows(nn, r, m, i_coinc).items():
        h = create(lib, Xs, perm, m, nn, i, i + 1)
        try:
            chk(lib, lib.gpbdev_vecchia_set_y(h, P(np.ascontiguousarray(y))))
            check_sums(grad_aniso(lib, h, cid, grp), r, np.arange(i, i + 1), sms, family + " row")
        finally:
            lib.gpbdev_vecchia_free(h)


@pytest.mark.gpu
@pytest.mark.parametrize("case", PRODUCT_CASES, ids=["d%d-m%d-%s-%s" % c for c in PRODUCT_CASES])
def test_product_route_matches_long_double(lib, sms, case):
    """the model's route: an unsearched engine on the original coordinates, device scaling (one rounded multiply per entry, as
    numpy's), device search, the pass; then scaling to a second parameter vector, searching and the pass again. The reference
    runs on host-scaled coordinates and the sets read back from the engine."""
    d, m, kernel, gk = case
    n = N_ROWS
    cid, grp = KERNELS[kernel], groups_of(gk, d)
    co, perm, y, _ = case_data(n, d, m, "unif", 900 + d + m)
    h = C.c_void_p()
    chk(lib, lib.gpbdev_vecchia_create_unsearched(C.byref(h), 0, C.c_int64(n), d, m, P(co), P(perm, C.c_int32), C.c_int64(0),
                                                   C.c_int64(n)))
    try:
        chk(lib, lib.gpbdev_vecchia_set_y(h, P(np.ascontiguousarray(y))))
        s1 = scales(n, d)[grp]  # one factor per group: the layout of a space-time or ARD parameter vector
        for s in (s1, s1 * np.linspace(1.7, 0.6, int(grp.max()) + 1)[grp]):
            chk(lib, lib.gpbdev_vecchia_set_coord_scale(h, P(np.ascontiguousarray(s))))
            chk(lib, lib.gpbdev_vecchia_search_neighbors(h))
            nn_d = np.empty((n, m), dtype=np.int32)
            chk(lib, lib.gpbdev_vecchia_get_nn(h, P(nn_d, C.c_int32)))
            Xs = np.ascontiguousarray(co * s)
            r = reference(Xs, nn_d, cid, grp, y[perm])
            check_sums(grad_aniso(lib, h, cid, grp), r, np.arange(n), sms, family_of(d, m) + " product")
    finally:
        lib.gpbdev_vecchia_free(h)
