"""The exact-GP (dense) engine against an extended-precision reference, at every tile edge of its blocked Cholesky.

`gpbdev_dense_eval` (gpboost_b200/csrc/dev/dense_api.cu) factorises the (n+1) x (n+1) matrix [[Psi, y], [y^T, *]] in 64 x 64
tiles, nt = ceil((n+1)/64) of them per side. The response y rides along as row n, so z = L^-1 y is row n of the factor. Block
column k pivots npiv = min(64, n - 64k) rows; the loop stops at the first tile with no pivot. `gpbdev_dense_grad` then forms
W = L^-1, P = Psi^-1 = W^T W (lower tiles only) and the gradient sums from P and alpha = Psi^-1 y.

Reference: the same operations restated in np.longdouble (x86-64: 64-bit mantissa, eps 1.1e-19) from the same fp64
coordinates, for n <= 800: a Cholesky of [[Psi, y], ...] giving L, z, log|Psi| and y^T Psi^-1 y; alpha by back
substitution; Psi^-1 by the backward recurrence L^T Psi^-1 = L^-1; the four gradient sums with dSigma/dlog(range) of
vecchia_factor.cuh::cov_eval. Above n = 800 the reference is fp64 LAPACK and only the scalar sums, z and alpha are compared.

Bars: Psi = I + v C with C a correlation matrix, so cond(Psi) <= 1 + v n is known before the run. Every quantity is held to
bar = 64 eps (1 + v n), capped at 1e-9, after a normalisation that keeps cancellation from hiding or inflating errors:
row r of L against sqrt(Psi_rr); P_ij against sqrt(P_ii P_jj); each gradient sum against the sum of its terms' magnitudes;
log|Psi| and y^T Psi^-1 y relative (all their terms are positive); z, alpha and yaux elementwise against their max norm.
The worst error/bar ratio of each quantity is printed when the module ends (run with -s to see it)."""
import ctypes as C
import functools
import math

import numpy as np
import pytest
from scipy.linalg import solve_triangular
from scipy.spatial.distance import cdist

LD = np.longdouble
EXTENDED = np.finfo(LD).eps <= 1e-18
EPS = np.finfo(np.float64).eps
C_BAR = 64.
NB = 64
LD_MAX_N = 800
COV_NAMES = ("exponential", "matern1.5", "matern2.5", "gaussian")   # gpbdev covariance ids 0..3
COV_MODEL = (("exponential", 0.5), ("matern", 1.5), ("matern", 2.5), ("gaussian", 0.))

# (n, d, cov id, v = sigma_1^2 / sigma^2, data)
#   synth  U[0,1]^d, long range (rho = 0.15 sqrt(d))
#   band   sorted U[0,1] (d = 1) with a short range rho = 3/n: for the Gaussian kernel dSigma/dlog(range) vanishes on every tile
#          more than one tile off the diagonal, so only the Psi^-1 read-back sees those tiles of P
#   offset U[0,1] + 1e6 (d = 1)
#   dup    exact duplicates and a cluster of coincident points, rows shuffled (distance 0: Sigma_ij = v, dSigma_ij = 0)
SMALL_N = (1, 2, 17, 62, 63, 64, 65, 127, 128, 129, 200)
CASES = [(n, 2, cov, 1., "synth") for n in SMALL_N for cov in range(4)]
CASES += [(333, 2, 0, 1., "synth"), (333, 2, 1, 10., "synth"), (333, 2, 2, 0.1, "synth"),
          (640, 2, 3, 1., "synth"), (640, 2, 0, 10., "synth"),
          (777, 2, 1, 1., "synth"), (777, 2, 2, 1., "synth"), (777, 2, 3, 0.1, "synth")]
CASES += [(63, 1, 0, 0.1, "synth"), (63, 3, 1, 1., "synth"), (63, 7, 2, 10., "synth"),
          (129, 1, 3, 10., "synth"), (129, 3, 0, 0.1, "synth"), (129, 7, 1, 1., "synth"),
          (333, 1, 2, 1., "synth"), (333, 3, 3, 10., "synth"), (333, 7, 0, 1., "synth")]
CASES += [(129, 1, 2, 1., "offset"), (200, 1, 0, 1., "offset")]
CASES += [(17, 2, 3, 10., "synth"), (65, 2, 1, 0.1, "synth"), (128, 2, 2, 10., "synth"), (200, 2, 0, 0.1, "synth")]
CASES += [(64, 2, 0, 1e3, "synth"), (65, 2, 1, 1e3, "synth"), (127, 2, 3, 1e3, "synth"), (129, 2, 2, 1e3, "synth")]
CASES += [(200, 1, 3, 1., "band"), (333, 1, 3, 1., "band"), (640, 1, 3, 10., "band")]
CASES += [(65, 2, 1, 1., "dup"), (65, 3, 3, 1., "dup"), (200, 2, 2, 1., "dup"), (200, 2, 3, 10., "dup")]
# fp64 LAPACK reference: scalar sums, z and alpha only
BIG_CASES = [(2000, 2, 0, 1., "synth"), (4095, 2, 1, 1., "synth"), (4096, 2, 2, 10., "synth"), (4097, 2, 3, 1., "synth"),
             (9000, 2, 1, 1., "synth")]

RATIOS = {}


def case_id(c):
    n, d, cov, v, data = c
    return "n%d-d%d-%s-v%g-%s" % (n, d, COV_NAMES[cov], v, data)


def tiles(n):
    """(nt, npiv of the last pivoted tile, tile and row of the response row) as dense_api.cu computes them"""
    nt = (n + 1 + NB - 1) // NB
    npiv = [max(0, min(NB, n - k * NB)) for k in range(nt)]
    return nt, npiv, n // NB, n % NB


def case_classes(c):
    n, d, cov, v, data = c
    nt, npiv, rt, rr = tiles(n)
    cls = {"nt=%s" % (nt if nt <= 3 else ">=10" if nt >= 10 else "4..9")}
    if nt == 1:
        cls.add("single tile")
    if rr == NB - 1:
        cls.add("response row ends a full tile")   # no padding row
    if rr == 0:
        cls.add("response row alone in its tile")   # npiv = 0 there: the factorisation loop stops before it
    if rr == 1:
        cls.add("response row after one pivot row")   # a last tile with npiv = 1
    cls.add("cov=%s" % COV_NAMES[cov])
    cls.add("d=%d" % d)
    cls.add("data=%s" % data)
    cls.add("v=%g" % v)
    return cls


def trans_range(cov, rho):
    """transformed range of cov_fcts.h:485-552 (REModel::TransformCovPars)"""
    return (1. / rho, math.sqrt(3.) / rho, math.sqrt(5.) / rho, 1. / (rho * rho))[cov]


def case_data(c, seed=None):
    n, d, cov, v, data = c
    rng = np.random.default_rng(seed if seed is not None else n * 1000 + d * 10 + cov)
    rho = 0.15 * math.sqrt(d)
    if data == "band":
        coords, rho = np.sort(rng.random(n))[:, None], 3. / n
    elif data == "offset":
        coords = rng.random((n, d)) + 1e6
    elif data == "dup":
        k = n // 5
        base = rng.random((n - 2 * k, d))
        coords = np.concatenate([base, base[:k], np.repeat(base[-1:], k, axis=0)])[rng.permutation(n)]
    else:
        coords = rng.random((n, d))
    y = np.sin(4. * coords[:, 0]) + 0.5 * rng.standard_normal(n)
    return np.ascontiguousarray(coords), y, v, trans_range(cov, rho)


def cov_and_grad(cov, dist, var, r):
    """Sigma and dSigma/dlog(range) (transformed scale) from distances — vecchia_factor.cuh::cov_eval restated"""
    rd = r * dist
    if cov == 0:
        val = var * np.exp(-rd)
        return val, -rd * val
    if cov == 1:
        e = np.exp(-rd)
        return var * (1 + rd) * e, -var * rd * rd * e
    if cov == 2:
        e = np.exp(-rd)
        return var * (1 + rd + rd * rd / 3) * e, -var * rd * rd / 3 * (1 + rd) * e
    val = var * np.exp(-r * dist * dist)
    return val, -r * dist * dist * val


def bar(n, v):
    return min(C_BAR * EPS * (1. + v * n), 1e-9)


def reference_ld(coords, y, cov, var, r):
    n = coords.shape[0]
    X = coords.astype(LD)
    D = np.sqrt(((X[:, None, :] - X[None, :, :]) ** 2).sum(-1))
    S, G = cov_and_grad(cov, D, LD(var), LD(r))
    Psi = S + np.eye(n, dtype=LD)
    # Cholesky of [[Psi, y], [y^T, *]], column by column: row n of the factor is z = L^-1 y
    A = np.concatenate([Psi, y.astype(LD)[None, :]])
    L = np.zeros((n + 1, n), dtype=LD)
    for j in range(n):
        s = A[j:, j] - L[j:, :j] @ L[j, :j]
        L[j, j] = np.sqrt(s[0])
        L[j + 1:, j] = s[1:] / L[j, j]
    L, z = L[:n], L[n]
    alpha = np.zeros(n, dtype=LD)
    for i in range(n - 1, -1, -1):
        alpha[i] = (z[i] - L[i + 1:, i] @ alpha[i + 1:]) / L[i, i]
    # Psi^-1 from L^T Psi^-1 = L^-1 (lower triangular, diagonal 1/L_jj): row j right of the diagonal from the trailing
    # block, then the diagonal entry from that row
    P = np.zeros((n, n), dtype=LD)
    for j in range(n - 1, -1, -1):
        lj = L[j + 1:, j]
        P[j, j + 1:] = -(lj @ P[j + 1:, j + 1:]) / L[j, j]
        P[j + 1:, j] = P[j, j + 1:]
        P[j, j] = (1. / L[j, j] - lj @ P[j + 1:, j]) / L[j, j]
    PG, aGa = P * G, alpha[:, None] * alpha[None, :] * G
    return dict(L=L, z=z, alpha=alpha, P=P, Psi_diag=np.diag(Psi),
                quad=z @ z, logdet=2 * np.log(np.diag(L)).sum(),
                out4=np.array([n - np.trace(P), PG.sum(), z @ z - alpha @ alpha, aGa.sum()]),
                scale4=np.array([n + np.abs(np.diag(P)).sum(), np.abs(PG).sum(), z @ z + alpha @ alpha, np.abs(aGa).sum()]))


def reference_fp64(coords, y, cov, var, r, with_psi_inv=True):
    """fp64 LAPACK through torch on the CPU (its threaded potrf is several times faster than scipy's here); Psi^-1 only for
    the trace sums. Row blocks keep the temporaries at a few n x n arrays."""
    import torch
    n = coords.shape[0]
    S, G = cov_and_grad(cov, cdist(coords, coords), var, r)
    S[np.diag_indices(n)] += 1.
    Lt = torch.linalg.cholesky(torch.from_numpy(S))
    del S
    Lc = Lt.numpy()
    z = solve_triangular(Lc, y, lower=True, check_finite=False)
    alpha = solve_triangular(Lc, z, lower=True, trans="T", check_finite=False)
    out4, scale4 = np.zeros(4), np.zeros(4)
    Ga = G @ alpha
    out4[2], scale4[2] = z @ z - alpha @ alpha, z @ z + alpha @ alpha
    out4[3], scale4[3] = alpha @ Ga, np.abs(alpha) @ (np.abs(G) @ np.abs(alpha))
    if with_psi_inv:
        W = torch.linalg.solve_triangular(Lt, torch.eye(n, dtype=torch.float64), upper=False)
        P = (W.T @ W).numpy()
        del W
        dP = np.diag(P).copy()
        out4[0], scale4[0] = n - dP.sum(), n + np.abs(dP).sum()
        for i0 in range(0, n, 512):   # strict lower triangle of P o G, doubled (G is symmetric with a zero diagonal)
            pg = np.tril(P[i0:i0 + 512] * G[i0:i0 + 512], i0 - 1)
            out4[1] += 2 * pg.sum()
            scale4[1] += 2 * np.abs(pg).sum()
    return dict(z=z, alpha=alpha, quad=z @ z, logdet=2 * np.log(np.diag(Lc)).sum(), out4=out4, scale4=scale4,
                with_psi_inv=with_psi_inv)


@functools.lru_cache(maxsize=None)
def reference(c):
    coords, y, var, r = case_data(c)
    if c[0] <= LD_MAX_N and EXTENDED:
        return reference_ld(coords, y, c[2], var, r)
    return reference_fp64(coords, y, c[2], var, r, with_psi_inv=c[0] <= 5000)


def record(qty, err, scale, b, what):
    """err <= b * scale, and keep the worst ratio per quantity"""
    err, scale = float(err), float(scale)
    ratio = err / (b * scale) if scale > 0 else (0. if err == 0 else math.inf)
    if ratio > RATIOS.get(qty, (0., ""))[0]:
        RATIOS[qty] = (ratio, what)
    assert ratio <= 1., "%s: error %.3e > bar %.3e x scale %.3e (%s)" % (qty, err, b, scale, what)


def vec_err(got, want):
    want64 = np.asarray(want, dtype=np.float64)
    return np.max(np.abs(np.asarray(got, dtype=LD) - np.asarray(want, dtype=LD))), np.max(np.abs(want64))


@pytest.fixture(scope="module", autouse=True)
def report_ratios():
    yield
    if RATIOS:
        print("\nworst error / bar per quantity (c = %g):" % C_BAR)
        for k in sorted(RATIOS):
            print("  %-10s %.3e  %s" % (k, RATIOS[k][0], RATIOS[k][1]))


def P_(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


@pytest.fixture(scope="module")
def lib(product_lib):
    product_lib.gpbdev_dense_last_error.restype = C.c_char_p
    return product_lib


@pytest.fixture(scope="module")
def gpu(lib):
    assert lib.gpbdev_device_count() > 0, "no CUDA device visible — GPU tests need an H100"
    return lib


def chk(lib, rc):
    assert rc == 0, lib.gpbdev_dense_last_error().decode()


def refused(lib, rc, msg):
    assert rc == -1
    assert msg in lib.gpbdev_dense_last_error().decode()


class Engine:
    def __init__(self, lib, coords, y):
        self.lib, self.n = lib, coords.shape[0]
        self.h = C.c_void_p()
        chk(lib, lib.gpbdev_dense_create(C.byref(self.h), 0, self.n, coords.shape[1], P_(coords)))
        self.set_y(y)

    def set_y(self, y):
        self.y = np.ascontiguousarray(y, dtype=np.float64)
        chk(self.lib, self.lib.gpbdev_dense_set_y(self.h, P_(self.y)))

    def eval(self, cov, var, r):
        o = np.zeros(3)
        chk(self.lib, self.lib.gpbdev_dense_eval(self.h, cov, C.c_double(var), C.c_double(r), P_(o)))
        return o

    def grad(self):
        o = np.zeros(4)
        chk(self.lib, self.lib.gpbdev_dense_grad(self.h, P_(o)))
        return o

    def yaux(self, scale):
        o = np.zeros(self.n)
        chk(self.lib, self.lib.gpbdev_dense_yaux(self.h, C.c_double(scale), P_(o)))
        return o

    def factor(self):
        L, z = np.full((self.n, self.n), np.nan), np.full(self.n, np.nan)
        chk(self.lib, self.lib.gpbdev_dense_get_factor(self.h, P_(L), P_(z)))
        return L, z

    def psi_inv(self):
        P = np.full((self.n, self.n), np.nan)
        chk(self.lib, self.lib.gpbdev_dense_get_psi_inv(self.h, P_(P)))
        return P

    def free(self):
        self.lib.gpbdev_dense_free(self.h)


def check_eval(ref, out3, b, what):
    assert out3[2] == 0, what
    record("quad", abs(LD(out3[0]) - ref["quad"]), abs(ref["quad"]), b, what)
    record("logdet", abs(LD(out3[1]) - ref["logdet"]), abs(ref["logdet"]), b, what)


def check_grad(ref, out4, b, what):
    names = ("tr(PS)", "sum(PG)", "aSa", "aGa")
    for k in range(4):
        if k < 2 and "P" not in ref and not ref.get("with_psi_inv"):
            continue
        record(names[k], abs(LD(out4[k]) - LD(ref["out4"][k])), ref["scale4"][k], b, what)


def check_factor(ref, L, z, b, what):
    if "L" in ref:
        assert np.all(np.triu(L, 1) == 0), what
        row_err = np.max(np.abs(L.astype(LD) - ref["L"]), axis=1) / np.sqrt(ref["Psi_diag"])
        record("L", np.max(row_err), 1., b, what)
    record("z", *vec_err(z, ref["z"]), b, what)


def check_psi_inv(ref, P, b, what):
    assert np.array_equal(P, P.T), what
    d = np.sqrt(np.diag(ref["P"]))
    record("Psi^-1", np.max(np.abs(P.astype(LD) - ref["P"]) / (d[:, None] * d[None, :])), 1., b, what)


def run_case(lib, c):
    n, d, cov, v, data = c
    what = case_id(c)
    coords, y, var, r = case_data(c)
    ref = reference(c)
    b = bar(n, v)
    e = Engine(lib, coords, y)
    try:
        check_eval(ref, e.eval(cov, var, r), b, what)
        L, z = e.factor()
        check_factor(ref, L, z, b, what)
        for s in (1., 0.37):
            record("yaux", *vec_err(e.yaux(s), ref["alpha"] * LD(s)), b, what + " scale %g" % s)
        check_grad(ref, e.grad(), b, what)
        if "P" in ref:
            check_psi_inv(ref, e.psi_inv(), b, what)
    finally:
        e.free()
    if n <= LD_MAX_N and not EXTENDED:
        pytest.skip("np.longdouble has no extended precision on this host: the fp64 LAPACK reference checked the sums, z and "
                    "alpha; L and Psi^-1 were not compared")


# ---------------------------------------------------------------------------------------------------------- CPU-only
def test_cases_reach_every_tile_class():
    """the tile arithmetic of dense_api.cu restated: the case list reaches every tile-edge class, dimension, data kind and
    conditioning band"""
    assert tiles(63) == (1, [63], 0, 63) and tiles(64) == (2, [64, 0], 1, 0) and tiles(65) == (2, [64, 1], 1, 1)
    assert tiles(127)[0] == 2 and tiles(128)[0] == 3 and tiles(777)[0] == 13 and tiles(4097)[0] == 65
    reached = set().union(*(case_classes(c) for c in CASES))
    need = {"single tile", "response row ends a full tile", "response row alone in its tile", "response row after one pivot row",
            "nt=1", "nt=2", "nt=3", "nt=>=10", "d=1", "d=2", "d=3", "d=7", "data=band", "data=offset", "data=dup",
            "v=0.1", "v=1", "v=10", "v=1000"}
    need |= {"cov=%s" % c for c in COV_NAMES}
    assert need <= reached, need - reached
    for cov in range(4):   # every covariance at every n <= 200, and at two multi-tile sizes above that
        assert {n for n in SMALL_N} <= {c[0] for c in CASES if c[2] == cov}
        assert len({c[0] for c in CASES if c[2] == cov and c[0] > 200}) >= 2, COV_NAMES[cov]
    assert {63, 129, 333} <= {c[0] for c in CASES if c[1] in (1, 3, 7)}
    assert all(c[0] <= 129 for c in CASES if c[3] >= 1e3)
    assert {65, 200} <= {c[0] for c in CASES if c[4] == "dup"}
    for c in CASES:   # every condition number bound keeps the bar at or below the 1e-9 of test_dense.py
        assert bar(c[0], c[3]) <= 1e-9
    big = {tiles(c[0])[3] for c in BIG_CASES}
    assert {63, 0, 1} <= big


def test_band_case_isolates_psi_inv_tiles():
    """the short-range Gaussian band: dSigma/dlog(range) is below 1e-30 on every tile more than one off the diagonal, so the
    gradient sums cannot see an error in those tiles of P; only the Psi^-1 read-back checks them"""
    for c in [c for c in CASES if c[4] == "band"]:
        coords, y, var, r = case_data(c)
        n = coords.shape[0]
        D = np.abs(coords[:, 0][:, None] - coords[:, 0][None, :])
        _, G = cov_and_grad(3, D, var, r)
        far = np.abs(np.arange(n)[:, None] // NB - np.arange(n)[None, :] // NB) > 1
        assert np.max(np.abs(G[far])) < 1e-30, case_id(c)


def test_reference_matches_lapack():
    """the longdouble restatement agrees with fp64 LAPACK to fp64 accuracy (guards the reference, not the device)"""
    if not EXTENDED:
        pytest.skip("np.longdouble has no extended precision on this host")
    for c in [(129, 3, 1, 10., "synth"), (65, 2, 3, 1., "dup")]:
        coords, y, var, r = case_data(c)
        a, f = reference_ld(coords, y, c[2], var, r), reference_fp64(coords, y, c[2], var, r)
        for k in ("quad", "logdet"):
            assert abs(float(a[k]) - f[k]) <= 1e-10 * abs(f[k])
        for k in range(4):
            assert abs(float(a["out4"][k]) - f["out4"][k]) <= 1e-10 * f["scale4"][k]
        assert np.max(np.abs(a["alpha"].astype(np.float64) - f["alpha"])) <= 1e-10 * np.max(np.abs(f["alpha"]))


def test_create_refuses_bad_sizes(lib):
    co = np.zeros(8)
    h = C.c_void_p()
    refused(lib, lib.gpbdev_dense_create(C.byref(h), 0, 0, 2, P_(co)), "need n > 0 and dim > 0")
    refused(lib, lib.gpbdev_dense_create(C.byref(h), 0, 4, 0, P_(co)), "need n > 0 and dim > 0")
    refused(lib, lib.gpbdev_dense_create(C.byref(h), 0, 46001, 1, P_(co)), "n is limited to 46000")


# ---------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_dense_engine_against_extended_reference(gpu, case):
    run_case(gpu, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", BIG_CASES, ids=case_id)
def test_dense_engine_large_n_against_lapack(gpu, case):
    run_case(gpu, case)


@pytest.mark.gpu
def test_engine_state_sequence(gpu):
    """one handle: covariance switch after W / P exist, repeated passes, a new response invalidating the factor"""
    lib = gpu
    n = 200
    ca, cb = (n, 2, 1, 1., "synth"), (n, 2, 3, 10., "synth")
    coords, y, var_a, r_a = case_data(ca, seed=5)
    _, _, var_b, r_b = case_data(cb, seed=5)
    y2 = np.cos(3. * coords[:, 1]) + 0.3 * np.random.default_rng(6).standard_normal(n)
    ref_a = reference_ld(coords, y, 1, var_a, r_a)
    ref_b = reference_ld(coords, y, 3, var_b, r_b)
    ref_c = reference_ld(coords, y2, 3, var_b, r_b)
    ba, bb = bar(n, var_a), bar(n, var_b)
    e = Engine(lib, coords, y)
    try:
        refused(lib, lib.gpbdev_dense_grad(e.h, P_(np.zeros(4))), "call gpbdev_dense_eval first")
        refused(lib, lib.gpbdev_dense_get_factor(e.h, P_(np.zeros((n, n))), None), "no current factor")
        # 1. Matern-1.5: eval, grad, yaux
        check_eval(ref_a, e.eval(1, var_a, r_a), ba, "state 1")
        refused(lib, lib.gpbdev_dense_get_psi_inv(e.h, P_(np.zeros((n, n)))), "no current Psi^-1")
        check_grad(ref_a, e.grad(), ba, "state 1")
        check_psi_inv(ref_a, e.psi_inv(), ba, "state 1")
        record("yaux", *vec_err(e.yaux(0.37), ref_a["alpha"] * LD(0.37)), ba, "state 1")
        # 2. Gaussian, other parameters: the gradient pass reuses W and P
        check_eval(ref_b, e.eval(3, var_b, r_b), bb, "state 2")
        refused(lib, lib.gpbdev_dense_get_psi_inv(e.h, P_(np.zeros((n, n)))), "no current Psi^-1")   # P is from state 1
        g1 = e.grad()
        check_grad(ref_b, g1, bb, "state 2")
        P1 = e.psi_inv()
        check_psi_inv(ref_b, P1, bb, "state 2")
        L1, z1 = e.factor()
        check_factor(ref_b, L1, z1, bb, "state 2")
        # 3. the reductions run in a fixed order: a second gradient pass is bit-identical
        assert np.array_equal(e.grad(), g1)
        assert np.array_equal(e.psi_inv(), P1)
        # 4. a new response invalidates the factor
        e.set_y(y2)
        refused(lib, lib.gpbdev_dense_grad(e.h, P_(np.zeros(4))), "call gpbdev_dense_eval first")
        refused(lib, lib.gpbdev_dense_yaux(e.h, C.c_double(1.), P_(np.zeros(n))), "call gpbdev_dense_eval first")
        refused(lib, lib.gpbdev_dense_get_factor(e.h, P_(np.zeros((n, n))), None), "no current factor")
        refused(lib, lib.gpbdev_dense_get_psi_inv(e.h, P_(np.zeros((n, n)))), "no current Psi^-1")
        # 5. eval, yaux with the new response; a repeated eval is bit-identical
        o3 = e.eval(3, var_b, r_b)
        check_eval(ref_c, o3, bb, "state 5")
        record("yaux", *vec_err(e.yaux(1.), ref_c["alpha"]), bb, "state 5")
        L2, z2 = e.factor()
        check_factor(ref_c, L2, z2, bb, "state 5")
        assert np.array_equal(L2, L1)   # the factor does not depend on y
        assert np.array_equal(e.eval(3, var_b, r_b), o3)
        L3, z3 = e.factor()
        assert np.array_equal(L3, L2) and np.array_equal(z3, z2)
    finally:
        e.free()


def ld_negll(coords, y, cov, cov_pars):
    """negative log-likelihood at original-scale (sigma^2, sigma_1^2, rho), and the sum of its terms' magnitudes"""
    s2, s1, rho = cov_pars
    v = s1 / s2
    ref = reference_ld(coords, y, cov, v, trans_range(cov, rho))
    terms = [ref["quad"] / 2 / LD(s2), ref["logdet"] / 2, len(y) / 2 * np.log(LD(s2)), len(y) / 2 * np.log(2 * np.pi, dtype=LD)]
    return sum(terms), sum(abs(t) for t in terms), v, ref


@pytest.mark.gpu
@pytest.mark.parametrize("d", [1, 3, 5])
@pytest.mark.parametrize("cov", range(4), ids=COV_NAMES)
def test_gpmodel_negll_against_extended_reference(gpu, d, cov):
    """GPModel(gp_approx="none"): the column-major -> row-major transpose of the coordinates and TransformCovPars"""
    from gpboost_b200 import GPModel
    if not EXTENDED:
        pytest.skip("np.longdouble has no extended precision on this host")
    n = 150
    rng = np.random.default_rng(40 + d + 10 * cov)
    coords = rng.random((n, d)) * np.arange(1, d + 1)   # unequal axes: a transposed matrix gives other distances
    y = np.sin(3. * coords[:, -1]) + 0.5 * rng.standard_normal(n)
    cp = (0.3, 1.2, 0.2 * math.sqrt(d))
    want, scale, v, _ = ld_negll(coords, y, cov, cp)
    shape = COV_MODEL[cov]
    m = GPModel(gp_coords=coords, cov_function=shape[0], cov_fct_shape=shape[1], gp_approx="none")
    got = m.neg_log_likelihood(np.array(cp), y)
    record("negll", abs(LD(got) - want), scale, bar(n, v), "GPModel d=%d %s" % (d, COV_NAMES[cov]))


@pytest.mark.gpu
def test_gpmodel_response_gradient_against_extended_reference(gpu):
    from gpboost_b200 import GPModel
    if not EXTENDED:
        pytest.skip("np.longdouble has no extended precision on this host")
    n, d = 300, 3
    rng = np.random.default_rng(77)
    coords = rng.random((n, d)) * np.array([1., 2., 0.5])
    y = np.cos(2. * coords[:, 1]) + 0.4 * rng.standard_normal(n)
    cp = np.array([0.4, 1.1, 0.3])
    _, _, v, ref = ld_negll(coords, y, 1, cp)
    m = GPModel(gp_coords=coords, cov_function="matern", cov_fct_shape=1.5, gp_approx="none")
    m.set_optim_params({"init_cov_pars": cp, "maxit": 0})
    m.fit(y)
    record("resp_grad", *vec_err(m.response_gradient(y), ref["alpha"] / LD(cp[0])), bar(n, v), "GPModel d=3 response_gradient")
