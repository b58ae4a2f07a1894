"""Every specialisation of the Vecchia factor kernels against the oracle.

`launch_eval` (gpboost_b200/csrc/dev/dev_api.cu) runs one of several separately compiled kernels, chosen by dimension d,
neighbour count m and mode:

  one-observation kernel  vecchia_factor_kernel<COV, MODE, DIM, cap>  DIM = 2 at d = 2 (unrolled gather), DIM = 0 (generic) else;
                          cap = 10 / 20 / 30 for m <= 10 / <= 20 / <= 30; at d = 2, cap 30 only for MODE_STORE_GRAD
  two-observation kernel  vecchia_nll2_kernel<COV, MODE>              d = 2, 20 < m <= 30, modes NLL / STORE / GRAD
  big kernel              vecchia_big_kernel<COV, BIG_*>              30 < m <= 60, any d

Each has its own gather, padding and unrolling, for 4 covariances and 4 modes. The cases below reach every (kernel, DIM, cap)
bucket for every covariance and every mode it serves (test_parametrisation_reaches_every_kernel_bucket checks that without a
GPU), including the band
edges m = 1, 10/11, 20/21, 30/31/32, rows that are all padding (n = m + 1), distance ties and coincident points.

Tolerances as in tests/test_vecchia_gpu.py: neighbour indices bit-exact; sums, gradients, A, D^-1 and Psi^-1 y <= 1e-8 relative.
The range grows with the typical neighbour spacing (~ n^(-1/d)) so the covariances between neighbours are neither ~1 nor ~0
in every dimension."""
import ctypes as C

import numpy as np
import pytest

import datagen
from oracle import laplace as ol
from oracle import predict as op
from oracle import vecchia as ov

REL = 1e-8
COVS = [("exponential", 0.5), ("matern", 1.5), ("matern", 2.5), ("gaussian", 0.)]
COV_IDS = ["exponential", "matern1.5", "matern2.5", "gaussian"]
MODE_NLL, MODE_STORE, MODE_GRAD, MODE_STORE_GRAD = 0, 1, 2, 3


def kernel_bucket(d, m, mode):
    """(kernel, DIM, cap) that launch_eval runs for one pass; restates dev_api.cu:pick_cap / pick_dim, the big-kernel branch of
    launch_eval (m > kMaxNeighbors = 30) and its two-observation branch (d = 2, m > 20)."""
    if m > 30:
        return ("big", 0, 60)
    if mode in (MODE_NLL, MODE_STORE, MODE_GRAD) and d == 2 and m > 20:
        return ("two_obs", 2, 30)
    return ("one_obs", 2 if d == 2 else 0, 10 if m <= 10 else (20 if m <= 20 else 30))


# (kernel, DIM, cap) run by NLL / STORE / GRAD; ("one_obs", 2, 30) serves MODE_STORE_GRAD only
ALL_BUCKETS = ({("one_obs", dim, cap) for dim in (2, 0) for cap in (10, 20, 30)} - {("one_obs", 2, 30)}) | {("two_obs", 2, 30), ("big", 0, 60)}
STORE_GRAD_BUCKETS = {("one_obs", dim, cap) for dim in (2, 0) for cap in (10, 20, 30)}

# (n, d, m, data): data "synth" = U[0,1]^d, "dup" = with repeated and coincident points, "lattice3" = 3-D integer grid
# (distance ties everywhere)
FACTOR_CASES = [(700, d, m, "synth") for d in (1, 2, 3, 5, 16) for m in (1, 10, 11, 20, 21, 30, 31, 32, 60)]
FACTOR_CASES += [(700, 2, 25, "synth"), (11, 1, 10, "synth"), (31, 2, 30, "synth"), (26, 3, 25, "synth"), (61, 5, 60, "synth"),
                 (900, 3, 25, "dup"), (900, 1, 12, "dup"), (900, 2, 40, "dup"),
                 (729, 3, 26, "lattice3"), (729, 3, 8, "lattice3"), (729, 3, 45, "lattice3")]

# (d, m): MODE_STORE_GRAD, the latent factor and its range derivative (Laplace path)
LATENT_CASES = [(d, m) for d in (1, 2, 3, 5) for m in (5, 15, 25, 30)]


def case_id(c):
    return "n%d-d%d-m%d-%s" % c


def P(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


@pytest.fixture(scope="module")
def lib(product_lib):
    assert product_lib.gpbdev_device_count() > 0, "no CUDA device visible — GPU tests need an H100"
    return product_lib


def chk(lib, rc):
    assert rc == 0, lib.gpbdev_last_error().decode()


def make_engine(lib, coords, m, seed=1):
    n, d = coords.shape
    perm = ov.random_order(n, seed)
    co = np.ascontiguousarray(coords[perm])
    h = C.c_void_p()
    chk(lib, lib.gpbdev_vecchia_create(C.byref(h), 0, C.c_int64(n), d, m, P(co), P(perm, C.c_int32), None, C.c_int64(0), C.c_int64(n)))
    return h, perm, co


def spread_range(n, d):
    return 2. * n ** (-1. / d)


def case_coords(n, d, data, seed):
    if data == "synth":
        return datagen.synth(n, d, seed)
    rng = np.random.default_rng(seed)
    if data == "lattice3":
        k = round(n ** (1. / 3.))
        g = np.arange(k) / k
        coords = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
        return coords, rng.standard_normal(coords.shape[0])
    base = rng.random((n - n // 3, d))  # "dup": exact repeats, near repeats (1e-13 apart) and a tight cluster
    coords = np.concatenate([base, base[:n // 6], base[:n // 12] + 1e-13, 1e-3 * rng.random((n // 3 - n // 6 - n // 12, d))])
    return coords, rng.standard_normal(n)


def check_engine_against_oracle(lib, h, perm, co, y, m, cov, shape, cp):
    """neighbours, the sums of every mode, the gradient, A, D^-1 and Psi^-1 y of one engine against the oracle"""
    n = co.shape[0]
    cid = ov.cov_id(cov, shape)
    s2, pt = ov.transform_cov_pars(cp, cov, shape)
    nn = np.empty((n, m), dtype=np.int32)
    chk(lib, lib.gpbdev_vecchia_get_nn(h, P(nn, C.c_int32)))
    nn_o = ov.knn(co, m)
    assert np.array_equal(nn, nn_o)
    chk(lib, lib.gpbdev_vecchia_set_y(h, P(np.ascontiguousarray(y))))
    A, Dinv, Ag, Dg, bad = ov.factor(co, nn_o, cid, pt, calc_grad=True)
    assert bad == 0
    yo = y[perm]
    ref = ov.nll_from_factor(nn_o, A, Dinv, yo, s2)
    g_ref = ov.grad_from_factor(nn_o, A, Dinv, Ag, Dg, yo, s2)
    ya_o = np.empty(n)
    ya_o[perm] = ov.yaux(nn_o, A, Dinv, yo)

    def check_factor():
        A_d = np.empty((n, m)); Di_d = np.empty(n)
        chk(lib, lib.gpbdev_vecchia_get_factor(h, P(A_d), P(Di_d)))
        assert np.abs(A_d - A).max() <= REL
        assert (np.abs(Di_d - Dinv) / Dinv).max() <= REL
        ya = np.empty(n)
        chk(lib, lib.gpbdev_vecchia_yaux(h, P(ya)))
        assert np.abs(ya - ya_o).max() <= REL * np.abs(ya_o).max()

    out = np.zeros(9)
    # STORE first (factor of the STORE pass), then GRAD: the two-observation gradient pass stores A, D^-1 and u again, and the
    # factor is read once more after it
    for mode in (MODE_STORE, MODE_GRAD, MODE_NLL):
        chk(lib, lib.gpbdev_vecchia_eval(h, cid, C.c_double(pt[0]), C.c_double(pt[1]), mode, P(out)))
        assert abs(out[0] - ref[1]) <= REL * abs(ref[1]), mode
        assert abs(out[1] - ref[2]) <= REL * max(1., abs(ref[2])), mode
        assert out[2] == 0
        if mode == MODE_STORE:
            check_factor()
        if mode == MODE_GRAD:
            g = np.array([(out[3 + k] - 0.5 * out[5 + k]) / s2 + 0.5 * out[7 + k] for k in range(2)])
            assert np.all(np.abs(g - g_ref) <= REL * np.maximum(1., np.abs(g_ref))), (g, g_ref)
            check_factor()


@pytest.mark.gpu
@pytest.mark.parametrize("cov,shape", COVS, ids=COV_IDS)
@pytest.mark.parametrize("case", FACTOR_CASES, ids=[case_id(c) for c in FACTOR_CASES])
def test_factor_kernel_matches_oracle(lib, cov, shape, case):
    n, d, m, data = case
    coords, y = case_coords(n, d, data, 13 + d)
    h, perm, co = make_engine(lib, coords, m)
    try:
        check_engine_against_oracle(lib, h, perm, co, y, m, cov, shape, [0.4, 1.3, spread_range(coords.shape[0], d)])
    finally:
        lib.gpbdev_vecchia_free(h)


@pytest.mark.gpu
def test_store_after_gradient_pass_launches_nothing(lib):
    """The two-observation gradient pass (d = 2, 20 < m <= 30) also writes the factor into the buffers a STORE pass allocated, so
    a STORE request at the parameters of that gradient pass launches nothing; the engine then still matches the oracle."""
    coords, y = datagen.synth(800, 2, 7)
    m, cov, shape = 30, "matern", 1.5
    cp = [0.4, 1.3, spread_range(800, 2)]
    cid = ov.cov_id(cov, shape)
    _, pt = ov.transform_cov_pars(cp, cov, shape)
    h, perm, co = make_engine(lib, coords, m)
    try:
        out = np.zeros(9)
        chk(lib, lib.gpbdev_vecchia_set_y(h, P(np.ascontiguousarray(y))))
        chk(lib, lib.gpbdev_vecchia_eval(h, cid, C.c_double(pt[0]), C.c_double(1.5 * pt[1]), MODE_STORE, P(out)))
        chk(lib, lib.gpbdev_vecchia_eval(h, cid, C.c_double(pt[0]), C.c_double(pt[1]), MODE_GRAD, P(out)))
        before = lib.gpbdev_vecchia_launch_count(h)
        chk(lib, lib.gpbdev_vecchia_eval(h, cid, C.c_double(pt[0]), C.c_double(pt[1]), MODE_STORE, P(out)))
        assert lib.gpbdev_vecchia_launch_count(h) == before
        check_engine_against_oracle(lib, h, perm, co, y, m, cov, shape, cp)
    finally:
        lib.gpbdev_vecchia_free(h)


def latent_coords(n, d, seed):
    """U[0,1]^d; in 1-D one point per cell of width 1/n: uniform points on a line come arbitrarily close (~1/n^2), and without a
    nugget the smooth kernels' neighbour blocks are then singular to fp64 (condition ~1e10, where two correct evaluation
    orders differ by ~1e-7 relative)."""
    rng = np.random.default_rng(seed)
    if d == 1:
        return ((np.arange(n) + 0.5 * rng.random(n)) / n)[:, None]
    return rng.random((n, d))


@pytest.mark.gpu
@pytest.mark.parametrize("cov,shape", COVS, ids=COV_IDS)
@pytest.mark.parametrize("d,m", LATENT_CASES)
def test_latent_factor_range_derivative_matches_oracle(lib, cov, shape, d, m):
    """MODE_STORE_GRAD (latent factor of the Laplace path and its derivative w.r.t. log range) at every cap and DIM, against
    oracle.laplace.factor_latent_grad. Bar as in tests/test_laplace_gpu.py: 1e-8 of the largest entry, 1e-6 for Matern-2.5 and
    the Gaussian kernel, whose latent neighbour blocks (no nugget, jitter 1e-10) reach condition numbers ~1e8 at these ranges."""
    n = 600
    coords = latent_coords(n, d, 40 + d)
    h, perm, co = make_engine(lib, coords, m)
    try:
        nn = np.empty((n, m), dtype=np.int32)
        chk(lib, lib.gpbdev_vecchia_get_nn(h, P(nn, C.c_int32)))
        assert np.array_equal(nn, ov.knn(co, m))
        cid = ov.cov_id(cov, shape)
        _, pt = ov.transform_cov_pars([1.0, 1.0, spread_range(n, d)], cov, shape)
        A = np.empty((n, m)); Dinv = np.empty(n); dA = np.empty((n, m)); dD = np.empty(n)
        chk(lib, lib.gpbdev_vecchia_latent_factor_grad(h, C.c_int(cid), C.c_double(1.0), C.c_double(pt[1]), P(A), P(Dinv), P(dA), P(dD)))
        A0, Dinv0, dA0, dD0, bad = ol.factor_latent_grad(co, nn, cid, 1.0, pt[1])
        assert bad == 0
        tol = 1e-6 if cid in (2, 3) else 1e-8
        for got, want, name in ((A, A0, "A"), (1. / Dinv, 1. / Dinv0, "D"), (dA, dA0, "dA"), (dD, dD0, "dD")):
            assert np.max(np.abs(got - want)) <= tol * np.max(np.abs(want)), name
    finally:
        lib.gpbdev_vecchia_free(h)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [31, 60])
def test_latent_factor_derivative_rejects_more_than_30_neighbours(lib, m):
    coords = latent_coords(200, 3, 1)
    h, _, _ = make_engine(lib, coords, m)
    try:
        buf = np.empty(200 * m)
        rc = lib.gpbdev_vecchia_latent_factor_grad(h, C.c_int(1), C.c_double(1.0), C.c_double(5.), P(buf), P(buf), P(buf), P(buf))
        assert rc != 0
        assert "supports num_neighbors <= 30" in lib.gpbdev_last_error().decode()
    finally:
        lib.gpbdev_vecchia_free(h)


# ---------------------------------------------------------------------------------------- Laplace off the plane
# (d, covariance, shape, n, m): d = 3 takes the Morton-ordered operator kernels, d = 1 and 4 the index-ordered ones
LAPLACE_CASES = [(1, "exponential", 0.5, 2000, 20),
                 (3, "matern", 1.5, 2500, 25),
                 (4, "gaussian", 0., 1500, 15)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", LAPLACE_CASES, ids=lambda c: "d%d-%s" % (c[0], c[1]))
def test_laplace_off_the_plane_matches_oracle(case):
    """bernoulli_logit at d = 1, 3, 4 against oracle.laplace.negll (iterative), on the bar of
    tests/test_laplace_gpu.py::test_mode_and_iterations_match_oracle"""
    from gpboost_b200 import GPModel
    d, cov, shape, n, m = case
    X, y, _ = datagen.binary_synth(n, 30 + d, False, d=d)
    cp = [1.0, spread_range(n, d)]
    gm = GPModel(likelihood="bernoulli_logit", gp_coords=X, cov_function=cov, cov_fct_shape=shape, gp_approx="vecchia",
                 num_neighbors=m, vecchia_ordering="random", seed=d, matrix_inversion_method="iterative")
    v = gm.neg_log_likelihood(np.array(cp), y)
    info = gm.laplace_info()
    vo = ov.VecchiaOracle(X, m, cov, shape, "random", d)
    _, pt = ov.transform_cov_pars([1.0] + cp, cov, shape)
    r = ol.negll(vo.coords, vo.nn, vo.cid, cp[0], pt[1], y[vo.perm], method="iterative")
    assert int(info[1]) == r["newton_it"]
    assert int(info[2]) == r["cg_it"]
    assert int(info[3]) == r["slq_it"]
    assert abs(info[4] - r["logdet"]) <= 1e-8 * abs(r["logdet"])
    mode = gm.laplace_mode()
    mode_oracle = np.empty_like(mode)
    mode_oracle[vo.perm] = r["mode"]
    assert np.max(np.abs(mode - mode_oracle)) <= 1e-5 * (1. + np.max(np.abs(mode_oracle)))
    assert abs(v - r["negll"]) <= 1e-9 * abs(r["negll"])


# ---------------------------------------------------------------------------------------- prediction off the plane
@pytest.mark.gpu
@pytest.mark.parametrize("cov,shape", COVS, ids=COV_IDS)
@pytest.mark.parametrize("d", [1, 3])
def test_prediction_off_the_plane_matches_oracle(cov, shape, d):
    """BIG_PRED at d = 1 and 3 through GPModel.predict against oracle.predict.predict_gaussian, every point, with prediction
    points that coincide with observed ones. 1e-8 relative; 1e-6 for the Gaussian kernel, whose neighbour blocks are
    ill-conditioned (as in tests/test_predict_gpu.py)."""
    from gpboost_b200 import GPModel
    n = 1500
    X, y = datagen.synth(n, d, 50 + d)
    Xp = np.concatenate([np.random.default_rng(d).random((120, d)), X[:30]])
    cp = np.array([0.3, 1.2, spread_range(n, d)])
    mdl = GPModel(gp_coords=X, cov_function=cov, cov_fct_shape=shape, gp_approx="vecchia", num_neighbors=15, seed=2)
    tol = 1e-6 if cov == "gaussian" else 1e-8
    for nnp in (7, 31, 60):
        r = mdl.predict(y, Xp, cp, predict_var=True, predict_response=False, num_neighbors_pred=nnp)
        mu, var = op.predict_gaussian(X, y, Xp, cp, cov, shape, 15, predict_response=False, num_neighbors_pred=nnp)
        assert np.abs(r["mu"] - mu).max() <= tol * np.abs(mu).max(), nnp
        assert np.abs(r["var"] - var).max() <= tol * np.abs(var).max(), nnp


# ---------------------------------------------------------------------------------------- coverage (no GPU)
def test_parametrisation_reaches_every_kernel_bucket():
    """Every (kernel, DIM, cap) bucket of launch_eval is run for every covariance and every mode it serves, so trimming the
    cases above cannot silently drop one."""
    reached = {(kernel_bucket(d, m, mode), mode) for n, d, m, _ in FACTOR_CASES for mode in (MODE_NLL, MODE_STORE, MODE_GRAD)}
    assert reached == {(b, mode) for b in ALL_BUCKETS for mode in (MODE_NLL, MODE_STORE, MODE_GRAD)}
    latent = {kernel_bucket(d, m, MODE_STORE_GRAD) for d, m in LATENT_CASES}
    assert latent == STORE_GRAD_BUCKETS
    # the one-observation cap-30 kernel at d = 2 serves MODE_STORE_GRAD only: NLL / STORE / GRAD there take the two-observation kernel
    assert ("one_obs", 2, 30) in STORE_GRAD_BUCKETS
    assert all(b != ("one_obs", 2, 30) for b, _ in reached)
    # band edges and padded rows
    ms = {m for _, _, m, _ in FACTOR_CASES}
    assert {1, 10, 11, 20, 21, 30, 31, 32, 60} <= ms
    assert any(n <= m + 1 for n, _, m, _ in FACTOR_CASES)
    assert {d for _, d, _, _ in FACTOR_CASES} >= {1, 2, 3, 5, 16}
