"""Pins oracle/laplace.py (Laplace-Vecchia, bernoulli_logit; SURVEY §8 a12) against
  * the R test's hard-coded value (test_GPModel_non_Gaussian_data.R:2541-2542, exact GP == Vecchia with all predecessors),
  * golden vectors produced by the unmodified reference library (tests/golden/make_laplace_golden.py), for both the
    sparse-Cholesky and the iterative (PCG + stochastic Lanczos quadrature, identical probe vectors) variants."""
import json
import os

import numpy as np
import pytest

import datagen
from oracle import laplace as ol
from oracle import vecchia as ov

HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(HERE, "golden", "laplace_golden.json")) as f:
    GOLD = json.load(f)["cases"]


def data_of(c):
    if c["name"] == "r_binary":
        X, y = datagen.r_binary_test_data()
        return X, y, None
    return datagen.binary_synth(c["n"], c["dseed"], c["offset"])


def oracle_negll(c, method):
    X, y, off = data_of(c)
    vo = ov.VecchiaOracle(X, c["m"], c["cov_function"], c["shape"], c["ordering"], c["seed"])
    _, pt = ov.transform_cov_pars([1.0] + list(c["cov_pars"]), c["cov_function"], c["shape"])
    fe = None if off is None else off[vo.perm]
    return ol.negll(vo.coords, vo.nn, vo.cid, c["cov_pars"][0], pt[1], y[vo.perm], fixed_effects=fe, method=method)


def test_r_known_answer():
    X, y = datagen.r_binary_test_data()
    vo = ov.VecchiaOracle(X, 99, "exponential", 0.5, "none", 0)
    r = ol.negll(vo.coords, vo.nn, vo.cid, 0.9, 1. / 0.2, y[vo.perm], method="cholesky")
    assert abs(r["negll"] - 66.299571) < 1e-6


@pytest.mark.parametrize("idx", range(len(GOLD)))
def test_golden_cholesky(idx):
    c = GOLD[idx]
    if c.get("n", 100) > 3000:
        pytest.skip("sparse LU of the larger case is slow in scipy")
    r = oracle_negll(c, "cholesky")
    assert abs(r["negll"] - c["negll_cholesky"]) <= 1e-9 * abs(c["negll_cholesky"])


@pytest.mark.parametrize("idx", range(len(GOLD)))
def test_golden_iterative(idx):
    c = GOLD[idx]
    r = oracle_negll(c, "iterative")
    # same probe vectors (std::mt19937 + seed_seq + normal_distribution) => deterministic agreement
    assert abs(r["negll"] - c["negll_iterative"]) <= 1e-9 * abs(c["negll_iterative"])


def oracle_grad(c, method):
    X, y, off = data_of(c)
    vo = ov.VecchiaOracle(X, c["m"], c["cov_function"], c["shape"], c["ordering"], c["seed"])
    _, pt = ov.transform_cov_pars([1.0] + list(c["cov_pars"]), c["cov_function"], c["shape"])
    fe = None if off is None else off[vo.perm]
    return ol.grad_negll(vo.coords, vo.nn, vo.cid, c["cov_pars"][0], pt[1], y[vo.perm], fixed_effects=fe, method=method)


@pytest.mark.parametrize("idx", range(len(GOLD)))
def test_golden_gradient_cholesky(idx):
    """Gradient w.r.t. (log variance, log range) of the Laplace-approximated likelihood, sparse-Cholesky branch of
    CalcGradNegMargLikelihoodLaplaceApproxVecchia, against the reference's own gradient (one gradient-descent step)."""
    c = GOLD[idx]
    if c.get("n", 100) > 2000:
        pytest.skip("the oracle inverts Sigma^-1 + W densely")
    r = oracle_grad(c, "cholesky")
    g = np.array(c["grad_cholesky"])
    assert np.all(np.abs(r["grad"] - g) <= 1e-7 * np.abs(g).max()), (r["grad"], g)


@pytest.mark.parametrize("idx", range(len(GOLD)))
def test_golden_gradient_iterative(idx):
    """Iterative branch: stochastic trace estimates with the SLQ probe vectors and their CG solutions, VADU variance
    reduction with the optimal c, implicit derivative by PCG — the same probes as the reference => deterministic agreement."""
    c = GOLD[idx]
    r = oracle_grad(c, "iterative")
    g = np.array(c["grad_iterative"])
    assert np.all(np.abs(r["grad"] - g) <= 1e-6 * np.abs(g).max()), (r["grad"], g)


@pytest.mark.parametrize("cov,shape", [("matern", 1.5), ("gaussian", 0.), ("exponential", 0.5)])
def test_gradient_is_the_derivative_of_the_likelihood(cov, shape):
    """Central differences of the oracle's own (pinned) likelihood w.r.t. (log variance, log range) against grad_consistent."""
    X, y, _ = datagen.binary_synth(400, 11, False)
    vo = ov.VecchiaOracle(X, 10, cov, shape, "random", 1)
    th = np.array([1.3, 0.12])

    def f(t):
        _, pt = ov.transform_cov_pars([1.0] + list(t), cov, shape)
        return ol.negll(vo.coords, vo.nn, vo.cid, t[0], pt[1], y[vo.perm], method="cholesky", delta_conv_mode_finding=1e-13)["negll"]
    _, pt = ov.transform_cov_pars([1.0] + list(th), cov, shape)
    g = ol.grad_negll(vo.coords, vo.nn, vo.cid, th[0], pt[1], y[vo.perm], method="cholesky", delta_conv_mode_finding=1e-13)["grad_consistent"]
    for j in range(2):
        e = np.zeros(2); e[j] = 1e-5
        fd = (f(th * np.exp(e)) - f(th * np.exp(-e))) / 2e-5
        # Gaussian kernel: the neighbour blocks are nearly singular, and the reference's shortcut dSigma^-1/dlog(var) = -Sigma^-1
        # ignores the jitter on their diagonal (Vecchia_utils.cpp:1607) — a 1e-5-level effect there, 1e-9 elsewhere
        tol = 1e-4 if cov == "gaussian" else 1e-6
        assert abs(fd - g[j]) <= tol * max(1., abs(g[j])), (cov, j, fd, g[j])


@pytest.mark.parametrize("idx", [i for i, c in enumerate(GOLD) if "fit_iterative" in c and c.get("n", 100) <= 2000])
def test_fit_glue_reproduces_reference_fit(idx):
    """GPB_OptimCovPar for the bernoulli_logit Vecchia model = the library's L-BFGS driver (GPB200_LbfgsMinimize: the code
    REModel::OptimCovParLaplace runs) on log(cov_pars), from the reference's initial values, with the Laplace likelihood and its
    gradient as objective. Here the objective is the pinned oracle (no device): same iteration count and optimum as the
    reference's own fit (tests/golden/make_laplace_golden.py)."""
    import ctypes as C
    from gpboost_b200.libpath import load_lib
    lib = load_lib()
    c = GOLD[idx]
    X, y, off = data_of(c)
    vo = ov.VecchiaOracle(X, c["m"], c["cov_function"], c["shape"], c["ordering"], c["seed"])
    fe = None if off is None else off[vo.perm]

    def obj(xp, n, gp, ctx):
        th = np.exp(np.array([xp[0], xp[1]]))
        _, pt = ov.transform_cov_pars([1.0] + list(th), c["cov_function"], c["shape"])
        if bool(gp):
            r = ol.grad_negll(vo.coords, vo.nn, vo.cid, th[0], pt[1], y[vo.perm], fixed_effects=fe, method="iterative")
            gp[0], gp[1] = r["grad"][0], r["grad"][1]
        else:
            r = ol.negll(vo.coords, vo.nn, vo.cid, th[0], pt[1], y[vo.perm], fixed_effects=fe, method="iterative")
        return float(r["negll"])
    cb = C.CFUNCTYPE(C.c_double, C.POINTER(C.c_double), C.c_int, C.POINTER(C.c_double), C.c_void_p)(obj)
    fit = c["fit_iterative"]
    x = np.log(np.array(fit["init_cov_pars"]))
    fx = C.c_double(0.); it = C.c_int(0)
    rc = lib.GPB200_LbfgsMinimize(cb, None, 2, x.ctypes.data_as(C.POINTER(C.c_double)), C.byref(fx), 1000, C.c_double(1e-6), 6,
                                  C.c_double(1.0), C.byref(it))
    assert rc == 0, lib.LGBM_GetLastError().decode()
    # the optimum is flat for the Gaussian kernel (ill-conditioned neighbour blocks): the run stops 3 iterations earlier at the
    # same likelihood (1e-6 relative); the other cases take exactly the reference's number of iterations
    assert abs(it.value - fit["num_it"]) <= (3 if c["cov_function"] == "gaussian" else 0), (it.value, fit["num_it"])
    assert np.all(np.abs(np.exp(x) - np.array(fit["cov_pars"])) <= 5e-3 * np.array(fit["cov_pars"])), (np.exp(x), fit["cov_pars"])
    assert abs(fx.value - fit["negll"]) <= 1e-5 * abs(fit["negll"])


@pytest.mark.parametrize("idx", [1, 4])
def test_device_gradient_schedule_matches_reference(idx):
    """The operator schedule of gpbdev_vecchia_laplace_grad (csrc/dev/laplace.cuh) replayed in numpy — the same sequence of
    products with B, B^T, B_grad, B_grad^T, the same coefficient vectors c1 = -D^-1 dD, c2 = D^-1 + W, c3 = 1 + W / D^-1, the same
    buffers and signs — on the oracle's factor, mode, probes and CG solutions: it must give the reference's gradient. (The kernels
    themselves are checked one by one against a longdouble reference in tests/test_laplace_kernels_gpu.py; this pins the algebra
    they are composed with.)"""
    import scipy.sparse as sp
    c = GOLD[idx]
    X, y, off = data_of(c)
    vo = ov.VecchiaOracle(X, c["m"], c["cov_function"], c["shape"], c["ordering"], c["seed"])
    _, pt = ov.transform_cov_pars([1.0] + list(c["cov_pars"]), c["cov_function"], c["shape"])
    fe = None if off is None else off[vo.perm]
    res = ol.grad_negll(vo.coords, vo.nn, vo.cid, c["cov_pars"][0], pt[1], y[vo.perm], fixed_effects=fe, method="iterative")
    st = res["_state"]
    B, Bt, Dinv, W, p_, cfg = st["B"], st["Bt"], st["Dinv"], st["W"], st["p"], st["cfg"]
    n = y.shape[0]; mode = res["mode"]; U = res["_AinvZ"]; Zp = res["_Zp"]
    A_, _, dA, dD, bad = ol.factor_latent_grad(vo.coords, vo.nn, vo.cid, c["cov_pars"][0], pt[1])
    assert bad == 0
    nn = np.asarray(vo.nn); m = nn.shape[1]
    rows = np.repeat(np.arange(n), m); mask = nn.ravel() >= 0
    MA = sp.csr_matrix((A_.ravel()[mask], (rows[mask], nn.ravel()[mask])), shape=(n, n))
    MdA = sp.csr_matrix((dA.ravel()[mask], (rows[mask], nn.ravel()[mask])), shape=(n, n))
    mv_B = lambda X_, Ds=None: (X_ - MA @ X_) * (Ds[:, None] if Ds is not None else 1.)   # mv_B_kernel
    mv_Bt = lambda T_: T_ - MA.T @ T_                                                    # mv_Bt_kernel (W = nullptr)
    mv_Bg = lambda X_: -(MdA @ X_)                                                       # mv_Bg_kernel
    mv_Bgt_acc = lambda T_, V_: V_ - MdA.T @ T_                                          # mv_Bgt_kernel (accumulate)
    dw = Dinv + W
    c1 = -Dinv * dD; c2 = Dinv + W; c3 = 1. + W / Dinv
    dWv = p_ * (1 - p_) * (1 - 2 * p_)
    sdet = [np.sum(Dinv * dD), np.sum(Dinv / dw), np.sum(Dinv ** 2 * dD / dw)]            # grad_coef_kernel
    Z = ol._vadu_solve(B, Bt, dw, Zp)                                                    # PI_Z
    T = mv_B(Z)
    ZA = U * dWv[:, None] * Z; ZP = T * dWv[:, None] * T                                 # stoch_dmode_kernel
    ma = ZA.mean(1); mp = ZP.mean(1)
    cc = ((ZA - ma[:, None]) * (ZP - mp[:, None])).mean(1); cv = ((ZP - mp[:, None]) ** 2).mean(1)
    copt = np.where(cv == 0, 1., cc / np.where(cv == 0, 1., cv))
    rhs = 0.5 * (ma + copt * (dWv / dw) - copt * mp)
    x, _ = ol.cg_vadu(B, Bt, Dinv, W, rhs, np.zeros(n), cfg["cg_max_num_it"], cfg["cg_delta_conv"], True)
    T1 = mv_B(Z, Dinv); V = mv_Bt(T1)                                                    # j = 0
    zP = -(Z * V).sum(0); zA = -(U * V).sum(0)
    tt = mv_B(mode[:, None], Dinv); v = mv_Bt(tt)[:, 0]
    tr1 = zA.mean(); trP = zP.mean(); cq = ol._optimal_c(zA, zP, tr1, trP)
    g0 = 0.5 * (-(mode @ v) + tr1 + n + cq * (-sdet[1]) - cq * trP) + x @ v
    Y = mv_Bg(Z)                                                                         # j = 1
    V = mv_Bgt_acc(T1, mv_Bt(Dinv[:, None] * Y + c1[:, None] * T1))
    zA = (U * V).sum(0)
    R = mv_Bgt_acc(c3[:, None] * T1, mv_Bt(c2[:, None] * Y + c1[:, None] * T1))
    zP = (Z * R).sum(0)
    yy = mv_Bg(mode[:, None])
    v = mv_Bgt_acc(tt, mv_Bt(Dinv[:, None] * yy + c1[:, None] * tt))[:, 0]
    tr1 = zA.mean(); trP = zP.mean(); cq = ol._optimal_c(zA, zP, tr1, trP)
    g1 = (0.5 * (mode @ v + tr1 + sdet[0] + cq * (-sdet[2]) - cq * trP) - x @ v) * (-0.5 if vo.cid == 3 else -1.)
    want = np.array(c["grad_iterative"])
    assert np.all(np.abs(np.array([g0, g1]) - want) <= 1e-6 * np.abs(want).max()), ([g0, g1], want)
