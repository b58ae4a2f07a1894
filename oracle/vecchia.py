"""TEST INFRASTRUCTURE ONLY — numpy front-end of the C restatement (oracle/vecchia_oracle.c).

High-level entry points mirror what the reference's C API computes for the hot path:
  * `neg_log_likelihood(...)`  ==  GPB_EvalNegLogLikelihood on a Gaussian GP (Vecchia or exact)
  * `factor(...)`              ==  B = I - A, D^-1 (+ gradients) of CalcCovFactorGradientVecchia
  * `nll_and_grad(...)`        ==  one EvalLLforLBFGSpp objective + gradient call (optim_utils.h:244-340)
"""
import ctypes as C
import math

import numpy as np

from .build import build_oracle

COV_IDS = {"exponential": 0, "matern0.5": 0, "matern1.5": 1, "matern2.5": 2, "gaussian": 3}

_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build_oracle())
        _lib.orc_vecchia_factor.restype = C.c_int
        _lib.orc_dense_nll.restype = C.c_int
        _lib.orc_knn_vecchia_range.restype = C.c_int
    return _lib


def _p(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


def cov_id(cov_function, shape=1.5):
    if cov_function == "matern":
        return COV_IDS["matern%.1f" % shape]
    return COV_IDS[cov_function]


def transform_cov_pars(cov_pars, cov_function, shape=1.5):
    """Original scale (sigma2, sigma1^2, rho) -> (sigma2, sigma1^2/sigma2, range_transformed):
    include/GPBoost/cov_fcts.h:485-552."""
    s2, s1, rho = [float(v) for v in cov_pars]
    cid = cov_id(cov_function, shape)
    rt = {0: 1. / rho, 1: np.sqrt(3.) / rho, 2: np.sqrt(5.) / rho, 3: 1. / (rho * rho)}[cid]
    return s2, np.array([s1 / s2, rt])


def random_order(n, seed):
    perm = np.empty(n, dtype=np.int32)
    lib().orc_vecchia_random_order(C.c_int(n), C.c_int(seed), _p(perm, C.c_int32))
    return perm


def knn(coords_ordered, m):
    """coords_ordered: (n, d) in Vecchia order. Returns int32 (n, m), -1 padded."""
    n, d = coords_ordered.shape
    cm = np.asfortranarray(coords_ordered, dtype=np.float64)
    nn = np.empty((n, m), dtype=np.int32)
    lib().orc_knn_vecchia(_p(cm), C.c_int(n), C.c_int(d), C.c_int(m), _p(nn, C.c_int32))
    return nn


def knn_range(coords, m, start_at, end_search_at):
    """The reference's search for the queries [start_at, n) of coords (n, d), candidates below min(i, end_search_at + 1).
    Model: start_at = 0, end_search_at = n - 2; prediction (observed points first): start_at = end_search_at + 1 = n_obs.
    m is clipped to end_search_at + 1. Returns int32 (n - start_at, m_clipped), -1 padded."""
    n, d = coords.shape
    cm = np.asfortranarray(coords, dtype=np.float64)
    nn = np.empty((n - start_at, m), dtype=np.int32)
    mc = lib().orc_knn_vecchia_range(_p(cm), C.c_int(n), C.c_int(d), C.c_int(m), C.c_int(start_at), C.c_int(end_search_at),
                                     _p(nn, C.c_int32))
    return np.ascontiguousarray(nn[:, :mc])


def sort_indices(v):
    """Indices sorting v ascending, by the same std::sort call as the reference (ties in its order)."""
    v = np.ascontiguousarray(v, dtype=np.float64)
    out = np.empty(v.shape[0], dtype=np.int32)
    lib().orc_sort_indices(_p(v), C.c_int(v.shape[0]), _p(out, C.c_int32))
    return out


def factor(coords_ordered, nn, cid, pars_trans, calc_grad=False):
    n, d = coords_ordered.shape
    m = nn.shape[1]
    cm = np.asfortranarray(coords_ordered, dtype=np.float64)
    A = np.empty((n, m)); Dinv = np.empty(n)
    Ag = np.empty((2, n, m)) if calc_grad else np.empty(1)
    Dg = np.empty((2, n)) if calc_grad else np.empty(1)
    pt = np.ascontiguousarray(pars_trans, dtype=np.float64)
    bad = lib().orc_vecchia_factor(_p(cm), C.c_int(n), C.c_int(d), C.c_int(m), _p(nn, C.c_int32), C.c_int(cid),
                                   _p(pt), _p(A), _p(Dinv), C.c_int(int(calc_grad)), _p(Ag), _p(Dg))
    return A, Dinv, (Ag if calc_grad else None), (Dg if calc_grad else None), bad


def nll_from_factor(nn, A, Dinv, y, sigma2):
    n, m = nn.shape
    out = np.empty(3)
    y = np.ascontiguousarray(y, dtype=np.float64)
    lib().orc_vecchia_nll(C.c_int(n), C.c_int(m), _p(nn, C.c_int32), _p(A), _p(Dinv), _p(y), C.c_double(sigma2), _p(out))
    return out  # negll, yTPsiInvy, log_det


def yaux(nn, A, Dinv, y):
    n, m = nn.shape
    out = np.empty(n)
    y = np.ascontiguousarray(y, dtype=np.float64)
    lib().orc_vecchia_yaux(C.c_int(n), C.c_int(m), _p(nn, C.c_int32), _p(A), _p(Dinv), _p(y), _p(out))
    return out


def grad_from_factor(nn, A, Dinv, Ag, Dg, y, sigma2):
    n, m = nn.shape
    g = np.empty(2)
    y = np.ascontiguousarray(y, dtype=np.float64)
    lib().orc_vecchia_grad(C.c_int(n), C.c_int(m), _p(nn, C.c_int32), _p(A), _p(Dinv), _p(Ag), _p(Dg), _p(y),
                           C.c_double(sigma2), _p(g))
    return g


class VecchiaOracle:
    """Ordering + neighbours fixed at construction (as GPB_CreateREModel does), evaluations afterwards."""

    def __init__(self, coords, num_neighbors=20, cov_function="matern", cov_fct_shape=1.5,
                 vecchia_ordering="random", seed=0):
        coords = np.asarray(coords, dtype=np.float64)
        n = coords.shape[0]
        self.n = n
        self.m = min(int(num_neighbors), n - 1)
        self.cov_function, self.shape = cov_function, cov_fct_shape
        self.cid = cov_id(cov_function, cov_fct_shape)
        if vecchia_ordering == "random":
            self.perm = random_order(n, seed)
        elif vecchia_ordering == "none":
            self.perm = np.arange(n, dtype=np.int32)
        else:
            raise ValueError(vecchia_ordering)
        self.coords = np.ascontiguousarray(coords[self.perm])
        self.nn = knn(self.coords, self.m)

    def neg_log_likelihood(self, cov_pars, y):
        s2, pt = transform_cov_pars(cov_pars, self.cov_function, self.shape)
        A, Dinv, _, _, _ = factor(self.coords, self.nn, self.cid, pt)
        return nll_from_factor(self.nn, A, Dinv, np.asarray(y, dtype=np.float64)[self.perm], s2)[0]

    def nll_and_grad_profiled(self, log_pars, y):
        """One L-BFGS objective call with the error variance profiled out (optim_utils.h:244-340):
        log_pars = log(sigma1^2/sigma2), log(range_transformed). Returns (negll, grad(2), sigma2)."""
        pt = np.exp(np.asarray(log_pars, dtype=np.float64))
        yo = np.asarray(y, dtype=np.float64)[self.perm]
        A, Dinv, Ag, Dg, _ = factor(self.coords, self.nn, self.cid, pt, calc_grad=True)
        _, ypy, ld = nll_from_factor(self.nn, A, Dinv, yo, 1.0)
        s2 = ypy / self.n  # ProfileOutSigma2, re_model_template.h:2640
        negll = ypy / 2. / s2 + ld / 2. + self.n / 2. * (np.log(s2) + np.log(2 * np.pi))
        g = grad_from_factor(self.nn, A, Dinv, Ag, Dg, yo, s2)
        return negll, g, s2

    def grad_response(self, cov_pars, y):
        """Psi^-1 y in the ORIGINAL data order: what REModel::CalcGradient writes back (re_model_template.h:3298)."""
        s2, pt = transform_cov_pars(cov_pars, self.cov_function, self.shape)
        A, Dinv, _, _, _ = factor(self.coords, self.nn, self.cid, pt)
        ya = yaux(self.nn, A, Dinv, np.asarray(y, dtype=np.float64)[self.perm])
        out = np.empty(self.n)
        out[self.perm] = ya
        return out, s2


def dense_neg_log_likelihood(coords, cov_pars, y, cov_function="matern", cov_fct_shape=1.5):
    coords = np.asarray(coords, dtype=np.float64)
    n, d = coords.shape
    s2, pt = transform_cov_pars(cov_pars, cov_function, cov_fct_shape)
    cm = np.asfortranarray(coords)
    out = np.empty(3)
    y = np.ascontiguousarray(y, dtype=np.float64)
    rc = lib().orc_dense_nll(_p(cm), C.c_int(n), C.c_int(d), C.c_int(cov_id(cov_function, cov_fct_shape)), _p(pt), _p(y),
                             C.c_double(s2), _p(out))
    if rc != 0:
        raise FloatingPointError("dense Cholesky failed")
    return out[0]


# ---- long-double per-row reference with error bounds (orc_vecchia_rows_ld)
ROWS_NOUT = 24
ROWS_COLS = ["D", "By", "u", "quad", "logD", "t3", "t4", "t5", "t6", "t7", "t8",
             "bD", "bBy", "bu", "bquad", "blogD", "bt3", "bt4", "bt5", "bt6", "bt7", "bt8", "kappa", "eps"]
# relative error of one fp64 covariance evaluation (exp to 2 ulp, the Matern polynomial, the products) and of one distance (d
# rounded squares summed, the square root, the pre-scaling by the range) in units of u = 2^-53: the c_v and c_r of the bound
COV_EVAL_ULPS = 8.


def dist_ulps(d):
    return d + 4.


def rows_ld(coords, nn_rows, cid, var, range_, diag_nb, diag_obs, y, row_begin=0, qcoords=None, cov_mult=1.0, drop=None):
    """Rows [row_begin, row_begin + len(nn_rows)) of the Vecchia factor in long double, with first-order bounds of an fp64
    evaluation (oracle/vecchia_oracle.c: orc_vecchia_rows_ld). coords (n, d) in Vecchia order; nn_rows the neighbour rows of these
    rows; qcoords (nrows, d): prediction rows (own point = query, y_i = 0; pass diag_obs = var). cov_mult / drop = (row, a, b):
    deliberate faults. Returns (dict column -> (nrows,) array, A (nrows, m), bound of A (nrows, m), number of bad rows)."""
    coords = np.asarray(coords, dtype=np.float64)
    n, d = coords.shape
    nn_rows = np.ascontiguousarray(nn_rows, dtype=np.int32)
    nrows, m = nn_rows.shape
    cm = np.asfortranarray(coords)
    qc = None if qcoords is None else np.asfortranarray(np.asarray(qcoords, dtype=np.float64).reshape(nrows, d))
    yy = np.ascontiguousarray(np.zeros(n) if y is None else y, dtype=np.float64)
    out = np.empty((nrows, ROWS_NOUT)); A = np.empty((nrows, m)); bA = np.empty((nrows, m))
    dr = None if drop is None else np.ascontiguousarray(drop, dtype=np.int64)
    L = lib()
    L.orc_vecchia_rows_ld.restype = C.c_int
    bad = L.orc_vecchia_rows_ld(
        _p(cm), C.c_int64(n), C.c_int(d), C.c_int(m), _p(nn_rows, C.c_int32), C.c_int(cid), C.c_double(var), C.c_double(range_),
        C.c_double(diag_nb), C.c_double(diag_obs), _p(yy), None if qc is None else _p(qc), C.c_int64(row_begin), C.c_int64(nrows),
        C.c_double(COV_EVAL_ULPS), C.c_double(dist_ulps(d)), C.c_double(cov_mult), None if dr is None else _p(dr, C.c_int64),
        _p(out), _p(A), _p(bA))
    return {k: out[:, j] for j, k in enumerate(ROWS_COLS)}, A, bA, bad


# ---- long-double per-row reference of the anisotropic gradient pass (orc_vecchia_rows_aniso_ld)
ANISO_COLS = ["D", "By", "u", "quad", "logD", "bD", "bBy", "bu", "bquad", "blogD", "kappa", "eps"]


def share_ulps(d, d_c):
    """extra relative error, in units of u, of one group entry g S_c / r^2 of the device over the isotropic derivative g: the
    division (1), S_c (d_c differences and their fused squares summed: d_c + 2), the r^2 it is divided by (d + 2) and the final
    multiply (1)"""
    return d + d_c + 6.


def rows_aniso_ld(coords_scaled, nn_rows, cid, var, group_of_coord, y, row_begin=0, group_mult=None, swap=None, drop=None,
                  unmasked=None):
    """Rows [row_begin, row_begin + len(nn_rows)) of the anisotropic gradient pass in long double at range 1 on the scaled
    coordinates (n, d) in Vecchia order, with first-order bounds of an fp64 evaluation (oracle/vecchia_oracle.c:
    orc_vecchia_rows_aniso_ld). Deliberate faults: group_mult = (c, 1 + delta), swap = (row, c1, c2), drop = (row, c, a, b) (a, b:
    points of the row, its neighbours in slot order then the row itself), unmasked = c. Returns (dict, bad): the columns of
    ANISO_COLS, "terms" (nrows, 3 (1 + C)) in the order of the device's sums 3.. and "bterms" their bounds."""
    coords = np.asarray(coords_scaled, dtype=np.float64)
    n, d = coords.shape
    nn_rows = np.ascontiguousarray(nn_rows, dtype=np.int32)
    nrows, m = nn_rows.shape
    grp = np.ascontiguousarray(group_of_coord, dtype=np.int32)
    ng = int(grp.max()) + 1
    np_ = 1 + ng
    ulps = np.array([share_ulps(d, int(np.sum(grp == c))) for c in range(ng)])
    out = np.empty((nrows, 12 + 6 * np_))
    mg, mult = (-1, 1.) if group_mult is None else (int(group_mult[0]), float(group_mult[1]))
    sw = None if swap is None else np.ascontiguousarray(swap, dtype=np.int64)
    dr = None if drop is None else np.ascontiguousarray(drop, dtype=np.int64)
    L = lib()
    L.orc_vecchia_rows_aniso_ld.restype = C.c_int
    bad = L.orc_vecchia_rows_aniso_ld(
        _p(np.asfortranarray(coords)), C.c_int64(n), C.c_int(d), C.c_int(m), _p(nn_rows, C.c_int32), C.c_int(cid), C.c_double(var),
        _p(grp, C.c_int32), C.c_int(ng), _p(np.ascontiguousarray(y, dtype=np.float64)), C.c_int64(row_begin), C.c_int64(nrows),
        C.c_double(COV_EVAL_ULPS), C.c_double(dist_ulps(d)), _p(ulps), C.c_int(mg), C.c_double(mult),
        None if sw is None else _p(sw, C.c_int64), None if dr is None else _p(dr, C.c_int64), C.c_int(-1 if unmasked is None else unmasked),
        _p(out))
    r = {k: out[:, j] for j, k in enumerate(ANISO_COLS)}
    r["terms"] = out[:, 12:12 + 3 * np_]
    r["bterms"] = out[:, 12 + 3 * np_:]
    return r, bad


# ---- long-double per-row reference of the factor derivatives (orc_vecchia_rows_dfactor_ld)
DF_COLS = ["D", "bD", "dD0", "bdD0", "dD1", "bdD1", "kappa", "eps", "rho0", "rho1"]
# relative error of one fp64 evaluation of the range derivative's closed form in units of u: the covariance's (COV_EVAL_ULPS) and
# up to four more products (range, distance and variance factors)
GRAD_EVAL_ULPS = COV_EVAL_ULPS + 4.
# the kernels' exp(-x) saturates at exp(-700) (vecchia_factor.cuh: exp_neg): the absolute error of exp(-x) for x > 700
EXP_FLOOR = math.exp(-700.)


def rows_dfactor_ld(coords, nn_rows, cid, var, range_, diag_nb, diag_obs, row_begin=0, range_mult=1.0, drop=None, g1_diag=0.0,
                    g0_shift=0.0):
    """Rows [row_begin, row_begin + len(nn_rows)) of the factor derivatives w.r.t. log var (k = 0) and log range (k = 1) in long
    double, dA_k = S_NN^-1 (g_k - G_k,NN A) and dD_k = b^T G_k b, with first-order bounds of an fp64 evaluation whose exp(-x) may
    saturate at EXP_FLOOR (oracle/vecchia_oracle.c: orc_vecchia_rows_dfactor_ld). diag_nb / diag_obs as rows_ld: var + 1 twice for the Gaussian factor,
    var (1 + 1e-10) and var for the latent one. Deliberate faults: range_mult scales the range derivative, drop = (row, a, b) removes
    one pair from it, g1_diag puts a value on its neighbour diagonal, g0_shift moves the variance derivative's diagonal. Returns
    (dict of DF_COLS -> (nrows,), dA (2, nrows, m), bound of dA (2, nrows, m), number of bad rows)."""
    coords = np.asarray(coords, dtype=np.float64)
    n, d = coords.shape
    nn_rows = np.ascontiguousarray(nn_rows, dtype=np.int32)
    nrows, m = nn_rows.shape
    out = np.empty((nrows, len(DF_COLS))); dA = np.empty((2, nrows, m)); bdA = np.empty((2, nrows, m))
    dr = None if drop is None else np.ascontiguousarray(drop, dtype=np.int64)
    L = lib()
    L.orc_vecchia_rows_dfactor_ld.restype = C.c_int
    bad = L.orc_vecchia_rows_dfactor_ld(
        _p(np.asfortranarray(coords)), C.c_int64(n), C.c_int(d), C.c_int(m), _p(nn_rows, C.c_int32), C.c_int(cid), C.c_double(var),
        C.c_double(range_), C.c_double(diag_nb), C.c_double(diag_obs), C.c_int64(row_begin), C.c_int64(nrows),
        C.c_double(COV_EVAL_ULPS), C.c_double(dist_ulps(d)), C.c_double(GRAD_EVAL_ULPS), C.c_double(EXP_FLOOR), C.c_double(range_mult),
        None if dr is None else _p(dr, C.c_int64), C.c_double(g1_diag), C.c_double(g0_shift), _p(out), _p(dA), _p(bdA))
    return {k: out[:, j] for j, k in enumerate(DF_COLS)}, dA, bdA, bad
