"""Every Laplace-Vecchia operator and solve kernel (gpboost_b200/csrc/dev/laplace.cuh) against an extended-precision reference.

`gpbdev_vecchia_laplace_apply` factors the latent model, installs W and dw = D^-1 + W and runs one operator through the same
dispatch the evaluation uses:
  op 0  D^-1 B X                  lap_mv_B      mv_B_kernel (G = ceil(t/32) column groups)
  op 1  B^T X + W X2, dots        lap_mv_Bt     mv_Bt_kernel
  op 2  (B^T D^-1 B + W) X, dots  lap_apply_op  t = 1: v_mv_B_kernel + v_mv_Bt_kernel, else ops 0 and 1
  op 3  P^-1 X, dots              lap_precond   t = 1: v_trs_bwd_kernel + v_trs_fwd_kernel, else trs_bwd_kernel + trs_fwd_kernel
  op 4  B^-T X                    the first solve of op 3
  op 5  B_grad X                  mv_Bg_kernel
  op 6  X2 + B_grad^T X           mv_Bgt_kernel with accumulate
with B = I - A, B_grad = -dA, P = B^T (D^-1 + W) B. The reference restates each operator in np.longdouble from the device's own
A, D^-1 and dA (read back with gpbdev_vecchia_latent_factor_grad, the same factor pass): B and B_grad products by gather, B^T
products by a scatter-add over the CSC entries, triangular solves by level-scheduled substitution vectorised over the t columns.
The chains of 1e5 rows are solved in fp64 by scipy.sparse.linalg.spsolve_triangular instead; there the bar below is doubled to
cover the reference's own rounding, which obeys the same bound.

Bars (derived from the standard rounding-error bounds, u = 2^-53, gamma_K = K u / (1 - K u); not fitted to any run):
  * Products. An entry that sums K terms, each at most one product, in any order is within gamma_K * M of the exact value, M = the
    same expression with every term replaced by its absolute value. Bar = 2 gamma_(K+1) M: K = the row's (column's) real entries
    + 2 covers the diagonal term, the W term, and the D^-1 scaling; the factor 2 leaves room for fused multiply-adds.
  * Solves. Substitution with the unit triangular L = I - A gives (L + dL) x^ = b, |dL| <= gamma_K |L| row by row, hence
    |x - x^| <= (I - |A|)^-1 diag(gamma_K) (I + |A|) |x^| (the Neumann series of the nilpotent A bounds |L^-1| by (I - |A|)^-1),
    evaluated with one more triangular solve on |A|; the transpose for B^-T. K = the row's (column's) entries + 2 (the division
    by dw adds one rounding to the right-hand side). Bar = 2 times that. P^-1 R propagates the bar of Y = B^-T R through the
    division by dw and the forward solve: (I - |A|)^-1 [diag(gamma_K)(I + |A|)|Z| + (u |Y| + bar_Y) / dw]. The product
    B^T D^-1 B + W carries the bar of D^-1 B X through |B^T|.
  * Dots. sum_j x_j v_j over the n rows: sum_j |x_j| bar_j (the error of v) + 2 gamma_n sum_j |x_j| |v_j| (per-warp partials
    and the fixed-order column reduction add at most n - 1 times).
  * P^-1 R again: P applied to the result in fp64 gives back R within |P| bar_Z + 2 gamma_(K_row + K_col + 3) |P| |Z|, with
    |P| <= (I + |A|^T) dw (I + |A|).
Every output must also be free of the solves' sentinel word 0x7ff8dead0badf00d, and a second call must be bit-identical.

The cases reach every dispatch bucket (test_cases_reach_every_dispatch_bucket restates the dispatch and checks it without a GPU):
t in {1, 2, 3, 31, 32, 33, 50, 63, 64, 65, 96, 97, 127, 128} (G = 1 ... 4), m in {1, 2, 5, 15, 16, 17, 29, 30}, n from 2 and
m + 1 (every row padded) up to 1e5, d in {1, 2, 3, 4} (Morton order at d = 2 and 3, index order at d = 1 and 4), W = 0,
W in (0, 0.25] and D^-1 spread over several decades, and hand-built neighbour patterns: a chain (depth n - 1, up to n = 1e5), a
star (column 0 has n - 1 entries), columns of exactly 15, 16, 17, 31, 32, 33, 127, 128 and 129 entries (around trs_bwd's 16-entry
batches, mv_Bt's 32-entry chunks and v_trs_bwd's 128-entry unrolled loop) and a comb (depth 1: every row depends on the first 30
rows).

End to end, GPModel at num_rand_vec_trace = t for t in {1, 2, 31, 32, 33, 64, 65, 97, 128} runs against oracle.laplace with the
same probe vectors: equal Newton, CG and SLQ iteration counts, log-det within 1e-8, NLL within 1e-9, mode within 1e-5 (the bars of
test_laplace_gpu.py::test_mode_and_iterations_match_oracle), and the gradient within 1e-6 of max|g| of the oracle's iterative
gradient."""
import ctypes as C
import functools

import numpy as np
import pytest

import datagen
from oracle import laplace as ol
from oracle import vecchia as ov

U = 2.0 ** -53
LD = np.longdouble
SENTINEL = 0x7ff8dead0badf00d
T_ALL = (1, 2, 3, 31, 32, 33, 50, 63, 64, 65, 96, 97, 127, 128)
OP_NAMES = ("DinvBX", "BtX+WX2", "SigmaI+W", "Pinv", "Bt_inv", "BgX", "X2+BgtX")
COL_COUNTS = (15, 16, 17, 31, 32, 33, 127, 128, 129)
WORST = {}  # op name -> worst error / bar ratio seen in this session


def gamma(k):
    k = np.asarray(k, dtype=np.float64)
    return k * U / (1. - k * U)


# ------------------------------------------------------------------------------------------------------------ patterns
def pad_rows(rows, m):
    nn = np.full((len(rows), m), -1, dtype=np.int32)
    for i, r in enumerate(rows):
        nn[i, :len(r)] = r
    return nn


def chain_nn(n):
    return pad_rows([[i - 1] if i else [] for i in range(n)], 1)


def star_nn(n, m):
    """every row depends on row 0 and on its m - 1 nearest predecessors: column 0 has n - 1 entries"""
    return pad_rows([sorted({0} | set(range(max(0, i - m + 1), i))) if i else [] for i in range(n)], m)


def colcount_nn(n):
    """columns 0 ... 8 have exactly COL_COUNTS entries: one from the row after them (every row also depends on its predecessor),
    the rest from consecutive blocks of later rows"""
    hubs = []
    for h, c in enumerate(COL_COUNTS):
        hubs += [h] * (c - 1)
    assert n >= len(COL_COUNTS) + len(hubs) + 10
    rows = [[] for _ in range(n)]
    for i in range(1, n):
        rows[i] = [i - 1]
    for k, h in enumerate(hubs):
        rows[len(COL_COUNTS) + k].append(h)
    return pad_rows(rows, 2)


def comb_nn(n, m=30):
    """the first m rows are unconditioned, every later row depends on exactly those m rows: depth 1, maximal fan-in"""
    return pad_rows([[] if i < m else list(range(m)) for i in range(n)], m)


def depth(nn):
    """length of the longest dependency path"""
    lev = np.zeros(nn.shape[0], dtype=np.int64)
    for i in range(nn.shape[0]):
        j = nn[i][nn[i] >= 0]
        if j.size:
            lev[i] = lev[j].max() + 1
    return int(lev.max())


def col_counts(nn):
    return np.bincount(nn[nn >= 0].ravel(), minlength=nn.shape[0])


# ------------------------------------------------------------------------------------------------- dispatch restatement
def engine_order(d):
    """laplace_ensure: Morton (Z-curve) order at d = 2 and 3, index order otherwise"""
    return "morton" if d in (2, 3) else "index"


def dispatch(op, t, d):
    """kernel buckets (family, G, order) one apply runs: lap_mv_B / lap_mv_Bt / lap_apply_op / lap_precond / the gradient launches.
    Only the gather operator kernels take the engine's row order; the single-vector, solve and gradient kernels go by index."""
    G = (t + 31) // 32
    mv = {("mv", G, engine_order(d))}
    if op in (0, 1):
        return mv
    if op == 2:
        return {("v_mv", 1, "index")} if t == 1 else mv
    if op in (3, 4):
        return {("v_trs", 1, "index")} if t == 1 else {("trs", G, "index")}
    return {("grad", G, "index")}


ALL_BUCKETS = ({("mv", G, o) for G in (1, 2, 3, 4) for o in ("morton", "index")} |
               {("v_mv", 1, "index"), ("v_trs", 1, "index")} | {("trs", G, "index") for G in (1, 2, 3, 4)} |
               {("grad", G, "index") for G in (1, 2, 3, 4)})


# ------------------------------------------------------------------------------------------------------------ the cases
# (name, n, d, m, pattern, ts, W regime, covariance id); pattern "knn" = the engine's own neighbour search
CASES = [
    ("tsweep", 600, 2, 15, "knn", T_ALL, "small", 0),
    ("tsweep-index", 500, 4, 15, "knn", (1, 3, 33, 65, 97, 128), "small", 1),
    ("n2-m1", 2, 1, 1, "knn", (1, 2, 33), "small", 0),
    ("n3-m2", 3, 4, 2, "knn", (1, 2, 65), "small", 0),
    ("n6-m5", 6, 3, 5, "knn", (1, 3, 97), "small", 1),
    ("n16-m15", 16, 2, 15, "knn", (1, 2, 64), "small", 0),
    ("n17-m16", 17, 1, 16, "knn", (1, 32, 128), "small", 0),
    ("n18-m17", 18, 1, 17, "knn", (1, 33), "small", 0),
    ("n30-m29", 30, 3, 29, "knn", (1, 63), "small", 0),
    ("n31-m30", 31, 4, 30, "knn", (1, 96), "small", 0),
    ("m30-n5000", 5000, 2, 30, "knn", (1, 50), "small", 0),
    ("m17-n3000", 3000, 3, 17, "knn", (1, 33), "small", 1),
    ("m5-n2000", 2000, 1, 5, "knn", (1, 65), "small", 0),
    ("m16-n2500", 2500, 4, 16, "knn", (1, 32), "small", 0),
    ("m1-n1500", 1500, 2, 1, "knn", (1, 97), "small", 0),
    ("m2-n1000", 1000, 3, 2, "knn", (1, 64, 127), "small", 0),
    ("m29-n1200", 1200, 1, 29, "knn", (1, 128), "small", 1),
    ("m15-n900", 900, 4, 15, "knn", (1, 31), "zero", 0),
    ("w0-d2", 1000, 2, 10, "knn", (1, 64), "zero", 0),
    ("dinv-spread", 1000, 2, 10, "knn", (1, 33), "small", 3),
    ("chain-3000", 3000, 2, 1, "chain", (1, 2, 65), "small", 0),
    ("chain-1e5", 100000, 2, 1, "chain", (1, 50), "small", 0),
    ("star-5000", 5000, 2, 5, "star", (1, 50), "small", 0),
    ("colcounts", 600, 2, 2, "cols", (1, 3, 33), "small", 0),
    ("colcounts-index", 600, 4, 2, "cols", (1, 64), "zero", 0),
    ("comb-3000", 3000, 2, 30, "comb", (1, 64), "small", 0),
]
CASE_T = [(c, t) for c in CASES for t in c[5]]


def case_coords(name, n, d, pattern):
    """distinct points; the chain and the star run along a path (x increases with the index), so that a row's predecessors are
    its spatial neighbours and the coefficients of the long dependency paths are large"""
    rng = np.random.default_rng(sum(map(ord, name)))
    if d == 1:
        co = ((rng.permutation(n) + 0.5 * rng.random(n)) / n)[:, None]
    elif pattern in ("chain", "star"):
        co = np.column_stack([(np.arange(n) + 0.5 * rng.random(n)) / n, 0.05 * rng.random((n, d - 1))])
    else:
        co = rng.random((n, d))
    return np.ascontiguousarray(co)


def case_nn(n, m, pattern):
    return {"chain": lambda: chain_nn(n), "star": lambda: star_nn(n, m), "cols": lambda: colcount_nn(n),
            "comb": lambda: comb_nn(n, m)}[pattern]()


def case_pars(n, d, pattern, cid):
    """(var, transformed range). The range follows the neighbour spacing 2 n^(-1/d) for the engine's own neighbour sets (with the
    Gaussian kernel the conditional variances then span several decades), is 50 path steps for the chain (coefficients ~0.98 along
    the whole chain) and 0.5 for the other hand-built patterns, whose neighbours are not the nearest points."""
    rho = {"knn": 2. * n ** (-1. / d), "chain": 50. / n}.get(pattern, 0.5)
    if cid == 3:
        return 1.0, 1. / rho ** 2
    return 0.7, {0: 1., 1: np.sqrt(3.), 2: np.sqrt(5.)}[cid] / rho


# ---------------------------------------------------------------------------------------------- longdouble reference
class Ref:
    """B = I - A, B_grad = -dA in the Vecchia order, products and substitutions in longdouble (fp64 + scipy for long chains)"""

    def __init__(self, nn, A, Dinv, dA, W, scipy_solves):
        n, m = nn.shape
        self.n, self.mask = n, nn >= 0
        self.idx = np.where(self.mask, nn, 0)
        self.A = np.where(self.mask, A, 0.).astype(LD)
        self.dA = np.where(self.mask, dA, 0.).astype(LD)
        self.Dinv, self.W = Dinv.astype(LD), W.astype(LD)
        self.dw = (Dinv + W).astype(LD)  # the device adds in fp64: same value
        rows = np.repeat(np.arange(n), m)[self.mask.ravel()]
        cols = nn.ravel()[self.mask.ravel()]
        o = np.argsort(cols, kind="stable")
        self.erow, self.ecol, self.epos = rows[o], cols[o], np.flatnonzero(self.mask.ravel())[o]
        self.krow = self.mask.sum(1)
        self.kcol = np.bincount(cols, minlength=n)
        self.scipy = scipy_solves
        if scipy_solves:
            import scipy.sparse as sp
            self.Am = sp.csr_matrix((A.ravel()[self.mask.ravel()], (rows, cols)), shape=(n, n))
            return
        lev = np.zeros(n, dtype=np.int64)  # forward levels: longest path to a row without dependencies
        for i in range(n):
            j = nn[i][self.mask[i]]
            if j.size:
                lev[i] = lev[j].max() + 1
        self.flev = [np.flatnonzero(lev == k) for k in range(lev.max() + 1)]
        blev = np.zeros(n, dtype=np.int64)  # backward levels: longest path to a row nobody depends on
        for i in range(n - 1, -1, -1):
            for j in nn[i][self.mask[i]]:
                blev[j] = max(blev[j], blev[i] + 1)
        self.blev = []
        for k in range(blev.max() + 1):
            cset = np.flatnonzero(blev == k)
            sel = np.flatnonzero(np.isin(self.ecol, cset))  # entries of these columns, sorted by column
            self.blev.append((cset, sel))

    # products --------------------------------------------------------------------------------------------------------
    def gather(self, coef, X):  # sum_k coef[i,k] X[nn[i,k]]
        return np.einsum("ik,ikc->ic", coef, X[self.idx])

    def scatter(self, coef_e, X):  # sum over the CSC entries of column j of coef_e X[row]
        out = np.zeros(X.shape, dtype=LD)
        if coef_e.size:
            starts = np.flatnonzero(np.r_[True, self.ecol[1:] != self.ecol[:-1]])
            out[self.ecol[starts]] = np.add.reduceat(coef_e[:, None] * X[self.erow], starts, axis=0)
        return out

    def a_e(self, coef):
        return coef.ravel()[self.epos]

    # solves: fwd  z = r + sum_k a[i,k] z[nn[i,k]]  (B z = r);  bwd  y_j = r_j + sum_e a_e y_row (B^T y = r) ------------------
    def fwd(self, R, absA=False):
        if self.scipy:
            return self._sp(R, absA, lower=True)
        a = np.abs(self.A) if absA else self.A
        Z = np.zeros(R.shape, dtype=LD)
        for rows in self.flev:
            Z[rows] = R[rows] + np.einsum("ik,ikc->ic", a[rows], Z[self.idx[rows]])
        return Z

    def bwd(self, R, absA=False):
        if self.scipy:
            return self._sp(R, absA, lower=False)
        a = self.a_e(np.abs(self.A) if absA else self.A)
        Y = np.array(R, dtype=LD)
        for cset, sel in self.blev:
            if sel.size:
                ec = self.ecol[sel]
                starts = np.flatnonzero(np.r_[True, ec[1:] != ec[:-1]])
                Y[ec[starts]] += np.add.reduceat(a[sel][:, None] * Y[self.erow[sel]], starts, axis=0)
        return Y

    def _sp(self, R, absA, lower):
        import scipy.sparse as sp
        from scipy.sparse.linalg import spsolve_triangular
        Am = abs(self.Am) if absA else self.Am
        Bm = (sp.identity(self.n, format="csr") - Am).tocsr()
        if not lower:
            Bm = Bm.T.tocsr()
        out = spsolve_triangular(Bm, np.asarray(R, dtype=np.float64), lower=lower, unit_diagonal=True)
        return np.asarray(out, dtype=LD).reshape(R.shape)

    # |B| and |B^T| applications for the bars
    def absB(self, X):
        return np.abs(X) + self.gather(np.abs(self.A), np.abs(X))

    def absBt(self, X):
        return np.abs(X) + self.scatter(self.a_e(np.abs(self.A)), np.abs(X))


def check(name, got, want, bar, what):
    """every entry within its bar; records the worst error / bar ratio of the operator"""
    err = np.abs(np.asarray(got, dtype=LD) - want)
    bar = np.asarray(bar, dtype=LD)
    bad = ~(err <= bar)
    assert not bad.any(), "%s: %d entries outside the bar, first at %s: got %r want %r bar %r" % (
        what, int(bad.sum()), np.argwhere(bad)[0], got[tuple(np.argwhere(bad)[0])], float(want[tuple(np.argwhere(bad)[0])]),
        float(bar[tuple(np.argwhere(bad)[0])]))
    pos = bar > 0
    ratio = float((err[pos] / bar[pos]).max()) if pos.any() else 0.
    WORST[name] = max(WORST.get(name, 0.), ratio)
    return ratio


def no_sentinel(a, what):
    words = np.ascontiguousarray(a).view(np.uint64)
    hit = np.flatnonzero(words == np.uint64(SENTINEL))
    assert hit.size == 0, "%s: %d output words still carry the solve's sentinel 0x7ff8dead0badf00d (first at flat index %d)" % (
        what, hit.size, hit[0])


# ------------------------------------------------------------------------------------------------------------ device
def P(a, t=C.c_double):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


@pytest.fixture(scope="module")
def lib(product_lib):
    assert product_lib.gpbdev_device_count() > 0, "no CUDA device visible — GPU tests need an H100"
    return product_lib


def chk(lib, rc):
    assert rc == 0, lib.gpbdev_last_error().decode()


def create(lib, co, m, nn=None):
    n, d = co.shape
    h = C.c_void_p()
    perm = np.arange(n, dtype=np.int32)
    chk(lib, lib.gpbdev_vecchia_create(C.byref(h), 0, C.c_int64(n), d, m, P(co), P(perm, C.c_int32),
                                       None if nn is None else P(np.ascontiguousarray(nn, dtype=np.int32), C.c_int32),
                                       C.c_int64(0), C.c_int64(n)))
    return h


def apply(lib, h, cid, var, rt, op, W, X, X2=None):
    n, t = X.shape
    out = np.empty((n, t)); dots = np.empty(t)
    chk(lib, lib.gpbdev_vecchia_laplace_apply(h, C.c_int(cid), C.c_double(var), C.c_double(rt), C.c_int(op), C.c_int(t), P(W),
                                              P(X), P(X2), P(out), P(dots)))
    return out, dots


@functools.lru_cache(maxsize=None)
def case_inputs(name):
    (_, n, d, m, pattern, ts, wmode, cid), = [c for c in CASES if c[0] == name]
    co = case_coords(name, n, d, pattern)
    nn = None if pattern == "knn" else case_nn(n, m, pattern)
    rng = np.random.default_rng(n + m)
    W = np.zeros(n) if wmode == "zero" else 0.25 * (1. - rng.random(n))  # (0, 0.25]
    return co, nn, W


def dot_bar(x, v, bar_v):
    return (np.abs(x) * bar_v).sum(0) + 2. * gamma(x.shape[0]) * (np.abs(x) * np.abs(v)).sum(0)


@pytest.mark.gpu
@pytest.mark.parametrize("case,t", CASE_T, ids=["%s-t%d" % (c[0], t) for c, t in CASE_T])
def test_operator_matches_extended_precision_reference(lib, case, t):
    name, n, d, m, pattern, _, wmode, cid = case
    co, nn, W = case_inputs(name)
    var, rt = case_pars(n, d, pattern, cid)
    h = create(lib, co, m, nn)
    try:
        nn_d = np.empty((n, m), dtype=np.int32)
        chk(lib, lib.gpbdev_vecchia_get_nn(h, P(nn_d, C.c_int32)))
        if nn is not None:
            assert np.array_equal(nn_d, nn)
        A = np.empty((n, m)); Dinv = np.empty(n); dA = np.empty((n, m)); dD = np.empty(n)
        chk(lib, lib.gpbdev_vecchia_latent_factor_grad(h, C.c_int(cid), C.c_double(var), C.c_double(rt), P(A), P(Dinv), P(dA), P(dD)))
        assert np.all(np.isfinite(A)) and np.all(np.isfinite(dA)) and np.all(Dinv > 0) and np.all(np.isfinite(Dinv))
        if name == "dinv-spread":
            assert Dinv.max() / Dinv.min() >= 1e3
        rng = np.random.default_rng(t * 1000 + n)
        X = rng.standard_normal((n, t)); X2 = rng.standard_normal((n, t))

        def run(op, X2arg=None):
            out, dots = apply(lib, h, cid, var, rt, op, W, X, X2arg)
            no_sentinel(out, "%s %s t=%d" % (name, OP_NAMES[op], t))
            if op in (1, 2, 3):
                no_sentinel(dots, "%s %s dots t=%d" % (name, OP_NAMES[op], t))
            out2, dots2 = apply(lib, h, cid, var, rt, op, W, X, X2arg)
            assert out.tobytes() == out2.tobytes(), "%s: repeated call differs" % OP_NAMES[op]
            if op in (1, 2, 3):
                assert dots.tobytes() == dots2.tobytes(), "%s: repeated dots differ" % OP_NAMES[op]
            return out, dots

        verify_operators(Ref(nn_d, A, Dinv, dA, W, scipy_solves=n > 20000), A, Dinv, W, X, X2, run)
        print("WORST-RATIOS %s t=%d %s" % (name, t, " ".join("%s=%.2e" % kv for kv in sorted(WORST.items()))))
    finally:
        lib.gpbdev_vecchia_free(h)


def verify_operators(R, A, Dinv, W, X, X2, run):
    """every operator's output (run(op, X2) -> (out, dots)) against the longdouble reference R, within the bars of the docstring"""
    c2 = 4. if R.scipy else 2.  # the fp64 reference solves obey the same bound as the device's
    XL, X2L, WL = X.astype(LD), X2.astype(LD), W.astype(LD)[:, None]
    Dv = R.Dinv[:, None]
    gr, gc = gamma(R.krow + 3)[:, None], gamma(R.kcol + 3)[:, None]
    # op 0: D^-1 B X
    out, _ = run(0)
    T = Dv * (XL - R.gather(R.A, XL))
    bar_T = 2. * gr * Dv * R.absB(XL)
    check(OP_NAMES[0], out, T, bar_T, "D^-1 B X")
    # op 1: B^T X + W X2, dots X2 . out
    out, dots = run(1, X2)
    V = XL - R.scatter(R.a_e(R.A), XL) + WL * X2L
    bar = 2. * gc * (R.absBt(XL) + np.abs(WL * X2L))
    check(OP_NAMES[1], out, V, bar, "B^T X + W X2")
    check(OP_NAMES[1], dots, (X2L * V).sum(0), dot_bar(X2L, out, bar), "B^T X + W X2 dots")
    # op 2: (B^T D^-1 B + W) X, dots X . out
    out, dots = run(2)
    V = T - R.scatter(R.a_e(R.A), T) + WL * XL
    bar = R.absBt(bar_T) + 2. * gc * (R.absBt(T) + np.abs(WL * XL))
    check(OP_NAMES[2], out, V, bar, "(B^T D^-1 B + W) X")
    check(OP_NAMES[2], dots, (XL * V).sum(0), dot_bar(XL, out, bar), "(B^T D^-1 B + W) X dots")
    # op 4: B^-T X
    out, _ = run(4)
    Y = R.bwd(XL)
    check(OP_NAMES[4], out, Y, c2 * R.bwd(gc * R.absBt(out), absA=True), "B^-T X")
    bar_Y = c2 * R.bwd(gc * R.absBt(Y), absA=True)
    # op 3: P^-1 X = B^-1 ((B^-T X) / dw), dots X . out
    out, dots = run(3)
    dwv = R.dw[:, None]
    Z = R.fwd(Y / dwv)
    bar_Z = c2 * R.fwd(gr * R.absB(out) + (U * np.abs(Y) + bar_Y) / dwv, absA=True)
    check(OP_NAMES[3], out, Z, bar_Z, "P^-1 X")
    check(OP_NAMES[3], dots, (XL * Z).sum(0), dot_bar(XL, out, bar_Z), "P^-1 X dots")
    # P applied to the result in fp64 gives back X
    Bz = out - np.einsum("ik,ikc->ic", np.where(R.mask, A, 0.), out[R.idx])
    PZ = Bz * (Dinv + W)[:, None]
    PZ = PZ - np.asarray(R.scatter(R.a_e(R.A), PZ.astype(LD)), dtype=np.float64)
    absP = lambda v: R.absBt(dwv * R.absB(v))
    check(OP_NAMES[3] + "(P Z - R)", PZ, XL, absP(bar_Z) + 2. * gamma(R.kcol + R.krow.max() + 3)[:, None] * absP(out),
          "P (P^-1 X) - X")
    # op 5: B_grad X
    out, _ = run(5)
    check(OP_NAMES[5], out, -R.gather(R.dA, XL), 2. * gr * R.gather(np.abs(R.dA), np.abs(XL)), "B_grad X")
    # op 6: X2 + B_grad^T X (accumulate)
    out, _ = run(6, X2)
    check(OP_NAMES[6], out, X2L - R.scatter(R.a_e(R.dA), XL),
          2. * gc * (np.abs(X2L) + R.scatter(R.a_e(np.abs(R.dA)), np.abs(XL))), "X2 + B_grad^T X")


@pytest.mark.gpu
@pytest.mark.parametrize("d,m", [(2, 10), (3, 20), (2, 30), (3, 30)])
def test_factor_of_rows_padded_beyond_m_matches_oracle(lib, d, m):
    """Supplied neighbour sets may pad any row with -1, also rows i >= m. The factor kernels took every row i >= m of a model with
    m equal to their capacity (10, 20, 30) for a row without dummy slots and built its covariance block from stale shared memory,
    so that D^-1 B X differed between two identical calls. Regression: rows i >= m keep 1 ... m of their
    nearest neighbours; the latent factor and its range derivative (one-observation kernel) and the Gaussian likelihood sums (at
    d = 2, m = 30 the two-observation kernel) must match the oracle and repeat bit for bit."""
    n = 700
    rng = np.random.default_rng(m + d)
    co = np.ascontiguousarray(rng.random((n, d)))
    nn = ov.knn(co, m).astype(np.int32)
    keep = rng.integers(1, m + 1, n)
    for i in range(m, n):
        nn[i, keep[i]:] = -1
    assert (nn[m:] < 0).any(axis=1).mean() > 0.8
    h = create(lib, co, m, nn)
    try:
        _, rt = case_pars(n, d, "knn", 0)
        got = []
        for _ in range(2):
            A = np.empty((n, m)); Dinv = np.empty(n); dA = np.empty((n, m)); dD = np.empty(n)
            chk(lib, lib.gpbdev_vecchia_latent_factor_grad(h, C.c_int(0), C.c_double(0.7), C.c_double(rt), P(A), P(Dinv), P(dA), P(dD)))
            got.append(b"".join(a.tobytes() for a in (A, Dinv, dA, dD)))
        assert got[0] == got[1]
        A0, Dinv0, dA0, dD0, bad = ol.factor_latent_grad(co, nn, 0, 0.7, rt)
        assert bad == 0
        mask = nn >= 0
        for g, w, name in ((np.where(mask, A, 0.), np.where(mask, A0, 0.), "A"), (1. / Dinv, 1. / Dinv0, "D"),
                           (np.where(mask, dA, 0.), np.where(mask, dA0, 0.), "dA"), (dD, dD0, "dD")):
            assert np.max(np.abs(g - w)) <= 1e-8 * np.max(np.abs(w)), name
        y = rng.standard_normal(n)
        s2, pt = ov.transform_cov_pars([0.4, 1.3, 2. * n ** (-1. / d)], "exponential", 0.5)
        chk(lib, lib.gpbdev_vecchia_set_y(h, P(y)))
        out = np.zeros(9)
        chk(lib, lib.gpbdev_vecchia_eval(h, 0, C.c_double(pt[0]), C.c_double(pt[1]), 1, P(out)))
        Af, Dinvf, _, _, bad = ov.factor(co, nn, 0, pt)
        ref = ov.nll_from_factor(nn, Af, Dinvf, y, s2)
        assert bad == 0 and abs(out[0] - ref[1]) <= 1e-8 * abs(ref[1]) and abs(out[1] - ref[2]) <= 1e-8 * max(1., abs(ref[2]))
    finally:
        lib.gpbdev_vecchia_free(h)


@pytest.mark.gpu
def test_apply_refuses_bad_requests_and_leaves_the_evaluation_clean(lib):
    n, m, t = 900, 10, 50
    X, y, _ = datagen.binary_synth(n, 5, False)
    co = np.ascontiguousarray(X)
    h = create(lib, co, m)
    h2 = create(lib, co, m)
    hb = create(lib, np.ascontiguousarray(X[:100]), 31)
    try:
        W = np.full(n, 0.1); Xm = np.ones((n, 4)); out = np.empty((n, 4)); dots = np.empty(4)
        f = lib.gpbdev_vecchia_laplace_apply

        def refused(rc, msg):
            assert rc != 0
            assert msg in lib.gpbdev_last_error().decode()

        refused(f(h, 0, C.c_double(1.), C.c_double(10.), 7, 4, P(W), P(Xm), P(Xm), P(out), P(dots)), "unknown operator 7")
        refused(f(h, 0, C.c_double(1.), C.c_double(10.), -1, 4, P(W), P(Xm), P(Xm), P(out), P(dots)), "unknown operator -1")
        for bad_t in (0, 129):
            refused(f(h, 0, C.c_double(1.), C.c_double(10.), 0, bad_t, P(W), P(Xm), P(Xm), P(out), P(dots)), "[1, 128]")
        refused(f(hb, 0, C.c_double(1.), C.c_double(10.), 0, 4, P(W[:100]), P(Xm[:100]), None, P(out[:100]), None), "<= 30")
        refused(f(h, 0, C.c_double(1.), C.c_double(10.), 0, 4, None, P(Xm), None, P(out), None), "null buffer")
        refused(f(h, 0, C.c_double(1.), C.c_double(10.), 0, 4, P(W), None, None, P(out), None), "null buffer")
        refused(f(h, 0, C.c_double(1.), C.c_double(10.), 0, 4, P(W), P(Xm), None, None, None), "null buffer")
        refused(f(h, 0, C.c_double(1.), C.c_double(10.), 1, 4, P(W), P(Xm), None, P(out), P(dots)), "null buffer")
        refused(f(h, 0, C.c_double(1.), C.c_double(10.), 6, 4, P(W), P(Xm), None, P(out), None), "null buffer")
        refused(f(h, 0, C.c_double(1.), C.c_double(10.), 3, 4, P(W), P(Xm), None, P(out), None), "null buffer")
        # an evaluation after every operator equals the evaluation of an untouched engine, bit for bit
        probes = np.asfortranarray(np.random.default_rng(3).standard_normal((n, t)))
        cfg = np.array([1000., 1e-8, 20., 1000., 1000., 1e-2, 1., 1e-4])
        outs = []
        for hh, touch in ((h, True), (h2, False)):
            chk(lib, lib.gpbdev_vecchia_set_y(hh, P(y)))
            chk(lib, lib.gpbdev_vecchia_laplace_set_probes(hh, P(probes), t))
            chk(lib, lib.gpbdev_vecchia_laplace_keep_solutions(hh, 1))
            if touch:
                o6 = np.empty(6)
                chk(lib, lib.gpbdev_vecchia_laplace_eval(hh, 1, C.c_double(1.), C.c_double(30.), None, P(cfg), P(o6)))
                for op in range(7):
                    for tt in (1, 3, 64):
                        Xt = np.ones((n, tt))
                        apply(lib, hh, 0, 0.5, 7., op, np.full(n, 0.2), Xt, Xt)
                g = np.empty(3)
                assert lib.gpbdev_vecchia_laplace_grad(hh, 1, C.c_double(1.), C.c_double(30.), P(cfg), P(g)) != 0
                assert "keep_solutions" in lib.gpbdev_last_error().decode()
            o = np.empty(6); g = np.empty(3); mode = np.empty(n)
            chk(lib, lib.gpbdev_vecchia_laplace_eval(hh, 1, C.c_double(1.), C.c_double(30.), None, P(cfg), P(o)))
            chk(lib, lib.gpbdev_vecchia_laplace_grad(hh, 1, C.c_double(1.), C.c_double(30.), P(cfg), P(g)))
            chk(lib, lib.gpbdev_vecchia_laplace_get_mode(hh, P(mode)))
            outs.append((o.tobytes(), g.tobytes(), mode.tobytes()))
        assert outs[0] == outs[1]
    finally:
        for hh in (h, h2, hb):
            lib.gpbdev_vecchia_free(hh)


# ------------------------------------------------------------------------------------------------ end to end, GPModel
# (d, covariance, shape, n, m, offset, t)
E2E = ([(2, "matern", 1.5, 1000, 10, False, t) for t in (1, 2, 31, 32, 33, 64, 65, 97, 128)] +
       [(3, "gaussian", 0., 800, 15, True, t) for t in (1, 33, 65, 128)])


@pytest.mark.gpu
@pytest.mark.parametrize("case", E2E, ids=["d%d-%s%s-t%d" % (c[0], c[1], "-offset" if c[5] else "", c[6]) for c in E2E])
def test_probe_count_end_to_end_matches_oracle(case):
    from gpboost_b200 import GPModel
    d, cov, shape, n, m, offset, t = case
    X, y, off = datagen.binary_synth(n, 60 + d, offset, d=d)
    cp = np.array([1.0, 2. * n ** (-1. / d)])
    gm = GPModel(likelihood="bernoulli_logit", gp_coords=X, cov_function=cov, cov_fct_shape=shape, gp_approx="vecchia",
                 num_neighbors=m, vecchia_ordering="random", seed=d, matrix_inversion_method="iterative")
    gm.set_optim_params({"num_rand_vec_trace": t})  # fresh model: the probes are drawn with run id 0
    negll = C.c_double(0.); g = np.zeros(2)
    offc = None if off is None else np.ascontiguousarray(off)
    rc = gm._LIB.GPB200_EvalLaplaceGradient(gm.handle, P(np.ascontiguousarray(y)), P(cp), P(offc), C.byref(negll), P(g))
    assert rc == 0, gm._LIB.LGBM_GetLastError().decode()
    info = gm.laplace_info()
    mode = gm.laplace_mode()
    vo = ov.VecchiaOracle(X, m, cov, shape, "random", d)
    _, pt = ov.transform_cov_pars([1.0] + list(cp), cov, shape)
    r = ol.grad_negll(vo.coords, vo.nn, vo.cid, cp[0], pt[1], y[vo.perm], fixed_effects=None if off is None else off[vo.perm],
                      method="iterative", num_rand_vec_trace=t)
    assert int(info[1]) == r["newton_it"]
    assert int(info[2]) == r["cg_it"]
    assert int(info[3]) == r["slq_it"]
    mode_oracle = np.empty_like(mode)
    mode_oracle[vo.perm] = r["mode"]
    ratios = dict(logdet=abs(info[4] - r["logdet"]) / (1e-8 * abs(r["logdet"])),
                  negll=abs(negll.value - r["negll"]) / (1e-9 * abs(r["negll"])),
                  mode=np.max(np.abs(mode - mode_oracle)) / (1e-5 * (1. + np.max(np.abs(mode_oracle)))),
                  grad=np.max(np.abs(g - r["grad"])) / (1e-6 * np.abs(r["grad"]).max()))
    print("E2E-RATIOS t=%d d=%d %s" % (t, d, " ".join("%s=%.2e" % kv for kv in sorted(ratios.items()))))
    for k, v in ratios.items():
        assert v <= 1., (k, v, g, r["grad"])


@pytest.mark.gpu
def test_probe_count_above_128_is_refused():
    from gpboost_b200 import GPModel, GPBoostError
    X, y, _ = datagen.binary_synth(300, 4, False)
    gm = GPModel(likelihood="bernoulli_logit", gp_coords=X, gp_approx="vecchia", num_neighbors=10, seed=1)
    gm.set_optim_params({"num_rand_vec_trace": 129})
    with pytest.raises(GPBoostError, match=r"num_rand_vec_trace must be in \[1, 128\]"):
        gm.neg_log_likelihood(np.array([1.0, 0.1]), y)


# ------------------------------------------------------------------------------------------------------- no GPU needed
def test_cases_reach_every_dispatch_bucket():
    reached = {b for (name, n, d, m, pattern, ts, _, _) in CASES for t in ts for op in range(7) for b in dispatch(op, t, d)}
    assert reached == ALL_BUCKETS, ALL_BUCKETS - reached
    assert {t for c in CASES for t in c[5]} == set(T_ALL)
    assert {c[3] for c in CASES} >= {1, 2, 5, 15, 16, 17, 29, 30}
    assert {c[2] for c in CASES} == {1, 2, 3, 4}
    assert any(c[1] == 2 for c in CASES) and all(any(c[1] == m + 1 and c[3] == m for c in CASES) for m in (1, 2, 5, 15, 16, 17, 29, 30))
    assert max(c[1] for c in CASES if c[4] == "knn") == 5000
    assert {c[6] for c in CASES} == {"zero", "small"} and any(c[0] == "dinv-spread" for c in CASES)
    # the long chain runs with the single-vector and the multi-vector solves
    assert {t for c in CASES if c[4] == "chain" and c[1] == 100000 for t in c[5]} == {1, 50}


def test_engineered_patterns_have_the_advertised_shape():
    for n in (3000, 100000):
        assert depth(chain_nn(n)) == n - 1
    nn = star_nn(5000, 5)
    assert col_counts(nn)[0] == 4999 and depth(nn) == 4999
    cc = col_counts(colcount_nn(600))
    assert list(cc[:len(COL_COUNTS)]) == list(COL_COUNTS) and set(cc[len(COL_COUNTS):]) <= {0, 1}
    nn = comb_nn(3000)
    assert depth(nn) == 1 and np.all(col_counts(nn)[:30] == 2970) and np.all(col_counts(nn)[30:] == 0)
    for nn in (chain_nn(50), star_nn(50, 5), colcount_nn(600), comb_nn(100)):
        for i in range(nn.shape[0]):
            r = nn[i][nn[i] >= 0]
            assert np.all(r < i) and len(set(r)) == r.size
        assert np.all(nn >= -1)


def test_create_rejects_neighbour_sets_that_are_not_earlier_rows(product_lib):
    """checked on the host before any device resource is taken (no GPU needed): a dependency on the row itself, on a later row,
    below -1, or twice in one row"""
    lib = product_lib
    n, m = 40, 3
    co = np.random.default_rng(0).random((n, 2))
    good = star_nn(n, m)
    cases = []
    bad = good.copy(); bad[7, 2] = 7; cases.append((bad, "neighbour 7 of row 7 is neither -1 nor an earlier row"))
    bad = good.copy(); bad[7, 2] = 20; cases.append((bad, "neighbour 20 of row 7 is neither -1 nor an earlier row"))
    bad = good.copy(); bad[0, 0] = 0; cases.append((bad, "neighbour 0 of row 0 is neither -1 nor an earlier row"))
    bad = good.copy(); bad[9, 1] = -2; cases.append((bad, "neighbour -2 of row 9 is neither -1 nor an earlier row"))
    bad = good.copy(); bad[9, 2] = bad[9, 1]; cases.append((bad, "neighbour %d appears twice in row 9" % good[9, 1]))
    perm = np.arange(n, dtype=np.int32)
    for nn, msg in cases:
        h = C.c_void_p()
        nn = np.ascontiguousarray(nn, dtype=np.int32)
        rc = lib.gpbdev_vecchia_create(C.byref(h), 0, C.c_int64(n), 2, m, P(co), P(perm, C.c_int32), P(nn, C.c_int32),
                                       C.c_int64(0), C.c_int64(n))
        assert rc != 0 and h.value is None
        assert lib.gpbdev_last_error().decode() == "gpbdev_vecchia_create: " + msg
