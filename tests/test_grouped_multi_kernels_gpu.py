"""The multi-factor grouped engine (K >= 2 crossed or nested random effects, gpboost_b200/csrc/dev/grouped_multi.cuh) against an
extended-precision reference, at the edges of its kernels.

spmm_kernel     Y = diag .* X + Off X; a warp per row, lane c + 32 q owns column c + 32 q of a G x t block (q < kPer = 4, so
                t > 96 runs the fourth lane group); grid-stride over rows, at most 16 SMs CTAs of 8 warps (a second sweep once
                G > 128 SMs rows)
tri_kernel      modes 0 / 1 (forward / backward solve with L D^-1/2, one launch per factor block), 2 (L D^-1/2 X), 3 (D^-1 upper(M) X);
                the same lanes and sweeps over the rows of a block
diag_kernel     diag(M) = 1 / v_k + counts and its scalings; grid-stride over 16 SMs x 256 threads
coldot_kernel   per-column dots over a row range: thread slices of per = ceil(len / 256) rows (a factor of 256 levels: per = 1; 257:
                per = 2; one level: all but one thread idle), then a tree; with no second operand the column sums of |A|
yaux_kernel     (y - Z x) scale, grid-stride over the observations

Cases: t in {1, 31, 32, 33, 64, 65, 127, 128}; K in {2, 3, 5, 8}; variance ratios v in {1e-6, 1e-2, 1, 1e2, 1e6} (the diagonal is
dominated by 1 / v or by the counts); a factor with one level (a dense CSR row, a block of one row), factors with 256 and 257 levels,
a nested pair, a level holding 2^18 observations (co-occurrence counts of that size), level counts above the largest index used
(empty CSR rows, count 0); a crossed case with G = 45 000 levels (a second sweep of spmm and tri_kernel) and one with 600 000
declared levels over 655 360 observations (a second sweep of diag_kernel and yaux_kernel).

Reference: M = Sigma^-1 + Z^T Z from explicit level counts (oracle/grouped_multi.Structure infers them from the data), every
product in np.longdouble. A factor's own levels never co-occur, so L is block lower-triangular with diagonal blocks and each
triangular solve is K vectorised block steps.

Bars and why:
- M X, L D^-1/2 X, D^-1 upper(M) X: |Y - Y_ref| <= 4 eps (w_i + 2) (|op| |X|)_ic, w_i the number of off-diagonal entries of row i:
  one chain of w_i additions plus the roundings of the diagonal scalings (1 / v + count, its inverse and square root);
- P^-1 X by its residual, which holds however ill-conditioned P is: with T = L D^-1/2, |T T^T Z - X| <= 6 eps (w + 2) |T| |T^T| |Z|
  (backward error of each of the two triangular solves), in longdouble; and Z against the float64 oracle at 1e-12 of the largest
  entry where the diagonal dominates (v <= 1e-2);
- CG and Lanczos iteration counts equal to oracle/grouped_multi.evaluate, quadratic form and log-det 1e-9 relative, gradient 1e-7
  relative to its largest entry (the bars of test_grouped_multi_gpu.py), also warm-started (the oracle's cg_vec from x_prev);
- set_y_device bitwise equal to set_y, yaux into a device buffer bitwise equal to the host result, repeated calls bitwise equal;
- yaux against y - Z x with x read back: eps (K + 2) (|y| + sum_k |x_{idx_k}|) scale per observation (K + 1 roundings);
- a right-hand side Z^T y with |Z^T y|_1 < 1e-100 (the reference's THRESHOLD_ZERO_RHS_CG_) gives x = 0 and yaux = y scale exactly."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import grouped_multi as gm

LD = np.longdouble
EPS = np.finfo(np.float64).eps
VS = (1e-6, 1e-2, 1., 1e2, 1e6)
TS = (1, 31, 32, 33, 64, 65, 127, 128)
SMALL = ("K2", "K3", "K5", "K8", "nested", "heavy")
H100_SMS = 132
CFG = (1000, 1000, 1e-2, 0)
DP = C.POINTER(C.c_double)


def structure(kind):
    """(idx K x n int32, declared level counts, response)"""
    rng = np.random.default_rng(sum(map(ord, kind)))

    def used(n, g):  # every one of g levels used, rows scrambled
        return rng.permutation(np.arange(n) % g)

    if kind == "K2":
        n, lv = 3000, [40, 300]
        idx = [used(n, g) for g in lv]
    elif kind == "K3":  # coldot slices per = 1 and 2, and a factor with one level (a dense row, a block of one row)
        n, lv = 6000, [256, 257, 1]
        idx = [used(n, g) for g in lv]
    elif kind == "K5":  # factors 2 and 4 declare more levels than they use: empty CSR rows with count 0
        n, lv = 4000, [17, 1, 95, 256, 40]
        idx = [used(n, g) for g in (17, 1, 90, 256, 33)]
    elif kind == "K8":
        n, lv = 6000, [5, 13, 64, 65, 100, 2, 257, 31]
        idx = [used(n, g) for g in lv]
    elif kind == "nested":
        n, lv = 4000, [50, 400]
        sub = used(n, 400)
        idx = [sub // 8, sub]
    elif kind == "heavy":  # level 0 of factor 0 holds 2^18 observations
        n, lv = (1 << 18) + 3000, [30, 200]
        f0 = np.zeros(n, dtype=np.int64)
        f0[1 << 18:] = 1 + np.arange(3000) % 29
        p = rng.permutation(n)
        idx = [f0[p], used(n, 200)]
    elif kind == "big":  # G = 45 000: spmm and tri_kernel sweep their rows more than once
        n, lv = 300000, [30000, 15000]
        idx = [used(n, g) for g in lv]
    else:
        assert kind == "huge"  # 600 000 declared levels over 655 360 observations: diag_kernel and yaux_kernel sweep twice
        n, lv = 655360, [600000, 3]
        idx = [rng.integers(0, 600000, n), used(n, 3)]
    idx = np.ascontiguousarray(np.stack(idx).astype(np.int32))
    y = sum(rng.standard_normal(g)[i] * (0.5 + k % 3) for k, (g, i) in enumerate(zip(lv, idx))) + 0.4 * rng.standard_normal(n)
    return idx, lv, y


class Ref:
    """M = Sigma^-1 + Z^T Z from explicit level counts; operators in np.longdouble"""

    def __init__(self, idx, levels):
        self.K, self.n = idx.shape
        self.levels = list(levels)
        self.cum = np.concatenate([[0], np.cumsum(levels)]).astype(np.int64)
        self.G = G = int(self.cum[-1])
        self.comp = np.repeat(np.arange(self.K), levels)
        self.cnt = np.concatenate([np.bincount(idx[k], minlength=levels[k]) for k in range(self.K)]).astype(np.float64)
        g = [idx[k].astype(np.int64) + self.cum[k] for k in range(self.K)]
        keys = np.concatenate([g[k] * G + g[l] for k in range(self.K) for l in range(self.K) if k != l])
        u, c = np.unique(keys, return_counts=True)
        self.row, self.col, self.val = u // G, u % G, c.astype(np.float64)
        self.w = np.bincount(self.row, minlength=G)
        self.lower = self.col < self.row
        self.Z = sp.csr_matrix((np.ones(self.K * self.n), (np.tile(np.arange(self.n), self.K), np.concatenate(g))), shape=(self.n, G))

    def at(self, v):
        v = np.asarray(v, dtype=LD)
        d = 1 / v[self.comp] + self.cnt.astype(LD)
        return dict(Mdiag=d, Dinv=1 / d, dis=1 / np.sqrt(d), ld=np.sqrt(d))

    def seg(self, sel, coef, X):
        """per row i: sum over the selected entries (i, j) of coef_e X[j] (entries sorted by row)"""
        Y = np.zeros((self.G, X.shape[1]), dtype=X.dtype)
        r, c = self.row[sel], self.col[sel]
        if r.size == 0:
            return Y
        start = np.flatnonzero(np.r_[True, r[1:] != r[:-1]])
        Y[r[start]] = np.add.reduceat(coef[sel][:, None] * X[c], start, axis=0)
        return Y

    def op(self, which, s, X):
        """0 M X, 2 L D^-1/2 X, 3 D^-1 upper(M) X, 4 (L D^-1/2)^T X"""
        X = np.asarray(X, dtype=LD)
        val = self.val.astype(LD)
        if which == 0:
            return s["Mdiag"][:, None] * X + self.seg(slice(None), val, X)
        if which == 2:
            return s["ld"][:, None] * X + self.seg(self.lower, val * s["dis"][self.col], X)
        if which == 3:
            return s["Dinv"][:, None] * (s["Mdiag"][:, None] * X + self.seg(~self.lower, val, X))
        return s["ld"][:, None] * X + s["dis"][:, None] * self.seg(~self.lower, val, X)

    def precond(self, s, X):
        """P^-1 X = (L D^-1/2)^-T (L D^-1/2)^-1 X: K block steps forward, K backward"""
        X = np.asarray(X, dtype=LD)
        val = self.val.astype(LD)
        W = np.zeros_like(X)
        for k in range(self.K):
            b = slice(self.cum[k], self.cum[k + 1])
            rb = (self.row >= self.cum[k]) & (self.row < self.cum[k + 1])
            W[b] = (X[b] - self.seg(rb & self.lower, val * s["dis"][self.col], W)[b]) / s["ld"][b, None]
        Z = np.zeros_like(X)
        for k in reversed(range(self.K)):
            b = slice(self.cum[k], self.cum[k + 1])
            rb = (self.row >= self.cum[k]) & (self.row < self.cum[k + 1])
            Z[b] = (W[b] - s["dis"][b, None] * self.seg(rb & ~self.lower, val, Z)[b]) / s["ld"][b, None]
        return Z

    def M64(self, v):
        """float64 scipy M for the oracle's SSOR"""
        off = sp.csr_matrix((self.val, (self.row, self.col)), shape=(self.G, self.G))
        return (off + sp.diags(1. / np.asarray(v, dtype=np.float64)[self.comp] + self.cnt)).tocsr()


def sweeps(rows, per_row_threads, sms):
    """grid-stride sweeps of a kernel launched by gm_grid (at most 16 SMs CTAs of 256 threads)"""
    ctas = max(1, min(-(-rows * per_row_threads // 256), sms * 16))
    return -(-rows * per_row_threads // (ctas * 256))


# ---------------------------------------------------------------------------------------------------------------------------
# CPU: the cases reach every edge, and the longdouble reference is the oracle's / the dense M


def test_cases_reach_every_edge():
    assert {(t - 1) // 32 for t in TS} == {0, 1, 2, 3} and {1, 32, 33, 128} <= set(TS)  # every lane group, full and partial
    ks = {k: structure(k) for k in SMALL + ("big",)}
    assert {len(ks[k][1]) for k in SMALL} >= {2, 3, 5, 8}
    assert any(1 in lv for _, lv, _ in ks.values()) and any({256, 257} <= set(lv) for _, lv, _ in ks.values())
    idx, lv, _ = ks["heavy"]
    assert np.bincount(idx[0]).max() == 1 << 18
    idx, lv, _ = ks["nested"]
    assert all(len(set(idx[0][idx[1] == s])) == 1 for s in range(0, 400, 37))
    idx, lv, _ = ks["K5"]
    assert any(idx[k].max() + 1 < lv[k] for k in range(len(lv)))
    idx, lv, _ = ks["big"]
    assert sum(lv) > 40000 and sweeps(sum(lv), 32, H100_SMS) > 1 and sweeps(max(lv), 32, H100_SMS) > 1
    assert sweeps(600003, 1, H100_SMS) > 1 and sweeps(655360, 1, H100_SMS) > 1  # "huge": diag and yaux


@pytest.mark.parametrize("kind", ["K3", "K5", "nested"])
def test_reference_matches_oracle(kind):
    """the block-step longdouble operators against the float64 oracle (dense M where levels are empty)"""
    idx, lv, y = structure(kind)
    r = Ref(idx, lv)
    v = np.array([0.3, 2., 0.7, 1.1, 5.][:r.K])
    M = r.M64(v)
    if kind != "K5":
        st = gm.Structure(idx.T)
        assert st.G == r.G and abs(st.ZtZ).sum() == r.val.sum() + r.cnt.sum()
    pc = gm.SSOR(M)
    X = np.random.default_rng(2).standard_normal((r.G, 5))
    s = r.at(v)
    want = [M @ X, None, pc.LD @ X, pc.Dinv[:, None] * (sp.triu(M, format="csr") @ X)]
    for which in (0, 2, 3):
        got = r.op(which, s, X).astype(np.float64)
        assert np.abs(got - want[which]).max() <= 1e-13 * np.abs(want[which]).max(), which
    Z = r.precond(s, X).astype(np.float64)
    assert np.abs(Z - pc.solve(X)).max() <= 1e-11 * np.abs(Z).max()
    assert np.abs((pc.LDt @ Z) - r.op(4, s, Z).astype(np.float64)).max() <= 1e-12 * np.abs(pc.LDt @ Z).max()
    assert r.Z.sum() == r.K * r.n and np.all(np.diff(r.Z.indptr) == r.K)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU


def _p(a):
    return a.ctypes.data_as(DP)


@pytest.fixture(scope="module")
def lib(product_lib):
    assert product_lib.gpbdev_device_count() > 0, "no CUDA device visible — GPU tests need an H100"
    product_lib.gpbdev_grouped_last_error.restype = C.c_char_p
    return product_lib


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


class Engine:
    def __init__(self, lib, idx, levels, y=None, probes=None):
        self.lib, self.K, self.n = lib, idx.shape[0], idx.shape[1]
        self.G = int(sum(levels))
        lv = np.array(levels, dtype=np.int32)
        self.h = C.c_void_p()
        self.ok(lib.gpbdev_grouped_multi_create(C.byref(self.h), 0, C.c_int64(self.n), self.K, idx.ctypes.data_as(C.POINTER(C.c_int32)),
                                                lv.ctypes.data_as(C.POINTER(C.c_int))))
        if y is not None:
            self.set_y(y)
        if probes is not None:
            self.set_probes(probes)

    def ok(self, rc):
        assert rc == 0, self.lib.gpbdev_grouped_last_error().decode()

    def set_y(self, y):
        self.ok(self.lib.gpbdev_grouped_multi_set_y(self.h, _p(np.ascontiguousarray(y, dtype=np.float64))))

    def set_y_device(self, y):
        import torch
        yt = torch.as_tensor(np.ascontiguousarray(y, dtype=np.float64)).cuda()
        torch.cuda.synchronize()  # the engine's stream does not wait for torch's
        self.ok(self.lib.gpbdev_grouped_multi_set_y_device(self.h, C.cast(C.c_void_p(yt.data_ptr()), DP)))

    def set_probes(self, probes):
        pr = np.asfortranarray(probes, dtype=np.float64)
        self.ok(self.lib.gpbdev_grouped_multi_set_probes(self.h, _p(pr.reshape(-1, order="F")), probes.shape[1]))

    def eval(self, v, cfg=CFG):
        out = np.zeros(5)
        self.ok(self.lib.gpbdev_grouped_multi_eval(self.h, _p(np.asarray(v, dtype=np.float64)), _p(np.asarray(cfg, dtype=np.float64)), _p(out)))
        return out

    def grad(self, sigma2):
        g = np.zeros(self.K)
        self.ok(self.lib.gpbdev_grouped_multi_grad(self.h, C.c_double(sigma2), _p(g)))
        return g

    def apply(self, v, which, X):
        X = np.ascontiguousarray(X, dtype=np.float64)
        Y = np.zeros_like(X)
        self.ok(self.lib.gpbdev_grouped_multi_apply(self.h, _p(np.asarray(v, dtype=np.float64)), which, _p(X), X.shape[1], _p(Y)))
        return Y

    def x(self):
        x = np.zeros(self.G)
        self.ok(self.lib.gpbdev_grouped_multi_apply(self.h, _p(np.ones(self.K)), 4, None, 1, _p(x)))
        return x

    def yaux(self, v, scale, cfg=CFG, device=False):
        its = C.c_int(0)
        if not device:
            out = np.full(self.n, np.nan)
            self.ok(self.lib.gpbdev_grouped_multi_yaux(self.h, _p(np.asarray(v, dtype=np.float64)), _p(np.asarray(cfg, dtype=np.float64)),
                                                       C.c_double(scale), _p(out), 0, C.byref(its)))
            return out, its.value
        import torch
        ot = torch.full((self.n,), float("nan"), dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        self.ok(self.lib.gpbdev_grouped_multi_yaux(self.h, _p(np.asarray(v, dtype=np.float64)), _p(np.asarray(cfg, dtype=np.float64)),
                                                   C.c_double(scale), C.cast(C.c_void_p(ot.data_ptr()), DP), 1, C.byref(its)))
        return ot.cpu().numpy(), its.value

    def __del__(self):
        self.lib.gpbdev_grouped_multi_free(self.h)


def check_operators(e, r, v, t, rng, oracle=False):
    X = rng.standard_normal((r.G, t)) * np.exp(rng.uniform(-2., 2., (r.G, 1)))
    s = r.at(v)
    w = (r.w + 2).astype(LD)[:, None]
    wn = r.w.copy()  # the residual of row i carries the solve errors of the rows it couples to
    np.maximum.at(wn, r.row, r.w[r.col])
    wn = (wn + 2).astype(LD)[:, None]
    for which in (0, 2, 3):
        got = e.apply(v, which, X)
        err = np.abs(got.astype(LD) - r.op(which, s, X))
        bad = err > 4 * EPS * w * r.op(which, s, np.abs(X))
        assert not bad.any(), (which, t, v, np.argwhere(bad)[:5])
    Z = e.apply(v, 1, X)
    res = np.abs(r.op(2, s, r.op(4, s, Z)) - X.astype(LD))
    mag = r.op(2, s, r.op(4, s, np.abs(Z)))
    bad = res > 6 * EPS * wn * mag
    assert not bad.any(), ("P^-1", t, v, np.argwhere(bad)[:5])
    if oracle:
        Zo = gm.SSOR(r.M64(v)).solve(X)
        assert np.abs(Z - Zo).max() <= 1e-12 * np.abs(Zo).max(), (t, v)
    assert np.array_equal(Z, e.apply(v, 1, X))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", SMALL)
def test_operators_against_longdouble_reference(lib, kind):
    idx, lv, y = structure(kind)
    r = Ref(idx, lv)
    e = Engine(lib, idx, lv, y, np.random.default_rng(1).standard_normal((r.G, 128)))
    rng = np.random.default_rng(len(lv))
    for t in TS:
        for v0 in VS:
            v = v0 * np.linspace(0.5, 2., r.K)
            check_operators(e, r, v, t, rng, oracle=v0 <= 1e-2 and t in (1, 33, 128))


@pytest.mark.gpu
@pytest.mark.parametrize("kind,ts", [("big", (1, 33)), ("huge", (1,))])
def test_operators_beyond_one_sweep(lib, sms, kind, ts):
    idx, lv, y = structure(kind)
    r = Ref(idx, lv)
    if kind == "big":
        assert sweeps(r.G, 32, sms) > 1 and sweeps(max(lv), 32, sms) > 1  # spmm, tri_kernel
    else:
        assert sweeps(r.G, 1, sms) > 1 and sweeps(r.n, 1, sms) > 1 and (r.cnt == 0).any()  # diag, yaux; empty rows
    e = Engine(lib, idx, lv, y, np.random.default_rng(1).standard_normal((r.G, max(ts))))
    rng = np.random.default_rng(3)
    for t in ts:
        for v0 in (1e-2, 1e2):
            check_operators(e, r, v0 * np.linspace(0.5, 2., r.K), t, rng)
    # yaux over every observation against y - Z x
    v = np.linspace(0.5, 2., r.K)
    out, _ = e.yaux(v, 0.7)
    check_yaux(e, r, y, out, 0.7)


def check_yaux(e, r, y, out, scale):
    """out = (y - Z x) scale with x read back: eps (K + 2) (|y| + sum_k |x_{idx_k}|) scale"""
    x = e.x()
    cols = r.Z.indices.reshape(r.n, r.K)  # the K levels of every observation (one entry per factor)
    want = (y.astype(LD) - x.astype(LD)[cols].sum(axis=1)) * LD(scale)
    bar = EPS * (r.K + 2) * (np.abs(y) + np.abs(x)[cols].sum(axis=1)) * scale
    bad = np.abs(out.astype(LD) - want) > bar
    assert not bad.any(), np.flatnonzero(bad)[:5]


def oracle_case(kind):
    """structure as oracle/grouped_multi.Structure numbers it (levels by first appearance), response"""
    idx, lv, y = structure(kind)
    st = gm.Structure(idx.T)
    return st, np.ascontiguousarray(np.stack(st.idx).astype(np.int32)), st.levels, y


@pytest.mark.gpu
@pytest.mark.parametrize("kind,t", [("K8", 1), ("K8", 33), ("K8", 128), ("big", 33)])
def test_eval_and_gradient_against_oracle(lib, kind, t):
    st, idx, lv, y = oracle_case(kind)
    r = gm.probes(st, t, 1)
    v = np.linspace(0.3, 1.7, st.K)
    want = gm.evaluate(st, y, v, sigma2=0.8, r=r, with_grad=True)
    e = Engine(lib, idx, lv, y, r)
    out = e.eval(v)
    assert out[2] == want["its"] and out[3] == want["its_tridiag"], (out, want["its"], want["its_tridiag"])
    assert abs(out[0] - want["quad"]) <= 1e-9 * abs(want["quad"])
    assert abs(out[1] - want["logdet"]) <= 1e-9 * abs(want["logdet"])
    assert np.abs(e.x() - want["x"]).max() <= 1e-10 * np.abs(want["x"]).max()
    g = e.grad(0.8)
    assert np.abs(g - want["grad"]).max() <= 1e-7 * np.abs(want["grad"]).max(), (g, want["grad"])
    assert np.array_equal(out, e.eval(v)) and np.array_equal(g, e.grad(0.8))


@pytest.mark.gpu
def test_warm_started_solve_against_oracle(lib):
    """cfg[3] = 1: the second solve starts from the first one's x, as the oracle's cg_vec(..., u0 = x_prev)"""
    st, idx, lv, y = oracle_case("K8")
    e = Engine(lib, idx, lv, y, gm.probes(st, 4, 1))
    warm = (1000, 1000, 1e-2, 1)
    v1 = np.linspace(0.3, 1.7, st.K)
    v2 = v1 * 1.05
    Zty = st.Z.T @ y
    M1 = st.M(v1)
    x1, its1 = gm.cg_vec(M1, gm.SSOR(M1), Zty, None, 1000, 1e-2)
    out1 = e.eval(v1, warm)  # no previous solution: from zero
    assert out1[2] == its1 and np.abs(e.x() - x1).max() <= 1e-10 * np.abs(x1).max()
    M2 = st.M(v2)
    x2, its2 = gm.cg_vec(M2, gm.SSOR(M2), Zty, x1, 1000, 1e-2)
    out2 = e.eval(v2, warm)
    assert out2[2] == its2, (out2[2], its2)
    assert np.abs(e.x() - x2).max() <= 1e-10 * np.abs(x2).max()
    cold, _ = gm.cg_vec(M2, gm.SSOR(M2), Zty, None, 1000, 1e-2)
    assert np.abs(cold - x2).max() > 1e-12 * np.abs(x2).max()  # the warm start is not a no-op
    _, its = e.yaux(v1, 1., warm)
    x3, its3 = gm.cg_vec(M1, gm.SSOR(M1), Zty, x2, 1000, 1e-2)
    assert its == its3 and np.abs(e.x() - x3).max() <= 1e-10 * np.abs(x3).max()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["K3", "K5"])
def test_response_paths_are_bitwise_and_yaux_is_y_minus_zx(lib, kind):
    idx, lv, y = structure(kind)
    r = Ref(idx, lv)
    probes = np.random.default_rng(4).standard_normal((r.G, 9))
    a, b = Engine(lib, idx, lv, y, probes), Engine(lib, idx, lv, None, probes)
    b.set_y_device(y)
    v = np.linspace(0.4, 2.5, r.K)
    out = a.eval(v)
    assert np.array_equal(out, b.eval(v)) and np.array_equal(a.grad(1.3), b.grad(1.3))
    host, its_h = a.yaux(v, 0.6)
    dev, its_d = a.yaux(v, 0.6, device=True)
    assert its_h == its_d and np.array_equal(host, dev)
    assert np.array_equal(host, a.yaux(v, 0.6)[0])
    check_yaux(a, r, y, host, 0.6)


@pytest.mark.gpu
def test_probe_count_grows_and_shrinks(lib):
    """set_probes 7 -> 128 -> 3 reallocates the work blocks once and keeps them; each evaluation equals the oracle, and the last one
    a fresh engine's with the same 3 probes bit for bit"""
    st, idx, lv, y = oracle_case("K3")
    v = np.array([0.5, 1.5, 0.9])
    e = Engine(lib, idx, lv, y)
    for t in (7, 128, 3):
        pr = gm.probes(st, t, t)
        e.set_probes(pr)
        out = e.eval(v)
        want = gm.evaluate(st, y, v, r=pr)
        assert out[2] == want["its"] and out[3] == want["its_tridiag"], (t, out)
        assert abs(out[0] - want["quad"]) <= 1e-9 * abs(want["quad"]) and abs(out[1] - want["logdet"]) <= 1e-9 * abs(want["logdet"])
    f = Engine(lib, idx, lv, y, pr)
    assert np.array_equal(out, f.eval(v)) and np.array_equal(e.grad(1.), f.grad(1.))


@pytest.mark.gpu
@pytest.mark.parametrize("l1", [1e-120, 0.])
def test_zero_right_hand_side(lib, l1):
    """|Z^T y|_1 below 1e-100: the reference returns x = 0 without an iteration, so y_aux = y scale exactly"""
    st, idx, lv, y0 = oracle_case("K2")
    y = y0 * (l1 / np.abs(st.Z.T @ y0).sum())
    assert np.abs(st.Z.T @ y).sum() < 1e-100 and (l1 == 0 or (st.Z.T @ y) @ (st.Z.T @ y) > 0)
    v = np.array([0.7, 1.3])
    x, its = gm.cg_vec(st.M(v), gm.SSOR(st.M(v)), st.Z.T @ y, None, 1000, 1e-2)
    assert its == 0 and not x.any()
    e = Engine(lib, idx, lv, y, gm.probes(st, 5, 1))
    out = e.eval(v)
    assert out[2] == 0 and not e.x().any() and abs(out[0] - y @ y) <= 1e-12 * (y @ y)
    ya, its = e.yaux(v, 0.25)
    assert its == 0 and np.array_equal(ya, y * 0.25)
