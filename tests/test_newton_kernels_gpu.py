"""The Newton leaf system of GPBoost with a Vecchia GP (gpbdev_vecchia_newton_system, gpboost_b200/csrc/dev/newton.cuh) against
an extended-precision reference, at the edges of its tiling.

newton_gram_kernel    grid (nchunks, npairs): CTA (chunk, pair) owns one 64 x 64 tile pair (ta, tb), ta >= tb, of the lower block
                      triangle of H^T B^T D^-1 B H, decoded from blockIdx.y; npairs = 1 / 3 / 6 / 10 for L <= 64 / 128 / 192 / 256.
                      Rows come in batches of 8, one per warp; the warp's lanes load the row's neighbours (lane < m, m <= 32), lane 0
                      builds the row of B H restricted to the two tiles, then every thread adds the batch's 8 weighted outer products.
                      nchunks = min(ceil(n / 256), max(1, 2 SMs / npairs)), rows_per_chunk = ceil(n / nchunks)
newton_reduce_kernel  M[a][b] = sum of the chunk partials of the lower-triangle entry, chunk order
newton_leafsum_*      rhs[l] = sum of g over the rows of leaf l: 4 SMs chunks, then a chunk-order sum

Cases: L in {1, 2, 63, 64, 65, 127, 128, 129, 192, 193, 255, 256} reaches every tile-pair count and every partial last tile;
m in {1, 10, 31, 32} (at 32 every lane of the neighbour load is live); engines with n <= m (every row padded, neighbour sets
supplied); n in {5, 257, 4000, 100 000}, which leave a partial 8-row batch at the end of a chunk, and n = 10^6 at L = 256 (ten
tile pairs, chunk count capped by the pair count). Leaf assignments: uniform, spatial strips (neighbours mostly share a leaf, so
the +1 and -A terms cancel), all rows on leaves 63 and 64 (the off-diagonal tile pair (1, 0) carries the mass), leaves of one row
each, and a leaf id without rows.

Reference: the rows of B H from the factor read back from the device (which isolates these kernels from the factor kernel):
+1 at leaf(perm[i]), -A[i, k] at leaf(perm[nn[i, k]]), -1 padding skipped. M_ref = sum_i D^-1_i r_i r_i^T and rhs_ref = H^T g are
accumulated in np.longdouble (np.add.at over the (m + 1)^2 slot pairs). At n = 10^6 the reference is the float64 scipy product
and the bar below is doubled.

Bars and why:
- |M - M_ref|_ab <= 4 eps (m + 2 + rows_per_chunk + nchunks) (|BH|^T D^-1 |BH|)_ab: each entry of a row of B H is a chain of up
  to m + 1 additions, the chunk adds its rows one after another, and the chunks are added in order; every addition of a chain of
  length c carries at most c eps relative to the sum of magnitudes, and the product D^-1 r_a r_b two more roundings;
- |rhs - rhs_ref|_l <= 4 eps (rows of a leaf-sum chunk + 4 SMs) sum_{i in l} |g_i|, for the same reason;
- a leaf without rows has an exactly zero row and column of M and an exactly zero rhs entry (no term ever touches them);
- M exactly symmetric (one partial serves both triangles) and a second call bitwise equal (every sum has a fixed order);
- through the Booster (fixed covariance parameters, leaves_newton_update): the new tree's leaf values equal the learning rate times
  the solve of the restated system (H^T Psi^-1 H)^-1 H^T Psi^-1 (y - F) with the factor of oracle/vecchia.py, 1e-8 relative (the
  bar of test_tree_gpu.py) or 1e-10 cond(H^T Psi^-1 H) where that is larger: the oracle's factor and the device's agree to the
  1e-10 of the Vecchia kernel tests, and leaves of a few rows make the system ill-conditioned (cond about 3e3 to 7e3 here);
- refusals (num_leaves 0 and 257, m = 33, no stored factor, a row-sharded engine) name the limit and leave the engine usable; a
  Booster with num_leaves = 300 and Newton updates is refused before it changes its scores."""
import ctypes as C
import math

import numpy as np
import pytest
import scipy.sparse as sp

import datagen
import ensemble_walk
from oracle import vecchia as ov

LD = np.longdouble
EPS = np.finfo(np.float64).eps
MODE_STORE = 1
TILE = 64
H100_SMS = 132
LS = (1, 2, 63, 64, 65, 127, 128, 129, 192, 193, 255, 256)
MS = (1, 10, 31, 32)
NS = (5, 257, 4000, 100000)
ASSIGN = ("uniform", "spatial", "tiles", "singletons", "empty")
# at n = 100 000 the longdouble reference costs seconds per call: a subset that still reaches 1, 3 and 10 tile pairs
BIG_N_LS = (63, 127, 256)
BIG_N_MS = (10, 32)


def P(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


def npairs(L):
    nt = (L + TILE - 1) // TILE
    return nt * (nt + 1) // 2


def chunking(n, L, sms):
    """(nchunks, rows_per_chunk) of the Gram kernel and (lchunks, rows per leaf-sum chunk), as gpbdev_vecchia_newton_system"""
    nchunks = min((n + 255) // 256, max(1, sms * 2 // npairs(L)))
    lchunks = 4 * sms
    return nchunks, -(-n // nchunks), lchunks, -(-n // lchunks)


def leaves(kind, L, n, coords, seed):
    """leaf of every row (original order), int32"""
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        return rng.integers(0, L, n).astype(np.int32)
    if kind == "spatial":  # strips along x: a row and its nearest earlier neighbours mostly share a leaf
        rank = np.empty(n, dtype=np.int64)
        rank[np.argsort(coords[:, 0], kind="stable")] = np.arange(n)
        return (rank * L // n).astype(np.int32)
    if kind == "tiles":  # leaves 63 and 64 only (tile pair (1, 0)); below 65 leaves the last two
        lo = 63 if L >= 65 else max(L - 2, 0)
        return (lo + rng.integers(0, min(2, L), n)).astype(np.int32)
    if kind == "singletons":  # leaves 0 .. L-2 hold one row each (as far as the rows go), the rest is on L-1
        leaf = np.full(n, L - 1, dtype=np.int32)
        k = min(L - 1, n)
        leaf[rng.permutation(n)[:k]] = np.arange(k, dtype=np.int32)
        return leaf
    assert kind == "empty"  # uniform over every leaf but L // 2 (for L = 1 the only leaf keeps its rows)
    if L == 1:
        return np.zeros(n, dtype=np.int32)
    leaf = rng.integers(0, L - 1, n).astype(np.int32)
    leaf[leaf >= L // 2] += 1
    return leaf


def slots(nn, A, perm, leaf):
    """columns (n, m + 1; -1 = padding) and coefficients of the rows of B H in Vecchia order"""
    n = nn.shape[0]
    cols = np.full((n, nn.shape[1] + 1), -1, dtype=np.int64)
    coef = np.zeros(cols.shape)
    cols[:, 0] = leaf[perm]
    coef[:, 0] = 1.
    live = nn >= 0
    cols[:, 1:][live] = leaf[perm[nn[live]]]
    coef[:, 1:][live] = -A[live]
    return cols, coef


def reference(nn, A, Dinv, perm, leaf, g, L):
    """M_ref, |BH|^T D^-1 |BH| (the bar's magnitude), rhs_ref, sum_{i in l} |g_i|: longdouble, vectorised over slot pairs"""
    cols, coef = slots(nn, A, perm, leaf)
    live = cols >= 0
    c = np.where(live, cols, 0)
    w = coef.astype(LD) * np.sqrt(Dinv.astype(LD))[:, None]
    wa = np.abs(coef) * np.sqrt(Dinv)[:, None]
    M = np.zeros(L * L, dtype=LD)
    Ma = np.zeros(L * L)  # a magnitude for the bar: float64 is plenty
    for s in range(cols.shape[1]):
        rows = live[:, s]
        if not rows.any():
            continue
        idx = c[rows, s:s + 1] * L + c[rows]
        msk = live[rows]
        np.add.at(M, idx[msk], (w[rows, s:s + 1] * w[rows])[msk])
        Ma += np.bincount(idx[msk], (wa[rows, s:s + 1] * wa[rows])[msk], L * L)
    rhs = np.zeros(L, dtype=LD)
    rhsa = np.zeros(L, dtype=LD)
    np.add.at(rhs, leaf, g.astype(LD))
    np.add.at(rhsa, leaf, np.abs(g).astype(LD))
    return M.reshape(L, L), Ma.reshape(L, L), rhs, rhsa


def reference_f64(nn, A, Dinv, perm, leaf, g, L):
    """the same in float64 through scipy (n = 10^6)"""
    cols, coef = slots(nn, A, perm, leaf)
    live = cols >= 0
    n = nn.shape[0]
    rows = np.repeat(np.arange(n), cols.shape[1]).reshape(cols.shape)
    BH = sp.csr_matrix((coef[live], (rows[live], cols[live])), shape=(n, L))
    BHa = sp.csr_matrix((np.abs(coef[live]), (rows[live], cols[live])), shape=(n, L))  # built from |A|, before duplicates add
    D = sp.diags(Dinv)
    M = (BH.T @ D @ BH).toarray()
    Ma = (BHa.T @ D @ BHa).toarray()
    return M, Ma, np.bincount(leaf, g, L), np.bincount(leaf, np.abs(g), L)


def cases():
    out = []
    for n in NS:
        for m in MS:
            if n >= 100000 and m not in BIG_N_MS:
                continue
            out.append((n, m))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# CPU: the cases reach every edge, and the longdouble reference is the dense product


def test_cases_reach_every_edge():
    """every tile-pair count with a full and a partial last tile, L = 1 and 64 exactly, m = 32, an engine with n <= m, a partial
    8-row batch at the end of a chunk, and the n = 10^6 case with its chunk count capped by the pair count (132 SMs of an H100)"""
    assert {npairs(L) for L in LS} == {1, 3, 6, 10}
    for p in (1, 3, 6, 10):
        tails = {L % TILE for L in LS if npairs(L) == p}
        assert 0 in tails and tails - {0}, (p, tails)
    assert 1 in LS and 64 in LS and 32 in MS
    assert any(n <= m for n, m in cases())
    partial = [(n, L) for n, _ in cases() for L in LS if chunking(n, L, H100_SMS)[1] % 8 and n > 8]
    assert partial
    nc, _, _, _ = chunking(10 ** 6, 256, H100_SMS)
    assert npairs(256) == 10 and nc == H100_SMS * 2 // 10 < (10 ** 6 + 255) // 256
    assert {npairs(L) for L in BIG_N_LS} >= {1, 3, 10} and 32 in BIG_N_MS
    # every assignment is a valid leaf vector; "tiles" touches the off-diagonal pair, "empty" leaves one leaf without rows
    coords = np.random.default_rng(0).random((300, 2))
    for kind in ASSIGN:
        for L in LS:
            lf = leaves(kind, L, 300, coords, 1)
            assert lf.min() >= 0 and lf.max() < L
    assert set(leaves("tiles", 129, 300, coords, 1)) == {63, 64}
    assert np.bincount(leaves("empty", 129, 300, coords, 1), minlength=129)[64] == 0
    assert (np.bincount(leaves("singletons", 129, 300, coords, 1), minlength=129)[:128] == 1).all()


def test_reference_is_the_dense_product():
    """the slot-pair longdouble accumulation against a dense B H built row by row (padding, repeated leaves, a leaf without rows)"""
    rng = np.random.default_rng(3)
    n, m, L = 40, 5, 7
    perm = rng.permutation(n).astype(np.int32)
    nn = np.full((n, m), -1, dtype=np.int32)
    for i in range(1, n):
        k = min(i, m)
        nn[i, :k] = rng.choice(i, k, replace=False)
    A = rng.standard_normal((n, m))
    Dinv = rng.random(n) + 0.5
    leaf = rng.integers(0, L - 1, n).astype(np.int32)  # leaf L-1 has no rows
    g = rng.standard_normal(n)
    BH = np.zeros((n, L))
    for i in range(n):
        BH[i, leaf[perm[i]]] += 1.
        for k in range(m):
            if nn[i, k] >= 0:
                BH[i, leaf[perm[nn[i, k]]]] -= A[i, k]
    want = BH.T @ (Dinv[:, None] * BH)
    M, Ma, rhs, rhsa = reference(nn, A, Dinv, perm, leaf, g, L)
    assert np.abs(M.astype(np.float64) - want).max() <= 1e-13 * np.abs(want).max()
    assert np.all(Ma * (1 + 1e-15) >= np.abs(M.astype(np.float64))) and np.all(Ma[L - 1] == 0) and rhs[L - 1] == 0
    assert np.allclose(rhs.astype(np.float64), [g[leaf == l].sum() for l in range(L)], rtol=0, atol=1e-14)
    M64, Ma64, rhs64, _ = reference_f64(nn, A, Dinv, perm, leaf, g, L)
    assert np.abs(M64 - want).max() <= 1e-13 * np.abs(want).max() and np.allclose(Ma64, Ma, rtol=1e-14)
    assert np.allclose(rhs64, rhs.astype(np.float64), rtol=0, atol=1e-14)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU


@pytest.fixture(scope="module")
def lib(product_lib):
    assert product_lib.gpbdev_device_count() > 0, "no CUDA device visible — GPU tests need an H100"
    return product_lib


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def chk(lib, rc):
    assert rc == 0, lib.gpbdev_last_error().decode()


def make_engine(lib, n, m, seed, row_range=None, store=True, nn_in=None):
    """engine on n synthetic points with the factor stored (matern 1.5); returns h, perm, nn, A, Dinv, coords.
    n <= m: every row padded, neighbour sets (all earlier rows) supplied"""
    coords, y = datagen.synth(n, 2, 11 + seed)
    perm = ov.random_order(n, seed)
    co = np.ascontiguousarray(coords[perm])
    if nn_in is None and n <= m:
        nn_in = np.full((n, m), -1, dtype=np.int32)
        for i in range(n):
            nn_in[i, :i] = np.arange(i)[::-1]
    r0, r1 = row_range or (0, n)
    h = C.c_void_p()
    nn_c = None if nn_in is None else P(np.ascontiguousarray(nn_in, dtype=np.int32), C.c_int32)
    chk(lib, lib.gpbdev_vecchia_create(C.byref(h), 0, C.c_int64(n), 2, m, P(co), P(perm, C.c_int32), nn_c, C.c_int64(r0), C.c_int64(r1)))
    chk(lib, lib.gpbdev_vecchia_set_y(h, P(np.ascontiguousarray(y, dtype=np.float64))))
    if not store:
        return h, perm, None, None, None, coords
    rho = 2. * n ** -0.5
    sums = np.zeros(9)
    chk(lib, lib.gpbdev_vecchia_eval(h, 1, C.c_double(1.3), C.c_double(math.sqrt(3.) / rho), MODE_STORE, P(sums)))
    nn = np.empty((n, m), dtype=np.int32)
    chk(lib, lib.gpbdev_vecchia_get_nn(h, P(nn, C.c_int32)))
    A = np.empty((n, m)); Dinv = np.empty(n)
    chk(lib, lib.gpbdev_vecchia_get_factor(h, P(A), P(Dinv)))
    if nn_in is not None:
        assert np.array_equal(nn, nn_in)
    return h, perm, nn, A, Dinv, coords


def newton_call(lib, h, leaf, L, g):
    """(rc, M, rhs) of one gpbdev_vecchia_newton_system call with the leaf ids and the gradient as CUDA tensors"""
    import torch
    lt = torch.as_tensor(np.ascontiguousarray(leaf, dtype=np.int32)).cuda()
    gt = torch.as_tensor(np.ascontiguousarray(g, dtype=np.float64)).cuda()
    torch.cuda.synchronize()  # the engine's stream does not wait for torch's
    M = np.full((max(L, 1), max(L, 1)), np.nan)
    rhs = np.full(max(L, 1), np.nan)
    rc = lib.gpbdev_vecchia_newton_system(h, C.c_void_p(lt.data_ptr()), L, C.c_void_p(gt.data_ptr()), P(M), P(rhs))
    return rc, M, rhs


def check_system(lib, h, nn, A, Dinv, perm, leaf, g, L, sms, f64=False):
    n, m = nn.shape
    rc, M, rhs = newton_call(lib, h, leaf, L, g)
    chk(lib, rc)
    Mr, Ma, rr, ra = (reference_f64 if f64 else reference)(nn, A, Dinv, perm, leaf, g, L)
    nchunks, rpc, lchunks, lrpc = chunking(n, L, sms)
    k = 2. if f64 else 1.
    err = np.abs(M.astype(LD) - Mr)
    bar = k * 4 * EPS * (m + 2 + rpc + nchunks) * Ma
    bad = err > bar
    assert not bad.any(), ("M", L, m, n, np.argwhere(bad)[:5], M[bad][:5], Mr[bad][:5])
    err = np.abs(rhs.astype(LD) - rr)
    bad = err > k * 4 * EPS * (lrpc + lchunks) * ra
    assert not bad.any(), ("rhs", L, np.flatnonzero(bad)[:5], rhs[bad][:5], rr[bad][:5])
    assert np.array_equal(M, M.T)
    empty = np.bincount(leaf, minlength=L) == 0
    assert np.all(M[empty] == 0) and np.all(M[:, empty] == 0) and np.all(rhs[empty] == 0)
    rc, M2, rhs2 = newton_call(lib, h, leaf, L, g)
    chk(lib, rc)
    assert np.array_equal(M, M2) and np.array_equal(rhs, rhs2)
    return M


@pytest.mark.gpu
@pytest.mark.parametrize("n,m", cases(), ids=["n%d-m%d" % c for c in cases()])
def test_newton_system_against_longdouble_reference(lib, sms, n, m):
    h, perm, nn, A, Dinv, coords = make_engine(lib, n, m, seed=m + n % 97)
    try:
        rng = np.random.default_rng(n + m)
        g = rng.standard_normal(n) * np.exp(rng.uniform(-3., 3., n))
        tiles_hit = False
        for L in (BIG_N_LS if n >= 100000 else LS):
            for kind in (ASSIGN if n < 100000 else ("uniform",) if m == 32 else ("uniform", "tiles")):
                leaf = leaves(kind, L, n, coords, seed=L)
                M = check_system(lib, h, nn, A, Dinv, perm, leaf, g, L, sms)
                if kind == "tiles" and L >= 65 and n > 8:
                    assert M[64, 63] != 0  # the off-diagonal tile pair (1, 0) carries the mass
                    tiles_hit = True
        assert tiles_hit or n <= 8 or (n >= 100000 and m == 32)
    finally:
        lib.gpbdev_vecchia_free(h)


@pytest.mark.gpu
def test_newton_system_at_one_million_rows(lib, sms):
    """L = 256 (ten tile pairs), chunk count 2 SMs / 10 < ceil(n / 256): float64 scipy reference, doubled bar"""
    n, m, L = 10 ** 6, 10, 256
    assert chunking(n, L, sms)[0] == max(1, 2 * sms // 10) < (n + 255) // 256
    h, perm, nn, A, Dinv, coords = make_engine(lib, n, m, seed=5)
    try:
        rng = np.random.default_rng(8)
        g = rng.standard_normal(n)
        for kind in ("uniform", "spatial"):
            check_system(lib, h, nn, A, Dinv, perm, leaves(kind, L, n, coords, seed=3), g, L, sms, f64=True)
    finally:
        lib.gpbdev_vecchia_free(h)


@pytest.mark.gpu
def test_refusals_leave_the_engine_usable(lib, sms):
    n = 500
    err = lambda: lib.gpbdev_last_error().decode()
    h, perm, nn, A, Dinv, coords = make_engine(lib, n, 10, seed=2)
    try:
        leaf = leaves("uniform", 100, n, coords, 1)
        g = np.random.default_rng(1).standard_normal(n)
        for bad_L in (0, 257):
            rc, _, _ = newton_call(lib, h, leaf if bad_L else leaf * 0, bad_L, g)
            assert rc != 0 and "num_leaves must be in [1, 256]" in err()
        check_system(lib, h, nn, A, Dinv, perm, leaf, g, 100, sms)
    finally:
        lib.gpbdev_vecchia_free(h)
    # m = 33: the neighbour load has 32 lanes
    h, perm, nn, A, Dinv, coords = make_engine(lib, n, 33, seed=3)
    try:
        rc, _, _ = newton_call(lib, h, np.zeros(n, dtype=np.int32), 4, np.ones(n))
        assert rc != 0 and "num_neighbors must be <= 32" in err()
        out = np.zeros(9)
        chk(lib, lib.gpbdev_vecchia_eval(h, 1, C.c_double(1.3), C.c_double(20.), MODE_STORE, P(out)))
        assert np.isfinite(out).all()
    finally:
        lib.gpbdev_vecchia_free(h)
    # before any STORE pass: refused, then usable once the factor is stored
    h, perm, _, _, _, coords = make_engine(lib, n, 10, seed=4, store=False)
    try:
        rc, _, _ = newton_call(lib, h, np.zeros(n, dtype=np.int32), 4, np.ones(n))
        assert rc != 0 and "the factor is not resident" in err()
        sums = np.zeros(9)
        chk(lib, lib.gpbdev_vecchia_eval(h, 1, C.c_double(1.3), C.c_double(math.sqrt(3.) / (2. * n ** -0.5)), MODE_STORE, P(sums)))
        nn = np.empty((n, 10), dtype=np.int32)
        chk(lib, lib.gpbdev_vecchia_get_nn(h, P(nn, C.c_int32)))
        A = np.empty((n, 10)); Dinv = np.empty(n)
        chk(lib, lib.gpbdev_vecchia_get_factor(h, P(A), P(Dinv)))
        check_system(lib, h, nn, A, Dinv, perm, leaves("uniform", 65, n, coords, 2), np.ones(n), 65, sms)
    finally:
        lib.gpbdev_vecchia_free(h)
    # a row-sharded engine (rows [0, n / 2))
    h, _, _, _, _, _ = make_engine(lib, n, 10, seed=6, row_range=(0, n // 2))
    try:
        rc, _, _ = newton_call(lib, h, np.zeros(n, dtype=np.int32), 4, np.ones(n))
        assert rc != 0 and "row-sharded" in err()
        sums = np.zeros(9)
        chk(lib, lib.gpbdev_vecchia_eval(h, 1, C.c_double(1.3), C.c_double(20.), MODE_STORE, P(sums)))
        assert np.isfinite(sums).all()
    finally:
        lib.gpbdev_vecchia_free(h)


# ---------------------------------------------------------------------------------------------------------------------------
# through the Booster

BOOST_N, BOOST_M, BOOST_COV = 6000, 10, [0.1, 0.4, 0.1]


def boost_data():
    rng = np.random.default_rng(21)
    X = rng.random((BOOST_N, 4))
    coords = rng.random((BOOST_N, 2))
    y = 2 * np.sin(3 * X[:, 0]) + X[:, 1] ** 2 + 0.5 * (X[:, 2] > 0.6) + np.sin(5 * coords[:, 0]) * np.cos(4 * coords[:, 1])
    return X, y + 0.3 * rng.standard_normal(BOOST_N), coords


def booster(num_leaves):
    from gpboost_b200 import GPModel
    from gpboost_b200.booster import Booster, Dataset
    X, y, coords = boost_data()
    params = {"objective": "regression", "num_leaves": num_leaves, "min_data_in_leaf": 5, "learning_rate": 0.1, "max_bin": 255,
              "verbose": -1, "train_gp_model_cov_pars": False, "leaves_newton_update": True}
    gp = GPModel(gp_coords=coords, cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia", num_neighbors=BOOST_M,
                 vecchia_ordering="random", seed=1)
    gp.set_optim_params({"init_cov_pars": np.array(BOOST_COV)})
    return Booster(params, Dataset(X, y, params=params), gp_model=gp), X, y, coords


@pytest.mark.gpu
@pytest.mark.parametrize("num_leaves", [64, 65, 200])
def test_booster_newton_leaf_values_against_restated_system(lib, num_leaves):
    """the second tree (the first carries BoostFromAverage's bias): leaf values = 0.1 (H^T Psi^-1 H)^-1 H^T Psi^-1 (y - F)"""
    from gpboost_b200.booster import parse_model_string
    b, X, y, coords = booster(num_leaves)
    b.update()
    F = b.inner_predict_train()
    b.update()
    tree = parse_model_string(b.model_to_string())[1]
    nl = tree["num_leaves"]
    assert nl > min(num_leaves - 1, 128), nl  # the tree reaches the tile edge the budget is chosen for
    leaf = ensemble_walk.leaf_of_rows(tree, X)
    vo = ov.VecchiaOracle(coords, BOOST_M, "matern", 1.5, "random", 1)
    _, pt = ov.transform_cov_pars(BOOST_COV, "matern", 1.5)
    A, Dinv, _, _, _ = ov.factor(vo.coords, vo.nn, vo.cid, pt)
    n = BOOST_N
    live = vo.nn >= 0
    rows = np.repeat(np.arange(n), vo.nn.shape[1]).reshape(vo.nn.shape)
    B = sp.eye(n, format="csr") - sp.csr_matrix((A[live], (rows[live], vo.nn[live])), shape=(n, n))
    H = sp.csr_matrix((np.ones(n), (np.arange(n), leaf[vo.perm])), shape=(n, nl))
    BH = B @ H
    Mr = (BH.T @ sp.diags(Dinv) @ BH).toarray()
    rhs = BH.T @ (Dinv * (B @ (y - F)[vo.perm]))
    want = 0.1 * np.linalg.solve(Mr, rhs)
    got = tree["leaf_value"]
    # the device's factor agrees with the oracle's to the 1e-10 of the Vecchia kernel tests; the solve amplifies that by cond(M)
    bar = max(1e-8, 1e-10 * np.linalg.cond(Mr)) * np.abs(want).max()
    assert np.abs(got - want).max() <= bar, (np.abs(got - want).max(), np.abs(want).max(), np.linalg.cond(Mr))
    assert abs(tree["shrinkage"] - 0.1) <= 1e-12


@pytest.mark.gpu
def test_booster_refuses_more_than_256_leaves(lib):
    """num_leaves = 300 with Newton updates: a GPBoostError that names the limit, before the scores change"""
    from gpboost_b200.basic import GPBoostError
    b, _, _, _ = booster(300)
    before = b.inner_predict_train().copy()
    for _ in range(2):
        with pytest.raises(GPBoostError, match="at most 256 leaves"):
            b.update()
        assert b.current_iteration() == 0
        assert np.array_equal(b.inner_predict_train(), before)
